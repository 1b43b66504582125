"""f14 redaction styles restated in numpy and Python ints (rf_b200.h rf_redact_style), on top of oracle/redact.py's f12 regions and
mosaic: byte for byte what the GPU writes for every style.

The regions, their order, the snapped rectangles and "original" are f12's (oracle/redact.py frame_regions).  A shape -- RECT: the
rectangle; ELLIPSE: the samples whose centres lie in the inscribed ellipse, u^2 H^2 + v^2 W^2 <= W^2 H^2 in exact integers; chroma on
the halved rectangle -- and a kind -- MOSAIC: f12's cells and cell values; BLUR: a triple-box blur of radius
a = clamp(ceil(max(W, H) / (2 detail)), 1, 127) (chroma (a + 1) >> 1) with replicate borders inside the plane, rounded
(S + (n^6 - 1) / 2) // n^6.  A sample takes its value from the lowest-index region whose SHAPE covers it; every other byte stays.
"""
from __future__ import annotations

from typing import NamedTuple, Sequence, Tuple

import numpy as np

from oracle.redact import DEFAULT_BLOCKS, Region, _mosaic, yuv_planes

MOSAIC, BLUR = 1, 2
RECT, ELLIPSE = 1, 2
DEFAULT_DETAIL, MAX_RADIUS = 4, 127


class Style(NamedTuple):
    """rf_redact_style with the defaults applied (blocks only for MOSAIC, detail only for BLUR)."""
    kind: int = MOSAIC
    shape: int = RECT
    blocks: int = DEFAULT_BLOCKS
    detail: int = 0


def style(kind: int = 0, shape: int = 0, blocks: int = 0, detail: int = 0) -> Style:
    """rf_redact_style's defaults: kind 0 -> BLUR, shape 0 -> ELLIPSE, blocks 0 -> 8 (mosaic), detail 0 -> 4 (blur)."""
    kind, shape = kind or BLUR, shape or ELLIPSE
    if kind == MOSAIC:
        return Style(MOSAIC, shape, blocks or DEFAULT_BLOCKS, 0)
    return Style(BLUR, shape, 0, detail or DEFAULT_DETAIL)


def blur_radius(region: Region, detail: int) -> int:
    """The luma / BGR radius a of a region: clamp(ceil(max(W, H) / (2 detail)), 1, 127)."""
    X0, Y0, X1, Y1 = region[:4]
    D = max(X1 - X0, Y1 - Y0)
    return min(max(-(-D // (2 * detail)), 1), MAX_RADIUS)


def kernel(a: int) -> np.ndarray:
    """k = box * box * box, box of width 2a + 1: 6a + 1 int64 taps summing to (2a + 1)^3."""
    box = np.ones(2 * a + 1, np.int64)
    return np.convolve(np.convolve(box, box), box)


def ellipse_mask(x0: int, y0: int, x1: int, y1: int, w: int, h: int) -> np.ndarray:
    """(h, w) bool: the samples (x, y) of a w x h plane whose centres lie in the ellipse inscribed in [x0, x1) x [y0, y1), exactly:
    u^2 H^2 + v^2 W^2 <= W^2 H^2 with u = 2x + 1 - x0 - x1, v = 2y + 1 - y0 - y1.  Per row the bound W^2 H^2 - v^2 W^2 is a Python
    int, and u^2 H^2 <= R is u^2 <= R // H^2 (H^2 > 0), which int64 holds for every u of the plane."""
    m = np.zeros((h, w), bool)
    W, H = x1 - x0, y1 - y0
    if W <= 0 or H <= 0:
        return m
    cx0, cx1, cy0, cy1 = max(x0, 0), min(x1, w), max(y0, 0), min(y1, h)
    if cx0 >= cx1 or cy0 >= cy1:
        return m
    u = 2 * np.arange(cx0, cx1, dtype=np.int64) + 1 - x0 - x1
    for y in range(cy0, cy1):
        v = 2 * y + 1 - y0 - y1
        R = W * W * H * H - v * v * W * W
        if R >= 0:
            m[y, cx0:cx1] = u * u <= R // (H * H)
    return m


def shape_mask(x0: int, y0: int, x1: int, y1: int, w: int, h: int, shape: int) -> np.ndarray:
    """(h, w) bool: the samples of a w x h plane a region's shape covers."""
    if shape == ELLIPSE:
        return ellipse_mask(x0, y0, x1, y1, w, h)
    m = np.zeros((h, w), bool)
    m[max(y0, 0):max(min(y1, h), 0), max(x0, 0):max(min(x1, w), 0)] = True
    return m


def _boxes3(x: np.ndarray, a: int, axis: int) -> np.ndarray:
    """Three un-normalised boxes of width 2a + 1 along axis (length L -> L - 6a), by cumulative sums in uint64: every difference is
    exact modulo 2^64 and every result is below 2^63."""
    n = 2 * a + 1
    for _ in range(3):
        c = np.cumsum(x, axis=axis, dtype=np.uint64)
        c = np.concatenate([np.zeros_like(np.take(c, [0], axis=axis)), c], axis=axis)
        L = c.shape[axis]
        x = np.take(c, np.arange(n, L), axis=axis) - np.take(c, np.arange(0, L - n), axis=axis)
    return x


def blur_plane(orig: np.ndarray, region: Tuple[int, int, int, int], a: int, direct: bool = False):
    """((rows, cols) slices, u8 values) of the blur of radius a over [x0, x1) x [y0, y1) clipped to the plane orig (h, w[, 3]), or
    None when it misses the plane: S = sum_ij k[i] k[j] P[clampY(y + j)][clampX(x + i)] (np.pad mode "edge" by 3a), rounded
    (S + (n^6 - 1) / 2) // n^6.  direct: the literal correlation with k in int64 (slow; for checking the cumulative sums)."""
    h, w = orig.shape[:2]
    x0, y0, x1, y1 = region
    cx0, cx1, cy0, cy1 = max(x0, 0), min(x1, w), max(y0, 0), min(y1, h)
    if cx0 >= cx1 or cy0 >= cy1:
        return None
    r = 3 * a
    rows = np.clip(np.arange(cy0 - r, cy1 + r), 0, h - 1)
    cols = np.clip(np.arange(cx0 - r, cx1 + r), 0, w - 1)
    win = orig[rows][:, cols].astype(np.int64)          # the plane padded by edge replication, cut to the taps' reach
    n6 = (2 * a + 1) ** 6
    if direct:
        k = kernel(a)
        hs = sum(k[i] * win[:, i:i + cx1 - cx0] for i in range(6 * a + 1))
        S = sum(k[j] * hs[j:j + cy1 - cy0] for j in range(6 * a + 1))
        return (slice(cy0, cy1), slice(cx0, cx1)), ((S + (n6 - 1) // 2) // n6).astype(np.uint8)
    S = _boxes3(_boxes3(win, a, 1), a, 0)
    return (slice(cy0, cy1), slice(cx0, cx1)), ((S + np.uint64((n6 - 1) // 2)) // np.uint64(n6)).astype(np.uint8)


def redact_planes(planes: Sequence[Tuple[np.ndarray, int]], regions: Sequence[Region], st: Style) -> None:
    """Writes the styled redaction into each (view, sub) in place, as oracle/redact.py redact_planes: sub 1 for a luma or (h, w, 3) BGR
    plane, 2 for a chroma plane (rectangles and cell side halved, blur radius (a + 1) >> 1).  MOSAIC uses the regions' cell side C."""
    for view, sub in planes:
        orig = view.copy()
        h, w = orig.shape[:2]
        for x0, y0, x1, y1, c in reversed(list(regions)):     # the lowest index is written last and wins
            rect = (x0 // sub, y0 // sub, x1 // sub, y1 // sub)
            if st.kind == MOSAIC:
                m = _mosaic(orig, *rect, c // sub)
            else:
                a = blur_radius((x0, y0, x1, y1), st.detail)
                m = blur_plane(orig, rect, a if sub == 1 else (a + 1) >> 1)
            if m is None:
                continue
            cover = shape_mask(*rect, w, h, st.shape)[m[0]]
            view[m[0]][cover] = m[1][cover]


def redact_yuv(buf: np.ndarray, layout: str, regions: Sequence[Region], st: Style, **surface) -> np.ndarray:
    """A styled, redacted copy of one YUV 4:2:0 frame buffer, as oracle/redact.py redact_yuv (surface: its pitched-surface keywords)."""
    out = np.array(buf, np.uint8, copy=True)
    if "width" not in surface:
        surface = dict(width=buf.shape[1], height=buf.shape[0] * 2 // 3)
    redact_planes(yuv_planes(out, layout, **surface), regions, st)
    return out


def redact_bgr(img: np.ndarray, regions: Sequence[Region], st: Style) -> np.ndarray:
    """A styled, redacted copy of one (h, w, 3) u8 BGR image."""
    out = np.array(img, np.uint8, copy=True)
    redact_planes([(out, 1)], regions, st)
    return out
