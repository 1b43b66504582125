"""f12 redaction restated in numpy and Python doubles (rf_b200.h rf_redact_yuv_device): the regions of a frame, their snapped
geometry, and the in-place mosaic of every plane, byte for byte what the GPU writes.

Regions: the frame's records j < min(count, max_faces) in rank order, each coordinate float32(x) * float32(scale) rounded to float
(__fmul_rn), then with tracks every RF_TRACK_LOST track in list order, box (kx1, ky1, kx2, ky2).  A box with a non-finite coordinate or
w <= 0 or h <= 0 is skipped.  Geometry in FP64, one rounding per step (Python floats):
    w = x2 - x1, h = y2 - y1, mx = margin * w, my = margin * h
    X0 = floor(max(x1 - mx, -65536)), X1 = floor(min(x2 + mx, 65536)) + 1, Y likewise; X0 = 2 floor(X0 / 2), X1 = 2 ceil(X1 / 2)
    C = 2 ceil(max(X1 - X0, Y1 - Y0) / (2 blocks))        (2 for a rectangle that is empty on both axes)
Cells are C x C squares from (X0, Y0); chroma planes use the rectangle and C halved.  A cell's value is (sum + cnt // 2) // cnt of the
ORIGINAL samples of the cell inside the plane; a sample covered by some region's rectangle takes its cell value in the lowest-index
region covering it; every other byte stays.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import numpy as np

RF_TRACK_LOST = 2
DEFAULT_BLOCKS, DEFAULT_MARGIN = 8, 0.25

Region = Tuple[int, int, int, int, int]      # X0, Y0, X1, Y1 (half-open, unclamped, even), C


def params(blocks: int = 0, margin: float = 0.0) -> Tuple[int, float]:
    """rf_redact_params with the defaults applied; margin as the float32 the C struct holds, widened."""
    return blocks or DEFAULT_BLOCKS, float(np.float32(margin or DEFAULT_MARGIN))


def geometry(x1, y1, x2, y2, margin: float, blocks: int) -> Optional[Region]:
    """The snapped rectangle and cell side of one box in frame pixels (floats), or None when the box is skipped."""
    x1, y1, x2, y2 = (float(np.float32(v)) for v in (x1, y1, x2, y2))
    if not all(math.isfinite(v) for v in (x1, y1, x2, y2)):
        return None
    w, h = x2 - x1, y2 - y1
    if not (w > 0 and h > 0):
        return None
    mx, my = margin * w, margin * h
    X0, X1 = math.floor(max(x1 - mx, -65536.0)), math.floor(min(x2 + mx, 65536.0)) + 1
    Y0, Y1 = math.floor(max(y1 - my, -65536.0)), math.floor(min(y2 + my, 65536.0)) + 1
    X0, Y0, X1, Y1 = 2 * (X0 // 2), 2 * (Y0 // 2), 2 * (-(-X1 // 2)), 2 * (-(-Y1 // 2))
    D = max(X1 - X0, Y1 - Y0)
    C = 2 * (-(-D // (2 * blocks))) if D > 0 else 2
    return X0, Y0, X1, Y1, C


def frame_regions(faces: np.ndarray, count: int, scale: Optional[float], margin: float, blocks: int, tracks=None,
                  max_faces: Optional[int] = None) -> List[Region]:
    """Frame i's regions in index order.  faces: (k, >= 5) float32 records (score, x1, y1, x2, y2, ...) in the network-input
    pixels the device call returned (scale None: already frame pixels); tracks: TRACK_DTYPE records of the frame's list, or None."""
    faces = np.asarray(faces, np.float32)
    k = min(int(count), faces.shape[0] if max_faces is None else max_faces)
    s = np.float32(1.0 if scale is None else scale)
    out = []
    for j in range(k):
        g = geometry(*(np.float32(faces[j, c]) * s for c in (1, 2, 3, 4)), margin, blocks)
        if g is not None:
            out.append(g)
    for t in (tracks if tracks is not None else ()):
        if int(t["state"]) == RF_TRACK_LOST:
            g = geometry(t["kx1"], t["ky1"], t["kx2"], t["ky2"], margin, blocks)
            if g is not None:
                out.append(g)
    return out


def _mosaic(orig: np.ndarray, x0: int, y0: int, x1: int, y1: int, c: int):
    """((rows, cols) slices, u8 fill) of one region on one plane of shape (h, w[, 3]), or None when it misses the plane."""
    h, w = orig.shape[:2]
    cx0, cx1, cy0, cy1 = max(x0, 0), min(x1, w), max(y0, 0), min(y1, h)
    if cx0 >= cx1 or cy0 >= cy1:
        return None
    sub = orig[cy0:cy1, cx0:cx1].astype(np.int64)
    colcell = (np.arange(cx0, cx1) - x0) // c
    rowcell = (np.arange(cy0, cy1) - y0) // c
    cstart = np.flatnonzero(np.r_[True, colcell[1:] != colcell[:-1]])
    rstart = np.flatnonzero(np.r_[True, rowcell[1:] != rowcell[:-1]])
    sums = np.add.reduceat(np.add.reduceat(sub, rstart, axis=0), cstart, axis=1)
    cnt = np.diff(np.r_[rstart, rowcell.size])[:, None] * np.diff(np.r_[cstart, colcell.size])[None, :]
    if sub.ndim == 3:
        cnt = cnt[..., None]
    mean = (sums + cnt // 2) // cnt
    fill = mean[rowcell - rowcell[0]][:, colcell - colcell[0]].astype(np.uint8)
    return (slice(cy0, cy1), slice(cx0, cx1)), fill


def redact_planes(planes: Sequence[Tuple[np.ndarray, int]], regions: Sequence[Region]) -> None:
    """Writes the mosaic into each (view, sub) in place: sub 1 for a luma or (h, w, 3) BGR plane, 2 for a chroma plane (rectangles
    and cell side halved).  Views may be strided (an NV12 chroma component, a pitched surface's rows)."""
    for view, sub in planes:
        orig = view.copy()
        for x0, y0, x1, y1, c in reversed(list(regions)):     # the lowest index is written last and wins
            m = _mosaic(orig, x0 // sub, y0 // sub, x1 // sub, y1 // sub, c // sub)
            if m is not None:
                view[m[0]] = m[1]


def yuv_planes(buf: np.ndarray, layout: str, width: int, height: int, y_pitch: Optional[int] = None, uv_offset: Optional[int] = None,
               uv_pitch: Optional[int] = None):
    """Writable (view, sub) planes of a frame held in one flat u8 buffer: OpenCV's single buffer by default, or a pitched surface
    (NVDEC: luma rows y_pitch apart, chroma at byte uv_offset, rows uv_pitch apart)."""
    flat = buf.reshape(-1)
    yp = y_pitch or width
    semi = layout in ("nv12", "nv21")
    cp = uv_pitch or (width if semi else width // 2)
    off = uv_offset if uv_offset is not None else yp * height
    y = flat[:yp * height].reshape(height, yp)[:, :width]
    ch = height // 2
    if semi:
        c = flat[off:off + cp * ch].reshape(ch, cp)[:, :width].reshape(ch, width // 2, 2)
        u, v = (c[..., 0], c[..., 1]) if layout == "nv12" else (c[..., 1], c[..., 0])
    else:
        a = flat[off:off + cp * ch].reshape(ch, cp)[:, :width // 2]
        b = flat[off + cp * ch:off + 2 * cp * ch].reshape(ch, cp)[:, :width // 2]
        u, v = (a, b) if layout == "i420" else (b, a)
    return [(y, 1), (u, 2), (v, 2)]


def redact_yuv(buf: np.ndarray, layout: str, regions: Sequence[Region], **surface) -> np.ndarray:
    """A redacted copy of one YUV 4:2:0 frame buffer (shape kept).  surface: yuv_planes' pitched-surface keywords, with width and
    height; without them buf is OpenCV's (h * 3 / 2, w) single buffer."""
    out = np.array(buf, np.uint8, copy=True)
    if "width" not in surface:
        surface = dict(width=buf.shape[1], height=buf.shape[0] * 2 // 3)
    redact_planes(yuv_planes(out, layout, **surface), regions)
    return out


def redact_bgr(img: np.ndarray, regions: Sequence[Region]) -> np.ndarray:
    """A redacted copy of one (h, w, 3) u8 BGR image."""
    out = np.array(img, np.uint8, copy=True)
    redact_planes([(out, 1)], regions)
    return out
