"""The letter-box kernel's own definition, restated in numpy (retinaface_b200/csrc/preprocess.cu): the geometry of both resize
branches, OpenCV's fixed-point bilinear taps, OpenCV's 2x area rule, NPP's coverage-weighted super-sampling and the EXIF
reflections / transposition, each in the kernel's operation order and precision (preprocess.cu is built with -fmad=false, so every
multiply and add rounds on its own).  Vectorised over the output.  Test infrastructure -- see ``oracle/__init__.py``.

``letterbox(img, box_w, box_h)`` is what k_letterbox_batch / k_letterbox_transposed write for one item: the resized displayed
image at the top left of a net_h x net_w canvas, zeros elsewhere.  It is checked against cv2 on the CPU
(tests/test_letterbox_cpu.py) and the kernels against it on the GPU (tests/test_gpu_letterbox_edges.py).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32

LB_FLIP_X, LB_FLIP_Y, LB_TRANSPOSE = 1, 2, 4
# EXIF orientation 1..8 -> LB_* bits (preprocess.cuh lb_orientation_bits)
ORIENTATION_BITS = {1: 0, 2: LB_FLIP_X, 3: LB_FLIP_X | LB_FLIP_Y, 4: LB_FLIP_Y, 5: LB_TRANSPOSE, 6: LB_TRANSPOSE | LB_FLIP_X,
                    7: LB_TRANSPOSE | LB_FLIP_X | LB_FLIP_Y, 8: LB_TRANSPOSE | LB_FLIP_Y}


def geometry(w: int, h: int, box_w: int, box_h: int):
    """letterbox_geometry: (dw, dh, scale) of OpenCV's branch.  sc = max(w / box_w, h / box_h, 1) in float, f = (double)(1 / sc),
    the resized size rounded half to even (saturate_cast<int>), clamped to the box; scale = 1 / f, the source pixels per output
    pixel.  A side that rounds to 0 (1 x 5000 into 448 x 448) leaves an empty resized image: the letter-box is all zero."""
    sw, sh = F32(1.0 * w / box_w), F32(1.0 * h / box_h)
    sc = sw if sw > sh else sh
    sc = sc if sc > F32(1) else F32(1)
    if sc > F32(1):
        f = float(F32(1) / sc)
        dw, dh, scale = int(np.rint(w * f)), int(np.rint(h * f)), 1.0 / f
    else:
        dw, dh, scale = w, h, 1.0
    return min(dw, box_w), min(dh, box_h), scale


def geometry_npp(w: int, h: int, box_w: int, box_h: int):
    """letterbox_geometry_npp (RF_FLAG_NPP_RESIZE): f = min(box_w / w, box_h / h) in double, never above 1; extent ceil(w f - 1e-9)."""
    f = min(box_w / w, box_h / h)
    if f >= 1.0:
        return min(w, box_w), min(h, box_h), 1.0
    return min(int(np.ceil(w * f - 1e-9)), box_w), min(int(np.ceil(h * f - 1e-9)), box_h), 1.0 / f


def displayed(img: np.ndarray, bits: int = 0) -> np.ndarray:
    """The image as the taps see it: stored pixel (x', y') for displayed (x, y), x' = FLIP_X ? sw-1-x : x, y' = FLIP_Y ? sh-1-y : y,
    read at stored column y', row x' under TRANSPOSE."""
    d = img.transpose(1, 0, 2) if bits & LB_TRANSPOSE else img
    if bits & LB_FLIP_X:
        d = d[:, ::-1]
    if bits & LB_FLIP_Y:
        d = d[::-1]
    return d


def tap_of(d: np.ndarray, sn: int, scale: float, horizontal: bool):
    """OpenCV's INTER_LINEAR coefficient of destination coordinates d: (s0, s1, a0, a1).  The source position in double, rounded to
    float; horizontal taps zero the fraction at the borders, vertical ones only clamp the source rows; weights rounded to 11 bits."""
    fx = ((np.asarray(d, np.float64) + 0.5) * scale - 0.5).astype(F32)
    s = np.floor(fx).astype(np.int64)
    fx = (fx - s.astype(F32)).astype(F32)
    if horizontal:
        lo = s < 0
        fx[lo], s[lo] = F32(0), 0
        hi = s >= sn - 1
        fx[hi], s[hi] = F32(0), sn - 1
    a0 = np.rint((F32(1) - fx) * F32(2048)).astype(np.int64)
    a1 = np.rint(fx * F32(2048)).astype(np.int64)
    return np.clip(s, 0, sn - 1), np.clip(s + 1, 0, sn - 1), a0, a1


def linear(src: np.ndarray, dw: int, dh: int, scale: float) -> np.ndarray:
    """linear_pixel over the dh x dw resized image of the displayed source: HResizeLinear in int, then VResizeLinear's
    ((a0 * (h0 >> 4)) >> 16) + ((a1 * (h1 >> 4)) >> 16) + 2 >> 2."""
    sh, sw = src.shape[:2]
    xs0, xs1, xa0, xa1 = tap_of(np.arange(dw), sw, scale, True)
    ys0, ys1, ya0, ya1 = tap_of(np.arange(dh), sh, scale, False)
    def p(ys, xs):
        return src[ys[:, None], xs[None, :]].astype(np.int64)
    xa0, xa1 = xa0[None, :, None], xa1[None, :, None]
    h0 = p(ys0, xs0) * xa0 + p(ys0, xs1) * xa1
    h1 = p(ys1, xs0) * xa0 + p(ys1, xs1) * xa1
    v = (((ya0[:, None, None] * (h0 >> 4)) >> 16) + ((ya1[:, None, None] * (h1 >> 4)) >> 16) + 2) >> 2
    return np.clip(v, 0, 255).astype(np.uint8)


def half(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """half_pixel: cv::resize's INTER_LINEAR at exactly 2x, OpenCV's fast area code.  The mean of source block [2x, 2x + 2) x
    [2y, 2y + 2): (sum + 2) >> 2 for a whole block; the sum over the pixels a block cut by the far edge has, divided in float and
    rounded half to even."""
    sh, sw = src.shape[:2]
    acc = np.zeros((dh, dw, 3), np.int64)
    cnt = np.zeros((dh, dw, 1), np.int64)
    for ky in (0, 1):
        for kx in (0, 1):
            ny, nx = max(0, min(dh, (sh - ky + 1) // 2)), max(0, min(dw, (sw - kx + 1) // 2))   # blocks that have this pixel
            acc[:ny, :nx] += src[ky:2 * ny:2, kx:2 * nx:2]
            cnt[:ny, :nx] += 1
    part = np.rint(acc.astype(F32) / np.maximum(cnt, 1).astype(F32)).astype(np.int64)
    return np.where(cnt == 4, (acc + 2) >> 2, part).astype(np.uint8)


def area(src: np.ndarray, dw: int, dh: int, scale: float) -> np.ndarray:
    """area_pixel (RF_FLAG_NPP_RESIZE): the coverage-weighted sum over source rectangle [x s, (x + 1) s) x [y s, (y + 1) s) in
    double, rows outer and columns inner as the kernel loops, samples beyond the image absent (weight lost, not renormalised), times
    1 / s^2, rounded half up."""
    sh, sw = src.shape[:2]

    def span(n, side):
        d = np.arange(n)
        a, b = d * scale, (d + 1) * scale
        return a, b, np.floor(a).astype(np.int64), np.minimum(np.ceil(b - 1e-12).astype(np.int64), side)
    ax, bx, x0, x1 = span(dw, sw)
    ay, by, y0, y1 = span(dh, sh)
    acc = np.zeros((dh, dw, 3), np.float64)
    for ky in range(int((y1 - y0).max(initial=0))):
        sy = y0 + ky
        rows = np.minimum(sy, sh - 1)
        wy = np.minimum(sy + 1.0, by) - np.maximum(sy.astype(np.float64), ay)
        for kx in range(int((x1 - x0).max(initial=0))):
            sx = x0 + kx
            wx = np.minimum(sx + 1.0, bx) - np.maximum(sx.astype(np.float64), ax)
            w = wy[:, None] * wx[None, :]
            term = w[..., None] * src[rows[:, None], np.minimum(sx, sw - 1)[None, :]].astype(np.float64)
            ok = (sy < y1)[:, None, None] & (sx < x1)[None, :, None]
            acc = np.where(ok, acc + term, acc)
    norm = 1.0 / (scale * scale)
    return np.clip(np.floor(acc * norm + 0.5), 0, 255).astype(np.uint8)


def resized(img: np.ndarray, dw: int, dh: int, scale: float, bits: int = 0, npp: bool = False, half_area: bool = True) -> np.ndarray:
    """lb_pixel over the whole dh x dw resized image of displayed(img, bits): the identity copy at scale 1, OpenCV's 2x area rule at
    scale 2 (half_area=False: the bilinear taps there instead, as the letter-box computed before it took OpenCV's branch), NPP's
    super-sampling with npp, OpenCV's bilinear taps otherwise."""
    src = displayed(img, bits)
    if dw <= 0 or dh <= 0:
        return np.zeros((max(dh, 0), max(dw, 0), 3), np.uint8)
    if scale == 1.0:
        return np.ascontiguousarray(src[:dh, :dw])
    if npp:
        return area(src, dw, dh, scale)
    if half_area and scale == 2.0:
        return half(src, dw, dh)
    return linear(src, dw, dh, scale)


def letterbox(img: np.ndarray, net_w: int, net_h: int, box=None, bits: int = 0, npp: bool = False, half_area: bool = True) -> np.ndarray:
    """letterbox_fill + k_letterbox_batch of one item: img (u8 BGR HWC, as stored) shown with LB_* `bits`, letter-boxed into `box`
    ((box_w, box_h), default the network) at the top left of a net_h x net_w canvas of zeros."""
    bw, bh = box or (net_w, net_h)
    h, w = img.shape[:2]
    if bits & LB_TRANSPOSE:
        w, h = h, w
    dw, dh, scale = (geometry_npp if npp else geometry)(w, h, bw, bh)
    out = np.zeros((net_h, net_w, 3), np.uint8)
    out[:max(dh, 0), :max(dw, 0)] = resized(img, dw, dh, scale, bits, npp, half_area)
    return out
