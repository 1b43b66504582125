"""f6 video frames: the numpy restatement of the YUV 4:2:0 -> BGR conversion the letter-box and alignment kernels fuse
(retinaface_b200/csrc/yuv.cuh).  Test infrastructure -- see ``oracle/__init__.py``.

BT.601 is OpenCV's COLOR_YUV2BGR_{NV12,NV21,I420,YV12} (nearest chroma, 20-bit fixed point, bit-equal to cv2.cvtColor).  BT.709
has no OpenCV counterpart: the same formula with round(c * 2^20) of the limited-range BT.709 matrix is its definition.  The
letter-box of a frame is then ``inputs.letterbox_bgr_u8(frame_to_bgr(...))`` and a crop ``align.warp_affine_fixed`` of it.
"""
from __future__ import annotations

import numpy as np

SHIFT = 20
# (CY, CUB, CUG, CVG, CVR)
BT601 = (1220542, 2116026, -409993, -852492, 1673527)      # OpenCV's ITUR_BT_601_* constants
BT709 = (1220945, 2215014, -223607, -558796, 1879825)
MATRICES = {"bt601": BT601, "bt709": BT709}
LAYOUTS = ("nv12", "nv21", "i420", "yv12")


def limited_range_coefficients(kr: float, kb: float):
    """round(c * 2^20) of the limited-range matrix with luma weights kr, kb (luma scale 255/219, chroma 255/224)."""
    kg = 1.0 - kr - kb
    cy, cc = 255.0 / 219.0, 255.0 / 224.0
    c = (cy, cc * 2 * (1 - kb), -cc * 2 * (1 - kb) * kb / kg, -cc * 2 * (1 - kr) * kr / kg, cc * 2 * (1 - kr))
    return tuple(int(round(v * (1 << SHIFT))) for v in c)


def yuv_to_bgr_samples(y, u, v, matrix: str = "bt601") -> np.ndarray:
    """Per-sample conversion of equally shaped Y, U, V arrays -> (..., 3) u8 BGR."""
    cy, cub, cug, cvg, cvr = MATRICES[matrix]
    y = np.maximum(np.asarray(y, np.int64) - 16, 0) * cy + (1 << (SHIFT - 1))
    u = np.asarray(u, np.int64) - 128
    v = np.asarray(v, np.int64) - 128
    bgr = [(y + cub * u) >> SHIFT, (y + cvg * v + cug * u) >> SHIFT, (y + cvr * v) >> SHIFT]
    return np.clip(np.stack(bgr, axis=-1), 0, 255).astype(np.uint8)


def float_bgr(y, u, v, kr: float, kb: float) -> np.ndarray:
    """The limited-range matrix evaluated in float64 (luma below 16 taken as 16, as the integer formula does), rounded half up and
    clamped: what the integer BT.709 formula approximates."""
    kg = 1.0 - kr - kb
    yy = (255.0 / 219.0) * np.maximum(np.asarray(y, np.float64) - 16, 0)
    cu = (255.0 / 224.0) * (np.asarray(u, np.float64) - 128)
    cv = (255.0 / 224.0) * (np.asarray(v, np.float64) - 128)
    r = yy + 2 * (1 - kr) * cv
    b = yy + 2 * (1 - kb) * cu
    g = yy - 2 * (1 - kb) * kb / kg * cu - 2 * (1 - kr) * kr / kg * cv
    return np.clip(np.floor(np.stack([b, g, r], axis=-1) + 0.5), 0, 255).astype(np.uint8)


def split_planes(buf: np.ndarray, layout: str):
    """OpenCV's single-buffer frame ((h * 3 / 2, w) u8) -> (Y (h, w), U (h/2, w/2), V (h/2, w/2))."""
    rows, w = buf.shape
    h = rows * 2 // 3
    y = buf[:h]
    if layout in ("nv12", "nv21"):
        c = buf[h:].reshape(h // 2, w // 2, 2)
        u, v = (c[..., 0], c[..., 1]) if layout == "nv12" else (c[..., 1], c[..., 0])
        return y, u, v
    flat = buf[h:].reshape(-1)
    q = (h // 2) * (w // 2)
    a, b = flat[:q].reshape(h // 2, w // 2), flat[q:].reshape(h // 2, w // 2)
    return (y, a, b) if layout == "i420" else (y, b, a)


def planes_to_bgr(y, u, v, matrix: str = "bt601") -> np.ndarray:
    """Nearest chroma: every 2 x 2 luma block takes its one (U, V) sample."""
    up = np.repeat(np.repeat(u, 2, axis=0), 2, axis=1)
    vp = np.repeat(np.repeat(v, 2, axis=0), 2, axis=1)
    return yuv_to_bgr_samples(y, up, vp, matrix)


def frame_to_bgr(buf: np.ndarray, layout: str, matrix: str = "bt601") -> np.ndarray:
    return planes_to_bgr(*split_planes(buf, layout), matrix)


def bgr_to_frame(bgr: np.ndarray, layout: str) -> np.ndarray:
    """A (h * 3 / 2, w) frame in `layout` from an even-sized BGR image via cv2.cvtColor(COLOR_BGR2YUV_I420) (test inputs)."""
    import cv2
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    if layout == "i420":
        return i420
    y, u, v = split_planes(i420, "i420")
    h, w = y.shape
    if layout == "yv12":
        return np.concatenate([y.reshape(-1), v.reshape(-1), u.reshape(-1)]).reshape(h * 3 // 2, w)
    first, second = (u, v) if layout == "nv12" else (v, u)
    return np.concatenate([y, np.stack([first, second], axis=-1).reshape(h // 2, w)])
