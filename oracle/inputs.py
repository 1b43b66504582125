"""Input preparation restating the reference's OpenCV preprocess branch, plus the seeded
synthetic inputs of SURVEY.md section 8d.  Test infrastructure -- see ``oracle/__init__.py``.
"""
from __future__ import annotations

import numpy as np


def letterbox_bgr_u8(img: np.ndarray, net_h: int, net_w: int) -> np.ndarray:
    """retinaface/RetinaFace.cpp:587-624 (non-NPP branch): isotropic shrink by
    1/max(cols/W, rows/H, 1) with cv::resize (INTER_LINEAR default), then zero-pad bottom /
    right to net_h x net_w (copyMakeBorder BORDER_CONSTANT 0).  Never up-scales."""
    import cv2
    rows, cols = img.shape[:2]
    sw = np.float32(1.0 * cols / net_w)
    sh = np.float32(1.0 * rows / net_h)
    scale = sw if sw > sh else sh
    scale = scale if scale > 1.0 else np.float32(1.0)
    if scale > 1:
        f = float(np.float32(1) / scale)
        res = cv2.resize(img, None, fx=f, fy=f)
    else:
        res = img
    out = np.zeros((net_h, net_w, 3), dtype=np.uint8)
    h = min(res.shape[0], net_h)
    w = min(res.shape[1], net_w)
    out[:h, :w] = res[:h, :w]
    return out


def s_real_batch(base: np.ndarray, batch: int) -> np.ndarray:
    """S-real (SURVEY.md 8d): element i = np.roll(base, 8*i, axis=1): same faces, distinct content."""
    return np.stack([np.roll(base, 8 * i, axis=1) for i in range(batch)])


def s_noise_batch(batch: int, net_h: int, net_w: int, seed: int = 0) -> np.ndarray:
    """S-noise (SURVEY.md 8d): uniform random u8, ~0 detections."""
    return np.random.default_rng(seed).integers(0, 256, (batch, net_h, net_w, 3), dtype=np.uint8)


def mixed_batch(photo: np.ndarray, n: int, net_h: int, net_w: int, start: int = 0) -> np.ndarray:
    """Neighbours as dissimilar as possible (the letter-boxed photo, noise, all-255, all-0, a rolled copy, a mirrored copy,
    other noise, an upside-down copy, cycled from `start`): a tile that reads the wrong image or a stale buffer changes
    bytes, and no two of any 8 consecutive images are the same."""
    inp = letterbox_bgr_u8(photo, net_h, net_w)
    noise = s_noise_batch(2, net_h, net_w, seed=21)
    pool = [inp, noise[0], np.full((net_h, net_w, 3), 255, np.uint8), np.zeros((net_h, net_w, 3), np.uint8),
            np.roll(inp, 37, axis=1), np.ascontiguousarray(inp[:, ::-1]), noise[1], np.ascontiguousarray(inp[::-1])]
    return np.stack([pool[(start + i) % len(pool)] for i in range(n)])
