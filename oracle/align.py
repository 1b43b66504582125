"""Face-alignment oracle (test infrastructure): the five-landmark similarity transform and the crop warp of
``rf_detect_align_batch``, restated in numpy.

* ``umeyama``            -- least-squares similarity by the SVD form of Umeyama (1991), the way
                            ``skimage.transform.SimilarityTransform.estimate`` computes it (insightface's ``norm_crop`` uses it).
* ``similarity_closed``  -- the centred closed form the kernel evaluates in FP64 (same minimiser).
* ``invert_affine``      -- ``cv::invertAffineTransform`` for double matrices.
* ``warp_affine_fixed``  -- ``cv2.warpAffine(img, M, (cw, ch), INTER_LINEAR, BORDER_CONSTANT, 0)`` on u8 images, restated in
                            OpenCV's fixed point: coordinates in 1/1024 then 1/32 pixel, integer bilinear weights summing to
                            32768, taps outside the image contribute 0.
* ``blob``               -- ``cv2.dnn.blobFromImages(crops, 1/std, size, (mean,) * 3, swapRB=True)`` of u8 BGR crops.
"""
from __future__ import annotations

import numpy as np

# ArcFace 112 x 112 template (insightface ``arcface_dst``): left eye, right eye, nose, left and right mouth corner.
ARCFACE_112 = np.array([[38.2946, 51.6963], [73.5318, 51.5014], [56.0252, 71.7366], [41.5493, 92.3655], [70.7299, 92.2041]],
                       dtype=np.float32)


def umeyama(src: np.ndarray, dst: np.ndarray) -> np.ndarray:
    """2 x 3 similarity (rotation, uniform scale, translation) minimising sum |M [src; 1] - dst|^2 (SVD form)."""
    src = np.asarray(src, dtype=np.float64)
    dst = np.asarray(dst, dtype=np.float64)
    num, dim = src.shape
    src_mean, dst_mean = src.mean(axis=0), dst.mean(axis=0)
    src_d, dst_d = src - src_mean, dst - dst_mean
    A = dst_d.T @ src_d / num
    d = np.ones(dim)
    if np.linalg.det(A) < 0:
        d[dim - 1] = -1
    T = np.eye(dim + 1)
    U, S, V = np.linalg.svd(A)
    rank = np.linalg.matrix_rank(A)
    if rank == 0:
        return np.zeros((2, 3))
    if rank == dim - 1:
        if np.linalg.det(U) * np.linalg.det(V) > 0:
            T[:dim, :dim] = U @ V
        else:
            s = d[dim - 1]
            d[dim - 1] = -1
            T[:dim, :dim] = U @ np.diag(d) @ V
            d[dim - 1] = s
    else:
        T[:dim, :dim] = U @ np.diag(d) @ V
    scale = 1.0 / src_d.var(axis=0).sum() * (S @ d)
    T[:dim, dim] = dst_mean - scale * (T[:dim, :dim] @ src_mean.T)
    T[:dim, :dim] *= scale
    return T[:2]


def similarity_closed(p: np.ndarray, q: np.ndarray) -> np.ndarray:
    """The kernel's closed form, in its order of operations: a = sum(p~ . q~) / sum |p~|^2,
    b = sum(p~x q~y - p~y q~x) / sum |p~|^2, M = [[a, -b, tx], [b, a, ty]].  All zeros when the landmarks coincide."""
    p = np.asarray(p, dtype=np.float64)
    q = np.asarray(q, dtype=np.float64)
    pmx = sum(float(v) for v in p[:, 0]) / 5.0
    pmy = sum(float(v) for v in p[:, 1]) / 5.0
    qmx = sum(float(v) for v in q[:, 0]) / 5.0
    qmy = sum(float(v) for v in q[:, 1]) / 5.0
    den = sxx = sxy = 0.0
    for k in range(5):
        ux, uy = float(p[k, 0]) - pmx, float(p[k, 1]) - pmy
        vx, vy = float(q[k, 0]) - qmx, float(q[k, 1]) - qmy
        den += ux * ux + uy * uy
        sxx += ux * vx + uy * vy
        sxy += ux * vy - uy * vx
    if den == 0.0:
        return np.zeros((2, 3))
    a, b = sxx / den, sxy / den
    return np.array([[a, -b, qmx - a * pmx + b * pmy], [b, a, qmy - b * pmx - a * pmy]])


def invert_affine(M: np.ndarray) -> np.ndarray:
    """cv::invertAffineTransform (double): D = M00 M11 - M01 M10 -> 1/D (0 when D = 0)."""
    m = np.asarray(M, dtype=np.float64).reshape(6)
    D = m[0] * m[4] - m[1] * m[3]
    D = 1.0 / D if D != 0 else 0.0
    a11, a22, a12, a21 = m[4] * D, m[0] * D, -m[1] * D, -m[3] * D
    b1 = -a11 * m[2] - a12 * m[5]
    b2 = -a21 * m[2] - a22 * m[5]
    return np.array([[a11, a12, b1], [a21, a22, b2]])


def warp_affine_fixed(img: np.ndarray, M: np.ndarray, size) -> np.ndarray:
    """cv2.warpAffine(img, M, size = (cw, ch), INTER_LINEAR, BORDER_CONSTANT, 0) for u8 H x W x 3 images, bit for bit."""
    cw, ch = size
    iM = invert_affine(M)
    h, w = img.shape[:2]
    x = np.arange(cw, dtype=np.float64)
    y = np.arange(ch, dtype=np.float64)
    adelta = np.rint(iM[0, 0] * x * 1024).astype(np.int64)
    bdelta = np.rint(iM[1, 0] * x * 1024).astype(np.int64)
    X0 = np.rint((iM[0, 1] * y + iM[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((iM[1, 1] * y + iM[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    src = img.astype(np.int64)
    acc = np.zeros((ch, cw, 3), dtype=np.int64)
    for dy, dx, wgt in ((0, 0, 32 * (32 - fx) * (32 - fy)), (0, 1, 32 * fx * (32 - fy)), (1, 0, 32 * (32 - fx) * fy), (1, 1, 32 * fx * fy)):
        tx, ty = sx + dx, sy + dy
        inside = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
        v = src[np.clip(ty, 0, h - 1), np.clip(tx, 0, w - 1)] * inside[..., None]
        acc += v * wgt[..., None]
    return ((acc + 16384) >> 15).astype(np.uint8)


def blob(crops_bgr: np.ndarray, mean: float = 127.5, std: float = 127.5) -> np.ndarray:
    """N x 3 x ch x cw float32, RGB planes, (u8 - mean) * (1 / std) in float32 (blobFromImages' arithmetic)."""
    x = np.asarray(crops_bgr)[..., ::-1].transpose(0, 3, 1, 2).astype(np.float32)
    return (x - np.float32(mean)) * np.float32(1.0 / std)
