"""f23 rotated views restated in Python (rf_b200.h rf_rotated_view): the angle reduction, the quarter turns' EXIF orientation, a warp
view's fit f and matrix M (the same libm cos / sin, the same operation order, so M is comparable bit for bit), its network input by
cv2.warpAffine, and the map-back of a warp view's records through cv::invertAffineTransform(M).  Test infrastructure -- see
``oracle/__init__.py``."""
from __future__ import annotations

import math

import numpy as np

from oracle.align import invert_affine

QUARTER = {0.0: 1, 90.0: 8, 180.0: 3, 270.0: 6}     # counter-clockwise quarter turn -> EXIF orientation of rf_detect_views_oriented


def reduce_angle(angle) -> float:
    """fmod(angle, 360) of the float32 angle, plus 360 when negative; a whole turn is 0."""
    a = math.fmod(float(np.float32(angle)), 360.0)
    if a < 0.0:
        a += 360.0
    return 0.0 if a == 360.0 else a


def shrink_box(net_w: int, net_h: int, shrink: float):
    """rf_detect_views' box: max(1, (int)(net * shrink)) with the product in float32."""
    s = np.float32(shrink)
    return max(1, int(np.float32(net_w) * s)), max(1, int(np.float32(net_h) * s))


def geometry(angle, w: int, h: int, box_w: int, box_h: int):
    """(orientation, f, M): a quarter turn's EXIF orientation with f = None, M = None; or 0, f and the 2 x 3 float64 M of a warp view."""
    a = reduce_angle(angle)
    if a in QUARTER:
        return QUARTER[a], None, None
    r = a * (math.pi / 180.0)
    c, s = math.cos(r), math.sin(r)
    W, H = float(w), float(h)
    wr, hr = abs(c) * W + abs(s) * H, abs(s) * W + abs(c) * H
    f = 1.0
    f = min(f, box_w / wr)
    f = min(f, box_h / hr)
    m00, m01, m10, m11 = f * c, f * s, -(f * s), f * c
    cx, cy = (W - 1.0) / 2.0, (H - 1.0) / 2.0
    tx = (f * wr - 1.0) / 2.0 - (m00 * cx + m01 * cy)
    ty = (f * hr - 1.0) / 2.0 - (m10 * cx + m11 * cy)
    return 0, f, np.array([[m00, m01, tx], [m10, m11, ty]])


def warp_view(img: np.ndarray, M: np.ndarray, net_w: int, net_h: int) -> np.ndarray:
    """The network input of a warp view: cv2.warpAffine(img, M, (net_w, net_h), INTER_LINEAR, BORDER_CONSTANT, 0)."""
    import cv2
    return cv2.warpAffine(img, M, (net_w, net_h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def map_back(faces: np.ndarray, M: np.ndarray, f: float) -> np.ndarray:
    """(k, 15) records of a warp view in network-input pixels -> image pixels: the box centre through iM, half sizes
    (x2 - x1) * (1 / (2 f)), each corner and landmark rounded to float32 once; landmark sides kept."""
    iM = invert_affine(M).reshape(6)
    half = 1.0 / (2.0 * f)
    out = np.array(faces, dtype=np.float32, copy=True)
    for row in out:
        x1, y1, x2, y2 = (float(v) for v in row[1:5])
        cx, cy = (x1 + x2) * 0.5, (y1 + y2) * 0.5
        X, Y = (iM[0] * cx + iM[1] * cy) + iM[2], (iM[3] * cx + iM[4] * cy) + iM[5]
        hw, hh = (x2 - x1) * half, (y2 - y1) * half
        row[1:5] = np.array([X - hw, Y - hh, X + hw, Y + hh], dtype=np.float32)
        lx, ly = [float(v) for v in row[5:10]], [float(v) for v in row[10:15]]
        row[5:10] = np.array([(iM[0] * x + iM[1] * y) + iM[2] for x, y in zip(lx, ly)], dtype=np.float32)
        row[10:15] = np.array([(iM[3] * x + iM[4] * y) + iM[5] for x, y in zip(lx, ly)], dtype=np.float32)
    return out
