"""f9 EXIF orientations restated in numpy: the displayed image of a stored one under each orientation (what cv2.imread applies), the
same on the planes of a single-buffer 4:2:0 frame, and its inverse.  The oriented letter-box, crop, tiling, tracking and redaction
kernels are held against their unoriented twins run on these materialised copies.  Test infrastructure -- see
``oracle/__init__.py``."""
from __future__ import annotations

import numpy as np

INVERSE = {6: 8, 8: 6}          # every other orientation is its own inverse


def orient(img, o):
    """T_o(img): the displayed image of a stored one under EXIF orientation o (what cv2.imread applies)."""
    return np.ascontiguousarray({1: lambda a: a, 2: lambda a: a[:, ::-1], 3: lambda a: a[::-1, ::-1], 4: lambda a: a[::-1],
                                 5: lambda a: a.swapaxes(0, 1), 6: lambda a: np.rot90(a, -1), 7: lambda a: a.swapaxes(0, 1)[::-1, ::-1],
                                 8: lambda a: np.rot90(a, 1)}[o](img))


def orient_planes(frame, layout, o):
    """The single-buffer 4:2:0 frame of T_o applied to each plane (chroma blocks of an even-sided frame map onto chroma blocks)."""
    rows, w = frame.shape
    h = rows * 2 // 3
    y = orient(frame[:h], o)
    if layout == "nv12":
        uv = orient(frame[h:].reshape(h // 2, w // 2, 2), o)
        return np.ascontiguousarray(np.concatenate([y, uv.reshape(uv.shape[0], -1)], axis=0))
    q = (h // 2) * (w // 2)
    flat = frame[h:].reshape(-1)
    u, v = orient(flat[:q].reshape(h // 2, w // 2), o), orient(flat[q:].reshape(h // 2, w // 2), o)
    return np.ascontiguousarray(np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(-1, y.shape[1]))


def unorient_planes(frame, layout, o):
    """The stored single-buffer 4:2:0 frame S whose orient_planes(S, layout, o) is `frame` (a displayed frame)."""
    return orient_planes(frame, layout, INVERSE.get(o, o))
