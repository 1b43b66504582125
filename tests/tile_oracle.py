"""Host restatement of f7 tiles (include/rf_b200.h rf_tile_layout, rf_detect_tiled): the layout, the bytes of each tile and the
float32 map-back + ownership filter of the merge, in the same operation order as the library.  Test infrastructure, kept with the
tiled tests that are its only users; it builds on oracle.inputs (the letter-box) and cv2.resize (the levels)."""
from __future__ import annotations

import numpy as np

from oracle.inputs import letterbox_bgr_u8

SIDE_LEFT, SIDE_TOP, SIDE_RIGHT, SIDE_BOTTOM = 0x1, 0x2, 0x4, 0x8
F32 = np.float32


def level_side(side: int, s) -> int:
    """cv::resize's size of a level, saturate_cast<int>(side * s): s a float32 widened to double, rounded half to even."""
    return int(np.rint(side * float(F32(s))))


def fitted_geometry(w: int, h: int, net_w: int, net_h: int):
    """(resized w, resized h, map-back factor) of the letter-box rf_detect_batch feeds the network (letterbox_bgr_u8's geometry)."""
    sc = max(F32(1.0 * w / net_w), F32(1.0 * h / net_h), F32(1.0))
    if sc > 1:
        f = float(F32(1) / sc)
        dw, dh = int(np.rint(w * f)), int(np.rint(h * f))
    else:
        dw, dh = w, h
    return min(dw, net_w), min(dh, net_h), sc


def axis_tiles(S: int, T: int, o: int):
    """Origins and half-open ownership cores of the tiles of one axis of a level of size S."""
    k = 1 if S <= T else -(-(S - o) // (T - o))
    origin = [0 if S <= T else min(i * (T - o), S - T) for i in range(k)]
    own = []
    for i in range(k):
        a = 0 if i == 0 else own[-1][1]
        b = origin[i] + T if i == k - 1 else (origin[i + 1] + origin[i] + T) // 2     # last: the far edge of the last tile
        own.append((a, b))
    return origin, own


def default_levels(w: int, h: int, net_w: int, net_h: int):
    levels, s = [], F32(1.0)
    while level_side(w, s) > net_w or level_side(h, s) > net_h:
        levels.append((float(s), 0))
        s = F32(s * F32(0.5))
    return levels + [(0.0, 0)]


def layout(net_w: int, net_h: int, w: int, h: int, levels=None, overlap: int = 0):
    """The tiles of a w x h image as dicts with rf_tile's fields, in candidate-id order."""
    o = overlap or 64
    levels = list(levels) if levels else default_levels(w, h, net_w, net_h)
    out = []
    for li, (s, flip) in enumerate(levels):
        s = F32(s)
        if s == 0:
            sw, sh, mb = fitted_geometry(w, h, net_w, net_h)
        else:
            sw, sh, mb = level_side(w, s), level_side(h, s), F32(1.0 / float(s))
        (ox, cx), (oy, cy) = axis_tiles(sw, net_w, o), axis_tiles(sh, net_h, o)
        for j, y0 in enumerate(oy):
            for i, x0 in enumerate(ox):
                sides = ((SIDE_LEFT if i > 0 else 0) | (SIDE_TOP if j > 0 else 0) | (SIDE_RIGHT if i + 1 < len(ox) else 0)
                         | (SIDE_BOTTOM if j + 1 < len(oy) else 0))
                out.append(dict(level=li, flip=int(bool(flip)), scaled_w=sw, scaled_h=sh, x0=x0, y0=y0, own_x0=cx[i][0], own_y0=cy[j][0],
                                own_x1=cx[i][1], own_y1=cy[j][1], shared_sides=sides, scale=float(s), map_back=float(mb)))
    return out


def level_image(img: np.ndarray, s: float, flip: bool) -> np.ndarray:
    """cv2.resize(cv2.flip(img) if flip else img, None, fx=s, fy=s) (INTER_LINEAR)."""
    import cv2
    src = cv2.flip(img, 1) if flip else img
    s = float(F32(s))
    return cv2.resize(src, None, fx=s, fy=s)


def tile_bytes(img: np.ndarray, tile: dict, net_w: int, net_h: int, level: np.ndarray = None) -> np.ndarray:
    """The network input of one tile: a slice of the resized level padded with zeros; the fitted level is the letter-box."""
    import cv2
    if tile["scale"] == 0:
        return letterbox_bgr_u8(cv2.flip(img, 1) if tile["flip"] else img, net_h, net_w)
    lev = level_image(img, tile["scale"], tile["flip"]) if level is None else level
    assert lev.shape[:2] == (tile["scaled_h"], tile["scaled_w"]), (lev.shape, tile)
    out = np.zeros((net_h, net_w, 3), np.uint8)
    crop = lev[tile["y0"]:tile["y0"] + net_h, tile["x0"]:tile["x0"] + net_w]
    out[:crop.shape[0], :crop.shape[1]] = crop
    return out


def map_tile(dets: np.ndarray, tile: dict, img_w: int, net_w: int, net_h: int) -> np.ndarray:
    """The merge of one tile's kept detections ((k, 15) float32 rows, network pixels): the ownership and seam filter, then the
    map-back to image pixels (un-mirrored, landmarks swapped), float32 operation by operation.  Returns the surviving rows, in order,
    and their ranks in the tile."""
    d = np.asarray(dets, F32).reshape(-1, 15)
    x0, y0, mb = F32(tile["x0"]), F32(tile["y0"]), F32(tile["map_back"])
    cx = (d[:, 1] + d[:, 3]) * F32(0.5)
    cy = (d[:, 2] + d[:, 4]) * F32(0.5)
    sides = tile["shared_sides"]
    keep = np.ones(len(d), bool)
    if sides & (SIDE_LEFT | SIDE_RIGHT):        # an axis held by one tile owns everything along it
        keep &= (cx >= F32(tile["own_x0"] - tile["x0"])) & (cx < F32(tile["own_x1"] - tile["x0"]))
    if sides & (SIDE_TOP | SIDE_BOTTOM):
        keep &= (cy >= F32(tile["own_y0"] - tile["y0"])) & (cy < F32(tile["own_y1"] - tile["y0"]))
    if sides & SIDE_LEFT:
        keep &= ~(d[:, 1] <= 0)
    if sides & SIDE_TOP:
        keep &= ~(d[:, 2] <= 0)
    if sides & SIDE_RIGHT:
        keep &= ~(d[:, 3] >= F32(net_w - 1))
    if sides & SIDE_BOTTOM:
        keep &= ~(d[:, 4] >= F32(net_h - 1))
    rank = np.nonzero(keep)[0]
    d = d[keep]

    def mx(v):
        return (v + x0) * mb if x0 != 0 else v * mb

    def my(v):
        return (v + y0) * mb if y0 != 0 else v * mb
    m = d.copy()
    m[:, 1], m[:, 3], m[:, 5:10] = mx(d[:, 1]), mx(d[:, 3]), mx(d[:, 5:10])
    m[:, 2], m[:, 4], m[:, 10:15] = my(d[:, 2]), my(d[:, 4]), my(d[:, 10:15])
    if tile["flip"]:
        wm1 = F32(img_w - 1)
        f = m.copy()
        f[:, 1], f[:, 3] = wm1 - m[:, 3], wm1 - m[:, 1]
        f[:, 5:10] = (wm1 - m[:, 5:10])[:, [1, 0, 2, 4, 3]]
        f[:, 10:15] = m[:, 10:15][:, [1, 0, 2, 4, 3]]
        m = f
    return m, rank
