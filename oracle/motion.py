"""f13 camera-motion oracle (rf_b200.h rf_tracker_set_motion): retinaface_b200/csrc/motion.cu restated in numpy integers and Python
doubles, every FP64 step one Python float operation (or one numpy float64 ufunc, which neither fuses nor reorders) in the kernel's
order, so every rf_motion compares bit for bit:

  thumbnail  D = ceil(max(W, H) / 320); tw = W // D, th = H // D; the rounded integer mean of each D x D luma box
  blocks     16 x 16 at (R + 16 i, R + 16 j), row by row; skipped when flat (256 sum p^2 - (sum p)^2 < 16 * 65536) or when a record
             grown by half its size on each side overlaps the block's frame rectangle
  match      exhaustive SAD over |dx|, |dy| <= R, minimum under (SAD, |dy| + |dx|, dy, dx); dropped on a shared minimum SAD or a
             border minimum; sub-pixel parabola per axis; p = (x0 + 7.5, y0 + 7.5), q = ((px + dx) + fx, (py + dy) + fy)
  fit        translations of each block and the similarities of blocks (k, k + N // 2); most inliers (|e| <= 1), lowest index;
             two rounds of inlier selection and centred least squares with the 32-lane sums
  frame      c = (D - 1) / 2;  tx' = ((D tx) + c) - ((a c) - (b c));  ty' = ((D ty) + c) - ((b c) + (a c))

`compensate` restates k_track_update's motion step on one oracle.track.Track, and `MotionTrackerOracle` is TrackerOracle with that
step after predict, before the first association stage (given the frame's rf_motion.m when its status is RF_MOTION_OK):

  s = sqrt(a a + b b), ss = s * s;  cx = ((a cx) - (b cy)) + tx;  cy = ((b cx) + (a cy)) + ty  (old cx, cy);  u_cx, u_cy likewise
  without t;  h = s h;  u_h = s u_h;  P00, P01, P11 = ss * P for cx, cy and h
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle.track import Track, TrackerOracle, map_faces

OK, FIRST, LOST = 0, 1, 2
THUMB, BLOCK, MIN_VAR, FACE_MARGIN, TOL = 320, 16, 16, 0.5, 1.0
MIN_SCALE, MAX_SCALE = 0.8, 1.25
DEFAULT_SEARCH, DEFAULT_MIN_INLIERS = 12, 12
IDENTITY = (1.0, 0.0, 0.0, 0.0, 1.0, 0.0)


def thumb_factor(width: int, height: int) -> int:
    return (max(width, height) + THUMB - 1) // THUMB


def thumbnail(luma: np.ndarray) -> Tuple[np.ndarray, int]:
    """(H, W) u8 luma -> ((th, tw) u8 thumbnail, D)."""
    H, W = luma.shape
    D = thumb_factor(W, H)
    th, tw = H // D, W // D
    s = luma[:th * D, :tw * D].astype(np.int64).reshape(th, D, tw, D).sum(axis=(1, 3))
    DD = D * D
    return ((s + DD // 2) // DD).astype(np.uint8), D


def block_grid(tw: int, th: int, R: int) -> List[Tuple[int, int]]:
    nbx = (tw - 2 * R) // BLOCK if tw - 2 * R >= BLOCK else 0
    nby = (th - 2 * R) // BLOCK if th - 2 * R >= BLOCK else 0
    return [(R + BLOCK * i, R + BLOCK * j) for j in range(nby) for i in range(nbx)]


def flat(block: np.ndarray) -> bool:
    p = block.astype(np.int64)
    return 256 * int((p * p).sum()) - int(p.sum()) ** 2 < MIN_VAR * 65536


def covered(x0: int, y0: int, D: int, boxes: List[Tuple[float, float, float, float]]) -> bool:
    X0, X1, Y0, Y1 = float(D * x0), float(D * (x0 + BLOCK)), float(D * y0), float(D * (y0 + BLOCK))
    for x1, y1, x2, y2 in boxes:
        w, h = x2 - x1, y2 - y1
        gx1, gx2 = x1 - FACE_MARGIN * w, x2 + FACE_MARGIN * w
        gy1, gy2 = y1 - FACE_MARGIN * h, y2 + FACE_MARGIN * h
        if gx1 < X1 and gx2 > X0 and gy1 < Y1 and gy2 > Y0:
            return True
    return False


def sad_table(cur: np.ndarray, ref: np.ndarray, x0: int, y0: int, R: int) -> np.ndarray:
    """SAD[sy, sx] of offset (dy, dx) = (sy - R, sx - R)."""
    blk = cur[y0:y0 + BLOCK, x0:x0 + BLOCK].astype(np.int64)
    win = ref[y0 - R:y0 + BLOCK + R, x0 - R:x0 + BLOCK + R].astype(np.int64)
    views = np.lib.stride_tricks.sliding_window_view(win, (BLOCK, BLOCK))
    return np.abs(views - blk).sum(axis=(2, 3))


def match_block(cur: np.ndarray, ref: np.ndarray, x0: int, y0: int, R: int) -> Optional[Tuple[float, float, float, float]]:
    """The block's (px, py, qx, qy), or None when the minimum is shared or on the border."""
    S = sad_table(cur, ref, x0, y0, R)
    side = 2 * R + 1
    keys = [(int(S[sy, sx]), abs(sy - R) + abs(sx - R), sy, sx) for sy in range(side) for sx in range(side)]
    smin, _, sy, sx = min(keys)
    if int((S == smin).sum()) > 1 or sx in (0, 2 * R) or sy in (0, 2 * R):
        return None
    xm, xp, ym, yp = int(S[sy, sx - 1]), int(S[sy, sx + 1]), int(S[sy - 1, sx]), int(S[sy + 1, sx])
    fx = float(xm - xp) / float(2 * (xm - 2 * smin + xp))
    fy = float(ym - yp) / float(2 * (ym - 2 * smin + yp))
    px, py = float(x0) + 7.5, float(y0) + 7.5
    return px, py, (px + float(sx - R)) + fx, (py + float(sy - R)) + fy


def lane_sum(vals) -> float:
    """The header's 32-lane sum: lane l adds terms l, l + 32, ... in order from 0.0, then lane l += lane l + o, o = 16 .. 1."""
    lanes = [0.0] * 32
    for j, v in enumerate(vals):
        lanes[j % 32] = lanes[j % 32] + v
    o = 16
    while o:
        for l in range(o):
            lanes[l] = lanes[l] + lanes[l + o]
        o //= 2
    return lanes[0]


def hypotheses(P: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """P (N, 4) = px, py, qx, qy -> ((H, 4) a, b, tx, ty, (H,) valid)."""
    N = len(P)
    px, py, qx, qy = P[:, 0], P[:, 1], P[:, 2], P[:, 3]
    trans = np.stack([np.ones(N), np.zeros(N), px - qx, py - qy], axis=1)
    k1 = np.arange(N // 2)
    k2 = k1 + N // 2
    dqx, dqy, dpx, dpy = qx[k2] - qx[k1], qy[k2] - qy[k1], px[k2] - px[k1], py[k2] - py[k1]
    den = dqx * dqx + dqy * dqy
    ok = den != 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        a = (dpx * dqx + dpy * dqy) / den
        b = (dpy * dqx - dpx * dqy) / den
    tx = px[k1] - (a * qx[k1] - b * qy[k1])
    ty = py[k1] - (b * qx[k1] + a * qy[k1])
    pair = np.stack([a, b, tx, ty], axis=1)
    return np.concatenate([trans, pair]), np.concatenate([np.ones(N, bool), ok])


def inliers(M: np.ndarray, P: np.ndarray) -> np.ndarray:
    """M (H, 4) models, P (N, 4) points -> (H, N) inlier mask."""
    a, b, tx, ty = (M[:, i:i + 1] for i in range(4))
    px, py, qx, qy = (P[None, :, i] for i in range(4))
    ex = ((a * qx - b * qy) + tx) - px
    ey = ((b * qx + a * qy) + ty) - py
    with np.errstate(invalid="ignore"):
        return ex * ex + ey * ey <= TOL * TOL


def ls_fit(P: np.ndarray, idx) -> Optional[Tuple[float, float, float, float]]:
    pts = [tuple(float(v) for v in P[k]) for k in idx]
    n = float(len(pts))
    mpx = lane_sum(p[0] for p in pts) / n
    mpy = lane_sum(p[1] for p in pts) / n
    mqx = lane_sum(p[2] for p in pts) / n
    mqy = lane_sum(p[3] for p in pts) / n
    dens, sas, sbs = [], [], []
    for px, py, qx, qy in pts:
        ux, uy, vx, vy = qx - mqx, qy - mqy, px - mpx, py - mpy
        dens.append(ux * ux + uy * uy)
        sas.append(ux * vx + uy * vy)
        sbs.append(ux * vy - uy * vx)
    den, sa, sb = lane_sum(dens), lane_sum(sas), lane_sum(sbs)
    if den == 0.0:
        return None
    a, b = sa / den, sb / den
    return a, b, (mpx - a * mqx) + b * mqy, (mpy - b * mqx) - a * mqy


def fit(P: np.ndarray, min_inliers: int) -> Tuple[int, int, Optional[Tuple[float, float, float, float]]]:
    """P (N, 4) kept point pairs in block order -> (status, inliers, (a, b, tx, ty) in thumbnail pixels or None)."""
    N = len(P)
    if N < min_inliers:
        return LOST, 0, None
    M, valid = hypotheses(P)
    counts = np.where(valid, inliers(M, P).sum(axis=1), 0)
    m = tuple(float(v) for v in M[int(np.argmax(counts))])
    n = 0
    for _ in range(2):
        idx = np.flatnonzero(inliers(np.array([m]), P)[0])
        n = len(idx)
        if n < min_inliers:
            return LOST, n, None
        m = ls_fit(P, idx)
        if m is None:
            return LOST, n, None
    return OK, n, m


def estimate(cur: np.ndarray, ref: Optional[np.ndarray], D: int, faces=None, count: Optional[int] = None, scale: Optional[float] = None,
             search: int = 0, min_inliers: int = 0) -> dict:
    """One frame: its thumbnail, the reference thumbnail (None: FIRST), D, the frame's records (K, 15) in network-input pixels
    (count: kept records; scale: map-back) -> rf_motion fields (status, blocks, inliers, m)."""
    R = search or DEFAULT_SEARCH
    mi = min_inliers or DEFAULT_MIN_INLIERS
    if ref is None:
        return dict(status=FIRST, blocks=0, inliers=0, m=IDENTITY)
    boxes = []
    if faces is not None:
        f = map_faces(np.asarray(faces, np.float32).reshape(-1, 15)[:count], scale)
        boxes = [(float(r[1]), float(r[2]), float(r[3]), float(r[4])) for r in f]
    th, tw = cur.shape
    pts = []
    for x0, y0 in block_grid(tw, th, R):
        if flat(cur[y0:y0 + BLOCK, x0:x0 + BLOCK]) or covered(x0, y0, D, boxes):
            continue
        pp = match_block(cur, ref, x0, y0, R)
        if pp is not None:
            pts.append(pp)
    P = np.array(pts, dtype=np.float64).reshape(-1, 4)
    status, n, m = fit(P, mi)
    out = dict(status=LOST, blocks=len(P), inliers=n, m=IDENTITY)
    if status != OK:
        return out
    a, b, tx, ty = m
    s = math.sqrt(a * a + b * b)
    if not (s >= MIN_SCALE and s <= MAX_SCALE):
        return out
    Dd = float(D)
    c = (Dd - 1.0) / 2.0
    out.update(status=OK, m=(a, -b, ((Dd * tx) + c) - ((a * c) - (b * c)), b, a, ((Dd * ty) + c) - ((b * c) + (a * c))))
    return out


def applied(rec: dict) -> Optional[Tuple[float, ...]]:
    """What the tracker applies for an rf_motion: its m on RF_MOTION_OK, else nothing."""
    return tuple(rec["m"]) if rec["status"] == OK else None


class MotionOracle:
    """Per-video references as rf_tracker_set_motion keeps them: the last frame's thumbnail and frame size."""

    def __init__(self, max_videos: int = 1, search: int = 0, min_inliers: int = 0):
        self.search, self.min_inliers = search, min_inliers
        self.ref: Dict[int, Tuple[np.ndarray, Tuple[int, int]]] = {}
        self.max_videos = max_videos

    def reset(self, video: int = -1):
        for v in (range(self.max_videos) if video < 0 else [video]):
            self.ref.pop(v, None)

    def update(self, video: int, luma: np.ndarray, faces=None, count: Optional[int] = None, scale: Optional[float] = None) -> dict:
        """One frame of `video` (its (H, W) u8 luma plane and records) -> rf_motion fields; the frame becomes the reference."""
        thumb, D = thumbnail(luma)
        size = (luma.shape[1], luma.shape[0])
        prev = self.ref.get(video)
        ref = prev[0] if prev is not None and prev[1] == size else None
        out = estimate(thumb, ref, D, faces, count, scale, self.search, self.min_inliers)
        self.ref[video] = (thumb, size)
        return out


def compensate(t: Track, m) -> None:
    """The motion step of k_track_update on track t, m = rf_motion.m = {a, -b, tx, b, a, ty}."""
    a, b, tx, ty = m[0], m[3], m[2], m[5]
    s = math.sqrt(a * a + b * b)
    ss = s * s
    cx, cy, ux, uy = t.m[0], t.m[1], t.u[0], t.u[1]
    t.m[0] = (a * cx - b * cy) + tx
    t.m[1] = (b * cx + a * cy) + ty
    t.u[0] = a * ux - b * uy
    t.u[1] = b * ux + a * uy
    t.m[3] = s * t.m[3]
    t.u[3] = s * t.u[3]
    for c in (0, 1, 3):
        t.p00[c] = ss * t.p00[c]
        t.p01[c] = ss * t.p01[c]
        t.p11[c] = ss * t.p11[c]


class MotionTrackerOracle(TrackerOracle):
    """TrackerOracle of a motion tracker: ``update(..., motion=m)`` moves every live track by m right after its predict (m: the
    frame's rf_motion.m on RF_MOTION_OK, ``applied``); motion None is TrackerOracle.update itself."""

    def update(self, video: int, faces: np.ndarray, scale: Optional[float] = None, max_align: int = 0, motion=None) -> List[dict]:
        if motion is None:
            return super().update(video, faces, scale, max_align)
        live = list(self.v[video]["tracks"])        # the tracks TrackerOracle.update predicts, in its order

        def moved(t):
            def predict():
                Track.predict(t)
                compensate(t, motion)
            return predict
        for t in live:
            t.predict = moved(t)                     # shadows Track.predict for this frame only
        try:
            return super().update(video, faces, scale, max_align)
        finally:
            for t in live:
                del t.predict
