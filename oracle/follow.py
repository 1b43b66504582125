"""f16 follow oracle (rf_b200.h rf_tracker_set_follow): luma templates cut on detect frames, the three-scale SAD search on follow
frames and the tracker step that replaces association there.

Plain numpy / Python restatement of retinaface_b200/csrc/follow.cu: every FP64 step is one Python float operation (IEEE double, one
rounding each, never fused) in the kernel's order, rint is half to even as __double2int_rn, and pixels are integers, so templates,
SADs, statuses, boxes and the FP64 Kalman state compare bit for bit.  Detect frames are oracle/track.py's update, unchanged.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

import math

from oracle.motion import MotionTrackerOracle, compensate
from oracle.track import CONFIRMED, LOST, TENTATIVE, measure

T = 32                      # RF_FOLLOW_TEMPLATE
MARGIN = 0.25               # RF_FOLLOW_MARGIN
SCALE = 1.05                # RF_FOLLOW_SCALE
MIN_VAR = 16                # RF_FOLLOW_MIN_VAR
MAX_SEARCH = 16             # RF_FOLLOW_MAX_SEARCH
OK, FLAT, BORDER, MISMATCH, OUTSIDE, LOST_STATUS = range(6)
GROW = 1.0 + 2.0 * MARGIN
MAX_BOX = 65536.0           # a predicted state beyond this is not searched


def config(search: int = 0, max_mad: float = 0.0) -> Tuple[int, float]:
    """rf_follow_config with the defaults applied (R, max_mad as float32); ValueError where rf_tracker_set_follow refuses."""
    R = int(search) or 8
    mad = float(np.float32(max_mad)) if max_mad else float(np.float32(24.0))
    if not 1 <= R <= MAX_SEARCH:
        raise ValueError(f"search {search}, must be 0 or in [1, {MAX_SEARCH}]")
    if not (np.isfinite(mad) and 0.0 < mad <= 255.0):
        raise ValueError(f"max_mad {max_mad}, must be 0 or finite in (0, 255]")
    return R, mad


def scale_of(k: int) -> float:
    return (1.0 / SCALE, 1.0, SCALE)[k]


def grid(cx: float, cy: float, w: float, h: float, c: float) -> Tuple[float, float, float, float]:
    """(px, py, ox, oy): template pixel (i, j) of the box at scale c is centred on (ox + px i, oy + py j)."""
    gw = (w * GROW) * c
    gh = (h * GROW) * c
    px = gw / float(T)
    py = gh / float(T)
    ox = ((cx - gw / 2.0) + px / 2.0) - 0.5
    oy = ((cy - gh / 2.0) + py / 2.0) - 0.5
    return px, py, ox, oy


def sample(luma: np.ndarray, px: float, py: float, X: float, Y: float, n: int) -> Tuple[np.ndarray, np.ndarray]:
    """n x n pixels of cv2.warpAffine(luma, [[px, 0, X], [0, py, Y]], INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT 0) and each
    pixel's INSIDE flag (its four taps in the frame)."""
    h, w = luma.shape
    i = np.arange(n, dtype=np.float64)
    Xf = (int(np.rint(X * 1024.0)) + 16 + np.rint((px * i) * 1024.0).astype(np.int64)) >> 5
    Yf = (np.rint((py * i + Y) * 1024.0).astype(np.int64) + 16) >> 5
    XX, YY = np.broadcast_to(Xf[None, :], (n, n)), np.broadcast_to(Yf[:, None], (n, n))
    sx, sy = np.clip(XX >> 5, -32768, 32767), np.clip(YY >> 5, -32768, 32767)
    fx, fy = XX & 31, YY & 31
    src = luma.astype(np.int64)
    acc = np.full((n, n), 16384, dtype=np.int64)
    cnt = np.zeros((n, n), dtype=np.int64)
    for dy, dx, wgt in ((0, 0, 32 * (32 - fx) * (32 - fy)), (0, 1, 32 * fx * (32 - fy)), (1, 0, 32 * (32 - fx) * fy), (1, 1, 32 * fx * fy)):
        tx, ty = sx + dx, sy + dy
        inside = (tx >= 0) & (tx < w) & (ty >= 0) & (ty < h)
        acc += src[np.clip(ty, 0, h - 1), np.clip(tx, 0, w - 1)] * wgt * inside
        cnt += inside
    return (acc >> 15).astype(np.uint8), cnt == 4


def face_grid(face) -> Tuple[float, float, float, float]:
    x1, y1 = float(face[1]), float(face[2])
    w = float(face[3]) - x1
    h = float(face[4]) - y1
    return grid(x1 + w / 2.0, y1 + h / 2.0, w, h, 1.0)


def cut(luma: np.ndarray, face) -> Tuple[np.ndarray, bool]:
    """The T x T template of a face record (frame pixels) and its FLAT test."""
    px, py, ox, oy = face_grid(face)
    tmpl, _ = sample(luma, px, py, ox, oy, T)
    p = tmpl.astype(np.int64)
    s1, s2 = int(p.sum()), int((p * p).sum())
    return tmpl, T * T * s2 - s1 * s1 < MIN_VAR * T ** 4


def sads(tmpl: np.ndarray, win: np.ndarray, R: int) -> np.ndarray:
    """SAD[dy + R, dx + R] of the template against every T x T sub-window of a (T + 2R)^2 window."""
    v = np.lib.stride_tricks.sliding_window_view(win.astype(np.int32), (T, T))
    return np.abs(v - tmpl.astype(np.int32)[None, None]).sum(axis=(2, 3))


def order_key(sad: int, k: int, dy: int, dx: int, R: int) -> int:
    """The minimum's order (SAD, |dx| + |dy|, k, dy, dx) as the kernel's 64-bit key."""
    return (sad << 20) | ((abs(dx) + abs(dy)) << 14) | (k << 12) | ((dy + R) << 6) | (dx + R)


def parabola(sm: int, s0: int, sp: int) -> float:
    d = 2 * (sm - 2 * s0 + sp)
    return 0.0 if d == 0 else (sm - sp) / d


def search(luma: np.ndarray, tmpl: Optional[np.ndarray], flat: bool, m: List[float], u: List[float], face: np.ndarray, R: int,
           max_mad: float, motion=None) -> Tuple[dict, Optional[np.ndarray]]:
    """One searched track: its state (m, u) before predict, its previous face, the frame's applied camera motion (rf_motion.m or
    None); -> (the rf_follow fields, the followed face record)."""
    pcx, pcy, pa, ph = m[0] + u[0], m[1] + u[1], m[2] + u[2], m[3] + u[3]
    if motion is not None:
        a, b = motion[0], motion[3]
        cx, cy = pcx, pcy
        pcx = (a * cx - b * cy) + motion[2]
        pcy = (b * cx + a * cy) + motion[5]
        ph = math.sqrt(a * a + b * b) * ph
    pw = pa * ph
    bounded = 0.0 < ph <= MAX_BOX and 0.0 < pw <= MAX_BOX and abs(pcx) <= MAX_BOX and abs(pcy) <= MAX_BOX
    if tmpl is None or not bounded:
        return dict(id=0, status=FLAT if bounded else MISMATCH, dx=0, dy=0, scale=0, sad=0, fx=0.0, fy=0.0, x1=0.0, y1=0.0, x2=0.0,
                    y2=0.0), None
    n = T + 2 * R
    grids, wins, ins, S = [], [], [], []
    for k in range(3):
        px, py, ox, oy = grid(pcx, pcy, pw, ph, scale_of(k))
        grids.append((px, py))
        win, inside = sample(luma, px, py, ox - float(R) * px, oy - float(R) * py, n)
        wins.append(win)
        ins.append(inside)
        S.append(sads(tmpl, win, R))
    best = None
    for k in range(3):
        Sk = S[k]
        dyy, dxx = np.meshgrid(np.arange(-R, R + 1), np.arange(-R, R + 1), indexing="ij")
        keys = (Sk.astype(np.int64) << 20) | ((np.abs(dxx) + np.abs(dyy)) << 14) | (k << 12) | ((dyy + R) << 6) | (dxx + R)
        kk = int(keys.min())
        best = kk if best is None else min(best, kk)
    k, wy, wx = (best >> 12) & 3, (best >> 6) & 63, best & 63
    dx, dy = wx - R, wy - R
    Sk = S[k]
    s0 = int(Sk[wy, wx])
    border = abs(dx) == R or abs(dy) == R
    fx = fy = 0.0
    if not border:
        fx = parabola(int(Sk[wy, wx - 1]), s0, int(Sk[wy, wx + 1]))
        fy = parabola(int(Sk[wy - 1, wx]), s0, int(Sk[wy + 1, wx]))
    px, py = grids[k]
    ncx = pcx + (float(dx) + fx) * px
    ncy = pcy + (float(dy) + fy) * py
    c = scale_of(k)
    nw, nh = pw * c, ph * c
    f32 = np.float32
    nf = np.array(face, dtype=np.float32).copy()
    nf[1], nf[2], nf[3], nf[4] = f32(ncx - nw / 2.0), f32(ncy - nh / 2.0), f32(ncx + nw / 2.0), f32(ncy + nh / 2.0)
    ow = float(face[3]) - float(face[1])
    oh = float(face[4]) - float(face[2])
    ocx = float(face[1]) + ow / 2.0
    ocy = float(face[2]) + oh / 2.0
    sx, sy = nw / ow, nh / oh
    for l in range(5):
        nf[5 + l] = f32(ncx + (float(face[5 + l]) - ocx) * sx)
        nf[10 + l] = f32(ncy + (float(face[10 + l]) - ocy) * sy)
    inside = int(ins[k][wy:wy + T, wx:wx + T].sum())
    empty = not (float(nf[3]) - float(nf[1]) > 0.0) or not (float(nf[4]) - float(nf[2]) > 0.0)
    if flat:
        status = FLAT
    elif 4 * inside < 3 * T * T:
        status = OUTSIDE
    elif border:
        status = BORDER
    elif float(s0) > float(np.float32(max_mad)) * float(T * T) or empty:
        status = MISMATCH
    else:
        status = OK
    rec = dict(id=0, status=status, dx=dx, dy=dy, scale=k, sad=s0, fx=f32(fx), fy=f32(fy), x1=nf[1], y1=nf[2], x2=nf[3], y2=nf[4])
    return rec, nf


def luma_of(buf: np.ndarray, w: int, h: int) -> np.ndarray:
    """The Y plane of a host 4:2:0 buffer (rows of any pitch >= w)."""
    return np.asarray(buf)[:h, :w]


class FollowTrackerOracle(MotionTrackerOracle):
    """The tracker oracle plus f16: `update` (detect frames) takes the frame's luma and cuts the templates; `follow` is a follow frame.
    motion: the frame's applied rf_motion.m (oracle/motion.py `applied`), or None."""

    def __init__(self, max_videos: int = 1, search: int = 0, max_mad: float = 0.0, **cfg):
        self.R, self.max_mad = config(search, max_mad)
        self.tmpl: Dict[int, Dict[int, Tuple[np.ndarray, bool]]] = {}
        super().__init__(max_videos, **cfg)

    def reset(self, video: int = -1):
        super().reset(video)
        for v in (range(self.max_videos) if video < 0 else [video]):
            self.tmpl[v] = {}

    def update(self, video: int, faces: np.ndarray, scale: Optional[float] = None, max_align: int = 0, motion=None,
               luma: Optional[np.ndarray] = None) -> List[dict]:
        out = super().update(video, faces, scale, max_align, motion=motion)
        for t in self.v[video]["tracks"]:
            if t.det >= 0:
                self.tmpl[video][t.id] = cut(luma, t.face)
        for r in out:
            r["followed"] = 0
        return out

    def mask_faces(self, video: int) -> np.ndarray:
        """The follow frame's f13 face mask: the faces of the video's TENTATIVE and CONFIRMED tracks, (K, 15) in frame pixels."""
        return np.array([t.face for t in self.v[video]["tracks"] if t.state != LOST], np.float32).reshape(-1, 15)

    def follow(self, video: int, luma: np.ndarray, motion=None) -> Tuple[List[dict], List[dict]]:
        """One follow frame of `video`: (the live tracks after it, as rf_track fields with `followed`; the rf_follow records in the same
        order)."""
        V = self.v[video]
        recs, keep, ok = {}, [], set()
        for t in V["tracks"]:
            st0 = t.state
            if st0 != LOST:
                tm = self.tmpl[video].get(t.id)
                rec, nf = search(luma, tm[0] if tm else None, tm[1] if tm else True, t.m, t.u, t.face, self.R, self.max_mad, motion)
                rec["id"] = t.id
                recs[t.id] = rec
            t.predict()
            if motion is not None:
                compensate(t, motion)
            t.age += 1
            t.det = -1
            if st0 != LOST and recs[t.id]["status"] == OK:
                t.update(measure(nf))
                t.lost = 0
                t.face = nf
                ok.add(t.id)
                keep.append(t)
                continue
            if st0 == TENTATIVE:
                continue
            if st0 == CONFIRMED:
                t.state, t.lost = LOST, 1
            else:
                t.lost += 1
            if t.lost <= self.max_lost:
                keep.append(t)
        V["frames"] += 1
        keep.sort(key=lambda t: t.id)
        V["tracks"] = keep
        tracks, follows = [], []
        for t in keep:
            r = t.record(-1)
            r["followed"] = int(t.id in ok)
            tracks.append(r)
            follows.append(recs[t.id] if t.id in recs else dict(id=t.id, status=LOST_STATUS, dx=0, dy=0, scale=0, sad=0, fx=0.0, fy=0.0,
                                                                  x1=0.0, y1=0.0, x2=0.0, y2=0.0))
        return tracks, follows
