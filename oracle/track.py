"""f10 tracker oracle (rf_b200.h rf_track_update): ByteTrack's association with SORT's constant-velocity Kalman filter.

`TrackerOracle` is a plain-Python scalar restatement of retinaface_b200/csrc/track.cu: every FP64 step is one Python float operation
(IEEE double, one rounding each, never fused) in the kernel's order, so ids, states and every float field compare bit for bit:

  predict   LOST: u_h = 0.  q_pos = sp * h, q_vel = sv * h (a: 1e-2, 1e-5), h the track's m_h;
            P00 = ((P00 + P01) + (P01 + P11)) + q_pos * q_pos;  P01 = P01 + P11;  P11 = P11 + q_vel * q_vel;  m = m + u
  update    r = sp * h (a: 1e-1), h = m_h before the step;  S = P00 + r * r;  K0 = P00 / S;  K1 = P01 / S;  y = z - m;
            m = m + K0 * y;  u = u + K1 * y;  P00 = P00 - (K0 * S) * K0;  P01 = P01 - (K0 * S) * K1;  P11 = P11 - (K1 * S) * K1
  birth     m = z;  u = 0;  P00 = ((2 * sp) * h)^2 (a: 1e-2^2);  P01 = 0;  P11 = ((10 * sv) * h)^2 (a: 1e-5^2)
  z         float32 record coordinates times the float32 scale (rounded to float32), widened: w = x2 - x1; h = y2 - y1;
            cx = x1 + w / 2; cy = y1 + h / 2; a = w / h (w <= 0 or h <= 0: ignored)
  box       w = a * h; x1 = cx - w / 2; y1 = cy - h / 2; x2 = x1 + w; y2 = y1 + h
  IoU       the reference NMS's +1 pixel convention, in double

`KalmanMatrix` is ByteTrack's 8 x 8 filter in numpy (its matrix form), which the scalar filter must equal to rounding.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

TENTATIVE, CONFIRMED, LOST = 0, 1, 2
SP, SV = 1.0 / 20.0, 1.0 / 160.0
DEFAULTS = dict(max_tracks=64, high_thresh=0.6, new_thresh=0.7, iou_high=0.2, iou_low=0.5, iou_tentative=0.3, max_lost=30)


def map_faces(faces: np.ndarray, scale: Optional[float]) -> np.ndarray:
    """(K, 15) float32 records in network-input pixels -> frame pixels: every coordinate times the float32 scale, rounded to
    float32 (__fmul_rn); scale None: 1."""
    f = np.array(faces, dtype=np.float32).reshape(-1, 15)
    if scale is not None:
        f[:, 1:] = f[:, 1:] * np.float32(scale)
    return f


def measure(face) -> Optional[List[float]]:
    x1, y1, x2, y2 = float(face[1]), float(face[2]), float(face[3]), float(face[4])
    w = x2 - x1
    h = y2 - y1
    if not (w > 0.0) or not (h > 0.0):
        return None
    return [x1 + w / 2.0, y1 + h / 2.0, w / h, h]


def box_of(m) -> List[float]:
    w = m[2] * m[3]
    x1 = m[0] - w / 2.0
    y1 = m[1] - m[3] / 2.0
    return [x1, y1, x1 + w, y1 + m[3]]


def iou(a, b) -> float:
    x, y = max(a[0], b[0]), max(a[1], b[1])
    w = (min(a[2], b[2]) - x) + 1.0
    h = (min(a[3], b[3]) - y) + 1.0
    if not (w > 0.0) or not (h > 0.0):
        return 0.0
    area1 = ((a[2] - a[0]) + 1.0) * ((a[3] - a[1]) + 1.0)
    area2 = ((b[2] - b[0]) + 1.0) * ((b[3] - b[1]) + 1.0)
    inter = w * h
    return inter / ((area1 + area2) - inter)


class Track:
    def __init__(self, tid: int, z: List[float], face: np.ndarray, state: int, det: int):
        self.id, self.state, self.hits, self.age, self.lost, self.det = tid, state, 1, 1, 0, det
        self.face = face.copy()
        h = z[3]
        self.m = list(z)
        self.u = [0.0] * 4
        self.p00, self.p01, self.p11 = [0.0] * 4, [0.0] * 4, [0.0] * 4
        for c in range(4):
            sp = 1e-2 if c == 2 else (2.0 * SP) * h
            sv = 1e-5 if c == 2 else (10.0 * SV) * h
            self.p00[c] = sp * sp
            self.p11[c] = sv * sv

    def predict(self):
        if self.state == LOST:
            self.u[3] = 0.0
        h = self.m[3]
        for c in range(4):
            qp = 1e-2 if c == 2 else SP * h
            qv = 1e-5 if c == 2 else SV * h
            p00, p01, p11 = self.p00[c], self.p01[c], self.p11[c]
            self.p00[c] = ((p00 + p01) + (p01 + p11)) + qp * qp
            self.p01[c] = p01 + p11
            self.p11[c] = p11 + qv * qv
            self.m[c] = self.m[c] + self.u[c]

    def update(self, z: List[float]):
        h = self.m[3]
        for c in range(4):
            r = 1e-1 if c == 2 else SP * h
            p00, p01, p11 = self.p00[c], self.p01[c], self.p11[c]
            S = p00 + r * r
            K0 = p00 / S
            K1 = p01 / S
            y = z[c] - self.m[c]
            self.m[c] = self.m[c] + K0 * y
            self.u[c] = self.u[c] + K1 * y
            self.p00[c] = p00 - (K0 * S) * K0
            self.p01[c] = p01 - (K0 * S) * K1
            self.p11[c] = p11 - (K1 * S) * K1

    def record(self, crop_slot: int = -1) -> dict:
        b = box_of(self.m)
        f32 = np.float32
        return dict(id=self.id, state=self.state, det=self.det, crop_slot=crop_slot, hits=self.hits, age=self.age, lost_frames=self.lost,
                    kx1=f32(b[0]), ky1=f32(b[1]), kx2=f32(b[2]), ky2=f32(b[3]), vx=f32(self.u[0]), vy=f32(self.u[1]), face=self.face.copy())

    def debug(self) -> List[float]:
        return [float(self.id), float(self.state), float(self.hits), float(self.age), float(self.lost)] + self.m + self.u + self.p00 + self.p01 + self.p11


def greedy(pairs):
    """Greedy by descending IoU, ties to the lower track id, then the lower record index: [(iou, id, det)] -> {id: det}."""
    out, used = {}, set()
    for _, tid, j in sorted(pairs, key=lambda p: (-p[0], p[1], p[2])):
        if tid not in out and j not in used:
            out[tid] = j
            used.add(j)
    return out


class TrackerOracle:
    """max_videos independent sequences; thresholds as the C ABI takes them (float32; 0 -> the defaults)."""

    def __init__(self, max_videos: int = 1, **cfg):
        c = dict(DEFAULTS)
        c.update({k: v for k, v in cfg.items() if v})
        self.T, self.max_lost = int(c["max_tracks"]), int(c["max_lost"])
        f = lambda k: float(np.float32(c[k]))   # noqa: E731
        self.high, self.new = f("high_thresh"), f("new_thresh")
        self.iou_high, self.iou_low, self.iou_tent = f("iou_high"), f("iou_low"), f("iou_tentative")
        self.max_videos = max_videos
        self.v: Dict[int, dict] = {}
        self.reset(-1)

    def reset(self, video: int = -1):
        for v in (range(self.max_videos) if video < 0 else [video]):
            self.v[v] = dict(issued=0, frames=0, overflow=0, tracks=[])

    def update(self, video: int, faces: np.ndarray, scale: Optional[float] = None, max_align: int = 0) -> List[dict]:
        """One frame of `video`: its kept records (K, 15) float32 in network-input pixels (best score first) and map-back scale.
        Returns the live tracks after the frame, sorted by id, as rf_track fields."""
        V = self.v[video]
        dets = map_faces(faces, scale)
        Z = [measure(d) for d in dets]
        tracks: List[Track] = V["tracks"]
        st0 = {}
        for t in tracks:
            st0[t.id] = t.state
            t.predict()
            t.age += 1
        match: Dict[int, int] = {}
        used = set()

        def stage(track_ok, det_ok, thr):
            pairs = []
            for t in tracks:
                if t.id in match or not track_ok(st0[t.id]):
                    continue
                p = box_of(t.m)
                for j, d in enumerate(dets):
                    if j in used or not det_ok(float(d[0])) or Z[j] is None:
                        continue
                    s = iou(p, [float(d[1]), float(d[2]), float(d[3]), float(d[4])])
                    if s > thr:
                        pairs.append((s, t.id, j))
            for tid, j in greedy(pairs).items():
                match[tid] = j
                used.add(j)

        hi = self.high
        stage(lambda s: s in (CONFIRMED, LOST), lambda sc: sc >= hi, self.iou_high)
        stage(lambda s: s == CONFIRMED, lambda sc: not (sc >= hi), self.iou_low)
        stage(lambda s: s == TENTATIVE, lambda sc: sc >= hi, self.iou_tent)
        due = set()
        keep = []
        for t in tracks:
            j = match.get(t.id, -1)
            if j >= 0:
                t.update(Z[j])
                t.hits += 1
                t.lost = 0
                t.face = dets[j].copy()
                t.det = j
                if st0[t.id] == TENTATIVE:
                    due.add(t.id)
                t.state = CONFIRMED
                keep.append(t)
                continue
            t.det = -1
            if st0[t.id] == TENTATIVE:
                continue
            if st0[t.id] == CONFIRMED:
                t.state, t.lost = LOST, 1
            else:
                t.lost += 1
            if t.lost <= self.max_lost:
                keep.append(t)
        first = V["frames"] == 0
        for j, d in enumerate(dets):
            if j in used or not (float(d[0]) >= hi) or not (float(d[0]) >= self.new) or Z[j] is None:
                continue
            if len(keep) == self.T:
                V["overflow"] += 1
                continue
            V["issued"] += 1
            keep.append(Track(V["issued"], Z[j], d, CONFIRMED if first else TENTATIVE, j))
            if first:
                due.add(V["issued"])
        V["frames"] += 1
        keep.sort(key=lambda t: t.id)
        V["tracks"] = keep
        out, k = [], 0
        for t in keep:
            slot = -1
            if t.id in due:
                slot = k if k < max_align else -1
                k += 1
            out.append(t.record(slot))
        return out

    def debug_state(self, video: int) -> np.ndarray:
        """rf_tracker_debug_state's doubles: live count, next id, frames, overflow, then 25 per live track in id order."""
        V = self.v[video]
        vals = [float(len(V["tracks"])), float(V["issued"] + 1), float(V["frames"]), float(V["overflow"])]
        for t in V["tracks"]:
            vals += t.debug()
        return np.array(vals, dtype=np.float64)


class KalmanMatrix:
    """ByteTrack's KalmanFilter (8 x 8, state (cx, cy, a, h) and velocities) in numpy: the matrix form the scalar filter decouples."""

    def __init__(self):
        self.F = np.eye(8)
        for i in range(4):
            self.F[i, 4 + i] = 1.0
        self.H = np.eye(4, 8)

    def initiate(self, z):
        h = z[3]
        std = [2 * SP * h, 2 * SP * h, 1e-2, 2 * SP * h, 10 * SV * h, 10 * SV * h, 1e-5, 10 * SV * h]
        return np.r_[np.asarray(z, float), np.zeros(4)], np.diag(np.square(std))

    def predict(self, mean, cov, lost=False):
        mean = mean.copy()
        if lost:
            mean[7] = 0.0
        h = mean[3]
        std = [SP * h, SP * h, 1e-2, SP * h, SV * h, SV * h, 1e-5, SV * h]
        return self.F @ mean, self.F @ cov @ self.F.T + np.diag(np.square(std))

    def update(self, mean, cov, z):
        h = mean[3]
        R = np.diag(np.square([SP * h, SP * h, 1e-1, SP * h]))
        S = self.H @ cov @ self.H.T + R
        K = np.linalg.solve(S, self.H @ cov).T
        return mean + K @ (np.asarray(z, float) - self.H @ mean), cov - K @ S @ K.T
