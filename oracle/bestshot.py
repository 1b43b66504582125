"""f11 best-shot oracle (rf_b200.h rf_tracker_create_best): the face quality of a crop and the per-track best-shot rule, restated in
numpy int64 and Python doubles.

* ``quality``         -- q and its terms for one crop, every FP64 step one Python float operation in the header's order (IEEE
                         double, one rounding each); INSIDE from the fixed-point tap coordinates of ``oracle.align.warp_affine_fixed``.
* ``grey``            -- cv2.cvtColor(BGR2GRAY) of u8 BGR pixels, (3735 B + 19235 G + 9798 R + 16384) >> 15.
* ``laplacian``       -- the 4-neighbour stencil of cv2.Laplacian(ksize=1) on the interior.
* ``BestShotOracle``  -- the store and the emission rule, fed ``TrackerOracle.update`` outputs frame by frame with each frame's
                         record crops and matrices.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from .align import ARCFACE_112, invert_affine
from .track import TENTATIVE

BEST_EXIT, BEST_FINISH = 0, 1
SHARP_HALF = 50.0


def grey(bgr: np.ndarray) -> np.ndarray:
    p = np.asarray(bgr).astype(np.int64)
    return (3735 * p[..., 0] + 19235 * p[..., 1] + 9798 * p[..., 2] + 16384) >> 15


def laplacian(g: np.ndarray) -> np.ndarray:
    """L(x, y) = g(x-1, y) + g(x+1, y) + g(x, y-1) + g(x, y+1) - 4 g(x, y) over 1 <= x <= w-2, 1 <= y <= h-2."""
    g = np.asarray(g, np.int64)
    return g[1:-1, :-2] + g[1:-1, 2:] + g[:-2, 1:-1] + g[2:, 1:-1] - 4 * g[1:-1, 1:-1]


def inside_mask(M: np.ndarray, frame_w: int, frame_h: int, size) -> np.ndarray:
    """(ch, cw) bool: the four bilinear taps of the crop pixel's cv::warpAffine sample all lie in the frame (the coordinates of
    warp_affine_fixed, after the saturate)."""
    cw, ch = size
    iM = invert_affine(M)
    x = np.arange(cw, dtype=np.float64)
    y = np.arange(ch, dtype=np.float64)
    adelta = np.rint(iM[0, 0] * x * 1024).astype(np.int64)
    bdelta = np.rint(iM[1, 0] * x * 1024).astype(np.int64)
    X0 = np.rint((iM[0, 1] * y + iM[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((iM[1, 1] * y + iM[1, 2]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + adelta[None, :]) >> 5
    Y = (Y0[:, None] + bdelta[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    return (sx >= 0) & (sx + 1 < frame_w) & (sy >= 0) & (sy + 1 < frame_h)


def quality(crop_u8: np.ndarray, face, M, frame_w: int, frame_h: int, template=ARCFACE_112, sharp_half: float = SHARP_HALF) -> dict:
    """q and its terms (Python floats) of one u8 BGR crop: face is the record's 15 floats in frame pixels (score, box, lx[5], ly[5]),
    M its 2 x 3 matrix, template the 5 x 2 crop-pixel targets (float32, as the C ABI takes them)."""
    face = np.asarray(face, np.float32).reshape(15)
    M = np.asarray(M, np.float64).reshape(2, 3)
    lx = [float(v) for v in face[5:10]]
    ly = [float(v) for v in face[10:15]]
    out = dict(score=float(face[0]), eye=0.0, frontal=0.0, sharpness=0.0, coverage=0.0, q=0.0)
    ex = lx[1] - lx[0]
    ey = ly[1] - ly[0]
    d2 = ex * ex + ey * ey
    if d2 == 0.0 or not M.any():
        return out
    ch, cw = crop_u8.shape[:2]
    eye = math.sqrt(d2)
    t = ((lx[2] - (lx[0] + lx[1]) / 2.0) * ex + (ly[2] - (ly[0] + ly[1]) / 2.0) * ey) / d2
    frontal = max(0.0, 1.0 - 2.0 * abs(t))
    tm = np.asarray(template, np.float32).reshape(10)
    tx = float(tm[2]) - float(tm[0])
    ty = float(tm[3]) - float(tm[1])
    eye_ref = math.sqrt(tx * tx + ty * ty)
    size = min(1.0, eye / eye_ref) if eye_ref > 0.0 else 1.0
    ins = inside_mask(M, frame_w, frame_h, (cw, ch))
    ok = ins[1:-1, 1:-1] & ins[1:-1, :-2] & ins[1:-1, 2:] & ins[:-2, 1:-1] & ins[2:, 1:-1]
    L = laplacian(grey(crop_u8))[ok]
    N, S1, S2 = int(L.size), int(L.sum()), int((L * L).sum())
    sharpness = float(N * S2 - S1 * S1) / (float(N) * float(N)) if N >= 2 else 0.0
    sharp = sharpness / (sharpness + float(np.float32(sharp_half)))
    coverage = float(int(ins.sum())) / float(cw * ch)
    q = (((float(face[0]) * frontal) * size) * sharp) * coverage
    out.update(eye=eye, frontal=frontal, sharpness=sharpness, coverage=coverage, q=q)
    return out


class BestShotOracle:
    """Per video: the best (q, crop, M, terms, record, frame) of every live track, and the emissions of each frame.  Thresholds as the
    C ABI takes them (float32; sharp_half 0 -> 50)."""

    def __init__(self, min_quality: float = 0.0, sharp_half: float = 0.0, template=ARCFACE_112):
        self.min_q = float(np.float32(min_quality))
        self.sharp_half = float(np.float32(sharp_half)) or SHARP_HALF
        self.template = np.asarray(template, np.float32)
        self.v: Dict[int, dict] = {}

    def reset(self, video: int):
        self.v[video] = dict(frames=0, best={}, live={})

    def _video(self, video: int) -> dict:
        if video not in self.v:
            self.reset(video)
        return self.v[video]

    @staticmethod
    def _shot(b: dict, tid: int, video: int, end_frame: int, hits: int, age: int, reason: int) -> dict:
        f32 = np.float32
        return dict(id=tid, video=video, frame=b["frame"], end_frame=end_frame, hits=hits, age=age, reason=reason, reserved=0,
                    quality=f32(b["q"]), score=f32(b["score"]), eye=f32(b["eye"]), frontal=f32(b["frontal"]),
                    sharpness=f32(b["sharpness"]), coverage=f32(b["coverage"]), face=b["face"].copy(), crop=b["crop"], M=b["M"])

    def update(self, video: int, tracks: List[dict], crops, mats, frame_w: int, frame_h: int) -> List[dict]:
        """One frame of `video`: the TrackerOracle.update output for it, and the u8 crop and M of each of the frame's records (indexed
        by record, i.e. rf_track.det).  Returns the frame's emissions in id order."""
        V = self._video(video)
        frame = V["frames"]
        now = {t["id"]: t for t in tracks}
        out = []
        for tid in sorted(V["live"]):
            if tid in now:
                continue
            prev = V["live"][tid]
            b = V["best"].pop(tid, None)
            if prev["state"] != TENTATIVE and b is not None and b["q"] >= self.min_q:
                out.append(self._shot(b, tid, video, frame, int(prev["hits"]), int(prev["age"]) + 1, BEST_EXIT))
        for t in tracks:
            j = int(t["det"])
            if j < 0:
                continue
            crop, M = np.asarray(crops[j]), np.asarray(mats[j], np.float64).reshape(2, 3)
            m = quality(crop, t["face"], M, frame_w, frame_h, self.template, self.sharp_half)
            b = V["best"].get(t["id"])
            if b is None or m["q"] > b["q"]:
                V["best"][t["id"]] = dict(m, frame=frame, face=np.asarray(t["face"], np.float32).copy(), crop=crop.copy(), M=M.copy())
        V["live"] = {t["id"]: dict(state=int(t["state"]), hits=int(t["hits"]), age=int(t["age"])) for t in tracks}
        V["frames"] = frame + 1
        return out

    def finish(self, video: int) -> List[dict]:
        """rf_tracker_finish: the shots of the live, ever-confirmed tracks in id order; the video then restarts."""
        V = self._video(video)
        out = []
        for tid in sorted(V["live"]):
            t = V["live"][tid]
            b = V["best"].get(tid)
            if t["state"] != TENTATIVE and b is not None and b["q"] >= self.min_q:
                out.append(self._shot(b, tid, video, V["frames"] - 1, t["hits"], t["age"], BEST_FINISH))
        self.reset(video)
        return out
