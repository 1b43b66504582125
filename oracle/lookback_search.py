"""f17 searching look-back restated in Python doubles (rf_b200.h rf_tracker_set_lookback_search), on top of oracle/lookback.py (f15's
frames, births, regions (a) (b) (c) and emission, unchanged) and oracle/follow.py (f16's cut and search, called as they are).

Chain of a birth on frame b with record box `face`: the template is f16's cut of `face` on frame b's luma; step k = 1 .. min(L, b)
searches frame e = b - k from the box of step k - 1 (`face` at k = 1):
    w = x2 - x1, h = y2 - y1, cx = x1 + w / 2, cy = y1 + h / 2
    with motion, frame e + 1's motion undone when OK (f15's step 2, the formulas of oracle/lookback.py's lookback_box)
    f16's search of the state (cx, cy, w / h, h) with zero velocity and no motion (pw = (w / h) h)
and the chain stops at the first status other than OK.  Regions of an emitted frame e: f15's, then (d) the box of step b - e of every
birth on frames e + 1 .. min(e + L, last) whose chain reached that step OK, frame by frame, id order within a frame.
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from oracle.follow import MISMATCH, OK, config as follow_config, cut, search
from oracle.lookback import MOTION_OK, Box, Emitted, LookbackOracle


def undo_motion(cx: float, cy: float, w: float, h: float, m: Sequence[float]) -> Tuple[float, float, float, float]:
    """One OK camera motion {a, -B, tx, B, a, ty} undone, as f15's step 2 states it."""
    a, b, tx, ty = float(m[0]), float(m[3]), float(m[2]), float(m[5])
    s2 = a * a + b * b
    dx, dy = cx - tx, cy - ty
    cx, cy = (a * dx + b * dy) / s2, (a * dy - b * dx) / s2
    s = math.sqrt(s2)
    return cx, cy, w / s, h / s


def unsearched(bid: int, status: int) -> dict:
    return dict(id=bid, status=status, dx=0, dy=0, scale=0, sad=0, fx=0.0, fy=0.0, x1=0.0, y1=0.0, x2=0.0, y2=0.0)


def chain(luma_b: np.ndarray, bid: int, face: Box, lumas: Sequence[np.ndarray], motions: Sequence, R: int, max_mad: float) -> List[dict]:
    """The rf_follow records of a birth's chain.  lumas[k - 1]: frame b - k's luma (len K); motions[k - 1]: frame b - k + 1's (status,
    m) or None without motion."""
    x1, y1, x2, y2 = (float(np.float32(v)) for v in face[:4])
    tmpl, flat = cut(luma_b, [0.0, x1, y1, x2, y2])
    steps: List[dict] = []
    for k, luma in enumerate(lumas, 1):
        w, h = x2 - x1, y2 - y1
        cx, cy = x1 + w / 2.0, y1 + h / 2.0
        mo = motions[k - 1]
        if mo is not None and int(mo[0]) == MOTION_OK:
            cx, cy, w, h = undo_motion(cx, cy, w, h, mo[1])
        if h == 0.0:          # w / h is infinite or NaN on the device: pw leaves the bound, not searched
            steps.append(unsearched(bid, MISMATCH))
            break
        prev = np.zeros(15, np.float32)
        prev[1:5] = (x1, y1, x2, y2)
        rec, nf = search(luma, tmpl, flat, [cx, cy, w / h, h], [0.0, 0.0, 0.0, 0.0], prev, R, max_mad, None)
        rec["id"] = bid
        steps.append(rec)
        if rec["status"] != OK:
            break
        x1, y1, x2, y2 = (float(nf[c]) for c in (1, 2, 3, 4))
    return steps


class SearchFrame(NamedTuple):
    """oracle/lookback.py's Frame plus each birth's chain (in births order)."""
    data: np.ndarray
    boxes: List[Box]
    births: List[Tuple[int, Box]]
    motion: Optional[Tuple[int, Sequence[float]]]
    chains: List[List[dict]]


class SearchLookbackOracle(LookbackOracle):
    """LookbackOracle with f17's chains: push() takes the frame's luma as well and computes the chains of its births before the frame
    enters the buffer (the device's order: search, then swap)."""

    def __init__(self, frames: int = 0, grow: float = 0.0, search: int = 0, max_mad: float = 0.0):
        super().__init__(frames, grow)
        self.R, self.max_mad = follow_config(search, max_mad)
        self.lumas: Dict[int, Dict[int, np.ndarray]] = {}

    def chains_of(self, video: int, num: int, luma: np.ndarray, births, motion) -> List[List[dict]]:
        L, K = self.L, min(self.L, num)
        lumas = [self.lumas[video][(num - k) % L] for k in range(1, K + 1)]
        mots = [motion if f == num else self.log[video][f % (2 * L)].motion for f in range(num, num - K, -1)]
        return [chain(luma, bid, face, lumas, mots, self.R, self.max_mad) for bid, face in births]

    def push(self, video: int, frame, luma: np.ndarray = None) -> Optional[Emitted]:
        num = self.count.get(video, 0)
        chains = self.chains_of(video, num, luma, frame.births, frame.motion)
        out = super().push(video, SearchFrame(frame.data, frame.boxes, frame.births, frame.motion, chains))
        self.lumas.setdefault(video, {})[num % self.L] = np.array(luma, copy=True)
        return out

    def _emit(self, video: int, e: int, last: int) -> Emitted:
        out = super()._emit(video, e, last)
        boxes = list(out.boxes)
        for b in range(e + 1, last + 1):
            for steps in self.log[video][b % (2 * self.L)].chains:
                k = b - e
                if len(steps) >= k and steps[k - 1]["status"] == OK:
                    s = steps[k - 1]
                    boxes.append(tuple(float(np.float32(s[c])) for c in ("x1", "y1", "x2", "y2")))
        return Emitted(out.video, out.number, out.data, boxes)
