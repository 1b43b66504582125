"""f22 live best shots (rf_b200.h rf_tracker_set_best_live), restated on top of oracle/bestshot.py's BestShotOracle in Python doubles.

* ``live_config``         -- rf_best_live_config with its defaults applied and its bounds checked, in the values the policy compares.
* ``live_emits``          -- the policy of one matched CONFIRMED track on one frame, as a pure function.
* ``max_live_shots``      -- the bound on a track's live shots, 1 + floor(ln(1 / first_quality) / ln(1 + improve)).
* ``LiveBestShotOracle``  -- BestShotOracle plus the live state; ``live=None`` is BestShotOracle exactly.  Follow frames need nothing
                             new: ``update`` fed FollowTrackerOracle.follow's tracks (all det = -1) emits only the removals.
"""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np

from oracle.align import ARCFACE_112
from oracle.bestshot import BestShotOracle
from oracle.track import CONFIRMED

BEST_LIVE = 2


def live_config(first_quality: float = 0.0, improve: float = 0.0, min_gap: int = 0) -> dict:
    """(first_quality, 1 + improve, min_gap) as doubles / int, from the float32 fields of the C struct (0: the defaults)."""
    fq = float(np.float32(first_quality)) or float(np.float32(0.3))
    imp = float(np.float32(improve)) or float(np.float32(0.2))
    gap = int(min_gap) or 30
    if not (0.0 < fq <= 1.0):
        raise ValueError(f"first_quality {first_quality}")
    if not (math.isfinite(imp) and imp > 0.0):
        raise ValueError(f"improve {improve}")
    if not (1 <= gap <= 1 << 20):
        raise ValueError(f"min_gap {min_gap}")
    return dict(first_quality=fq, improve=imp, ratio=1.0 + imp, min_gap=gap)


def live_emits(q: float, n: int, q_l: float, e_l: int, frame: int, cfg: dict, min_quality: float) -> bool:
    """Whether a matched CONFIRMED track with stored best q and n live shots so far (the last one q_l, on frame e_l) emits on frame."""
    if n == 0:
        return q >= cfg["first_quality"] and q >= min_quality
    return frame - e_l >= cfg["min_gap"] and q > q_l * cfg["ratio"]


def max_live_shots(cfg: dict) -> int:
    return 1 + math.floor(math.log(1.0 / cfg["first_quality"]) / math.log(cfg["ratio"]))


class LiveBestShotOracle(BestShotOracle):
    """BestShotOracle with the f22 live policy (``live``: ``live_config``'s keywords, or None for none)."""

    def __init__(self, min_quality: float = 0.0, sharp_half: float = 0.0, template=ARCFACE_112, live: Optional[dict] = None):
        super().__init__(min_quality, sharp_half, template)
        self.live = None if live is None else live_config(**live)

    def reset(self, video: int):
        super().reset(video)
        self.v[video]["shots"] = {}          # id -> (n, q_l, e_l)

    def update(self, video: int, tracks: List[dict], crops, mats, frame_w: int, frame_h: int) -> List[dict]:
        frame = self._video(video)["frames"]
        out = super().update(video, tracks, crops, mats, frame_w, frame_h)
        if self.live is None:
            return out
        V = self.v[video]
        now = {t["id"] for t in tracks}
        V["shots"] = {i: s for i, s in V["shots"].items() if i in now}
        for t in tracks:
            if int(t["det"]) < 0 or int(t["state"]) != CONFIRMED:
                continue
            tid = int(t["id"])
            b = V["best"][tid]
            n, q_l, e_l = V["shots"].get(tid, (0, 0.0, 0))
            if live_emits(b["q"], n, q_l, e_l, frame, self.live, self.min_q):
                out.append(self._shot(b, tid, video, frame, int(t["hits"]), int(t["age"]), BEST_LIVE))
                V["shots"][tid] = (n + 1, b["q"], frame)
        out.sort(key=lambda s: s["id"])
        return out
