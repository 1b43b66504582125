"""f18 following look-back restated (rf_b200.h rf_tracker_set_lookback_follow): oracle/follow.py's FollowTrackerOracle, unchanged,
tracks the detect and follow frames; oracle/lookback.py's LookbackOracle (or oracle/lookback_search.py's SearchLookbackOracle on a
searching tracker), unchanged, buffers, emits, drains and resets.

What each frame logs:
    detect frame   Frame(data, frame_boxes(records, count, scale, tracks), births(tracks), motion) -- f15's, as on a look-back tracker;
    follow frame   Frame(data, every OK-followed face's box in id order + every LOST track's box in id order, [], motion) -- what
                   f16's redaction draws on the frame, and no births.
Detect and follow frames share each video's count, so emission, the (c) motion chain and f17's (d) steps run through both kinds.
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from oracle.follow import FollowTrackerOracle
from oracle.lookback import Box, Emitted, Frame, LookbackOracle, births, frame_boxes
from oracle.lookback_search import SearchLookbackOracle
from oracle.redact import RF_TRACK_LOST


def follow_boxes(tracks) -> List[Box]:
    """A follow frame's (a) + (b): the OK-followed faces (followed == 1) in id order, then the LOST tracks in id order."""
    ok = [tuple(float(np.float32(v)) for v in t["face"][1:5]) for t in tracks if int(t["followed"])]
    lost = [tuple(float(t[f]) for f in ("kx1", "ky1", "kx2", "ky2")) for t in tracks if int(t["state"]) == RF_TRACK_LOST]
    return ok + lost


def detect_frame(data: np.ndarray, records: np.ndarray, count: int, scale: Optional[float], tracks, motion=None) -> Frame:
    return Frame(data, frame_boxes(records, count, scale, tracks), births(tracks), motion)


def follow_frame(data: np.ndarray, tracks, motion=None) -> Frame:
    return Frame(data, follow_boxes(tracks), [], motion)


class LookbackFollowOracle:
    """A following look-back tracker of max_videos videos.  motion (status, m) is the frame's rf_motion as the log keeps it, applied
    its oracle/motion.py `applied` form for the tracker (both None without motion); luma is the frame's Y plane."""

    def __init__(self, max_videos: int = 1, frames: int = 0, grow: float = 0.0, search: Optional[dict] = None,
                 follow: Optional[dict] = None, **cfg):
        self.tracker = FollowTrackerOracle(max_videos, **(follow or {}), **cfg)
        self.searching = search is not None
        self.lookback = SearchLookbackOracle(frames, grow, **search) if self.searching else LookbackOracle(frames, grow)

    def _push(self, video: int, frame: Frame, luma: np.ndarray) -> Optional[Emitted]:
        return self.lookback.push(video, frame, luma) if self.searching else self.lookback.push(video, frame)

    def detect(self, video: int, data: np.ndarray, luma: np.ndarray, records: np.ndarray, scale: Optional[float], motion=None,
               applied=None):
        """A detect frame: (the tracker's lists, what the frame emits or None)."""
        tracks = self.tracker.update(video, records, scale, motion=applied, luma=luma)
        return tracks, self._push(video, detect_frame(data, records, len(records), scale, tracks, motion), luma)

    def follow(self, video: int, data: np.ndarray, luma: np.ndarray, motion=None, applied=None):
        """A follow frame: (the tracker's lists, the rf_follow records, what the frame emits or None)."""
        tracks, recs = self.tracker.follow(video, luma, motion=applied)
        return tracks, recs, self._push(video, follow_frame(data, tracks, motion), luma)

    def drain(self, video: int) -> List[Emitted]:
        out = self.lookback.drain(video)
        self.tracker.reset(video)
        return out

    def reset(self, video: int) -> None:
        self.lookback.reset(video)
        self.tracker.reset(video)

