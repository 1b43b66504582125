"""f15 look-back redaction restated in Python doubles (rf_b200.h rf_detect_yuv_redact_lookback_device): which frame each call emits,
the look-back box of every birth, and the regions of an emitted frame, on top of oracle/redact.py's geometry and
oracle/redact_style.py's styles.

Each video numbers its frames from 0 since create, reset or drain.  Frame num emits frame num - L once num >= L; a drain emits the
last min(L, frames) buffered frames.  An emitted frame e is redacted, over its ORIGINAL bytes, with the regions
    (a) its records in rank order, __fmul_rn(x, scale);  (b) its LOST tracks in id order, (kx1, ky1, kx2, ky2);
    (c) the look-back boxes of the births (tracks with age == 1, id order) on frames e + 1 .. min(e + L, last frame seen), frame by frame.
Look-back box of a birth on frame b at k = b - e frames back, every FP64 step one rounding (Python floats):
    w = x2 - x1, h = y2 - y1, cx = x1 + w / 2, cy = y1 + h / 2
    with motion, for f = b, b - 1, ..., e + 1 and frame f's {a, -B, tx, B, a, ty} of status OK: s2 = a a + B B, dx = cx - tx,
        dy = cy - ty, cx = (a dx + B dy) / s2, cy = (a dy - B dx) / s2, s = sqrt(s2), w = w / s, h = h / s
    g = 0.5 + grow k, ex = g w, ey = g h; the box (cx - ex, cy - ey, cx + ex, cy + ey), each rounded to float32.
LookbackOracle keeps, like the device, each video's last L frames in a ring of L slots and its last 2 L frames' logs.
"""
from __future__ import annotations

import math
from typing import Dict, List, NamedTuple, Optional, Sequence, Tuple

import numpy as np

from oracle.redact import RF_TRACK_LOST, geometry, yuv_planes

DEFAULT_FRAMES, MAX_FRAMES = 15, 64
MOTION_OK = 0

Box = Tuple[float, float, float, float]     # float32 values, frame pixels


def config(frames: int = 0, grow: float = 0.0) -> Tuple[int, float]:
    """rf_lookback_config with the defaults applied: (L, grow as the float32 the struct holds, widened).  Bad values: ValueError."""
    L = frames or DEFAULT_FRAMES
    g = float(np.float32(grow or 0.1))
    if not 1 <= L <= MAX_FRAMES:
        raise ValueError(f"frames {frames}: 0 or 1..{MAX_FRAMES}")
    if not (math.isfinite(g) and 0.0 < g <= 1.0):
        raise ValueError(f"grow {grow}: 0 or finite in (0, 1]")
    return L, g


def lookback_box(face: Sequence[float], k: int, grow: float, motions: Sequence[Tuple[int, Sequence[float]]] = ()) -> Box:
    """The look-back box of a birth with record box `face` (x1, y1, x2, y2) k frames back.  motions: (status, m[6]) of frames
    b, b - 1, ..., e + 1 (k of them), or empty without motion."""
    x1, y1, x2, y2 = (float(np.float32(v)) for v in face[:4])
    w, h = x2 - x1, y2 - y1
    cx, cy = x1 + w / 2.0, y1 + h / 2.0
    for status, m in motions:
        if status != MOTION_OK:
            continue
        a, b, tx, ty = float(m[0]), float(m[3]), float(m[2]), float(m[5])
        s2 = a * a + b * b
        dx, dy = cx - tx, cy - ty
        cx, cy = (a * dx + b * dy) / s2, (a * dy - b * dx) / s2
        s = math.sqrt(s2)
        w, h = w / s, h / s
    g = 0.5 + grow * float(k)
    ex, ey = g * w, g * h
    return tuple(float(np.float32(v)) for v in (cx - ex, cy - ey, cx + ex, cy + ey))


def frame_boxes(faces: np.ndarray, count: int, scale: Optional[float], tracks=None, max_faces: Optional[int] = None) -> List[Box]:
    """A frame's (a) + (b) boxes as floats: its records in rank order times scale (float32 products), then its LOST tracks."""
    faces = np.asarray(faces, np.float32)
    k = min(int(count), faces.shape[0] if max_faces is None else max_faces)
    s = np.float32(1.0 if scale is None else scale)
    out = [tuple(float(np.float32(faces[j, c]) * s) for c in (1, 2, 3, 4)) for j in range(k)]
    for t in (tracks if tracks is not None else ()):
        if int(t["state"]) == RF_TRACK_LOST:
            out.append(tuple(float(t[f]) for f in ("kx1", "ky1", "kx2", "ky2")))
    return out


def births(tracks) -> List[Tuple[int, Box]]:
    """(id, face box) of every track born on the frame (age == 1), in list (id) order."""
    return [(int(t["id"]), tuple(float(v) for v in t["face"][1:5])) for t in (tracks if tracks is not None else ()) if int(t["age"]) == 1]


def regions(boxes: Sequence[Box], margin: float, blocks: int):
    """f12's snapped regions of the boxes, skipped boxes dropped."""
    out = []
    for b in boxes:
        g = geometry(*b, margin, blocks)
        if g is not None:
            out.append(g)
    return out


class Frame(NamedTuple):
    """What the log keeps of one frame: its original bytes, its (a) + (b) boxes, its births and its motion (status, m) or None."""
    data: np.ndarray
    boxes: List[Box]
    births: List[Tuple[int, Box]]
    motion: Optional[Tuple[int, Sequence[float]]]


class Emitted(NamedTuple):
    video: int
    number: int
    data: np.ndarray          # the frame's original bytes
    boxes: List[Box]          # (a) + (b) + (c)


class LookbackOracle:
    """The device's per-video state: a frame counter, the frame bytes in L slots (num mod L) and the log in 2 L slots (num mod 2 L)."""

    def __init__(self, frames: int = 0, grow: float = 0.0):
        self.L, self.grow = config(frames, grow)
        self.count: Dict[int, int] = {}
        self.buf: Dict[int, Dict[int, np.ndarray]] = {}
        self.log: Dict[int, Dict[int, Frame]] = {}

    def _emit(self, video: int, e: int, last: int) -> Emitted:
        L, log = self.L, self.log[video]
        boxes = list(log[e % (2 * L)].boxes)
        for b in range(e + 1, last + 1):
            for _, face in log[b % (2 * L)].births:
                mot = [log[f % (2 * L)].motion for f in range(b, e, -1)]
                boxes.append(lookback_box(face, b - e, self.grow, [] if mot[0] is None else mot))
        return Emitted(video, e, self.buf[video][e % L], boxes)

    def push(self, video: int, frame: Frame) -> Optional[Emitted]:
        """One frame of a call, in call order; returns what it emits (frame num - L) or None."""
        num = self.count.get(video, 0)
        self.count[video] = num + 1
        self.log.setdefault(video, {})[num % (2 * self.L)] = frame
        buf = self.buf.setdefault(video, {})
        out = None
        if num >= self.L:
            out = self._emit(video, num - self.L, num)
        buf[num % self.L] = np.array(frame.data, copy=True)
        return out

    def drain(self, video: int) -> List[Emitted]:
        """rf_tracker_drain: the last min(L, frames) frames in frame order, windows ending at the last frame seen; then the video restarts."""
        n = self.count.get(video, 0)
        out = [self._emit(video, e, n - 1) for e in range(max(0, n - self.L), n)]
        self.reset(video)
        return out

    def reset(self, video: int) -> None:
        self.count[video] = 0


def emit_into(out: np.ndarray, data: np.ndarray, layout: str, **surface) -> np.ndarray:
    """A copy of the out frame buffer `out` with the planes of `data` (the same layout and surface keywords as `out`, or a packed
    buffer when `data_surface` is given) written over its planes; its pitch padding stays."""
    src_surface = surface.pop("data_surface", surface)
    res = np.array(out, np.uint8, copy=True)
    for (d, _), (s, _) in zip(yuv_planes(res, layout, **surface), yuv_planes(np.asarray(data), layout, **src_surface)):
        d[...] = s
    return res
