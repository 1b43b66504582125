"""f17 searching look-back without a GPU: oracle/lookback_search.py's chains against a literal per-step restatement over
oracle/follow.py's search (with and without motion, stopping, FLAT templates, frame 0 and resets), the chain on a synthetic fast face
against its true path, f15's regions kept exactly with (d) appended, rf_follow_config's bounds, the C layout and link of the new
symbols, the no-spill build of k_lookback_search and the C++ shell."""
import math
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from oracle.follow import FLAT, MISMATCH, OK, cut, search
from oracle.lookback import Frame, LookbackOracle, lookback_box
from oracle.lookback_search import SearchLookbackOracle, chain, undo_motion

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "retinaface_b200", "csrc")
FW, FH = 720, 360
SPEED = 40


def _texture(rng, h, w, sigma):
    return cv2.GaussianBlur(rng.integers(0, 256, (h, w)).astype(np.float32), (0, 0), sigma)


def _norm(a):
    a = a - a.min()
    return (a * (255.0 / max(a.max(), 1e-6))).astype(np.uint8)


def _fast_video(seed=0, n=12, w0=150.0, grow=1.03, x0=60.0):
    """Luma frames of a textured face patch crossing a faintly textured scene at SPEED px per frame, its size changing by `grow` per frame,
    and each frame's true box (float32 values)."""
    rng = np.random.default_rng(seed)
    # a face has far more structure than what lies behind it: the template's context (f16's margin) is scene, which stays put
    scene = (96 + _norm(_texture(rng, FH, FW, 8)) // 5).astype(np.uint8)
    face = _norm(_texture(rng, 256, 208, 6))
    frames, truth = [], []
    for t in range(n):
        w = w0 * grow ** t
        h = 1.25 * w
        cx, cy = x0 + SPEED * t + w / 2, 170.0
        x1, y1 = int(round(cx - w / 2)), int(round(cy - h / 2))
        pw, ph = int(round(w)), int(round(h))
        f = scene.copy()
        p = cv2.resize(face, (pw, ph), interpolation=cv2.INTER_AREA)
        xa, ya, xb, yb = max(x1, 0), max(y1, 0), min(x1 + pw, FW), min(y1 + ph, FH)
        if xb > xa and yb > ya:
            f[ya:yb, xa:xb] = p[ya - y1:yb - y1, xa - x1:xb - x1]
        frames.append(f)
        truth.append(tuple(float(np.float32(v)) for v in (x1, y1, x1 + pw, y1 + ph)))
    return frames, truth


def _iou(a, b):
    iw, ih = min(a[2], b[2]) - max(a[0], b[0]), min(a[3], b[3]) - max(a[1], b[1])
    if iw <= 0 or ih <= 0:
        return 0.0
    i = iw * ih
    return i / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - i)


def _literal_chain(luma_b, bid, face, lumas, motions, R, mad):
    """The definition step by step: the template of `face` on frame b, then each step from the last OK box, motion undone by f15's
    step 2 (here as lookback_box's formulas at g = 0.5: the box it returns is exactly the undone box), f16's search of the state."""
    tmpl, flat = cut(luma_b, [0.0] + list(face))
    box = [float(np.float32(v)) for v in face]
    out = []
    for k in range(1, len(lumas) + 1):
        x1, y1, x2, y2 = box
        w, h = x2 - x1, y2 - y1
        cx, cy = x1 + w / 2, y1 + h / 2
        mo = motions[k - 1]
        if mo is not None and mo[0] == 0:
            a, b, tx, ty = mo[1][0], mo[1][3], mo[1][2], mo[1][5]
            s2 = a * a + b * b
            cx, cy = (a * (cx - tx) + b * (cy - ty)) / s2, (a * (cy - ty) - b * (cx - tx)) / s2
            w, h = w / math.sqrt(s2), h / math.sqrt(s2)
        prev = np.zeros(15, np.float32)
        prev[1:5] = box
        rec, nf = search(lumas[k - 1], tmpl, flat, [cx, cy, w / h, h], [0.0] * 4, prev, R, mad)
        rec["id"] = bid
        out.append(rec)
        if rec["status"] != OK:
            break
        box = [float(nf[c]) for c in (1, 2, 3, 4)]
    return out


def _same_chain(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert {k: float(v) for k, v in g.items()} == {k: float(v) for k, v in w.items()}


@pytest.mark.parametrize("motion", [False, True])
def test_chain_equals_the_literal_steps(motion):
    frames, truth = _fast_video(1)
    b = 10
    rng = np.random.default_rng(3)
    mots = [None] * b
    if motion:      # small OK motions, one FIRST and one LOST on the way: only OK ones move the box
        mots = [(int(s), (1 + rng.uniform(-0.01, 0.01), -0.002, rng.uniform(-2, 2), 0.002, 1 + rng.uniform(-0.01, 0.01), rng.uniform(-2, 2)))
                for s in [0, 0, 1, 0, 2, 0, 0, 0, 0, 0]]
    lumas = [frames[b - k] for k in range(1, b + 1)]
    for R, mad in ((8, 24.0), (3, 24.0), (16, 2.0)):
        got = chain(frames[b], 7, truth[b], lumas, mots, R, mad)
        _same_chain(got, _literal_chain(frames[b], 7, truth[b], lumas, mots, R, mad))
        assert all(s["status"] == OK for s in got[:-1]) and all(s["id"] == 7 for s in got)
        if got[-1]["status"] != OK:
            assert len(got) <= b       # it stopped at its first failure


def test_undo_is_f15s_step():
    """undo_motion, then the growth at k, is exactly lookback_box's box: the same operations in the same order."""
    rng = np.random.default_rng(4)
    for _ in range(200):
        x, y, s = rng.uniform(0, 1800), rng.uniform(0, 900), rng.uniform(10, 300)
        face = tuple(float(np.float32(v)) for v in (x, y, x + s, y + 1.2 * s))
        m = (1 + rng.uniform(-0.1, 0.1), -0.03, rng.uniform(-50, 50), 0.03, 1 + rng.uniform(-0.1, 0.1), rng.uniform(-20, 20))
        w, h = face[2] - face[0], face[3] - face[1]
        cx, cy, w, h = undo_motion(face[0] + w / 2, face[1] + h / 2, w, h, m)
        g = 0.5 + 0.1 * 1
        mine = tuple(float(np.float32(v)) for v in (cx - g * w, cy - g * h, cx + g * w, cy + g * h))
        assert mine == lookback_box(face, 1, 0.1, [(0, m)])


def test_flat_template_stops_at_once_and_gives_no_region():
    flat = np.full((FH, FW), 128, np.uint8)
    st = chain(flat, 3, (100.0, 100.0, 200.0, 220.0), [flat] * 5, [None] * 5, 8, 24.0)
    assert len(st) == 1 and st[0]["status"] == FLAT
    o = SearchLookbackOracle(3)
    for t in range(5):
        births = [(1, (100.0, 100.0, 200.0, 220.0))] if t == 2 else []
        o.push(0, Frame(np.zeros(2, np.uint8), [], births, None), flat)
    plain = LookbackOracle(3)
    for t in range(5):
        plain.push(0, Frame(np.zeros(2, np.uint8), [], [(1, (100.0, 100.0, 200.0, 220.0))] if t == 2 else [], None))
    assert [e.boxes for e in o.drain(0)] == [e.boxes for e in plain.drain(0)]


def test_unbounded_and_empty_boxes_are_not_searched():
    luma = _fast_video(2)[0][5]
    for face in ((100.0, 100.0, 100.0, 220.0), (100.0, 100.0, 200.0, 100.0), (1e6, 100.0, 1e6 + 50, 160.0)):
        st = chain(luma, 1, face, [luma] * 3, [None] * 3, 8, 24.0)
        assert len(st) == 1 and st[0]["status"] in (MISMATCH, FLAT), (face, st)


def test_chains_stop_at_frame_0_and_at_a_reset():
    frames, truth = _fast_video(5, n=8)
    L = 6
    o = SearchLookbackOracle(L)
    for t in range(8):
        if t == 4:
            o.reset(0)              # numbering restarts: frame 4 is number 0
        births = [(t + 1, truth[t])] if t in (2, 5, 7) else []
        o.push(0, Frame(np.zeros(2, np.uint8), [], births, None), frames[t])
        ch = o.log[0][o.count[0] - 1 if t < 4 else (t - 4) % (2 * L)].chains
        num = t if t < 4 else t - 4
        for steps in ch:
            assert 1 <= len(steps) <= min(L, num) or (num == 0 and steps == [])
    # births on number 0 (frame 4 after the reset would be one, frame 0 before it) have no steps
    assert o.chains_of(0, 0, frames[0], [(9, truth[0])], None) == [[]]


def test_fast_face_chain_recovers_the_true_path():
    """A face 150 px wide crossing at 40 px per frame, 3 % larger every frame: the chain from its true box on frame b recovers the
    true box (IoU >= 0.7) on every step where the face is inside the frame, while f15's growth box misses part of the true box from
    some k <= 5 on."""
    frames, truth = _fast_video(0, n=10)
    b = 9
    lumas = [frames[b - k] for k in range(1, b + 1)]
    st = chain(frames[b], 1, truth[b], lumas, [None] * b, 8, 24.0)
    inside = [k for k in range(1, b + 1) if truth[b - k][0] >= 0 and truth[b - k][2] <= FW]
    assert inside and all(len(st) >= k and st[k - 1]["status"] == OK for k in inside), [s["status"] for s in st]
    for k in inside:
        s = st[k - 1]
        assert _iou((s["x1"], s["y1"], s["x2"], s["y2"]), truth[b - k]) >= 0.7, k
    miss = [k for k in range(1, 6) if not (lambda g, t: g[0] <= t[0] and g[1] <= t[1] and g[2] >= t[2] and g[3] >= t[3])(
        lookback_box(truth[b], k, 0.1), truth[b - k])]
    assert miss, "the growth box alone covers the face: the test video is too slow"


def _rand_log(rng, n, motion, frames):
    out, nid = [], 1
    for t in range(n):
        boxes = [tuple(float(np.float32(v)) for v in rng.uniform(0, 300, 4)) for _ in range(rng.integers(0, 3))]
        births = []
        for _ in range(rng.integers(0, 3)):
            x, y, s = rng.uniform(0, 400), rng.uniform(0, 150), rng.uniform(100, 180)
            births.append((nid, tuple(float(np.float32(v)) for v in (x, y, x + s, y + 1.2 * s))))
            nid += 1
        mo = None
        if motion:
            mo = (int(rng.choice([0, 0, 1, 2])), (1 + rng.uniform(-0.02, 0.02), -0.01, rng.uniform(-5, 5), 0.01, 1 + rng.uniform(-0.02, 0.02),
                                                 rng.uniform(-5, 5)))
        out.append((Frame(np.full(4, t, np.uint8), boxes, births, mo), frames[t % len(frames)]))
    return out


@pytest.mark.parametrize("L,motion", [(1, False), (4, True)])
def test_f15_regions_kept_and_d_appended(L, motion):
    """With chains present the first regions of every emitted frame are the unchanged f15 oracle's, and the rest are (d): each birth
    of frames e + 1 .. last, frame by frame, in births order, with its step b - e when that step is OK."""
    rng = np.random.default_rng(L)
    frames = _fast_video(6, n=6)[0]
    log = _rand_log(rng, 3 * L + 4, motion, frames)
    plain, srch = LookbackOracle(L), SearchLookbackOracle(L)
    for t, (fr, luma) in enumerate(log):
        a, b = plain.push(0, fr), srch.push(0, fr, luma)
        if a is None:
            assert b is None
            continue
        _check_emission(a, b, srch, L, t)
    drained = list(zip(plain.drain(0), srch.drain(0)))
    assert drained
    for a, b in drained:             # a drain's windows end at the last frame seen
        _check_emission(a, b, srch, L, len(log) - 1)


def _check_emission(a, b, o, L, last):
    assert b.number == a.number and np.array_equal(a.data, b.data)
    assert b.boxes[:len(a.boxes)] == a.boxes
    want = []
    for f in range(a.number + 1, last + 1):
        for steps in o.log[0][f % (2 * L)].chains:
            k = f - a.number
            if len(steps) >= k and steps[k - 1]["status"] == OK:
                want.append(tuple(float(np.float32(steps[k - 1][c])) for c in ("x1", "y1", "x2", "y2")))
    assert b.boxes[len(a.boxes):] == want


def test_config_bounds():
    from oracle.follow import config
    assert config() == (8, 24.0)
    for bad in ((17, 0.0), (-1, 0.0), (0, 256.0), (0, -1.0), (0, float("nan"))):
        with pytest.raises(ValueError):
            config(*bad)


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = capi.load_library()
    for s in ("rf_tracker_set_lookback_search", "rf_tracker_lookback_search"):
        assert hasattr(lib, s)
    src = tmp_path / "lbs.c"
    src.write_text('#include "rf_b200.h"\n#include <stddef.h>\n'
                   '_Static_assert(sizeof(rf_follow) == 48 && sizeof(rf_follow_config) == 8, "layout");\n'
                   'int main(void) {\n'
                   '    rf_follow_config c = {0, 0.f};\n'
                   '    const rf_follow *s; const int32_t *n;\n'
                   '    return rf_tracker_set_lookback_search(NULL, &c) == RF_ERR_INVALID_ARG &&\n'
                   '           rf_tracker_lookback_search(NULL, &s, &n) == RF_ERR_INVALID_ARG ? 0 : 1;\n'
                   '}\n')
    exe = tmp_path / "lbs"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L",
                           os.path.dirname(capi.lib_path()), "-lrf_b200", "-Wl,-rpath," + os.path.dirname(capi.lib_path())])
    assert subprocess.run([str(exe)]).returncode == 0


def test_kernel_builds_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "lookback_search.cu"), "-o",
                                                   str(tmp_path / "lbs.o")], capture_output=True, text=True, check=True)
    assert re.findall(r"Compiling entry function '\S*(k_lookback_search)", r.stderr) == ["k_lookback_search"]
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert spills and all(s == ("0", "0", "0") for s in spills), r.stderr


def test_host_shell_compiles_with_lookback_search(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    with open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.h")) as f:
        assert "bool lookback_search" in f.read()
