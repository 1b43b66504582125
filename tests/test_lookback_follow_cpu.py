"""f18 following look-back without a GPU: oracle/lookback_follow.py against a literal restatement over plain per-frame lists (emitted
numbers, region order, drain and reset; k = 2, 3, 5 and L = 1, 4, 15, with and without motion and search); a face revealed on a follow
frame covered from the reveal on when L >= k - 1 and not when L < k - 1; rf_follow_config's bounds, the C layout and link of the new
symbols, the no-spill build of the look-back kernels and the C++ shell with lookback and detect_every together."""
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from oracle.follow import OK
from oracle.lookback import lookback_box, regions
from oracle.lookback_follow import LookbackFollowOracle
from oracle.lookback_search import chain
from oracle.redact import RF_TRACK_LOST, params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "retinaface_b200", "csrc")
FW, FH = 320, 240
GROW = float(np.float32(0.1))


def _texture(rng, h, w, sigma):
    a = cv2.GaussianBlur(rng.integers(0, 256, (h, w)).astype(np.float32), (0, 0), sigma)
    a -= a.min()
    return (a * (255.0 / max(a.max(), 1e-6))).astype(np.uint8)


def _video(seed, n, faces):
    """n luma frames of a faint scene with textured faces; faces: (first frame, x0, y0, size, dx per frame).  Returns the frames and
    per frame the true boxes of the faces in view."""
    rng = np.random.default_rng(seed)
    scene = (96 + _texture(rng, FH, FW, 6) // 6).astype(np.uint8)
    patches = [_texture(rng, int(1.25 * s), s, 3) for _, _, _, s, _ in faces]
    frames, truth = [], []
    for t in range(n):
        f = scene.copy()
        boxes = []
        for (t0, x0, y0, s, dx), p in zip(faces, patches):
            if t < t0:
                continue
            x = int(x0 + dx * (t - t0))
            h = p.shape[0]
            if x < 0 or x + s > FW:
                continue
            f[y0:y0 + h, x:x + s] = p
            boxes.append((float(x), float(y0), float(x + s), float(y0 + h)))
        frames.append(f)
        truth.append(boxes)
    return frames, truth


def _records(boxes):
    """The detector's records of a key frame: each true box, score 0.9, landmarks inside it, in frame pixels (scale 1)."""
    r = np.zeros((len(boxes), 15), np.float32)
    for j, (x1, y1, x2, y2) in enumerate(boxes):
        r[j, :5] = (0.9, x1, y1, x2, y2)
        r[j, 5:10] = np.linspace(x1 + 0.3 * (x2 - x1), x2 - 0.3 * (x2 - x1), 5)
        r[j, 10:15] = np.linspace(y1 + 0.4 * (y2 - y1), y2 - 0.3 * (y2 - y1), 5)
    return r


def _motion(rng):
    return (int(rng.choice([0, 0, 1, 2])), (1 + rng.uniform(-0.02, 0.02), -0.01, rng.uniform(-3, 3), 0.01, 1 + rng.uniform(-0.02, 0.02),
                                            rng.uniform(-3, 3)))


class _Literal:
    """The definition over plain lists: per video since its restart, each frame's (data, (a) + (b) boxes, births, motion, luma)."""

    def __init__(self, L, search):
        self.L, self.search, self.f = L, search, []

    def push(self, data, ab, births, motion, luma):
        self.f.append((data, ab, births, motion, luma))
        num = len(self.f) - 1
        return None if num < self.L else self.emit(num - self.L, num)

    def emit(self, e, last):
        boxes = list(self.f[e][1])
        for b in range(e + 1, min(e + self.L, last) + 1):            # (c), motion undone frame by frame from b down to e + 1
            for _, face in self.f[b][2]:
                mot = [self.f[g][3] for g in range(b, e, -1)]
                boxes.append(lookback_box(face, b - e, GROW, [] if mot[0] is None else mot))
        if self.search:                                               # (d): the birth's step b - e, when OK
            for b in range(e + 1, min(e + self.L, last) + 1):
                K = min(self.L, b)
                lumas = [self.f[b - q][4] for q in range(1, K + 1)]
                mots = [self.f[b - q + 1][3] for q in range(1, K + 1)]
                for bid, face in self.f[b][2]:
                    steps = chain(self.f[b][4], bid, face, lumas, mots, 8, 24.0)
                    if len(steps) >= b - e and steps[b - e - 1]["status"] == OK:
                        boxes.append(tuple(float(np.float32(steps[b - e - 1][c])) for c in ("x1", "y1", "x2", "y2")))
        return e, self.f[e][0], boxes

    def drain(self):
        n = len(self.f)
        out = [self.emit(e, n - 1) for e in range(max(0, n - self.L), n)]
        self.f = []
        return out


def _lists_ab(kind, records, tracks):
    lost = [tuple(float(t[c]) for c in ("kx1", "ky1", "kx2", "ky2")) for t in tracks if int(t["state"]) == RF_TRACK_LOST]
    if kind == "detect":
        return [tuple(float(v) for v in r[1:5]) for r in records] + lost, [
            (int(t["id"]), tuple(float(v) for v in t["face"][1:5])) for t in tracks if int(t["age"]) == 1]
    return [tuple(float(np.float32(v)) for v in t["face"][1:5]) for t in tracks if int(t["followed"])] + lost, []


@pytest.mark.parametrize("motion,search", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("L", [1, 4, 15])
@pytest.mark.parametrize("k", [2, 3, 5])
def test_composed_oracle_equals_the_literal_definition(k, L, motion, search):
    rng = np.random.default_rng(100 * k + L)
    n = 2 * L + 12
    frames, truth = _video(k, n, [(0, 20, 40, 56, 3), (k + 1, 200, 100, 64, -2), (2 * k + 3, 120, 20, 48, 0)])
    o = LookbackFollowOracle(1, L, search={} if search else None)
    lit = _Literal(L, search)
    # a drain mid-interval, frames again, a reset mid-interval, frames again, a final drain
    plan = [("frames", range(0, L + 5)), ("drain", None), ("frames", range(L + 5, 2 * L + 8)), ("reset", None),
            ("frames", range(2 * L + 8, n)), ("drain", None)]
    emitted = follows = 0
    for what, rg in plan:
        if what == "drain":
            got, want = o.drain(0), lit.drain()
            assert [(e.number, e.boxes) for e in got] == [(w[0], w[2]) for w in want]
            assert all(np.array_equal(e.data, w[1]) for e, w in zip(got, want))
            continue
        if what == "reset":
            o.reset(0)
            lit.f = []
            continue
        for num, t in enumerate(rg):
            data = frames[t] // 2 + num             # the bytes an emitted frame carries
            mot = _motion(rng) if motion else None
            if num % k == 0:
                rec = _records(truth[t])
                tracks, em = o.detect(0, data, frames[t], rec, None, mot)
                ab, births = _lists_ab("detect", rec, tracks)
            else:
                tracks, _, em = o.follow(0, data, frames[t], mot)
                ab, births = _lists_ab("follow", None, tracks)
                assert births == [] and all(int(r["age"]) > 1 for r in tracks)
                follows += sum(int(r["followed"]) for r in tracks)
            want = lit.push(data, ab, births, mot, frames[t])
            assert (em is None) == (want is None), (t, num)
            if em is not None:
                assert (em.number, em.boxes) == (want[0], want[2]) and np.array_equal(em.data, want[1]), (t, num)
                emitted += 1
    assert emitted > 0 and follows > 0


def _covered(box, em, m, b):
    x1, y1, x2, y2 = box
    return any(X0 <= x1 and Y0 <= y1 and X1 >= x2 and Y1 >= y2 for X0, Y0, X1, Y1, _ in regions(em.boxes, m, b))


@pytest.mark.parametrize("k,L", [(3, 2), (5, 4), (5, 6), (5, 2), (3, 1)])
def test_face_revealed_on_a_follow_frame(k, L):
    """A still face revealed on a follow frame r and first detected on the next key frame b: with L >= k - 1 every out frame from r on
    covers its true box with a region's rectangle; with L < k - 1 the frames before b - L go out uncovered."""
    r = k + 1                                       # a follow frame (k + 1 is not a multiple of k for k >= 2)
    n = 4 * k + L + 2
    frames, truth = _video(7, n, [(r, 140, 60, 60, 0)])
    o = LookbackFollowOracle(1, L)
    bb, mm = params(0, 0.0)
    ems = {}
    for t in range(n):
        if t % k == 0:
            _, em = o.detect(0, frames[t], frames[t], _records(truth[t]), None)
        else:
            _, _, em = o.follow(0, frames[t], frames[t])
        if em is not None:
            ems[em.number] = em
    for em in o.drain(0):
        ems[em.number] = em
    b = -(-r // k) * k
    uncovered = [e for e in range(r, n) if not _covered(truth[e][0], ems[e], mm, bb)]
    if L >= k - 1:
        assert uncovered == [], (k, L, b, uncovered)
    else:
        assert uncovered and all(e < b - L for e in uncovered), (k, L, b, uncovered)


def test_config_bounds():
    from oracle.follow import config
    assert config() == (8, 24.0)
    for bad in ((17, 0.0), (-1, 0.0), (0, 256.0), (0, -1.0), (0, float("nan"))):
        with pytest.raises(ValueError):
            config(*bad)


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = capi.load_library()
    for s in ("rf_tracker_set_lookback_follow", "rf_track_follow_redact_lookback_device"):
        assert hasattr(lib, s) and s in capi.EXPORTS
    src = tmp_path / "lbf.c"
    src.write_text('#include "rf_b200.h"\n#include <stddef.h>\n'
                   '_Static_assert(sizeof(rf_follow_config) == 8 && sizeof(rf_follow) == 48, "layout");\n'
                   'int main(void) {\n'
                   '    rf_follow_config c = {0, 0.f};\n'
                   '    rf_yuv_frame f = {0}, o = {0};\n'
                   '    int v = 0; int32_t num = 0;\n'
                   '    const rf_track *tr; const int32_t *tc;\n'
                   '    return rf_tracker_set_lookback_follow(NULL, &c) == RF_ERR_INVALID_ARG &&\n'
                   '           rf_track_follow_redact_lookback_device(NULL, &f, &v, 1, NULL, &o, &num, &tr, &tc) == RF_ERR_INVALID_ARG ? 0 : 1;\n'
                   '}\n')
    exe = tmp_path / "lbf"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L",
                           os.path.dirname(capi.lib_path()), "-lrf_b200", "-Wl,-rpath," + os.path.dirname(capi.lib_path())])
    assert subprocess.run([str(exe)]).returncode == 0


def test_lookback_kernels_build_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "lookback.cu"), "-o",
                                                   str(tmp_path / "lb.o")], capture_output=True, text=True, check=True)
    names = re.findall(r"Compiling entry function '\S*(k_lookback_\w+?)E", r.stderr)
    assert sorted(set(names)) == ["k_lookback_boxes", "k_lookback_log", "k_lookback_swap"], names
    spills = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(spills) == 3 and all(s == ("0", "0", "0") for s in spills), r.stderr


def test_host_shell_combines_lookback_and_detect_every(built_lib, tmp_path):
    """A user's program setting RedactOptions::lookback together with RetinaFaceOptions::detect_every compiles and links."""
    from retinaface_b200.build import HERE, build_host
    assert os.path.exists(build_host())
    host = os.path.join(HERE, "host")
    src = tmp_path / "user.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    if (argc < 2) return 0;\n'
                   '    string model = argv[1];\n'
                   '    RetinaFaceOptions opt;\n'
                   '    opt.detect_every = 3;\n'
                   '    RetinaFace rf(model, "net3", 0.4f, opt);\n'
                   '    vector<rf_yuv_frame> frames(4), outs(4);\n'
                   '    vector<int> videos(4, 0);\n'
                   '    RedactOptions ro;\n'
                   '    ro.lookback = 2;\n'
                   '    ro.style = RF_REDACT_BLUR;\n'
                   '    rf.redactYUV(frames, &videos, 0.5f, ro, &outs);\n'
                   '    const vector<int32_t> &nums = rf.lastFrameNumbers();\n'
                   '    return (int)nums.size() + (int)rf.drainVideo(0, outs, ro).size();\n'
                   '}\n')
    exe = tmp_path / "user"
    subprocess.check_call(["g++", "-std=c++14", "-O0", "-I", host, "-I", os.path.join(ROOT, "include"), str(src),
                           os.path.join(host, "RetinaFace.cpp"), "-o", str(exe), "-L", HERE, "-lrf_b200", "-Wl,-rpath," + HERE])
    assert subprocess.run([str(exe)]).returncode == 0          # no model: it only shows the program runs to its first line
