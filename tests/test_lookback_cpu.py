"""f15 look-back redaction without a GPU: oracle/lookback.py against a literal restatement of the definition (emitted numbers, windows,
region order, drain and reset), the look-back box against exact rational arithmetic rounded once per step, the inverse-motion chain
against composed 3 x 3 inverses, rf_lookback_config, the C layout and link, the no-spill build and the C++ shell."""
import ctypes as C
import math
import os
import re
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from oracle.lookback import Frame, LookbackOracle, config, lookback_box

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "retinaface_b200", "csrc")


def _rand_frames(rng, n, motion):
    """n synthetic log frames: bytes, 0-3 (a)+(b) boxes, 0-2 births with rising ids, and a motion (OK, FIRST or LOST) or None."""
    out, nid = [], 1
    for t in range(n):
        boxes = [tuple(float(np.float32(v)) for v in rng.uniform(0, 500, 4)) for _ in range(rng.integers(0, 4))]
        births = []
        for _ in range(rng.integers(0, 3)):
            x, y, s = rng.uniform(0, 800), rng.uniform(0, 400), rng.uniform(20, 150)
            births.append((nid, tuple(float(np.float32(v)) for v in (x, y, x + s, y + 1.2 * s))))
            nid += 1
        mo = None
        if motion:
            a, b = 1 + rng.uniform(-0.05, 0.05), rng.uniform(-0.03, 0.03)
            mo = (int(rng.choice([0, 0, 0, 1, 2])), (a, -b, rng.uniform(-30, 30), b, a, rng.uniform(-10, 10)))
        out.append(Frame(np.full(4, t, np.uint8), boxes, births, mo))
    return out


def _literal(frames, L, grow, e, last):
    """The regions of emitted frame e, straight from the definition: e's boxes, then for b = e + 1 .. last every birth's box."""
    boxes = list(frames[e].boxes)
    for b in range(e + 1, last + 1):
        for _, face in frames[b].births:
            chain = [frames[f].motion for f in range(b, e, -1)] if frames[b].motion is not None else []
            boxes.append(lookback_box(face, b - e, grow, chain))
    return boxes


@pytest.mark.parametrize("L,motion", [(1, False), (3, True), (15, True), (64, False)])
def test_oracle_equals_the_literal_definition(L, motion):
    """Two interleaved videos pushed frame by frame, one reset and one drain: every emission's number, bytes and box list equal the
    literal restatement over plain lists of frames."""
    rng = np.random.default_rng(L)
    grow = config(L, 0.0)[1]
    o = LookbackOracle(L)
    vids = {0: _rand_frames(rng, 3 * L + 5, motion), 1: _rand_frames(rng, 2 * L + 3, motion)}
    seen = {0: [], 1: []}
    order = [0] * (L + 2) + [1, 0] * (2 * L + 3) + [0] * (3 * L + 5)
    pos = {0: 0, 1: 0}
    for v in order:
        if pos[v] >= len(vids[v]):
            continue
        if v == 1 and pos[v] == L + 1:          # a reset in the middle of video 1: it starts again at frame 0
            o.reset(1)
            seen[1] = []
        f = vids[v][pos[v]]
        pos[v] += 1
        seen[v].append(f)
        num = len(seen[v]) - 1
        got = o.push(v, f)
        if num < L:
            assert got is None
            continue
        e = num - L
        assert got.number == e and got.video == v
        assert np.array_equal(got.data, seen[v][e].data)
        assert got.boxes == _literal(seen[v], L, grow, e, num), (L, v, e)
    for v in (0, 1):
        n = len(seen[v])
        got = o.drain(v)
        assert [g.number for g in got] == list(range(max(0, n - L), n))
        for g in got:
            assert np.array_equal(g.data, seen[v][g.number].data)
            assert g.boxes == _literal(seen[v], L, grow, g.number, n - 1)
        assert o.drain(v) == []                  # the drain restarted the video


def _rn(x: Fraction) -> Fraction:
    return Fraction(float(x))                     # round to the nearest double


def _box_fraction(face, k, grow, motions):
    x1, y1, x2, y2 = (Fraction(float(np.float32(v))) for v in face)
    w, h = _rn(x2 - x1), _rn(y2 - y1)
    cx, cy = _rn(x1 + _rn(w / 2)), _rn(y1 + _rn(h / 2))
    for status, m in motions:
        if status != 0:
            continue
        a, b, tx, ty = (Fraction(float(m[i])) for i in (0, 3, 2, 5))
        s2 = _rn(_rn(a * a) + _rn(b * b))
        dx, dy = _rn(cx - tx), _rn(cy - ty)
        cx, cy = _rn(_rn(_rn(a * dx) + _rn(b * dy)) / s2), _rn(_rn(_rn(a * dy) - _rn(b * dx)) / s2)
        s = Fraction(math.sqrt(float(s2)))        # IEEE sqrt is correctly rounded
        w, h = _rn(w / s), _rn(h / s)
    g = _rn(Fraction(1, 2) + _rn(Fraction(grow) * k))
    ex, ey = _rn(g * w), _rn(g * h)
    return tuple(float(np.float32(float(_rn(v)))) for v in (cx - ex, cy - ey, cx + ex, cy + ey))


def test_box_equals_rational_arithmetic():
    rng = np.random.default_rng(5)
    for trial in range(300):
        face = tuple(np.float32(v) for v in (rng.uniform(-50, 1800), rng.uniform(-50, 1000)))
        s = rng.uniform(8, 300)
        face = face + (np.float32(face[0] + s), np.float32(face[1] + 1.3 * s))
        k = int(rng.integers(1, 65))
        grow = float(np.float32(rng.uniform(0.01, 1.0)))
        motions = []
        if trial % 2:
            for _ in range(k):
                a, b = 1 + rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05)
                motions.append((int(rng.choice([0, 0, 1, 2])), (a, -b, rng.uniform(-80, 80), b, a, rng.uniform(-40, 40))))
        assert lookback_box(face, k, grow, motions) == _box_fraction(face, k, grow, motions), trial


def test_inverse_motion_chain_equals_composed_inverses():
    """Undoing frames b .. e + 1 one by one moves the centre where the inverse of their composed similarities does (1e-12 relative),
    and the size by the product of 1 / s."""
    rng = np.random.default_rng(9)
    for trial in range(100):
        k = int(rng.integers(1, 65))
        ms = []
        for _ in range(k):
            a, b = 1 + rng.uniform(-0.1, 0.1), rng.uniform(-0.05, 0.05)
            ms.append((0, (a, -b, rng.uniform(-50, 50), b, a, rng.uniform(-30, 30))))
        face = (500.0, 300.0, 620.0, 450.0)
        got = lookback_box(face, k, 0.5, ms)          # g = 0.5 + 0.5 k
        M = np.eye(3)
        for _, m in ms:                                # frame f's motion maps f - 1 -> f; ms[0] is frame b's
            M = M @ np.array([[m[0], m[1], m[2]], [m[3], m[4], m[5]], [0, 0, 1]])
        # M maps frame e -> frame b; its inverse takes the birth's centre back to frame e
        c = np.linalg.solve(M, np.array([560.0, 375.0, 1.0]))
        s = np.prod([math.hypot(m[0], m[3]) for _, m in ms])
        g = 0.5 + 0.5 * k
        want = (c[0] - g * 120 / s, c[1] - g * 150 / s, c[0] + g * 120 / s, c[1] + g * 150 / s)
        assert np.allclose(got, want, rtol=1e-6, atol=0), (trial, got, want)     # float32 output
        assert abs((got[0] + got[2]) / 2 - c[0]) <= 1e-4 * max(1.0, abs(c[0]))
        # the chain in doubles, before the float rounding, within 1e-12
        cx, cy = 560.0, 375.0
        for _, m in ms:
            a, b = m[0], m[3]
            s2 = a * a + b * b
            dx, dy = cx - m[2], cy - m[5]
            cx, cy = (a * dx + b * dy) / s2, (a * dy - b * dx) / s2
        assert abs(cx - c[0]) <= 1e-12 * abs(c[0]) and abs(cy - c[1]) <= 1e-12 * max(abs(c[1]), 1.0), trial


def test_config_defaults_and_bounds():
    assert config() == (15, float(np.float32(0.1)))
    assert config(64, 1.0) == (64, 1.0)
    for bad in ((65, 0.0), (-1, 0.0), (0, 1.5), (0, -0.1), (0, float("nan")), (0, float("inf"))):
        with pytest.raises(ValueError):
            config(*bad)


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = capi.load_library()
    for s in ("rf_tracker_set_lookback", "rf_detect_yuv_redact_lookback_device", "rf_tracker_drain"):
        assert hasattr(lib, s)
    assert C.sizeof(capi.LookbackConfig) == 8 and capi.LookbackConfig.grow.offset == 4
    src = tmp_path / "lb.c"
    src.write_text('#include "rf_b200.h"\n#include <stddef.h>\n'
                   '_Static_assert(sizeof(rf_lookback_config) == 8 && offsetof(rf_lookback_config, grow) == 4, "layout");\n'
                   'int main(void) { rf_lookback_config c = {0, 0.f}; return rf_tracker_set_lookback(NULL, &c) == RF_ERR_INVALID_ARG ? 0 : 1; }\n')
    exe = tmp_path / "lb"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L",
                           os.path.dirname(capi.lib_path()), "-lrf_b200", "-Wl,-rpath," + os.path.dirname(capi.lib_path())])
    assert subprocess.run([str(exe)]).returncode == 0


def test_kernels_build_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "lookback.cu"), "-o",
                                                   str(tmp_path / "lb.o")], capture_output=True, text=True, check=True)
    names = re.findall(r"Compiling entry function '\S*(k_lookback_\w+?)E", r.stderr)
    assert sorted(set(n.rstrip("0123456789_") for n in names)) == ["k_lookback_boxes", "k_lookback_log", "k_lookback_swap"], names
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert spills and all(a == "0" and b == "0" for a, b in spills), r.stderr


def test_host_shell_compiles(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
