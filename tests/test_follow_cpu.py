"""f16 following without a GPU: oracle/follow.py's search against a literal per-candidate loop, its templates against cv2.warpAffine on
the luma plane, the tie order and the sub-pixel step against exact rationals, the four failure statuses on constructed frames,
rf_follow_config's bounds, the C layout and link, and the no-spill build of the new kernels."""
import ctypes as C
import os
import re
import subprocess
from fractions import Fraction

import cv2
import numpy as np
import pytest

from oracle.follow import (BORDER, FLAT, MISMATCH, OK, OUTSIDE, T, config, cut, face_grid, grid, order_key, parabola, sample,
                           scale_of, search)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "retinaface_b200", "csrc")


def _texture(rng, h=360, w=640):
    """Smooth random texture (blurred noise), so that every sub-pixel shift changes the SAD."""
    t = cv2.GaussianBlur(rng.integers(0, 256, (h, w), dtype=np.uint8), (0, 0), 2.0)
    return cv2.normalize(t, None, 0, 255, cv2.NORM_MINMAX)


def _face(x1, y1, x2, y2, score=0.9):
    f = np.zeros(15, np.float32)
    f[:5] = (score, x1, y1, x2, y2)
    f[5:10] = np.linspace(x1 + 10, x2 - 10, 5)
    f[10:15] = np.linspace(y1 + 10, y2 - 10, 5)
    return f


def _state(face):
    """(m, u) of a track whose predicted box is the face's box: m = z of the face, u = 0."""
    x1, y1 = float(face[1]), float(face[2])
    w, h = float(face[3]) - x1, float(face[4]) - y1
    return [x1 + w / 2.0, y1 + h / 2.0, w / h, h], [0.0] * 4


def test_template_equals_cv2_warp_affine():
    """The sampler is cv2.warpAffine(INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT 0) on the luma plane, byte for byte, inside
    and across the frame's edges, at every scale."""
    rng = np.random.default_rng(1)
    luma = rng.integers(0, 256, (240, 320), dtype=np.uint8)
    for trial in range(200):
        x1, y1 = rng.uniform(-60, 300), rng.uniform(-60, 220)
        s = rng.uniform(4, 180)
        face = _face(x1, y1, x1 + s, y1 + s * rng.uniform(0.8, 1.5))
        for c in (scale_of(0), 1.0, scale_of(2)):
            x1f, y1f = float(face[1]), float(face[2])
            w, h = float(face[3]) - x1f, float(face[4]) - y1f
            px, py, ox, oy = grid(x1f + w / 2.0, y1f + h / 2.0, w, h, c)
            R = int(rng.integers(0, 17))
            n = T + 2 * R
            X, Y = ox - float(R) * px, oy - float(R) * py
            got, _ = sample(luma, px, py, X, Y, n)
            want = cv2.warpAffine(luma, np.array([[px, 0.0, X], [0.0, py, Y]]), (n, n), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                                  borderMode=cv2.BORDER_CONSTANT, borderValue=0)
            assert np.array_equal(got, want), (trial, c, R)
        tm, _ = cut(luma, face)
        px, py, ox, oy = face_grid(face)
        assert np.array_equal(tm, cv2.warpAffine(luma, np.array([[px, 0.0, ox], [0.0, py, oy]]), (T, T),
                                                 flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP)), trial


def _literal_search(luma, tmpl, m, u, R):
    """The definition's search as a literal loop over candidates: every (k, dy, dx) in the stated order, ties to the first."""
    pcx, pcy, pa, ph = m[0] + u[0], m[1] + u[1], m[2] + u[2], m[3] + u[3]
    pw = pa * ph
    best = None
    tab = {}
    for k in range(3):
        px, py, ox, oy = grid(pcx, pcy, pw, ph, scale_of(k))
        win, _ = sample(luma, px, py, ox - float(R) * px, oy - float(R) * py, T + 2 * R)
        for dy in range(-R, R + 1):
            for dx in range(-R, R + 1):
                sad = 0
                for j in range(T):
                    for i in range(0, T, 8):
                        a = tmpl[j, i:i + 8].astype(int)
                        b = win[R + dy + j, R + dx + i:R + dx + i + 8].astype(int)
                        sad += int(np.abs(a - b).sum())
                tab[k, dy, dx] = sad
                cand = (sad, abs(dx) + abs(dy), k, dy, dx)
                if best is None or cand < best:
                    best = cand
    return best, tab


def test_search_equals_a_literal_loop():
    rng = np.random.default_rng(2)
    luma = _texture(rng)
    for trial in range(4):
        x1, y1, s = rng.uniform(150, 400), rng.uniform(80, 200), rng.uniform(40, 90)
        face = _face(x1, y1, x1 + s, y1 + 1.2 * s)
        tmpl, flat = cut(luma, face)
        m, u = _state(face)
        u = [rng.uniform(-6, 6), rng.uniform(-6, 6), 0.0, rng.uniform(-1, 1)]       # a predicted motion the search must undo
        R = int(rng.integers(2, 6))
        rec, nf = search(luma, tmpl, flat, m, u, face, R, 24.0)
        best, tab = _literal_search(luma, tmpl, m, u, R)
        assert (rec["sad"], abs(rec["dx"]) + abs(rec["dy"]), rec["scale"], rec["dy"], rec["dx"]) == best, trial
        assert rec["sad"] == tab[rec["scale"], rec["dy"], rec["dx"]]


def test_tie_order_and_subpixel_step():
    """The packed key orders exactly as the tuple (SAD, |dx| + |dy|, k, dy, dx); the parabola is the exact rational rounded once."""
    rng = np.random.default_rng(3)
    R = 16
    cands = [(int(rng.integers(0, 4)), int(rng.integers(0, 3)), int(rng.integers(-R, R + 1)), int(rng.integers(-R, R + 1)))
             for _ in range(3000)]
    by_key = sorted(cands, key=lambda c: order_key(c[0], c[1], c[2], c[3], R))
    by_tuple = sorted(cands, key=lambda c: (c[0], abs(c[3]) + abs(c[2]), c[1], c[2], c[3]))
    assert by_key == by_tuple
    assert order_key(T * T * 255, 2, R, R, R) < 1 << 63
    for _ in range(5000):
        s0 = int(rng.integers(0, 200000))
        sm, sp = s0 + int(rng.integers(0, 5000)), s0 + int(rng.integers(0, 5000))
        d = 2 * (sm - 2 * s0 + sp)
        want = 0.0 if d == 0 else float(Fraction(sm - sp, d))
        assert parabola(sm, s0, sp) == want
        assert abs(want) <= 0.5
    assert parabola(7, 7, 7) == 0.0


def test_failure_statuses():
    """FLAT (a flat template), OUTSIDE (the window off the frame), BORDER (a jump past R), MISMATCH (a flat patch over the face) and
    OK (the face moved inside R) on constructed frames."""
    rng = np.random.default_rng(4)
    luma = _texture(rng)
    face = _face(280, 120, 360, 220)
    tmpl, flat = cut(luma, face)
    assert not flat
    m, u = _state(face)
    moved = np.roll(luma, (3, -5), axis=(0, 1))
    rec, _ = search(moved, tmpl, flat, m, u, face, 8, 24.0)
    assert rec["status"] == OK and (rec["dx"], rec["dy"]) != (0, 0)
    # FLAT: the template of a uniform wall
    wall = np.full_like(luma, 90)
    ft, fflat = cut(wall, face)
    assert fflat and search(luma, ft, fflat, m, u, face, 8, 24.0)[0]["status"] == FLAT
    # BORDER: the face jumped far past R template pixels
    far = np.roll(luma, 60, axis=1)
    assert search(far, tmpl, flat, m, u, face, 2, 255.0)[0]["status"] == BORDER
    # MISMATCH: a flat patch over the face
    occ = luma.copy()
    occ[60:300, 200:440] = 128
    assert search(occ, tmpl, flat, m, u, face, 8, 24.0)[0]["status"] == MISMATCH
    # OUTSIDE: the predicted box mostly off the frame
    edge = _face(600, 120, 700, 220)
    em, eu = _state(edge)
    assert search(luma, tmpl, flat, em, eu, edge, 8, 255.0)[0]["status"] == OUTSIDE


def test_config_defaults_and_bounds():
    assert config() == (8, 24.0)
    assert config(16, 255.0) == (16, 255.0)
    for bad in ((17, 0.0), (-1, 0.0), (0, 256.0), (0, -1.0), (0, float("nan")), (0, float("inf"))):
        with pytest.raises(ValueError):
            config(*bad)


def test_header_constants_match_the_oracle():
    from oracle import follow
    hdr = open(os.path.join(ROOT, "include", "rf_b200.h")).read()
    want = dict(TEMPLATE=follow.T, MARGIN=follow.MARGIN, SCALE=follow.SCALE, MIN_VAR=follow.MIN_VAR, MAX_SEARCH=follow.MAX_SEARCH,
                OK=follow.OK, FLAT=follow.FLAT, BORDER=follow.BORDER, MISMATCH=follow.MISMATCH, OUTSIDE=follow.OUTSIDE, LOST=follow.LOST_STATUS)
    for k, v in want.items():
        m = re.search(rf"#define RF_FOLLOW_{k}\s+(\S+)", hdr)
        assert m and float(m.group(1)) == v, k


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = capi.load_library()
    for s in ("rf_tracker_set_follow", "rf_track_follow_device", "rf_tracker_follow"):
        assert hasattr(lib, s)
    assert C.sizeof(capi.FollowConfig) == 8 and capi.FollowConfig.max_mad.offset == 4
    assert C.sizeof(capi.FollowRecord) == 48 == capi.FOLLOW_DTYPE.itemsize and capi.FollowRecord.x1.offset == 32
    assert capi.TRACK_DTYPE.fields["followed"][1] == capi.TrackRecord.followed.offset == 28
    src = tmp_path / "fo.c"
    src.write_text('#include "rf_b200.h"\n#include <stddef.h>\n'
                   '_Static_assert(sizeof(rf_follow_config) == 8 && offsetof(rf_follow_config, max_mad) == 4, "layout");\n'
                   '_Static_assert(sizeof(rf_follow) == 48 && offsetof(rf_follow, x1) == 32 && offsetof(rf_follow, sad) == 20, "layout");\n'
                   '_Static_assert(sizeof(rf_track) == 116 && offsetof(rf_track, followed) == 28, "layout");\n'
                   'int main(void) { rf_follow_config c = {0, 0.f}; const rf_follow *f = 0;\n'
                   '  return rf_tracker_set_follow(NULL, &c) == RF_ERR_INVALID_ARG && rf_tracker_follow(NULL, &f) == RF_ERR_INVALID_ARG &&\n'
                   '         rf_track_follow_device(NULL, NULL, NULL, 0, NULL, NULL) == RF_ERR_INVALID_ARG ? 0 : 1; }\n')
    exe = tmp_path / "fo"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L",
                           os.path.dirname(capi.lib_path()), "-lrf_b200", "-Wl,-rpath," + os.path.dirname(capi.lib_path())])
    assert subprocess.run([str(exe)]).returncode == 0


def test_kernels_build_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "follow.cu"), "-o",
                                                   str(tmp_path / "fo.o")], capture_output=True, text=True, check=True)
    names = re.findall(r"Compiling entry function '\S*(k_follow_\w+?)E", r.stderr)
    assert sorted(set(n.rstrip("0123456789_") for n in names)) == ["k_follow_cut", "k_follow_mask", "k_follow_search", "k_follow_update"], names
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert frames and all(f == ("0", "0", "0") for f in frames), r.stderr


def test_host_shell_detect_every_compiles(built_lib, tmp_path):
    """The C++ shell's RetinaFaceOptions::detect_every and lastFollow() as a user writes them."""
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "de.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int use(RetinaFace &rf) { RetinaFaceOptions o; o.detect_every = 3; o.track_motion = true;\n'
                   '  const RetinaFace::DeviceFollow &f = rf.lastFollow(); return o.detect_every + f.n + (f.follow ? 1 : 0); }\n')
    subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-I", host, "-I", os.path.join(ROOT, "include"), str(src)])


def test_interval_calls_keep_each_videos_order():
    """RetinaFace's split of a call into detect and follow calls: every frame once, each video's frames in order, runs of one kind."""
    from types import SimpleNamespace
    from retinaface_b200.detector import RetinaFace
    rng = np.random.default_rng(5)
    for k in (2, 3, 5):
        holder, nums = SimpleNamespace(), {}
        for _ in range(30):
            vids = [int(v) for v in rng.integers(0, 3, int(rng.integers(1, 9)))]
            calls = RetinaFace._interval_calls(holder, vids, k)
            issued = [i for _, idx in calls for i in idx]
            assert sorted(issued) == list(range(len(vids)))
            for v in set(vids):
                mine = [i for i in issued if vids[i] == v]
                assert mine == sorted(mine)
            for det, idx in calls:
                for i in idx:
                    n = nums.get(vids[i], 0) + sum(1 for j in range(i) if vids[j] == vids[i])
                    assert det == (n % k == 0)
            for v in vids:
                nums[v] = nums.get(v, 0) + 1
