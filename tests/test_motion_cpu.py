"""CPU: f13 camera motion without a GPU -- oracle/motion.py against literal loops of rf_b200.h's definition, recovery of known
similarities and robustness on synthetic frames, the compensation against ByteTrack's 8 x 8 filter, the ctypes layout against the
header, the C link of the new symbols, the kernels' build and the C++ shell."""
import ctypes as C
import math
import os
import subprocess

import cv2
import numpy as np
import pytest

from conftest import ROOT
from oracle.motion import FIRST, LOST, OK, MotionOracle, MotionTrackerOracle, compensate, estimate, match_block, sad_table, thumbnail
from oracle.track import KalmanMatrix, Track, TrackerOracle

W, H = 1920, 1080
R = 12
# Recovery tolerances, fixed from the oracle before any GPU run: the frame centre maps within half a thumbnail pixel (D / 2 = 3 frame
# pixels at 1080p) of the true transform, and a, b within 0.005.  The oracle meets them with a wide margin (0.25 px, 2e-4).
TOL_CENTRE = 3.0
TOL_AB = 0.005


def scene(seed: int, w: int = 2600, h: int = 1700) -> np.ndarray:
    """A seeded textured luma scene: coarse and fine band-limited noise."""
    r = np.random.default_rng(seed)
    a = cv2.resize(r.integers(0, 256, (h // 24, w // 24)).astype(np.uint8), (w, h), interpolation=cv2.INTER_CUBIC).astype(np.float32)
    b = cv2.resize(r.integers(0, 256, (h // 6, w // 6)).astype(np.uint8), (w, h), interpolation=cv2.INTER_CUBIC).astype(np.float32)
    return np.clip(0.6 * a + 0.4 * b, 0, 255).astype(np.uint8)


def view(S: np.ndarray, M: np.ndarray, ox: int = 300, oy: int = 300) -> np.ndarray:
    """The W x H window at (ox, oy) of the scene moved by M (frame pixels of the window: x' = M x)."""
    A = M[:, :2]
    t = M[:, 2] - A @ np.array([ox, oy], float)
    return cv2.warpAffine(S, np.c_[A, t], (W, H), flags=cv2.INTER_LINEAR)


def similarity(angle_deg: float, scale: float, tx: float, ty: float) -> np.ndarray:
    M = cv2.getRotationMatrix2D((W / 2, H / 2), angle_deg, scale)
    M[:, 2] += (tx, ty)
    return M


def centre_error(m, M) -> float:
    c = np.array([W / 2, H / 2])
    got = np.array([m[0] * c[0] + m[1] * c[1] + m[2], m[3] * c[0] + m[4] * c[1] + m[5]])
    return float(np.abs(got - M @ np.r_[c, 1.0]).max())


def test_thumbnail_equals_literal_loop():
    rng = np.random.default_rng(0)
    for w, h in ((646, 330), (322, 200), (1000, 1282), (64, 48)):
        luma = rng.integers(0, 256, (h, w), dtype=np.uint8)
        th, D = thumbnail(luma)
        assert D == math.ceil(max(w, h) / 320) and th.shape == (h // D, w // D)
        for y in range(0, th.shape[0], 7):
            for x in range(0, th.shape[1], 5):
                s = sum(int(luma[D * y + r, D * x + c]) for r in range(D) for c in range(D))
                assert th[y, x] == (s + D * D // 2) // (D * D)


def test_block_match_equals_brute_force_argmin():
    rng = np.random.default_rng(1)
    S = scene(5, 400, 300)
    for trial in range(40):
        r = int(rng.integers(2, 9))
        cur = S[50:150, 60:180].copy()
        dy, dx = rng.integers(-r, r + 1, 2)
        ref = S[50 + dy:150 + dy, 60 + dx:180 + dx].copy()
        if trial % 4 == 0:          # ties: a flat reference gives a shared minimum
            ref[:] = 128
        x0, y0 = r + 16, r + 16
        got = match_block(cur, ref, x0, y0, r)
        best, ties = None, 0
        for oy in range(-r, r + 1):
            for ox in range(-r, r + 1):
                s = sum(abs(int(cur[y0 + i, x0 + j]) - int(ref[y0 + oy + i, x0 + ox + j])) for i in range(16) for j in range(16))
                key = (s, abs(oy) + abs(ox), oy, ox)
                best = key if best is None or key < best else best
        T = sad_table(cur, ref, x0, y0, r)
        ties = int((T == best[0]).sum())
        if ties > 1 or abs(best[2]) == r or abs(best[3]) == r:
            assert got is None, trial
            continue
        assert got is not None
        assert got[2] - got[0] == pytest.approx(best[3], abs=0.5) and got[3] - got[1] == pytest.approx(best[2], abs=0.5)
        assert math.floor(got[2] - got[0] + 0.5) == best[3] and math.floor(got[3] - got[1] + 0.5) == best[2]


@pytest.mark.parametrize("k", range(8))
def test_recovers_known_similarities(k):
    rng = np.random.default_rng(100 + k)
    S = scene(10 + k)
    # rotations up to 3 degrees, scales 0.9 .. 1.1, translations up to R * D = 72 frame pixels less the rotation's and the zoom's
    # share at the blocks; k = 0: a pure translation of 11 thumbnail pixels (R itself lies on the search border, which drops a block)
    M = similarity(rng.uniform(-3, 3), rng.uniform(0.9, 1.1), *rng.uniform(-60, 60, 2))
    if k == 0:
        M = similarity(0.0, 1.0, 66.0, -66.0)
    mo = MotionOracle()
    assert mo.update(0, view(S, np.eye(3)[:2]))["status"] == FIRST
    r = mo.update(0, view(S, M))
    assert r["status"] == OK, r
    assert centre_error(r["m"], M) <= TOL_CENTRE and abs(r["m"][0] - M[0, 0]) <= TOL_AB and abs(r["m"][3] - M[1, 0]) <= TOL_AB


def test_independent_patch_is_ignored():
    """A patch covering 30 % of the blocks moves on its own: the estimate stays within the tolerances."""
    S = scene(21)
    M = similarity(1.5, 1.04, 40.0, -25.0)
    prev, cur = view(S, np.eye(3)[:2]), view(S, M)
    patch = scene(99, 900, 700)
    # the patch sits at the same frame position in both frames but its content moves by (+30, +20): it matches elsewhere
    x0, y0, pw, ph = 300, 200, 1000, 420          # about 30 % of the 18 x 9 block grid
    big = cv2.resize(patch, (pw + 60, ph + 60))
    prev[y0:y0 + ph, x0:x0 + pw] = big[20:20 + ph, 30:30 + pw]
    cur[y0:y0 + ph, x0:x0 + pw] = big[:ph, :pw]
    mo = MotionOracle()
    mo.update(0, prev)
    r = mo.update(0, cur)
    assert r["status"] == OK and centre_error(r["m"], M) <= TOL_CENTRE
    assert abs(r["m"][0] - M[0, 0]) <= TOL_AB and abs(r["m"][3] - M[1, 0]) <= TOL_AB


def test_flat_frame_and_scene_cut_are_lost_and_first_is_first():
    S = scene(31)
    mo = MotionOracle()
    assert mo.update(0, view(S, np.eye(3)[:2]))["status"] == FIRST
    r = mo.update(0, np.full((H, W), 117, np.uint8))
    assert r["status"] == LOST and r["blocks"] == 0 and r["m"] == (1.0, 0.0, 0.0, 0.0, 1.0, 0.0)
    mo.update(0, view(S, np.eye(3)[:2]))
    assert mo.update(0, view(scene(77), np.eye(3)[:2]))["status"] == LOST          # a different scene
    # a new frame size has no reference; nor has a reset video
    assert mo.update(0, view(S, np.eye(3)[:2])[:720, :1280])["status"] == FIRST
    mo.reset(0)
    assert mo.update(0, view(S, np.eye(3)[:2])[:720, :1280])["status"] == FIRST


def test_records_exclude_blocks():
    S = scene(41)
    cur, prev = view(S, similarity(0, 1, 20, 10)), view(S, np.eye(3)[:2])
    th, D = thumbnail(cur)
    tp, _ = thumbnail(prev)
    all_ = estimate(th, tp, D)
    face = np.zeros((1, 15), np.float32)
    face[0, :5] = (0.9, 400, 300, 700, 700)          # network-input pixels, scale 2 -> frame pixels 800..1400 x 600..1400
    part = estimate(th, tp, D, face, 1, 2.0)
    assert all_["status"] == OK and part["status"] == OK and part["blocks"] < all_["blocks"]


def _A8(a, b, s):
    A = np.zeros((8, 8))
    for o in (0, 4):
        A[o:o + 2, o:o + 2] = [[a, -b], [b, a]]
        A[o + 2, o + 2] = 1.0
        A[o + 3, o + 3] = s
    return A


def test_compensation_equals_matrix_form_and_keeps_cx_cy_equal():
    rng = np.random.default_rng(5)
    K = KalmanMatrix()
    for _ in range(200):
        z = [rng.uniform(50, 1800), rng.uniform(50, 1000), rng.uniform(0.5, 1.2), rng.uniform(20, 300)]
        t = Track(1, z, np.zeros(15, np.float32), 1, 0)
        mean, cov = K.initiate(z)
        for _ in range(int(rng.integers(0, 4))):
            zz = [v + rng.normal(0, 3) for v in z]
            t.predict()
            t.update(zz)
            mean, cov = K.predict(mean, cov)
            mean, cov = K.update(mean, cov, zz)
        t.predict()
        mean, cov = K.predict(mean, cov)
        ang, sc = rng.uniform(-0.05, 0.05), rng.uniform(0.9, 1.1)
        a, b = sc * math.cos(ang), sc * math.sin(ang)
        m = (a, -b, rng.uniform(-80, 80), b, a, rng.uniform(-80, 80))
        compensate(t, m)
        s = math.sqrt(a * a + b * b)
        A = _A8(a, b, s)
        mean = A @ mean
        mean[:2] += (m[2], m[5])
        cov = A @ cov @ A.T
        state = np.r_[t.m, t.u]
        assert np.allclose(state, mean, rtol=1e-12, atol=0)
        for c in range(4):
            for got, ref in ((t.p00[c], cov[c, c]), (t.p01[c], cov[c, 4 + c]), (t.p11[c], cov[4 + c, 4 + c])):
                assert got == pytest.approx(ref, rel=1e-12)
        assert abs(cov[0, 1]) <= 1e-12 * cov[0, 0] and abs(cov[0, 5]) <= 1e-12 * abs(cov[0, 4]) + 1e-300


def test_cx_cy_covariances_equal_bit_for_bit_in_an_oracle_run():
    rng = np.random.default_rng(9)
    tr = MotionTrackerOracle(1)
    faces = np.zeros((3, 15), np.float32)
    faces[:, 0] = 0.95
    pos = np.array([[100, 100], [400, 200], [800, 500]], np.float32)
    for k in range(40):
        ang = rng.uniform(-0.03, 0.03)
        a, b = 1.02 * math.cos(ang), 1.02 * math.sin(ang)
        m = (a, -b, rng.uniform(-40, 40), b, a, rng.uniform(-40, 40))
        pos = pos + rng.normal(0, 2, pos.shape).astype(np.float32)
        faces[:, 1:3] = pos
        faces[:, 3:5] = pos + np.float32([60, 80])
        keep = faces[: 3 if k % 7 else 1]                  # LOST stretches too
        tr.update(0, keep, None, motion=m if k % 3 else None)
        for t in tr.v[0]["tracks"]:
            assert t.p00[0] == t.p00[1] and t.p01[0] == t.p01[1] and t.p11[0] == t.p11[1]


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    src = tmp_path / "mo.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rf_b200.h"\nint main(void){\n'
                   'printf("%zu %zu %zu %zu\\n", sizeof(rf_motion), offsetof(rf_motion, m), sizeof(rf_motion_config), offsetof(rf_motion_config, min_inliers));\n'
                   'const rf_motion *p = 0; rf_motion_config c = {0, 0};\n'
                   'printf("%d %d\\n", rf_tracker_set_motion(NULL, &c) == RF_ERR_INVALID_ARG, rf_tracker_motion(NULL, &p) == RF_ERR_INVALID_ARG);\n'
                   'return 0;}\n')
    exe = tmp_path / "mo"
    libdir = os.path.dirname(built_lib)
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lrf_b200",
                           "-Wl,-rpath," + libdir])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(capi.Motion), capi.Motion.m.offset, C.sizeof(capi.MotionConfig), capi.MotionConfig.min_inliers.offset, 1, 1]
    assert capi.MOTION_DTYPE.itemsize == C.sizeof(capi.Motion) == 64
    assert {"rf_tracker_set_motion", "rf_tracker_motion"} <= set(capi.EXPORTS)


def test_entry_points_refuse_null_handles_without_gpu(built_lib):
    from retinaface_b200 import capi
    lib = capi.load_library()
    cfg = capi.motion_config()
    assert lib.rf_tracker_set_motion(None, C.byref(cfg)) == -1
    p = C.c_void_p()
    assert lib.rf_tracker_motion(None, C.byref(p)) == -1


def test_motion_kernels_compile_for_sm90a_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, CSRC, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "motion.cu"), "-o",
                                                   str(tmp_path / "m.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for k in ("k_motion_thumb", "k_motion_match", "k_motion_fit", "k_motion_commit"):
        assert k in r.stderr, k
    assert r.stderr.count("0 bytes spill stores") >= 4 and "bytes spill stores" not in r.stderr.replace("0 bytes spill stores", ""), r.stderr


def test_cpp_shell_compiles_motion_calls(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    src = open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.cpp")).read()
    assert "rf_tracker_set_motion" in src and "rf_tracker_motion" in src


def test_motion_tracker_oracle_is_the_tracker_oracle_plus_the_motion_step():
    """Without motion MotionTrackerOracle is TrackerOracle bit for bit; with it, on a frame without records (nothing matches, so no
    Kalman update follows), every track's state is exactly Track.predict then compensate, applied once."""
    import copy
    rng = np.random.default_rng(13)
    plain, moved = TrackerOracle(1), MotionTrackerOracle(1)
    faces = np.zeros((2, 15), np.float32)
    faces[:, 0] = 0.95
    pos = np.array([[100, 100], [500, 300]], np.float32)
    m = (1.01, -0.004, 3.0, 0.004, 1.01, -2.0)
    for k in range(12):
        pos = pos + rng.normal(0, 2, pos.shape).astype(np.float32)
        faces[:, 1:3] = pos
        faces[:, 3:5] = pos + np.float32([60, 80])
        plain.update(0, faces, None)
        moved.update(0, faces, None)
        assert np.array_equal(plain.debug_state(0).view(np.uint64), moved.debug_state(0).view(np.uint64)), k
    want = copy.deepcopy(moved.v[0]["tracks"])
    for t in want:
        t.predict()
        compensate(t, m)
    moved.update(0, np.zeros((0, 15), np.float32), None, motion=m)
    got = moved.v[0]["tracks"]
    assert len(got) == len(want) == 2
    for g, w in zip(got, want):
        assert "predict" not in g.__dict__
        assert [g.m, g.u, g.p00, g.p01, g.p11] == [w.m, w.u, w.p00, w.p01, w.p11]
