"""CPU: f10 tracking without a GPU -- the scalar oracle against ByteTrack's 8 x 8 Kalman filter, the greedy stages against the
optimal assignment, the lifecycle rules on hand-built sequences, the ctypes layouts against the header, and the builds."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

from conftest import ROOT
from oracle.track import CONFIRMED, LOST, TENTATIVE, KalmanMatrix, Track, TrackerOracle, box_of, greedy, iou, measure


def _face(x1, y1, x2, y2, score=0.9):
    f = np.zeros(15, np.float32)
    f[:5] = (score, x1, y1, x2, y2)
    return f


def _faces(*boxes):
    return np.array([_face(*b) for b in boxes], np.float32).reshape(-1, 15)


def test_scalar_filter_equals_matrix_form():
    """Random predict / update / lost sequences: the four scalar filters equal ByteTrack's 8 x 8 filter to 1e-9 relative."""
    rng = np.random.default_rng(5)
    km = KalmanMatrix()
    for _ in range(50):
        p, s = rng.uniform(0, 500, 2), rng.uniform(20, 200, 2)
        z = measure(_face(p[0], p[1], p[0] + s[0], p[1] + s[1]))
        t = Track(1, z, _face(0, 0, 1, 1), CONFIRMED, 0)
        mean, cov = km.initiate(z)
        for step in range(30):
            lost = rng.random() < 0.2
            t.state = LOST if lost else CONFIRMED
            t.predict()
            mean, cov = km.predict(mean, cov, lost)
            if not lost:
                b = box_of(t.m)
                zz = measure(_face(*(np.array(b) + rng.normal(0, 0.03 * s.min(), 4))))
                if zz is None:      # the random walk collapsed the box
                    break
                t.update(zz)
                mean, cov = km.update(mean, cov, zz)
            got_m = np.array(t.m + t.u)
            got_c = np.zeros((8, 8))
            for c in range(4):
                got_c[c, c], got_c[c, 4 + c], got_c[4 + c, c], got_c[4 + c, 4 + c] = t.p00[c], t.p01[c], t.p01[c], t.p11[c]
            assert np.allclose(got_m, mean, rtol=1e-9, atol=1e-9 * np.abs(mean).max()), step
            assert np.allclose(got_c, cov, rtol=1e-9, atol=1e-9 * np.abs(cov).max()), step


def test_greedy_equals_optimal_assignment_without_rivals():
    """On every random frame where no track has two candidates above the threshold, the greedy stage is the optimal assignment."""
    rng = np.random.default_rng(7)
    checked = 0
    for _ in range(400):
        tr = [list(rng.uniform(0, 400, 2)) for _ in range(rng.integers(1, 8))]
        tr = [[x, y, x + 60, y + 80] for x, y in tr]
        de = [[b[0] + rng.normal(0, 25), b[1] + rng.normal(0, 25), b[2] + rng.normal(0, 25), b[3] + rng.normal(0, 25)]
              for b in tr if rng.random() < 0.8]
        M = np.array([[iou(t, d) for d in de] for t in tr]).reshape(len(tr), len(de))
        cand = M > 0.2
        if len(de) == 0 or (cand.sum(1) > 1).any():
            continue
        pairs = [(M[i, j], i + 1, j) for i in range(len(tr)) for j in range(len(de)) if cand[i, j]]
        g = greedy(pairs)
        r, c = linear_sum_assignment(np.where(cand, -M, 0.0))
        opt = {i + 1: j for i, j in zip(r, c) if cand[i, j]}
        assert g == opt
        checked += 1
    assert checked > 100


def _ids(tracks, state=None):
    return [t["id"] for t in tracks if state is None or t["state"] == state]


def test_lifecycle_rules():
    o = TrackerOracle(2, max_tracks=3, max_lost=2)
    a, b = (100, 100, 160, 180), (400, 100, 460, 180)
    # first frame: births are confirmed at once, in record (score) order
    out = o.update(0, _faces(a + (0.95,), b + (0.8,)))
    assert _ids(out, CONFIRMED) == [1, 2] and [t["det"] for t in out] == [0, 1]
    # a later birth is tentative and confirmed on its second matched frame; a low-score record never starts a track
    c = (700, 100, 760, 180)
    out = o.update(0, _faces(a, b, c, (900, 100, 960, 180, 0.65)))
    assert [(t["id"], t["state"]) for t in out] == [(1, CONFIRMED), (2, CONFIRMED), (3, TENTATIVE)]
    out = o.update(0, _faces(a, b, c))
    assert out[2]["state"] == CONFIRMED and out[2]["hits"] == 2
    # a tentative track unmatched on its next frame is removed
    o.update(1, _faces(a))
    o.update(1, _faces(a, b))
    assert _ids(o.update(1, _faces(a))) == [1]
    # a lost track comes back with its id; one lost for more than max_lost frames is removed
    out = o.update(0, _faces(a, c))
    assert [(t["id"], t["state"], t["lost_frames"]) for t in out] == [(1, CONFIRMED, 0), (2, LOST, 1), (3, CONFIRMED, 0)]
    out = o.update(0, _faces(a, b, c))
    assert [(t["id"], t["state"]) for t in out] == [(1, CONFIRMED), (2, CONFIRMED), (3, CONFIRMED)]
    for k in (1, 2):
        out = o.update(0, _faces(a, c))
        assert out[1]["lost_frames"] == k
    assert _ids(o.update(0, _faces(a, c))) == [1, 3]
    # low records keep a confirmed track (stage 2) but never a lost one
    out = o.update(0, _faces(a + (0.5,), c))
    assert [(t["id"], t["state"], t["det"]) for t in out] == [(1, CONFIRMED, 0), (3, CONFIRMED, 1)]
    # overflow at max_tracks: births beyond it are skipped and counted
    o.update(0, _faces(a, c, b, (1000, 100, 1060, 180), (1200, 100, 1260, 180)))
    assert len(o.v[0]["tracks"]) == 3 and o.v[0]["overflow"] == 2 and o.v[0]["issued"] == 4
    o.reset(0)
    assert _ids(o.update(0, _faces(b))) == [1] and o.v[1]["issued"] == 2


def test_crop_slots_go_to_new_identities_in_id_order():
    o = TrackerOracle(1)
    out = o.update(0, _faces((0, 0, 50, 60), (200, 0, 250, 60), (400, 0, 450, 60)), max_align=2)
    assert [t["crop_slot"] for t in out] == [0, 1, -1]
    out = o.update(0, _faces((0, 0, 50, 60), (600, 0, 650, 60)), max_align=2)
    assert all(t["crop_slot"] == -1 for t in out)
    out = o.update(0, _faces((0, 0, 50, 60), (600, 0, 650, 60)), max_align=2)
    assert [(t["id"], t["crop_slot"]) for t in out if t["crop_slot"] >= 0] == [(4, 0)]


def test_ctypes_layout_matches_header(built_lib, tmp_path):
    from retinaface_b200 import capi
    src = tmp_path / "lay.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rf_b200.h"\nint main(void){\n'
                   'printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(rf_track), offsetof(rf_track, kx1), offsetof(rf_track, vx),'
                   ' offsetof(rf_track, face), sizeof(rf_track_config), offsetof(rf_track_config, iou_high), offsetof(rf_track_config, max_lost));\n'
                   'return 0;}\n')
    exe = tmp_path / "lay"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    T, K = capi.TrackRecord, capi.TrackConfig
    assert got == [C.sizeof(T), T.kx1.offset, T.vx.offset, T.face.offset, C.sizeof(K), K.iou_high.offset, K.max_lost.offset]
    assert capi.TRACK_DTYPE.itemsize == C.sizeof(T) and capi.TRACK_DTYPE.fields["face"][1] == T.face.offset


def test_cpp_shell_compiles_track_calls(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    src = open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.cpp")).read()
    assert "rf_detect_yuv_track_device" in src and "rf_tracker_destroy" in src


def test_track_kernel_compiles_for_sm90a_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, CSRC, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "track.cu"), "-o",
                                                   str(tmp_path / "t.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "k_track_update" in r.stderr and "0 bytes spill stores" in r.stderr, r.stderr


def test_tracker_refuses_bad_handles_without_gpu(built_lib):
    from retinaface_b200 import capi
    lib = capi.load_library()
    cfg = capi.TrackConfig(1, 0, 0, 0, 0, 0, 0, 0)
    t = C.c_void_p()
    assert lib.rf_tracker_create(None, C.byref(cfg), C.byref(t)) == -1
    assert lib.rf_track_update(None, None, 0, None, None, None, None, None) == -1
    assert lib.rf_tracker_reset(None, -1) == -1
    assert lib.rf_tracker_debug_state(None, 0, None, 0) == -1
    lib.rf_tracker_destroy(None)
