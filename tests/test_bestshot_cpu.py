"""CPU: f11 best shots without a GPU -- the quality's grey and Laplacian against OpenCV, its terms on hand-built faces, the store and
emission rule of oracle/bestshot.py on a scripted track history, the ctypes layouts against the header, and the sm_90a build."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from conftest import ROOT
from oracle.align import ARCFACE_112, similarity_closed, warp_affine_fixed
from oracle.bestshot import BEST_EXIT, BEST_FINISH, BestShotOracle, grey, inside_mask, laplacian, quality
from oracle.track import CONFIRMED, LOST, TENTATIVE


def test_grey_equals_cvtcolor_on_every_triple():
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert np.array_equal(grey(img), cv2.cvtColor(img, cv2.COLOR_BGR2GRAY).astype(np.int64))


def test_stencil_equals_cv2_laplacian_in_the_interior():
    rng = np.random.default_rng(3)
    for shape in ((112, 112), (37, 61), (8, 8)):
        g = rng.integers(0, 256, shape).astype(np.uint8)
        ref = cv2.Laplacian(g, cv2.CV_16S, ksize=1)[1:-1, 1:-1]
        assert np.array_equal(laplacian(g), ref.astype(np.int64)), shape


def _face(lm, score=0.9):
    lm = np.asarray(lm, np.float32).reshape(5, 2)
    f = np.zeros(15, np.float32)
    f[0] = score
    f[1:5] = (lm[:, 0].min() - 10, lm[:, 1].min() - 10, lm[:, 0].max() + 10, lm[:, 1].max() + 10)
    f[5:10], f[10:15] = lm[:, 0], lm[:, 1]
    return f


def _case(lm, frame, score=0.9):
    f = _face(lm, score)
    M = similarity_closed(f[5:15].reshape(2, 5).T, ARCFACE_112)
    crop = warp_affine_fixed(frame, M, (112, 112))
    return quality(crop, f, M, frame.shape[1], frame.shape[0]), crop, M


def _textured(h, w, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3)).astype(np.uint8)


def test_template_landmarks_are_frontal_and_full_size():
    frame = _textured(300, 300)
    lm = ARCFACE_112.astype(np.float64) + 80
    q, _, M = _case(lm, frame)
    assert q["frontal"] > 0.99 and q["coverage"] == 1.0 and q["eye"] == pytest.approx(35.24, abs=0.01)
    # the exact template (nose on the eyes' perpendicular bisector, up to the template's own 0.03 px) in a frame it fits
    sym = ARCFACE_112.astype(np.float64).copy()
    sym[2, 0] = (sym[0, 0] + sym[1, 0]) / 2
    sym[0, 1] = sym[1, 1] = 51.5
    q2, _, _ = _case(sym * 2 + 50, frame)
    assert q2["frontal"] == 1.0 and q2["eye"] > 35.24 and q2["q"] > 0


def test_nose_on_an_eye_is_not_frontal_and_mirroring_keeps_it():
    frame = _textured(300, 300, 1)
    lm = np.round(ARCFACE_112.astype(np.float64) * 64) / 64 + 60      # coarse: 300 - x is exact in float32
    on_eye = lm.copy()
    on_eye[2] = lm[0]
    q, _, _ = _case(on_eye, frame)
    assert q["frontal"] == 0.0 and q["q"] == 0.0
    turned = lm.copy()
    turned[2, 0] += 6
    mirrored = turned.copy()
    mirrored[:, 0] = 300 - turned[:, 0]
    mirrored[[0, 1]] = mirrored[[1, 0]]
    mirrored[[3, 4]] = mirrored[[4, 3]]
    a, _, _ = _case(turned, frame)
    b, _, _ = _case(mirrored, frame)
    assert 0 < a["frontal"] < 1 and a["frontal"] == pytest.approx(b["frontal"], abs=1e-12)


def test_degenerate_landmarks_give_zero():
    frame = _textured(200, 200, 2)
    same = np.full((5, 2), 100.0)
    q, crop, M = _case(same, frame)
    assert not M.any() and q["q"] == 0.0 and q["eye"] == 0.0 and q["coverage"] == 0.0 and q["sharpness"] == 0.0
    eyes_together = ARCFACE_112.astype(np.float64) + 40
    eyes_together[1] = eyes_together[0]
    q, _, _ = _case(eyes_together, frame)
    assert q["q"] == 0.0 and q["eye"] == 0.0 and q["frontal"] == 0.0


def test_identity_like_M_inside_the_frame_has_full_coverage():
    M = np.array([[1.0, 0.0, -20.0], [0.0, 1.0, -30.0]])
    assert inside_mask(M, 200, 200, (112, 112)).all()
    frame = _textured(200, 200, 4)
    crop = warp_affine_fixed(frame, M, (112, 112))
    assert np.array_equal(crop, frame[30:142, 20:132])
    f = _face(ARCFACE_112 + np.float32([20, 30]))
    q = quality(crop, f, M, 200, 200)
    assert q["coverage"] == 1.0 and q["sharpness"] > 1000


def test_a_crop_hanging_off_an_edge_counts_its_inside_pixels():
    # crop x = frame x - 150 on a 200-wide frame: columns whose taps x, x + 1 both lie below 200 are x <= 48
    M = np.array([[1.0, 0.0, -150.0], [0.0, 1.0, -10.0]])
    ins = inside_mask(M, 200, 200, (112, 112))
    assert ins[:, :49].all() and not ins[:, 49:].any()
    frame = _textured(200, 200, 5)
    crop = warp_affine_fixed(frame, M, (112, 112))
    q = quality(crop, _face(ARCFACE_112 + np.float32([150, 10])), M, 200, 200)
    assert q["coverage"] == 49 * 112 / (112 * 112)
    # sharpness from the inside pixels only: the black part contributes nothing
    g = grey(crop)
    L = laplacian(g)[:, :47]
    N = L.size
    assert q["sharpness"] == float(N * int((L * L).sum()) - int(L.sum()) ** 2) / (float(N) * float(N))


def _track(tid, state, det, hits, age, face):
    return dict(id=tid, state=state, det=det, hits=hits, age=age, face=face)


def test_oracle_selection_on_a_scripted_history():
    """Tie keeps the earlier frame, a better frame replaces, TENTATIVE never emits, LOST-and-removed emits on its removal frame with
    hits and age + 1, min_quality filters, finish emits live confirmed tracks in id order."""
    frame = _textured(400, 400, 6)
    blurred = cv2.GaussianBlur(frame, (0, 0), 2)
    lm = ARCFACE_112.astype(np.float64) + 100
    f = _face(lm)
    M = similarity_closed(f[5:15].reshape(2, 5).T, ARCFACE_112)
    sharp_crop, blur_crop = warp_affine_fixed(frame, M, (112, 112)), warp_affine_fixed(blurred, M, (112, 112))
    qs, qb = quality(sharp_crop, f, M, 400, 400)["q"], quality(blur_crop, f, M, 400, 400)["q"]
    assert qs > qb > 0
    o = BestShotOracle()
    upd = lambda tracks, crops: o.update(0, tracks, crops, [M] * len(crops), 400, 400)   # noqa: E731
    # frame 0: track 1 (blurred), frame 1: a tie, frame 2: sharp, frame 3: blurred again; track 2 tentative on frame 1 only
    assert upd([_track(1, CONFIRMED, 0, 1, 1, f)], [blur_crop]) == []
    assert upd([_track(1, CONFIRMED, 0, 2, 2, f), _track(2, TENTATIVE, 1, 1, 1, f)], [blur_crop, sharp_crop]) == []
    assert upd([_track(1, CONFIRMED, 0, 3, 3, f)], [sharp_crop]) == []          # track 2 removed while TENTATIVE: no shot
    assert upd([_track(1, CONFIRMED, 0, 4, 4, f), _track(3, CONFIRMED, 1, 1, 1, f)], [blur_crop, blur_crop]) == []
    assert upd([_track(1, LOST, -1, 4, 5, f), _track(3, CONFIRMED, 0, 2, 2, f)], [blur_crop]) == []
    out = upd([_track(3, CONFIRMED, 0, 3, 3, f)], [blur_crop])                   # track 1 removed on frame 5
    assert [(s["id"], s["frame"], s["end_frame"], s["hits"], s["age"], s["reason"]) for s in out] == [(1, 2, 5, 4, 6, BEST_EXIT)]
    assert out[0]["quality"] == np.float32(qs) and np.array_equal(out[0]["crop"], sharp_crop)
    # a tie keeps the earlier frame: track 3's frames 3..5 are all blurred, the shot is frame 3's
    fin = o.finish(0)
    assert [(s["id"], s["frame"], s["end_frame"], s["reason"]) for s in fin] == [(3, 3, 5, BEST_FINISH)]
    assert o.finish(0) == [] and o.v[0]["frames"] == 0
    # min_quality above every q: nothing is emitted
    o = BestShotOracle(min_quality=1.0)
    o.update(0, [_track(1, CONFIRMED, 0, 1, 1, f), _track(2, CONFIRMED, 1, 1, 1, f)], [sharp_crop, sharp_crop], [M, M], 400, 400)
    assert o.update(0, [_track(2, LOST, -1, 1, 2, f)], [], [], 400, 400) == []
    assert o.finish(0) == []


def test_ctypes_layout_matches_header(built_lib, tmp_path):
    from retinaface_b200 import capi
    src = tmp_path / "lay.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rf_b200.h"\nint main(void){\n'
                   'printf("%zu %zu %zu %zu %zu %zu %zu %zu\\n", sizeof(rf_best_shot), offsetof(rf_best_shot, end_frame),'
                   ' offsetof(rf_best_shot, quality), offsetof(rf_best_shot, coverage), offsetof(rf_best_shot, face),'
                   ' sizeof(rf_best_config), offsetof(rf_best_config, min_quality), offsetof(rf_best_config, sharp_half));\n'
                   'printf("%d %d\\n", RF_BEST_EXIT, RF_BEST_FINISH);\nreturn 0;}\n')
    exe = tmp_path / "lay"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    S, B = capi.BestShot, capi.BestConfig
    assert got == [C.sizeof(S), S.end_frame.offset, S.quality.offset, S.coverage.offset, S.face.offset, C.sizeof(B), B.min_quality.offset,
                   B.sharp_half.offset, capi.BEST_EXIT, capi.BEST_FINISH]
    assert capi.BEST_DTYPE.itemsize == C.sizeof(S) and capi.BEST_DTYPE.fields["face"][1] == S.face.offset
    assert set(("rf_tracker_create_best", "rf_detect_yuv_track_best_device", "rf_tracker_finish")) <= set(capi.EXPORTS)


def test_best_kernels_compile_for_sm90a_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, CSRC, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "best.cu"), "-o",
                                                   str(tmp_path / "b.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for k in ("k_best_measure", "k_best_select", "k_best_emit", "k_best_commit", "k_best_finish"):
        assert k in r.stderr, k
    assert r.stderr.count("0 bytes spill stores") >= 5 and "bytes spill stores" not in r.stderr.replace("0 bytes spill stores", ""), r.stderr


def test_best_entry_points_refuse_bad_handles_without_gpu(built_lib):
    from retinaface_b200 import capi
    lib = capi.load_library()
    cfg = capi.TrackConfig(1, 0, 0, 0, 0, 0, 0, 0)
    best = capi.best_config()
    t = C.c_void_p()
    assert lib.rf_tracker_create_best(None, C.byref(cfg), C.byref(best), C.byref(t)) == -1
    assert lib.rf_tracker_finish(None, 0, None, None, None, None) == -1
    assert lib.rf_detect_yuv_track_best_device(None, None, None, None, 0, 0, 0.5, 0.4, None, None, None, None, None, None, None, None,
                                               None) == -1


def test_cpp_shell_compiles_best_shot_calls(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    src = open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.cpp")).read()
    assert "rf_detect_yuv_track_best_device" in src and "rf_tracker_finish" in src and "rf_tracker_create_best" in src
