"""CPU: the face-alignment oracle (oracle/align.py) against OpenCV and skimage's estimator form, and the C-ABI surface of
rf_detect_align_batch (exported symbols, rf_align_params layout as capi.py declares it)."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np

from conftest import ROOT
from oracle.align import ARCFACE_112, similarity_closed, umeyama, warp_affine_fixed


def _cv2_warp(img, M, size):
    return cv2.warpAffine(img, M, size, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def test_fixed_point_warp_equals_cv2_on_random_similarities():
    """Random rotations / scales / translations into crops of 8..160 px, many of them hanging off one or more image edges
    (translations place the crop across every border), and identity-like warps at every 1/32 sub-pixel phase."""
    rng = np.random.default_rng(7)
    img = rng.integers(0, 256, (173, 251, 3), dtype=np.uint8)
    off_edge = 0
    for _ in range(400):
        s, th = rng.uniform(0.15, 4.0), rng.uniform(-np.pi, np.pi)
        cw, ch = int(rng.integers(8, 161)), int(rng.integers(8, 161))
        M = np.array([[s * np.cos(th), -s * np.sin(th), 0.0], [s * np.sin(th), s * np.cos(th), 0.0]])
        # a source point anywhere from beyond the left / top edge to beyond the right / bottom edge maps to the crop centre
        sx, sy = rng.uniform(-60, img.shape[1] + 60), rng.uniform(-60, img.shape[0] + 60)
        M[:, 2] = np.array([cw / 2, ch / 2]) - M[:, :2] @ np.array([sx, sy])
        want = _cv2_warp(img, M, (cw, ch))
        assert np.array_equal(warp_affine_fixed(img, M, (cw, ch)), want)
        off_edge += int((want == 0).all(axis=2).any())
    assert off_edge > 100
    small = rng.integers(0, 256, (5, 6, 3), dtype=np.uint8)
    for fy in range(32):
        for fx in range(32):
            M = np.array([[1.0, 0.0, -(1 + fx / 32)], [0.0, 1.0, -(2 + fy / 32)]])
            assert np.array_equal(warp_affine_fixed(small, M, (6, 5)), _cv2_warp(small, M, (6, 5))), (fx, fy)


def test_closed_form_equals_umeyama():
    rng = np.random.default_rng(3)
    worst = 0.0
    for k in range(300):
        q = ARCFACE_112 * (128 / 112) if k % 2 else ARCFACE_112
        p = (rng.uniform(0, 2000, 2) + rng.uniform(-150, 150, (5, 2))).astype(np.float32)
        a, b = umeyama(p, q), similarity_closed(p, q)
        worst = max(worst, float(np.abs(a - b).max() / np.abs(a).max()))
    assert worst < 1e-12, worst
    assert not similarity_closed(np.full((5, 2), 7.0), ARCFACE_112).any()   # coincident landmarks: all zeros


def test_align_entry_points_and_params_layout(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = C.CDLL(built_lib)
    for name in ("rf_detect_align_batch", "rf_detect_align_batch_device"):
        assert name in capi.EXPORTS and hasattr(lib, name), name
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rf_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu %d %d %d\\n", sizeof(rf_align_params),'
                   ' offsetof(rf_align_params, crop_w), offsetof(rf_align_params, crop_h), offsetof(rf_align_params, template_xy),'
                   ' offsetof(rf_align_params, max_faces), offsetof(rf_align_params, format), offsetof(rf_align_params, mean),'
                   ' offsetof(rf_align_params, std), RF_CROP_BGR_U8, RF_CROP_RGB_F32, RF_CROP_RGB_F16); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    P = capi.AlignParams
    want = [C.sizeof(P)] + [getattr(P, f).offset for f in ("crop_w", "crop_h", "template_xy", "max_faces", "format", "mean", "std")]
    want += [capi.RF_CROP_BGR_U8, capi.RF_CROP_RGB_F32, capi.RF_CROP_RGB_F16]
    assert got == want
    p = capi.align_params(crop=(96, 112), template=ARCFACE_112 - [8, 0], fmt="rgb_f16", max_faces=3)
    assert (p.crop_w, p.crop_h, p.max_faces, p.format) == (96, 112, 3, capi.RF_CROP_RGB_F16)
    assert np.allclose(np.array(p.template_xy).reshape(5, 2), ARCFACE_112 - [8, 0])
    assert capi.crop_shape("rgb_f32", (96, 112)) == ((3, 112, 96), np.float32)
    assert capi.crop_shape("bgr_u8", (0, 0)) == ((112, 112, 3), np.uint8)
