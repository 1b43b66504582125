"""f24 rotated views of device frames without a GPU: the exported signatures of the new entry points, the YUV view oracle (a warp view
of cv2.cvtColor(frame)) for every layout and matrix, and the angle sweep detectAnyAngle and detectAnyAngleFrames share, in Python and in
the C++ shell."""
import ctypes as C
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from conftest import ROOT
from oracle import rotate, yuv
from test_signatures_cpu import _exact_types, _prototypes, _squash

NEW = ("rf_detect_views_rotated_device", "rf_detect_yuv_views_rotated_device", "rf_preprocess_yuv_rotated", "rf_fetch_dets")
CVT = {"nv12": cv2.COLOR_YUV2BGR_NV12, "nv21": cv2.COLOR_YUV2BGR_NV21, "i420": cv2.COLOR_YUV2BGR_I420, "yv12": cv2.COLOR_YUV2BGR_YV12}


def test_new_prototypes_have_exact_signatures(built_lib):
    """Structures by class, input arrays typed, outputs as addresses."""
    from retinaface_b200 import capi
    protos, _ = _prototypes()
    exact = dict(_exact_types(), **{"const rf_rotated_view*": C.POINTER(capi._RotatedView)})
    lib = capi.load_library()
    for name in NEW:
        ret, params = protos[name]
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == len(params), name
        for p, got in zip(params, fn.argtypes):
            t = _squash(re.sub(r"\s*\w+$", "", p))
            want = exact.get(_squash(p), exact.get(t, C.c_void_p))
            assert t in exact or t.endswith("*"), (name, p)
            assert got == want, (name, p, got, want)


def _frame(golden_image, size):
    return cv2.resize(golden_image, size)


@pytest.mark.parametrize("layout", yuv.LAYOUTS)
@pytest.mark.parametrize("angle", (30.0, -60.0, 200.0))
def test_yuv_view_oracle_is_warp_affine_of_cvt_color(golden_image, layout, angle):
    """BT.601: rotate.warp_view on yuv.frame_to_bgr is cv2.warpAffine(cv2.cvtColor(frame), M) byte for byte."""
    frame = yuv.bgr_to_frame(_frame(golden_image, (640, 442)), layout)
    bgr = cv2.cvtColor(frame, CVT[layout])
    assert np.array_equal(yuv.frame_to_bgr(frame, layout, "bt601"), bgr)
    _, _, M = rotate.geometry(angle, 640, 442, 448, 448)
    want = cv2.warpAffine(bgr, M, (448, 448), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(rotate.warp_view(yuv.frame_to_bgr(frame, layout, "bt601"), M, 448, 448), want)


@pytest.mark.parametrize("layout", yuv.LAYOUTS)
def test_bt709_yuv_view_oracle_is_within_one_of_the_float_matrix(golden_image, layout):
    """BT.709 has no cv2.cvtColor: the view of the oracle's conversion is cv2.warpAffine of it, and within 1 of the warp of the
    float-matrix conversion (each tap is within 1, and a bilinear weight set sums to one)."""
    frame = yuv.bgr_to_frame(_frame(golden_image, (640, 442)), layout)
    ours = yuv.frame_to_bgr(frame, layout, "bt709")
    y, u, v = yuv.split_planes(frame, layout)
    up, vp = (np.repeat(np.repeat(c, 2, axis=0), 2, axis=1) for c in (u, v))
    ref = yuv.float_bgr(y, up, vp, 0.2126, 0.0722)
    _, _, M = rotate.geometry(45.0, 640, 442, 448, 448)
    got = rotate.warp_view(ours, M, 448, 448)
    assert np.array_equal(got, cv2.warpAffine(ours, M, (448, 448), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0))
    assert np.abs(got.astype(np.int16) - rotate.warp_view(ref, M, 448, 448).astype(np.int16)).max() <= 1


def test_python_angle_sweep_is_shared_and_refuses_more_than_sixteen_views():
    from retinaface_b200 import RetinaFace
    from retinaface_b200.detector import angle_sweep
    assert angle_sweep(30.0) == [(30.0 * k, 1.0) for k in range(12)]
    assert angle_sweep(22.5) == [(22.5 * k, 1.0) for k in range(16)]
    assert angle_sweep(400.0) == [(0.0, 1.0)]
    det = object.__new__(RetinaFace)          # the step is checked before the engine is used
    for step in (20.0, 1.0, 0.0, -30.0, float("nan")):
        with pytest.raises(ValueError):
            angle_sweep(step)
        with pytest.raises(ValueError):
            det.detectAnyAngleFrames([object()], step=step)
        with pytest.raises(ValueError):
            det.detectAnyAngle(np.zeros((8, 8, 3), np.uint8), step=step)


CPP_SWEEP = r'''
#include "RetinaFace.h"
#include <cstdio>
#include <stdexcept>
// prints the sweep of each step in argv, or "refused" when angleSweep throws
int main(int argc, char **argv) {
    for (int i = 1; i < argc; i++) {
        try {
            const auto v = RetinaFace::angleSweep("detectAnyAngleYUV", (float)atof(argv[i]));
            printf("%zu", v.size());
            for (const auto &x : v) printf(" %g/%g", x.angle, x.shrink);
            printf("\n");
        } catch (const std::invalid_argument &) {
            printf("refused\n");
        }
    }
    return 0;
}
void use(RetinaFace &r, const std::vector<rf_yuv_frame> &f) { r.detectAnyAngleYUV(f, 0.5f, 30.f); }
'''


def test_cpp_shell_angle_sweep(built_lib, tmp_path):
    """RetinaFace::angleSweep, which detectAnyAngle and detectAnyAngleYUV share: 12 views at 30 degrees, 16 at 22.5, and a refusal
    of more than RF_MAX_VIEWS views or a step that is not positive (linked against the library; no GPU is touched)."""
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "sweep.cpp"
    src.write_text(CPP_SWEEP)
    exe = tmp_path / "sweep"
    libdir = os.path.dirname(built_lib)
    subprocess.check_call(["g++", "-std=c++14", "-I", host, "-I", os.path.join(ROOT, "include"), str(src), os.path.join(host, "RetinaFace.cpp"),
                           "-o", str(exe), "-L", libdir, "-lrf_b200", "-Wl,-rpath," + libdir])
    out = subprocess.check_output([str(exe), "30", "22.5", "20", "0", "-5"], text=True).splitlines()
    assert out[0] == "12 " + " ".join(f"{30 * k:g}/1" for k in range(12))
    assert out[1] == "16 " + " ".join(f"{22.5 * k:g}/1" for k in range(16))
    assert out[2:] == ["refused"] * 3
