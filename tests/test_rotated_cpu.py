"""f23 rotated views without a GPU: oracle/rotate.py's geometry against cv2 and the kernel's fixed-point warp, the angle classification,
the map-back as the inverse of M, the recall gain of a rotated view on a tilted photo with the CPU network and post-process oracles, the
exported signatures and the C++ shell's new call."""
import ctypes as C
import math
import os
import re
import subprocess

import cv2
import numpy as np
import pytest

from conftest import ROOT, caffemodel
from oracle import rotate
from oracle.align import warp_affine_fixed
from test_signatures_cpu import _exact_types, _prototypes, _squash

ANGLES = (7.5, 30.0, 45.0, 135.0, -60.0, 359.9)


@pytest.mark.parametrize("angle", ANGLES)
def test_warp_view_is_cv2_warp_affine_of_the_rotation(golden_image, angle):
    """M is cv2.getRotationMatrix2D's rotation about the image centre at scale f, moved to the box's top-left; the view's bytes are
    the kernel's fixed-point warp (oracle.align) of that M, byte for byte."""
    h, w = golden_image.shape[:2]
    o, f, M = rotate.geometry(angle, w, h, 448, 448)
    assert o == 0 and 0 < f <= 1
    R = cv2.getRotationMatrix2D(((w - 1) / 2, (h - 1) / 2), float(np.float32(angle)), f)
    assert np.allclose(M[:, :2], R[:, :2], rtol=0, atol=1e-12)
    shift = M[:, 2] - R[:, 2]
    a = rotate.reduce_angle(angle) * math.pi / 180
    wr, hr = abs(math.cos(a)) * w + abs(math.sin(a)) * h, abs(math.sin(a)) * w + abs(math.cos(a)) * h
    centre = M @ np.array([(w - 1) / 2, (h - 1) / 2, 1.0])
    assert np.allclose(centre, [(f * wr - 1) / 2, (f * hr - 1) / 2], atol=1e-9) and np.isfinite(shift).all()
    view = rotate.warp_view(golden_image, M, 448, 448)
    assert np.array_equal(view, warp_affine_fixed(golden_image, M, (448, 448)))
    assert view.any() and not view[int(math.ceil(f * hr)) + 1:].any() and not view[:, int(math.ceil(f * wr)) + 1:].any()


@pytest.mark.parametrize("size", [(1280, 886), (300, 200), (3840, 2160), (1, 1), (17, 900)])
@pytest.mark.parametrize("shrink", [1.0, 0.6, 0.05])
def test_image_corners_land_inside_the_shrink_box(size, shrink):
    w, h = size
    for net in ((448, 448), (1280, 896)):
        bw, bh = rotate.shrink_box(net[0], net[1], shrink)
        for angle in ANGLES + (200.0, 1.0, 89.0, 271.5):
            o, f, M = rotate.geometry(angle, w, h, bw, bh)
            assert o == 0 and f <= 1
            corners = np.array([[0, 0, 1], [w - 1, 0, 1], [0, h - 1, 1], [w - 1, h - 1, 1]], np.float64).T
            p = M @ corners
            assert (p[0] >= -0.5 - 1e-9).all() and (p[0] <= bw - 0.5 + 1e-9).all(), (size, angle, p)
            assert (p[1] >= -0.5 - 1e-9).all() and (p[1] <= bh - 0.5 + 1e-9).all(), (size, angle, p)
            if (w, h) == (300, 200) and shrink == 1.0:
                assert f == 1.0, (net, angle)      # the rotated 300x200 image fits: never up-scaled


def test_angle_classification():
    for angle, o in ((0, 1), (90, 8), (180, 3), (270, 6), (-90, 6), (450, 8), (360, 1), (-360, 1), (-0.0, 1), (720, 1), (-1e-30, 1)):
        assert rotate.geometry(angle, 640, 480, 448, 448)[0] == o, angle
    for angle in (359.999, 0.001, 89.99, 45.0, -45.0, 1e-5):
        assert rotate.geometry(angle, 640, 480, 448, 448)[0] == 0, angle


@pytest.mark.parametrize("angle", ANGLES + (200.0,))
def test_map_back_inverts_m(angle):
    """Landmarks and a face box carried into the view by M (rounded to float) map back within 1e-3 px; the box keeps its size."""
    rng = np.random.default_rng(int(abs(angle) * 10))
    w, h = 1280, 886
    o, f, M = rotate.geometry(angle, w, h, 448, 448)
    rows = []
    truth = []
    for _ in range(20):
        cx, cy, s = rng.uniform(100, w - 100), rng.uniform(100, h - 100), rng.uniform(20, 90)
        lm = np.stack([cx + rng.uniform(-s, s, 5) / 2, cy + rng.uniform(-s, s, 5) / 2], 1)
        v = (M @ np.vstack([lm.T, np.ones(5)])).T
        vc = M @ np.array([cx, cy, 1.0])
        half = s * f / 2
        rows.append(np.concatenate([[0.9], [vc[0] - half, vc[1] - half, vc[0] + half, vc[1] + half], v[:, 0], v[:, 1]]).astype(np.float32))
        truth.append((cx, cy, s, lm))
    back = rotate.map_back(np.stack(rows), M, f)
    for r, (cx, cy, s, lm) in zip(back, truth):
        assert np.allclose(r[5:10], lm[:, 0], atol=1e-3) and np.allclose(r[10:15], lm[:, 1], atol=1e-3)
        assert np.allclose([(r[1] + r[3]) / 2, (r[2] + r[4]) / 2], [cx, cy], atol=1e-3)
        assert np.allclose([r[3] - r[1], r[4] - r[2]], [s, s], atol=1e-3)


def _count(net, post, img):
    from oracle.mnet_numpy import preprocess_bgr_u8
    from oracle.topology import OUTPUT_BLOBS
    net.setInput(preprocess_bgr_u8(img))
    heads = [o[0] for o in net.forward(OUTPUT_BLOBS)]
    return len(post.postprocess(heads, 448, 448, 0.5, 0.4)["faces"])


def test_rotated_view_recovers_a_tilted_photo(golden_image):
    """The golden photo tilted 45 degrees counter-clockwise onto an expanded canvas: its plain letter-box finds at most one face, the
    view rotated back by the tilt at least four (cv2.dnn on the committed model, the C post-process oracle)."""
    from oracle.inputs import letterbox_bgr_u8
    from oracle.postproc import PostprocOracle
    h, w = golden_image.shape[:2]
    R = cv2.getRotationMatrix2D((w / 2, h / 2), 45.0, 1.0)
    c, s = abs(R[0, 0]), abs(R[0, 1])
    W, H = int(h * s + w * c), int(h * c + w * s)
    R[0, 2] += W / 2 - w / 2
    R[1, 2] += H / 2 - h / 2
    tilted = cv2.warpAffine(golden_image, R, (W, H))
    net = cv2.dnn.readNetFromCaffe(os.path.join(ROOT, "tests", "golden", "weights", "mnet25.prototxt"), caffemodel("mnet25"))
    post = PostprocOracle()
    plain = _count(net, post, letterbox_bgr_u8(tilted, 448, 448))
    o, f, M = rotate.geometry(-45.0, W, H, 448, 448)
    back = _count(net, post, rotate.warp_view(tilted, M, 448, 448))
    print(f"\n45 degree tilt: {plain} faces plain, {back} in the -45 degree view")
    assert plain <= 1 and back >= 4


def test_new_prototypes_have_exact_signatures(built_lib):
    from retinaface_b200 import capi
    protos, _ = _prototypes()
    exact = dict(_exact_types(), **{"const rf_rotated_view*": C.POINTER(capi._RotatedView)})
    lib = capi.load_library()
    for name in ("rf_detect_views_rotated", "rf_preprocess_rotated"):
        ret, params = protos[name]
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == len(params), name
        for p, got in zip(params, fn.argtypes):
            t = _squash(re.sub(r"\s*\w+$", "", p))              # the type without the parameter name
            want = exact.get(_squash(p), exact.get(t, C.c_void_p))
            assert t in exact or t.endswith("*"), (name, p)
            assert got == want, (name, p, got, want)


def test_cpp_shell_compiles_detect_any_angle(tmp_path):
    """RetinaFace::detectAnyAngle is declared and defined: the C++ shell compiles (no link, no GPU)."""
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "use.cpp"
    src.write_text('#include "RetinaFace.h"\nvoid use(RetinaFace &r, const cv::Mat &m) {\n'
                   '    AlignOptions a;\n    auto f = r.detectAnyAngle(m, 0.5f, 30.f, &a);\n    (void)f;\n}\n')
    for cpp in (str(src), os.path.join(host, "RetinaFace.cpp")):
        subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-I", host, "-I", os.path.join(ROOT, "include"), cpp])


def test_detect_any_angle_refuses_more_than_sixteen_views():
    from retinaface_b200 import RetinaFace
    det = object.__new__(RetinaFace)          # the step is checked before the engine is used
    img = np.zeros((8, 8, 3), np.uint8)
    for step in (20.0, 1.0, 0.0, -30.0):
        with pytest.raises(ValueError):
            det.detectAnyAngle(img, step=step)
