"""CPU: the YUV 4:2:0 oracle (oracle/yuv.py) against cv2.cvtColor and the BT.709 matrix, the single-buffer / plane descriptors
capi.py builds, and the C-ABI surface of f6 (exported symbols, rf_yuv_frame layout, the C++ shell's detectYUV)."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from conftest import ROOT
from oracle.yuv import (BT709, LAYOUTS, bgr_to_frame, float_bgr, frame_to_bgr, limited_range_coefficients, planes_to_bgr,
                        split_planes, yuv_to_bgr_samples)

CODES = dict(nv12=cv2.COLOR_YUV2BGR_NV12, nv21=cv2.COLOR_YUV2BGR_NV21, i420=cv2.COLOR_YUV2BGR_I420, yv12=cv2.COLOR_YUV2BGR_YV12)


def test_bt601_equals_cv2_on_every_triple():
    """All 2^24 (Y, U, V) triples as one 4096 x 4096 NV12 frame: chroma block b carries (U, V) = divmod(b >> 6, 256) and its four
    luma samples 4 (b & 63) .. 4 (b & 63) + 3, so the 64 blocks of one (U, V) pair hold every Y once."""
    b = np.arange(1 << 22, dtype=np.int64).reshape(2048, 2048)
    uv, k = b >> 6, b & 63
    y = np.empty((4096, 4096), np.uint8)
    for dy in range(2):
        for dx in range(2):
            y[dy::2, dx::2] = 4 * k + 2 * dy + dx
    chroma = np.stack([uv >> 8, uv & 255], axis=-1).astype(np.uint8).reshape(2048, 4096)
    frame = np.concatenate([y, chroma])
    assert np.array_equal(frame_to_bgr(frame, "nv12"), cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_NV12))


@pytest.mark.parametrize("layout", LAYOUTS)
def test_layouts_equal_cv2_on_odd_quarter_sizes(layout):
    """1282 x 722 (both = 2 mod 4: the planar chroma planes do not split into whole rows of w) with random bytes, and frames made
    from a BGR image the way test inputs are."""
    rng = np.random.default_rng(11)
    frame = rng.integers(0, 256, (722 * 3 // 2, 1282), dtype=np.uint8)
    assert np.array_equal(frame_to_bgr(frame, layout), cv2.cvtColor(frame, CODES[layout]))
    img = rng.integers(0, 256, (240, 320, 3), dtype=np.uint8)
    made = bgr_to_frame(img, layout)
    assert made.shape == (360, 320)
    assert np.array_equal(frame_to_bgr(made, layout), cv2.cvtColor(made, CODES[layout]))
    assert np.array_equal(frame_to_bgr(made, layout), frame_to_bgr(bgr_to_frame(img, "i420"), "i420"))


def test_pitched_planes_equal_packed():
    """Planes cut out of wider allocations (non-zero padding) convert like the packed frame."""
    rng = np.random.default_rng(5)
    frame = rng.integers(0, 256, (180 * 3 // 2, 200), dtype=np.uint8)
    y, u, v = split_planes(frame, "i420")
    pad = [np.full((a.shape[0], a.shape[1] + 37), 0xEE, np.uint8) for a in (y, u, v)]
    for p, a in zip(pad, (y, u, v)):
        p[:, :a.shape[1]] = a
    views = [p[:, :a.shape[1]] for p, a in zip(pad, (y, u, v))]
    assert np.array_equal(planes_to_bgr(*views), cv2.cvtColor(frame, cv2.COLOR_YUV2BGR_I420))


def test_bt709_constants_and_bound_against_the_float_matrix():
    assert limited_range_coefficients(0.2126, 0.0722) == BT709
    a = np.arange(1 << 24, dtype=np.int64)
    y, u, v = a >> 16, (a >> 8) & 255, a & 255
    d = np.abs(yuv_to_bgr_samples(y, u, v, "bt709").astype(np.int16) - float_bgr(y, u, v, 0.2126, 0.0722).astype(np.int16))
    assert d.max() <= 1
    assert (d.max(axis=1) > 0).mean() <= 1e-4


def test_capi_descriptors_of_every_form():
    from retinaface_b200 import capi
    h, w = 6, 8
    buf = np.arange(h * 3 // 2 * w, dtype=np.uint8).reshape(h * 3 // 2, w)
    p = buf.ctypes.data
    want = {"nv12": (p, p + 48, p + 49, 8, 8, 2), "nv21": (p, p + 49, p + 48, 8, 8, 2),
            "i420": (p, p + 48, p + 60, 8, 4, 1), "yv12": (p, p + 60, p + 48, 8, 4, 1)}
    for layout, (y, u, v, yp, uvp, step) in want.items():
        f, dev = capi.yuv_frame(buf, layout)
        assert not dev and (f.y, f.u, f.v, f.y_pitch, f.uv_pitch, f.uv_step, f.width, f.height) == (y, u, v, yp, uvp, step, w, h), layout
    big = np.zeros((20, 64), np.uint8)
    yv, uvv = big[:6, 3:11], big[10:13, 5:13]
    f, _ = capi.yuv_frame((yv, uvv), "nv21")
    assert (f.y, f.v, f.u, f.y_pitch, f.uv_pitch, f.uv_step) == (yv.ctypes.data, uvv.ctypes.data, uvv.ctypes.data + 1, 64, 64, 2)
    f, _ = capi.yuv_frame((yv, big[10:13, 0:4], big[14:17, 0:4]), "i420")
    assert (f.uv_step, f.uv_pitch, f.u, f.v) == (1, 64, big[10:].ctypes.data, big[14:].ctypes.data)
    for bad in (buf[:, :7], np.zeros((10, 8), np.uint8), buf[::2]):
        with pytest.raises(ValueError):
            capi.yuv_frame(bad, "nv12")
    with pytest.raises(ValueError):
        capi.yuv_frame(buf, "yuyv")
    with pytest.raises(ValueError):
        capi.yuv_frame((yv, uvv), "i420")


def test_yuv_entry_points_and_frame_layout(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = C.CDLL(built_lib)
    for name in ("rf_detect_yuv_batch", "rf_detect_yuv_batch_device", "rf_preprocess_yuv"):
        assert name in capi.EXPORTS and hasattr(lib, name), name
    src = tmp_path / "layout.c"
    fields = ("y", "u", "v", "y_pitch", "uv_pitch", "uv_step", "width", "height")
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rf_b200.h"\n'
                   'int main(void) { printf("%zu' + " %zu" * len(fields) + ' %d %d\\n", sizeof(rf_yuv_frame), '
                   + ", ".join(f"offsetof(rf_yuv_frame, {f})" for f in fields) + ", RF_YUV_BT601, RF_YUV_BT709); return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(t) for t in subprocess.check_output([str(exe)], text=True).split()]
    F = capi.YuvFrame
    assert got == [C.sizeof(F)] + [getattr(F, f).offset for f in fields] + [capi.RF_YUV_BT601, capi.RF_YUV_BT709]


def test_cpp_shell_compiles_a_detect_yuv_call(built_lib, tmp_path):
    from retinaface_b200.build import build_host
    build_host()
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "yuv_call.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    string dir = argc > 1 ? argv[1] : ".";\n'
                   '    RetinaFace rf(dir);\n'
                   '    vector<unsigned char> buf(1080 * 3 / 2 * 1920, 128);\n'
                   '    vector<Mat> frames(1, Mat(1080 * 3 / 2, 1920, CV_8UC1, buf.data(), 1920));\n'
                   '    AlignOptions a;\n'
                   '    rf.detectYUV(frames, RetinaFace::YUV_NV12, 0.9f, &a);\n'
                   '    rf.detectYUV(frames, RetinaFace::YUV_I420, 0.9f);\n'
                   '    return (int)rf.lastBatchFaces().size() + (int)rf.lastCrops().size() - 2;\n'
                   '}\n')
    exe = tmp_path / "yuv_call"
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", host, "-I", os.path.join(ROOT, "include"), str(src),
                           os.path.join(host, "RetinaFace.cpp"), "-o", str(exe), "-L", os.path.dirname(built_lib), "-lrf_b200",
                           "-Wl,-rpath," + os.path.dirname(built_lib)])
    assert os.path.exists(exe)
