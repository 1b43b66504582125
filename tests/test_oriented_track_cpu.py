"""CPU: f20 oriented videos in tracker calls without a GPU -- the stored frame of a displayed one (unorient_planes, the inverse of
orient_planes) for every orientation and layout, pitched planes included; the stored-address map the redaction kernels use (yuv.cuh
plane_map, restated here as the header states it) against orient_planes at luma and chroma granularity; the new entry points in the
built library and the binding's signature table; and the C++ shell compiling setVideoOrientation.
unorient_planes and orient_planes are oracle/orient.py's."""
import os

import numpy as np
import pytest

from conftest import ROOT
from oracle.orient import orient, orient_planes, unorient_planes

ALL = list(range(1, 9))
BITS = {1: 0, 2: 1, 3: 3, 4: 2, 5: 4, 6: 5, 7: 7, 8: 6}      # EXIF -> LB_FLIP_X 1 | LB_FLIP_Y 2 | LB_TRANSPOSE 4


def plane_map(bits, dw, dh, pitch, step):
    """yuv.cuh plane_map: (off, xs, ys) with displayed sample (x, y) of a dw x dh plane at off + x xs + y ys of its stored plane."""
    fx, fy, tr = bits & 1, bits & 2, bits & 4
    a, b = (pitch, step) if tr else (step, pitch)
    return (a * (dw - 1) if fx else 0) + (b * (dh - 1) if fy else 0), -a if fx else a, -b if fy else b


def _gather(flat, off, xs, ys, dw, dh):
    ys_, xs_ = np.mgrid[0:dh, 0:dw]
    return flat[off + xs_ * xs + ys_ * ys]


@pytest.mark.parametrize("layout", ["nv12", "i420"])
@pytest.mark.parametrize("o", ALL)
@pytest.mark.parametrize("size", [(6, 4), (1282, 722), (20, 34)])
def test_unorient_inverts_orient(layout, o, size):
    w, h = size
    rng = np.random.default_rng(o)
    shown = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    stored = unorient_planes(shown, layout, o)
    assert np.array_equal(orient_planes(stored, layout, o), shown)
    assert np.array_equal(unorient_planes(orient_planes(shown, layout, o), layout, o), shown)


@pytest.mark.parametrize("layout", ["nv12", "i420"])
@pytest.mark.parametrize("o", ALL)
@pytest.mark.parametrize("pitch_pad", [0, 3, 61])
def test_plane_map_is_orient_planes(layout, o, pitch_pad):
    """Displayed luma and chroma samples read through plane_map from pitched stored planes (odd pitches included) equal
    orient_planes of the packed frame, at luma and at chroma granularity."""
    w, h = 14, 10
    rng = np.random.default_rng(10 * o + pitch_pad)
    frame = rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    shown = orient_planes(frame, layout, o)
    bits = BITS[o]
    dw, dh = (h, w) if bits & 4 else (w, h)
    yp = w + pitch_pad
    luma = np.zeros(yp * h, np.uint8)
    luma.reshape(h, yp)[:, :w] = frame[:h]
    assert np.array_equal(_gather(luma, *plane_map(bits, dw, dh, yp, 1), dw, dh), shown[:dh])
    if layout == "nv12":
        cp = w + pitch_pad
        chroma = np.zeros(cp * (h // 2), np.uint8)
        chroma.reshape(h // 2, cp)[:, :w] = frame[h:]
        off, xs, ys = plane_map(bits, dw // 2, dh // 2, cp, 2)
        pairs = shown[dh:].reshape(dh // 2, dw // 2, 2)
        assert np.array_equal(_gather(chroma, off, xs, ys, dw // 2, dh // 2), pairs[..., 0])           # U
        assert np.array_equal(_gather(chroma, off + 1, xs, ys, dw // 2, dh // 2), pairs[..., 1])       # V
    else:
        cp = w // 2 + pitch_pad
        q = (h // 2) * (w // 2)
        flat = frame[h:].reshape(-1)
        sq = (dh // 2) * (dw // 2)
        shown_c = shown[dh:].reshape(-1)
        for k in range(2):
            plane = np.zeros(cp * (h // 2), np.uint8)
            plane.reshape(h // 2, cp)[:, :w // 2] = flat[k * q:(k + 1) * q].reshape(h // 2, w // 2)
            got = _gather(plane, *plane_map(bits, dw // 2, dh // 2, cp, 1), dw // 2, dh // 2)
            assert np.array_equal(got, shown_c[k * sq:(k + 1) * sq].reshape(dh // 2, dw // 2))


def test_plane_map_matches_the_header_table():
    """Luma through plane_map is A_o of rf_b200.h's f9 table, sample by sample."""
    from test_oriented_cpu import stored_of
    w, h = 7, 5
    stored = np.arange(w * h, dtype=np.int32).reshape(h, w)
    for o in ALL:
        bits = BITS[o]
        dw, dh = (h, w) if bits & 4 else (w, h)
        shown = _gather(stored.reshape(-1), *plane_map(bits, dw, dh, w, 1), dw, dh)
        ys, xs = np.mgrid[0:dh, 0:dw]
        sx, sy = stored_of(o, xs, ys, w, h)
        assert np.array_equal(shown, stored[sy, sx]) and np.array_equal(shown, orient(stored, o)), o


def test_new_entry_points_are_exported(built_lib):
    import ctypes as C
    from retinaface_b200 import capi
    lib = C.CDLL(built_lib)
    for name in ("rf_tracker_set_orientation", "rf_redact_yuv_oriented_device_style"):
        assert hasattr(lib, name) and name in capi.EXPORTS, name
    with open(os.path.join(ROOT, "include", "rf_b200.h")) as f:
        hdr = f.read()
    assert "int rf_tracker_set_orientation(rf_tracker t, int video, int orientation);" in hdr
    assert "int rf_redact_yuv_oriented_device_style(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n," in hdr


def test_cpp_shell_compiles_set_video_orientation(built_lib, tmp_path):
    import subprocess
    from retinaface_b200.build import build_host
    build_host()
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "oriented_track.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    string dir = argv[1];\n'
                   '    RetinaFace rf(dir);\n'
                   '    rf.setVideoOrientation(0, 6);\n'
                   '    rf.setVideoOrientation(-1, 1);\n'
                   '    return 0;\n'
                   '}\n')
    subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-I", host, "-I", os.path.join(ROOT, "include"), str(src)])
