"""CPU: the f8 surface without a GPU -- the four tiled entry points exported with the ctypes signatures their header prototypes have,
the C++ shell compiling a detectTiled call with crops, and the Python device wrappers refusing host arrays before any call."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT

NEW = ("rf_detect_tiled_align", "rf_detect_yuv_tiled_align", "rf_detect_tiled_device", "rf_detect_yuv_tiled_device")


def _prototype(name):
    """The parameter types of `name` in include/rf_b200.h, whitespace-normalised."""
    text = open(os.path.join(ROOT, "include", "rf_b200.h")).read()
    m = re.search(r"\bint " + name + r"\(([^;]*)\);", text)
    assert m, name
    return [re.sub(r"\s+", " ", p.strip()) for p in m.group(1).split(",")]


def _ctype_of(param):
    """The ctypes type capi should declare for one C parameter."""
    from retinaface_b200 import capi
    t = re.sub(r"\s*\*\s*", "*", re.sub(r"\s*\w+$", "", param))      # the type without the parameter name
    simple = {"rf_handle": C.c_void_p, "int": C.c_int, "float": C.c_float}
    if t in simple:
        return simple[t]
    ptrs = {"const uint8_t*const*": C.POINTER(C.c_void_p), "const int*": C.POINTER(C.c_int), "const rf_tiling*": C.POINTER(capi.Tiling),
            "const rf_align_params*": C.POINTER(capi.AlignParams), "const rf_yuv_frame*": C.POINTER(capi.YuvFrame),
            "const rf_det**": C.POINTER(C.c_void_p), "const int32_t**": C.POINTER(C.c_void_p)}
    if t in ptrs:
        return ptrs[t]
    assert t.endswith("*"), t                      # output arrays and buffers: plain addresses
    return C.c_void_p


def test_entry_points_and_signatures(built_lib):
    from retinaface_b200 import capi
    lib = capi.load_library()
    raw = C.CDLL(built_lib)
    for name in NEW:
        assert name in capi.EXPORTS and hasattr(raw, name), name
        params = _prototype(name)
        want = [_ctype_of(p) for p in params]
        got = getattr(lib, name).argtypes
        assert len(got) == len(want), (name, len(got), len(want))
        for p, g, w in zip(params, got, want):
            assert g == w, (name, p, g, w)


def test_cpp_shell_compiles_a_detect_tiled_call_with_crops(built_lib, tmp_path):
    from retinaface_b200.build import build_host
    build_host()
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "tiled_align_call.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    string dir = argc > 1 ? argv[1] : ".";\n'
                   '    RetinaFace rf(dir);\n'
                   '    vector<unsigned char> buf(2160 * 3840 * 3, 0);\n'
                   '    vector<Mat> imgs(1, Mat(2160, 3840, CV_8UC3, buf.data(), 3840 * 3));\n'
                   '    AlignOptions align;\n'
                   '    align.max_faces = 4;\n'
                   '    rf.detectTiled(imgs, 0.9f, vector<float>(), false, 0, &align);\n'
                   '    rf.detectTiled(imgs, 0.9f, vector<float>{1.f, 0.f}, true, 96, &align);\n'
                   '    return (int)rf.lastCrops().size() - 1;\n'
                   '}\n')
    exe = tmp_path / "tiled_align_call"
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", host, "-I", os.path.join(ROOT, "include"), str(src),
                           os.path.join(host, "RetinaFace.cpp"), "-o", str(exe), "-L", os.path.dirname(built_lib), "-lrf_b200",
                           "-Wl,-rpath," + os.path.dirname(built_lib)])
    assert os.path.exists(exe)


def test_device_wrappers_refuse_host_arrays(built_lib):
    from retinaface_b200 import capi
    eng = object.__new__(capi.Engine)        # no handle: the wrappers must refuse before calling the library
    eng.lib, eng.h = capi.load_library(), None
    img = np.zeros((64, 96, 3), np.uint8)
    frame = np.zeros((96, 64), np.uint8)
    with pytest.raises(ValueError):
        eng.detect_tiled_device([img], 0.5, 0.4)
    with pytest.raises(ValueError):
        eng.detect_yuv_tiled_device([frame], 0.5, 0.4)
    with pytest.raises(ValueError):
        eng.detect_yuv_tiled_device([(frame[:64], frame[64:])], 0.5, 0.4, layout="nv12")
    with pytest.raises(ValueError):
        eng.detect_tiled_device([img], 0.5, 0.4, align={}, dev_crops_ptr=0)
