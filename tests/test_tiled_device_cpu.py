"""CPU: the f8 surface without a GPU -- the C++ shell compiling a detectTiled call with crops, and the Python device wrappers refusing
host arrays before any call (the four tiled entry points' signatures are checked in test_signatures_cpu.py)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

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
