"""f25 rotated views as a tracker's detector, without a GPU: the exported signature of rf_tracker_set_views, the EXIF composition table
the oriented quarter-turn views read through (all 64 pairs against oracle/orient.py), the resources of the oriented warp instantiation,
the Python surfaces' refusals, and the C++ shell's track_any_angle_step."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle.orient import orient
from test_signatures_cpu import _exact_types, _prototypes, _squash

CSRC = os.path.join(ROOT, "retinaface_b200", "csrc")


def test_set_views_has_an_exact_signature(built_lib):
    from retinaface_b200 import capi
    protos, _ = _prototypes()
    exact = dict(_exact_types(), **{"const rf_rotated_view*": C.POINTER(capi._RotatedView)})
    fn = getattr(capi.load_library(), "rf_tracker_set_views")
    ret, params = protos["rf_tracker_set_views"]
    assert fn.restype is C.c_int and len(fn.argtypes) == len(params) == 3
    for p, got in zip(params, fn.argtypes):
        t = _squash(re.sub(r"\s*\w+$", "", p))
        assert got == exact.get(_squash(p), exact.get(t, C.c_void_p)), p


def _compose_table():
    src = open(os.path.join(CSRC, "preprocess.cuh")).read()
    body = re.search(r"kExifCompose\[8\]\[8\] = \{(.*?)\};", src, re.S).group(1)
    rows = re.findall(r"\{([^{}]*)\}", body)
    return np.array([[int(x) for x in r.split(",")] for r in rows])


def test_exif_composition_table_for_all_64_pairs():
    """T_{table[inner][outer]}(S) = T_outer(T_inner(S)) for every pair, on a non-square array whose every element differs, so that a
    wrong orientation, a wrong transpose or a wrong size cannot pass."""
    table = _compose_table()
    assert table.shape == (8, 8)
    s = np.arange(3 * 5).reshape(3, 5)
    for inner in range(1, 9):
        for outer in range(1, 9):
            want = orient(orient(s, inner), outer)
            got = orient(s, int(table[inner - 1, outer - 1]))
            assert got.shape == want.shape and np.array_equal(got, want), (inner, outer)
    # orientation 1 is the identity on either side, and the LB_* bits round trip through lb_exif
    assert list(table[0]) == list(range(1, 9)) and list(table[:, 0]) == list(range(1, 9))
    src = open(os.path.join(CSRC, "preprocess.cuh")).read()
    bits = [int(eval(b.strip().replace("LB_FLIP_X", "1").replace("LB_FLIP_Y", "2").replace("LB_TRANSPOSE", "4")))
            for b in re.search(r"static const int bits\[9\] = \{-1, (.*?)\};", src, re.S).group(1).split(",")]
    exif = [int(x) for x in re.search(r"static const int exif\[8\] = \{(.*?)\};", src).group(1).split(",")]
    assert [exif[b] for b in bits] == list(range(1, 9))


def test_oriented_warp_instantiation_does_not_spill(built_lib):
    """Every k_letterbox_warp instantiation in the built object, the oriented YUV one included (there is no oriented BGR one): no local
    memory (spills), 56 registers or fewer."""
    obj = os.path.join(CSRC, "build", "preprocess.o")
    out = subprocess.check_output(["/usr/local/cuda/bin/cuobjdump", "-res-usage", obj], text=True)
    found = {}
    lines = out.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function (\S*k_letterbox_warp\S*):", line)
        if m:
            res = lines[i + 1]
            found[m.group(1)] = (int(re.search(r"REG:(\d+)", res).group(1)), int(re.search(r"LOCAL:(\d+)", res).group(1)))
    assert len(found) == 3, found                       # BGR upright, YUV upright and oriented
    assert [k for k in found if "Lb1E" in k and "YuvPlanes" in k] == [k for k in found if "Lb1E" in k] != [], found
    for k, (reg, local) in found.items():
        assert local == 0 and reg <= 56, (k, reg, local)


def test_detector_surfaces_refuse_any_angle_with_tiling():
    from retinaface_b200.detector import RetinaFace
    rf = RetinaFace.__new__(RetinaFace)
    with pytest.raises(ValueError, match="exclusive"):
        rf.trackFrames([], [], any_angle=45, tiling=True)
    with pytest.raises(ValueError, match="exclusive"):
        rf.redactFrames([], [], any_angle=45, tiling={"overlap": 48})
    with pytest.raises(ValueError, match="needs videos"):
        rf.redactFrames([], None, any_angle=45)
    assert RetinaFace._views(None) is None
    assert RetinaFace._views(45) == [(45.0 * k, 1.0) for k in range(8)]
    with pytest.raises(ValueError):
        RetinaFace._views(20)            # 18 views


CPP_SHELL = r'''
#include "RetinaFace.h"
#include <cstdio>
#include <stdexcept>
// Compiles the option, and runs the shared sweep the option uses (no GPU is touched).
static void sweep(float step) {
    try {
        const vector<rf_rotated_view> v = RetinaFace::angleSweep("track_any_angle_step", step);
        printf("%d", (int)v.size());
        for (const auto &x : v) printf(" %g/%g", x.angle, x.shrink);
        printf("\n");
    } catch (const std::invalid_argument &e) { printf("refused %s\n", e.what()); }
}
int main() {
    RetinaFaceOptions opt;
    printf("%g\n", opt.track_any_angle_step);
    opt.track_any_angle_step = 45.f;
    sweep(opt.track_any_angle_step);
    sweep(-1.f);
    return 0;
}
'''


def test_cpp_shell_track_any_angle_step(built_lib, tmp_path):
    """RetinaFaceOptions::track_any_angle_step defaults to 0 (off); at 45 the tracker's views are detectAnyAngleYUV's eight."""
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "opt.cpp"
    src.write_text(CPP_SHELL)
    exe = tmp_path / "opt"
    libdir = os.path.dirname(built_lib)
    subprocess.check_call(["g++", "-std=c++14", "-I", host, "-I", os.path.join(ROOT, "include"), str(src), os.path.join(host, "RetinaFace.cpp"),
                           "-o", str(exe), "-L", libdir, "-lrf_b200", "-Wl,-rpath," + libdir])
    out = subprocess.check_output([str(exe)], text=True).splitlines()
    assert out[0] == "0"
    assert out[1] == "8 " + " ".join(f"{45 * k:g}/1" for k in range(8))
    assert out[2] == "refused track_any_angle_step: step_deg must be positive"
