"""CPU: f21 oriented tiled detection without a GPU -- a mirrored level of the displayed image read through the composed LB bits
(lb_orientation_bits(o) ^ LB_FLIP_X, restated here) against cv2.flip(orient(img, o), 1), the layout of a portrait 4K frame from the
tiling rule, the exact ctypes signatures of the five f21 entry points, and the C++ shell compiling the detectTiled overload."""
import ctypes as C
import os
import re

import cv2
import numpy as np
import pytest

from conftest import ROOT
from oracle.orient import orient
from test_signatures_cpu import _exact_types, _prototypes, _squash

LB_FLIP_X, LB_FLIP_Y, LB_TRANSPOSE = 1, 2, 4
BITS = {1: 0, 2: LB_FLIP_X, 3: LB_FLIP_X | LB_FLIP_Y, 4: LB_FLIP_Y, 5: LB_TRANSPOSE, 6: LB_TRANSPOSE | LB_FLIP_X,
        7: LB_TRANSPOSE | LB_FLIP_X | LB_FLIP_Y, 8: LB_TRANSPOSE | LB_FLIP_Y}      # preprocess.cuh lb_orientation_bits
F21 = ("rf_detect_tiled_oriented", "rf_detect_tiled_oriented_device", "rf_detect_yuv_tiled_oriented_device", "rf_preprocess_tile_oriented",
       "rf_preprocess_yuv_tile_oriented")


def read_displayed(stored, bits):
    """The displayed image an LbItem with `bits` reads (preprocess.cu col_of / row_of / stored_pixel): displayed (x, y) of the
    sw x sh displayed frame reads x' = FLIP_X ? sw-1-x : x, y' = FLIP_Y ? sh-1-y : y, at stored column y', row x' when TRANSPOSE."""
    h, w = stored.shape[:2]
    sw, sh = (h, w) if bits & LB_TRANSPOSE else (w, h)
    x, y = np.meshgrid(np.arange(sw), np.arange(sh))
    xs = sw - 1 - x if bits & LB_FLIP_X else x
    ys = sh - 1 - y if bits & LB_FLIP_Y else y
    return stored[xs, ys] if bits & LB_TRANSPOSE else stored[ys, xs]


@pytest.mark.parametrize("o", range(1, 9))
def test_mirrored_level_bits_read_the_flipped_displayed_image(o):
    """A mirrored level of D = T_o(S) is an item with bits lb_orientation_bits(o) ^ LB_FLIP_X: the flip acts on displayed x before the
    transpose, so the pixels read are cv2.flip(orient(S, o), 1) byte for byte (and bits alone read orient(S, o)); odd sides on both
    axes."""
    img = np.random.default_rng(o).integers(0, 256, (37, 53, 3), np.uint8)
    assert np.array_equal(read_displayed(img, BITS[o]), orient(img, o))
    assert np.array_equal(read_displayed(img, BITS[o] ^ LB_FLIP_X), cv2.flip(orient(img, o), 1))


def _tiles_of(w, h, net=448, o=64):
    """The tile count of the default pyramid from the layout rule of rf_b200.h: levels 1, 1/2, ... while the level does not fit, then
    the fitted level (one tile); per axis one tile when S <= T, else ceil((S - o) / (T - o))."""
    axis = lambda s: 1 if s <= net else -(-(s - o) // (net - o))
    count, s = 1, 1.0
    while round(w * s) > net or round(h * s) > net:
        count += axis(int(round(w * s))) * axis(int(round(h * s)))
        s *= 0.5
    return count


def test_portrait_4k_layout_has_the_landscape_tile_count(built_lib):
    """A 3840 x 2160 frame shown at 6 is tiled as 2160 x 3840: 84 tiles, like the landscape frame, by the rule and by rf_tile_layout."""
    from retinaface_b200 import capi
    assert _tiles_of(2160, 3840) == _tiles_of(3840, 2160) == 84
    portrait = capi.tile_layout(448, 448, 2160, 3840)
    assert len(portrait) == len(capi.tile_layout(448, 448, 3840, 2160)) == 84
    assert {(t["scaled_w"], t["scaled_h"]) for t in portrait if t["level"] == 0} == {(2160, 3840)}


def test_f21_entry_points_have_their_exact_ctypes_types(built_lib):
    """Each parameter of the five f21 entry points: structures by their ctypes class, input arrays (orientations included) as typed
    pointers, every other pointer as a plain address."""
    from retinaface_b200 import capi
    protos, _ = _prototypes()
    lib, exact = capi.load_library(), _exact_types()
    for name in F21:
        ret, params = protos[name]
        fn = getattr(lib, name)
        assert fn.restype is C.c_int and len(fn.argtypes) == len(params), name
        for p, got in zip(params, fn.argtypes):
            t = _squash(re.sub(r"\s*\w+$", "", p))
            assert t in exact or t.endswith("*"), (name, p)
            assert got == exact.get(t, C.c_void_p), (name, p, got)
        assert sum(1 for p in params if re.search(r"\borientations?\b", p)) == 1, name


def test_cpp_shell_compiles_the_oriented_detect_tiled(built_lib, tmp_path):
    import subprocess
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "oriented_tiled_call.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    string dir = argv[1];\n'
                   '    RetinaFace rf(dir);\n'
                   '    vector<Mat> imgs(2, Mat(2160, 3840, CV_8UC3));\n'
                   '    AlignOptions a;\n'
                   '    rf.detectTiled(imgs, vector<int>{6, 1}, 0.5f, vector<float>{1.f, 0.f}, true, 64, &a);\n'
                   '    rf.detectTiled(imgs, vector<int>(2, 8));\n'
                   '    rf.detectTiled(imgs, 0.5f);\n'
                   '    return (int)rf.lastBatchFaces().size();\n'
                   '}\n')
    subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-I", host, "-I", os.path.join(ROOT, "include"), str(src)])
