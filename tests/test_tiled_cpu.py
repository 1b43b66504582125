"""CPU: f7 tile geometry -- rf_tile_layout against the host restatement (tests/tile_oracle.py) field for field, the properties the
seam rule relies on (cores partition each level, tiles cover it, neighbours share the overlap, a face smaller than the overlap is
whole in the tile that owns it), the fitted level against the letter-box, bad tilings, and the C-ABI structure layouts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from tile_oracle import SIDE_BOTTOM, SIDE_LEFT, SIDE_RIGHT, SIDE_TOP, fitted_geometry, layout

NETS = [(448, 448), (1280, 896)]      # (net_w, net_h)


def _capi(built_lib):
    from retinaface_b200 import capi
    return capi


def _random_levels(rng, w, h):
    """1..4 explicit levels, flipped or not, scales in [0.05, 3.5] (s > 1 included) or the fitted level, kept within RF_MAX_TILES
    for a 448 network."""
    levels = []
    for _ in range(rng.integers(1, 5)):
        s = 0.0 if rng.random() < 0.2 else float(np.float32(rng.uniform(0.05, 3.5)))
        levels.append((s, int(rng.random() < 0.5)))
    return levels


def test_layout_equals_the_oracle(built_lib):
    capi = _capi(built_lib)
    rng = np.random.default_rng(7)
    checked = capacity = 0
    for _ in range(300):
        w, h = int(rng.integers(1, 4097)), int(rng.integers(1, 3073))
        for net_w, net_h in NETS:
            for levels in (None, _random_levels(rng, w, h)):
                overlap = int(rng.choice([0, 16, 48, 96, min(net_w, net_h) // 2]))
                want = layout(net_w, net_h, w, h, levels, overlap)
                if any(min(t["scaled_w"], t["scaled_h"]) < 1 for t in want):
                    with pytest.raises(capi.RfError) as e:
                        capi.tile_layout(net_w, net_h, w, h, levels, overlap)
                    assert e.value.status == -1
                    continue
                if len(want) > capi.MAX_TILES:
                    with pytest.raises(capi.RfError) as e:
                        capi.tile_layout(net_w, net_h, w, h, levels, overlap)
                    assert e.value.status == -6
                    capacity += 1
                    continue
                got = capi.tile_layout(net_w, net_h, w, h, levels, overlap)
                assert len(got) == len(want), (w, h, net_w, net_h, levels, overlap)
                for g, t in zip(got, want):
                    assert g == t, (w, h, net_w, net_h, levels, overlap, g, t)
                checked += 1
    assert checked > 800 and capacity > 0


def test_default_pyramid_counts(built_lib):
    """The counts the documentation quotes: a 4K frame is 84 tiles at 448x448 and 17 at 1280x896 (overlap 64); an image that fits
    the network gets the fitted level alone."""
    capi = _capi(built_lib)
    assert len(capi.tile_layout(448, 448, 3840, 2160)) == 84
    assert len(capi.tile_layout(1280, 896, 3840, 2160)) == 17
    assert [t["scale"] for t in capi.tile_layout(448, 448, 448, 300)] == [0.0]
    assert [t["scale"] for t in capi.tile_layout(448, 448, 449, 300)] == [1.0, 1.0, 0.0]


@pytest.mark.parametrize("net", NETS)
def test_layout_properties(built_lib, net):
    capi = _capi(built_lib)
    net_w, net_h = net
    rng = np.random.default_rng(11)
    for _ in range(60):
        w, h = int(rng.integers(16, 2049)), int(rng.integers(16, 1537))
        o = int(rng.choice([16, 64, 100, min(net) // 2]))
        for level in ((1.0, 0), (0.5, 1), (1.7, 0), (0.0, 0)):     # one layout per level: all four can exceed RF_MAX_TILES
            ts = capi.tile_layout(net_w, net_h, w, h, [level], o)
            S, Sh = ts[0]["scaled_w"], ts[0]["scaled_h"]
            owner = np.zeros((Sh, S), np.int32)
            for t in ts:
                owner[t["own_y0"]:t["own_y1"], t["own_x0"]:t["own_x1"]] += 1
                # within the level (or at 0 when the level is smaller than the tile), the core inside the tile
                for a0, side, T, c0, c1 in (("x0", S, net_w, "own_x0", "own_x1"), ("y0", Sh, net_h, "own_y0", "own_y1")):
                    if side <= T:
                        assert t[a0] == 0
                    else:
                        assert 0 <= t[a0] <= side - T
                    assert t[a0] <= t[c0] < t[c1] <= t[a0] + T
            assert (owner == 1).all(), "the cores partition the level"
            assert ts[-1]["own_x1"] == max(S, net_w) and ts[-1]["own_y1"] == max(Sh, net_h)   # the far edge of the last tile
            cover = np.zeros((Sh, S), bool)
            for t in ts:
                cover[t["y0"]:t["y0"] + net_h, t["x0"]:t["x0"] + net_w] = True
            assert cover.all()
            xs = sorted({t["x0"] for t in ts})
            ys = sorted({t["y0"] for t in ts})
            for a, b in zip(xs, xs[1:]):
                assert a + net_w - b >= o
            for a, b in zip(ys, ys[1:]):
                assert a + net_h - b >= o
            for t in ts:           # shared sides are exactly the sides with a neighbour; a core edge keeps >= o / 2 from them
                assert bool(t["shared_sides"] & SIDE_LEFT) == (t["x0"] != xs[0])
                assert bool(t["shared_sides"] & SIDE_RIGHT) == (t["x0"] != xs[-1])
                assert bool(t["shared_sides"] & SIDE_TOP) == (t["y0"] != ys[0])
                assert bool(t["shared_sides"] & SIDE_BOTTOM) == (t["y0"] != ys[-1])
                if t["shared_sides"] & SIDE_LEFT:
                    assert t["own_x0"] - t["x0"] >= o // 2
                if t["shared_sides"] & SIDE_RIGHT:
                    assert t["x0"] + net_w - t["own_x1"] >= o // 2
                if t["shared_sides"] & SIDE_TOP:
                    assert t["own_y0"] - t["y0"] >= o // 2
                if t["shared_sides"] & SIDE_BOTTOM:
                    assert t["y0"] + net_h - t["own_y1"] >= o // 2


def test_fitted_level_is_the_letterbox(built_lib):
    """Size and map-back factor of the fitted level equal what the letter-box of rf_detect_batch (cv2.resize by the reference's
    float factor) produces."""
    import cv2
    capi = _capi(built_lib)
    rng = np.random.default_rng(5)
    for _ in range(40):
        w, h = int(rng.integers(1, 4097)), int(rng.integers(1, 3073))
        for net_w, net_h in NETS:
            (t,) = capi.tile_layout(net_w, net_h, w, h, [(0.0, 0)])
            sc = max(np.float32(1.0 * w / net_w), np.float32(1.0 * h / net_h), np.float32(1.0))
            if sc > 1:
                f = float(np.float32(1) / sc)
                rh, rw = cv2.resize(np.zeros((h, w), np.uint8), None, fx=f, fy=f).shape
            else:
                rh, rw = h, w
            assert (t["scaled_w"], t["scaled_h"]) == (min(rw, net_w), min(rh, net_h))
            assert np.float32(t["map_back"]) == sc
            # one tile on both axes: it owns everything, its core reported as the whole tile
            assert (t["x0"], t["y0"], t["shared_sides"], t["own_x0"], t["own_y0"], t["own_x1"], t["own_y1"]) == (0, 0, 0, 0, 0, net_w, net_h)
            assert fitted_geometry(w, h, net_w, net_h)[:2] == (t["scaled_w"], t["scaled_h"])


@pytest.mark.parametrize("net", NETS)
def test_halving_pyramid_owns_every_box_once_and_whole_somewhere(built_lib, net):
    """Default pyramid, random boxes of side 16 px .. min(w, h) inside random images (fixed seed): at every level the box's centre
    lies in exactly one core, and in at least one level the owning tile holds the whole box -- in particular at every tiled level
    where the box's side is below the overlap (the rule the seam filter relies on)."""
    capi = _capi(built_lib)
    net_w, net_h = net
    rng = np.random.default_rng(23)
    for _ in range(12):
        w, h = int(rng.integers(600, 4097)), int(rng.integers(400, 3073))
        tiles = capi.tile_layout(net_w, net_h, w, h)
        o = 64
        nlev = tiles[-1]["level"] + 1
        for _ in range(200):
            d = float(rng.uniform(16, min(w, h)))
            x1, y1 = rng.uniform(0, w - d), rng.uniform(0, h - d)
            whole_somewhere = False
            for lv in range(nlev):
                ts = [t for t in tiles if t["level"] == lv]
                k = ts[0]["scaled_w"] / w          # level pixels per image pixel (the fitted level's resize included)
                bx1, by1, bd = x1 * k, y1 * k, d * k
                cx, cy = bx1 + bd / 2, by1 + bd / 2
                own = [t for t in ts if t["own_x0"] <= cx < t["own_x1"] and t["own_y0"] <= cy < t["own_y1"]]
                if cx >= ts[0]["scaled_w"] or cy >= ts[0]["scaled_h"]:
                    continue                        # rounding of the level size: the centre fell off the last pixel
                assert len(own) == 1, (w, h, lv, d)
                t = own[0]
                whole = (bx1 >= t["x0"] - 1 and by1 >= t["y0"] - 1 and bx1 + bd <= t["x0"] + net_w + 1 and by1 + bd <= t["y0"] + net_h + 1)
                if len(ts) > 1 and bd < o - 2:
                    assert whole, (w, h, lv, d, t)
                whole_somewhere |= whole
            assert whole_somewhere


def test_bad_tilings_return_their_status(built_lib):
    capi = _capi(built_lib)
    bad = [([(-0.5, 0)], 0), ([(float("nan"), 0)], 0), ([(float("inf"), 0)], 0), ([(5.0, 0)], 0),   # 4000 * 5 > 16384
           ([(1e-6, 0)], 0), (None, 15), (None, 225), (None, -3), ([(1.0, 0)] * 9, 0)]
    for levels, overlap in bad:
        with pytest.raises(capi.RfError) as e:
            capi.tile_layout(448, 448, 4000, 3000, levels, overlap)
        assert e.value.status == -1, (levels, overlap)
    with pytest.raises(capi.RfError) as e:                  # 10 x 7 tiles at s = 1 and 25 x 18 at s = 2.5
        capi.tile_layout(448, 448, 4000, 3000, [(1.0, 0), (2.5, 0)], 0)
    assert e.value.status == -6
    lib = capi.load_library()
    t = capi.tiling()
    assert lib.rf_tile_layout(448, 448, 0, 100, C.byref(t), None, 0) == -1
    assert lib.rf_tile_layout(0, 448, 100, 100, C.byref(t), None, 0) == -1
    assert lib.rf_tile_layout(448, 448, 100, 100, C.byref(t), None, 1) == -1       # cap without an array
    assert lib.rf_tile_layout(448, 448, 100, 100, None, None, 0) == 1            # NULL tiling: the default pyramid
    nolevels = capi.Tiling(None, 2, 0)
    assert lib.rf_tile_layout(448, 448, 100, 100, C.byref(nolevels), None, 0) == -1
    assert capi.tile_layout(448, 448, 2000, 1500, None, 16)    # the bounds themselves are valid
    assert capi.tile_layout(448, 448, 2000, 1500, None, 224)


def test_tile_entry_points_and_struct_layout(built_lib, tmp_path):
    from retinaface_b200 import capi
    lib = C.CDLL(built_lib)
    for name in ("rf_tile_layout", "rf_detect_tiled", "rf_detect_yuv_tiled", "rf_preprocess_tile"):
        assert name in capi.EXPORTS and hasattr(lib, name), name
    src = tmp_path / "layout.c"
    tf = [f for f, _ in capi.Tile._fields_]
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "rf_b200.h"\n'
                   'int main(void) {\n'
                   '    printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(rf_tile_level), offsetof(rf_tile_level, flip), sizeof(rf_tiling), '
                   'offsetof(rf_tiling, levels), offsetof(rf_tiling, nlevels), offsetof(rf_tiling, overlap), sizeof(rf_tile));\n'
                   '    printf("' + " ".join(["%zu"] * len(tf)) + '\\n", ' + ", ".join(f"offsetof(rf_tile, {f})" for f in tf) + ');\n'
                   '    printf("%d %d %d %d %d %d\\n", RF_MAX_TILE_LEVELS, RF_MAX_TILES, RF_TILE_SIDE_LEFT, RF_TILE_SIDE_TOP, RF_TILE_SIDE_RIGHT, '
                   'RF_TILE_SIDE_BOTTOM);\n'
                   '    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    lines = subprocess.check_output([str(exe)], text=True).splitlines()
    got = [[int(v) for v in ln.split()] for ln in lines]
    assert got[0] == [C.sizeof(capi.TileLevel), capi.TileLevel.flip.offset, C.sizeof(capi.Tiling), capi.Tiling.levels.offset,
                      capi.Tiling.nlevels.offset, capi.Tiling.overlap.offset, C.sizeof(capi.Tile)]
    assert got[1] == [getattr(capi.Tile, f).offset for f in tf]
    assert got[2] == [capi.MAX_TILE_LEVELS, capi.MAX_TILES, capi.TILE_SIDE_LEFT, capi.TILE_SIDE_TOP, capi.TILE_SIDE_RIGHT,
                      capi.TILE_SIDE_BOTTOM]


def test_cpp_shell_compiles_a_detect_tiled_call(built_lib, tmp_path):
    from retinaface_b200.build import build_host
    build_host()
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "tiled_call.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    string dir = argc > 1 ? argv[1] : ".";\n'
                   '    RetinaFace rf(dir);\n'
                   '    vector<unsigned char> buf(2160 * 3840 * 3, 0);\n'
                   '    vector<Mat> imgs(1, Mat(2160, 3840, CV_8UC3, buf.data(), 3840 * 3));\n'
                   '    rf.detectTiled(imgs, 0.9f);\n'
                   '    rf.detectTiled(imgs, 0.9f, vector<float>{1.5f, 0.f}, true, 96);\n'
                   '    return (int)rf.lastBatchFaces().size() - 1;\n'
                   '}\n')
    exe = tmp_path / "tiled_call"
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", host, "-I", os.path.join(ROOT, "include"), str(src),
                           os.path.join(host, "RetinaFace.cpp"), "-o", str(exe), "-L", os.path.dirname(built_lib), "-lrf_b200",
                           "-Wl,-rpath," + os.path.dirname(built_lib)])
    assert os.path.exists(exe)


def _half_area(img):
    """The rule k_letterbox_batch applies to tile levels of scale 0.5 (preprocess.cu half_pixel), restated in numpy: the mean of
    each 2 x 2 source block, (sum + 2) >> 2 for a whole block, sum / count rounded half to even for a block cut by the far edge."""
    h, w = img.shape[:2]
    dw, dh = int(np.rint(w * 0.5)), int(np.rint(h * 0.5))
    pad = np.zeros((2 * dh, 2 * dw, 3), np.int64)
    cnt = np.zeros((2 * dh, 2 * dw, 1), np.int64)
    hh, ww = min(h, 2 * dh), min(w, 2 * dw)     # a side of 1 mod 4 halves down: its last pixel is not read
    pad[:hh, :ww] = img[:hh, :ww]
    cnt[:hh, :ww] = 1
    s = pad.reshape(dh, 2, dw, 2, 3).sum(axis=(1, 3))
    n = cnt.reshape(dh, 2, dw, 2, 1).sum(axis=(1, 3))
    whole = (s + 2) >> 2
    part = np.rint(s.astype(np.float32) / n.astype(np.float32)).astype(np.int64)
    return np.where(n == 4, whole, part).astype(np.uint8)


@pytest.mark.parametrize("hw", [(335, 519), (63, 107), (71, 123), (333, 517), (48, 64), (886, 1280), (5, 3), (3, 7)])
def test_half_scale_level_is_opencvs_area_rule(hw):
    """cv2.resize(INTER_LINEAR) at fx = fy = 0.5 runs OpenCV's fast 2x INTER_AREA code: on sides of 3 mod 4 the last column / row
    averages the pixels it has, rounded half to even, which the bilinear taps would round up.  The rule the tile letter-box uses
    for levels of scale 0.5 equals cv2 on every size, plain and mirrored."""
    import cv2
    img = np.random.default_rng(hw[0] * 7 + hw[1]).integers(0, 256, hw + (3,), dtype=np.uint8)
    for src in (img, cv2.flip(img, 1)):
        assert np.array_equal(_half_area(src), cv2.resize(src, None, fx=0.5, fy=0.5))
