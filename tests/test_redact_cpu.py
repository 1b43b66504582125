"""CPU: f12 redaction without a GPU -- oracle/redact.py (vectorised) against a literal per-sample loop of rf_b200.h's definition on
random small frames (boxes off every edge and wholly outside, odd coordinates, overlaps, blocks 1 / 8 / 32, NV12 / I420 / BGR), the
geometry's properties, the ctypes layout against the header, the kernels' build and the C link of the new symbols."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from oracle.redact import frame_regions, geometry, params, redact_bgr, redact_planes, redact_yuv, yuv_planes
from oracle.yuv import split_planes

W, H = 46, 34


def _literal(orig: np.ndarray, sub: int, regions) -> np.ndarray:
    """The definition sample by sample: the lowest-index region whose rectangle covers the sample's luma position, the sample's cell
    (side C / sub, anchored at (X0 / sub, Y0 / sub)), the rounded mean of that cell's original samples inside the plane."""
    h, w = orig.shape[:2]
    out = orig.copy()
    means = {}
    for y in range(h):
        for x in range(w):
            for idx, (X0, Y0, X1, Y1, Cs) in enumerate(regions):
                if not (X0 <= x * sub < X1 and Y0 <= y * sub < Y1):
                    continue
                cs, ax, ay = Cs // sub, X0 // sub, Y0 // sub
                cx, cy = (x - ax) // cs, (y - ay) // cs
                key = (idx, cx, cy)
                if key not in means:
                    vals = [orig[yy, xx].astype(np.int64) for yy in range(max(ay + cy * cs, 0), min(ay + (cy + 1) * cs, Y1 // sub, h))
                            for xx in range(max(ax + cx * cs, 0), min(ax + (cx + 1) * cs, X1 // sub, w))]
                    s, n = np.sum(vals, axis=0), len(vals)
                    means[key] = (s + n // 2) // n
                out[y, x] = means[key]
                break
    return out


def _boxes(rng, k):
    """k random (score, x1, y1, x2, y2) records around and beyond a W x H frame, with fractional (odd-snapping) coordinates."""
    f = np.zeros((k, 15), np.float32)
    for j in range(k):
        x1, y1 = rng.uniform(-20, W + 5), rng.uniform(-20, H + 5)
        f[j, :5] = (0.9, x1, y1, x1 + rng.uniform(1, 30), y1 + rng.uniform(1, 25))
    return f


EDGE_BOXES = np.array([[0.9, -8.3, 5.1, 6.7, 17.2],        # off the left edge
                       [0.9, 39.5, 3.0, 55.0, 12.9],       # off the right edge
                       [0.9, 10.2, -9.9, 22.4, 4.1],       # off the top
                       [0.9, 12.0, 28.7, 30.3, 44.0],      # off the bottom
                       [0.9, 60.0, 50.0, 70.0, 60.0],      # wholly outside
                       [0.9, 13.0, 9.0, 27.0, 21.0],       # overlaps the next
                       [0.9, 19.1, 13.3, 35.5, 27.9]], np.float32)
EDGE_BOXES = np.pad(EDGE_BOXES, ((0, 0), (0, 10)))


@pytest.mark.parametrize("blocks", [1, 8, 32])
@pytest.mark.parametrize("layout", ["nv12", "i420", "bgr"])
def test_oracle_equals_the_literal_definition(layout, blocks):
    rng = np.random.default_rng(blocks * 7 + len(layout))
    for trial in range(4):
        faces = EDGE_BOXES if trial == 0 else _boxes(rng, int(rng.integers(1, 6)))
        scale = 1.0 if trial < 2 else float(rng.uniform(0.5, 2.0))
        _, margin = params(0, float(rng.choice([0.0, 0.1, 1.0])))
        regions = frame_regions(faces / np.float32([1, scale, scale, scale, scale] + [1] * 10), len(faces), scale, margin, blocks)
        if layout == "bgr":
            img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
            assert np.array_equal(redact_bgr(img, regions), _literal(img, 1, regions)), trial
            continue
        buf = rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
        got = split_planes(redact_yuv(buf, layout, regions), layout)
        for plane, orig, sub in zip(got, split_planes(buf, layout), (1, 2, 2)):
            assert np.array_equal(plane, _literal(orig, sub, regions)), (trial, sub)


def test_geometry_properties():
    """C is even and at least 2, rectangles are even and contain the box, the chroma grid is the luma grid halved, and no region has
    more than blocks cells across either side."""
    rng = np.random.default_rng(11)
    for _ in range(3000):
        x1, y1 = rng.uniform(-2000, 5000, 2)
        x2, y2 = x1 + rng.uniform(0.01, 900), y1 + rng.uniform(0.01, 900)
        blocks = int(rng.integers(1, 33))
        margin = float(np.float32(rng.uniform(0.001, 1.0)))
        X0, Y0, X1, Y1, c = geometry(x1, y1, x2, y2, margin, blocks)
        assert c >= 2 and c % 2 == 0 and X0 % 2 == 0 and X1 % 2 == 0 and Y0 % 2 == 0 and Y1 % 2 == 0
        assert X0 <= math.floor(np.float32(x1)) and X1 > math.floor(np.float32(x2)) and Y0 <= math.floor(np.float32(y1))
        assert math.ceil((X1 - X0) / c) <= blocks and math.ceil((Y1 - Y0) / c) <= blocks
        # chroma sample j lies in luma columns 2j, 2j + 1: both in the same luma cell, the chroma cell of the halved grid
        j = np.arange(X0 // 2, X1 // 2)
        assert np.array_equal((2 * j - X0) // c, (j - X0 // 2) // (c // 2)) and np.array_equal((2 * j + 1 - X0) // c, (j - X0 // 2) // (c // 2))


def test_skipped_boxes_and_bounds():
    assert geometry(10, 10, 10, 20, 0.25, 8) is None                 # w == 0
    assert geometry(10, 10, 5, 20, 0.25, 8) is None                  # w < 0
    assert geometry(np.nan, 10, 20, 20, 0.25, 8) is None
    assert geometry(0, 0, np.inf, 20, 0.25, 8) is None
    X0, Y0, X1, Y1, c = geometry(-1e30, -1e30, 1e30, 1e30, 0.25, 8)
    assert (X0, Y0, X1, Y1) == (-65536, -65536, 65538, 65538) and c == 2 * math.ceil(131074 / 16)
    X0, _, X1, _, c = geometry(1e6, 0, 2e6, 10, 0.25, 8)            # beyond +65536: an empty rectangle that covers nothing
    assert X1 <= X0
    img = np.random.default_rng(1).integers(0, 256, (H, W, 3), dtype=np.uint8)
    regions = [geometry(1e6, 0, 2e6, 10, 0.25, 8), geometry(70000, 70000, 80000, 80000, 0.25, 1)]
    assert np.array_equal(redact_bgr(img, regions), img)
    # skipped records do not take an index: the regions of the valid ones are those of the valid ones alone
    recs = np.zeros((4, 15), np.float32)
    recs[:, 1:5] = [[5, 5, 15, 15], [np.nan, 1, 2, 3], [3, 3, 3, 9], [8, 8, 30, 20]]
    assert frame_regions(recs, 4, None, 0.25, 8) == frame_regions(recs[[0, 3]], 2, None, 0.25, 8)
    assert frame_regions(recs, 4, None, 0.25, 8, max_faces=1) == frame_regions(recs[:1], 1, None, 0.25, 8)


def test_lowest_index_wins_and_originals_are_read():
    """Two overlapping regions: the overlap takes region 0's cells; region 1's cells are means of the ORIGINAL samples."""
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    r0, r1 = geometry(4, 4, 20, 20, 0.1, 1), geometry(12, 12, 40, 30, 0.1, 1)
    out = redact_bgr(img, [r0, r1])
    m0 = redact_bgr(img, [r0])
    m1 = redact_bgr(img, [r1])
    in0 = np.zeros((H, W), bool)
    in0[max(r0[1], 0):r0[3], max(r0[0], 0):r0[2]] = True
    in1 = np.zeros((H, W), bool)
    in1[max(r1[1], 0):min(r1[3], H), max(r1[0], 0):min(r1[2], W)] = True
    assert (in0 & in1).any()
    assert np.array_equal(out[in0], m0[in0]) and np.array_equal(out[in1 & ~in0], m1[in1 & ~in0]) and np.array_equal(out[~in0 & ~in1], img[~in0 & ~in1])


def test_lost_tracks_only():
    from retinaface_b200.capi import TRACK_DTYPE
    tr = np.zeros(3, TRACK_DTYPE)
    tr["state"] = [1, 2, 0]
    for k, f in enumerate(("kx1", "ky1", "kx2", "ky2")):
        tr[f] = [[1, 2, 11, 12][k], [5, 6, 25, 26][k], [3, 3, 9, 9][k]]
    regions = frame_regions(np.zeros((0, 15), np.float32), 0, 1.0, 0.25, 8, tracks=tr)
    assert regions == [geometry(5, 6, 25, 26, 0.25, 8)]


def test_pitched_surface_padding_untouched():
    """An NVDEC-like surface (pitch 64, chroma at pitch x (H + 2)): only plane bytes of regions change."""
    pitch, uv_off = 64, 64 * (H + 2)
    surf = np.random.default_rng(2).integers(0, 256, uv_off + pitch * H // 2, dtype=np.uint8)
    regions = [geometry(-3, 5, 50, 20, 0.25, 8)]
    out = redact_yuv(surf, "nv12", regions, width=W, height=H, y_pitch=pitch, uv_offset=uv_off, uv_pitch=pitch)
    mask = np.zeros(surf.size, bool)
    for view, _ in yuv_planes(np.arange(surf.size).astype(np.int64), "nv12", W, H, pitch, uv_off, pitch):
        mask[view.reshape(-1)] = True
    assert np.array_equal(out[~mask], surf[~mask]) and not np.array_equal(out, surf)
    ref = np.array(surf)
    redact_planes(yuv_planes(ref, "nv12", W, H, pitch, uv_off, pitch), regions)
    assert np.array_equal(out, ref)


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    src = tmp_path / "red.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rf_b200.h"\nint main(void){\n'
                   'printf("%zu %zu\\n", sizeof(rf_redact_params), offsetof(rf_redact_params, margin));\n'
                   'void *f[3] = {(void *)rf_redact_yuv_device, (void *)rf_redact_device, (void *)rf_detect_yuv_redact_device};\n'
                   'printf("%d\\n", rf_redact_yuv_device(NULL, NULL, 0, NULL, NULL, NULL, NULL, NULL, NULL, NULL) == RF_ERR_INVALID_ARG && f[1] && f[2]);\n'
                   'return 0;}\n')
    exe = tmp_path / "red"
    libdir = os.path.dirname(built_lib)
    subprocess.check_call(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir, "-lrf_b200",
                           "-Wl,-rpath," + libdir])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(capi.RedactParams), capi.RedactParams.margin.offset, 1]
    assert {"rf_redact_yuv_device", "rf_redact_device", "rf_detect_yuv_redact_device"} <= set(capi.EXPORTS)


def test_entry_points_refuse_null_handles_without_gpu(built_lib):
    from retinaface_b200 import capi
    lib = capi.load_library()
    assert lib.rf_redact_yuv_device(None, None, 0, None, None, None, None, None, None, None) == -1
    assert lib.rf_redact_device(None, None, None, None, None, 0, None, None, None, None, None, None, None) == -1
    assert lib.rf_detect_yuv_redact_device(None, None, None, None, 0, 0, 0.5, 0.4, None, None, None, None, None, None) == -1


def test_redact_kernels_compile_for_sm90a_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, CSRC, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "redact.cu"), "-o",
                                                   str(tmp_path / "r.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    for k in ("k_redact_regions", "k_redact_measure", "k_redact_apply"):
        assert r.stderr.count(k) >= 2, k          # the YUV and the BGR instantiation
    assert r.stderr.count("0 bytes spill stores") >= 6 and "bytes spill stores" not in r.stderr.replace("0 bytes spill stores", ""), r.stderr


def test_cpp_shell_compiles_redact_calls(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    src = open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.cpp")).read()
    assert "rf_detect_yuv_redact_device" in src
