"""CPU: f14 redaction styles without a GPU -- the blur kernel and its sliding-sum cascade, oracle/redact_style.py's blur against a
literal per-sample loop of rf_b200.h's definition, the integer bounds at radius 127, the exact ellipse test against fractions.Fraction, the
ownership of overlapping regions, {MOSAIC, RECT} against f12, the privacy of the default blur on the golden photo, and the C layout,
link, build and C++ shell of the new surface."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle.redact import frame_regions, geometry, params
from oracle.redact import redact_bgr as f12_bgr
from oracle.redact import redact_yuv as f12_yuv
from oracle.redact_style import (BLUR, ELLIPSE, MOSAIC, RECT, _boxes3, blur_plane, blur_radius, ellipse_mask, kernel, redact_bgr, redact_yuv,
                                 shape_mask, style)
from oracle.yuv import split_planes

W, H = 46, 34


def _literal_blur(orig: np.ndarray, x: int, y: int, a: int) -> np.ndarray:
    """The definition at one sample: S = sum_ij k[i] k[j] P[clampY(y + j)][clampX(x + i)] in Python ints, rounded."""
    h, w = orig.shape[:2]
    k = [int(v) for v in kernel(a)]
    S = 0
    for j in range(-3 * a, 3 * a + 1):
        for i in range(-3 * a, 3 * a + 1):
            S = S + k[i + 3 * a] * k[j + 3 * a] * orig[min(max(y + j, 0), h - 1), min(max(x + i, 0), w - 1)].astype(object)
    n6 = (2 * a + 1) ** 6
    return (S + (n6 - 1) // 2) // n6


def _literal_ellipse(x0, y0, x1, y1, x, y) -> bool:
    """The ellipse inscribed in [x0, x1) x [y0, y1) contains the centre (x + 1/2, y + 1/2), in rationals."""
    W_, H_ = x1 - x0, y1 - y0
    if W_ <= 0 or H_ <= 0:
        return False
    cx, cy = Fraction(x0 + x1, 2), Fraction(y0 + y1, 2)
    dx, dy = Fraction(2 * x + 1, 2) - cx, Fraction(2 * y + 1, 2) - cy
    return (dx / Fraction(W_, 2)) ** 2 + (dy / Fraction(H_, 2)) ** 2 <= 1


@pytest.mark.parametrize("a", [1, 2, 19, 63, 127])
def test_kernel_is_three_boxes_and_the_cascade_is_the_correlation(a):
    n = 2 * a + 1
    k = kernel(a)
    box = np.ones(n, np.int64)
    assert len(k) == 6 * a + 1 and k.sum() == n ** 3 and np.array_equal(k, np.convolve(np.convolve(box, box), box))
    assert np.array_equal(k, k[::-1]) and k[3 * a] == k.max()
    rng = np.random.default_rng(a)
    x = rng.integers(0, 256, (3, 6 * a + 40), dtype=np.int64)
    direct = np.stack([np.correlate(r, k, mode="valid") for r in x])
    assert np.array_equal(_boxes3(x, a, 1).astype(np.int64), direct)
    # the device's form: three running sums of q(t) - 3 q(t - n) + 3 q(t - 2n) - q(t - 3n), modulo 2^32
    q = np.concatenate([np.zeros(3 * n, np.int64), x[0]])
    d = (q[3 * n:] - 3 * q[2 * n:-n] + 3 * q[n:-2 * n] - q[:-3 * n]) % 2 ** 32
    c3 = np.cumsum(np.cumsum(np.cumsum(d) % 2 ** 32) % 2 ** 32) % 2 ** 32
    assert np.array_equal(c3[6 * a:], direct[0])


def test_blur_plane_equals_the_literal_definition():
    """Small planes, regions touching or leaving every edge, luma-sized and chroma-sized radii; BGR channels independently."""
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (18, 23, 3), dtype=np.uint8)
    for region, a in [((-6, -4, 8, 6), 1), ((16, 10, 30, 24), 2), ((-20, -20, 40, 40), 3), ((4, 2, 10, 8), 5), ((22, 0, 24, 18), 1)]:
        sl, got = blur_plane(img, region, a)
        _, direct = blur_plane(img, region, a, direct=True)
        assert np.array_equal(got, direct), region
        for yy in range(sl[0].start, sl[0].stop, 3):
            for xx in range(sl[1].start, sl[1].stop, 2):
                assert np.array_equal(got[yy - sl[0].start, xx - sl[1].start], _literal_blur(img, xx, yy, a)), (region, xx, yy)
    assert blur_plane(img, (30, 0, 40, 10), 1) is None and blur_plane(img, (0, 0, 0, 10), 1) is None


def test_integer_bounds_at_the_largest_radius():
    """a = 127 on an all-255 plane: a one-axis sum 255 n^3 = 255^4 < 2^32, S = 255 n^6 = 255^7 < 2^63, and the value 255."""
    a, n = 127, 255
    assert 255 * n ** 3 == 255 ** 4 < 2 ** 32 and 255 * n ** 6 == 255 ** 7 < 2 ** 63
    assert blur_radius((0, 0, 4000, 10), 1) == 127 and blur_radius((0, 0, 2, 2), 64) == 1 and blur_radius((0, 0, 0, 0), 4) == 1
    plane = np.full((40, 30), 255, np.uint8)
    row = _boxes3(np.full((2, 6 * a + 30), 255, np.int64), a, 1)
    assert row.shape == (2, 30) and (row == 255 ** 4).all()
    sl, v = blur_plane(plane, (-10, -10, 50, 50), a)
    assert (v == 255).all() and v.shape == (40, 30)


def test_ellipse_test_is_exact():
    """ellipse_mask against fractions.Fraction on random, thin, boundary and +-65536-clamped rectangles."""
    rng = np.random.default_rng(2)
    rects = [(0, 0, 2, 2), (0, 0, 2, 40), (-6, -4, 20, 12), (-65536, -65536, 65538, 65538), (-65536, 4, 65538, 30),
             (10, -65536, 30, 65538), (0, 0, 30, 30), (8, 8, 8, 20), (8, 20, 30, 10)]
    for _ in range(40):
        x0, y0 = 2 * int(rng.integers(-20, 30)), 2 * int(rng.integers(-20, 20))
        rects.append((x0, y0, x0 + 2 * int(rng.integers(1, 30)), y0 + 2 * int(rng.integers(1, 25))))
    for x0, y0, x1, y1 in rects:
        m = ellipse_mask(x0, y0, x1, y1, W, H)
        for y in range(H):
            for x in range(W):
                assert m[y, x] == _literal_ellipse(x0, y0, x1, y1, x, y), (x0, y0, x1, y1, x, y)
    # the clamp: W^2 H^2 above int64 -- a sample inside near the centre and the corner outside
    big = ellipse_mask(-65536, -65536, 65538, 65538, 4, 4)
    assert big.all() and (-65536 - 1) ** 2 * 131074 ** 2 > 2 ** 63


def test_default_margin_ellipse_contains_the_box():
    """With margin 0.25 every pixel centre of the box lies in the ellipse; at 0.15 some corner does not."""
    rng = np.random.default_rng(3)
    for _ in range(300):
        x1, y1 = rng.uniform(0, 60, 2)
        x2, y2 = x1 + rng.uniform(2, 60), y1 + rng.uniform(2, 60)
        X0, Y0, X1, Y1, _ = geometry(x1, y1, x2, y2, params(0, 0.25)[1], 8)
        m = ellipse_mask(X0, Y0, X1, Y1, 140, 140)
        fx1, fy1, fx2, fy2 = (float(np.float32(v)) for v in (x1, y1, x2, y2))
        xs = [x for x in range(140) if fx1 <= x + 0.5 <= fx2]
        ys = [y for y in range(140) if fy1 <= y + 0.5 <= fy2]
        assert m[np.ix_(ys, xs)].all()
    X0, Y0, X1, Y1, _ = geometry(20, 20, 100, 100, params(0, 0.15)[1], 8)
    assert not ellipse_mask(X0, Y0, X1, Y1, 140, 140)[20, 20]


@pytest.mark.parametrize("shape", [RECT, ELLIPSE])
def test_overlaps_read_only_originals(shape):
    """Two overlapping regions of different radii: the overlap takes region 0's shape's value, region 1's samples elsewhere the blur of
    the ORIGINAL plane with its own radius, and nothing outside the shapes changes."""
    rng = np.random.default_rng(4)
    img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    r0, r1 = geometry(4, 4, 14, 14, 0.1, 8), geometry(10, 8, 44, 32, 0.1, 8)
    st = style(BLUR, shape, 0, 2)
    assert blur_radius(r0, 2) != blur_radius(r1, 2)
    out = redact_bgr(img, [r0, r1], st)
    m0, m1 = redact_bgr(img, [r0], st), redact_bgr(img, [r1], st)
    s0, s1 = shape_mask(*r0[:4], W, H, shape), shape_mask(*r1[:4], W, H, shape)
    assert (s0 & s1).any() and (s1 & ~s0).any()
    assert np.array_equal(out[s0], m0[s0]) and np.array_equal(out[s1 & ~s0], m1[s1 & ~s0]) and np.array_equal(out[~s0 & ~s1], img[~s0 & ~s1])


@pytest.mark.parametrize("layout", ["nv12", "i420", "bgr"])
def test_mosaic_rect_style_is_f12(layout):
    rng = np.random.default_rng(5)
    faces = np.zeros((4, 15), np.float32)
    faces[:, 1:5] = [[-8.3, 5.1, 6.7, 17.2], [13, 9, 27, 21], [19.1, 13.3, 35.5, 27.9], [39.5, 3.0, 55.0, 12.9]]
    regions = frame_regions(faces, 4, None, 0.25, 6)
    st = style(MOSAIC, RECT, 6)
    if layout == "bgr":
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
        assert np.array_equal(redact_bgr(img, regions, st), f12_bgr(img, regions))
        return
    buf = rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
    assert np.array_equal(redact_yuv(buf, layout, regions, st), f12_yuv(buf, layout, regions))
    # mosaic over the ellipse: f12's cell values on exactly the ellipse's samples
    e = split_planes(redact_yuv(buf, layout, regions, style(MOSAIC, ELLIPSE, 6)), layout)
    r = split_planes(f12_yuv(buf, layout, regions), layout)
    o = split_planes(buf, layout)
    for pe, pr, po, sub in zip(e, r, o, (1, 2, 2)):
        cover = np.zeros(po.shape, bool)
        for X0, Y0, X1, Y1, _ in reversed(regions):
            m = ellipse_mask(X0 // sub, Y0 // sub, X1 // sub, Y1 // sub, po.shape[1], po.shape[0])
            cover |= m
        assert np.array_equal(pe[~cover], po[~cover])
        first = np.zeros(po.shape, bool)      # samples whose lowest covering rectangle is also the lowest covering ellipse
        for idx, (X0, Y0, X1, Y1, _) in enumerate(regions):
            m = ellipse_mask(X0 // sub, Y0 // sub, X1 // sub, Y1 // sub, po.shape[1], po.shape[0])
            if idx == 0:
                first |= m
        assert np.array_equal(pe[first], pr[first])


def test_chroma_uses_the_halved_radius_and_ellipse():
    rng = np.random.default_rng(6)
    buf = rng.integers(0, 256, (H * 3 // 2, W), dtype=np.uint8)
    reg = geometry(6, 4, 36, 26, 0.25, 8)
    st = style(BLUR, ELLIPSE, 0, 1)
    a = blur_radius(reg, 1)
    out = split_planes(redact_yuv(buf, "i420", [reg], st), "i420")
    orig = split_planes(buf, "i420")
    for plane, po, sub in zip(out, orig, (1, 2, 2)):
        rect = tuple(v // sub for v in reg[:4])
        m = ellipse_mask(*rect, po.shape[1], po.shape[0])
        sl, v = blur_plane(po, rect, a if sub == 1 else (a + 1) >> 1)
        want = po.copy()
        want[sl][m[sl]] = v[m[sl]]
        assert np.array_equal(plane, want), sub
    assert (a + 1) >> 1 != a


def test_privacy_on_the_golden_photo(golden_image):
    """The default blur (detail 4, ellipse, margin 0.25) of the golden photo's six faces (the 1280x896 FP32 records at threshold 0.5,
    in photo pixels): the variance of cv2.Laplacian inside each face box falls below 2.5.  The photo's face boxes have variances of
    145 to 267; the oracle's blur (a = 27 on these faces) leaves 1.64 to 1.94, so the bound is the oracle's with a margin."""
    faces = np.load(os.path.join(GOLDEN, "dets_mnet25_896x1280.npz"))["faces_thr0.5"]
    regions = frame_regions(faces, len(faces), None, 0.25, 8)
    out = redact_bgr(golden_image, regions, style())
    lap0 = cv2.Laplacian(cv2.cvtColor(golden_image, cv2.COLOR_BGR2GRAY), cv2.CV_64F)
    lap1 = cv2.Laplacian(cv2.cvtColor(out, cv2.COLOR_BGR2GRAY), cv2.CV_64F)
    assert len(faces) == 6
    for f in faces:
        x1, y1, x2, y2 = (int(v) for v in f[1:5])
        assert lap0[y1:y2, x1:x2].var() > 100 and lap1[y1:y2, x1:x2].var() < 2.5, (x1, y1, x2, y2)


def test_ctypes_layout_and_c_link(built_lib, tmp_path):
    from retinaface_b200 import capi
    src = tmp_path / "sty.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "rf_b200.h"\nint main(void){\n'
                   'printf("%zu %zu %zu %d %d %d %d\\n", sizeof(rf_redact_style), offsetof(rf_redact_style, detail), offsetof(rf_redact_style, margin),'
                   ' RF_REDACT_MOSAIC, RF_REDACT_BLUR, RF_REDACT_RECT, RF_REDACT_ELLIPSE);\n'
                   'void *f[3] = {(void *)rf_redact_yuv_device_style, (void *)rf_redact_device_style, (void *)rf_detect_yuv_redact_device_style};\n'
                   'printf("%d\\n", rf_redact_yuv_device_style(NULL, NULL, 0, NULL, NULL, NULL, NULL, NULL, NULL, NULL) == RF_ERR_INVALID_ARG && f[1] && f[2]);\n'
                   'return 0;}\n')
    exe = tmp_path / "sty"
    libdir = os.path.dirname(built_lib)
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                           "-L", libdir, "-lrf_b200", "-Wl,-rpath," + libdir])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(capi.RedactStyle), capi.RedactStyle.detail.offset, capi.RedactStyle.margin.offset, capi.RF_REDACT_MOSAIC,
                   capi.RF_REDACT_BLUR, capi.RF_REDACT_RECT, capi.RF_REDACT_ELLIPSE, 1]
    assert {"rf_redact_yuv_device_style", "rf_redact_device_style", "rf_detect_yuv_redact_device_style"} <= set(capi.EXPORTS)
    lib = capi.load_library()
    assert lib.rf_redact_device_style(None, None, None, None, None, 0, None, None, None, None, None, None, None) == -1
    assert lib.rf_detect_yuv_redact_device_style(None, None, None, None, 0, 0, 0.5, 0.4, None, None, None, None, None, None) == -1


def test_python_keywords_pick_the_call():
    from retinaface_b200 import capi
    assert capi.redact_style() is None and capi.redact_style(blocks=5, margin=0.3) is None
    st = capi.redact_style("blur", "ellipse", 0, 6, 0.3)
    assert (st.kind, st.shape, st.blocks, st.detail) == (2, 2, 0, 6) and abs(st.margin - 0.3) < 1e-7
    st = capi.redact_style("mosaic", "ellipse", 5)
    assert (st.kind, st.shape, st.blocks, st.detail) == (1, 2, 5, 0)
    with pytest.raises(ValueError):
        capi.redact_style("gauss")


def test_blur_kernels_compile_for_sm90a_without_spills(tmp_path):
    from retinaface_b200.build import ARCH, COMMON, CSRC, nvcc
    r = subprocess.run([nvcc()] + ARCH + COMMON + ["-fmad=false", "-Xptxas", "-v", "-c", os.path.join(CSRC, "redact.cu"), "-o",
                                                   str(tmp_path / "r.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stderr.count("k_redact_blur") >= 4 and r.stderr.count("k_redact_apply") >= 8
    assert "bytes spill stores" not in r.stderr.replace("0 bytes spill stores", ""), r.stderr


def test_cpp_shell_calls_the_style_entry_point(built_lib):
    from retinaface_b200.build import build_host
    assert os.path.exists(build_host())
    src = open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.cpp")).read()
    hdr = open(os.path.join(ROOT, "retinaface_b200", "host", "RetinaFace.h")).read()
    assert "rf_detect_yuv_redact_device_style" in src and "int style = RF_REDACT_MOSAIC" in hdr and "int shape = RF_REDACT_RECT" in hdr
