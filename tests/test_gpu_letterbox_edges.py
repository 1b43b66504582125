"""GPU (-m gpu): every letter-box entry point against the kernel's definition (oracle/letterbox.py, itself held to cv2 by
tests/test_letterbox_cpu.py), byte for byte, on the shapes where cv::resize changes its code path: exactly 2x with every residue
mod 4 of the other side, the identity and one pixel over the box, round-half-to-even ties of the resized size, one-pixel sides and
extreme aspect ratios (an all-zero letter-box).  Then the detect paths at exactly 2x against rf_forward_heads + the post-process
oracle on the cv2 letter-box, and the degenerate shapes through them: their status or no faces, with nothing written past it."""
import ctypes as C

import cv2
import numpy as np
import pytest

from conftest import caffemodel
from oracle import letterbox as lb
from oracle.inputs import letterbox_bgr_u8
from oracle.postproc import PostprocOracle
from oracle.postproc import compare_dets
from oracle.yuv import bgr_to_frame, frame_to_bgr
from test_letterbox_cpu import thin_shapes, tie_shapes

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
NETS = [(448, 448), (160, 96)]          # (net_w, net_h)


def _engine(net=(448, 448), **kw):
    from retinaface_b200 import RF_PREC_FP16, Engine
    kw.setdefault("max_batch", 2)
    kw.setdefault("max_image", (5000, 5000))
    return Engine(caffemodel("mnet25"), net[1], net[0], precision=RF_PREC_FP16, **kw)


def edge_shapes(bw, bh):
    """(h, w): exactly 2x with the other side of each residue mod 4 (both ways round), the identity and one pixel over, two ties,
    and the one-pixel and extreme sides."""
    two = [(2 * bh - r, 2 * bw) for r in range(4)] + [(2 * bh, 2 * bw - r) for r in range(1, 4)]
    near = [(bh, bw), (bh, bw + 1), (bh + 1, bw), (bh - 1, bw - 3)]
    return list(dict.fromkeys(two + near + tie_shapes(bw, bh, per=1)[:4] + thin_shapes(bw, bh)))


def _random(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, shape + (3,), dtype=np.uint8)


def _want(img, net_w, net_h, **kw):
    """The definition, and cv2's letter-box wherever cv2 accepts the size (the two agree there: tests/test_letterbox_cpu.py)."""
    want = lb.letterbox(img, net_w, net_h, **kw)
    if not kw and min(lb.geometry(img.shape[1], img.shape[0], net_w, net_h)[:2]) > 0:
        assert np.array_equal(want, letterbox_bgr_u8(img, net_h, net_w)), img.shape
    return want


@pytest.fixture(scope="module")
def post_oracle():
    return PostprocOracle()


@pytest.mark.parametrize("net", NETS, ids=[f"{w}x{h}" for w, h in NETS])
def test_preprocess_pageable_pinned_and_strided(net):
    """rf_preprocess from a pageable, a pinned and a row-strided source (a slice of a wider buffer) == the definition."""
    import torch
    net_w, net_h = net
    eng = _engine(net)
    try:
        for i, hw in enumerate(edge_shapes(net_w, net_h)):
            img = _random(hw, i)
            want = _want(img, net_w, net_h)
            assert np.array_equal(eng.preprocess(img), want), ("pageable", hw)
            pinned = torch.empty(hw + (3,), dtype=torch.uint8).pin_memory().numpy()
            pinned[:] = img
            assert np.array_equal(eng.preprocess(pinned), want), ("pinned", hw)
            wide = np.full((hw[0], hw[1] + 7, 3), 0xA5, np.uint8)
            wide[:, :hw[1]] = img
            out = np.empty((net_h, net_w, 3), np.uint8)
            assert eng.lib.rf_preprocess(eng.h, wide.ctypes.data, hw[1], hw[0], wide.strides[0], out.ctypes.data) == 0
            assert np.array_equal(out, want), ("strided", hw)
    finally:
        eng.close()


def _pitched(frame, layout, pad=64):
    """The frame's planes in buffers whose rows are `pad` bytes longer than the plane (an NVDEC-like pitch)."""
    rows, w = frame.shape
    h = rows * 2 // 3

    def plane(a):
        buf = np.full((a.shape[0], a.shape[1] + pad), 0x3C, np.uint8)
        buf[:, :a.shape[1]] = a
        return buf[:, :a.shape[1]]
    if layout == "nv12":
        return plane(frame[:h]), plane(frame[h:])
    q = (h // 2) * (w // 2)
    flat = frame[h:].reshape(-1)
    return plane(frame[:h]), plane(flat[:q].reshape(h // 2, w // 2)), plane(flat[q:].reshape(h // 2, w // 2))


@pytest.mark.parametrize("layout", ["nv12", "i420"])
@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
def test_preprocess_yuv_single_buffer_and_pitched(layout, matrix):
    """rf_preprocess_yuv == the definition on the frame's BGR conversion (oracle/yuv.py), for OpenCV's single buffer and for planes
    with their own pitches, on the even edge shapes (4:2:0 frames have even sides)."""
    eng = _engine()
    try:
        shapes = [hw for hw in edge_shapes(448, 448) if hw[0] % 2 == 0 and hw[1] % 2 == 0]
        assert len(shapes) >= 6
        for i, hw in enumerate(shapes):
            frame = bgr_to_frame(_random(hw, 50 + i), layout)
            want = lb.letterbox(frame_to_bgr(frame, layout, matrix), 448, 448)
            assert np.array_equal(eng.preprocess_yuv(frame, layout=layout, matrix=matrix), want), (hw, "single buffer")
            assert np.array_equal(eng.preprocess_yuv(_pitched(frame, layout), layout=layout, matrix=matrix), want), (hw, "pitched")
    finally:
        eng.close()


@pytest.mark.parametrize("o", range(1, 9))
def test_preprocess_oriented(o):
    """rf_preprocess_oriented in every EXIF orientation (5..8: the transposed kernel) == the definition of the oriented item."""
    eng = _engine()
    try:
        for i, hw in enumerate(edge_shapes(448, 448)):
            img = _random(hw, 100 + i)
            assert np.array_equal(eng.preprocess_oriented(img, o), lb.letterbox(img, 448, 448, bits=lb.ORIENTATION_BITS[o])), (hw, o)
    finally:
        eng.close()


def test_preprocess_tile_fitted_and_half_levels():
    """rf_preprocess_tile at the fitted level and at s = 0.5, plain and mirrored: the fitted level is the letter-box, a tile of the
    0.5 level a window of the definition's 2x image (zeros past its edge)."""
    from retinaface_b200 import capi
    eng = _engine()
    levels = [(0.5, 0), (0.5, 1), (0.0, 0), (0.0, 1)]
    try:
        for i, hw in enumerate([(503, 896), (896, 503), (895, 896), (1023, 1795), (448, 449)]):
            img = _random(hw, 200 + i)
            tiles = capi.tile_layout(448, 448, hw[1], hw[0], levels)
            for k, t in enumerate(tiles):
                bits = lb.LB_FLIP_X if t["flip"] else 0
                if t["scale"] == 0:
                    want = lb.letterbox(img, 448, 448, bits=bits)
                else:
                    level = lb.resized(img, t["scaled_w"], t["scaled_h"], 2.0, bits)
                    want = np.zeros((448, 448, 3), np.uint8)
                    win = level[t["y0"]:t["y0"] + 448, t["x0"]:t["x0"] + 448]
                    want[:win.shape[0], :win.shape[1]] = win
                assert np.array_equal(eng.preprocess_tile(img, k, levels), want), (hw, k, t)
    finally:
        eng.close()


def _npp_shapes():
    return [(503, 896), (896, 503), (895, 896), (449, 448), (448, 449), (886, 1280), (333, 1000), (181, 297), (80, 100), (1, 449),
            (449, 1), (700, 900), (1023, 1795), (3, 1795), (2000, 31), (897, 897)]


def test_npp_branch_equals_its_definition_and_npp():
    """RF_FLAG_NPP_RESIZE: the kernel == the definition's area rule byte for byte (plain and in orientations 2 and 6), and within
    1 LSB of NPP itself (nppiResizeSqrPixel_8u_C3R, NPPI_INTER_SUPER) on at most 0.5 % of the bytes, on 16 shapes."""
    from oracle.npp import npp_letterbox
    from retinaface_b200.capi import RF_FLAG_NPP_RESIZE
    eng = _engine(flags=RF_FLAG_NPP_RESIZE)
    try:
        exact = 0
        for i, hw in enumerate(_npp_shapes()):
            img = _random(hw, 300 + i)
            got = eng.preprocess(img)
            assert np.array_equal(got, lb.letterbox(img, 448, 448, npp=True)), hw
            for o in (2, 6):
                assert np.array_equal(eng.preprocess_oriented(img, o), lb.letterbox(img, 448, 448, bits=lb.ORIENTATION_BITS[o], npp=True)), (hw, o)
            if min(hw) < 16:
                continue        # NPP itself is compared where its ROI is not a sliver
            diff = np.abs(got.astype(int) - npp_letterbox(img, 448, 448).astype(int))
            frac = np.count_nonzero(diff) / diff.size
            print(f"{hw[1]}x{hw[0]}: NPP max diff {diff.max()}, {frac:.4%} of the bytes")
            assert diff.max() <= 1 and frac <= 5e-3, (hw, diff.max(), frac)
            exact += int(diff.max() == 0)
        assert exact >= 4
    finally:
        eng.close()


def _exact_2x_photos(golden_image):
    """The photo at exactly 2x into 448 x 448 with the other side 3 mod 4: 896 x 619 (last row one source row) and a portrait
    891 x 896 crop (last column one source column)."""
    return [cv2.resize(golden_image, (896, 619)), cv2.resize(np.ascontiguousarray(golden_image[:, 190:1100]), (891, 896))]


def test_detect_batch_at_exact_2x_equals_heads_of_the_cv2_letterbox(golden_image, post_oracle):
    """rf_detect_batch on images that are exactly twice the network with a side of 3 mod 4 == rf_forward_heads of the cv2
    letter-box through the post-process oracle: the same faces, in order, with the same anchor indices."""
    eng = _engine(max_image=(1024, 1024))
    try:
        for img in _exact_2x_photos(golden_image):
            inp = letterbox_bgr_u8(img, 448, 448)
            assert np.array_equal(eng.preprocess(img), inp), img.shape
            faces, idx = eng.detect_batch([img], THR, NMS, want_index=True)
            heads = eng.forward_heads(inp[None])
            compare_dets(faces[0], idx[0], post_oracle.postprocess([x[0] for x in heads], 448, 448, THR, NMS), str(img.shape))
            assert len(faces[0]) >= 1, img.shape
    finally:
        eng.close()


def test_detect_views_at_half_shrink_equals_heads_of_the_cv2_letterbox(golden_image, post_oracle):
    """rf_detect_views with one shrink-0.5 view of a 1280 x 719 image on a 1280 x 896 network: the view's box is 640 x 448, exactly
    half the image's width, and 719 is 3 mod 4.  Its faces == rf_forward_heads of the cv2 letter-box into the box, post-processed by
    the oracle and scaled by the view's map-back factor."""
    eng = _engine((1280, 896), max_batch=1, max_image=(896, 1280))
    try:
        img = np.ascontiguousarray(golden_image[:719])
        faces, view_of, scales = eng.detect_views(img, [(0.5, False)], THR, NMS)
        assert scales[0] == 2.0
        canvas = np.zeros((896, 1280, 3), np.uint8)
        canvas[:448, :640] = letterbox_bgr_u8(img, 448, 640)
        assert np.array_equal(canvas, lb.letterbox(img, 1280, 896, box=(640, 448)))
        # the view's network input, as the call left it in the input tensor
        assert np.array_equal(eng._fetch(eng.device_input_ptr(), np.uint8, 896, 1280, 3), canvas)
        heads = eng.forward_heads(canvas[None])
        ref = post_oracle.postprocess([x[0] for x in heads], 896, 1280, THR, NMS)["faces"].copy()
        ref[:, 1:] *= np.float32(scales[0])          # the map-back: coordinates only
        assert faces.shape == ref.shape and len(faces) >= 1 and (view_of == 0).all()
        assert np.array_equal(faces[:, 0], ref[:, 0]) and np.array_equal(faces[:, 5:], ref[:, 5:])
        assert np.allclose(faces[:, 1:5], ref[:, 1:5], rtol=4e-6, atol=2e-4)
    finally:
        eng.close()


CANARY = np.float32(-12345.5)


def test_degenerate_shapes_detect_nothing_and_write_nothing_past_their_counts(golden_image):
    """1 x 5000 and 5000 x 1 letter-box to an all-zero network input (the resized side rounds to 0): rf_detect_batch and
    rf_detect_views return RF_OK and no faces for them, rf_detect_tiled's default pyramid refuses them (RF_ERR_INVALID_ARG: a level
    side of 0), and none of them writes a face record, count or index past what it reports -- while the photo in the same batch
    gets exactly what it gets beside an all-zero network input."""
    from retinaface_b200 import capi
    eng = _engine()
    try:
        want, want_idx = eng.detect_batch([np.zeros((448, 448, 3), np.uint8), golden_image], THR, NMS, want_index=True)
        assert len(want[0]) == 0 and len(want[1]) >= 5
        mf = eng.max_faces
        for hw in ((1, 5000), (5000, 1), (2, 5000)):
            thin = _random(hw, 7)
            assert min(lb.geometry(hw[1], hw[0], 448, 448)[:2]) == 0
            assert not eng.preprocess(thin).any(), hw
            keep, ptrs, ws, hs, rs = eng._host_images([thin, golden_image])
            faces = np.full((2, mf, 15), CANARY, np.float32)
            counts = np.full(2, -7, np.int32)
            idx = np.full((2, mf), -9, np.int32)
            assert eng.lib.rf_detect_batch(eng.h, ptrs, ws, hs, rs, 2, THR, NMS, faces.ctypes.data, counts.ctypes.data, idx.ctypes.data) == 0
            assert counts.tolist() == [0, len(want[1])], (hw, counts)
            assert np.array_equal(faces[1, :counts[1]], want[1]) and np.array_equal(idx[1, :counts[1]], want_idx[1]), hw
            for i in range(2):
                assert (faces[i, counts[i]:] == CANARY).all() and (idx[i, counts[i]:] == -9).all(), (hw, i)
            vf = np.full((mf, 15), CANARY, np.float32)
            vo = np.full(mf, -9, np.int32)
            cnt = C.c_int(-7)
            views = (capi._View * 1)(capi._View(0.5, 0))
            assert eng.lib.rf_detect_views(eng.h, thin.ctypes.data, hw[1], hw[0], 0, views, 1, THR, NMS, vf.ctypes.data, C.byref(cnt),
                                           vo.ctypes.data, None) == 0
            assert cnt.value == 0 and (vf == CANARY).all() and (vo == -9).all(), hw
            t = capi.tiling()
            tf = np.full((1, mf, 15), CANARY, np.float32)
            tc = np.full(1, -7, np.int32)
            rc = eng.lib.rf_detect_tiled(eng.h, ptrs, ws, hs, rs, 1, C.byref(t), THR, NMS, tf.ctypes.data, tc.ctypes.data, None)
            assert rc == -1 and (tf == CANARY).all() and tc[0] == -7, (hw, rc)
        assert np.array_equal(eng.detect_batch([np.zeros((448, 448, 3), np.uint8), golden_image], THR, NMS)[1], want[1])
    finally:
        eng.close()
