"""GPU (-m gpu): f8 tiled detection of device-resident images and frames, and the crops of every tiled path -- rf_detect_tiled_device
/ rf_detect_yuv_tiled_device against the blocking rf_detect_tiled / rf_detect_yuv_tiled bit for bit, rf_detect_tiled_align /
rf_detect_yuv_tiled_align crops against cv2.warpAffine of the original, several device calls in flight over the slot ring, and
that nothing else changes.  Every comparison goes through the C ABI."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.align import ARCFACE_112, blob, umeyama
from oracle.yuv import bgr_to_frame, frame_to_bgr, split_planes

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
F32 = np.float32
LEVELS = [(1.0, 0), (0.5, 1), (0.0, 0)]


def _engine(prec="fp16", net=(448, 448), **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (2160, 3840))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), net[1], net[0], precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), net[1], net[0], precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


def _canvas(golden_image, w=3840, h=2160, xs=(32, 704, 1376, 2048, 2720), ys=(32, 512, 992)):
    """The f7 seam canvas: half-scale copies of the golden photo (640 x 443, faces about 50 x 70 px) on black, at 32-aligned
    positions."""
    half = cv2.resize(golden_image, (640, 443), interpolation=cv2.INTER_AREA)
    c = np.zeros((h, w, 3), np.uint8)
    for y in ys:
        for x in xs:
            c[y:y + 443, x:x + 640] = half
    return c, half, [(x, y) for y in ys for x in xs]


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _to_i420(nv12):
    y, u, v = split_planes(nv12, "nv12")
    return np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(nv12.shape)


def _nvdec_like(frame, pitch, coded_h):
    """NV12 on the device as NVDEC maps it: luma rows of `pitch` bytes, the interleaved chroma plane at pitch * coded height; the
    padding is 0xEE.  Returns the (y, uv) plane views and the surface."""
    import torch
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]
    surf = torch.full((coded_h + coded_h // 2, pitch), 0xEE, dtype=torch.uint8, device="cuda")
    surf[:h, :w] = _cuda(frame[:h])
    surf[coded_h:coded_h + h // 2, :w] = _cuda(frame[h:])
    return (surf[:h, :w], surf[coded_h:coded_h + h // 2, :w]), surf


def _warp(img, M, size=(112, 112)):
    return cv2.warpAffine(img, M, size, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def _assert_same(dev, host, tile_of, mf, what):
    faces, ids = dev
    for i, (f, want) in enumerate(zip(faces, host)):
        assert f.shape == want.shape and np.array_equal(f, want), (what, i, f.shape, want.shape)
        assert np.array_equal(ids[i] // mf, tile_of[i]), (what, i)


def _mixed_images(golden_image):
    rng = np.random.default_rng(11)
    canvas, _, _ = _canvas(golden_image)
    return [canvas, golden_image, golden_image[:, ::-1].copy(), cv2.resize(golden_image, (1279, 887)),   # sides of 3 mod 4
            cv2.resize(golden_image, (1920, 1080)), golden_image[100:700, 200:1100].copy(), rng.integers(0, 256, (500, 700, 3), np.uint8),
            golden_image]                                                                              # the last one: a strided view


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_device_bgr_equals_host(golden_image, prec):
    """Eight mixed images (the 4K canvas, the golden photo, a mirrored copy, 1279 x 887, 1920 x 1080, a crop, noise, and a row-strided
    view of a larger device tensor), levels {1, 0.5 mirrored, fitted} and the default pyramid: rf_detect_tiled_device records equal
    rf_detect_tiled's faces in value and order, and anchor_index / max_faces == out_tile_of."""
    import torch
    imgs = _mixed_images(golden_image)
    eng = _engine(prec)
    try:
        big = torch.full((886, 1300, 3), 0x5A, dtype=torch.uint8, device="cuda")
        big[:, :1280] = _cuda(golden_image)
        dev = [_cuda(im) for im in imgs[:-1]] + [big[:, :1280]]
        assert dev[-1].stride(0) == 3900
        torch.cuda.synchronize()
        for levels in (LEVELS, None):
            want, tile_of = eng.detect_tiled(imgs, THR, NMS, levels=levels)
            d, c = eng.detect_tiled_device(dev, THR, NMS, levels=levels)
            eng.synchronize()
            _assert_same(eng.read_dets(d, c, 8), want, tile_of, eng.max_faces, (prec, levels))
            assert sum(len(f) for f in want) >= 30
    finally:
        eng.close()


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_device_yuv_equals_host(golden_image, prec):
    """rf_detect_yuv_tiled_device on NV12 BT.601 and I420 BT.709 device frames (the 4K canvas, the golden photo, 1920 x 1080, 1038 x 670
    -- sides of 3 mod 4 at s = 0.5 -- and an NVDEC-like NV12 surface, luma pitch 2048, chroma at pitch x 1088) equals
    rf_detect_yuv_tiled on host copies, and anchor_index / max_faces == out_tile_of."""
    import torch
    canvas, _, _ = _canvas(golden_image)
    bgr = [canvas, golden_image, cv2.resize(golden_image, (1920, 1080)), cv2.resize(golden_image, (1038, 670))]
    eng = _engine(prec)
    try:
        for layout, matrix in (("nv12", "bt601"), ("i420", "bt709")):
            frames = [bgr_to_frame(b, "nv12") for b in bgr]
            if layout == "i420":
                frames = [_to_i420(f) for f in frames]
            dev = [_cuda(f) for f in frames]
            surf = None
            if layout == "nv12":
                planes, surf = _nvdec_like(frames[2], 2048, 1088)
                dev.append(planes)
                frames.append(frames[2])
            torch.cuda.synchronize()
            n = len(frames)
            for levels in (LEVELS, None):
                want, tile_of = eng.detect_yuv_tiled(frames, THR, NMS, layout, matrix, levels=levels)
                d, c = eng.detect_yuv_tiled_device(dev, THR, NMS, layout, matrix, levels=levels)
                eng.synchronize()
                _assert_same(eng.read_dets(d, c, n), want, tile_of, eng.max_faces, (prec, layout, levels))
                assert sum(len(f) for f in want) >= 20
            del surf
    finally:
        eng.close()


def _cut(eng, golden_image):
    """The golden photo cut through its right-most face (the crop of that face reaches past the image border)."""
    right = int(eng.detect_batch([golden_image], 0.9, NMS)[0][:, 3].max() * max(F32(1280 / 448), F32(886 / 448))) + 1
    return np.ascontiguousarray(golden_image[:, :right + (right & 1)])


def test_crops_of_every_tiled_path(golden_image):
    """Host _align and device variants, BGR and NV12, on the golden photo, the 4K canvas and the photo cut through a face, u8 / F32 /
    F16: faces bit-equal to the tiled call without crops; u8 crops == cv2.warpAffine(img, M_returned) (of cvtColor(frame) for NV12);
    M within 1e-9 relative of Umeyama on the returned landmarks; F32 within 1e-6 of blobFromImages(u8), F16 == F32 rounded; device
    crops and matrices == host ones."""
    import torch
    canvas, _, _ = _canvas(golden_image)
    eng = _engine("fp16")
    try:
        cut = _cut(eng, golden_image)
        zero_cols = 0
        for name, img in (("golden", golden_image), ("canvas", canvas), ("cut", cut)):
            frame = bgr_to_frame(img, "nv12")
            conv = frame_to_bgr(frame, "nv12")
            for kind, src in (("bgr", img), ("nv12", frame)):
                ref = conv if kind == "nv12" else img
                if kind == "bgr":
                    plain, plain_tile = eng.detect_tiled([src], THR, NMS)
                    faces, tile_of, u8, mats = eng.detect_tiled([src], THR, NMS, align=dict(want_mats=True))
                    f32 = eng.detect_tiled([src], THR, NMS, align=dict(fmt="rgb_f32"))[2]
                    f16 = eng.detect_tiled([src], THR, NMS, align=dict(fmt="rgb_f16"))[2]
                else:
                    plain, plain_tile = eng.detect_yuv_tiled([src], THR, NMS)
                    faces, tile_of, u8, mats = eng.detect_yuv_tiled([src], THR, NMS, align=dict(want_mats=True))
                    f32 = eng.detect_yuv_tiled([src], THR, NMS, align=dict(fmt="rgb_f32"))[2]
                    f16 = eng.detect_yuv_tiled([src], THR, NMS, align=dict(fmt="rgb_f16"))[2]
                assert np.array_equal(faces[0], plain[0]) and np.array_equal(tile_of[0], plain_tile[0]), (name, kind)
                assert len(u8[0]) == len(faces[0]) >= 3, (name, kind)
                for f, crop, M in zip(faces[0], u8[0], mats[0]):
                    assert np.array_equal(crop, _warp(ref, M)), (name, kind)
                    lm = np.stack([f[5:10], f[10:15]], axis=1).astype(np.float64)
                    want_m = umeyama(lm, ARCFACE_112)
                    assert np.abs(M - want_m).max() <= 1e-9 * np.abs(want_m).max(), (name, kind)
                if name == "cut":
                    zero_cols = max(zero_cols, max(int((c == 0).all(axis=2).any(axis=0).sum()) for c in u8[0]))
                assert np.abs(f32[0] - blob(u8[0])).max() <= 1e-6 and np.array_equal(f16[0], f32[0].astype(np.float16)), (name, kind)
                # the device variant into torch buffers
                A = eng.max_faces
                for fmt, host in (("bgr_u8", u8[0]), ("rgb_f16", f16[0])):
                    shape = (1, A, 112, 112, 3) if fmt == "bgr_u8" else (1, A, 3, 112, 112)
                    dt = torch.uint8 if fmt == "bgr_u8" else torch.float16
                    crops = torch.full(shape, 7, dtype=dt, device="cuda")
                    dmats = torch.zeros((1, A, 2, 3), dtype=torch.float64, device="cuda")
                    if kind == "bgr":
                        d, c = eng.detect_tiled_device([_cuda(src)], THR, NMS, align=dict(fmt=fmt), dev_crops_ptr=crops.data_ptr(),
                                                       dev_mats_ptr=dmats.data_ptr())
                    else:
                        d, c = eng.detect_yuv_tiled_device([_cuda(src)], THR, NMS, align=dict(fmt=fmt), dev_crops_ptr=crops.data_ptr(),
                                                           dev_mats_ptr=dmats.data_ptr())
                    eng.synchronize()
                    df, ids = eng.read_dets(d, c, 1)
                    k = len(faces[0])
                    assert np.array_equal(df[0], faces[0]) and np.array_equal(ids[0] // eng.max_faces, tile_of[0])
                    assert np.array_equal(crops[0, :k].cpu().numpy(), host) and (crops[0, k:] == 7).all(), (name, kind, fmt)
                    assert np.array_equal(dmats[0, :k].cpu().numpy(), mats[0]), (name, kind, fmt)
        assert zero_cols > 4, zero_cols          # the face cut by the image border is zero-filled beyond it
    finally:
        eng.close()


def test_max_faces_writes_only_the_top_crops(golden_image):
    """align max_faces = 2 on two images (the golden photo and noise without faces): the host and device crops are the first two of the
    unlimited call's, slots without a face and the bytes after the buffer keep their canary."""
    import torch
    eng = _engine("fp16")
    try:
        imgs = [golden_image, np.random.default_rng(5).integers(0, 256, (400, 300, 3), np.uint8)]
        faces, _, full = eng.detect_tiled(imgs, THR, NMS, align={})
        _, _, top = eng.detect_tiled(imgs, THR, NMS, align=dict(max_faces=2))
        counts = [len(f) for f in faces]
        assert counts[0] > 2 and counts[1] < 2, counts
        for i in range(2):
            assert np.array_equal(top[i], full[i][:2])
        A, cb = 2, 112 * 112 * 3
        buf = torch.full((2 * A * cb + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
        eng.detect_tiled_device([_cuda(im) for im in imgs], THR, NMS, align=dict(max_faces=2), dev_crops_ptr=buf.data_ptr())
        eng.synchronize()
        got = buf.cpu().numpy()
        for i in range(2):
            for j in range(A):
                s = got[(i * A + j) * cb:(i * A + j + 1) * cb]
                if j < counts[i]:
                    assert np.array_equal(s.reshape(112, 112, 3), full[i][j]), (i, j)
                else:
                    assert (s == 0xA5).all(), (i, j)
        assert (got[2 * A * cb:] == 0xA5).all()
    finally:
        eng.close()


def _iou(a, b):
    iw = min(a[3], b[3]) - max(a[1], b[1]) + 1
    ih = min(a[4], b[4]) - max(a[2], b[2]) + 1
    inter = max(iw, 0) * max(ih, 0)
    return inter / ((a[3] - a[1] + 1) * (a[4] - a[2] + 1) + (b[3] - b[1] + 1) * (b[4] - b[2] + 1) - inter)


def test_small_faces_get_crops(golden_image):
    """The seam canvas (15 half-scale golden-photo copies on 3840 x 2160), the default pyramid with crops: one crop per found face, every
    expected face matched (IoU >= 0.5), every crop == its warp byte for byte, host and device alike; rf_detect_align_batch on the canvas
    finds strictly fewer faces."""
    import torch
    canvas, half, pos = _canvas(golden_image)
    one = _engine("fp16", net=(672, 448), max_batch=1, max_image=(448, 672))
    try:
        ref = one.detect_batch([half], 0.9, NMS)[0]
    finally:
        one.close()
    assert len(ref) >= 3
    expected = []
    for x, y in pos:
        e = ref.copy()
        e[:, [1, 3]] += F32(x)
        e[:, [2, 4]] += F32(y)
        expected.append(e)
    expected = np.concatenate(expected)
    eng = _engine("fp16")
    try:
        faces, _, crops, mats = eng.detect_tiled([canvas], THR, NMS, align=dict(want_mats=True))
        assert len(crops[0]) == len(faces[0])
        for e in expected:
            assert any(_iou(e, f) >= 0.5 for f in faces[0]), e[:5]
        for crop, M in zip(crops[0], mats[0]):
            assert np.array_equal(crop, _warp(canvas, M))
        A = eng.max_faces
        buf = torch.zeros((1, A, 112, 112, 3), dtype=torch.uint8, device="cuda")
        eng.detect_tiled_device([_cuda(canvas)], THR, NMS, align={}, dev_crops_ptr=buf.data_ptr())
        eng.synchronize()
        assert np.array_equal(buf[0, :len(crops[0])].cpu().numpy(), np.stack(crops[0]))
        plain, _ = eng.detect_align([canvas], THR, NMS)
        print(f"small faces: {len(expected)} expected, tiled {len(faces[0])} faces / crops, rf_detect_align_batch {len(plain[0])}")
        assert len(plain[0]) < len(expected) <= len(faces[0])
    finally:
        eng.close()


def _in_flight(eng, golden_image, streams, sizes):
    """2 streams + 1 device tiled calls, alternating BGR and NV12, each image set different (rolled), crops into a torch buffer per
    call, an rf_detect_batch_device call between each two, no host synchronise; then every crop buffer == its blocking twin's crops, the
    records of the last `streams` calls == the blocking results, and the frames' checksums are unchanged."""
    import torch
    from oracle.inputs import letterbox_bgr_u8
    calls = 2 * streams + 1
    A = eng.max_faces
    net_in = _cuda(np.stack([letterbox_bgr_u8(golden_image, 448, 448)] * 2))
    host, dev, out, bufs = [], [], [], []
    for k in range(calls):
        w, h = sizes(k)
        base = cv2.resize(golden_image, (w, h)) if (w, h) != (1280, 886) else golden_image
        imgs = [np.roll(base, 16 * (2 * k + i) + 8, axis=1) for i in range(2)]
        kind = "bgr" if k % 2 == 0 else "nv12"
        srcs = imgs if kind == "bgr" else [bgr_to_frame(im, "nv12") for im in imgs]
        host.append((kind, srcs))
        dev.append([_cuda(s) for s in srcs])
        bufs.append(torch.full((2, A, 3, 112, 112), 7.0, dtype=torch.float16, device="cuda"))
    torch.cuda.synchronize()
    sums = [[int(t.to(torch.int64).sum()) for t in d] for d in dev]
    for k in range(calls):
        kind = host[k][0]
        fn = eng.detect_tiled_device if kind == "bgr" else eng.detect_yuv_tiled_device
        out.append(fn(dev[k], THR, NMS, align=dict(fmt="rgb_f16"), dev_crops_ptr=bufs[k].data_ptr()))
        eng.detect_device(2, THR, NMS, net_in.data_ptr())
    eng.synchronize()
    for k in range(calls):
        kind, srcs = host[k]
        if kind == "bgr":
            faces, tile_of, crops = eng.detect_tiled(srcs, THR, NMS, align=dict(fmt="rgb_f16"))
        else:
            faces, tile_of, crops = eng.detect_yuv_tiled(srcs, THR, NMS, align=dict(fmt="rgb_f16"))
        for i in range(2):
            kk = len(crops[i])
            assert kk > 0 and np.array_equal(bufs[k][i, :kk].cpu().numpy(), crops[i]), (k, i)
            assert (bufs[k][i, kk:] == 7.0).all(), (k, i)
        if k >= calls - streams:
            _assert_same(eng.read_dets(out[k][0], out[k][1], 2), faces, tile_of, eng.max_faces, k)
    assert [[int(t.to(torch.int64).sum()) for t in d] for d in dev] == sums


@pytest.mark.parametrize("streams", [2, 8])
def test_several_calls_in_flight(golden_image, streams):
    eng = _engine("fp16", max_batch=4, streams=streams)
    try:
        _in_flight(eng, golden_image, streams, lambda k: (1920, 1080))
    finally:
        eng.close()
    # slot growth mid-sequence: the first calls have small layouts, the later ones 4K layouts, so each reused slot grows
    eng = _engine("fp16", max_batch=4, streams=streams)
    try:
        _in_flight(eng, golden_image, streams, lambda k: (1280, 886) if k == 0 else (3840, 2160))
    finally:
        eng.close()


def test_nothing_else_changes_and_bad_calls_launch_nothing(golden_image):
    import torch
    from retinaface_b200 import RfError, capi
    imgs = [golden_image, cv2.resize(golden_image, (1920, 1080))]
    big = cv2.resize(golden_image, (3840, 2160))
    eng = _engine("fp16")
    try:
        before = eng.detect_batch(imgs, THR, NMS, want_index=True)
        tiled_before = eng.detect_tiled(imgs, THR, NMS, levels=LEVELS)
        launches = eng.launches_per_batch(8)
        dev = [_cuda(im) for im in imgs]
        frame = bgr_to_frame(imgs[1], "nv12")
        eng.detect_tiled_device(dev, THR, NMS)
        eng.detect_yuv_tiled_device([_cuda(frame)], THR, NMS, align={}, dev_crops_ptr=torch.empty(256 * 112 * 112 * 3, dtype=torch.uint8,
                                                                                                   device="cuda").data_ptr())
        eng.detect_tiled(imgs, THR, NMS, align={})
        eng.detect_yuv_tiled([frame], THR, NMS, align={})
        eng.synchronize()
        after = eng.detect_batch(imgs, THR, NMS, want_index=True)
        for a, b in zip(before, after):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
        tiled_after = eng.detect_tiled(imgs, THR, NMS, levels=LEVELS)
        for a, b in zip(tiled_before, tiled_after):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
        assert eng.launches_per_batch(8) == launches

        lib, h = eng.lib, eng.h
        d_big = _cuda(big)
        canary = torch.full((4096,), 0xA5, dtype=torch.uint8, device="cuda")
        good_t = capi.tiling()
        good_a = capi.align_params()
        bad_a = capi.align_params(crop=(4, 4))

        def dev_bgr(ptrs, ws, hs, rs, n, t=good_t, align=None, crops=canary.data_ptr()):
            """rf_detect_tiled_device with raw arguments; returns (status, dets pointer untouched)."""
            d, c = C.c_void_p(), C.c_void_p()
            rc = lib.rf_detect_tiled_device(h, ptrs, ws, hs, rs, n, C.byref(t), THR, NMS, C.byref(align) if align is not None else None, crops,
                                            None, C.byref(d), C.byref(c))
            return rc, d.value is None and c.value is None

        def arr(T, vals):
            return (T * len(vals))(*vals)

        P, I = C.c_void_p, C.c_int
        one = (arr(P, [d_big.data_ptr()]), arr(I, [3840]), arr(I, [2160]), arr(I, [0]))
        cases = [
            (dev_bgr(None, one[1], one[2], None, 1), -1),                                            # NULL arrays
            (dev_bgr(arr(P, [None]), one[1], one[2], None, 1), -1),                                   # empty image
            (dev_bgr(one[0], arr(I, [0]), one[2], None, 1), -1),
            (dev_bgr(one[0], one[1], one[2], arr(I, [3840 * 3 - 1]), 1), -1),                         # row stride below 3 w
            (dev_bgr(one[0], arr(I, [3842]), one[2], None, 1), -6),                                   # above max_image
            (dev_bgr(arr(P, [d_big.data_ptr()] * 9), arr(I, [3840] * 9), arr(I, [2160] * 9), None, 9), -6),   # n > max_batch
            (dev_bgr(*one, 1, t=capi.tiling([(-1.0, 0)])), -1),                                       # tile_layout's statuses
            (dev_bgr(*one, 1, t=capi.tiling([(2.0, 0), (1.0, 0)])), -6),
            (dev_bgr(*one, 1, t=capi.tiling(overlap=8)), -1),
            (dev_bgr(*one, 1, align=bad_a), -1),                                                      # bad align params
            (dev_bgr(*one, 1, align=good_a, crops=None), -1),                                         # align without dev_crops
        ]
        for k, ((rc, untouched), status) in enumerate(cases):
            assert rc == status and untouched, (k, rc, status)

        d_frame = _cuda(bgr_to_frame(big, "nv12"))
        f = capi.yuv_frame(d_frame, "nv12")[0]
        odd = capi.yuv_frame(d_frame, "nv12")[0]
        odd.width = 3839
        for fr, align, crops, status in ((odd, None, None, -1), (f, bad_a, canary.data_ptr(), -1), (f, good_a, None, -1)):
            d, c = C.c_void_p(), C.c_void_p()
            rc = lib.rf_detect_yuv_tiled_device(h, C.byref(fr), 1, 0, C.byref(good_t), THR, NMS, C.byref(align) if align is not None else None,
                                                crops, None, C.byref(d), C.byref(c))
            assert rc == status and d.value is None, (rc, status)
        d, c = C.c_void_p(), C.c_void_p()
        assert lib.rf_detect_yuv_tiled_device(h, C.byref(f), 1, 7, C.byref(good_t), THR, NMS, None, None, None, C.byref(d), C.byref(c)) == -1

        # host _align variants: outputs keep their canaries
        faces = np.full((2, eng.max_faces, 15), -3.0, np.float32)
        counts = np.full(2, -3, np.int32)
        crops = np.full(2 * eng.max_faces * 112 * 112 * 3, 0xA5, np.uint8)
        ptrs = arr(P, [big.ctypes.data])
        for align, out_crops, status in ((bad_a, crops.ctypes.data, -1), (good_a, None, -1), (None, crops.ctypes.data, -1)):
            rc = lib.rf_detect_tiled_align(h, ptrs, arr(I, [3840]), arr(I, [2160]), None, 1, C.byref(good_t), THR, NMS,
                                           C.byref(align) if align is not None else None, faces.ctypes.data, counts.ctypes.data, None,
                                           out_crops, None)
            assert rc == status, (rc, status)
        h_frame = bgr_to_frame(big, "nv12")
        fr = capi.yuv_frame(h_frame, "nv12")[0]
        for align, out_crops in ((bad_a, crops.ctypes.data), (good_a, None), (None, crops.ctypes.data)):
            rc = lib.rf_detect_yuv_tiled_align(h, C.byref(fr), 1, 0, C.byref(good_t), THR, NMS, C.byref(align) if align is not None else None,
                                               faces.ctypes.data, counts.ctypes.data, None, out_crops, None)
            assert rc == -1, rc
        assert (faces == -3.0).all() and (counts == -3).all() and (crops == 0xA5).all()
        torch.cuda.synchronize()
        assert (canary == 0xA5).all()
        again = eng.detect_batch(imgs, THR, NMS, want_index=True)
        for a, b in zip(before, again):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        eng.close()
    # more images than raw buffers: the host _align variants cannot keep every original resident
    few = _engine("fp16", max_image=(8192, 16384))
    try:
        with pytest.raises(RfError) as e:
            few.detect_tiled([golden_image] * 8, THR, NMS, align={})
        assert e.value.status == -6
        frame = bgr_to_frame(golden_image, "nv12")
        with pytest.raises(RfError) as e:
            few.detect_yuv_tiled([frame] * 8, THR, NMS, align={})
        assert e.value.status == -6
        assert len(few.detect_tiled([golden_image] * 8, THR, NMS)[0]) == 8       # without crops the call groups its uploads
    finally:
        few.close()
    npp = _engine("fp16", flags=capi.RF_FLAG_NPP_RESIZE)
    try:
        for call in (lambda: npp.detect_tiled([golden_image], THR, NMS, align={}),
                     lambda: npp.detect_yuv_tiled([bgr_to_frame(golden_image, "nv12")], THR, NMS, align={}),
                     lambda: npp.detect_tiled_device([_cuda(golden_image)], THR, NMS),
                     lambda: npp.detect_yuv_tiled_device([_cuda(bgr_to_frame(golden_image, "nv12"))], THR, NMS)):
            with pytest.raises(RfError) as e:
                call()
            assert e.value.status == -7
    finally:
        npp.close()


def test_detector_detect_tiled_with_crops(golden_image):
    """RetinaFace.detectTiled(align=...): (FaceDetectInfo, crop) pairs equal to Engine.detect_tiled's faces and crops."""
    from retinaface_b200 import RetinaFace
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(2160, 3840))
    canvas, _, _ = _canvas(golden_image)
    per = rf.detectTiled([canvas, golden_image], 0.5, align={})
    faces, _, crops = rf.engine.detect_tiled([canvas, golden_image], 0.5, 0.4, align={})
    assert [len(p) for p in per] == [len(f) for f in faces] and len(per[0]) > 20
    for p, f, c in zip(per, faces, crops):
        for (info, crop), row, want in zip(p, f, c):
            assert info.score == float(row[0]) and np.array_equal(crop, want)
