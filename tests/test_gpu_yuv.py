"""GPU (-m gpu): f6 video frames -- rf_preprocess_yuv / rf_detect_yuv_batch / rf_detect_yuv_batch_device against the BGR paths run
on oracle/yuv.py's conversion of the same frames (== cv2.cvtColor for BT.601), through the C ABI."""
import ctypes as C

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.inputs import letterbox_bgr_u8
from oracle.yuv import LAYOUTS, bgr_to_frame, frame_to_bgr, split_planes

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4


def _engine(prec="fp16", **kw):
    import os
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (1088, 1920))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


def _scale(w, h):
    return max(np.float32(w / 448), np.float32(h / 448), np.float32(1.0))


def _even(img):
    return np.ascontiguousarray(img[:img.shape[0] // 2 * 2, :img.shape[1] // 2 * 2])


def _pitched(frame, layout, pad=37):
    """The frame's planes cut out of wider allocations whose padding is 0xEE."""
    planes = split_planes(frame, layout)
    if layout in ("nv12", "nv21"):
        h = planes[0].shape[0]
        planes = (planes[0], frame[h:])
    out = []
    for p in planes:
        buf = np.full((p.shape[0], p.shape[1] + pad), 0xEE, np.uint8)
        buf[:, :p.shape[1]] = p
        out.append(buf[:, :p.shape[1]])
    return tuple(out)


def _nvdec_like(frame, pitch=2048, coded_h=1088):
    """NV12 as NVDEC maps it: luma rows of `pitch` bytes, the interleaved chroma plane at pitch * coded_height."""
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]
    surf = np.full((coded_h + coded_h // 2, pitch), 0xEE, np.uint8)
    surf[:h, :w] = frame[:h]
    surf[coded_h:coded_h + h // 2, :w] = frame[h:]
    return surf[:h, :w], surf[coded_h:coded_h + h // 2, :w]


def _frames_of(golden_image):
    rng = np.random.default_rng(3)
    return {
        "448x448": bgr_to_frame(letterbox_bgr_u8(golden_image, 448, 448), "i420"),
        "1920x1080": bgr_to_frame(cv2.resize(golden_image, (1920, 1080)), "i420"),
        "1282x722": rng.integers(0, 256, (722 * 3 // 2, 1282), dtype=np.uint8),
        "320x240": bgr_to_frame(cv2.resize(golden_image, (320, 240), interpolation=cv2.INTER_AREA), "i420"),
    }


def _relayout(i420, layout):
    """The same samples in another layout (no colour round trip)."""
    y, u, v = split_planes(i420, "i420")
    h, w = y.shape
    if layout == "i420":
        return i420
    if layout == "yv12":
        return np.concatenate([y.reshape(-1), v.reshape(-1), u.reshape(-1)]).reshape(h * 3 // 2, w)
    a, b = (u, v) if layout == "nv12" else (v, u)
    return np.concatenate([y, np.stack([a, b], axis=-1).reshape(h // 2, w)])


@pytest.mark.parametrize("matrix", ["bt601", "bt709"])
def test_preprocess_equals_letterbox_of_converted_frame(golden_image, matrix):
    eng = _engine(max_batch=1)
    try:
        for name, i420 in _frames_of(golden_image).items():
            for layout in LAYOUTS:
                frame = _relayout(i420, layout)
                want = letterbox_bgr_u8(frame_to_bgr(frame, layout, matrix), 448, 448)
                assert np.array_equal(eng.preprocess_yuv(frame, layout, matrix), want), (name, layout)
                assert np.array_equal(eng.preprocess_yuv(_pitched(frame, layout), layout, matrix), want), (name, layout, "pitched")
        f = _relayout(_frames_of(golden_image)["1920x1080"], "nv12")
        want = letterbox_bgr_u8(frame_to_bgr(f, "nv12", matrix), 448, 448)
        assert np.array_equal(eng.preprocess_yuv(_nvdec_like(f), "nv12", matrix), want)
    finally:
        eng.close()


def test_npp_resize_equals_bgr_path(golden_image):
    from retinaface_b200.capi import RF_FLAG_NPP_RESIZE
    eng = _engine(max_batch=1, flags=RF_FLAG_NPP_RESIZE)
    try:
        for name, i420 in _frames_of(golden_image).items():
            for layout in LAYOUTS:
                frame = _relayout(i420, layout)
                for matrix in ("bt601", "bt709"):
                    want = eng.preprocess(frame_to_bgr(frame, layout, matrix))
                    assert np.array_equal(eng.preprocess_yuv(frame, layout, matrix), want), (name, layout, matrix)
                    assert np.array_equal(eng.preprocess_yuv(_pitched(frame, layout), layout, matrix), want), (name, layout, matrix)
    finally:
        eng.close()


def _mixed_frames(golden_image, n):
    g = _even(golden_image)
    pool = [bgr_to_frame(g, "nv12"), bgr_to_frame(cv2.resize(golden_image, (1920, 1080)), "nv12"),
            bgr_to_frame(letterbox_bgr_u8(golden_image, 448, 448), "nv12"), bgr_to_frame(_even(golden_image[100:700, 200:1100]), "nv12"),
            bgr_to_frame(cv2.resize(golden_image, (640, 442)), "nv12"), bgr_to_frame(np.roll(g, 40, axis=1), "nv12"),
            bgr_to_frame(cv2.resize(golden_image, (1282, 722)), "nv12"), bgr_to_frame(g[::-1].copy(), "nv12")]
    return pool[:n]


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_detect_host_and_device_equal_bgr_detect(golden_image, prec):
    import torch
    eng = _engine(prec)
    try:
        for n in (1, 3, 8):
            for layout, matrix in (("nv12", "bt601"), ("i420", "bt709")):
                frames = [f if layout == "nv12" else _to_i420(f) for f in _mixed_frames(golden_image, n)]
                bgr = [frame_to_bgr(f, layout, matrix) for f in frames]
                ref, ref_idx = eng.detect_batch(bgr, THR, NMS, want_index=True)
                want = []
                for im, r in zip(bgr, ref):
                    w = r.copy()
                    w[:, 1:] = r[:, 1:] * _scale(im.shape[1], im.shape[0])
                    want.append(w)
                faces, idx = eng.detect_yuv(frames, THR, NMS, layout, matrix, want_index=True)
                pinned = [torch.from_numpy(f).pin_memory().numpy() for f in frames]
                pf, pidx = eng.detect_yuv(pinned, THR, NMS, layout, matrix, want_index=True)
                dev = [torch.from_numpy(f).cuda() for f in frames]
                torch.cuda.synchronize()
                d, c, scales = eng.detect_yuv_device(dev, THR, NMS, layout, matrix)
                df, didx = eng.read_dets(d, c, n)
                for i in range(n):
                    assert np.array_equal(faces[i], want[i]) and np.array_equal(idx[i], ref_idx[i]), (n, layout, i)
                    assert np.array_equal(pf[i], want[i]) and np.array_equal(pidx[i], ref_idx[i])
                    assert np.array_equal(df[i], ref[i]) and np.array_equal(didx[i], ref_idx[i])
                    assert scales[i] == _scale(bgr[i].shape[1], bgr[i].shape[0])
                assert sum(len(f) for f in faces) >= n
    finally:
        eng.close()


def _to_i420(nv12):
    y, u, v = split_planes(nv12, "nv12")
    return np.concatenate([y.reshape(-1), u.reshape(-1), v.reshape(-1)]).reshape(nv12.shape)


def _warp(img, M, size=(112, 112)):
    return cv2.warpAffine(img, M, size, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def test_crops_equal_warp_of_converted_frame(golden_image):
    from oracle.align import blob
    eng = _engine()
    try:
        g = _even(golden_image)
        right = int(eng.detect_batch([g], 0.9, NMS)[0][:, 3].max() * _scale(g.shape[1], g.shape[0])) + 1
        cut = _even(g[:, :right + (right & 1)])
        for src in (g, cut):
            for layout in ("nv12", "yv12"):
                frame = _relayout(bgr_to_frame(src, "i420"), layout)
                bgr = frame_to_bgr(frame, layout)
                _, _, ref_m = eng.detect_align([bgr], THR, NMS, want_mats=True)
                faces, crops, mats = eng.detect_yuv([frame], THR, NMS, layout, align=dict(want_mats=True))
                assert len(crops[0]) >= 1 and np.array_equal(mats[0], ref_m[0])
                for crop, M in zip(crops[0], mats[0]):
                    assert np.array_equal(crop, _warp(bgr, M))
                f32 = eng.detect_yuv([frame], THR, NMS, layout, align=dict(fmt="rgb_f32"))[1][0]
                f16 = eng.detect_yuv([frame], THR, NMS, layout, align=dict(fmt="rgb_f16"))[1][0]
                assert np.abs(f32 - blob(crops[0])).max() <= 1e-6 and np.array_equal(f16, f32.astype(np.float16))
        zero_cols = [(c == 0).all(axis=2).any(axis=0).sum() for c in crops[0]]
        assert max(zero_cols) > 4, zero_cols           # the last source is the cut frame: its edge face is zero-filled
    finally:
        eng.close()


def test_device_calls_over_two_contexts_leave_frames_untouched(golden_image):
    import torch
    eng = _engine(streams=2, max_batch=4)
    try:
        g = _even(golden_image)
        batches = [[bgr_to_frame(np.roll(g, 24 * (4 * b + i), axis=1), "nv12") for i in range(4)] for b in range(4)]
        dev = [[torch.from_numpy(f).cuda() for f in fs] for fs in batches]
        torch.cuda.synchronize()
        sums = [[int(t.to(torch.int64).sum()) for t in fs] for fs in dev]
        A = eng.max_faces
        crops = [torch.full((4, A, 3, 112, 112), 7.0, dtype=torch.float16, device="cuda") for _ in range(4)]
        mats = [torch.zeros((4, A, 2, 3), dtype=torch.float64, device="cuda") for _ in range(4)]
        out = []
        for b in range(4):
            out.append(eng.detect_yuv_device(dev[b], THR, NMS, "nv12", align=dict(fmt="rgb_f16"), dev_crops_ptr=crops[b].data_ptr(),
                                             dev_mats_ptr=mats[b].data_ptr()))
        eng.synchronize()
        for b in range(4):
            ref = eng.detect_batch([frame_to_bgr(f, "nv12") for f in batches[b]], THR, NMS)
            _, want_c, want_m = eng.detect_yuv(batches[b], THR, NMS, "nv12", align=dict(fmt="rgb_f16", want_mats=True))
            # out[b]'s device records were overwritten by later calls on the same context only after 2 more calls: re-run alone
            d, c, _ = eng.detect_yuv_device(dev[b], THR, NMS, "nv12")
            faces, _ = eng.read_dets(d, c, 4)
            for i in range(4):
                k = len(want_c[i])
                assert k > 0 and np.array_equal(faces[i], ref[i])
                assert np.array_equal(crops[b][i, :k].cpu().numpy(), want_c[i]) and np.array_equal(mats[b][i, :k].cpu().numpy(), want_m[i])
                assert (crops[b][i, k:] == 7.0).all()
        assert [[int(t.to(torch.int64).sum()) for t in fs] for fs in dev] == sums
    finally:
        eng.close()


def test_yuv_calls_change_nothing_for_bgr_detect_and_reject_bad_frames(golden_image):
    import torch
    from retinaface_b200 import RfError, capi
    eng = _engine()
    try:
        imgs = [golden_image, letterbox_bgr_u8(golden_image, 448, 448)]
        launches = eng.launches_per_batch(2)
        before = eng.detect_batch(imgs, THR, NMS, want_index=True)
        frame = bgr_to_frame(_even(golden_image), "nv12")
        eng.detect_yuv([frame], THR, NMS, align=dict())
        eng.detect_yuv_device([torch.from_numpy(frame).cuda()], THR, NMS)
        eng.synchronize()
        after = eng.detect_batch(imgs, THR, NMS, want_index=True)
        for a, b in zip(before[0] + before[1], after[0] + after[1]):
            assert np.array_equal(a, b)
        assert eng.launches_per_batch(2) == launches

        good, _ = capi.yuv_frame(frame, "nv12")

        def bad(**kw):
            f = capi.YuvFrame.from_buffer_copy(good)
            for k, v in kw.items():
                setattr(f, k, v)
            return f
        cases = [(bad(width=1279), -1), (bad(height=0), -1), (bad(y=None), -1), (bad(v=None), -1), (bad(uv_step=3), -1),
                 (bad(v=good.u + 2), -1), (bad(y_pitch=1278), -1), (bad(uv_pitch=1278), -1),
                 (bad(width=2048, y_pitch=2048, uv_pitch=2048), -6)]
        faces = np.empty((8, eng.max_faces, 15), np.float32)
        counts = np.zeros(8, np.int32)
        out = np.empty((448, 448, 3), np.uint8)
        for f, status in cases:
            arr = (capi.YuvFrame * 1)(f)
            assert eng.lib.rf_detect_yuv_batch(eng.h, arr, 1, 0, THR, NMS, None, faces.ctypes.data, counts.ctypes.data, None, None, None) == status
            assert eng.lib.rf_preprocess_yuv(eng.h, arr, 0, out.ctypes.data) == status
            d, c = C.c_void_p(), C.c_void_p()
            assert eng.lib.rf_detect_yuv_batch_device(eng.h, arr, 1, 0, THR, NMS, None, None, None, C.byref(d), C.byref(c), None) == status
        arr = (capi.YuvFrame * 9)(*([good] * 9))
        assert eng.lib.rf_detect_yuv_batch(eng.h, arr, 9, 0, THR, NMS, None, faces.ctypes.data, counts.ctypes.data, None, None, None) == -6
        assert eng.lib.rf_detect_yuv_batch(eng.h, arr, 1, 2, THR, NMS, None, faces.ctypes.data, counts.ctypes.data, None, None, None) == -1
        p = capi.align_params()
        p.format = 7
        assert eng.lib.rf_detect_yuv_batch(eng.h, arr, 1, 0, THR, NMS, C.byref(p), faces.ctypes.data, counts.ctypes.data, None, out.ctypes.data,
                                           None) == -1
        assert eng.launches_per_batch(2) == launches
        after2 = eng.detect_batch(imgs, THR, NMS, want_index=True)
        for a, b in zip(before[0] + before[1], after2[0] + after2[1]):
            assert np.array_equal(a, b)
    finally:
        eng.close()


def test_python_class_surface(golden_image):
    from retinaface_b200 import RetinaFace
    rf = RetinaFace(GOLDEN + "/weights", model_file="mnet-deconv-0517.caffemodel")
    frame = bgr_to_frame(_even(golden_image), "i420")
    bgr = frame_to_bgr(frame, "i420")
    per = rf.detectFrames([frame], 0.9, layout="i420")[0]
    ref = rf.detectAndAlign([bgr], 0.9)[0]
    assert len(per) == len(ref) == 5 and all(a == b for a, (b, _) in zip(per, ref))
    pairs = rf.detectFrames([frame], 0.9, layout="i420", align=dict())[0]
    assert all(np.array_equal(c, rc) for (_, c), (_, rc) in zip(pairs, ref))
