"""GPU (-m gpu): f5 face alignment -- rf_detect_align_batch / rf_detect_align_batch_device against rf_detect_batch, the numpy
Umeyama estimator and cv2.warpAffine / cv2.dnn.blobFromImages (oracle/align.py), through the C ABI."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.align import ARCFACE_112, blob, umeyama
from oracle.inputs import letterbox_bgr_u8

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4


def _engine(prec=None, **kw):
    from retinaface_b200 import RF_PREC_FP16, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (1024, 1536))
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP16 if prec is None else prec, **kw)


def _scale(img):
    """The letter-box's map-back factor, in float32 the way it computes it."""
    h, w = img.shape[:2]
    return max(np.float32(w / 448), np.float32(h / 448), np.float32(1.0))


def _warp(img, M, size):
    return cv2.warpAffine(img, M, size, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def _check_image(img, faces, crops, mats, ref_net, size=(112, 112), template=ARCFACE_112):
    """faces == rf_detect_batch x scale bit for bit; M == numpy Umeyama to 1e-9; crops == cv2.warpAffine(img, M) byte for byte
    and within 1 LSB on <= 0.1 % of the bytes of cv2.warpAffine(img, numpy M)."""
    want = ref_net.copy()
    want[:, 1:] = ref_net[:, 1:] * _scale(img)
    assert faces.dtype == np.float32 and np.array_equal(faces, want)
    assert len(crops) == len(faces) and len(mats) == len(faces)
    for f, crop, M in zip(faces, crops, mats):
        p = np.stack([f[5:10], f[10:15]], axis=1)
        Mn = umeyama(p, np.asarray(template, np.float32))
        assert np.abs(M - Mn).max() <= 1e-9 * np.abs(Mn).max(), (M, Mn)
        assert np.array_equal(crop, _warp(img, M, size))
        d = np.abs(crop.astype(int) - _warp(img, Mn, size).astype(int))
        assert d.max() <= 1 and (d > 0).mean() <= 1e-3


@pytest.mark.parametrize("prec", ["fp32", "fp16"])
def test_golden_photo_faces_matrices_and_crops(golden_image, prec):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32
    eng = _engine(RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16)
    try:
        ref = eng.detect_batch([golden_image], THR, NMS)[0]
        faces, crops, mats = eng.detect_align([golden_image], THR, NMS, want_mats=True)
        assert len(ref) >= 5
        _check_image(golden_image, faces[0], crops[0], mats[0], ref)
    finally:
        eng.close()


def _cut_image(golden_image, eng):
    """The photo cropped at the right edge of its right-most face's box: the template crop reaches past the box, so part of that
    face's crop lies outside the image and is zero-filled."""
    f = eng.detect_batch([golden_image], 0.9, NMS)[0]
    right = int(f[:, 3].max() * _scale(golden_image)) + 1
    return np.ascontiguousarray(golden_image[:, :right])


@pytest.mark.parametrize("n", [1, 3, 8])
def test_mixed_batches_sizes_strides_pinned_and_pageable(golden_image, n):
    import torch
    eng = _engine()
    try:
        net = letterbox_bgr_u8(golden_image, 448, 448)
        big = np.zeros((1000, 1500, 3), np.uint8)
        big[57:57 + 886, 91:91 + 1280] = golden_image
        strided = big[57:57 + 886, 91:91 + 1280]                    # row stride 4500 bytes
        small = np.ascontiguousarray(cv2.resize(golden_image, (420, 291), interpolation=cv2.INTER_AREA))
        cut = _cut_image(golden_image, eng)
        pool = [cut, net, golden_image, small, strided, np.roll(net, 40, axis=1), golden_image[100:700, 200:1100], net[::-1].copy()]
        imgs = pool[:n] if n > 1 else [cut]
        ref = eng.detect_batch([np.ascontiguousarray(im) for im in imgs], THR, NMS)
        faces, crops, mats = eng.detect_align(imgs, THR, NMS, want_mats=True)
        pinned = [torch.from_numpy(np.ascontiguousarray(im)).pin_memory().numpy() for im in imgs]
        pf, pc, pm = eng.detect_align(pinned, THR, NMS, want_mats=True)
        for i, im in enumerate(imgs):
            _check_image(np.ascontiguousarray(im), faces[i], crops[i], mats[i], ref[i])
            assert np.array_equal(pf[i], faces[i]) and np.array_equal(pc[i], crops[i]) and np.array_equal(pm[i], mats[i])
        zero_filled = [(c == 0).all(axis=2).any(axis=0).sum() for c in crops[0]]
        assert len(crops[0]) > 0 and max(zero_filled) > 4, zero_filled     # the cut face: columns of border zeros
    finally:
        eng.close()


def test_float_formats_and_templates(golden_image):
    eng = _engine()
    try:
        u8, = eng.detect_align([golden_image], THR, NMS)[1]
        f32, = eng.detect_align([golden_image], THR, NMS, fmt="rgb_f32")[1]
        f16, = eng.detect_align([golden_image], THR, NMS, fmt="rgb_f16")[1]
        assert f32.shape == (len(u8), 3, 112, 112) and f32.dtype == np.float32
        assert np.abs(f32 - blob(u8)).max() <= 1e-6
        want = cv2.dnn.blobFromImages(list(u8), 1 / 127.5, (112, 112), (127.5, 127.5, 127.5), swapRB=True)
        assert np.abs(f32 - want).max() <= 1e-6
        assert f16.dtype == np.float16 and np.array_equal(f16, f32.astype(np.float16))
        f32b, = eng.detect_align([golden_image], THR, NMS, fmt="rgb_f32", mean=100.0, std=50.0)[1]
        assert np.abs(f32b - blob(u8, 100.0, 50.0)).max() <= 1e-6
        ref = eng.detect_batch([golden_image], THR, NMS)[0]
        for size, tmpl in (((128, 128), ARCFACE_112 * np.float32(128 / 112)), ((96, 112), ARCFACE_112 - np.float32([8, 0])),
                           ((101, 77), ARCFACE_112 * np.float32(0.7))):
            faces, crops, mats = eng.detect_align([golden_image], THR, NMS, crop=size, template=tmpl, want_mats=True)
            assert crops[0].shape[1:] == (size[1], size[0], 3)
            _check_image(golden_image, faces[0], crops[0], mats[0], ref, size=size, template=tmpl)
            f32s, = eng.detect_align([golden_image], THR, NMS, crop=size, template=tmpl, fmt="rgb_f32")[1]
            assert np.abs(f32s - blob(crops[0])).max() <= 1e-6
    finally:
        eng.close()


def test_face_limit_leaves_other_slots_untouched(golden_image):
    """max_faces = 2: the two best faces' crops only; canary bytes after them and in the slots of a face-less image stay."""
    from retinaface_b200 import capi
    eng = _engine()
    try:
        imgs = [golden_image, np.zeros((300, 500, 3), np.uint8), letterbox_bgr_u8(golden_image, 448, 448)]
        n, A, cb = len(imgs), 2, 112 * 112 * 3
        faces, crops = eng.detect_align(imgs, THR, NMS)
        p = capi.align_params(max_faces=A)
        buf = np.full(n * A * cb + 4096, 0xA5, np.uint8)
        out_faces = np.empty((n, eng.max_faces, 15), np.float32)
        counts = np.zeros(n, np.int32)
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in imgs])
        ws, hs = (C.c_int * n)(*[im.shape[1] for im in imgs]), (C.c_int * n)(*[im.shape[0] for im in imgs])
        eng._check(eng.lib.rf_detect_align_batch(eng.h, ptrs, ws, hs, None, n, THR, NMS, C.byref(p), out_faces.ctypes.data,
                                                 counts.ctypes.data, buf.ctypes.data, None))
        assert counts[0] >= 5 and counts[1] == 0 and counts[2] >= 2
        slots = buf[:n * A * cb].reshape(n, A, 112, 112, 3)
        assert np.array_equal(slots[0], crops[0][:2]) and np.array_equal(slots[2], crops[2][:2])
        assert (slots[1] == 0xA5).all() and (buf[n * A * cb:] == 0xA5).all()
        f2, c2 = eng.detect_align(imgs, THR, NMS, max_faces=A)
        assert [len(c) for c in c2] == [2, 0, 2] and all(np.array_equal(a, b) for a, b in zip(f2, faces))
    finally:
        eng.close()


def test_device_variant_four_calls_over_two_contexts(golden_image):
    import torch
    eng = _engine(streams=2, max_batch=4)
    try:
        net = letterbox_bgr_u8(golden_image, 448, 448)
        batches = [np.stack([np.roll(net, 24 * (4 * b + i), axis=1) for i in range(4)]) for b in range(4)]
        dev = [torch.from_numpy(b).cuda() for b in batches]
        torch.cuda.synchronize()
        A = eng.max_faces
        outs = [torch.full((4, A, 3, 112, 112), 7.0, dtype=torch.float16, device="cuda") for _ in range(4)]
        mats = [torch.zeros((4, A, 2, 3), dtype=torch.float64, device="cuda") for _ in range(4)]
        cnt = []
        for b in range(4):
            _, cptr = eng.detect_align_device(4, THR, NMS, outs[b].data_ptr(), fmt="rgb_f16", dev_mats_ptr=mats[b].data_ptr(), dev_ptr=dev[b].data_ptr())
            cnt.append(cptr)
        eng.synchronize()
        got = [o.cpu().numpy() for o in outs]
        got_m = [m.cpu().numpy() for m in mats]
        for b in range(4):
            faces, crops, want_m = eng.detect_align(list(batches[b]), THR, NMS, fmt="rgb_f16", want_mats=True)
            for i in range(4):
                k = len(crops[i])
                assert k > 0 and np.array_equal(got[b][i, :k], crops[i]) and np.array_equal(got_m[b][i, :k], want_m[i])
                assert (got[b][i, k:] == 7.0).all()
    finally:
        eng.close()


def test_align_changes_nothing_for_detect_and_rejects_bad_params(golden_image):
    import torch
    from retinaface_b200 import RfError, capi
    eng = _engine()
    try:
        imgs = [golden_image, letterbox_bgr_u8(golden_image, 448, 448)]
        launches = eng.launches_per_batch(2)
        before = eng.detect_batch(imgs, THR, NMS, want_index=True)
        eng.detect_align(imgs, THR, NMS, fmt="rgb_f32", want_mats=True)
        scratch = torch.empty((eng.max_faces, 112, 112, 3), dtype=torch.uint8, device="cuda")
        eng.detect_align_device(1, THR, NMS, scratch.data_ptr())
        eng.synchronize()
        after = eng.detect_batch(imgs, THR, NMS, want_index=True)
        for a, b in zip(before[0] + before[1], after[0] + after[1]):
            assert np.array_equal(a, b)
        assert eng.launches_per_batch(2) == launches
        for kw in (dict(crop=(4, 112)), dict(crop=(112, 513)), dict(max_faces=eng.max_faces + 1), dict(mean=1.0, std=0.0)):
            with pytest.raises(RfError) as e:
                eng.detect_align(imgs, THR, NMS, **kw)
            assert e.value.status == -1, kw
        p = capi.align_params()
        p.format = 7
        with pytest.raises(RfError) as e:
            eng._check(eng.lib.rf_detect_align_batch_device(eng.h, eng.device_input_ptr(), 1, THR, NMS, C.byref(p), eng.device_input_ptr(), None,
                                                            None, None))
        assert e.value.status == -1
    finally:
        eng.close()
    # more originals than raw buffers: refused before anything runs
    big = _engine(max_batch=6, max_image=(13000, 13000))     # 4 raw buffers of 13000 x 13000 x 3
    try:
        small = [np.ascontiguousarray(golden_image[:300 + 10 * i, :400]) for i in range(5)]
        with pytest.raises(RfError) as e:
            big.detect_align(small, THR, NMS)
        assert e.value.status == -6 and "split the batch" in str(e.value)
        assert len(big.detect_align(small[:4], THR, NMS)[1]) == 4
    finally:
        big.close()


def test_cpp_class_detect_and_align(golden_image, tmp_path):
    """RetinaFace::detectAndAlign / lastCrops through the main.cpp-style driver == the Python mirror."""
    from retinaface_b200 import RetinaFace
    from retinaface_b200.build import build_host
    exe = build_host()
    raw = tmp_path / "img.bgr"
    raw.write_bytes(np.ascontiguousarray(golden_image).tobytes())
    out = tmp_path / "crops.bgr"
    r = subprocess.run([exe, os.path.join(GOLDEN, "weights"), "--image", str(raw), "1280", "886", "--net", "448", "448", "--iters", "1",
                        "--align", str(out)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet-deconv-0517.caffemodel")
    per = rf.detectAndAlign([golden_image], 0.9)[0]
    assert f"aligned {len(per)} crops" in r.stdout and len(per) == 5
    got = np.frombuffer(out.read_bytes(), np.uint8).reshape(len(per), 112, 112, 3)
    for (face, crop), c in zip(per, got):
        assert np.array_equal(crop, c)
    lines = [ln for ln in r.stdout.splitlines() if "image-pixel landmarks" in ln]
    for (face, _), ln in zip(per, lines):
        vals = [float(v) for v in ln.split()[2:]]
        assert np.allclose(vals, [face.pts_x[0], face.pts_y[0], face.pts_x[4], face.pts_y[4]], atol=1e-3)
