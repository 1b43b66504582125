"""GPU (-m gpu): the image-source layer every detect entry point goes through -- batches that cross the 64-item chunks of the
letter-box and crop tables, the row-stride rule of every BGR entry point, and checks that run before anything is staged."""
import ctypes as C

import cv2
import numpy as np
import pytest

from conftest import caffemodel
from oracle.inputs import letterbox_bgr_u8

pytestmark = pytest.mark.gpu

THR, NMS, A = 0.5, 0.4, 4


def _engine(**kw):
    from retinaface_b200 import RF_PREC_FP16, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (1024, 1536))
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP16, **kw)


def _host_batch(golden_image, n=70):
    """n host images, all different, of every kind a batch mixes: network-sized (the direct copy) at four places, and other sizes
    with packed or strided rows, in pageable or pinned memory -- more than 64 of those, so their letter-box items fill one 64-item
    launch and spill into a second."""
    import torch
    net = letterbox_bgr_u8(golden_image, 448, 448)
    imgs = []
    for i in range(n):
        if i in (5, 30, 47, 66):
            im = np.roll(net, 9 * i, axis=1)
            imgs.append(torch.from_numpy(im).pin_memory().numpy() if i % 2 else im)
            continue
        src = np.roll(golden_image, 11 * i, axis=1)
        kind = i % 4
        if kind == 1:
            src = cv2.resize(src, (400 + 3 * i, 280 + 2 * i), interpolation=cv2.INTER_AREA)
        if kind == 2:        # strided rows: a view into a wider buffer
            hgt, w = src.shape[:2]
            big = np.zeros((hgt + 9, w + 13, 3), np.uint8)
            big[4:4 + hgt, 6:6 + w] = src
            src = big[4:4 + hgt, 6:6 + w]
        if kind == 3:
            src = torch.from_numpy(np.ascontiguousarray(src)).pin_memory().numpy()
        imgs.append(src)
    assert sum(im.shape[:2] != (448, 448) for im in imgs) == n - 4 > 64
    return imgs


def test_align_batches_across_table_chunks_equal_single_calls(golden_image):
    """66 of 70 host images are letter-boxed, which crosses the 64-item chunk of the letter-box launch, and all 70 are cropped, which
    crosses the 64-image chunk of the crop table: faces, crops and matrices equal n = 1 calls."""
    eng = _engine(max_batch=72)
    try:
        imgs = _host_batch(golden_image)
        faces, crops, mats = eng.detect_align(imgs, THR, NMS, max_faces=A, want_mats=True)
        assert sum(len(c) > 0 for c in crops) > 64
        for i, im in enumerate(imgs):
            f1, c1, m1 = eng.detect_align([im], THR, NMS, max_faces=A, want_mats=True)
            assert np.array_equal(faces[i], f1[0]) and np.array_equal(crops[i], c1[0]) and np.array_equal(mats[i], m1[0]), i
    finally:
        eng.close()


def test_oriented_batches_across_table_chunks_equal_single_calls(golden_image):
    """The same 70 images in orientations 1..8: both letter-box kernels (reflections, transpositions) split across the 64-item chunks,
    and the oriented crop table crosses 64 images; faces, anchor indices, crops and matrices equal n = 1 calls."""
    eng = _engine(max_batch=72)
    try:
        imgs = _host_batch(golden_image)
        orient = [i % 8 + 1 for i in range(len(imgs))]
        faces, crops, mats, idx = eng.detect_oriented(imgs, orient, THR, NMS, align=dict(max_faces=A, want_mats=True), want_index=True)
        # the network misses most faces turned 90 degrees or more: the upright and reflected images carry the crops, in both chunks
        assert sum(len(c) > 0 for c in crops[:64]) >= 16 and sum(len(c) > 0 for c in crops[64:]) >= 2
        for i, im in enumerate(imgs):
            f1, c1, m1, x1 = eng.detect_oriented([im], [orient[i]], THR, NMS, align=dict(max_faces=A, want_mats=True), want_index=True)
            assert np.array_equal(faces[i], f1[0]) and np.array_equal(idx[i], x1[0]), i
            assert np.array_equal(crops[i], c1[0]) and np.array_equal(mats[i], m1[0]), i
    finally:
        eng.close()


def test_device_align_batches_across_table_chunks_equal_single_calls(golden_image):
    import torch
    eng = _engine(max_batch=72)
    try:
        net = letterbox_bgr_u8(golden_image, 448, 448)
        n, cb = 70, 112 * 112 * 3
        batch = torch.from_numpy(np.stack([np.roll(net, 8 * i, axis=1) for i in range(n)])).cuda()
        crops = torch.full((n, A, cb), 7, dtype=torch.uint8, device="cuda")
        mats = torch.zeros((n, A, 6), dtype=torch.float64, device="cuda")
        eng.detect_align_device(n, THR, NMS, crops.data_ptr(), max_faces=A, dev_mats_ptr=mats.data_ptr(), dev_ptr=batch.data_ptr())
        eng.synchronize()
        one_c = torch.full((n, A, cb), 7, dtype=torch.uint8, device="cuda")
        one_m = torch.zeros((n, A, 6), dtype=torch.float64, device="cuda")
        for i in range(n):
            eng.detect_align_device(1, THR, NMS, one_c[i].data_ptr(), max_faces=A, dev_mats_ptr=one_m[i].data_ptr(), dev_ptr=batch[i].data_ptr())
            eng.synchronize()
        assert (crops != 7).any(dim=2).any(dim=1).sum().item() == n        # every image has crops
        assert torch.equal(crops, one_c) and torch.equal(mats, one_m)
    finally:
        eng.close()


def _bgr_calls(eng, img, stride):
    """Every BGR entry point on one image with row stride `stride`: name -> status."""
    from retinaface_b200 import capi
    lib, h, mf = eng.lib, eng.h, eng.max_faces
    w, hgt = img.shape[1], img.shape[0]
    ptrs, ws, hs, rs = (C.c_void_p * 1)(img.ctypes.data), (C.c_int * 1)(w), (C.c_int * 1)(hgt), (C.c_int * 1)(stride)
    o = (C.c_int * 1)(6)
    p = capi.align_params(max_faces=A)
    faces = np.empty((mf, 15), np.float32)
    counts, idx = np.zeros(1, np.int32), np.empty(mf, np.int32)
    crops, mats = np.empty(A * 112 * 112 * 3, np.uint8), np.empty(A * 6)
    out = np.empty((448, 448, 3), np.uint8)
    cnt = C.c_int(0)
    t = capi.tiling()
    views = (capi._View * 1)(capi._View(1.0, 0))
    oviews = (capi._OrientedView * 1)(capi._OrientedView(1.0, 6))
    return {
        "rf_detect_batch": lib.rf_detect_batch(h, ptrs, ws, hs, rs, 1, THR, NMS, faces.ctypes.data, counts.ctypes.data, None),
        "rf_detect_align_batch": lib.rf_detect_align_batch(h, ptrs, ws, hs, rs, 1, THR, NMS, C.byref(p), faces.ctypes.data, counts.ctypes.data,
                                                           crops.ctypes.data, mats.ctypes.data),
        "rf_detect_oriented_batch": lib.rf_detect_oriented_batch(h, ptrs, ws, hs, rs, o, 1, THR, NMS, C.byref(p), faces.ctypes.data,
                                                                 counts.ctypes.data, idx.ctypes.data, crops.ctypes.data, None),
        "rf_detect_tiled": lib.rf_detect_tiled(h, ptrs, ws, hs, rs, 1, C.byref(t), THR, NMS, faces.ctypes.data, counts.ctypes.data, None),
        "rf_detect_tiled_align": lib.rf_detect_tiled_align(h, ptrs, ws, hs, rs, 1, C.byref(t), THR, NMS, C.byref(p), faces.ctypes.data,
                                                           counts.ctypes.data, None, crops.ctypes.data, None),
        "rf_detect_views": lib.rf_detect_views(h, img.ctypes.data, w, hgt, stride, views, 1, THR, NMS, faces.ctypes.data, C.byref(cnt), None,
                                               None),
        "rf_detect_views_oriented": lib.rf_detect_views_oriented(h, img.ctypes.data, w, hgt, stride, oviews, 1, THR, NMS, faces.ctypes.data,
                                                                 C.byref(cnt), None, None),
        "rf_preprocess": lib.rf_preprocess(h, img.ctypes.data, w, hgt, stride, out.ctypes.data),
        "rf_preprocess_oriented": lib.rf_preprocess_oriented(h, img.ctypes.data, w, hgt, stride, 6, out.ctypes.data),
        "rf_preprocess_tile": lib.rf_preprocess_tile(h, img.ctypes.data, w, hgt, stride, C.byref(t), 0, out.ctypes.data),
    }


def test_row_stride_below_three_widths_is_refused_by_every_bgr_entry_point(golden_image):
    import torch
    eng = _engine()
    try:
        before = eng.detect_batch([golden_image], THR, NMS)[0]
        img = np.ascontiguousarray(golden_image[:300, :400])
        ok = _bgr_calls(eng, img, 0)
        assert all(v == 0 for v in ok.values()), ok
        bad = _bgr_calls(eng, img, 3 * 400 - 1)
        assert all(v == -1 for v in bad.values()), bad
        dev = torch.from_numpy(img).cuda()
        from retinaface_b200 import capi
        t = capi.tiling()
        d, c = C.c_void_p(), C.c_void_p()
        for stride, want in ((0, 0), (3 * 400 - 3, -1)):
            rc = eng.lib.rf_detect_tiled_device(eng.h, (C.c_void_p * 1)(dev.data_ptr()), (C.c_int * 1)(400), (C.c_int * 1)(300),
                                                (C.c_int * 1)(stride), 1, C.byref(t), THR, NMS, None, None, None, C.byref(d), C.byref(c))
            assert rc == want, (stride, rc)
        eng.synchronize()
        after = eng.detect_batch([golden_image], THR, NMS)[0]
        assert len(before) >= 5 and np.array_equal(before, after)
    finally:
        eng.close()


def test_bad_last_image_is_refused_before_anything_is_staged(golden_image):
    """rf_detect_batch checks every image before the first copy: a batch whose last image is empty or too large returns its status
    without touching the pinned staging mirror (which a pageable network-sized image ahead of it would be copied into), and the next
    call detects what a fresh handle detects."""
    from retinaface_b200 import RfError
    net = letterbox_bgr_u8(golden_image, 448, 448)
    imgs = [golden_image, net, np.ascontiguousarray(golden_image[:500, :700]), np.roll(net, 40, axis=1)]
    fresh = _engine()
    try:
        want = fresh.detect_batch(imgs, THR, NMS, want_index=True)
    finally:
        fresh.close()
    eng = _engine()
    try:
        mirror = eng.pinned_input()
        for last, status in ((np.zeros((0, 10, 3), np.uint8), -1), (np.zeros((1100, 1600, 3), np.uint8), -6)):
            mirror[:] = 0xA5
            with pytest.raises(RfError) as e:
                eng.detect_batch(imgs[:3] + [last], THR, NMS)
            assert e.value.status == status
            assert (mirror == 0xA5).all()
            got = eng.detect_batch(imgs, THR, NMS, want_index=True)
            for a, b in zip(want[0] + want[1], got[0] + got[1]):
                assert np.array_equal(a, b)
    finally:
        eng.close()
