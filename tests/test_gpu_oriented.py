"""GPU (-m gpu): f9 rotated and mirrored images -- every oriented entry point against its unoriented twin run on the rotated copy
(orient() of oracle/orient.py), bit for bit: letter-box bytes, faces, anchor indices, matrices and crops; the device YUV path on
oriented surfaces; oriented views against host map-back; the any-orientation sweep finding the upright photo's faces on a photo
stored sideways; invalid orientations refused with nothing written; and that nothing else changes.  Everything goes through the C ABI."""
import ctypes as C
import math
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.inputs import letterbox_bgr_u8
from oracle.yuv import bgr_to_frame, frame_to_bgr
from oracle.orient import orient, orient_planes
from test_oriented_cpu import stored_faces

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
ALL = list(range(1, 9))


def _engine(prec="fp16", net=(448, 448), **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (2160, 3840))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), net[1], net[0], precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), net[1], net[0], precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _sources(golden_image):
    rng = np.random.default_rng(9)
    g = golden_image
    return {"golden": g, "517x333": cv2.resize(g, (517, 333)), "519x335": cv2.resize(g, (519, 335)),
            "448x448": np.ascontiguousarray(g[:448, 300:748]), "1920x1080": cv2.resize(g, (1920, 1080)),
            "strided": g[100:700, 200:1100], "noise": rng.integers(0, 256, (301, 203, 3), dtype=np.uint8)}


@pytest.mark.parametrize("o", ALL)
def test_letterbox_bytes_equal_the_rotated_copy(eng, golden_image, o):
    for name, img in _sources(golden_image).items():
        got = eng.preprocess_oriented(img, o)
        assert np.array_equal(got, letterbox_bgr_u8(orient(img, o), 448, 448)), (name, o)


def test_letterbox_from_pinned_source(eng, golden_image):
    import torch
    pinned = torch.from_numpy(golden_image.copy()).pin_memory().numpy()
    for o in ALL:
        assert np.array_equal(eng.preprocess_oriented(pinned, o), letterbox_bgr_u8(orient(golden_image, o), 448, 448)), o


def test_npp_letterbox_equals_the_rotated_copy(golden_image):
    from retinaface_b200.capi import RF_FLAG_NPP_RESIZE
    e = _engine(flags=RF_FLAG_NPP_RESIZE)
    try:
        for img in (golden_image, cv2.resize(golden_image, (519, 335))):
            for o in ALL:
                assert np.array_equal(e.preprocess_oriented(img, o), e.preprocess(orient(img, o))), o
    finally:
        e.close()


@pytest.mark.parametrize("layout,matrix", [("nv12", "bt601"), ("i420", "bt709")])
def test_yuv_letterbox_equals_the_rotated_frame(eng, golden_image, layout, matrix):
    frame = bgr_to_frame(cv2.resize(golden_image, (1282, 722)), layout)
    for o in ALL:
        got = eng.preprocess_yuv_oriented(frame, o, layout=layout, matrix=matrix)
        assert np.array_equal(got, eng.preprocess_yuv(orient_planes(frame, layout, o), layout=layout, matrix=matrix)), o
        if matrix == "bt601":
            assert np.array_equal(got, letterbox_bgr_u8(orient(frame_to_bgr(frame, layout), o), 448, 448)), o


def test_yuv_letterbox_of_a_pitched_surface(eng, golden_image):
    frame = bgr_to_frame(cv2.resize(golden_image, (1282, 722)), "nv12")
    pitched = np.zeros((frame.shape[0], 1536), np.uint8)          # NVDEC-like: rows padded to a 512-byte pitch
    pitched[:, :1282] = frame
    y, uv = pitched[:722, :1282], pitched[722:, :1282]
    for o in ALL:
        assert np.array_equal(eng.preprocess_yuv_oriented((y, uv), o), letterbox_bgr_u8(orient(frame_to_bgr(frame, "nv12"), o), 448, 448)), o


def _mixed(golden_image, n):
    imgs = [golden_image, cv2.resize(golden_image, (640, 443)), np.ascontiguousarray(golden_image[:448, 400:848]),
            golden_image[50:850, 100:1200], cv2.resize(golden_image, (1920, 1329))]
    return [imgs[i % len(imgs)] for i in range(n)], [ALL[(3 * i + 5) % 8] for i in range(n)]


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_detect_oriented_equals_detect_align_on_the_rotated_copy(golden_image, prec, n):
    e = _engine(prec)
    try:
        imgs, os_ = _mixed(golden_image, n)
        if n == 1:
            os_ = [6]
        shown = [orient(im, o) for im, o in zip(imgs, os_)]
        al = dict(want_mats=True)
        f, c, m, idx = e.detect_oriented(imgs, os_, THR, NMS, align=al, want_index=True)
        rf, rc_, rm = e.detect_align(shown, THR, NMS, want_mats=True)
        _, ridx = e.detect_batch(shown, THR, NMS, want_index=True)
        for i in range(n):
            assert np.array_equal(f[i], rf[i]) and np.array_equal(idx[i], ridx[i]), (prec, i)
            assert np.array_equal(m[i], rm[i]) and np.array_equal(c[i], rc_[i]), (prec, i)
            for j in range(len(c[i])):
                warp = cv2.warpAffine(shown[i], m[i][j], (112, 112), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
                assert np.array_equal(c[i][j], warp), (prec, i, j)
        # without crops: the same faces
        f2 = e.detect_oriented(imgs, os_, THR, NMS)
        assert all(np.array_equal(a, b) for a, b in zip(f, f2))
        # float crops: equal to the twin's
        for fmt in ("rgb_f32", "rgb_f16"):
            _, cf = e.detect_oriented(imgs, os_, THR, NMS, align=dict(fmt=fmt))
            _, rcf = e.detect_align(shown, THR, NMS, fmt=fmt)
            assert all(np.array_equal(a, b) for a, b in zip(cf, rcf)), fmt
    finally:
        e.close()


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_device_yuv_oriented_equals_the_rotated_surfaces(eng, golden_image):
    import torch
    base = [bgr_to_frame(cv2.resize(golden_image, s), "nv12") for s in ((1920, 1080), (1282, 722), (640, 444))]
    frames = [base[i % 3] for i in range(8)]
    os_ = [ALL[(5 * i + 2) % 8] for i in range(8)]
    dev = [_cuda(f) for f in frames]
    rot = [_cuda(orient_planes(f, "nv12", o)) for f, o in zip(frames, os_)]
    sums = [int(d.sum()) for d in dev]
    A = eng.max_faces
    crops = torch.zeros((8, A, 112, 112, 3), dtype=torch.uint8, device="cuda")
    crops_ref = torch.zeros_like(crops)
    mats = torch.zeros((8, A, 6), dtype=torch.float64, device="cuda")
    mats_ref = torch.zeros_like(mats)
    d, c, sc = eng.detect_yuv_oriented_device(dev, os_, THR, NMS, align={}, dev_crops_ptr=crops.data_ptr(), dev_mats_ptr=mats.data_ptr())
    eng.synchronize()
    got, got_idx = eng.read_dets(d, c, 8)
    d2, c2, sc2 = eng.detect_yuv_device(rot, THR, NMS, align={}, dev_crops_ptr=crops_ref.data_ptr(), dev_mats_ptr=mats_ref.data_ptr())
    eng.synchronize()
    ref, ref_idx = eng.read_dets(d2, c2, 8)
    assert np.array_equal(sc, sc2)
    for i in range(8):
        assert np.array_equal(got[i], ref[i]) and np.array_equal(got_idx[i], ref_idx[i]), i
        k = len(got[i])
        assert torch.equal(crops[i, :k], crops_ref[i, :k]) and torch.equal(mats[i, :k], mats_ref[i, :k]), i
    assert [int(x.sum()) for x in dev] == sums                          # the surfaces are read, never written
    # the host path's crops of the same displayed frames
    hf, hc = eng.detect_oriented([frame_to_bgr(f, "nv12") for f in frames], os_, THR, NMS, align={})
    for i in range(8):
        assert np.array_equal(crops[i, :len(hc[i])].cpu().numpy(), hc[i]), i


def test_views_oriented(eng, golden_image):
    img = cv2.resize(golden_image, (900, 620))
    h, w = img.shape[:2]
    # orientations 1 / 2 are rf_detect_views' flip 0 / 1, bit for bit
    for o, flip in ((1, 0), (2, 1)):
        a = eng.detect_views_oriented(img, [(1.0, o), (0.6, o)], THR, NMS)
        b = eng.detect_views(img, [(1.0, flip), (0.6, flip)], THR, NMS)
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), o
    # one view: the twin's faces on the rotated copy, mapped back into stored pixels on the host
    for o in ALL:
        for shrink in (1.0, 0.7):
            f, view_of, sc = eng.detect_views_oriented(img, [(shrink, o)], THR, NMS)
            rf, _, rsc = eng.detect_views(orient(img, o), [(shrink, 0)], THR, NMS)
            assert np.array_equal(sc, rsc) and np.array_equal(view_of, np.zeros(len(f), np.int32))
            assert np.array_equal(f, stored_faces(o, rf, w, h)), (o, shrink)


def _iou(a, b):
    ix = max(0.0, min(a[2], b[2]) - max(a[0], b[0]))
    iy = max(0.0, min(a[3], b[3]) - max(a[1], b[1]))
    inter = ix * iy
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)


def _angle(M):
    return math.degrees(math.atan2(M[1, 0], M[0, 0]))


def test_any_orientation_sweep_finds_the_upright_faces(eng, golden_image):
    from oracle.align import ARCFACE_112, umeyama
    upright = golden_image
    stored = np.ascontiguousarray(cv2.rotate(upright, cv2.ROTATE_90_CLOCKWISE))     # the photo stored lying on its side
    H = upright.shape[0]
    ref = eng.detect_align([upright], THR, NMS)[0][0]
    plain = eng.detect_align([stored], THR, NMS)[0][0]
    print(f"\nrf_detect_batch on the sideways photo: {len(plain)} faces (upright: {len(ref)})")
    faces, view_of, _ = eng.detect_views_oriented(stored, [(1.0, o) for o in (1, 6, 3, 8)], THR, NMS)
    assert len(ref) > 0
    for r in ref:
        # upright (x, y) -> stored (H-1-y, x): the clockwise turn
        box = [H - 1 - r[4], r[1], H - 1 - r[2], r[3]]
        best = max(faces, key=lambda f: _iou(box, f[1:5]))
        assert _iou(box, best[1:5]) > 0.6
        lx, ly = H - 1 - r[10:15], r[5:10]
        assert np.allclose(best[5:10], lx, atol=0.25 * (box[2] - box[0])) and np.allclose(best[10:15], ly, atol=0.25 * (box[3] - box[1]))
        # the crops fitted on the stored-frame landmarks come out upright: M's angle = the upright M's composed with the turn
        M = umeyama(np.stack([best[5:10], best[10:15]], 1).astype(np.float64), ARCFACE_112)[:2]
        Mu = umeyama(np.stack([r[5:10], r[10:15]], 1).astype(np.float64), ARCFACE_112)[:2]
        d = (_angle(M) - (_angle(Mu) - 90.0) + 180.0) % 360.0 - 180.0
        assert abs(d) < 10.0, (d, _angle(M), _angle(Mu))


def test_invalid_orientations_change_nothing(eng, golden_image):
    from retinaface_b200 import capi
    lib, h = eng.lib, eng.h
    img = np.ascontiguousarray(golden_image)
    out = np.full((448, 448, 3), 7, np.uint8)
    for bad in (0, 9, -1):
        assert lib.rf_preprocess_oriented(h, img.ctypes.data, img.shape[1], img.shape[0], 0, bad, out.ctypes.data) == -1
        assert (out == 7).all()
        ptrs = (C.c_void_p * 1)(img.ctypes.data)
        ws, hs, os_ = (C.c_int * 1)(img.shape[1]), (C.c_int * 1)(img.shape[0]), (C.c_int * 1)(bad)
        faces = np.full((1, eng.max_faces, 15), 7, np.float32)
        counts = np.full(1, 7, np.int32)
        assert lib.rf_detect_oriented_batch(h, ptrs, ws, hs, None, os_, 1, THR, NMS, None, faces.ctypes.data, counts.ctypes.data, None, None, None) == -1
        assert (faces == 7).all() and (counts == 7).all()
        v = (capi._OrientedView * 1)(capi._OrientedView(1.0, bad))
        cnt = C.c_int(7)
        assert lib.rf_detect_views_oriented(h, img.ctypes.data, img.shape[1], img.shape[0], 0, v, 1, THR, NMS, faces.ctypes.data, C.byref(cnt),
                                            None, None) == -1
        assert cnt.value == 7 and (faces == 7).all()
        fr = bgr_to_frame(cv2.resize(golden_image, (640, 444)), "nv12")
        arr = eng._frames([fr], "nv12", False)
        assert lib.rf_preprocess_yuv_oriented(h, arr, 0, bad, out.ctypes.data) == -1 and (out == 7).all()
        dframe = _cuda(fr)
        darr = eng._frames([dframe], "nv12", True)
        d, c = C.c_void_p(7), C.c_void_p(7)
        scales = np.full(1, 7, np.float32)
        assert lib.rf_detect_yuv_oriented_device(h, darr, os_, 1, 0, THR, NMS, None, None, None, C.byref(d), C.byref(c), scales.ctypes.data) == -1
        assert d.value == 7 and c.value == 7 and (scales == 7).all()
    # NULL orientations
    assert lib.rf_detect_oriented_batch(h, (C.c_void_p * 1)(img.ctypes.data), (C.c_int * 1)(img.shape[1]), (C.c_int * 1)(img.shape[0]), None,
                                        None, 1, THR, NMS, None, faces.ctypes.data, counts.ctypes.data, None, None, None) == -1
    with pytest.raises(ValueError):
        eng.detect_oriented([img], [1, 2], THR, NMS)


def test_nothing_else_changes(golden_image):
    import torch
    e = _engine()
    try:
        imgs = [golden_image, cv2.resize(golden_image, (640, 443))]
        frame = bgr_to_frame(cv2.resize(golden_image, (1282, 722)), "nv12")
        dframe = _cuda(frame)
        launches = e.launches_per_batch(2)

        def plain():
            f, idx = e.detect_batch(imgs, THR, NMS, want_index=True)
            d, c, sc = e.detect_yuv_device([dframe], THR, NMS)
            e.synchronize()
            return (f, idx, *e.read_dets(d, c, 1), sc)
        before = plain()
        e.detect_oriented(imgs, [6, 7], THR, NMS, align={})
        e.detect_yuv_oriented_device([dframe], [8], THR, NMS)
        e.detect_views_oriented(imgs[0], [(1.0, o) for o in (1, 6, 3, 8)], THR, NMS)
        e.synchronize()
        after = plain()
        for a, b in zip(before, after):
            if isinstance(a, list):
                assert all(np.array_equal(x, y) for x, y in zip(a, b))
            else:
                assert np.array_equal(a, b)
        assert e.launches_per_batch(2) == launches
        assert torch.equal(dframe.cpu(), torch.from_numpy(frame))
    finally:
        e.close()
