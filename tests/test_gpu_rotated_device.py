"""GPU (-m gpu): f24 rotated views of device frames through the C ABI, against the host call rf_detect_views_rotated as the oracle, bit
for bit: rf_preprocess_yuv_rotated against the YUV view oracle, device BGR and YUV records, view scales and M, crops, a rebuild from the
library's parts, calls in flight over the rotated ring beside the tiled one, a tilted video through the tracker and the redaction, and the
refusals."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle import rotate
from oracle.align import ARCFACE_112, blob, similarity_closed, warp_affine_fixed
from oracle.yuv import LAYOUTS, bgr_to_frame, frame_to_bgr
from test_gpu_redact_blur import _regions, _style
from test_gpu_rotated import ANGLES, QUARTERS, SWEEP, _engine, _expected, _tilted
from test_gpu_tiled_device import _cuda, _nvdec_like, _to_i420
from test_gpu_track import _same

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
VIEW_SETS = ([(a, 1.0) for a in (0, 30, 45, 135, 270)], [(a, 1.0) for a in SWEEP], [(a, 0.75) for a in SWEEP[:7]] + [(315.0, 1.0)])


def _planes(frame, layout, pad):
    """The host frame as planes whose rows are `pad` bytes longer than the plane (a padded pitch)."""
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]

    def padded(p):
        out = np.full((p.shape[0], p.shape[1] + pad), 0xEE, np.uint8)
        out[:, :p.shape[1]] = p
        return out[:, :p.shape[1]]
    if layout in ("nv12", "nv21"):
        return (padded(frame[:h]), padded(frame[h:]))
    flat, q = frame[h:].reshape(-1), (h // 2) * (w // 2)
    a, b = flat[:q].reshape(h // 2, w // 2), flat[q:].reshape(h // 2, w // 2)
    return (padded(frame[:h]), padded(a), padded(b)) if layout == "i420" else (padded(frame[:h]), padded(b), padded(a))


@pytest.mark.parametrize("net", [(448, 448), (1280, 896)])
def test_preprocess_yuv_bytes_and_matrix(golden_image, net):
    """rf_preprocess_yuv_rotated: bytes = warp_view(frame_to_bgr(frame)) and M = rotate.geometry at f23's angles, shrink 1 and 0.6, all
    four layouts, both matrices, packed and padded pitches; quarter turns = rf_preprocess_yuv_oriented with zero M."""
    e = _engine(net=net)
    try:
        for bgr in (golden_image, cv2.resize(golden_image, (640, 442))):
            h, w = bgr.shape[:2]
            for layout in LAYOUTS:
                frame = bgr_to_frame(bgr, layout)
                for matrix in ("bt601", "bt709"):
                    conv = frame_to_bgr(frame, layout, matrix)
                    for src in (frame, _planes(frame, layout, 64)):
                        for angle in ANGLES:
                            for shrink in (1.0, 0.6):
                                got, M = e.preprocess_yuv_rotated(src, angle, shrink, layout, matrix)
                                o, f, want_M = rotate.geometry(angle, w, h, *rotate.shrink_box(net[0], net[1], shrink))
                                assert o == 0 and M.tobytes() == want_M.tobytes(), (layout, matrix, angle, shrink)
                                assert np.array_equal(got, rotate.warp_view(conv, want_M, net[0], net[1])), (layout, matrix, angle, shrink)
                        for angle, o in QUARTERS:
                            got, M = e.preprocess_yuv_rotated(src, angle, 1.0, layout, matrix)
                            assert np.array_equal(got, e.preprocess_yuv_oriented(src, o, layout, matrix)) and not M.any(), (layout, angle)
    finally:
        e.close()


def _host(e, imgs, views, align=None):
    return [e.detect_views_rotated(im, views, THR, NMS, align=align) for im in imgs]


def _assert_records(e, d, c, host, scales, mats, what):
    faces, ids = e.read_dets(d, c, len(host))
    mf = e.max_faces
    for i, want in enumerate(host):
        assert np.array_equal(faces[i], want[0]) and np.array_equal(ids[i] // mf, want[1]), (what, i, len(faces[i]), len(want[0]))
        assert np.array_equal(scales[i], want[2]) and mats[i].tobytes() == want[3].tobytes(), (what, i)


def _bgr_frames(golden_image):
    """Eight frames of different sizes; the last one a row-strided view of a larger device tensor."""
    import torch
    tilted = _tilted(golden_image, 40.0)[0]
    imgs = [golden_image, tilted, cv2.resize(golden_image, (1100, 760)), cv2.resize(tilted, (900, 900)), golden_image[100:700, 200:1100].copy(),
            cv2.resize(golden_image, (1920, 1080)), np.ascontiguousarray(golden_image[:, ::-1]), golden_image]
    big = torch.full((886, 1300, 3), 0x5A, dtype=torch.uint8, device="cuda")
    big[:, :1280] = _cuda(golden_image)
    dev = [_cuda(im) for im in imgs[:-1]] + [big[:, :1280]]
    assert dev[-1].stride(0) == 3900
    return imgs, dev, big


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_bgr_device_records_equal_the_host_call(golden_image, prec):
    """n = 1, 3 and max_batch frames of different sizes and strides, three view sets: per frame, records, view of each face, view scales
    and M equal rf_detect_views_rotated on the host copy; the tilted frame also equals the rebuild from the library's parts."""
    import torch
    e = _engine(prec)
    try:
        imgs, dev, big = _bgr_frames(golden_image)
        torch.cuda.synchronize()
        for views in VIEW_SETS:
            host = _host(e, imgs, views)
            for n in (1, 3, 8):
                d, c, sc, mats = e.detect_views_rotated_device(dev[8 - n:], views, THR, NMS)
                _assert_records(e, d, c, host[8 - n:], sc, mats, (prec, len(views), n))
            assert sum(len(h[0]) for h in host) >= 20
        for views in VIEW_SETS[:2]:
            want_f, want_v = _expected(e, imgs[1], views)
            d, c, _, _ = e.detect_views_rotated_device([dev[1]], views, THR, NMS)
            faces, ids = e.read_dets(d, c, 1)
            assert np.array_equal(faces[0], want_f) and np.array_equal(ids[0] // e.max_faces, want_v), (prec, len(views))
        del big
    finally:
        e.close()


@pytest.mark.parametrize("prec", ["fp16", "int8"])
def test_a_chunk_of_more_than_sixteen_warp_views(golden_image, prec):
    """A max_batch 32 handle: 3 frames x 12 views make a first chunk of 32 network inputs, 24 of them warp views (two warp and two merge
    launches), and the records still equal the host call's."""
    import torch
    e = _engine(prec, max_batch=32)
    try:
        imgs, dev, big = _bgr_frames(golden_image)
        torch.cuda.synchronize()
        views = VIEW_SETS[1]
        host = _host(e, imgs, views)
        for sel in ((0, 1, 2), tuple(range(8))):
            d, c, sc, mats = e.detect_views_rotated_device([dev[i] for i in sel], views, THR, NMS)
            _assert_records(e, d, c, [host[i] for i in sel], sc, mats, (prec, sel))
        del big
    finally:
        e.close()


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_yuv_device_records_equal_the_host_call(golden_image, prec):
    """NV12 BT.601 (with an NVDEC-like surface, luma pitch 2048) and I420 BT.709 device frames: per frame, records, view of each face,
    scales and M equal rf_detect_views_rotated on cv2.cvtColor(frame) (the oracle's conversion for BT.709)."""
    import torch
    tilted = _tilted(golden_image, 45.0)[0]
    bgr = [golden_image, cv2.resize(tilted, (1000, 1000)), cv2.resize(golden_image, (1920, 1080)), cv2.resize(tilted, (638, 638))]
    e = _engine(prec)
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
            for views in VIEW_SETS[:2]:
                host = _host(e, [frame_to_bgr(f, layout, matrix) for f in frames], views)
                d, c, sc, mats = e.detect_yuv_views_rotated_device(dev, views, THR, NMS, layout, matrix)
                _assert_records(e, d, c, host, sc, mats, (prec, layout, len(views)))
                assert sum(len(h[0]) for h in host) >= 10
            del surf
    finally:
        e.close()


@pytest.mark.parametrize("fmt", ["bgr_u8", "rgb_f16"])
def test_crops_equal_the_host_call_and_the_align_oracle(golden_image, fmt):
    """u8 and F16 crops and matrices of both device calls equal the host call's and oracle/align.py's."""
    import torch
    e = _engine("fp16")
    try:
        tilted = _tilted(golden_image, 30.0)[0]
        bgr = [np.ascontiguousarray(tilted[:tilted.shape[0] // 2 * 2, :tilted.shape[1] // 2 * 2]), cv2.resize(golden_image, (1100, 760))]
        views = VIEW_SETS[1]
        A = e.max_faces
        shape = (112, 112, 3) if fmt == "bgr_u8" else (3, 112, 112)
        dt = torch.uint8 if fmt == "bgr_u8" else torch.float16
        for kind in ("bgr", "nv12"):
            srcs = bgr if kind == "bgr" else [frame_to_bgr(bgr_to_frame(b, "nv12"), "nv12") for b in bgr]
            dev = [_cuda(b) for b in bgr] if kind == "bgr" else [_cuda(bgr_to_frame(b, "nv12")) for b in bgr]
            crops = torch.full((2, A) + shape, 7, dtype=dt, device="cuda")
            mats = torch.full((2, A, 2, 3), 7.0, dtype=torch.float64, device="cuda")
            fn = e.detect_views_rotated_device if kind == "bgr" else e.detect_yuv_views_rotated_device
            d, c, _, _ = fn(dev, views, THR, NMS, align={"fmt": fmt}, dev_crops_ptr=crops.data_ptr(), dev_mats_ptr=mats.data_ptr())
            faces, _ = e.read_dets(d, c, 2)
            for i, img in enumerate(srcs):
                f, _, _, _, hc, hm = e.detect_views_rotated(img, views, THR, NMS, align={"fmt": fmt, "want_mats": True})
                k = len(f)
                assert k > 0 and np.array_equal(faces[i], f), (kind, i)
                assert np.array_equal(crops[i, :k].cpu().numpy(), hc) and mats[i, :k].cpu().numpy().tobytes() == hm.tobytes(), (kind, i)
                assert (crops[i, k:] == 7).all(), (kind, i)
                for j, r in enumerate(f):
                    M = similarity_closed(np.stack([r[5:10], r[10:15]], 1).astype(np.float64), ARCFACE_112.astype(np.float64))
                    assert hm[j].tobytes() == M.tobytes(), (kind, i, j)
                    u8 = warp_affine_fixed(img, M, (112, 112))
                    assert np.array_equal(hc[j], u8 if fmt == "bgr_u8" else blob(u8[None])[0].astype(np.float16)), (kind, i, j)
    finally:
        e.close()


@pytest.mark.parametrize("streams", [2, 3])
def test_calls_in_flight_and_the_separate_rings(golden_image, streams):
    """A tiled device call, then 2 streams + 1 rotated device calls (BGR and NV12 alternating, crops into a buffer per call) with an
    rf_detect_batch_device call between each two, no host synchronise: every call's crops equal the host call's, the records of the
    last `streams` rotated calls equal it, the tiled call's records are still its own, and the frames are unchanged."""
    import torch
    from oracle.inputs import letterbox_bgr_u8
    e = _engine("fp16", max_batch=4, streams=streams)
    try:
        calls = 2 * streams + 1
        views = [(a, 1.0) for a in (0, 45, 90, 200, 315)]
        net_in = _cuda(np.stack([letterbox_bgr_u8(golden_image, 448, 448)] * 2))
        tiled_img = cv2.resize(golden_image, (1920, 1080))
        want_tiled, tile_of = e.detect_tiled([tiled_img], THR, NMS)
        d_tiled = _cuda(tiled_img)
        host, dev, bufs, out = [], [], [], []
        for k in range(calls):
            imgs = [np.roll(_tilted(golden_image, 15.0 * (k % 4))[0], 16 * (2 * k + i), axis=1) for i in range(2)]
            imgs = [im[:im.shape[0] // 2 * 2, :im.shape[1] // 2 * 2] for im in imgs]
            kind = "bgr" if k % 2 == 0 else "nv12"
            srcs = [np.ascontiguousarray(im) for im in imgs] if kind == "bgr" else [bgr_to_frame(im, "nv12") for im in imgs]
            host.append([im if kind == "bgr" else frame_to_bgr(s, "nv12") for im, s in zip(imgs, srcs)])
            dev.append((kind, [_cuda(s) for s in srcs]))
            bufs.append(torch.full((2, e.max_faces, 3, 112, 112), 7.0, dtype=torch.float16, device="cuda"))
        torch.cuda.synchronize()
        sums = [[int(t.to(torch.int64).sum()) for t in d] for _, d in dev]
        td, tc = e.detect_tiled_device([d_tiled], THR, NMS)
        for k in range(calls):
            kind, d = dev[k]
            fn = e.detect_views_rotated_device if kind == "bgr" else e.detect_yuv_views_rotated_device
            out.append(fn(d, views, THR, NMS, align=dict(fmt="rgb_f16"), dev_crops_ptr=bufs[k].data_ptr()))
            e.detect_device(2, THR, NMS, net_in.data_ptr())
        e.synchronize()
        for k in range(calls):
            want = _host(e, host[k], views, align=dict(fmt="rgb_f16"))
            for i in range(2):
                kk = len(want[i][4])
                assert np.array_equal(bufs[k][i, :kk].cpu().numpy(), want[i][4]), (k, i)
                assert (bufs[k][i, kk:] == 7.0).all(), (k, i)
            assert sum(len(w[0]) for w in want) > 0, k
            if k >= calls - streams:
                _assert_records(e, out[k][0], out[k][1], want, out[k][2], out[k][3], k)
        faces, ids = e.read_dets(td, tc, 1)
        assert np.array_equal(faces[0], want_tiled[0]) and np.array_equal(ids[0] // e.max_faces, tile_of[0])
        assert [[int(t.to(torch.int64).sum()) for t in d] for _, d in dev] == sums
    finally:
        e.close()


def _tilted_video(golden_image, frames=12):
    """The golden photo tilted 45 degrees at 0.6x, drifting 9 px right and 5 px down a frame on a 1280 x 960 NV12 canvas."""
    t = cv2.resize(_tilted(golden_image, 45.0)[0], None, fx=0.6, fy=0.6, interpolation=cv2.INTER_AREA)
    out = []
    for k in range(frames):
        c = np.zeros((960, 1280, 3), np.uint8)
        x, y = 40 + 9 * k, 10 + 5 * k
        h, w = min(t.shape[0], 960 - y), min(t.shape[1], 1280 - x)
        c[y:y + h, x:x + w] = t[:h, :w]
        out.append(bgr_to_frame(c, "nv12"))
    return out


def test_tilted_video_through_the_tracker_and_the_redaction(golden_image):
    """The rotated sweep's records (scales NULL) through rf_track_update equal oracle/track.py, and rf_redact_yuv_device_style writes
    oracle/redact_style.py's bytes on the same records; the sweep keeps more faces tracked than rf_detect_yuv_track_device."""
    from oracle.redact_style import redact_yuv
    from oracle.track import CONFIRMED, TrackerOracle
    frames = _tilted_video(golden_image)
    e = _engine("fp16")
    trk, plain = e.tracker(), e.tracker()
    try:
        o = TrackerOracle(1)
        views = [(a, 1.0) for a in SWEEP]
        st = _style("blur", "ellipse")
        tracked = plain_tracked = 0
        for s in range(0, len(frames), 4):
            chunk = frames[s:s + 4]
            dev = [_cuda(f) for f in chunk]
            d, c, _, _ = e.detect_yuv_views_rotated_device(dev, views, THR, NMS)
            tp, tcn = trk.update([0] * 4, d, c)
            recs = e.read_dets(d, c, 4)[0]
            tracks = trk.read(tp, tcn, 4)
            for i in range(4):
                _same(tracks[i], o.update(0, recs[i], None), f"frame {s + i}")
                tracked += sum(int(r["state"]) == CONFIRMED for r in tracks[i])
            e.redact_yuv_device(dev, d, c, None, style="blur", shape="ellipse")
            e.synchronize()
            regs = _regions(recs, None)
            for i in range(4):
                assert np.array_equal(dev[i].cpu().numpy(), redact_yuv(chunk[i], "nv12", regs[i], st)), s + i
            ptp, ptc, _, _, _ = plain.detect_yuv_device([_cuda(f) for f in chunk], [0] * 4, THR, NMS)
            plain_tracked += sum(sum(int(r["state"]) == CONFIRMED for r in t) for t in plain.read(ptp, ptc, 4))
        print(f"\ntilted video: {tracked} confirmed track-frames with the 30-degree sweep, {plain_tracked} with rf_detect_yuv_track_device")
        assert tracked > plain_tracked and tracked >= len(frames)
    finally:
        trk.close()
        plain.close()
        e.close()


def test_refusals_and_other_calls(golden_image):
    """Each refusal returns its status before anything is launched or written (dets pointers, view scales, M and crops untouched); n = 0
    launches nothing; rf_detect_views_rotated, the tiled device calls and rf_detect_yuv_batch_device return what they did before."""
    import math

    import torch
    from retinaface_b200 import capi
    e = _engine("fp16")
    try:
        lib, h = e.lib, e.h
        img = cv2.resize(golden_image, (1100, 760))
        frame = bgr_to_frame(img, "nv12")
        d_img, d_frame = _cuda(img), _cuda(frame)
        views = VIEW_SETS[0]

        def plain():
            out = [e.detect_views_rotated(img, views, THR, NMS)]
            d, c = e.detect_tiled_device([d_img], THR, NMS)
            out.append(e.read_dets(d, c, 1))
            d, c = e.detect_yuv_tiled_device([d_frame], THR, NMS)
            out.append(e.read_dets(d, c, 1))
            d, c, sc = e.detect_yuv_device([d_frame], THR, NMS)
            out.append(e.read_dets(d, c, 1) + ([sc],))
            return out
        before = plain()
        e.detect_views_rotated_device([d_img], VIEW_SETS[1], THR, NMS)
        e.detect_yuv_views_rotated_device([d_frame], VIEW_SETS[2], THR, NMS, align={}, dev_crops_ptr=torch.empty(
            e.max_faces * 112 * 112 * 3, dtype=torch.uint8, device="cuda").data_ptr())
        after = plain()

        def flat(x):
            return [z for y in x for z in flat(y)] if isinstance(x, (list, tuple)) else [x]
        a, b = flat(before), flat(after)
        assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))

        canary = torch.full((4096,), 0xA5, dtype=torch.uint8, device="cuda")
        good, bad = capi.align_params(), capi.align_params(crop=(4, 4))
        yf = capi.yuv_frame(d_frame, "nv12")[0]

        def call(kind, vs, nv=None, n=1, align=None, crops=canary.data_ptr(), frames=None, matrix=0):
            scales = np.full(64, 7, np.float32)
            mats = np.full(64 * 6, 7, np.float64)
            varr = None if vs is None else (capi._RotatedView * max(len(vs), 1))(*[capi._RotatedView(a, s) for a, s in vs])
            nv = len(vs) if nv is None else nv
            d, c = C.c_void_p(), C.c_void_p()
            al = C.byref(align) if align is not None else None
            if kind == "bgr":
                P, I = C.c_void_p, C.c_int
                m = max(n, 1)
                rc = lib.rf_detect_views_rotated_device(h, (P * m)(*[d_img.data_ptr()] * m), (I * m)(*[1100] * m), (I * m)(*[760] * m), None, n,
                                                        varr, nv, THR, NMS, al, crops, None, C.byref(d), C.byref(c), scales.ctypes.data,
                                                        mats.ctypes.data)
            else:
                arr = frames if frames is not None else (capi.YuvFrame * max(n, 1))(*[yf] * max(n, 1))
                rc = lib.rf_detect_yuv_views_rotated_device(h, arr, n, matrix, varr, nv, THR, NMS, al, crops, None, C.byref(d), C.byref(c),
                                                            scales.ctypes.data, mats.ctypes.data)
            return rc, d.value is None and c.value is None and (scales == 7).all() and (mats == 7).all()

        bad_frame = capi.YuvFrame(yf.y, yf.u, yf.v, yf.y_pitch, yf.uv_pitch, 2, 1101, 760)
        one = [(30.0, 1.0)]
        cases = [(("bgr", one), dict(n=9), -6), (("yuv", one), dict(n=9), -6),                    # n > max_batch
                 (("yuv", one), dict(frames=(capi.YuvFrame * 1)(bad_frame)), -1),                 # odd width
                 (("yuv", one), dict(matrix=5), -1),                                              # unknown matrix
                 (("bgr", None), dict(nv=1), -1), (("yuv", None), dict(nv=1), -1),               # views NULL
                 (("bgr", one), dict(nv=0), -6), (("yuv", [(30.0, 1.0)] * 17), {}, -6),           # the view count
                 (("bgr", [(math.nan, 1.0)]), {}, -1), (("yuv", [(30.0, 1.0), (math.inf, 1.0)]), {}, -1),
                 (("bgr", [(30.0, 0.0)]), {}, -1), (("yuv", [(30.0, 1.5)]), {}, -1),             # shrink outside (0, 1]
                 (("bgr", one), dict(align=bad), -1), (("yuv", one), dict(align=good, crops=None), -1)]
        for k, ((kind, vs), kw, status) in enumerate(cases):
            rc, untouched = call(kind, vs, **kw)
            assert rc == status and untouched, (k, rc, status)
        for kind in ("bgr", "yuv"):
            assert call(kind, one, n=0) == (0, True)
        e.synchronize()
        assert (canary == 0xA5).all()
        out = np.full((448, 448, 3), 7, np.uint8)
        m6 = np.full(6, 7, np.float64)
        host_frame = (capi.YuvFrame * 1)(capi.yuv_frame(frame, "nv12")[0])
        for angle, shrink in ((math.nan, 1.0), (math.inf, 1.0), (30.0, 0.0), (30.0, 1.5)):
            assert lib.rf_preprocess_yuv_rotated(h, host_frame, 0, angle, shrink, out.ctypes.data, m6.ctypes.data) == -1
            assert (out == 7).all() and (m6 == 7).all()
    finally:
        e.close()


def test_detector_any_angle_frames(golden_image):
    """RetinaFace.detectAnyAngleFrames: per frame, detectAnyAngle's faces on cv2.cvtColor(frame)."""
    from retinaface_b200 import RetinaFace
    from conftest import caffemodel
    import os
    rf = RetinaFace(os.path.dirname(caffemodel("mnet25")), model_file="mnet25.caffemodel")
    try:
        bgr = [_tilted(golden_image, 45.0)[0][:1530, :1530], cv2.resize(golden_image, (1100, 760))]
        frames = [bgr_to_frame(b, "nv12") for b in bgr]
        got = rf.detectAnyAngleFrames([_cuda(f) for f in frames], 0.5, step=45.0)
        for g, f in zip(got, frames):
            want = rf.detectAnyAngle(frame_to_bgr(f, "nv12"), 0.5, step=45.0)
            assert len(g) == len(want) > 0 and all(a == b for a, b in zip(g, want))
    finally:
        rf.engine.close()
