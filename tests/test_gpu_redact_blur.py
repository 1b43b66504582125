"""GPU (-m gpu): f14 redaction styles -- rf_redact_yuv_device_style, rf_redact_device_style and rf_detect_yuv_redact_device_style
against oracle/redact_style.py byte for byte (every plane byte, pitch padding included): the elliptical and rectangular blur and
the elliptical mosaic on detected and synthetic records, {MOSAIC, RECT} against the f12 calls, radii 1 and 127, LOST tracks with and
without motion, the combined call against its parts, tiled 4K records, calls in flight, and the refusals."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle.redact import frame_regions, params
from oracle.redact_style import redact_bgr, redact_yuv, shape_mask, style
from oracle.yuv import bgr_to_frame
from test_gpu_redact import (NMS, SURF, SYNTH, THR, H, W, _canvas, _clones, _cuda, _det_array, _engine, _moving, _planes,
                             _surface)

pytestmark = pytest.mark.gpu

KINDS = {"mosaic": 1, "blur": 2}
SHAPES = {"rect": 1, "ellipse": 2}
STYLES = [("blur", "ellipse"), ("blur", "rect"), ("mosaic", "ellipse")]


def _style(kind, shape, blocks=0, detail=0):
    return style(KINDS[kind], SHAPES[shape], blocks, detail)


def _regions(recs, scales, blocks=0, margin=0.0, tracks=None):
    b, m = params(blocks, margin)
    return [frame_regions(r, len(r), None if scales is None else scales[i], m, b, tracks=None if tracks is None else tracks[i])
            for i, r in enumerate(recs)]


def _owned_luma(regions, shape, w, h):
    m = np.zeros((h, w), bool)
    for X0, Y0, X1, Y1, _ in regions:
        m |= shape_mask(X0, Y0, X1, Y1, w, h, SHAPES[shape])
    return m


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_styles_equal_the_oracle(golden_image, prec):
    """NV12 BT.601 surfaces (pitch 2048), I420 BT.709 buffers and strided BGR images of the golden photo on a 1080p canvas: detect,
    redact with each style, every byte equal to oracle/redact_style.py fed the fetched records and scales; only owned luma samples change."""
    eng = _engine(prec)
    imgs = [_canvas(golden_image, 37 * k, 23 * k) for k in range(3)]
    for kind, shape in STYLES:
        st = _style(kind, shape)
        surfs = [_surface(im) for im in imgs]
        dev = [_cuda(s) for s in surfs]
        frames = [_planes(d) for d in dev]
        d, c, sc = eng.detect_yuv_device(frames, THR, NMS, matrix="bt601")
        recs = eng.read_dets(d, c, 3)[0]
        assert all(len(r) >= 3 for r in recs)
        eng.redact_yuv_device(frames, d, c, sc, style=kind, shape=shape)
        eng.synchronize()
        regs = _regions(recs, sc)
        for k in range(3):
            want = redact_yuv(surfs[k], "nv12", regs[k], st, **SURF)
            got = dev[k].cpu().numpy()
            assert np.array_equal(got, want), (prec, kind, shape, k)
            y0 = surfs[k][:H * 2048].reshape(H, 2048)[:, :W]
            y1 = got[:H * 2048].reshape(H, 2048)[:, :W]
            changed = y0 != y1
            assert changed.any() and not (changed & ~_owned_luma(regs[k], shape, W, H)).any()
        # I420 BT.709, margin 0.5, detail 2
        bufs = [bgr_to_frame(im, "i420") for im in imgs]
        devi = [_cuda(b) for b in bufs]
        d, c, sc = eng.detect_yuv_device(devi, THR, NMS, layout="i420", matrix="bt709")
        recs = eng.read_dets(d, c, 3)[0]
        det = 2 if kind == "blur" else 0
        eng.redact_yuv_device(devi, d, c, sc, layout="i420", margin=0.5, style=kind, shape=shape, detail=det)
        eng.synchronize()
        for k in range(3):
            want = redact_yuv(bufs[k], "i420", _regions(recs, sc, 0, 0.5)[k], _style(kind, shape, detail=det))
            assert np.array_equal(devi[k].cpu().numpy(), want), (prec, kind, shape, "i420", k)
        # BGR rows 64 bytes beyond 3 w
        big = [np.full((H, 3 * W + 64), 0xEE, np.uint8) for _ in imgs]
        for b, im in zip(big, imgs):
            b[:, :3 * W] = im.reshape(H, 3 * W)
        devb = [_cuda(b) for b in big]
        views = [t[:, :3 * W].view(H, W, 3) for t in devb]
        eng.redact_device(views, d, c, sc, style=kind, shape=shape)
        eng.synchronize()
        for k in range(3):
            want = big[k].copy()
            want[:, :3 * W] = redact_bgr(imgs[k], _regions(recs, sc)[k], st).reshape(H, 3 * W)
            assert np.array_equal(devb[k].cpu().numpy(), want), (prec, kind, shape, "bgr", k)
    eng.close()


def test_mosaic_rect_style_equals_f12(golden_image):
    """{MOSAIC, RECT} through the _style calls writes the f12 calls' bytes, on detected and synthetic records, YUV and BGR."""
    import torch
    from retinaface_b200 import capi
    eng = _engine("fp16", max_faces=16)
    imgs = [_canvas(golden_image, 37 * k, 23 * k) for k in range(2)]
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    d, c, sc = eng.detect_yuv_device(a, THR, NMS)
    eng.synchronize()
    for blocks, margin in ((0, 0.0), (13, 0.6)):
        eng.redact_yuv_device(a, d, c, sc, blocks=blocks, margin=margin)
        st = capi.RedactStyle(1, 1, blocks, 0, margin)
        arr = eng._frames(b, "nv12", True)
        s = np.ascontiguousarray(sc, np.float32)
        eng._check(eng.lib.rf_redact_yuv_device_style(eng.h, arr, 2, d, c, s.ctypes.data, None, None, None, C.byref(st)))
        eng.synchronize()
        assert all(torch.equal(x, y) for x, y in zip(a, b)), (blocks, margin)
    rng = np.random.default_rng(3)
    dets, counts = _det_array(SYNTH[:2], eng.max_faces)
    dd, dc = _cuda(dets), _cuda(counts)
    scales = np.array([1.0, 1.5], np.float32)
    imgs = [rng.integers(0, 256, (360, 640, 3), dtype=np.uint8) for _ in range(2)]
    x, y = [_cuda(i) for i in imgs], [_cuda(i) for i in imgs]
    eng.redact_device(x, dd.data_ptr(), dc.data_ptr(), scales, blocks=5)
    ptrs, ws, hs, rs = eng._device_images(y)
    st = capi.RedactStyle(1, 1, 5, 0, 0.0)
    eng._check(eng.lib.rf_redact_device_style(eng.h, ptrs, ws, hs, rs, 2, dd.data_ptr(), dc.data_ptr(), scales.ctypes.data, None, None, None,
                                              C.byref(st)))
    eng.synchronize()
    assert all(torch.equal(p, q) for p, q in zip(x, y))
    eng.close()


@pytest.mark.parametrize("kind,shape,detail,margin", [("blur", "ellipse", 0, 0.0), ("blur", "rect", 1, 0.1), ("blur", "ellipse", 64, 1.0),
                                                      ("mosaic", "ellipse", 0, 0.33)])
def test_synthetic_records(kind, shape, detail, margin):
    """Device rf_det arrays with overlaps of different radii, zero and negative widths, NaN, boxes beyond +-65536 and frame edges, on
    I420 and BGR frames, and a frame with max_faces regions: identical bytes."""
    eng = _engine("fp16", max_faces=16)
    rng = np.random.default_rng(detail + 7)
    w, h = 640, 360
    boxes = [list(f) for f in SYNTH]
    boxes[2] = [(float(x), float(y), float(x + 40 + 9 * j), float(y + 50 + 5 * j)) for j, (x, y) in
                enumerate(zip(rng.uniform(-30, w - 20, 16), rng.uniform(-30, h - 20, 16)))]     # max_faces regions, overlapping
    dets, counts = _det_array(boxes, eng.max_faces)
    scales = np.array([1.0, 1.5, 1.0], np.float32)
    dd, dc = _cuda(dets), _cuda(counts)
    bufs = [rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8) for _ in range(3)]
    devi = [_cuda(b) for b in bufs]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(3)]
    devb = [_cuda(b) for b in imgs]
    blocks = 5 if kind == "mosaic" else 0
    kw = dict(blocks=blocks, margin=margin, style=kind, shape=shape, detail=detail)
    eng.redact_yuv_device(devi, dd.data_ptr(), dc.data_ptr(), scales, layout="i420", **kw)
    eng.redact_device(devb, dd.data_ptr(), dc.data_ptr(), scales, **kw)
    eng.synchronize()
    recs = [dets[i, :counts[i], :15] for i in range(3)]
    regs = _regions(recs, scales, blocks, margin)
    st = _style(kind, shape, blocks, detail)
    assert len(regs[2]) == 16
    for k in range(3):
        assert np.array_equal(devi[k].cpu().numpy(), redact_yuv(bufs[k], "i420", regs[k], st)), k
        assert np.array_equal(devb[k].cpu().numpy(), redact_bgr(imgs[k], regs[k], st)), k
    eng.close()


def test_largest_radius_on_4k():
    """detail 1 on a 3840x2160 NV12 frame: regions of radius 127 (and a chroma radius of 64) whose 3a halos leave the frame on every
    side, and a small region of radius 1 at detail 64 in the same call's neighbour frame."""
    eng = _engine("fp16", max_batch=2, max_image=(2160, 3840))
    rng = np.random.default_rng(5)
    w, h = 3840, 2160
    bufs = [rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8) for _ in range(2)]
    for b in bufs:        # smooth content as well, so that rounding carries differ across the halo
        b[:h] = cv2.GaussianBlur(b[:h], (0, 0), 9)
    boxes = [[(-300, -200, 900, 700), (3000, 1500, 4100, 2400), (1200, 600, 2400, 1600)], [(100, 100, 104, 103), (3830, 2150, 3900, 2200)]]
    for detail in (1, 64):
        dets, counts = _det_array(boxes, eng.max_faces)
        dd, dc = _cuda(dets), _cuda(counts)
        dev = [_cuda(b) for b in bufs]
        eng.redact_yuv_device(dev, dd.data_ptr(), dc.data_ptr(), None, style="blur", shape="ellipse", detail=detail)
        eng.synchronize()
        regs = _regions([dets[i, :counts[i], :15] for i in range(2)], None)
        st = _style("blur", "ellipse", detail=detail)
        for k in range(2):
            assert np.array_equal(dev[k].cpu().numpy(), redact_yuv(bufs[k], "nv12", regs[k], st)), (detail, k)
    eng.close()


@pytest.mark.parametrize("motion", [False, True])
def test_lost_tracks_stay_covered(golden_image, motion):
    """The moving photo with the faces blanked on frames 5 and 6, through the combined call with a tracker: every frame equals the
    oracle fed the returned records and tracks, and on the blanked frames LOST tracks still add blurred ellipses."""
    eng = _engine("fp16")
    trk = eng.tracker(motion=True if motion else None)
    imgs = _moving(golden_image, 9)
    lost_frames = 0
    for t, im in enumerate(imgs):
        if t in (5, 6):
            im = np.full_like(im, 128)
            im[::7] = 60          # texture that a blur changes
        buf = bgr_to_frame(im, "nv12")
        f = _cuda(buf)
        tp, tc, d, c, sc = trk.detect_yuv_redact_device([f], [0], THR, NMS, style="blur", shape="ellipse")
        rec = eng.read_dets(d, c, 1)[0][0]
        tracks = trk.read(tp, tc, 1)[0]
        regs = _regions([rec], sc, tracks=[tracks])[0]
        assert np.array_equal(f.cpu().numpy(), redact_yuv(buf, "nv12", regs, _style("blur", "ellipse"))), t
        if t in (5, 6):
            assert len(rec) == 0 and (tracks["state"] == 2).sum() >= 3, t
            assert not np.array_equal(f.cpu().numpy(), buf)
            lost_frames += 1
    assert lost_frames == 2
    trk.close()
    eng.close()


def test_combined_call_equals_its_parts(golden_image):
    """rf_detect_yuv_redact_device_style against rf_detect_yuv_batch_device + rf_redact_yuv_device_style, and with a tracker against
    rf_detect_yuv_track_device + the primitive: records, tracks and frames bit-equal."""
    import torch
    eng = _engine("fp16")
    imgs = _moving(golden_image, 8)
    kw = dict(style="blur", shape="ellipse", detail=3, margin=0.3)
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    for s in range(0, 8, 4):
        d1, c1, s1 = eng.detect_yuv_redact_device(a[s:s + 4], THR, NMS, **kw)
        r1 = eng.read_dets(d1, c1, 4)[0]
        d2, c2, s2 = eng.detect_yuv_device(b[s:s + 4], THR, NMS)
        r2 = eng.read_dets(d2, c2, 4)[0]
        eng.redact_yuv_device(b[s:s + 4], d2, c2, s2, **kw)
        eng.synchronize()
        assert all(np.array_equal(x, y) for x, y in zip(r1, r2)) and np.array_equal(s1, s2)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    t1, t2 = eng.tracker(), eng.tracker()
    for s in range(0, 8, 2):
        tp1, tc1, d1, c1, s1 = t1.detect_yuv_redact_device(a[s:s + 2], [0] * 2, THR, NMS, style="mosaic", shape="ellipse")
        tp2, tc2, d2, c2, s2 = t2.detect_yuv_device(b[s:s + 2], [0] * 2, THR, NMS)
        eng.redact_yuv_device(b[s:s + 2], d2, c2, s2, tracker=t2, tracks_ptr=tp2, track_counts_ptr=tc2, style="mosaic", shape="ellipse")
        eng.synchronize()
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(t1.read(tp1, tc1, 2), t2.read(tp2, tc2, 2)))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    t1.close()
    t2.close()
    eng.close()


def test_tiled_4k_records(golden_image):
    """A 3840x2160 canvas of half-scale photos through rf_detect_yuv_tiled_device, blurred with scales = NULL: equal to the oracle."""
    eng = _engine("fp16", max_image=(2160, 3840))
    half = cv2.resize(golden_image, None, fx=0.5, fy=0.5)
    img = np.full((2160, 3840, 3), 128, np.uint8)
    for x, y in [(200, 150), (2000, 300), (900, 1300), (2900, 1500)]:
        img[y:y + half.shape[0], x:x + half.shape[1]] = half
    buf = bgr_to_frame(img, "nv12")
    dev = _cuda(buf)
    d, c = eng.detect_yuv_tiled_device([dev], THR, NMS)
    rec = eng.read_dets(d, c, 1)[0][0]
    assert len(rec) >= 12
    eng.redact_yuv_device([dev], d, c, None, style="blur", shape="ellipse")
    eng.synchronize()
    assert np.array_equal(dev.cpu().numpy(), redact_yuv(buf, "nv12", _regions([rec], None)[0], _style("blur", "ellipse")))
    eng.close()


@pytest.mark.parametrize("streams", [2, 8])
def test_calls_in_flight(golden_image, streams):
    """2 streams + 1 combined blur calls in flight, each on its own frames, against the same calls synchronised one by one."""
    import torch
    eng = _engine("fp16", streams=streams)
    k = 2 * streams + 1
    imgs = _moving(golden_image, 4 * k)
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    for s in range(k):
        eng.detect_yuv_redact_device(a[4 * s:4 * s + 4], THR, NMS, style="blur", shape="ellipse")
    eng.synchronize()
    for s in range(k):
        eng.detect_yuv_redact_device(b[4 * s:4 * s + 4], THR, NMS, style="blur", shape="ellipse")
        eng.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    eng.close()


def test_invalid_styles_launch_nothing(golden_image):
    import torch
    from retinaface_b200 import capi
    eng = _engine("fp16", max_batch=2)
    lib = eng.lib
    buf = bgr_to_frame(_canvas(golden_image), "nv12")
    f = [_cuda(buf), _cuda(buf)]
    d, c, sc = eng.detect_yuv_device(f, THR, NMS)
    eng.synchronize()
    before = _clones(f)
    arr = eng._frames(f, "nv12", True)
    s = np.ascontiguousarray(sc, np.float32)
    bad = [(3, 0, 0, 0, 0.0), (-1, 0, 0, 0, 0.0), (0, 3, 0, 0, 0.0), (2, 0, 8, 0, 0.0), (2, 0, 0, 65, 0.0), (2, 0, 0, -1, 0.0),
           (1, 0, 0, 4, 0.0), (1, 0, 33, 0, 0.0), (0, 0, 0, 0, 1.5), (0, 0, 0, 0, float("nan"))]
    ptrs, ws, hs, rs = eng._device_images([t.view(-1)[:64 * 8 * 3].view(8, 64, 3) for t in f])
    outs = [C.c_void_p(0x5EED) for _ in range(4)]
    for v in bad:
        st = capi.RedactStyle(*v)
        assert lib.rf_redact_yuv_device_style(eng.h, arr, 2, d, c, s.ctypes.data, None, None, None, C.byref(st)) == -1, v
        assert lib.rf_redact_device_style(eng.h, ptrs, ws, hs, rs, 2, d, c, None, None, None, None, C.byref(st)) == -1, v
        assert lib.rf_detect_yuv_redact_device_style(eng.h, None, arr, None, 2, 0, THR, NMS, C.byref(st), *(C.byref(o) for o in outs), None) == -1, v
    # f12's statuses come first, in f12's order
    arr3 = eng._frames([f[0]] * 3, "nv12", True)
    st = capi.RedactStyle(7, 0, 0, 0, 0.0)
    assert lib.rf_redact_yuv_device_style(eng.h, arr3, 3, d, c, None, None, None, None, C.byref(st)) == -6
    assert lib.rf_redact_yuv_device_style(eng.h, arr3, 3, d, c, None, None, None, None, None) == -6
    eng.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(f, before))
    assert all(o.value == 0x5EED for o in outs)
    eng.close()


def test_detector_redact_frames_blur(golden_image):
    """RetinaFace.redactFrames(style="blur", shape="ellipse") is the combined call."""
    import os
    import torch
    from conftest import GOLDEN
    from retinaface_b200.detector import RetinaFace
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    eng = det.engine
    buf = bgr_to_frame(_canvas(golden_image), "nv12")
    a, b = _cuda(buf), _cuda(buf)
    det.redactFrames([a], threshold=THR, style="blur", shape="ellipse", detail=6)
    d, c, sc = eng.detect_yuv_device([b], THR, det.nms_threshold)
    eng.redact_yuv_device([b], d, c, sc, style="blur", shape="ellipse", detail=6)
    eng.synchronize()
    assert torch.equal(a, b) and not np.array_equal(a.cpu().numpy(), buf)
