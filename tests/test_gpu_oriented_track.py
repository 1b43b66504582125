"""GPU (-m gpu): f20 oriented videos in tracker calls.  Every case runs a tracker on stored frames S with a video at orientation o against
a twin tracker at orientation 1 on the materialised displayed frames orient_planes(S, o) (oracle/orient.py), and holds
them equal bit for bit: records, out_scales, track lists, rf_tracker_debug_state, crops and matrices, and the written frames as
orient_planes(S_out, o) == twin_out.  Also: rf_redact_yuv_oriented_device_style against rf_redact_yuv_device_style on the rotated
copies, a portrait phone video whose faces a tracker without the orientation leaves uncovered, pitched surfaces whose padding stays
untouched, calls in flight, the drivers, and every refusal with nothing changed."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.orient import orient_planes, unorient_planes
from oracle.yuv import bgr_to_frame

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
ALL = list(range(1, 9))
SOME = [2, 5, 6, 8]
W, H = 1280, 720            # the stored (landscape) frame; orientations 5..8 display it as 720 x 1280
INVALID, UNSUPPORTED = -1, -7


def _engine(prec="fp16", **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (1920, 1920))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


@pytest.fixture(scope="module")
def eng():
    e = _engine(streams=2)
    yield e
    e.close()


def _cuda(a):
    """A device copy, complete before the library's streams (which do not wait for torch's) read it."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


SHAKE = [(0, 0), (47, -41), (-38, 52), (61, 40), (-52, -47), (44, 66), (-63, 35), (40, -58)]


def _displayed(golden, o, k, w=W, h=H, scale=0.5, faces=True, shake=False):
    """Displayed BGR frame k of a video shown in orientation o: the golden photo, scaled, moving on a grey canvas of the displayed size
    (shake: jumping 40-70 px between frames, as a shaking camera moves the scene)."""
    dw, dh = (h, w) if o >= 5 else (w, h)
    if shake:          # the whole scene moves: texture everywhere for the motion estimate
        return np.ascontiguousarray(np.roll(cv2.resize(golden, (dw, dh)), (SHAKE[k % 8][1], SHAKE[k % 8][0]), axis=(0, 1)))
    img = np.full((dh, dw, 3), 128, np.uint8)
    if faces:
        g = cv2.resize(golden, None, fx=scale, fy=scale)
        x, y = 10 + 9 * k, 30 + 13 * k
        g = g[:dh - y, :dw - x]
        img[y:y + g.shape[0], x:x + g.shape[1]] = g
    return img


def _video(golden, o, layout, n, blank=0, **kw):
    """(stored frames S, displayed frames D = orient_planes(S, o)) of n frames, host single buffers; the first `blank` without faces."""
    shown = [bgr_to_frame(_displayed(golden, o, k, faces=k >= blank, **kw), layout) for k in range(n)]
    stored = [unorient_planes(d, layout, o) for d in shown]
    for s, d in zip(stored, shown):
        assert np.array_equal(orient_planes(s, layout, o), d)
    return stored, shown


def _bytes(recs):
    return [np.ascontiguousarray(r).tobytes() for r in recs]


def _same_lists(ta, tb, a, b, n):
    assert _bytes(ta.read(*a, n)) == _bytes(tb.read(*b, n))


def _same_dets(eng, a, b, n):
    fa, ia = eng.read_dets(*a, n)
    fb, ib = eng.read_dets(*b, n)
    assert _bytes(fa) == _bytes(fb) and _bytes(ia) == _bytes(ib)
    return fa


def _same_state(ta, tb, videos):
    for v in videos:
        ha, ra = ta.debug_state(v)
        hb, rb = tb.debug_state(v)
        assert np.array_equal(ha, hb) and np.array_equal(ra, rb), v


def _redact_pair(eng, golden, o, layout, matrix, calls, per, style, shape, detail=0):
    """A plain redacting tracker on S at orientation o and its twin at orientation 1 on D, `calls` calls of `per` frames of video 0."""
    S, D = _video(golden, o, layout, calls * per)
    s_dev, d_dev = [_cuda(f) for f in S], [_cuda(f) for f in D]
    ta, tb = eng.tracker(max_videos=2), eng.tracker(max_videos=2)
    ta.set_orientation(0, o)
    kw = dict(layout=layout, matrix=matrix, style=style, shape=shape, detail=detail)
    for c in range(calls):
        fa, fb = s_dev[c * per:(c + 1) * per], d_dev[c * per:(c + 1) * per]
        ra = ta.detect_yuv_redact_device(fa, [0] * per, THR, NMS, **kw)
        eng.synchronize()
        recs = _same_dets(eng, ra[2:4], ra[2:4], per)      # read before the twin's call reuses the context
        la = ta.read(ra[0], ra[1], per)
        rb = tb.detect_yuv_redact_device(fb, [0] * per, THR, NMS, **kw)
        eng.synchronize()
        fb_, ib_ = eng.read_dets(rb[2], rb[3], per)
        assert _bytes(recs) == _bytes(fb_), (o, c)
        assert np.array_equal(ra[4], rb[4]), (o, c)
        assert _bytes(la) == _bytes(tb.read(rb[0], rb[1], per)), (o, c)
    _same_state(ta, tb, [0])
    for k, (a, b) in enumerate(zip(s_dev, d_dev)):
        got = orient_planes(a.cpu().numpy(), layout, o)
        want = b.cpu().numpy()
        assert np.array_equal(got, want), (o, k)
        assert not np.array_equal(want, D[k]), (o, k)          # something was written
    ta.close()
    tb.close()


@pytest.mark.parametrize("style,shape", [("mosaic", "rect"), ("blur", "ellipse")])
@pytest.mark.parametrize("o", ALL)
def test_plain_redaction_every_orientation(eng, golden_image, o, style, shape):
    _redact_pair(eng, golden_image, o, "nv12", "bt601", calls=3, per=2, style=style, shape=shape)


@pytest.mark.parametrize("per", [1, 4, 8])
def test_frames_per_call(eng, golden_image, per):
    _redact_pair(eng, golden_image, 6, "nv12", "bt601", calls=2, per=per, style="mosaic", shape="ellipse")


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("layout,matrix", [("nv12", "bt601"), ("i420", "bt709")])
def test_crops_and_blur_across_engines(golden_image, prec, layout, matrix):
    """New-identity crops and matrices of rf_detect_yuv_track_device, and a blur / rect redaction, for {2, 5, 6, 8}."""
    import torch
    e = _engine(prec)
    try:
        A, n = 8, 3
        for o in SOME:
            S, D = _video(golden_image, o, layout, n)
            ta, tb = e.tracker(), e.tracker()
            ta.set_orientation(0, o)
            out = []
            for t, frames in ((ta, S), (tb, D)):
                dev = [_cuda(f) for f in frames]
                crops = torch.zeros((n, A, 112, 112, 3), dtype=torch.uint8, device="cuda")
                mats = torch.zeros((n, A, 6), dtype=torch.float64, device="cuda")
                torch.cuda.synchronize()
                res = []
                for i in range(n):       # one frame per call: tracks are confirmed over the calls, and crops cut on confirmation
                    r = t.detect_yuv_device(dev[i:i + 1], [0], THR, NMS, layout=layout, matrix=matrix, align=dict(max_faces=A),
                                            dev_crops_ptr=crops[i].data_ptr(), dev_mats_ptr=mats[i].data_ptr())
                    e.synchronize()
                    res.append((_bytes(e.read_dets(r[2], r[3], 1)[0]), r[4].tobytes(), _bytes(t.read(r[0], r[1], 1))))
                out.append((res, crops.cpu().numpy(), mats.cpu().numpy()))
            assert out[0][0] == out[1][0], (prec, o)
            assert np.array_equal(out[0][1], out[1][1]) and np.array_equal(out[0][2], out[1][2]), (prec, o)
            assert out[0][1].any(), (prec, o)                   # some identity was cropped
            _same_state(ta, tb, [0])
            ta.close()
            tb.close()
            _redact_pair(e, golden_image, o, layout, matrix, calls=2, per=2, style="blur", shape="rect", detail=2)
    finally:
        e.close()


def test_two_videos_interleaved(eng, golden_image):
    """Video 0 at orientation 6 and video 1 upright, interleaved in one call: each equals its own twin."""
    S0, D0 = _video(golden_image, 6, "nv12", 4)
    S1, _ = _video(golden_image, 1, "nv12", 4, scale=0.4)
    a = [_cuda(f) for f in (S0[0], S1[0], S0[1], S1[1], S0[2], S1[2], S0[3], S1[3])]
    b = [_cuda(f) for f in (D0[0], S1[0], D0[1], S1[1], D0[2], S1[2], D0[3], S1[3])]
    videos = [0, 1] * 4
    ta, tb = eng.tracker(max_videos=2), eng.tracker(max_videos=2)
    ta.set_orientation(0, 6)
    for half in range(2):
        sl = slice(4 * half, 4 * half + 4)
        ra = ta.detect_yuv_redact_device(a[sl], videos[sl], THR, NMS, style="blur", shape="ellipse")
        eng.synchronize()
        fa = eng.read_dets(ra[2], ra[3], 4)[0]
        la = ta.read(ra[0], ra[1], 4)
        rb = tb.detect_yuv_redact_device(b[sl], videos[sl], THR, NMS, style="blur", shape="ellipse")
        eng.synchronize()
        assert _bytes(fa) == _bytes(eng.read_dets(rb[2], rb[3], 4)[0]) and np.array_equal(ra[4], rb[4])
        assert _bytes(la) == _bytes(tb.read(rb[0], rb[1], 4))
    _same_state(ta, tb, [0, 1])
    for k in range(8):
        got = a[k].cpu().numpy()
        if k % 2 == 0:
            got = orient_planes(got, "nv12", 6)
        assert np.array_equal(got, b[k].cpu().numpy()), k
    ta.close()
    tb.close()


def test_pitched_surfaces_keep_their_padding(eng, golden_image):
    """NV12 stored surfaces with rows 1536 bytes apart and chroma from its own allocation: the padding stays 0xEE."""
    P = 1536
    for o in (3, 6, 7):
        S, D = _video(golden_image, o, "nv12", 2)
        surfs = []
        for s in S:
            y = np.full((H, P), 0xEE, np.uint8)
            uv = np.full((H // 2, P), 0xEE, np.uint8)
            y[:, :W], uv[:, :W] = s[:H], s[H:]
            surfs.append((_cuda(y), _cuda(uv)))
        ta, tb = eng.tracker(), eng.tracker()
        ta.set_orientation(0, o)
        d_dev = [_cuda(f) for f in D]
        ta.detect_yuv_redact_device([(y[:, :W], uv[:, :W]) for y, uv in surfs], [0, 0], THR, NMS, style="mosaic", shape="rect")
        tb.detect_yuv_redact_device(d_dev, [0, 0], THR, NMS, style="mosaic", shape="rect")
        eng.synchronize()
        for (y, uv), b in zip(surfs, d_dev):
            yh, uvh = y.cpu().numpy(), uv.cpu().numpy()
            assert (yh[:, W:] == 0xEE).all() and (uvh[:, W:] == 0xEE).all(), o
            got = np.concatenate([yh[:, :W], uvh[:, :W]])
            assert np.array_equal(orient_planes(got, "nv12", o), b.cpu().numpy()), o
        ta.close()
        tb.close()


def test_calls_in_flight_equal_blocking_runs(eng, golden_image):
    """2 streams + 1 = 5 calls issued back to back equal the same calls each followed by a synchronize."""
    o, n = 8, 5
    S, _ = _video(golden_image, o, "nv12", 2 * n)
    outs = []
    for blocking in (False, True):
        t = eng.tracker()
        t.set_orientation(0, o)
        dev = [_cuda(f) for f in S]
        lists = []
        for c in range(n):
            r = t.detect_yuv_redact_device(dev[2 * c:2 * c + 2], [0, 0], THR, NMS, style="blur", shape="ellipse")
            if blocking:
                eng.synchronize()
            lists.append(r)
        eng.synchronize()
        outs.append(([d.cpu().numpy().tobytes() for d in dev], t.debug_state(0)[1].tobytes(), _bytes(t.read(lists[-1][0], lists[-1][1], 2))))
        t.close()
    assert outs[0] == outs[1]


@pytest.mark.parametrize("layout,matrix", [("nv12", "bt601"), ("i420", "bt709")])
def test_standalone_oriented_redaction(eng, golden_image, layout, matrix):
    """rf_redact_yuv_oriented_device_style on rf_detect_yuv_oriented_device records, with and without rf_track_update lists, equals
    rf_redact_yuv_device_style on the rotated copies, mapped back; at orientation 1 it writes the unoriented call's bytes."""
    os_ = [6, 2, 5, 8]
    shown = [bgr_to_frame(_displayed(golden_image, o, k), layout) for k, o in enumerate(os_)]
    blank = [bgr_to_frame(_displayed(golden_image, o, 4 + k, faces=False), layout) for k, o in enumerate(os_)]
    for kind, shape in (("mosaic", "rect"), ("blur", "ellipse"), ("mosaic", "ellipse")):
        ta, tb = eng.tracker(max_videos=4), eng.tracker(max_videos=4)
        for step, D in enumerate((shown, blank)):      # the blank frames leave every track LOST: region (b)
            S = [unorient_planes(d, layout, o) for d, o in zip(D, os_)]
            a, b = [_cuda(f) for f in S], [_cuda(f) for f in D]
            d, c, sc = eng.detect_yuv_oriented_device(a, os_, THR, NMS, layout=layout, matrix=matrix)
            tp, tc = ta.update(range(4), d, c, sc)
            eng.redact_yuv_oriented_device(a, os_, d, c, sc, layout=layout, tracker=ta, tracks_ptr=tp, track_counts_ptr=tc, style=kind,
                                           shape=shape)
            eng.synchronize()
            recs = eng.read_dets(d, c, 4)[0]
            la = ta.read(tp, tc, 4)
            d2, c2, sc2 = eng.detect_yuv_device(b, THR, NMS, layout=layout, matrix=matrix)
            tp2, tc2 = tb.update(range(4), d2, c2, sc2)
            eng.redact_yuv_device(b, d2, c2, sc2, layout=layout, tracker=tb, tracks_ptr=tp2, track_counts_ptr=tc2, style=kind, shape=shape)
            eng.synchronize()
            assert _bytes(recs) == _bytes(eng.read_dets(d2, c2, 4)[0]) and np.array_equal(sc, sc2)
            assert _bytes(la) == _bytes(tb.read(tp2, tc2, 4))
            if step == 1:
                assert any((t["state"] == 2).any() for t in la), "no LOST track"      # RF_TRACK_LOST
            for k in range(4):
                assert np.array_equal(orient_planes(a[k].cpu().numpy(), layout, os_[k]), b[k].cpu().numpy()), (kind, shape, step, k)
            # without track lists
            a, b = [_cuda(f) for f in S], [_cuda(f) for f in D]
            d, c, sc = eng.detect_yuv_oriented_device(a, os_, THR, NMS, layout=layout, matrix=matrix)
            eng.redact_yuv_oriented_device(a, os_, d, c, sc, layout=layout, style=kind, shape=shape)
            eng.synchronize()
            d2, c2, sc2 = eng.detect_yuv_device(b, THR, NMS, layout=layout, matrix=matrix)
            eng.redact_yuv_device(b, d2, c2, sc2, layout=layout, style=kind, shape=shape)
            eng.synchronize()
            for k in range(4):
                assert np.array_equal(orient_planes(a[k].cpu().numpy(), layout, os_[k]), b[k].cpu().numpy()), (kind, shape, "untracked", k)
        ta.close()
        tb.close()
    # orientation 1: the unoriented call's bytes
    a, b = [_cuda(f) for f in shown], [_cuda(f) for f in shown]
    d, c, sc = eng.detect_yuv_device(a, THR, NMS, layout=layout, matrix=matrix)
    eng.synchronize()
    eng.redact_yuv_oriented_device(a, [1] * 4, d, c, sc, layout=layout, style="blur", shape="ellipse")
    eng.redact_yuv_device(b, d, c, sc, layout=layout, style="blur", shape="ellipse")
    eng.synchronize()
    assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a, b))


def _covered(before, after, boxes, w, h):
    """Per box: whether the luma inside its central half changed on at least half of its samples."""
    out = []
    for x1, y1, x2, y2 in boxes:
        cx, cy, bw, bh = (x1 + x2) / 2, (y1 + y2) / 2, (x2 - x1) / 4, (y2 - y1) / 4
        X0, X1 = int(max(cx - bw, 0)), int(min(cx + bw, w))
        Y0, Y1 = int(max(cy - bh, 0)), int(min(cy + bh, h))
        out.append((before[Y0:Y1, X0:X1] != after[Y0:Y1, X0:X1]).mean() >= 0.5)
    return out


def test_portrait_phone_video_is_covered(golden_image):
    """A 1920x1080 stored video of moving faces shown at orientation 6.  A redacting tracker without the orientation sees the faces
    lying on their side and leaves most of them uncovered; with it, every face the upright twin finds lies inside a written region on
    every frame."""
    e = _engine("fp16")
    try:
        o, n = 6, 12
        S, D = _video(golden_image, o, "nv12", n, w=1920, h=1080, scale=0.8)
        boxes = []
        for k in range(n):      # the faces: what the detector finds on the displayed frame
            d, c, sc = e.detect_yuv_device([_cuda(D[k])], THR, NMS)
            f = e.read_dets(d, c, 1)[0][0]
            boxes.append([tuple(float(v) * sc[0] for v in r[1:5]) for r in f])
        assert all(len(b) >= 1 for b in boxes)
        dh, dw = 1920, 1080
        res = {}
        for oriented in (False, True):
            t = e.tracker()
            if oriented:
                t.set_orientation(0, o)
            dev = [_cuda(f) for f in S]
            for c in range(0, n, 4):
                t.detect_yuv_redact_device(dev[c:c + 4], [0] * 4, THR, NMS)
            e.synchronize()
            cov = []
            for k in range(n):
                shown_out = orient_planes(dev[k].cpu().numpy(), "nv12", o)
                cov.append(_covered(D[k][:dh], shown_out[:dh], boxes[k], dw, dh))
            res[oriented] = cov
            t.close()
        assert all(all(c) for c in res[True]), res[True]
        assert np.mean([np.mean(c) for c in res[False]]) < 0.5, res[False]
    finally:
        e.close()


def test_refusals_change_nothing(eng, golden_image):
    from retinaface_b200 import capi
    lib = eng.lib
    t = eng.tracker(max_videos=2)
    for bad in (0, 9, -1):
        assert lib.rf_tracker_set_orientation(t.t, 0, bad) == INVALID
    for v in (-2, 2):
        assert lib.rf_tracker_set_orientation(t.t, v, 6) == INVALID
    assert lib.rf_tracker_set_orientation(None, 0, 6) == INVALID
    # the orientation holds from a video's first frame call to its next restart
    S, D = _video(golden_image, 6, "nv12", 2)
    assert lib.rf_tracker_set_orientation(t.t, 0, 6) == 0
    t.detect_yuv_redact_device([_cuda(S[0])], [0], THR, NMS)
    for v, o in ((0, 1), (-1, 6), (0, 6)):
        assert lib.rf_tracker_set_orientation(t.t, v, o) == INVALID, (v, o)
    assert lib.rf_tracker_set_orientation(t.t, 1, 3) == 0        # video 1 has not started
    t.reset(0)
    assert lib.rf_tracker_set_orientation(t.t, 0, 6) == 0        # reset keeps it and frees the setter again
    t.close()
    # the reset kept orientation 6: a fresh call equals a twin on the displayed frame
    ta, tb = eng.tracker(), eng.tracker()
    ta.set_orientation(-1, 6)
    ta.reset()
    a, b = _cuda(S[1]), _cuda(D[1])
    ra = ta.detect_yuv_redact_device([a], [0], THR, NMS)
    rb = tb.detect_yuv_redact_device([b], [0], THR, NMS)
    eng.synchronize()
    assert np.array_equal(orient_planes(a.cpu().numpy(), "nv12", 6), b.cpu().numpy()) and np.array_equal(ra[4], rb[4])
    ta.close()
    tb.close()
    # orientation 1 is accepted on every kind; drain and finish restart a video, which frees the setter again
    lb = eng.tracker(lookback=2)
    lb.set_orientation(0, 1)
    out = [_cuda(S[0])]
    lb.detect_yuv_redact_lookback_device([_cuda(S[0])], [0], out, THR, NMS)
    assert lib.rf_tracker_set_orientation(lb.t, 0, 1) == INVALID
    lb.drain(0, [_cuda(S[0])])
    assert lib.rf_tracker_set_orientation(lb.t, 0, 1) == 0
    lb.close()
    import torch
    bt = eng.tracker(best={})
    crops = torch.zeros((1, 64, 112, 112, 3), dtype=torch.uint8, device="cuda")
    bt.detect_yuv_best_device([_cuda(S[0])], [0], THR, NMS, crops.data_ptr())
    assert lib.rf_tracker_set_orientation(bt.t, 0, 1) == INVALID
    bt.finish(0, crops.data_ptr())
    assert lib.rf_tracker_set_orientation(bt.t, 0, 1) == 0
    assert lib.rf_tracker_set_orientation(bt.t, 0, 6) == 0
    bt.close()
    # tiling, in either order: RF_ERR_UNSUPPORTED, nothing changed
    x = eng.tracker(tiling=True)
    assert lib.rf_tracker_set_orientation(x.t, 0, 6) == UNSUPPORTED
    assert lib.rf_tracker_set_orientation(x.t, -1, 6) == UNSUPPORTED
    assert lib.rf_tracker_set_orientation(x.t, 0, 1) == 0
    x.close()
    y = eng.tracker(max_videos=2)
    y.set_orientation(1, 8)
    with pytest.raises(capi.RfError) as e:
        y.set_tiling()
    assert e.value.status == UNSUPPORTED
    assert lib.rf_tracker_set_orientation(y.t, 1, 1) == 0
    y.set_tiling()                          # every video upright again: tiling is accepted
    y.close()
    # every other option, before or after the orientation
    for opt in ("motion", "follow", "lookback"):
        x = eng.tracker(**{opt: True})
        assert lib.rf_tracker_set_orientation(x.t, 0, 6) == 0, opt
        x.close()
        y = eng.tracker()
        y.set_orientation(0, 8)
        getattr(y, "set_" + opt)()
        y.close()
    # the standalone call: bad orientations, nothing written
    f = [_cuda(S[0])]
    d, c, sc = eng.detect_yuv_oriented_device(f, [6], THR, NMS)
    eng.synchronize()
    before = f[0].cpu().numpy()
    arr = eng._frames(f, "nv12", True)
    st = capi.RedactStyle(1, 1, 0, 0, 0.0)
    for bad in (0, 9):
        o = (C.c_int * 1)(bad)
        s = np.ascontiguousarray(sc, np.float32)
        assert lib.rf_redact_yuv_oriented_device_style(eng.h, arr, o, 1, d, c, s.ctypes.data, None, None, None, C.byref(st)) == INVALID
    assert lib.rf_redact_yuv_oriented_device_style(eng.h, arr, None, 1, d, c, None, None, None, None, C.byref(st)) == INVALID
    eng.synchronize()
    assert np.array_equal(f[0].cpu().numpy(), before)


def test_python_driver_equals_the_c_calls(golden_image):
    """RetinaFace.setVideoOrientation with trackFrames / redactFrames equals the same calls by hand on a tracker set to the same
    orientations, set before the tracker exists and at once after."""
    from retinaface_b200.detector import RetinaFace
    o = 5
    S, _ = _video(golden_image, o, "nv12", 4)
    S3, _ = _video(golden_image, 3, "nv12", 2, scale=0.4)
    eng = _engine("fp16")
    try:
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        rf.setVideoOrientation(0, o)
        a = [_cuda(f) for f in S]
        rf.redactFrames(a[:2], [0, 0], THR, max_videos=2, style="blur", shape="ellipse")
        rf.setVideoOrientation(1, 3)          # the tracker exists: applied at once
        got = rf.trackFrames([_cuda(f) for f in S3], [1, 1], THR)[0]
        rf.redactFrames(a[2:], [0, 0], THR, style="blur", shape="ellipse")
        eng.synchronize()
        t = eng.tracker(max_videos=2)
        t.set_orientation(0, o)
        t.set_orientation(1, 3)
        b = [_cuda(f) for f in S]
        t.detect_yuv_redact_device(b[:2], [0, 0], THR, NMS, style="blur", shape="ellipse")
        tp, tc, _, _, _ = t.detect_yuv_device([_cuda(f) for f in S3], [1, 1], THR, NMS)
        want = RetinaFace._lists(t.read(tp, tc, 2))
        t.detect_yuv_redact_device(b[2:], [0, 0], THR, NMS, style="blur", shape="ellipse")
        eng.synchronize()
        assert got == want
        assert all(np.array_equal(x.cpu().numpy(), y.cpu().numpy()) for x, y in zip(a, b))
        t.close()
        rf._tracker.close()
    finally:
        eng.close()


CPP_PROGRAM = r'''
#include "RetinaFace.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <fstream>
// argv: model directory, frames file (n NV12 1280x720 stored frames), out file, n.  Video 0 shown at orientation 6, redactYUV two
// frames a call, then the bytes.
int main(int argc, char **argv) {
    string model = argv[1];
    const int n = atoi(argv[4]), w = 1280, h = 720;
    const size_t bytes = (size_t)w * h * 3 / 2;
    std::vector<unsigned char> buf(bytes * n);
    std::ifstream(argv[2], std::ios::binary).read((char *)buf.data(), buf.size());
    RetinaFaceOptions opt;
    opt.net_w = opt.net_h = 448;
    opt.model_file = "mnet25.caffemodel";
    RetinaFace rf(model, "net3", 0.4f, opt);
    rf.setVideoOrientation(0, 6);
    unsigned char *d = nullptr;
    if (cudaMalloc(&d, buf.size()) != cudaSuccess) return 2;
    cudaMemcpy(d, buf.data(), buf.size(), cudaMemcpyHostToDevice);
    RedactOptions ro;
    for (int s = 0; s < n; s += 2) {
        std::vector<rf_yuv_frame> frames;
        std::vector<int> videos;
        for (int i = s; i < s + 2 && i < n; i++) {
            unsigned char *y = d + bytes * i, *uv = y + (size_t)w * h;
            frames.push_back(rf_yuv_frame{y, uv, uv + 1, w, w, 2, w, h});
            videos.push_back(0);
        }
        rf.redactYUV(frames, &videos, 0.5f, ro);
    }
    cudaDeviceSynchronize();
    cudaMemcpy(buf.data(), d, buf.size(), cudaMemcpyDeviceToHost);
    std::ofstream(argv[3], std::ios::binary).write((const char *)buf.data(), buf.size());
    cudaFree(d);
    return 0;
}
'''


def test_host_shell_set_video_orientation_equals_c_calls(golden_image, tmp_path):
    """The C++ RetinaFace::setVideoOrientation + redactYUV gives the bytes of the same C calls."""
    import subprocess
    from conftest import ROOT
    from retinaface_b200.build import HERE, build_host
    from retinaface_b200 import Engine, RF_PREC_FP16
    build_host()
    S, _ = _video(golden_image, 6, "nv12", 4)
    (tmp_path / "in.bin").write_bytes(b"".join(f.tobytes() for f in S))
    src = tmp_path / "user.cpp"
    src.write_text(CPP_PROGRAM)
    exe = tmp_path / "user"
    cuda = "/usr/local/cuda"
    hostdir = os.path.join(HERE, "host")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", hostdir, "-I", os.path.join(ROOT, "include"), "-I", cuda + "/include", str(src),
                           os.path.join(hostdir, "RetinaFace.cpp"), "-o", str(exe), "-L", HERE, "-lrf_b200", "-L", cuda + "/lib64", "-lcudart",
                           "-Wl,-rpath," + HERE + ":" + cuda + "/lib64"])
    subprocess.check_call([str(exe), os.path.dirname(caffemodel("mnet25")), str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(len(S))])
    got = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.uint8).reshape(len(S), *S[0].shape)
    eng = Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP16, max_batch=8, max_faces=256, max_image=(3072, 4096), network="net3")
    try:
        trk = eng.tracker(max_videos=16)
        trk.set_orientation(0, 6)
        dev = [_cuda(f) for f in S]
        for s in (0, 2):
            trk.detect_yuv_redact_device(dev[s:s + 2], [0, 0], 0.5, 0.4)
        eng.synchronize()
        want = [d.cpu().numpy() for d in dev]
        trk.close()
    finally:
        eng.close()
    assert any(not np.array_equal(g, f) for g, f in zip(got, S))
    for i in range(len(S)):
        assert np.array_equal(got[i], want[i]), i


# ---- every other kind: {2, 5, 6, 8} across FP32 / FP16 / INT8, NV12 / I420 and BT.601 / BT.709 ------------------------------------------
KINDS = ["best", "motion", "follow", "lookback", "lookback_search", "lookback_follow"]
PRECS = ["fp32", "fp16", "int8"]
LAYOUTS = [("nv12", "bt601"), ("i420", "bt709")]


@pytest.fixture(scope="module")
def engines():
    made = {}

    def get(prec):
        if prec not in made:
            made[prec] = _engine(prec)
        return made[prec]
    yield get
    for e in made.values():
        e.close()


def _make(e, kind):
    return {"best": lambda: e.tracker(best={}), "motion": lambda: e.tracker(motion=True), "follow": lambda: e.tracker(follow=True),
            "lookback": lambda: e.tracker(lookback=15), "lookback_search": lambda: e.tracker(lookback=15, lookback_search=True),
            "lookback_follow": lambda: e.tracker(lookback=4, lookback_follow=True)}[kind]()


def _kind_run(e, t, kind, frames, outs, layout, matrix):
    """kind's calls over the device frames of video 0 on tracker t; returns every host result in call order.  outs: look-back out frames."""
    import torch
    kw = dict(layout=layout, matrix=matrix)
    n, res = len(frames), []

    def lists(tp, tc, m):
        return _bytes(t.read(tp, tc, m))
    if kind == "best":
        crops = torch.zeros((2, t.max_tracks, 112, 112, 3), dtype=torch.uint8, device="cuda")
        mats = torch.zeros((2, t.max_tracks, 6), dtype=torch.float64, device="cuda")
        for c in range(0, n, 2):
            r = t.detect_yuv_best_device(frames[c:c + 2], [0, 0], THR, NMS, crops.data_ptr(), mats.data_ptr(), **kw)
            e.synchronize()
            res.append((_bytes(t.read_best(r[0], r[1], 2)), crops.cpu().numpy().tobytes(), mats.cpu().numpy().tobytes(), lists(r[2], r[3], 2),
                        _bytes(e.read_dets(r[4], r[5], 2)[0]), r[6].tobytes()))
        crops.zero_()
        torch.cuda.synchronize()
        bp, bc = t.finish(0, crops.data_ptr(), mats.data_ptr())
        e.synchronize()
        shots = t.read_best(bp, bc, 1)
        assert len(shots[0]) > 0
        res.append((_bytes(shots), crops[0].cpu().numpy().tobytes(), mats[0].cpu().numpy().tobytes()))
    elif kind == "motion":
        for c in range(0, n, 2):
            r = t.detect_yuv_device(frames[c:c + 2], [0, 0], THR, NMS, **kw)
            e.synchronize()
            m = t.motion(2)
            res.append((m.tobytes(), lists(r[0], r[1], 2), r[4].tobytes()))
        assert m["blocks"].any(), m                   # the estimate matched blocks of the shaking scene
    elif kind == "follow":
        for c in range(n):                            # detect every 3rd frame, follow the others (k = 3)
            if c % 3 == 0:
                r = t.detect_yuv_device(frames[c:c + 1], [0], THR, NMS, **kw)
                tp, tc = r[0], r[1]
            else:
                tp, tc = t.follow_redact_device(frames[c:c + 1], [0], layout=layout, style="blur", shape="ellipse")
            e.synchronize()
            k = len(t.read(tp, tc, 1)[0])         # the follow records of the list; the rest of the row is not written
            res.append((lists(tp, tc, 1), t.follow(1)[0, :k].tobytes() if c % 3 else b""))
    else:
        L = 4 if kind == "lookback_follow" else 15
        for c in range(0, n, 2):
            if kind == "lookback_follow" and (c // 2) % 5:          # detect every 5th call (k = 5), follow the others
                nums, tp, tc = t.follow_redact_lookback_device(frames[c:c + 2], [0, 0], outs[c:c + 2], layout=layout, style="blur")
            else:
                nums, tp, tc, d, cc, sc = t.detect_yuv_redact_lookback_device(frames[c:c + 2], [0, 0], outs[c:c + 2], THR, NMS, style="blur", **kw)
            e.synchronize()
            step = ()
            if kind == "lookback_search":         # each chain's steps up to its length; the rest is not written
                st, ln = t.lookback_search(2)
                step = (b"".join(st[i, r, :ln[i, r]].tobytes() for i in range(2) for r in range(st.shape[1])), ln.tobytes())
            res.append((nums.tobytes(), lists(tp, tc, 2)) + step)
        if kind == "lookback_search":
            assert any(np.frombuffer(r[3], np.int32).any() for r in res), "no chain was searched"
        drained = [o.clone() for o in outs[:L]]
        torch.cuda.synchronize()
        res.append((t.drain(0, drained, layout=layout, style="blur").tobytes(),))
        outs.extend(drained)
    return res


@pytest.mark.parametrize("o", SOME)
@pytest.mark.parametrize("kind", KINDS)
def test_every_kind_equals_its_twin(engines, golden_image, kind, o):
    i = KINDS.index(kind) + SOME.index(o)
    prec, (layout, matrix) = PRECS[i % 3], LAYOUTS[i % 2]
    e = engines(prec)
    n = {"best": 6, "motion": 8, "follow": 7, "lookback": 20, "lookback_search": 20, "lookback_follow": 20}[kind]
    blank = 4 if kind.startswith("lookback") else 0         # faces born after the buffer holds frames: look-back has work
    S, D = _video(golden_image, o, layout, n, blank=blank, shake=kind == "motion")
    got = []
    for t_o, frames in ((o, S), (1, D)):
        t = _make(e, kind)
        t.set_orientation(0, t_o)
        dev = [_cuda(f) for f in frames]
        outs = [_cuda(np.zeros_like(f)) for f in frames]
        r = _kind_run(e, t, kind, dev, outs, layout, matrix)
        state = t.debug_state(0)
        e.synchronize()
        got.append((r, state, [d.cpu().numpy() for d in dev], [x.cpu().numpy() for x in outs]))
        t.close()
    (ra, sa, fa, oa), (rb, sb, fb, ob) = got
    assert ra == rb, (kind, o, prec)
    assert np.array_equal(sa[0], sb[0]) and np.array_equal(sa[1], sb[1]), (kind, o)
    for k in range(n):
        assert np.array_equal(orient_planes(fa[k], layout, o), fb[k]), (kind, o, "frame", k)
    for k in range(len(oa)):
        assert np.array_equal(orient_planes(oa[k], layout, o), ob[k]), (kind, o, "out", k)
    if kind.startswith("lookback"):
        assert any(not np.array_equal(x, d) for x, d in zip(ob[:n], D)), "nothing was redacted"


def test_portrait_video_with_interval_and_lookback_is_covered(golden_image):
    """The portrait phone video with look-back L = 4, detecting every frame and, on a following look-back tracker, every 3rd.  With
    the orientation the emitted frames equal the upright twin's, mapped back, and with detection on every frame every face the upright
    detector finds lies inside a written region of every emitted frame."""
    e = _engine("fp16")
    try:
        o, n, L = 6, 12, 4
        S, D = _video(golden_image, o, "nv12", n, w=1920, h=1080, scale=0.8)
        boxes = []
        for k in range(n):
            d, c, sc = e.detect_yuv_device([_cuda(D[k])], THR, NMS)
            boxes.append([tuple(float(v) * sc[0] for v in r[1:5]) for r in e.read_dets(d, c, 1)[0][0]])
        assert all(len(b) >= 1 for b in boxes)
        dh, dw = 1920, 1080
        for every in (1, 3):
            emitted = []
            for t_o, frames in ((o, S), (1, D)):
                t = e.tracker(lookback=L, lookback_follow=every > 1)
                t.set_orientation(0, t_o)
                dev = [_cuda(f) for f in frames]
                outs = [_cuda(np.zeros_like(f)) for f in frames]
                for k in range(n):
                    if k % every == 0:
                        t.detect_yuv_redact_lookback_device(dev[k:k + 1], [0], outs[k:k + 1], THR, NMS)
                    else:
                        t.follow_redact_lookback_device(dev[k:k + 1], [0], outs[k:k + 1])
                tail = [_cuda(np.zeros_like(frames[0])) for _ in range(L)]
                t.drain(0, tail)
                e.synchronize()
                emitted.append([x.cpu().numpy() for x in outs[L:] + tail])       # frame k, redacted
                t.close()
            shown = [orient_planes(x, "nv12", o) for x in emitted[0]]
            assert all(np.array_equal(a, b) for a, b in zip(shown, emitted[1])), every
            if every == 1:
                for k in range(n):
                    assert all(_covered(D[k][:dh], shown[k][:dh], boxes[k], dw, dh)), (every, k)
    finally:
        e.close()
