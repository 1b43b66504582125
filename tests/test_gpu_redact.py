"""GPU (-m gpu): f12 redaction -- rf_redact_yuv_device, rf_redact_device and rf_detect_yuv_redact_device against oracle/redact.py byte
for byte (every plane byte, pitch padding included) on detected and on synthetic records, the combined call against its parts, the LOST
tracks that close the detector's leak, tiled 4K records, calls in flight over the contexts, the refusals, and that nothing else
changes."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.redact import frame_regions, params, redact_bgr, redact_yuv
from oracle.yuv import bgr_to_frame

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
W, H = 1920, 1080
PITCH, UV_ROW = 2048, 1088          # an NVDEC surface: luma rows 2048 bytes apart, chroma from row 1088


def _engine(prec="fp16", **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (H, W))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


def _cuda(a):
    """A device copy, complete before the library's streams (which do not wait for torch's) read it."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def _clones(ts):
    import torch
    out = [t.clone() for t in ts]
    torch.cuda.synchronize()
    return out


def _canvas(golden, dx=0, dy=0, scale=1.0):
    img = np.full((H, W, 3), 128, np.uint8)
    g = golden if scale == 1.0 else cv2.resize(golden, None, fx=scale, fy=scale)
    img[40 + dy:40 + dy + g.shape[0], 100 + dx:100 + dx + g.shape[1]] = g
    return img


def _surface(bgr):
    """NV12 of bgr in an NVDEC-like surface (host), 0xEE padding."""
    buf = bgr_to_frame(bgr, "nv12")
    h, w = bgr.shape[:2]
    surf = np.full(PITCH * (UV_ROW + h // 2), 0xEE, np.uint8)
    surf[:h * PITCH].reshape(h, PITCH)[:, :w] = buf[:h]
    surf[PITCH * UV_ROW:].reshape(h // 2, PITCH)[:, :w] = buf[h:]
    return surf


def _planes(dev, h=H, w=W):
    return (dev[:h * PITCH].view(h, PITCH)[:, :w], dev[PITCH * UV_ROW:PITCH * UV_ROW + PITCH * h // 2].view(h // 2, PITCH)[:, :w])


SURF = dict(width=W, height=H, y_pitch=PITCH, uv_offset=PITCH * UV_ROW, uv_pitch=PITCH)


def _regions(recs, scales, blocks=0, margin=0.0, tracks=None):
    b, m = params(blocks, margin)
    return [frame_regions(r, len(r), None if scales is None else scales[i], m, b, tracks=None if tracks is None else tracks[i])
            for i, r in enumerate(recs)]


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_redaction_equals_the_oracle(golden_image, prec):
    """NV12 BT.601 surfaces (pitch 2048), I420 BT.709 buffers and strided BGR images of the golden photo on a 1080p canvas: detect with
    rf_detect_yuv_batch_device, redact, every byte equal to oracle/redact.py fed the fetched records and scales."""
    eng = _engine(prec)
    imgs = [_canvas(golden_image, 37 * k, 23 * k) for k in range(3)]
    surfs = [_surface(im) for im in imgs]
    dev = [_cuda(s) for s in surfs]
    frames = [_planes(d) for d in dev]
    d, c, sc = eng.detect_yuv_device(frames, THR, NMS, matrix="bt601")
    recs = eng.read_dets(d, c, 3)[0]
    assert all(len(r) >= 3 for r in recs)
    eng.redact_yuv_device(frames, d, c, sc)
    eng.synchronize()
    for k in range(3):
        want = redact_yuv(surfs[k], "nv12", _regions(recs, sc)[k], **SURF)
        assert np.array_equal(dev[k].cpu().numpy(), want), (prec, k)
        assert not np.array_equal(want, surfs[k])
    # I420 BT.709, blocks 1 / 32, margin 0.5
    bufs = [bgr_to_frame(im, "i420") for im in imgs]
    devi = [_cuda(b) for b in bufs]
    d, c, sc = eng.detect_yuv_device(devi, THR, NMS, layout="i420", matrix="bt709")
    recs = eng.read_dets(d, c, 3)[0]
    for blocks in (1, 32):
        eng.redact_yuv_device(devi, d, c, sc, layout="i420", blocks=blocks, margin=0.5)
        eng.synchronize()
        for k in range(3):
            bufs[k] = redact_yuv(bufs[k], "i420", _regions(recs, sc, blocks, 0.5)[k])
            assert np.array_equal(devi[k].cpu().numpy(), bufs[k]), (prec, blocks, k)
    # BGR rows 64 bytes beyond 3 w, the NV12 records
    d, c, sc = eng.detect_yuv_device(frames, THR, NMS)
    recs = eng.read_dets(d, c, 3)[0]
    big = [np.full((H, 3 * W + 64), 0xEE, np.uint8) for _ in imgs]
    for b, im in zip(big, imgs):
        b[:, :3 * W] = im.reshape(H, 3 * W)
    devb = [_cuda(b) for b in big]
    views = [t[:, :3 * W].view(H, W, 3) for t in devb]
    eng.redact_device(views, d, c, sc)
    eng.synchronize()
    for k in range(3):
        want = big[k].copy()
        want[:, :3 * W] = redact_bgr(imgs[k], _regions(recs, sc)[k]).reshape(H, 3 * W)
        assert np.array_equal(devb[k].cpu().numpy(), want), (prec, "bgr", k)
    eng.close()


def _det_array(boxes_per_frame, F):
    a = np.zeros((len(boxes_per_frame), F, 16), np.float32)
    counts = np.zeros(len(boxes_per_frame), np.int32)
    for i, boxes in enumerate(boxes_per_frame):
        for j, b in enumerate(boxes):
            a[i, j, 0] = 0.9
            a[i, j, 1:5] = b
        counts[i] = len(boxes)
    return a, counts


SYNTH = [[(100, 100, 300, 320), (250, 200, 420, 380), (50, 60, 50, 90), (70, 90, 40, 120), (np.nan, 10, 40, 50), (-1e6, -1e6, -9e5, 100),
          (1e6, 10, 2e6, 50), (-40.5, 300.25, 60.75, 381.5), (560.3, 330.1, 700.9, 420.0), (3.5, 3.5, 9.5, 9.5)],
         [(10, 10, 630, 350), (200, 100, 260, 170), (-1e9, -1e9, 1e9, 1e9)],
         []]


@pytest.mark.parametrize("blocks,margin", [(0, 0.0), (1, 0.1), (32, 1.0), (5, 0.33)])
def test_synthetic_records(blocks, margin):
    """Device rf_det arrays with overlaps, zero and negative widths, NaN, boxes beyond +-65536 and frame edges cutting cells, on I420 and
    BGR frames: identical bytes; the skipped boxes change nothing."""
    import torch
    eng = _engine("fp16", max_faces=16)
    rng = np.random.default_rng(blocks)
    w, h = 640, 360
    dets, counts = _det_array(SYNTH, eng.max_faces)
    scales = np.array([1.0, 1.5, 2.0], np.float32)
    dd, dc = _cuda(dets), _cuda(counts)
    bufs = [rng.integers(0, 256, (h * 3 // 2, w), dtype=np.uint8) for _ in range(3)]
    devi = [_cuda(b) for b in bufs]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(3)]
    devb = [_cuda(b) for b in imgs]
    eng.redact_yuv_device(devi, dd.data_ptr(), dc.data_ptr(), scales, layout="i420", blocks=blocks, margin=margin)
    eng.redact_device(devb, dd.data_ptr(), dc.data_ptr(), scales, blocks=blocks, margin=margin)
    eng.synchronize()
    recs = [dets[i, :counts[i], :15] for i in range(3)]
    regs = _regions(recs, scales, blocks, margin)
    for k in range(3):
        assert np.array_equal(devi[k].cpu().numpy(), redact_yuv(bufs[k], "i420", regs[k])), k
        assert np.array_equal(devb[k].cpu().numpy(), redact_bgr(imgs[k], regs[k])), k
    # the same frames with the skipped records removed: the same bytes
    keep = [[b for b in f if np.isfinite(b).all() and b[2] > b[0] and b[3] > b[1]] for f in SYNTH]
    dets2, counts2 = _det_array(keep, eng.max_faces)
    dd2, dc2 = _cuda(dets2), _cuda(counts2)
    devi2 = [_cuda(b) for b in bufs]
    eng.redact_yuv_device(devi2, dd2.data_ptr(), dc2.data_ptr(), scales, layout="i420", blocks=blocks, margin=margin)
    eng.synchronize()
    for a, b in zip(devi, devi2):
        assert torch.equal(a, b)
    eng.close()


def _moving(golden, n):
    return [_canvas(golden, 7 * t % 350, 3 * t % 150) for t in range(n)]


def test_combined_call_equals_its_parts(golden_image):
    """rf_detect_yuv_redact_device against rf_detect_yuv_batch_device + rf_redact_yuv_device, and with a tracker against
    rf_detect_yuv_track_device + the primitive: records, tracks and frames bit-equal."""
    import torch
    eng = _engine("fp16")
    imgs = _moving(golden_image, 12)
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    for s in range(0, 12, 4):
        d1, c1, s1 = eng.detect_yuv_redact_device(a[s:s + 4], THR, NMS, blocks=12, margin=0.3)
        r1 = eng.read_dets(d1, c1, 4)[0]
        d2, c2, s2 = eng.detect_yuv_device(b[s:s + 4], THR, NMS)
        r2 = eng.read_dets(d2, c2, 4)[0]
        eng.redact_yuv_device(b[s:s + 4], d2, c2, s2, blocks=12, margin=0.3)
        eng.synchronize()
        assert all(np.array_equal(x, y) for x, y in zip(r1, r2)) and np.array_equal(s1, s2)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    t1, t2 = eng.tracker(), eng.tracker()
    for s in range(0, 12, 3):
        tp1, tc1, d1, c1, s1 = t1.detect_yuv_redact_device(a[s:s + 3], [0] * 3, THR, NMS)
        tp2, tc2, d2, c2, s2 = t2.detect_yuv_device(b[s:s + 3], [0] * 3, THR, NMS)
        eng.redact_yuv_device(b[s:s + 3], d2, c2, s2, tracker=t2, tracks_ptr=tp2, track_counts_ptr=tc2)
        eng.synchronize()
        assert all(np.array_equal(x, y) for x, y in zip(eng.read_dets(d1, c1, 3)[0], eng.read_dets(d2, c2, 3)[0]))
        assert all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(t1.read(tp1, tc1, 3), t2.read(tp2, tc2, 3)))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    t1.close()
    t2.close()
    eng.close()


def test_tracking_closes_the_leak(golden_image):
    """The moving photo with the best face's record deleted from the device records on frames 5-7, through rf_track_update: with tracks
    its LOST track's predicted box is redacted, equal to the oracle; without tracks its pixels are the input's."""
    import torch
    from retinaface_b200.capi import device_view
    eng = _engine("fp16")
    trk = eng.tracker()
    imgs = _moving(golden_image, 10)
    leaked = 0
    for t, im in enumerate(imgs):
        buf = bgr_to_frame(im, "nv12")
        f1, f2 = _cuda(buf), _cuda(buf)
        d, c, sc = eng.detect_yuv_device([f1], THR, NMS)
        rec = eng.read_dets(d, c, 1)[0][0]
        if 5 <= t <= 7:             # the detector misses face 0 on these frames
            raw = device_view(d, (1, eng.max_faces, 16), "<f4")
            raw[0, :len(rec) - 1] = raw[0, 1:len(rec)].clone()
            device_view(c, (1,), "<i4").sub_(1)
            torch.cuda.synchronize()
            gone, rec = rec[0], rec[1:]
        tp, tc = trk.update([0], d, c, sc)
        eng.redact_yuv_device([f1], d, c, sc, tracker=trk, tracks_ptr=tp, track_counts_ptr=tc)
        eng.redact_yuv_device([f2], d, c, sc)
        eng.synchronize()
        tracks = trk.read(tp, tc, 1)[0]
        want = redact_yuv(buf, "nv12", _regions([rec], sc, tracks=[tracks])[0])
        assert np.array_equal(f1.cpu().numpy(), want), t
        assert np.array_equal(f2.cpu().numpy(), redact_yuv(buf, "nv12", _regions([rec], sc)[0])), t
        if 5 <= t <= 7:
            assert (tracks["state"] == 2).sum() >= 1, t
            x1, y1, x2, y2 = (int(v) for v in np.round(gone[1:5] * sc[0]))
            y = buf[:H]
            others = np.zeros((H, W), bool)
            for X0, Y0, X1, Y1, _ in _regions([rec], sc)[0]:
                others[max(Y0, 0):Y1, max(X0, 0):X1] = True
            face = np.zeros((H, W), bool)
            face[y1:y2, x1:x2] = True
            own = face & ~others
            assert own.sum() > 100
            assert np.array_equal(f2.cpu().numpy()[:H][own], y[own])          # the leak
            assert not np.array_equal(f1.cpu().numpy()[:H][own], y[own])      # closed by the LOST track
            leaked += 1
    assert leaked == 3
    trk.close()
    eng.close()


def test_tiled_4k_records(golden_image):
    """A 3840x2160 canvas of half-scale photos through rf_detect_yuv_tiled_device, redacted with scales = NULL: equal to the oracle, and
    every planted photo's faces redacted."""
    eng = _engine("fp16", max_image=(2160, 3840))
    half = cv2.resize(golden_image, None, fx=0.5, fy=0.5)
    img = np.full((2160, 3840, 3), 128, np.uint8)
    spots = [(200, 150), (2000, 300), (900, 1300), (2900, 1500)]
    for x, y in spots:
        img[y:y + half.shape[0], x:x + half.shape[1]] = half
    buf = bgr_to_frame(img, "nv12")
    dev = _cuda(buf)
    d, c = eng.detect_yuv_tiled_device([dev], THR, NMS)
    rec = eng.read_dets(d, c, 1)[0][0]
    eng.redact_yuv_device([dev], d, c, None)
    eng.synchronize()
    out = dev.cpu().numpy()
    assert np.array_equal(out, redact_yuv(buf, "nv12", _regions([rec], None)[0]))
    for x, y in spots:
        inside = [r for r in rec if x <= r[1] and r[3] <= x + half.shape[1] and y <= r[2] and r[4] <= y + half.shape[0]]
        assert len(inside) >= 3, (x, y)
        for r in inside:
            x1, y1, x2, y2 = (int(v) for v in r[1:5])
            assert not np.array_equal(out[y1:y2, x1:x2], buf[y1:y2, x1:x2])
    eng.close()


@pytest.mark.parametrize("streams", [2, 8])
def test_calls_in_flight(golden_image, streams):
    """2 streams + 1 combined calls in flight, each on its own frames, against the same calls synchronised one by one: bit-equal."""
    import torch
    eng = _engine("fp16", streams=streams)
    k = 2 * streams + 1
    imgs = _moving(golden_image, 4 * k)
    a = [_cuda(bgr_to_frame(im, "nv12")) for im in imgs]
    b = _clones(a)
    for s in range(k):
        eng.detect_yuv_redact_device(a[4 * s:4 * s + 4], THR, NMS)
    eng.synchronize()
    for s in range(k):
        eng.detect_yuv_redact_device(b[4 * s:4 * s + 4], THR, NMS)
        eng.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    eng.close()


def test_invalid_arguments_launch_nothing(golden_image):
    import torch
    from retinaface_b200 import capi
    eng = _engine("fp16", max_batch=2)
    other = _engine("fp16", max_batch=2)
    lib = eng.lib
    buf = bgr_to_frame(_canvas(golden_image), "nv12")
    f = [_cuda(buf), _cuda(buf)]
    d, c, sc = eng.detect_yuv_device(f, THR, NMS)
    eng.synchronize()
    before = _clones(f)
    trk, otrk = eng.tracker(), other.tracker()
    tp, tc = trk.update([0, 0], d, c, sc)
    best = eng.tracker(best={})

    def arr(frames):
        return eng._frames(frames, "nv12", True)

    def red(frames, n=None, scales=sc, t=None, tracks=None, counts=None, blocks=0, margin=0.0, dets=d):
        s = None if scales is None else np.ascontiguousarray(scales, np.float32)
        p = capi.RedactParams(blocks, margin)
        return lib.rf_redact_yuv_device(eng.h, arr(frames), len(frames) if n is None else n, dets, c, s.ctypes.data if s is not None else None,
                                        t, tracks, counts, C.byref(p))

    odd = (f[1][:H].view(H, W)[:, :W - 2], f[1][H:].view(H // 2, W)[:, :W - 2])
    odd = capi.yuv_frame(odd, "nv12")[0]
    odd.width = W - 1
    cases = [
        ("n > max_batch", lib.rf_redact_yuv_device(eng.h, arr([f[0]] * 3), 3, d, c, None, None, None, None, None), -6),
        ("blocks 33", red(f, blocks=33), -1), ("blocks -1", red(f, blocks=-1), -1),
        ("margin 1.5", red(f, margin=1.5), -1), ("margin -0.5", red(f, margin=-0.5), -1), ("margin nan", red(f, margin=float("nan")), -1),
        ("tracker of another handle", red(f, t=otrk.t, tracks=tp, counts=tc), -1),
        ("tracks without the tracker", red(f, tracks=tp, counts=tc), -1),
        ("tracker without tracks", red(f, t=trk.t), -1),
        ("scale 0", red(f, scales=[1.0, 0.0]), -1), ("scale nan", red(f, scales=[float("nan"), 1.0]), -1),
        ("scale -1", red(f, scales=[-1.0, 1.0]), -1),
        ("overlapping frames", red([f[0], f[0]]), -1),
        ("NULL records", red(f, dets=None), -1),
        ("odd width", lib.rf_redact_yuv_device(eng.h, (capi.YuvFrame * 1)(odd), 1, d, c, None, None, None, None, None), -1),
    ]
    ptr1 = (C.c_void_p * 1)(f[0].data_ptr())
    cases.append(("bgr stride below 3 w", lib.rf_redact_device(eng.h, ptr1, (C.c_int * 1)(64), (C.c_int * 1)(8), (C.c_int * 1)(100), 1, d, c, None,
                                                               None, None, None, None), -1))
    ptrs2 = (C.c_void_p * 2)(f[0].data_ptr(), f[0].data_ptr() + 10)
    cases.append(("bgr overlap", lib.rf_redact_device(eng.h, ptrs2, (C.c_int * 2)(64, 64), (C.c_int * 2)(8, 8), None, 2, d, c, None, None, None,
                                                      None, None), -1))
    canary = 0x5EED
    outs = [C.c_void_p(canary) for _ in range(4)]
    scales_out = np.full(2, 7.0, np.float32)
    cases.append(("best-shot tracker", lib.rf_detect_yuv_redact_device(eng.h, best.t, arr(f), (C.c_int * 2)(0, 0), 2, 0, THR, NMS, None,
                                                                       *(C.byref(o) for o in outs), scales_out.ctypes.data), -1))
    cases.append(("combined: bad blocks", lib.rf_detect_yuv_redact_device(eng.h, None, arr(f), None, 2, 0, THR, NMS,
                                                                          C.byref(capi.RedactParams(40, 0.0)), *(C.byref(o) for o in outs),
                                                                          scales_out.ctypes.data), -1))
    cases.append(("combined: overlapping frames", lib.rf_detect_yuv_redact_device(eng.h, None, arr([f[0], f[0]]), None, 2, 0, THR, NMS, None,
                                                                                  *(C.byref(o) for o in outs), scales_out.ctypes.data), -1))
    cases.append(("combined: tracker without videos", lib.rf_detect_yuv_redact_device(eng.h, trk.t, arr(f), None, 2, 0, THR, NMS, None,
                                                                                      *(C.byref(o) for o in outs), scales_out.ctypes.data), -1))
    cases.append(("combined: n > max_batch", lib.rf_detect_yuv_redact_device(eng.h, None, arr([f[0]] * 3), None, 3, 0, THR, NMS, None,
                                                                             *(C.byref(o) for o in outs), scales_out.ctypes.data), -6))
    eng.synchronize()
    for what, rc, want in cases:
        assert rc == want, (what, rc, lib.rf_last_error(eng.h))
    assert all(torch.equal(x, y) for x, y in zip(f, before))
    assert all(o.value == canary for o in outs) and (scales_out == 7.0).all()
    for t in (trk, otrk, best):
        t.close()
    other.close()
    eng.close()


def test_nothing_else_changes(golden_image):
    """rf_detect_batch, rf_detect_yuv_batch_device and rf_launches_per_batch are the same before and after redaction calls."""
    eng = _engine("fp16")
    inp = cv2.resize(golden_image, (448, 448))
    buf = bgr_to_frame(_canvas(golden_image), "nv12")

    def snapshot():
        faces = eng.detect_batch([inp, inp], THR, NMS)
        d, c, sc = eng.detect_yuv_device([_cuda(buf)], THR, NMS)
        return faces, eng.read_dets(d, c, 1)[0], sc, eng.launches_per_batch(8)

    a = snapshot()
    for blocks in (1, 8, 32):
        eng.detect_yuv_redact_device([_cuda(buf), _cuda(buf)], THR, NMS, blocks=blocks)
    eng.synchronize()
    b = snapshot()
    assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and np.array_equal(a[1][0], b[1][0]) and np.array_equal(a[2], b[2])
    assert a[3] == b[3]
    eng.close()


def test_detector_redact_frames(golden_image):
    """RetinaFace.redactFrames: the combined call, with and without tracking."""
    import torch
    from retinaface_b200.detector import RetinaFace
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    eng = det.engine
    buf = bgr_to_frame(_canvas(golden_image), "nv12")
    a, b = _cuda(buf), _cuda(buf)
    det.redactFrames([a], threshold=THR)
    d, c, sc = eng.detect_yuv_device([b], THR, det.nms_threshold)
    eng.redact_yuv_device([b], d, c, sc)
    eng.synchronize()
    assert torch.equal(a, b) and not np.array_equal(a.cpu().numpy(), buf)
    v = _cuda(buf)
    det.redactFrames([v], videos=[0], threshold=THR)
    eng.synchronize()
    assert torch.equal(v, b)
