"""GPU (-m gpu): f11 best shots -- rf_detect_yuv_track_best_device and rf_tracker_finish against oracle/bestshot.py bit for bit (every
emitted record, crop and M), the behaviour on a synthetic 30-frame 1080p video (blurred except a sharp window, an occluded face, a
face entering across the right edge, a face shown on one frame), the float formats, unchanged tracks, the ordering rules and the
refusals."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.align import blob
from oracle.bestshot import BEST_EXIT, BEST_FINISH, BestShotOracle
from oracle.track import TrackerOracle
from oracle.yuv import bgr_to_frame, frame_to_bgr

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
W, H, NF = 1920, 1080, 30
X0, Y0 = 100, 40
SHARP = range(10, 15)
OCCLUDE_FROM, MAX_LOST = 17, 3
ENTER_FROM, ONE_FRAME = 2, 6
SHOT_INTS = ("id", "video", "frame", "end_frame", "hits", "age", "reason", "reserved")
SHOT_FLOATS = ("quality", "score", "eye", "frontal", "sharpness", "coverage")


def _engine(prec="fp16", **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (H, W))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def video(golden_image):
    """30 NV12 frames: the golden photo moving (3, 1) px per frame on grey, GaussianBlur(sigma 2) on every frame outside SHARP, a grey
    occluder over its best face from OCCLUDE_FROM on, a 2x copy of that face entering across the right edge from ENTER_FROM (4 px
    per frame to the left) and another 2x copy, below it, shown on frame ONE_FRAME only.  Returns (nv12 frames, bgr frames)."""
    eng = _engine("fp32")
    faces = eng.detect_batch([golden_image], 0.8, NMS)[0]
    eng.close()
    sc = max(golden_image.shape[1] / 448, golden_image.shape[0] / 448, 1.0)
    x1, y1, x2, y2 = (faces[0, 1:5] * sc).astype(int)
    face = golden_image[max(y1 - 20, 0):y2 + 20, max(x1 - 20, 0):x2 + 20]
    big = cv2.resize(face, (face.shape[1] * 2, face.shape[0] * 2))
    frames, bgr = [], []
    for t in range(NF):
        img = np.full((H, W, 3), 128, np.uint8)
        ox, oy = X0 + 3 * t, Y0 + t
        img[oy:oy + golden_image.shape[0], ox:ox + golden_image.shape[1]] = golden_image
        if t >= OCCLUDE_FROM:
            img[oy + y1 - 10:oy + y2 + 10, ox + x1 - 10:ox + x2 + 10] = 128
        if t >= ENTER_FROM:
            fx = W - big.shape[1] + 40 - 4 * (t - ENTER_FROM)
            cols = min(big.shape[1], W - fx)
            img[200:200 + big.shape[0], fx:fx + cols] = big[:, :cols]
        if t == ONE_FRAME:
            img[H - big.shape[0] - 10:H - 10, 1450:1450 + big.shape[1]] = big
        if t not in SHARP:
            img = cv2.GaussianBlur(img, (0, 0), 2)
        frames.append(bgr_to_frame(img, "nv12"))
        bgr.append(frame_to_bgr(frames[-1], "nv12"))
    return frames, bgr


def _best_run(eng, trk, dev, per_call, crops, mats=None, videos=None):
    """The frames through rf_detect_yuv_track_best_device, per_call per call; per frame (shots, tracks, records, scale)."""
    out = []
    for s in range(0, len(dev), per_call):
        chunk = dev[s:s + per_call]
        vids = videos[s:s + per_call] if videos is not None else [0] * len(chunk)
        bp, bc, tp, tc, d, c, sc = trk.detect_yuv_best_device(chunk, vids, THR, NMS, crops[s:s + per_call].data_ptr(),
                                                               mats[s:s + per_call].data_ptr() if mats is not None else None)
        shots = trk.read_best(bp, bc, len(chunk))
        tracks = trk.read(tp, tc, len(chunk))
        recs = eng.read_dets(d, c, len(chunk))[0]
        out += [(shots[i], tracks[i], recs[i], sc[i]) for i in range(len(chunk))]
    return out


def _same_shot(r, w, what):
    for f in SHOT_INTS:
        assert int(r[f]) == int(w[f]), (what, f, int(r[f]), int(w[f]))
    for f in SHOT_FLOATS:
        assert np.float32(r[f]).tobytes() == np.float32(w[f]).tobytes(), (what, f, r[f], w[f])
    assert np.array_equal(np.asarray(r["face"], np.float32).view(np.uint32), np.asarray(w["face"], np.float32).view(np.uint32)), what


def _oracle_video(eng, dev, bgr, min_quality=0.0):
    """oracle/bestshot.py fed TrackerOracle and the crops / matrices rf_detect_yuv_batch_device cuts for every record."""
    import torch
    mf = eng.max_faces
    to, bo = TrackerOracle(1, max_lost=MAX_LOST), BestShotOracle(min_quality=min_quality)
    per_frame, seen = [], []
    for t in range(len(dev)):
        crops = torch.zeros((1, mf, 112, 112, 3), dtype=torch.uint8, device="cuda")
        mats = torch.zeros((1, mf, 6), dtype=torch.float64, device="cuda")
        d, c, sc = eng.detect_yuv_device([dev[t]], THR, NMS, align=dict(), dev_crops_ptr=crops.data_ptr(), dev_mats_ptr=mats.data_ptr())
        recs = eng.read_dets(d, c, 1)[0][0]
        tracks = to.update(0, recs, sc[0])
        cr, mt = crops[0].cpu().numpy(), mats[0].cpu().numpy()
        per_frame.append(bo.update(0, tracks, cr, mt, W, H))
        seen.append({t_["id"]: bo.v[0]["best"].get(t_["id"]) for t_ in tracks})
    return per_frame, bo.finish(0), seen


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_shots_equal_the_oracle(video, prec):
    """Every emitted record equals the oracle's bit for bit, each u8 crop is the crop of the matched record on its frame and
    cv2.warpAffine(cvtColor(frame), M), M bit-equal; finish emits the rest, and the next frame's ids restart at 1."""
    import torch
    frames, bgr = video
    dev = [_cuda(f) for f in frames]
    eng = _engine(prec)
    want, want_fin, _ = _oracle_video(eng, dev, bgr)
    trk = eng.tracker(max_lost=MAX_LOST, best=dict())
    T = trk.max_tracks
    crops = torch.full((NF, T, 112, 112, 3), 0xA5, dtype=torch.uint8, device="cuda")
    mats = torch.zeros((NF, T, 6), dtype=torch.float64, device="cuda")
    got = _best_run(eng, trk, dev, 8, crops, mats)
    crops_h, mats_h = crops.cpu().numpy(), mats.cpu().numpy()
    emitted = 0
    for t, (shots, _, _, _) in enumerate(got):
        assert len(shots) == len(want[t]), (prec, t, [int(s["id"]) for s in shots], [w["id"] for w in want[t]])
        for k, (s, w) in enumerate(zip(shots, want[t])):
            _same_shot(s, w, f"{prec} frame {t}")
            assert np.array_equal(crops_h[t, k], w["crop"]), (prec, t, k)
            assert mats_h[t, k].tobytes() == w["M"].reshape(6).tobytes(), (prec, t, k)
            ref = cv2.warpAffine(bgr[int(s["frame"])], mats_h[t, k].reshape(2, 3), (112, 112), flags=cv2.INTER_LINEAR,
                                 borderMode=cv2.BORDER_CONSTANT, borderValue=0)
            assert np.array_equal(crops_h[t, k], ref), (prec, t, k)
            emitted += 1
        assert (crops_h[t, len(shots):] == 0xA5).all(), t
    fc = torch.full((T, 112, 112, 3), 0x5A, dtype=torch.uint8, device="cuda")
    fm = torch.zeros((T, 6), dtype=torch.float64, device="cuda")
    bp, bc = trk.finish(0, fc.data_ptr(), fm.data_ptr())
    fin = trk.read_best(bp, bc, 1)[0]
    assert len(fin) == len(want_fin) >= 3
    for k, (s, w) in enumerate(zip(fin, want_fin)):
        _same_shot(s, w, f"{prec} finish")
        assert np.array_equal(fc[k].cpu().numpy(), w["crop"]) and fm[k].cpu().numpy().tobytes() == w["M"].reshape(6).tobytes()
    assert emitted >= 1
    # the video restarted: ids from 1
    _, _, tp, tc, _, _, _ = trk.detect_yuv_best_device([dev[0]], [0], THR, NMS, crops.data_ptr())
    ids = [int(r["id"]) for r in trk.read(tp, tc, 1)[0]]
    assert ids == list(range(1, len(ids) + 1))
    trk.close()
    eng.close()


def test_behaviour_on_the_synthetic_video(video):
    import torch
    frames, bgr = video
    dev = [_cuda(f) for f in frames]
    eng = _engine("fp16")
    _, _, seen = _oracle_video(eng, dev, bgr)
    trk = eng.tracker(max_lost=MAX_LOST, best=dict())
    T = trk.max_tracks
    crops = torch.zeros((NF, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
    got = _best_run(eng, trk, dev, 4, crops)
    first = [int(r["id"]) for r in got[0][1]]
    assert len(first) >= 3
    exits = {int(s["id"]): (t, s) for t, (shots, _, _, _) in enumerate(got) for s in shots}
    # the occluded face: emitted with reason EXIT on exactly its removal frame (lost from OCCLUDE_FROM, removed past max_lost)
    occluded = [i for i in first if any(int(r["id"]) == i and r["det"] < 0 for r in got[OCCLUDE_FROM][1])]
    assert occluded
    for i in occluded:
        t, s = exits[i]
        assert t == OCCLUDE_FROM + MAX_LOST and int(s["end_frame"]) == t and int(s["reason"]) == BEST_EXIT, (i, t)
        assert not any(int(r["id"]) == i for r in got[t][1]) and any(int(r["id"]) == i for r in got[t - 1][1])
    fc = torch.zeros((T, 112, 112, 3), dtype=torch.uint8, device="cuda")
    bp, bc = trk.finish(0, fc.data_ptr())
    fin = trk.read_best(bp, bc, 1)[0]
    assert [int(s["id"]) for s in fin] == sorted(int(s["id"]) for s in fin)
    assert all(int(s["reason"]) == BEST_FINISH and int(s["end_frame"]) == NF - 1 for s in fin)
    shots = {int(s["id"]): s for s in fin}
    shots.update({i: s for i, (_, s) in exits.items()})
    # every first-frame face's shot comes from the sharp window
    for i in first:
        assert int(shots[i]["frame"]) in SHARP, (i, int(shots[i]["frame"]))
    # the entering face: born at the right edge with coverage < 1, its shot is fully inside
    entering = [int(r["id"]) for t in range(ENTER_FROM, ENTER_FROM + 6) for r in got[t][1]
                if int(r["id"]) not in first and r["face"][1] > 1500 and r["face"][2] < 700]
    assert entering, "the entering face was never tracked"
    e = entering[0]
    first_seen = min(t for t in range(NF) if e in seen[t])
    assert seen[first_seen][e]["coverage"] < 1.0
    assert e in shots and float(shots[e]["coverage"]) == 1.0
    # the one-frame face is never emitted
    one = [int(r["id"]) for r in got[ONE_FRAME][1] if int(r["id"]) not in first and r["face"][2] > 700]
    assert one and not any(i in shots for i in one)
    trk.close()
    # min_quality = 1 emits nothing
    trk = eng.tracker(max_lost=MAX_LOST, best=dict(min_quality=1.0))
    got = _best_run(eng, trk, dev, 8, crops)
    assert all(len(s) == 0 for s, _, _, _ in got)
    bp, bc = trk.finish(0, fc.data_ptr())
    assert len(trk.read_best(bp, bc, 1)[0]) == 0
    trk.close()
    eng.close()


def test_float_formats_and_unchanged_tracks(video):
    """F32 / F16 shots are blob() of the u8 shot (F16 = F32 rounded); the best call's tracks, records and scales equal a plain
    tracker's rf_detect_yuv_track_device bit for bit."""
    import torch
    frames, _ = video
    dev = [_cuda(f) for f in frames]
    eng = _engine("fp16")
    res = {}
    for fmt, dt, shape in (("bgr_u8", torch.uint8, (112, 112, 3)), ("rgb_f32", torch.float32, (3, 112, 112)),
                           ("rgb_f16", torch.float16, (3, 112, 112))):
        trk = eng.tracker(max_lost=MAX_LOST, best=dict(fmt=fmt))
        crops = torch.zeros((NF, trk.max_tracks) + shape, dtype=dt, device="cuda")
        got = _best_run(eng, trk, dev, 8, crops)
        fc = torch.zeros((trk.max_tracks,) + shape, dtype=dt, device="cuda")
        bp, bc = trk.finish(0, fc.data_ptr())
        fin = trk.read_best(bp, bc, 1)[0]
        out = [crops[t, k].cpu().numpy() for t, (s, _, _, _) in enumerate(got) for k in range(len(s))] + \
              [fc[k].cpu().numpy() for k in range(len(fin))]
        res[fmt] = (out, got)
        trk.close()
    u8 = np.array(res["bgr_u8"][0])
    assert len(u8) >= 3
    f32 = blob(u8)
    assert np.array_equal(np.array(res["rgb_f32"][0]).view(np.uint32), f32.view(np.uint32))
    assert np.array_equal(np.array(res["rgb_f16"][0]).view(np.uint16), f32.astype(np.float16).view(np.uint16))
    plain = eng.tracker(max_lost=MAX_LOST)
    for s in range(0, NF, 8):
        chunk = dev[s:s + 8]
        tp, tc, d, c, sc = plain.detect_yuv_device(chunk, [0] * len(chunk), THR, NMS)
        tr, recs = plain.read(tp, tc, len(chunk)), eng.read_dets(d, c, len(chunk))[0]
        for i in range(len(chunk)):
            _, btr, brec, bsc = res["bgr_u8"][1][s + i]
            assert btr.tobytes() == tr[i].tobytes() and np.array_equal(brec, recs[i]) and bsc == sc[i], s + i
    plain.close()
    eng.close()


def _shot_bytes(got, crops):
    return [(s.tobytes(), crops[t, :len(s)].cpu().numpy().tobytes()) for t, (s, _, _, _) in enumerate(got)]


def test_ordering_rules(video, golden_image):
    import torch
    frames, _ = video
    dev = [_cuda(f) for f in frames]
    eng = _engine("fp16")
    T = 64
    # 8 frames per call == 1 frame per call
    a, b = eng.tracker(max_lost=MAX_LOST, best=dict()), eng.tracker(max_lost=MAX_LOST, best=dict())
    ca = torch.zeros((NF, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
    cb = torch.zeros_like(ca)
    assert _shot_bytes(_best_run(eng, a, dev, 8, ca), ca) == _shot_bytes(_best_run(eng, b, dev, 1, cb), cb)
    a.close()
    b.close()
    # 8 videos in one call == 8 calls (video v starts v frames in)
    a, b = eng.tracker(max_videos=8, max_lost=MAX_LOST, best=dict()), eng.tracker(max_videos=8, max_lost=MAX_LOST, best=dict())
    one, sep = [], []
    for s in range(0, NF - 8):
        fr = [dev[v + s] for v in range(8)]
        c8 = torch.zeros((8, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
        one += _shot_bytes(_best_run(eng, a, fr, 8, c8, videos=list(range(8))), c8)
        for v in range(8):
            c1 = torch.zeros((1, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
            sep += _shot_bytes(_best_run(eng, b, [fr[v]], 1, c1, videos=[v]), c1)
    assert one == sep and any(x[0] for x in one)
    a.close()
    b.close()
    eng.close()
    # a slot freed and reused on one frame inside one call: face A on frames 0-3, nothing on 4, face B elsewhere on 5-7; with
    # max_lost 1, A is removed on frame 5 (emitting its frame-0..3 scratch crop) as B is born into its slot
    x1, y1 = 300, 300
    crop_a = golden_image[100:500, 200:600]
    seq = []
    for t in range(8):
        img = np.full((H, W, 3), 128, np.uint8)
        if t <= 3:
            img[y1:y1 + 400, x1:x1 + 400] = crop_a
        if t >= 5:
            img[500:900, 1300:1700] = crop_a
        seq.append(_cuda(bgr_to_frame(img, "nv12")))
    eng = _engine("fp16")
    runs = []
    for per_call in (8, 1):
        k = eng.tracker(max_lost=1, max_tracks=8, best=dict())
        cr = torch.zeros((8, 8, 112, 112, 3), dtype=torch.uint8, device="cuda")
        got = _best_run(eng, k, seq, per_call, cr)
        runs.append(_shot_bytes(got, cr))
        if per_call == 8:
            assert len(got[5][0]) >= 1 and all(int(s["frame"]) <= 3 and int(s["end_frame"]) == 5 for s in got[5][0])
        k.close()
    assert runs[0] == runs[1]
    eng.close()
    # 2 * streams + 1 calls in flight on streams 2 and 8 == the same calls synchronised one by one
    for streams in (2, 8):
        res = []
        for sync in (False, True):
            e = _engine("fp16", streams=streams)
            k = e.tracker(max_videos=2, max_lost=MAX_LOST, best=dict())
            n_calls = 2 * streams + 1
            cr = torch.zeros((n_calls, 2, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
            ptrs = []
            for i in range(n_calls):
                ptrs.append(k.detect_yuv_best_device([dev[i % NF], dev[NF - 1 - i % NF]], [0, 1], THR, NMS, cr[i].data_ptr()))
                if sync:
                    e.synchronize()
            bp, bc = ptrs[-1][:2]
            fc = torch.zeros((T, 112, 112, 3), dtype=torch.uint8, device="cuda")
            fp, fcnt = k.finish(0, fc.data_ptr())
            last = k.read_best(bp, bc, 2)
            fin = k.read_best(fp, fcnt, 1)[0]
            res.append(([x.tobytes() for x in last], fin.tobytes(), fc[:len(fin)].cpu().numpy().tobytes(), cr.cpu().numpy().tobytes()))
            k.close()
            e.close()
        assert res[0] == res[1], streams


def test_refusals_and_isolation(video, golden_image):
    import torch
    from retinaface_b200 import capi
    frames, _ = video
    dev = [_cuda(f) for f in frames[:2]]
    eng = _engine("fp16")
    base = eng.detect_batch([golden_image], THR, NMS)[0]
    plain = eng.tracker(max_videos=2)
    tp, tc, _, _, _ = plain.detect_yuv_device(dev, [0, 1], THR, NMS)
    plain_tracks = plain.read(tp, tc, 2)
    plain.close()
    launches = eng.launches_per_batch(2)
    lib = eng.lib
    trk = eng.tracker(max_videos=2, best=dict())
    crops = torch.zeros((2, trk.max_tracks, 112, 112, 3), dtype=torch.uint8, device="cuda")
    trk.detect_yuv_best_device(dev, [0, 1], THR, NMS, crops.data_ptr())
    state = [trk.debug_state(v)[0].tobytes() + trk.debug_state(v)[1].tobytes() for v in (0, 1)]
    arr = eng._frames(dev, "nv12", True)
    vids, bad_v = (C.c_int * 2)(0, 1), (C.c_int * 2)(0, 2)
    outs = [C.c_void_p(0x1000 + k) for k in range(6)]

    def call(t, v, n, m, cr):
        return lib.rf_detect_yuv_track_best_device(eng.h, t, arr, v, n, m, THR, NMS, cr, None, *[C.byref(o) for o in outs], None)
    cp = crops.data_ptr()
    for args, status in (((trk.t, bad_v, 2, 0, cp), -1), ((trk.t, None, 2, 0, cp), -1), ((trk.t, vids, 2, 5, cp), -1),
                         ((trk.t, vids, 2, 0, None), -1), ((trk.t, vids, 9, 0, cp), -6), ((None, vids, 2, 0, cp), -1)):
        assert call(*args) == status, args
        assert [o.value for o in outs] == [0x1000 + k for k in range(6)]
    # cross-use: a plain tracker here, a best-shot tracker in the plain calls, finish on a plain tracker
    other = eng.tracker()
    assert call(other.t, vids, 2, 0, cp) == -1
    can = C.c_void_p(0x77)
    assert lib.rf_tracker_finish(other.t, 0, cp, None, C.byref(can), None) == -1 and can.value == 0x77
    other.close()
    assert lib.rf_detect_yuv_track_device(eng.h, trk.t, arr, vids, 2, 0, THR, NMS, None, None, None, C.byref(can), None, None, None,
                                          None) == -1
    d, c, _ = eng.detect_yuv_device(dev, THR, NMS)
    assert lib.rf_track_update(trk.t, vids, 2, d, c, None, C.byref(can), None) == -1 and can.value == 0x77
    assert lib.rf_tracker_finish(trk.t, 2, cp, None, C.byref(can), None) == -1 and can.value == 0x77
    assert lib.rf_tracker_finish(trk.t, 0, None, None, C.byref(can), None) == -1 and can.value == 0x77
    cfg = capi.TrackConfig(1, 0, 0, 0, 0, 0, 0, 0)
    bad = [capi.best_config(max_faces=4), capi.best_config(min_quality=1.5), capi.best_config(min_quality=-0.1),
           capi.best_config(sharp_half=-1.0), capi.best_config(sharp_half=float("nan")), capi.best_config(sharp_half=float("inf")),
           capi.best_config(crop=(4, 4))]
    for b in bad:
        out = C.c_void_p(0x42)
        assert lib.rf_tracker_create_best(eng.h, C.byref(cfg), C.byref(b), C.byref(out)) == -1
    big = capi.TrackConfig(4096, 1024, 0, 0, 0, 0, 0, 0)
    out = C.c_void_p(0x42)
    assert lib.rf_tracker_create_best(eng.h, C.byref(big), C.byref(capi.best_config()), C.byref(out)) == -6
    assert lib.rf_tracker_create_best(eng.h, C.byref(capi.TrackConfig(0, 0, 0, 0, 0, 0, 0, 0)), C.byref(capi.best_config()),
                                      C.byref(out)) == -1
    assert [trk.debug_state(v)[0].tobytes() + trk.debug_state(v)[1].tobytes() for v in (0, 1)] == state
    # the other paths are as they were
    trk.close()
    assert np.array_equal(eng.detect_batch([golden_image], THR, NMS)[0], base)
    plain = eng.tracker(max_videos=2)
    tp, tc, _, _, _ = plain.detect_yuv_device(dev, [0, 1], THR, NMS)
    assert [a.tobytes() for a in plain.read(tp, tc, 2)] == [a.tobytes() for a in plain_tracks]
    plain.close()
    assert eng.launches_per_batch(2) == launches
    eng.close()


def test_detector_best_shots(video):
    from retinaface_b200 import RetinaFace
    frames, _ = video
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    dev = [_cuda(f) for f in frames[:4]]
    tracks, shots = rf.trackFrames(dev, [0] * 4, THR, best=dict(), max_videos=2)
    assert len(tracks) == 4 and len(tracks[0]) >= 3 and all(s == [] for s in shots)
    fin = rf.finishVideo(0)
    assert [int(s["id"]) for s, _ in fin] == [i for i, st, _ in tracks[3] if st != 0]
    assert all(tuple(c.shape) == (112, 112, 3) for _, c in fin)
