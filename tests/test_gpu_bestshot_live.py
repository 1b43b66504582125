"""GPU (-m gpu): f22 best shots for live cameras -- rf_tracker_set_best_live against tests/bestshot_live_oracle.py bit for bit (every
LIVE, EXIT and FINISH record, crop and M) on f11's synthetic 30-frame 1080p video, live shots strictly additive to f11's, the behaviour in
the sharp window; following best-shot trackers (rf_tracker_set_best_follow, rf_track_follow_best_device) at k = 2, 3 and 5 against a
follow tracker and FollowTrackerOracle -> the live oracle; tiling, calls in flight, the refusals and the drivers."""
import ctypes as C
import os

import numpy as np
import pytest

from bestshot_live_oracle import BEST_LIVE, LiveBestShotOracle
from conftest import GOLDEN
from oracle.bestshot import BEST_EXIT, BEST_FINISH, quality
from oracle.follow import FollowTrackerOracle, luma_of
from test_gpu_bestshot import MAX_LOST, NF, NMS, SHARP, THR, ONE_FRAME, H, W, _cuda, _engine, _same_shot, video  # noqa: F401

pytestmark = pytest.mark.gpu

T = 64
LIVE_CFG = dict(first_quality=0.05, improve=0.2, min_gap=2)


def _dev(frames):
    return [_cuda(f) for f in frames]


def _call(eng, trk, chunk, vids, detect, crops, mats=None):
    """One best-shot call (detect, or follow on a following best-shot tracker): (shots, tracks, records or follow records, scales)."""
    m = len(chunk)
    if detect:
        bp, bc, tp, tc, d, c, sc = trk.detect_yuv_best_device(chunk, vids, THR, NMS, crops.data_ptr(), mats.data_ptr() if mats is not None else None)
        recs = eng.read_dets(d, c, m)[0]
    else:
        bp, bc, tp, tc = trk.follow_best_device(chunk, vids, crops.data_ptr(), mats.data_ptr() if mats is not None else None)
        sc = [None] * m
    shots, tracks = trk.read_best(bp, bc, m), trk.read(tp, tc, m)
    if not detect:
        fo = trk.follow(m)
        recs = [fo[i, :len(tracks[i])] for i in range(m)]
    return [(shots[i], tracks[i], recs[i], sc[i]) for i in range(m)]


def _runs(k, s, m):
    out = []
    for t in range(s, s + m):
        d = t % k == 0
        if out and out[-1][0] == d:
            out[-1][2] += 1
        else:
            out.append([d, t, 1])
    return out


def _drive(eng, trk, dev, per_call, k=1):
    """Every frame of video 0, per_call frames per call split into detect and follow runs (frame t detected when t % k == 0).  Returns
    per frame (kind, shots, tracks, records, scale) and the host crops / matrices of each frame's shots."""
    import torch
    crops = torch.full((NF, T, 112, 112, 3), 0xA5, dtype=torch.uint8, device="cuda")
    mats = torch.zeros((NF, T, 6), dtype=torch.float64, device="cuda")
    got = []
    for s in range(0, len(dev), per_call):
        for det, t0, m in _runs(k, s, min(per_call, len(dev) - s)):
            got += [(det,) + r for r in _call(eng, trk, dev[t0:t0 + m], [0] * m, det, crops[t0:t0 + m], mats[t0:t0 + m])]
    return got, crops.cpu().numpy(), mats.cpu().numpy()


def _finish(trk, video=0):
    import torch
    fc = torch.full((T, 112, 112, 3), 0x5A, dtype=torch.uint8, device="cuda")
    fm = torch.zeros((T, 6), dtype=torch.float64, device="cuda")
    bp, bc = trk.finish(video, fc.data_ptr(), fm.data_ptr())
    return trk.read_best(bp, bc, 1)[0], fc.cpu().numpy(), fm.cpu().numpy()


def _record_crops(eng, frame):
    """The crop and M rf_detect_yuv_batch_device cuts for every record of one frame (the oracle's inputs)."""
    import torch
    mf = eng.max_faces
    crops = torch.zeros((1, mf, 112, 112, 3), dtype=torch.uint8, device="cuda")
    mats = torch.zeros((1, mf, 6), dtype=torch.float64, device="cuda")
    d, c, sc = eng.detect_yuv_device([frame], THR, NMS, align=dict(), dev_crops_ptr=crops.data_ptr(), dev_mats_ptr=mats.data_ptr())
    return eng.read_dets(d, c, 1)[0][0], sc[0], crops[0].cpu().numpy(), mats[0].cpu().numpy()


def _oracle(eng, dev, frames, k=1, live=LIVE_CFG, min_quality=0.0):
    """FollowTrackerOracle (detect frames t % k == 0, follow frames otherwise) -> LiveBestShotOracle: per frame its shots, finish, and
    each matched track's q on the frame."""
    fo, bo = FollowTrackerOracle(1, max_lost=MAX_LOST), LiveBestShotOracle(min_quality=min_quality, live=live)
    out, qs = [], []
    for t in range(len(dev)):
        luma = luma_of(frames[t], W, H)
        if t % k == 0:
            recs, sc, cr, mt = _record_crops(eng, dev[t])
            tracks = fo.update(0, recs, sc, luma=luma)
        else:
            tracks, _ = fo.follow(0, luma)
            cr = mt = None
        out.append(bo.update(0, tracks, cr, mt, W, H))
        qs.append({int(x["id"]): quality(cr[int(x["det"])], x["face"], mt[int(x["det"])], W, H)["q"] for x in tracks if int(x["det"]) >= 0})
    return out, bo.finish(0), qs


def _check_shots(got, crops, mats, want, tag):
    n = 0
    for t, (_, shots, _, _, _) in enumerate(got):
        assert len(shots) == len(want[t]), (tag, t, [(int(s["id"]), int(s["reason"])) for s in shots], [(w["id"], w["reason"]) for w in want[t]])
        for kk, (s, w) in enumerate(zip(shots, want[t])):
            _same_shot(s, w, f"{tag} frame {t}")
            assert np.array_equal(crops[t, kk], w["crop"]), (tag, t, kk)
            assert mats[t, kk].tobytes() == w["M"].reshape(6).tobytes(), (tag, t, kk)
            n += int(s["reason"]) == BEST_LIVE
        assert (crops[t, len(shots):] == 0xA5).all(), (tag, t)
    return n


def _check_finish(fin, fc, fm, want_fin, tag):
    assert len(fin) == len(want_fin), tag
    for kk, (s, w) in enumerate(zip(fin, want_fin)):
        _same_shot(s, w, f"{tag} finish")
        assert np.array_equal(fc[kk], w["crop"]) and fm[kk].tobytes() == w["M"].reshape(6).tobytes(), tag


@pytest.mark.parametrize("prec,per_call", [("fp32", 8), ("fp16", 1), ("fp16", 4), ("fp16", 8), ("int8", 8)])
def test_live_shots_equal_the_oracle(video, prec, per_call):
    frames, _ = video
    dev = _dev(frames)
    eng = _engine(prec)
    want, want_fin, _ = _oracle(eng, dev, frames)
    trk = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=LIVE_CFG)
    got, crops, mats = _drive(eng, trk, dev, per_call)
    assert _check_shots(got, crops, mats, want, prec) >= 2
    _check_finish(*_finish(trk), want_fin, prec)
    trk.close()
    eng.close()


def test_two_videos_interleaved(video):
    """Video 0 from frame 0 and video 1 from frame 7, frames alternating in each call, equal the oracle per video."""
    import torch
    frames, _ = video
    dev = _dev(frames)
    eng = _engine("fp16")
    want0, fin0, _ = _oracle(eng, dev, frames)
    want1, fin1, _ = _oracle(eng, dev[7:], frames[7:])
    trk = eng.tracker(max_videos=2, max_lost=MAX_LOST, best=dict(), best_live=LIVE_CFG)
    seq = [(0, t) for t in range(NF)]
    seq = [x for pair in zip(seq, [(1, t) for t in range(NF - 7)] + [None] * 7) for x in pair if x is not None]
    got = {0: [], 1: []}
    for s in range(0, len(seq), 8):
        part = seq[s:s + 8]
        cr = torch.full((len(part), T, 112, 112, 3), 0xA5, dtype=torch.uint8, device="cuda")
        mt = torch.zeros((len(part), T, 6), dtype=torch.float64, device="cuda")
        res = _call(eng, trk, [dev[t + 7 * v] for v, t in part], [v for v, _ in part], True, cr, mt)
        crh, mth = cr.cpu().numpy(), mt.cpu().numpy()
        for i, (v, t) in enumerate(part):
            got[v].append((res[i][0], crh[i], mth[i]))
    for v, want, fin in ((0, want0, fin0), (1, want1, fin1)):
        assert len(got[v]) == len(want)
        for t, (shots, crh, mth) in enumerate(got[v]):
            assert len(shots) == len(want[t]), (v, t)
            for kk, (s, w) in enumerate(zip(shots, want[t])):
                _same_shot(s, dict(w, video=v), f"video {v} frame {t}")
                assert np.array_equal(crh[kk], w["crop"]) and mth[kk].tobytes() == w["M"].reshape(6).tobytes()
        f, fc, fm = _finish(trk, v)
        _check_finish(f, fc, fm, [dict(w, video=v) for w in fin], f"video {v}")
    trk.close()
    eng.close()


def test_live_is_additive(video):
    """The live tracker's lists equal a plain best-shot tracker's, and without its LIVE shots each frame's shots and crops are the
    plain tracker's, in order."""
    frames, _ = video
    dev = _dev(frames)
    eng = _engine("fp16")
    plain = eng.tracker(max_lost=MAX_LOST, best=dict())
    live = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=dict(first_quality=0.01, improve=0.05, min_gap=1))
    gp, cp, _ = _drive(eng, plain, dev, 8)
    gl, cl, _ = _drive(eng, live, dev, 8)
    nlive = 0
    for t in range(NF):
        assert gp[t][2].tobytes() == gl[t][2].tobytes(), t
        keep = [kk for kk, s in enumerate(gl[t][1]) if int(s["reason"]) != BEST_LIVE]
        nlive += len(gl[t][1]) - len(keep)
        assert gl[t][1][keep].tobytes() == gp[t][1].tobytes(), t
        assert np.array_equal(cl[t, keep], cp[t, :len(gp[t][1])]), t
    assert nlive >= 3
    assert _finish(plain)[0].tobytes() == _finish(live)[0].tobytes()
    plain.close()
    live.close()
    eng.close()


def test_behaviour_on_the_synthetic_video(video):
    frames, _ = video
    dev = _dev(frames)
    eng = _engine("fp16")
    _, _, qs = _oracle(eng, dev, frames, live=None)
    blurred = max(q for t, per in enumerate(qs) if t not in SHARP for q in per.values())
    sharp_ids = {i for t in SHARP for i, q in qs[t].items() if q > blurred}
    assert sharp_ids
    # first_quality above every blurred frame's q: a face detected in the sharp window gets its first LIVE shot there
    fq = float(np.nextafter(np.float32(blurred), np.float32(1)))
    trk = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=dict(first_quality=fq, min_gap=1))
    got, _, _ = _drive(eng, trk, dev, 4)
    first_live = {}
    for t, (_, shots, _, _, _) in enumerate(got):
        for s in shots:
            if int(s["reason"]) == BEST_LIVE:
                first_live.setdefault(int(s["id"]), t)
    for i in sharp_ids:
        assert first_live.get(i) in SHARP, (i, first_live.get(i))
    one = [int(r["id"]) for r in got[ONE_FRAME][2] if r["face"][2] > 700 and int(r["id"]) not in first_live]
    trk.close()
    # a low first_quality and min_gap 2: a blurred-frame LIVE shot first, an improved one in the sharp window
    trk = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=dict(first_quality=0.01, min_gap=2))
    got, _, _ = _drive(eng, trk, dev, 4)
    lives = {}
    for t, (_, shots, _, _, _) in enumerate(got):
        for s in shots:
            if int(s["reason"]) == BEST_LIVE:
                lives.setdefault(int(s["id"]), []).append(int(s["frame"]))
    assert any(fr[0] not in SHARP and any(f in SHARP for f in fr[1:]) for fr in lives.values()), lives
    # the face shown on one frame never emits
    ids_one = [int(r["id"]) for r in got[ONE_FRAME][2] if r["face"][2] > 700 and int(r["state"]) == 0]
    assert (ids_one or one) and not any(i in lives for i in ids_one)
    fin = _finish(trk)[0]
    assert not any(int(s["id"]) in ids_one for s in fin) and all(int(s["reason"]) == BEST_FINISH for s in fin)
    trk.close()
    eng.close()


@pytest.mark.parametrize("prec,k,per_call,live", [("fp16", 3, 8, True), ("fp32", 2, 4, False), ("int8", 5, 8, True), ("fp16", 5, 1, False),
                                                  ("fp16", 2, 8, True)])
def test_interval_equals_follow_and_the_oracle(video, prec, k, per_call, live):
    frames, _ = video
    dev = _dev(frames)
    eng = _engine(prec)
    # lists and rf_follow records: a follow tracker's, fed the same split
    fol = eng.tracker(max_lost=MAX_LOST, follow=True)
    want_l = []
    for s in range(0, NF, per_call):
        for det, t0, m in _runs(k, s, min(per_call, NF - s)):
            if det:
                tp, tc, _, _, _ = fol.detect_yuv_device(dev[t0:t0 + m], [0] * m, THR, NMS)
                tr = fol.read(tp, tc, m)
                want_l += [(tr[i], None) for i in range(m)]
            else:
                tp, tc = fol.follow_device(dev[t0:t0 + m], [0] * m)
                tr, fo = fol.read(tp, tc, m), fol.follow(m)
                want_l += [(tr[i], fo[i, :len(tr[i])]) for i in range(m)]
    fol.close()
    trk = eng.tracker(max_lost=MAX_LOST, best=dict(), best_follow=True, best_live=LIVE_CFG if live else None)
    got, crops, mats = _drive(eng, trk, dev, per_call, k)
    for t, (det, _, tracks, recs, _) in enumerate(got):
        assert tracks.tobytes() == want_l[t][0].tobytes(), (k, t)
        if not det:
            assert recs.tobytes() == want_l[t][1].tobytes(), (k, t)
    want, want_fin, _ = _oracle(eng, dev, frames, k=k, live=LIVE_CFG if live else None)
    n = _check_shots(got, crops, mats, want, f"{prec} k={k}")
    assert (n > 0) == live
    assert any(int(s["reason"]) == BEST_EXIT for t in range(NF) for s in got[t][1])
    _check_finish(*_finish(trk), want_fin, f"{prec} k={k}")
    trk.close()
    eng.close()


def test_interval_twins(video):
    """Detect calls only: a following best-shot tracker equals a best-shot tracker.  With motion: the lists equal a motion follow
    tracker's.  Tiling levels {{0, 0}}: everything equals the untiled twin."""
    frames, _ = video
    dev = _dev(frames)
    eng = _engine("fp16")
    a = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=LIVE_CFG)
    b = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=LIVE_CFG, best_follow=True)
    ga, ca, ma = _drive(eng, a, dev, 8)
    gb, cb, mb = _drive(eng, b, dev, 8)
    assert [(x[1].tobytes(), x[2].tobytes()) for x in ga] == [(x[1].tobytes(), x[2].tobytes()) for x in gb]
    assert np.array_equal(ca, cb) and np.array_equal(ma, mb) and _finish(a)[0].tobytes() == _finish(b)[0].tobytes()
    a.close()
    b.close()
    # motion on a shaking video: the same shake as the follow tests' (the frames shifted by a few pixels)
    import cv2
    shake = [cv2.warpAffine(np.ascontiguousarray(f), np.float32([[1, 0, 0], [0, 1, (t % 3) * 2]]), (f.shape[1], f.shape[0]),
                            flags=cv2.INTER_NEAREST) for t, f in enumerate(frames)]
    sdev = _dev(shake)
    res = []
    for kind in ("follow", "best"):
        trk = eng.tracker(max_lost=MAX_LOST, motion=True, follow=kind == "follow", best=dict() if kind == "best" else None,
                          best_follow=kind == "best")
        lists = []
        for s in range(0, NF, 8):
            for det, t0, m in _runs(3, s, min(8, NF - s)):
                import torch
                cr = torch.zeros((m, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
                if kind == "best":
                    lists += [(x[1].tobytes(), x[2].tobytes() if not det else b"") for x in _call(eng, trk, sdev[t0:t0 + m], [0] * m, det, cr)]
                elif det:
                    tp, tc, _, _, _ = trk.detect_yuv_device(sdev[t0:t0 + m], [0] * m, THR, NMS)
                    lists += [(x.tobytes(), b"") for x in trk.read(tp, tc, m)]
                else:
                    tp, tc = trk.follow_device(sdev[t0:t0 + m], [0] * m)
                    tr, fo = trk.read(tp, tc, m), trk.follow(m)
                    lists += [(tr[i].tobytes(), fo[i, :len(tr[i])].tobytes()) for i in range(m)]
        res.append(lists)
        trk.close()
    assert res[0] == res[1]
    # tiling {{0, 0}} against the untiled twin, at k = 3 with live shots
    runs = []
    for tiling in ({"levels": [(0.0, 0)]}, None):
        trk = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=LIVE_CFG, best_follow=True, tiling=tiling)
        g, c, m = _drive(eng, trk, dev, 8, 3)
        runs.append(([(x[1].tobytes(), x[2].tobytes()) for x in g], c.tobytes(), m.tobytes(), _finish(trk)[0].tobytes()))
        trk.close()
    assert runs[0] == runs[1]
    eng.close()


def test_oriented_twin(video):
    """Orientation 6 on stored frames equals orientation 1 on the materialised portrait frames (oracle/orient.py), at k = 3 with live
    shots."""
    from oracle.orient import orient_planes
    frames, _ = video
    stored = frames[:12]                                              # shown at EXIF 6
    portrait = [orient_planes(f, "nv12", 6) for f in stored]         # the displayed frames, materialised
    eng = _engine("fp16", max_image=(W, W))
    res = []
    for ori, imgs in ((6, stored), (1, portrait)):
        dev = _dev(imgs)
        trk = eng.tracker(max_lost=MAX_LOST, best=dict(), best_live=LIVE_CFG, best_follow=True)
        trk.set_orientation(0, ori)
        import torch
        crops = torch.zeros((len(dev), T, 112, 112, 3), dtype=torch.uint8, device="cuda")
        out = []
        for s in range(0, len(dev), 4):
            for det, t0, m in _runs(3, s, min(4, len(dev) - s)):
                out += [(x[1].tobytes(), x[2].tobytes()) for x in _call(eng, trk, dev[t0:t0 + m], [0] * m, det, crops[t0:t0 + m])]
        res.append((out, crops.cpu().numpy().tobytes(), _finish(trk)[0].tobytes()))
        trk.close()
    assert res[0] == res[1]
    eng.close()


def test_calls_in_flight(video):
    import torch
    frames, _ = video
    dev = _dev(frames)
    for streams in (2, 4):
        res = []
        for sync in (False, True):
            e = _engine("fp16", streams=streams)
            k = e.tracker(max_videos=2, max_lost=MAX_LOST, best=dict(), best_live=dict(first_quality=0.01, min_gap=1), best_follow=True)
            n_calls = 2 * streams + 1
            cr = torch.zeros((n_calls, 2, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
            last = None
            for i in range(n_calls):
                fr = [dev[i % NF], dev[NF - 1 - i % NF]]
                if i % 3 == 0:
                    last = k.detect_yuv_best_device(fr, [0, 1], THR, NMS, cr[i].data_ptr())[:2]
                else:
                    last = k.follow_best_device(fr, [0, 1], cr[i].data_ptr())[:2]
                if sync:
                    e.synchronize()
            shots = k.read_best(last[0], last[1], 2)
            fin = _finish(k)[0]
            res.append(([x.tobytes() for x in shots], fin.tobytes(), cr.cpu().numpy().tobytes()))
            k.close()
            e.close()
        assert res[0] == res[1], streams


def _status(eng, fn, *args):
    rc = fn(*args)
    return rc, (eng.lib.rf_last_error(eng.h) or b"").decode()


def test_refusals(video):
    import torch
    from retinaface_b200 import capi
    frames, _ = video
    dev = _dev(frames[:2])
    eng = _engine("fp16")
    lib = eng.lib
    arr = eng._frames(dev, "nv12", True)
    vids = (C.c_int * 2)(0, 0)
    cr = torch.zeros((2, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
    fc = capi.FollowConfig(0, 0.0)
    good = capi.BestLiveConfig(0.0, 0.0, 0)
    # other kinds refuse both setters
    plain, fol = eng.tracker(), eng.tracker(follow=True)
    for t in (plain, fol):
        assert _status(eng, lib.rf_tracker_set_best_live, t.t, C.byref(good)) == (-1, "rf_tracker_set_best_live: not a best-shot tracker "
                                                                                      "(rf_tracker_create_best)")
        assert _status(eng, lib.rf_tracker_set_best_follow, t.t, C.byref(fc))[0] == -1
    outs = [C.c_void_p(0x1000 + i) for i in range(4)]
    rc, err = _status(eng, lib.rf_track_follow_best_device, fol.t, arr, vids, 2, cr.data_ptr(), None, *[C.byref(o) for o in outs])
    assert rc == -1 and err == "rf_track_follow_best_device: not a following best-shot tracker (rf_tracker_set_best_follow)"
    assert [o.value for o in outs] == [0x1000 + i for i in range(4)]
    plain.close()
    fol.close()
    # bad values, a second call, a call after an update; rf_tracker_set_follow keeps its message on a best-shot tracker
    b = eng.tracker(best=dict())
    for bad in ((float("nan"), 0, 0), (1.5, 0, 0), (-0.1, 0, 0), (0, float("nan"), 0), (0, -0.2, 0), (0, float("inf"), 0), (0, 0, -1),
                (0, 0, (1 << 20) + 1)):
        assert _status(eng, lib.rf_tracker_set_best_live, b.t, C.byref(capi.BestLiveConfig(*bad)))[0] == -1, bad
    assert _status(eng, lib.rf_tracker_set_best_follow, b.t, C.byref(capi.FollowConfig(99, 0.0)))[0] == -1
    assert _status(eng, lib.rf_tracker_set_follow, b.t, C.byref(fc)) == (-1, "rf_tracker_set_follow: a best-shot tracker cannot follow")
    # a plain best-shot tracker refuses the follow-best call, nothing launched
    rc, err = _status(eng, lib.rf_track_follow_best_device, b.t, arr, vids, 2, cr.data_ptr(), None, *[C.byref(o) for o in outs])
    assert rc == -1 and err == "rf_track_follow_best_device: not a following best-shot tracker (rf_tracker_set_best_follow)"
    assert b.best_live_on is False
    b.set_best_live()
    assert _status(eng, lib.rf_tracker_set_best_live, b.t, C.byref(good)) == (-1, "rf_tracker_set_best_live: live shots are already on")
    b.set_best_follow()
    assert _status(eng, lib.rf_tracker_set_best_follow, b.t, C.byref(fc)) == (-1, "rf_tracker_set_best_follow: best-shot following is "
                                                                                  "already on")
    only = "a best-shot tracker takes frames only through rf_detect_yuv_track_best_device and rf_track_follow_best_device"
    for fn, args in ((lib.rf_track_follow_device, (b.t, arr, vids, 2, None, None)),
                     (lib.rf_track_follow_redact_device, (b.t, arr, vids, 2, None, None, None))):
        rc, err = _status(eng, fn, *args)
        assert rc == -1 and err.endswith(only), err
    rc, err = _status(eng, lib.rf_track_follow_best_device, b.t, arr, vids, 2, None, None, *[C.byref(o) for o in outs])
    assert rc == -1 and err == "rf_track_follow_best_device: dev_best_crops is NULL"
    assert [o.value for o in outs] == [0x1000 + i for i in range(4)]
    b.detect_yuv_best_device(dev, [0, 0], THR, NMS, cr.data_ptr())
    state = b.debug_state(0)[0].tobytes()
    for fn, cfg in ((lib.rf_tracker_set_best_live, good), (lib.rf_tracker_set_best_follow, fc)):
        rc, err = _status(eng, fn, b.t, C.byref(cfg))
        assert rc == -1 and err.endswith("already on") or err.endswith("the tracker has already been updated"), err
    a2 = eng.tracker(best=dict())
    a2.detect_yuv_best_device(dev[:1], [0], THR, NMS, cr.data_ptr())
    for fn, cfg, who in ((lib.rf_tracker_set_best_live, good, "rf_tracker_set_best_live"), (lib.rf_tracker_set_best_follow, fc,
                                                                                            "rf_tracker_set_best_follow")):
        assert _status(eng, fn, a2.t, C.byref(cfg)) == (-1, f"{who}: the tracker has already been updated")
    assert b.debug_state(0)[0].tobytes() == state
    a2.close()
    b.close()
    eng.close()


def test_drivers(video):
    """RetinaFace.trackFrames(best, live, detect_every=3) equals the direct calls."""
    from retinaface_b200 import RetinaFace
    frames, _ = video
    dev = _dev(frames[:12])
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    live = dict(first_quality=0.05, min_gap=2)
    got = []
    for s in range(0, 12, 4):
        tracks, shots = rf.trackFrames(dev[s:s + 4], [0] * 4, THR, best=dict(), live=live, detect_every=3, max_videos=1)
        got += [([(i, st) for i, st, _ in tr], [(s_.tobytes(), c.cpu().numpy().tobytes()) for s_, c in sh]) for tr, sh in zip(tracks, shots)]
    fin = [(s_.tobytes(), c.cpu().numpy().tobytes()) for s_, c in rf.finishVideo(0)]
    eng = rf.engine
    trk = eng.tracker(max_videos=1, best=dict(), best_live=live, best_follow=True)
    want = []
    import torch
    for s in range(0, 12, 4):
        for det, t0, m in _runs(3, s, 4):
            cr = torch.zeros((m, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
            for i, (shots, tracks, _, _) in enumerate(_call(eng, trk, dev[t0:t0 + m], [0] * m, det, cr)):
                want.append(([(int(r["id"]), int(r["state"])) for r in tracks],
                             [(x.tobytes(), cr[i, kk].cpu().numpy().tobytes()) for kk, x in enumerate(shots)]))
    wfin = _finish(trk)
    assert got == want
    assert fin == [(x.tobytes(), wfin[1][kk].tobytes()) for kk, x in enumerate(wfin[0])]
    assert any(int(np.frombuffer(x, dtype=np.int32)[6]) == BEST_LIVE for _, sh in got for x, _ in sh)
    trk.close()
    with pytest.raises(ValueError):
        rf.trackFrames(dev[:1], [0], THR, live=live)
