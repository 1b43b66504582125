"""GPU (-m gpu): f16 following between detections -- rf_track_follow_device and the detect calls of a follow tracker against
oracle/follow.py bit for bit (track lists, rf_follow records, the FP64 Kalman state), fed the device's records; that detect calls on a
follow tracker return exactly a plain tracker's lists and bytes; that planted faces keep their ids and boxes across follow frames;
that a face replaced by a flat patch is dropped rather than left on the background; reset and the refusals."""
import numpy as np
import pytest

from oracle.follow import FLAT, MISMATCH, FollowTrackerOracle, luma_of
from oracle.track import LOST
from test_gpu_lookback import FACE, NF, PY, _in_frames, _patch, _planted, _views
from test_gpu_motion import _same, _scene
from test_gpu_redact import _engine

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
W, H = 1920, 1080
REC = ("id", "status", "dx", "dy", "scale", "sad")


@pytest.fixture(scope="module")
def planted(golden_image):
    return _planted(golden_image)


@pytest.fixture(scope="module")
def moving(golden_image):
    """NF BGR frames of the textured scene with two copies of the planted face moving inside the frame -- right and down at (6, 2) px
    per frame, left at 4 px per frame -- and their true face boxes per frame."""
    S = _scene(3, 2400, 1400)
    p = _patch(golden_image)
    ph, pw = p.shape[:2]
    frames, truth = [], []
    for t in range(NF):
        f = S[:H, :W].copy()
        pos = {"right": (200 + 6 * t, 40 + 2 * t), "left": (1400 - 4 * t, PY)}
        for x, y in pos.values():
            f[y:y + ph, x:x + pw] = p
        frames.append(f)
        truth.append({k: (x + FACE[0], y + FACE[1], x + FACE[2], y + FACE[3]) for k, (x, y) in pos.items()})
    return frames, truth


def _runs(k, s, m):
    """Frames s .. s + m - 1 as consecutive runs of one kind: (detect?, first, count); frame t is a detect frame when t % k == 0."""
    out = []
    for t in range(s, s + m):
        d = t % k == 0
        if out and out[-1][0] == d:
            out[-1][2] += 1
        else:
            out.append([d, t, 1])
    return out


def _drive(eng, trk, views, host, k, per_call, layout, redact=False):
    """Every frame of video 0 through the follow tracker, per_call frames per call split into detect and follow runs.  Returns per
    frame (kind, tracks, records or follow records, scale)."""
    got = []
    for s in range(0, len(views), per_call):
        for det, t0, m in _runs(k, s, min(per_call, len(views) - s)):
            chunk = views[t0:t0 + m]
            if det:
                call = trk.detect_yuv_redact_device if redact else trk.detect_yuv_device
                tp, tc, d, c, sc = call(chunk, [0] * m, THR, NMS, layout=layout)
                recs = eng.read_dets(d, c, m)[0]
                tr = trk.read(tp, tc, m)
                got += [("detect", tr[i], recs[i], sc[i]) for i in range(m)]
            else:
                tp, tc = trk.follow_device(chunk, [0] * m, layout=layout)
                tr = trk.read(tp, tc, m)
                fo = trk.follow(m)
                got += [("follow", tr[i], fo[i, :len(tr[i])], None) for i in range(m)]
    eng.synchronize()
    return got


def _check_oracle(got, host, tag, **cfg):
    o = FollowTrackerOracle(1, **cfg)
    for t, (kind, tracks, recs, sc) in enumerate(got):
        luma = luma_of(host[t], W, H)
        if kind == "detect":
            want = o.update(0, recs, sc, luma=luma)
        else:
            want, wf = o.follow(0, luma)
            assert len(recs) == len(wf), (tag, t)
            for r, w in zip(recs, wf):
                for f in REC:
                    assert int(r[f]) == int(w[f]), (tag, t, f, r, w)
                for f in ("fx", "fy", "x1", "y1", "x2", "y2"):
                    assert np.float32(r[f]).tobytes() == np.float32(w[f]).tobytes(), (tag, t, f, r[f], w[f])
        _same(tracks, want, f"{tag} frame {t}")
        assert [int(r["followed"]) for r in tracks] == [w["followed"] for w in want], (tag, t)
    return o


@pytest.mark.parametrize("prec,layout,k,per_call", [("fp16", "nv12", 3, 8), ("fp32", "i420", 2, 1), ("int8", "nv12", 5, 4),
                                                    ("fp16", "i420", 5, 8), ("fp16", "nv12", 2, 4)])
def test_follow_equals_the_oracle(planted, prec, layout, k, per_call):
    frames, _ = planted
    dev, host = _in_frames(frames, layout)
    eng = _engine(prec)
    trk = eng.tracker(follow=True)
    got = _drive(eng, trk, _views(dev, layout), host, k, per_call, layout)
    o = _check_oracle(got, host, f"{prec} {layout} k={k} per_call={per_call}")
    hdr, rows = trk.debug_state(0)
    assert np.array_equal(np.r_[hdr, rows.reshape(-1)].view(np.uint64), o.debug_state(0).view(np.uint64))
    assert any(int(r["followed"]) for kind, tr, _, _ in got if kind == "follow" for r in tr)
    trk.close()
    eng.close()


def test_detect_calls_equal_a_plain_tracker(planted):
    """Only detect calls (tracked, then tracked + redacted): a follow tracker's lists, Kalman state and redacted bytes are a plain
    tracker's."""
    import torch
    frames, _ = planted
    eng = _engine("fp16")
    outs = {}
    for follow in (False, True):
        dev, host = _in_frames(frames[:16], "nv12")
        trk = eng.tracker(follow=follow)
        got = _drive(eng, trk, _views(dev, "nv12"), host, 1, 8, "nv12", redact=True)
        outs[follow] = (got, trk.debug_state(0), [d.cpu().numpy() for d in dev])
        torch.cuda.synchronize()
        trk.close()
    (g0, s0, b0), (g1, s1, b1) = outs[False], outs[True]
    for (_, t0, r0, c0), (_, t1, r1, c1) in zip(g0, g1):
        assert t0.tobytes() == t1.tobytes() and np.array_equal(r0, r1) and c0 == c1
    assert all(np.array_equal(a, b) for a, b in zip(s0, s1))
    assert all(np.array_equal(a, b) for a, b in zip(b0, b1))
    eng.close()


def _iou(a, b):
    x1, y1, x2, y2 = max(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2]), min(a[3], b[3])
    inter = max(0.0, x2 - x1) * max(0.0, y2 - y1)
    return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)


@pytest.mark.parametrize("k", [3, 5])
def test_moving_faces_keep_their_ids(moving, k):
    """Each moving face, once tracked on a detect frame, keeps one id on every later frame, and its box (the followed box on follow
    frames) has IoU >= 0.5 with the true box."""
    frames, truth = moving
    dev, host = _in_frames(frames, "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(follow=True)
    got = _drive(eng, trk, _views(dev, "nv12"), host, k, 8, "nv12")
    ids = {}
    checked = 0
    for t, (kind, tracks, _, _) in enumerate(got):
        for name, box in truth[t].items():
            best = max(((_iou(tuple(float(v) for v in r["face"][1:5]), box), int(r["id"])) for r in tracks if int(r["state"]) != LOST),
                       default=(0.0, 0))
            if name not in ids:
                if kind == "detect" and best[0] >= 0.5:
                    ids[name] = best[1]
                continue
            assert best[1] == ids[name] and best[0] >= 0.5, (k, t, name, best, ids[name])
            checked += kind == "follow"
    assert set(ids) == {"right", "left"} and checked > 0, (ids, checked)
    trk.close()
    eng.close()


def test_flat_patch_ends_lost(planted):
    """The still face replaced by a flat patch on follow frames: its track fails with MISMATCH or FLAT and becomes LOST, and no
    followed box stays on the patch."""
    frames, truth = planted
    frames = [f.copy() for f in frames[:14]]
    x1, y1, x2, y2 = truth[0]["still"]
    for t in (11, 12):                      # follow frames at k = 5
        frames[t][y1 - 30:y2 + 30, max(x1 - 30, 0):x2 + 30] = 128
    dev, host = _in_frames(frames, "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(follow=True)
    got = _drive(eng, trk, _views(dev, "nv12"), host, 5, 1, "nv12")
    _check_oracle(got, host, "flat patch")
    before = [r for r in got[10][1] if _iou(tuple(float(v) for v in r["face"][1:5]), truth[10]["still"]) >= 0.5]
    assert before, "the still face is tracked before the patch"
    sid = int(before[0]["id"])
    kind, tracks, fo, _ = got[11]
    assert kind == "follow"
    rec = [r for r in fo if int(r["id"]) == sid][0]
    assert int(rec["status"]) in (MISMATCH, FLAT), rec
    tr = [r for r in tracks if int(r["id"]) == sid][0]
    assert int(tr["state"]) == LOST and int(tr["followed"]) == 0
    for t in (11, 12):
        for r in got[t][1]:
            if int(r["followed"]):
                assert _iou(tuple(float(v) for v in r["face"][1:5]), truth[t]["still"]) < 0.3, (t, r)
    trk.close()
    eng.close()


def test_reset_and_refusals(planted):
    """Refused calls launch nothing (the Kalman state and the follow records stay as they were); reset drops the templates."""
    from retinaface_b200.capi import RfError
    frames, _ = planted
    dev, host = _in_frames(frames[:4], "nv12")
    views = _views(dev, "nv12")
    eng = _engine("fp16")
    plain = eng.tracker()
    with pytest.raises(RfError):
        plain.follow_device(views[:1], [0])
    with pytest.raises(RfError):
        plain.follow(1)
    for kw in (dict(best={}), dict(lookback=True)):
        with pytest.raises(RfError):
            eng.tracker(follow=True, **kw)
    trk = eng.tracker(follow=True)
    with pytest.raises(RfError):
        trk.set_follow()                       # a second call
    for bad in (dict(search=17), dict(max_mad=300.0), dict(max_mad=float("nan"))):
        with pytest.raises(RfError):
            eng.tracker(**{"follow": bad})
    tp, tc, d, c, sc = trk.detect_yuv_device(views[:2], [0, 0], THR, NMS)
    trk.follow_device(views[2:3], [0])
    state = trk.debug_state(0)
    fo = trk.follow(1)
    with pytest.raises(RfError):
        trk.update([0], d, c, sc[:1])          # no pixels
    with pytest.raises(RfError):
        trk.follow_device(views[3:4], [1])     # video outside max_videos
    with pytest.raises(RfError):
        trk.set_motion()
    with pytest.raises(RfError):
        trk.set_lookback()
    after = trk.debug_state(0)
    assert all(np.array_equal(a.view(np.uint64), b.view(np.uint64)) for a, b in zip(state, after))
    assert trk.follow(1).tobytes() == fo.tobytes()
    assert state[0][0] > 0
    trk.reset(0)
    tp, tc = trk.follow_device(views[3:4], [0])
    assert len(trk.read(tp, tc, 1)[0]) == 0
    trk.close()
    plain.close()
    eng.close()


def _calls(vids, k, per_call):
    """The driver's calls: per chunk of per_call frames, the detect and follow sub-calls RetinaFace.trackFrames issues for them."""
    from types import SimpleNamespace
    from retinaface_b200.detector import RetinaFace
    holder = SimpleNamespace()
    out = []
    for s in range(0, len(vids), per_call):
        for det, idx in RetinaFace._interval_calls(holder, vids[s:s + per_call], k):
            out.append((det, [s + i for i in idx]))
    return out


def _drive_many(eng, trk, views, vids, k, per_call, layout, style=None, sync=True):
    """Every frame through the follow tracker (frame i of video vids[i]); style: redact every call with it.  Returns the issue order
    and, per frame, (kind, tracks, records or follow records, scale, motion) -- with sync False only the last call's lists are read."""
    got, order = {}, []
    calls = _calls(vids, k, per_call)
    for n_call, (det, idx) in enumerate(calls):
        chunk, vv, m = [views[i] for i in idx], [vids[i] for i in idx], len(idx)
        order += idx
        kw = dict(style=style[0], shape=style[1]) if style else {}
        if det:
            call = trk.detect_yuv_redact_device if style else trk.detect_yuv_device
            tp, tc, d, c, sc = call(chunk, vv, THR, NMS, layout=layout, **kw)
        else:
            tp, tc = (trk.follow_redact_device if style else trk.follow_device)(chunk, vv, layout=layout, **kw)
        if not sync and n_call < len(calls) - 1:
            continue
        tr = trk.read(tp, tc, m)
        mo = trk.motion(m) if trk.motion_on else [None] * m
        if det:
            recs = eng.read_dets(d, c, m)[0]
            for j, i in enumerate(idx):
                got[i] = ("detect", tr[j], recs[j], sc[j], mo[j])
        else:
            fo = trk.follow(m)
            for j, i in enumerate(idx):
                got[i] = ("follow", tr[j], fo[j, :len(tr[j])], None, mo[j])
    eng.synchronize()
    return order, got


def _oracle_run(host, vids, order, got, nv, motion, check=True, tag=""):
    """The oracle over the frames in issue order, fed the device's records; checks every frame in `got` (check).  Returns the
    trackers' oracle and per frame the oracle's lists."""
    from oracle.motion import MotionOracle, applied
    from test_gpu_motion import _same_motion
    o = FollowTrackerOracle(nv)
    mo = MotionOracle(nv) if motion else None
    lists = {}
    for i in order:
        kind, tracks, recs, sc, mrec = got[i]
        v, luma = vids[i], luma_of(host[i], W, H)
        if kind == "detect":
            wm = mo.update(v, luma, recs, len(recs), float(sc)) if motion else None
            want = o.update(v, recs, sc, motion=applied(wm) if motion else None, luma=luma)
        else:
            faces = o.mask_faces(v)
            wm = mo.update(v, luma, faces, len(faces), None) if motion else None
            want, wf = o.follow(v, luma, motion=applied(wm) if motion else None)
            if check:
                assert len(recs) == len(wf), (tag, i)
                for r, w in zip(recs, wf):
                    assert all(int(r[f]) == int(w[f]) for f in REC), (tag, i, r, w)
                    assert all(np.float32(r[f]).tobytes() == np.float32(w[f]).tobytes() for f in ("fx", "fy", "x1", "y1", "x2", "y2")), (tag, i)
        if check:
            if motion:
                _same_motion(mrec, wm, f"{tag} frame {i}")
            _same(tracks, want, f"{tag} frame {i}")
            assert [int(r["followed"]) for r in tracks] == [w["followed"] for w in want], (tag, i)
        lists[i] = want
    return o, lists


def test_follow_with_motion_equals_the_oracle(golden_image):
    """On a motion tracker, follow frames are estimated with the tracks' faces as the mask and searched from the moved prediction:
    motions, lists, follow records and the FP64 state equal the oracles' on the shaking video."""
    from test_gpu_motion import _shake
    frames = _shake(golden_image)[0]
    dev, host = _in_frames(frames, "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(follow=True, motion=True)
    vids = [0] * len(frames)
    order, got = _drive_many(eng, trk, _views(dev, "nv12"), vids, 3, 4, "nv12")
    o, _ = _oracle_run(host, vids, order, got, 1, True, "motion")
    hdr, rows = trk.debug_state(0)
    assert np.array_equal(np.r_[hdr, rows.reshape(-1)].view(np.uint64), o.debug_state(0).view(np.uint64))
    assert any(int(m["status"]) == 0 for kind, *_, m in got.values() if kind == "follow")
    assert any(int(r["followed"]) for kind, tr, *_ in got.values() if kind == "follow" for r in tr)
    trk.close()
    eng.close()


@pytest.mark.parametrize("st,layout", [(("mosaic", "rect"), "nv12"), (("blur", "ellipse"), "i420")])
def test_follow_redaction_equals_the_oracle_and_covers(moving, st, layout):
    """rf_track_follow_redact_device: every byte of every frame (detect frames through the tracked redaction) equals f12 / f14's
    oracle over the OK-followed faces and the LOST tracks, and every moving face's true box lies inside a region on every frame."""
    from oracle.redact import frame_regions, params
    from oracle.redact_style import redact_yuv, style
    from test_gpu_lookback import PITCH, _surface
    frames, truth = moving
    dev, host = _in_frames(frames, layout)
    eng = _engine("fp16")
    trk = eng.tracker(follow=True)
    vids = [0] * len(frames)
    order, got = _drive_many(eng, trk, _views(dev, layout), vids, 3, 8, layout, style=st)
    _, lists = _oracle_run(host, vids, order, got, 1, False, "redact")
    b, m = params(0, 0.0)
    sty = style(1 if st[0] == "mosaic" else 2, 1 if st[1] == "rect" else 2)
    surf = _surface(layout, PITCH)
    for i in range(len(frames)):
        kind, tracks, recs, sc, _ = got[i]
        want = lists[i]
        _same(tracks, want, f"redact frame {i}")
        if kind == "detect":
            regs = frame_regions(recs, len(recs), float(sc), m, b, tracks=want)
        else:
            faces = np.array([w["face"] for w in want if w["followed"]], np.float32).reshape(-1, 15)
            regs = frame_regions(faces, len(faces), None, m, b, tracks=want)
        exp = redact_yuv(host[i], layout, regs, sty, **surf)
        assert np.array_equal(dev[i].cpu().numpy(), exp), (st, i, kind)
        for name, (x1, y1, x2, y2) in truth[i].items():
            assert any(r[0] <= x1 and r[1] <= y1 and r[2] >= x2 and r[3] >= y2 for r in regs), (i, name, regs)
    trk.close()
    eng.close()


def test_two_videos_over_two_contexts_in_flight(planted, moving):
    """Two videos interleaved in every call (two frames of each: two rounds), on a two-context engine, every list equal to the
    oracle's; then 2 streams + 1 calls issued without waiting, the final lists and both videos' FP64 state equal to the oracle's."""
    fa, fb = planted[0][:20], moving[0][:20]
    frames, vids = [], []
    for t in range(0, 20, 2):
        frames += [fa[t], fb[t], fa[t + 1], fb[t + 1]]
        vids += [0, 1, 0, 1]
    dev, host = _in_frames(frames, "nv12")
    sync_got = None
    for sync in (True, False):
        eng = _engine("fp16", streams=2)
        trk = eng.tracker(max_videos=2, follow=True)
        order, got = _drive_many(eng, trk, _views(dev, "nv12"), vids, 3, 4, "nv12", sync=sync)
        if sync:
            o, _ = _oracle_run(host, vids, order, got, 2, False, True, "two videos")
        else:
            last = [i for i in order if i in got]
            full = {i: got.get(i) for i in order}
            # the frames before the last call are replayed from the synchronous run's records
            for i in order:
                if full[i] is None:
                    full[i] = sync_got[i]
            o, lists = _oracle_run(host, vids, order, full, 2, False, "in flight")
            for i in last:
                _same(got[i][1], lists[i], f"in flight frame {i}")
        for v in (0, 1):
            hdr, rows = trk.debug_state(v)
            assert np.array_equal(np.r_[hdr, rows.reshape(-1)].view(np.uint64), o.debug_state(v).view(np.uint64)), (sync, v)
        sync_got = got
        trk.close()
        eng.close()


def test_detector_detect_every(moving):
    """RetinaFace.trackFrames(detect_every=3) and redactFrames(detect_every=3) issue the detect and follow calls a follow tracker
    takes: the lists equal a capi-driven tracker's; best / look-back with an interval and a plain tracker with one are refused."""
    import os
    from conftest import GOLDEN
    from retinaface_b200.detector import RetinaFace
    frames = moving[0][:10]
    dev, host = _in_frames(frames, "nv12")
    views = _views(dev, "nv12")
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    eng = det.engine
    vids = [0] * len(frames)
    got = []
    for s in range(0, len(frames), 4):
        got += det.trackFrames(views[s:s + 4], vids[s:s + 4], threshold=THR, detect_every=3, max_videos=1)[0]
    trk = eng.tracker(max_videos=1, follow=True)
    order, ref = _drive_many(eng, trk, views, vids, 3, 4, "nv12")
    for i in range(len(frames)):
        assert [(a, b) for a, b, _ in got[i]] == [(int(r["id"]), int(r["state"])) for r in ref[i][1]], i
        assert [f.rect for _, _, f in got[i]] == [tuple(float(x) for x in r["face"][1:5]) for r in ref[i][1]], i
    with pytest.raises(ValueError):
        det.trackFrames(views[:1], [0], detect_every=2, best={})
    with pytest.raises(ValueError):
        det.redactFrames(views[:1], [0], detect_every=2, lookback=3)
    with pytest.raises(ValueError):
        det.redactFrames(views[:1], None, detect_every=2)
    plain = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    plain.trackFrames(views[:1], [0], threshold=THR)
    with pytest.raises(ValueError):
        plain.trackFrames(views[1:2], [0], threshold=THR, detect_every=3)
    det2 = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    dev2, _ = _in_frames(frames[:4], "nv12")
    det2.redactFrames(_views(dev2, "nv12"), [0] * 4, threshold=THR, detect_every=2)
    assert det2._tracker.follow_on
    trk.close()
