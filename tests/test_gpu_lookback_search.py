"""GPU (-m gpu): f17 searching look-back -- every out and drained frame of a searching look-back tracker against
oracle/lookback_search.py byte for byte, and every rf_follow step record and chain length against the oracle's chains; bytes outside
the (d) regions equal a plain look-back tracker's; a fast face is covered on the frames before its first detection where f15's growth
boxes miss it; call shapes, drain and reset; the refusals; RetinaFace.redactFrames(lookback_search=...)."""
import ctypes as C

import numpy as np
import pytest

from oracle.lookback import Frame, births, emit_into, frame_boxes, regions
from oracle.lookback_search import SearchLookbackOracle
from oracle.motion import MotionOracle, MotionTrackerOracle, applied
from oracle.redact import params
from oracle.redact_style import redact_yuv, style
from oracle.track import TrackerOracle
from test_gpu_lookback import (FACE, H, NMS, OPITCH, PITCH, PY, STYLES, THR, W, _in_frames, _lap_var, _out_frames, _patch, _surface,
                               _views)
from test_gpu_motion import _same, _same_motion, _scene
from test_gpu_redact import _engine

pytestmark = pytest.mark.gpu

NF = 24
FAST, SEEN = 40, 16             # the fast face crosses at 40 px per frame (about 2 x grow * w for its ~220 px); detected from frame 16
X0 = 480
NONE = 1.0                      # the decode keeps scores above the threshold, and no score exceeds 1: the calls before SEEN return
                                # no records, whatever the precision
# The detector finds this ~220 px face even blurred with sigma 24 (score > 0.8 at 448 x 448), so the frames before its first detection
# are made by the calls' threshold, not by the pixels: the face is in full view on every frame, and only the records are withheld.


def _thr(t, seen=SEEN):
    return NONE if t < seen else THR


def _fast(golden):
    """NF BGR frames of a face crossing a textured scene from x X0 at FAST px per frame, and each frame's ground-truth face box."""
    S = _scene(3, 2400, 1400)
    p = _patch(golden)
    ph, pw = p.shape[:2]
    frames, truth = [], []
    for t in range(NF):
        f = S[:H, :W].copy()
        x = X0 + FAST * t
        f[PY:PY + ph, x:x + pw] = p
        frames.append(f)
        truth.append((x + FACE[0], PY + FACE[1], x + FACE[2], PY + FACE[3]))
    return frames, truth


@pytest.fixture(scope="module")
def fast(golden_image):
    return _fast(golden_image)


@pytest.fixture(scope="module")
def shaking(golden_image):
    from test_gpu_motion import _shake
    return _shake(golden_image)[0]


def _run(eng, trk, dev, layout, matrix, per_call, st, outs=None, videos=None, seen=SEEN):
    """The frames through the look-back call, per_call per call, at _thr(first frame of the call, seen); per frame (number, tracks,
    records, scale, motion, steps, lengths) and the out frames."""
    outs = outs if outs is not None else _out_frames(len(dev), layout)
    views, oviews = _views(dev, layout), _views(outs, layout)
    got = []
    for s in range(0, len(dev), per_call):
        m = min(per_call, len(dev) - s)
        vids = [0] * m if videos is None else videos[s:s + m]
        nums, tp, tc, d, c, sc = trk.detect_yuv_redact_lookback_device(views[s:s + m], vids, oviews[s:s + m], _thr(s, seen), NMS, layout=layout,
                                                                       matrix=matrix, style=st[0], shape=st[1])
        recs = eng.read_dets(d, c, m)[0]
        tr = trk.read(tp, tc, m)
        mo = trk.motion(m) if trk.motion_on else [None] * m
        steps, lens = trk.lookback_search(m) if trk.lookback_search_on else ([None] * m, [None] * m)
        got += [(int(nums[i]), tr[i], recs[i], sc[i], mo[i], steps[i], lens[i]) for i in range(m)]
    eng.synchronize()
    return got, outs


def _same_steps(steps, lens, want, tag):
    assert all(int(n) == 0 for n in lens[len(want):]), tag
    for r, ch in enumerate(want):
        assert int(lens[r]) == len(ch), (tag, r, int(lens[r]), len(ch))
        for k, w in enumerate(ch):
            g = steps[r][k]
            for f in ("id", "status", "dx", "dy", "scale", "sad"):
                assert int(g[f]) == int(w[f]), (tag, r, k, f, g, w)
            for f in ("fx", "fy", "x1", "y1", "x2", "y2"):
                assert np.float32(g[f]) == np.float32(w[f]), (tag, r, k, f, g, w)


def _check_oracle(got, host, outs, layout, st, L, motion, drained=None, tag="", search=(0, 0.0)):
    """Every emitted (and drained) out frame against the searching oracle over the oracle trackers' lists, every chain against the
    oracle's; returns the oracle's emissions by number and the number of non-empty chains."""
    b, m = params(0, 0.0)
    sty = style(*(1 if st[0] == "mosaic" else 2, 1 if st[1] == "rect" else 2))
    lo = SearchLookbackOracle(L, search=search[0], max_mad=search[1])
    to = MotionTrackerOracle(1) if motion else TrackerOracle(1)
    mo = MotionOracle(1) if motion else None
    isurf, osurf = _surface(layout, PITCH), _surface(layout, OPITCH)
    canary = np.full(outs[0].shape, 0x5A, np.uint8)
    ems, chains = {}, 0
    for t, (num, tracks, recs, sc, mrec, steps, lens) in enumerate(got):
        luma = np.ascontiguousarray(host[t][:H, :W])
        if motion:
            want_m = mo.update(0, luma, recs, len(recs), float(sc))
            _same_motion(mrec, want_m, f"{tag} frame {t}")
            want = to.update(0, recs, sc, motion=applied(want_m))
        else:
            want = to.update(0, recs, sc)
        _same(tracks, want, f"{tag} frame {t}")
        fr = Frame(host[t], frame_boxes(recs, len(recs), float(sc), want), births(want),
                   (int(mrec["status"]), tuple(mrec["m"])) if motion else None)
        em = lo.push(0, fr, luma)
        ch = lo.log[0][t % (2 * L)].chains
        _same_steps(steps, lens, ch, f"{tag} frame {t}")
        chains += sum(1 for c in ch if c)
        assert num == (-1 if em is None else em.number), (tag, t, num)
        got_out = outs[t].cpu().numpy()
        if em is None:
            assert np.array_equal(got_out, canary), (tag, t)
            continue
        ems[em.number] = em
        exp = emit_into(canary, em.data, layout, data_surface=isurf, **osurf)
        exp = redact_yuv(exp, layout, regions(em.boxes, m, b), sty, **osurf)
        assert np.array_equal(got_out, exp), (tag, t, em.number)
    if drained is not None:
        nums, douts = drained
        want = lo.drain(0)
        assert list(nums) == [e.number for e in want], (tag, list(nums))
        for e, o in zip(want, douts):
            ems[e.number] = e
            exp = emit_into(canary, e.data, layout, data_surface=isurf, **osurf)
            exp = redact_yuv(exp, layout, regions(e.boxes, m, b), sty, **osurf)
            assert np.array_equal(o.cpu().numpy(), exp), (tag, "drain", e.number)
    return ems, chains


@pytest.mark.parametrize("prec,st,layout,L,motion,video", [("fp16", "blur", "nv12", 15, False, "fast"),
                                                            ("fp32", "mosaic", "i420", 1, True, "fast"),
                                                            ("int8", "blur", "i420", 64, True, "shaking"),
                                                            ("fp16", "mosaic", "nv12", 15, True, "fast")])
def test_out_frames_and_chains_equal_the_oracle(fast, shaking, prec, st, layout, L, motion, video):
    frames = fast[0] if video == "fast" else shaking
    matrix = "bt601" if layout == "nv12" else "bt709"
    dev, host = _in_frames(frames, layout)
    eng = _engine(prec)
    trk = eng.tracker(motion=motion or None, lookback=dict(frames=L), lookback_search=True)
    got, outs = _run(eng, trk, dev, layout, matrix, min(4, L), STYLES[st], seen=SEEN if video == "fast" else 8)
    k = min(L, len(frames))
    douts = _out_frames(k, layout)
    nums = trk.drain(0, _views(douts, layout), layout=layout, style=STYLES[st][0], shape=STYLES[st][1])
    eng.synchronize()
    tag = f"{prec} {st} {layout} L{L} {video}"
    ems, chains = _check_oracle(got, host, outs, layout, STYLES[st], L, motion, (nums, douts), tag)
    assert len(ems) == len(frames) and chains >= 1, (tag, chains)
    trk.close()
    eng.close()


@pytest.mark.parametrize("R,mad,layout,motion", [(16, 40.0, "nv12", False), (2, 10.0, "i420", True)])
def test_search_radius_extremes_equal_the_oracle(fast, R, mad, layout, motion):
    """R = 16 (64-pixel windows filling the shared arrays) and R = 2 (a 40 px step is out of reach: BORDER), with their own max_mad:
    out frames, step records and lengths equal the oracle's."""
    frames = fast[0]
    L = 15
    dev, host = _in_frames(frames, layout)
    eng = _engine("fp16")
    trk = eng.tracker(motion=motion or None, lookback=dict(frames=L), lookback_search=dict(search=R, max_mad=mad))
    got, outs = _run(eng, trk, dev, layout, "bt601", 4, STYLES["mosaic"])
    douts = _out_frames(L, layout)
    nums = trk.drain(0, _views(douts, layout), layout=layout, style=STYLES["mosaic"][0], shape=STYLES["mosaic"][1])
    eng.synchronize()
    ems, chains = _check_oracle(got, host, outs, layout, STYLES["mosaic"], L, motion, (nums, douts), f"R{R}", search=(R, mad))
    assert len(ems) == len(frames) and chains >= 1
    trk.close()
    eng.close()


def _d_mask(em, plain_count, m, b):
    """Luma and chroma masks of the samples the emission's (d) regions could cover (their snapped rectangles, one sample wider)."""
    ym = np.zeros((H, W), bool)
    for X0, Y0, X1, Y1, _ in regions(em.boxes[plain_count:], m, b):
        ym[max(int(Y0) - 1, 0):min(int(Y1) + 2, H), max(int(X0) - 1, 0):min(int(X1) + 2, W)] = True
    cm = ym.reshape(H // 2, 2, W // 2, 2).any(axis=(1, 3))
    return ym, cm


def test_bytes_outside_d_equal_plain_lookback_and_fast_face_is_covered(fast):
    """The same frames through a plain and a searching look-back tracker (FP16, NV12, blur + ellipse, L = 15): every byte outside
    the (d) regions is equal.  For the fast face, first born on frame b, on frames max(0, b - L) .. b - 1 where it lies wholly in the
    frame: its true box lies inside a (d) rectangle and the Laplacian variance inside it is below f14's bound of 2.5 (below 4 on the
    few far frames where a (c) growth region's edge crosses the face and two blur radii meet), while the plain tracker leaves it above
    2.5 on at least one of those frames."""
    frames, truth = fast
    L = 15
    dev, host = _in_frames(frames, "nv12")
    eng = _engine("fp16")
    outs = {}
    got = {}
    for name, kw in (("plain", {}), ("search", dict(lookback_search=True))):
        trk = eng.tracker(high_thresh=THR, new_thresh=THR, lookback=dict(frames=L), **kw)
        o = _out_frames(NF, "nv12")
        res = []
        views, ov = _views(dev, "nv12"), _views(o, "nv12")
        for s in range(0, NF, 4):
            r = trk.detect_yuv_redact_lookback_device(views[s:s + 4], [0] * 4, ov[s:s + 4], _thr(s), NMS, style="blur", shape="ellipse")
            res.append(trk.read(r[1], r[2], 4))
        d = _out_frames(L, "nv12")
        trk.drain(0, _views(d, "nv12"), style="blur", shape="ellipse")
        eng.synchronize()
        outs[name] = [x.cpu().numpy() for x in o[L:]] + [x.cpu().numpy() for x in d]       # frame e at index e
        got[name] = [t for r in res for t in r]
        trk.close()
    b_, m_ = params(0, 0.0)
    # the oracle's (d) boxes of each frame, from the device's lists (test_out_frames_and_chains_equal_the_oracle checks them bit for bit)
    lo = SearchLookbackOracle(L)
    ems = {}
    for t in range(NF):
        tr = got["search"][t]
        em = lo.push(0, Frame(host[t], [], births(tr), None), np.ascontiguousarray(host[t][:H, :W]))
        if em is not None:
            ems[em.number] = em
    for em in lo.drain(0):
        ems[em.number] = em
    plain_lo = __import__("oracle.lookback", fromlist=["LookbackOracle"]).LookbackOracle(L)
    counts = {}
    for t in range(NF):
        e = plain_lo.push(0, Frame(host[t], [], births(got["plain"][t]), None))
        if e is not None:
            counts[e.number] = len(e.boxes)
    for e in plain_lo.drain(0):
        counts[e.number] = len(e.boxes)
    for e in range(NF):
        ym, cm = _d_mask(ems[e], counts[e], m_, b_)
        a, s = outs["plain"][e], outs["search"][e]
        assert np.array_equal(a[:H, :W][~ym], s[:H, :W][~ym]), e
        ca, cs = a[H:H + H // 2, :W].reshape(H // 2, W // 2, 2), s[H:H + H // 2, :W].reshape(H // 2, W // 2, 2)
        assert np.array_equal(ca[~cm], cs[~cm]), e
    first = None
    for t, tracks in enumerate(got["search"]):
        for r in tracks:
            cx = (r["face"][1] + r["face"][3]) / 2
            x1, y1, x2, y2 = truth[t]
            if int(r["age"]) == 1 and x1 <= cx <= x2 and first is None:
                first = t
    assert first == SEEN, first
    bad, missed, checked, split = [], 0, 0, 0
    for e in range(max(0, first - L), first):
        gt = truth[e]
        if gt[2] > W:
            continue
        checked += 1
        d = regions(ems[e].boxes[counts[e]:], m_, b_)
        inside = any(X0 <= gt[0] and Y0 <= gt[1] and X1 >= gt[2] and Y1 >= gt[3] for X0, Y0, X1, Y1, _ in d)
        # a (c) growth region whose edge crosses the face owns part of it: two blur radii meet there (see DESIGN f17)
        crossed = any(X0 < gt[2] and X1 > gt[0] and Y0 < gt[3] and Y1 > gt[1] and not (X0 <= gt[0] and Y0 <= gt[1] and X1 >= gt[2] and
                                                                                     Y1 >= gt[3])
                      for X0, Y0, X1, Y1, _ in regions(ems[e].boxes[:counts[e]], m_, b_))
        v = _lap_var(outs["search"][e][:H, :W], gt)
        split += crossed
        if not inside or (not crossed and v >= 2.5) or v >= 4.0:
            bad.append((e, inside, crossed, round(float(v), 3)))
        missed += _lap_var(outs["plain"][e][:H, :W], gt) >= 2.5
    assert checked >= 10 and not bad and split <= 3, (first, checked, split, bad)
    assert missed >= 1, "f15's growth boxes alone cover the fast face: the video does not exercise the search"
    eng.close()


def _outs_of(eng, trk, dev, per_call, inplace=False, videos=None):
    if inplace:
        views = _views(dev, "nv12")
        for s in range(0, len(dev), per_call):
            m = min(per_call, len(dev) - s)
            trk.detect_yuv_redact_lookback_device(views[s:s + m], [0] * m if videos is None else videos[s:s + m], views[s:s + m], _thr(s),
                                                  NMS, style="mosaic", shape="ellipse")
        eng.synchronize()
        return dev
    return _run(eng, trk, dev, "nv12", "bt601", per_call, ("mosaic", "ellipse"), videos=videos)[1]


def test_call_shapes(fast):
    """1, 4 and 8 frames per call (the chains then read earlier frames of the call), in place and into out frames, two contexts, two
    interleaved videos, eight videos in one call against eight calls, and 2 streams + 1 calls in flight: bit-equal out frames."""
    import torch
    frames = fast[0]
    L = 8
    ref = None
    for per_call, inplace, streams in ((1, False, 1), (4, False, 1), (8, False, 1), (8, True, 2)):
        dev, _ = _in_frames(frames, "nv12")
        eng = _engine("fp16", streams=streams)
        trk = eng.tracker(lookback=dict(frames=L), lookback_search=True)
        outs = _outs_of(eng, trk, dev, per_call, inplace)
        planes = [o[:H + H // 2, :W].cpu() for o in outs[L:]]
        if ref is None:
            ref = planes
        assert all(torch.equal(a, b) for a, b in zip(ref, planes)), (per_call, inplace, streams)
        trk.close()
        eng.close()
    eng = _engine("fp16", streams=2)
    trk = eng.tracker(max_videos=2, lookback=dict(frames=L), lookback_search=True)
    dev, _ = _in_frames(frames + frames, "nv12")
    order = [i // 2 + NF * (i % 2) for i in range(2 * NF)]
    outs = _run(eng, trk, [dev[i] for i in order], "nv12", "bt601", 4, ("mosaic", "ellipse"), videos=[i % 2 for i in range(2 * NF)],
                seen=2 * SEEN)[1]
    for i in range(2 * NF):
        if i // 2 >= L:
            assert torch.equal(outs[i][:H + H // 2, :W].cpu(), ref[i // 2 - L]), i
    trk.close()
    eng.close()
    # eight videos, one frame of each per call, against each video alone
    n8 = 12
    eng = _engine("fp16")
    a = eng.tracker(max_videos=8, lookback=dict(frames=4), lookback_search=True)
    dev, _ = _in_frames(frames[:n8], "nv12")
    outs8 = _out_frames(8 * n8, "nv12")
    views, ov = _views(dev, "nv12"), _views(outs8, "nv12")
    for t in range(n8):
        a.detect_yuv_redact_lookback_device([views[(t + v) % n8] for v in range(8)], list(range(8)), ov[8 * t:8 * t + 8], _thr(t, 5),
                                            NMS, style="blur", shape="ellipse")
    eng.synchronize()
    for v in (0, 3, 7):
        b = eng.tracker(lookback=dict(frames=4), lookback_search=True)
        single = _run(eng, b, [dev[(t + v) % n8] for t in range(n8)], "nv12", "bt601", 1, ("blur", "ellipse"), seen=5)[1]
        for t in range(4, n8):
            assert torch.equal(single[t], outs8[8 * t + v]), (v, t)
        b.close()
    a.close()
    eng.close()
    for streams in (2,):
        k = 2 * streams + 1
        eng = _engine("fp16", streams=streams)
        res = []
        for sync in (False, True):
            trk = eng.tracker(lookback=dict(frames=2), lookback_search=True)
            dev, _ = _in_frames(frames[:k], "nv12")
            outs = _out_frames(k, "nv12")
            views, ov = _views(dev, "nv12"), _views(outs, "nv12")
            for s in range(k):
                trk.detect_yuv_redact_lookback_device([views[s]], [0], [ov[s]], _thr(s, 2), NMS, style="blur", shape="ellipse")
                if sync:
                    eng.synchronize()
            eng.synchronize()
            res.append([o.cpu() for o in outs])
            trk.close()
        assert all(torch.equal(x, y) for x, y in zip(*res)), streams
        eng.close()


def test_drain_and_reset_restart_the_chains(fast):
    """Across a reset the numbering restarts, so the first frame after it has no steps; drained frames carry (d) as the oracle does."""
    frames = fast[0]
    L = 6
    dev, host = _in_frames(frames[:8], "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(lookback=dict(frames=L), lookback_search=True)
    got, outs = _run(eng, trk, dev[:4], "nv12", "bt601", 2, STYLES["mosaic"], seen=2)
    douts = _out_frames(L, "nv12")
    nums = trk.drain(0, _views(douts, "nv12"), style="mosaic", shape="rect")
    eng.synchronize()
    _check_oracle(got, host[:4], outs, "nv12", STYLES["mosaic"], L, False, (nums, douts), "drain")
    trk.reset(0)
    got2, outs2 = _run(eng, trk, dev[4:], "nv12", "bt601", 2, STYLES["mosaic"], seen=0)
    assert all(int(n) == 0 for n in got2[0][6])            # number 0 after the reset: no frame before it
    _check_oracle(got2, host[4:], outs2, "nv12", STYLES["mosaic"], L, False, None, "after reset")
    trk.close()
    eng.close()


def test_refusals_launch_nothing(fast):
    """Each refusal returns RF_ERR_INVALID_ARG and changes nothing: the frames keep their bytes, a refused tracker then gives exactly
    the out frames, step records and lengths of a tracker that never saw the refused calls, and a tracker refused after an update
    stays a plain look-back tracker."""
    import torch
    from retinaface_b200 import capi
    eng = _engine("fp16", max_batch=4)
    lib = eng.lib
    dev, _ = _in_frames(fast[0][:4], "nv12")
    outs = {k: _out_frames(4, "nv12") for k in ("lb", "ref", "later", "plain_ref")}
    ins0, outs0 = [d.clone() for d in dev], [x.clone() for x in outs["lb"]]
    torch.cuda.synchronize()
    plain = eng.tracker()
    lb = eng.tracker(lookback=dict(frames=2))
    cfg = capi.FollowConfig(0, 0.0)
    p, q = C.c_void_p(), C.c_void_p()
    assert lib.rf_tracker_set_lookback_search(plain.t, C.byref(cfg)) == -1                 # not a look-back tracker
    for bad in ((17, 0.0), (-1, 0.0), (0, 256.0), (0, -1.0), (0, float("nan"))):
        assert lib.rf_tracker_set_lookback_search(lb.t, C.byref(capi.FollowConfig(*bad))) == -1, bad
    assert lib.rf_tracker_set_lookback_search(lb.t, None) == -1
    assert lib.rf_tracker_lookback_search(lb.t, C.byref(p), C.byref(q)) == -1             # refused: still not searching
    lb.set_lookback_search()
    assert lib.rf_tracker_set_lookback_search(lb.t, C.byref(capi.FollowConfig(3, 9.0))) == -1   # a second call
    assert lib.rf_tracker_lookback_search(lb.t, C.byref(p), C.byref(q)) == 0 and not p.value and not q.value
    eng.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(dev, ins0)) and all(torch.equal(a, b) for a, b in zip(outs["lb"], outs0))
    # the refused tracker against one that never saw a refusal: its first frame is number 0, and the second call kept the defaults
    ref = eng.tracker(lookback=dict(frames=2), lookback_search=True)
    later = eng.tracker(lookback=dict(frames=2))
    plain_ref = eng.tracker(lookback=dict(frames=2))
    res = {}
    for name, trk in (("lb", lb), ("ref", ref), ("later", later), ("plain_ref", plain_ref)):
        got, _ = _run(eng, trk, dev[:2], "nv12", "bt601", 1, ("blur", "ellipse"), outs=outs[name][:2], seen=1)
        if name == "later":
            assert lib.rf_tracker_set_lookback_search(later.t, C.byref(cfg)) == -1        # after an update
            assert lib.rf_tracker_lookback_search(later.t, C.byref(p), C.byref(q)) == -1
        views, ov = _views(dev[2:], "nv12"), _views(outs[name][2:], "nv12")
        for i in range(2):
            trk.detect_yuv_redact_lookback_device(views[i:i + 1], [0], ov[i:i + 1], THR, NMS, style="blur", shape="ellipse")
        eng.synchronize()
        res[name] = got
    assert [g[0] for g in res["lb"]] == [-1, -1]
    for a, b in zip(res["lb"], res["ref"]):       # lengths, and the steps taken (the rest of the rows is not written)
        assert np.array_equal(a[6], b[6]) and all(np.array_equal(a[5][r][:n], b[5][r][:n]) for r, n in enumerate(a[6]))
    assert int(res["ref"][1][6][0]) == 1, "the face born on frame 1 has no chain: the comparison checks nothing"
    assert all(torch.equal(a, b) for a, b in zip(outs["lb"], outs["ref"]))
    assert all(torch.equal(a, b) for a, b in zip(outs["later"], outs["plain_ref"]))
    for x in (plain, lb, ref, later, plain_ref):
        x.close()
    eng.close()


def test_detector_redact_frames_lookback_search(fast):
    import os
    import torch
    from conftest import GOLDEN
    from retinaface_b200.detector import RetinaFace
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    eng = det.engine
    with pytest.raises(ValueError):
        det.redactFrames([], [], lookback_search=True)
    dev, _ = _in_frames(fast[0][:6], "nv12")
    views = _views(dev, "nv12")
    a, b = _out_frames(6, "nv12"), _out_frames(6, "nv12")
    trk = eng.tracker(max_videos=64, lookback=dict(frames=3), lookback_search=True)
    for t in range(6):
        det.redactFrames([views[t]], [0], threshold=_thr(t, 2), lookback=3, lookback_search=True, out=_views(a[t:t + 1], "nv12"))
        trk.detect_yuv_redact_lookback_device([views[t]], [0], _views(b[t:t + 1], "nv12"), _thr(t, 2), det.nms_threshold)
    da, db = _out_frames(3, "nv12"), _out_frames(3, "nv12")
    assert list(det.drainVideo(0, _views(da, "nv12"))) == list(trk.drain(0, _views(db, "nv12")))
    eng.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a + da, b + db))
    trk.close()
