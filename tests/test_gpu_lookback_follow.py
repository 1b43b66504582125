"""GPU (-m gpu): f18 following look-back -- a look-back tracker that also takes follow frames.  Every out and drained frame of
rf_detect_yuv_redact_lookback_device and rf_track_follow_redact_lookback_device against oracle/lookback_follow.py byte for byte (pitch
padding included), fed the device's records; the lists, rf_follow records, motions, step records and the FP64 state against the
oracles'; the tracking equals a follow tracker's, k = 1 equals a plain look-back tracker, and bytes outside (c) and (d) equal the
undelayed f16 redaction; a face revealed on a follow frame is covered from the reveal on; call shapes, drain and reset mid-interval,
RetinaFace.redactFrames(lookback=L, detect_every=k); the admission table of the new kind."""
import ctypes as C

import numpy as np
import pytest

from oracle.follow import luma_of
from oracle.lookback import emit_into, regions
from oracle.lookback_follow import LookbackFollowOracle
from oracle.motion import MotionOracle, applied
from oracle.redact import params
from oracle.redact_style import redact_yuv, style
from test_gpu_follow import REC, _calls
from test_gpu_lookback import (H, OPITCH, PITCH, REVEAL, STYLES, W, _in_frames, _lap_var, _out_frames, _planted, _surface, _views)
from test_gpu_lookback_search import _same_steps
from test_gpu_motion import _same, _same_motion
from test_gpu_redact import _engine

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
TCFG = dict(high_thresh=THR, new_thresh=THR)


@pytest.fixture(scope="module")
def planted(golden_image):
    return _planted(golden_image)


@pytest.fixture(scope="module")
def shaking(golden_image):
    from test_gpu_motion import _shake
    return _shake(golden_image)[0]


def _st(name):
    return STYLES[name] if isinstance(name, str) else name


def _drive(eng, trk, views, oviews, vids, k, per_call, layout="nv12", matrix="bt601", st="mosaic", sync=True):
    """Every frame through the following look-back tracker: per chunk of per_call frames, the detect and follow sub-calls
    RetinaFace._interval_calls makes (numbering from 0).  Returns the issue order and per frame (kind, number, tracks, records or
    follow records, scale, motion, steps, lengths); with sync False nothing is read back."""
    st = _st(st)
    got, order = {}, []
    for det, idx in _calls(vids, k, per_call):
        fr, vv, oo, m = [views[i] for i in idx], [vids[i] for i in idx], [oviews[i] for i in idx], len(idx)
        order += idx
        if det:
            nums, tp, tc, d, c, sc = trk.detect_yuv_redact_lookback_device(fr, vv, oo, THR, NMS, layout=layout, matrix=matrix, style=st[0],
                                                                           shape=st[1])
        else:
            nums, tp, tc = trk.follow_redact_lookback_device(fr, vv, oo, layout=layout, style=st[0], shape=st[1])
        if not sync:
            continue
        tr = trk.read(tp, tc, m)
        mo = trk.motion(m) if trk.motion_on else [None] * m
        if det:
            recs = eng.read_dets(d, c, m)[0]
            steps, lens = trk.lookback_search(m) if trk.lookback_search_on else ([None] * m, [None] * m)
            for j, i in enumerate(idx):
                got[i] = ("detect", int(nums[j]), tr[j], recs[j], sc[j], mo[j], steps[j], lens[j])
        else:
            fo = trk.follow(m)
            for j, i in enumerate(idx):
                got[i] = ("follow", int(nums[j]), tr[j], fo[j, :len(tr[j])], None, mo[j], None, None)
    eng.synchronize()
    return order, got


class _Check:
    """The composed oracle fed the device's records in issue order; checks every frame's lists, follow records, motion, steps, number
    and out frame, and drained frames."""

    def __init__(self, layout, st, L, motion, search, nv=1, tag=""):
        self.o = LookbackFollowOracle(nv, L, search={} if search else None, **TCFG)
        self.mo = MotionOracle(nv) if motion else None
        self.layout, self.L, self.tag = layout, L, tag
        st = _st(st)
        self.b, self.m = params(0, 0.0)
        self.sty = style(1 if st[0] == "mosaic" else 2, 1 if st[1] == "rect" else 2)
        self.isurf, self.osurf = _surface(layout, PITCH), _surface(layout, OPITCH)
        self.emitted = self.followed = self.chains = 0
        self.ems = {}             # (video, number) -> (index of the frame that emitted it, Emitted, its own (a) + (b) boxes)

    def _out(self, canary, em, got_out, what):
        exp = emit_into(canary, em.data, self.layout, data_surface=self.isurf, **self.osurf)
        exp = redact_yuv(exp, self.layout, regions(em.boxes, self.m, self.b), self.sty, **self.osurf)
        assert np.array_equal(got_out, exp), (self.tag, what, em.number)

    def frames(self, order, got, host, vids, outs):
        canary = np.full(outs[0].shape, 0x5A, np.uint8)
        for i in order:
            kind, num, tracks, recs, sc, mrec, steps, lens = got[i]
            v, luma = vids[i], np.ascontiguousarray(luma_of(host[i], W, H))
            what = f"{self.tag} frame {i} ({kind})"
            mot = (int(mrec["status"]), tuple(mrec["m"])) if self.mo else None
            if kind == "detect":
                wm = self.mo.update(v, luma, recs, len(recs), float(sc)) if self.mo else None
                want, em = self.o.detect(v, host[i], luma, recs, sc, mot, applied(wm) if self.mo else None)
                if self.o.searching:
                    ch = self.o.lookback.log[v][(self.o.lookback.count[v] - 1) % (2 * self.L)].chains
                    _same_steps(steps, lens, ch, what)
                    self.chains += sum(1 for c in ch if c)
            else:
                faces = self.o.tracker.mask_faces(v)
                wm = self.mo.update(v, luma, faces, len(faces), None) if self.mo else None
                want, wf, em = self.o.follow(v, host[i], luma, mot, applied(wm) if self.mo else None)
                assert len(recs) == len(wf), what
                for r, w in zip(recs, wf):
                    assert all(int(r[f]) == int(w[f]) for f in REC), (what, r, w)
                    assert all(np.float32(r[f]).tobytes() == np.float32(w[f]).tobytes() for f in ("fx", "fy", "x1", "y1", "x2", "y2")), what
                self.followed += sum(int(r["followed"]) for r in tracks)
            if self.mo:
                _same_motion(mrec, wm, what)
            _same(tracks, want, what)
            assert [int(r["followed"]) for r in tracks] == [int(w["followed"]) for w in want], what
            assert num == (-1 if em is None else em.number), (what, num)
            got_out = outs[i].cpu().numpy()
            if em is None:
                assert np.array_equal(got_out, canary), what
            else:
                self._out(canary, em, got_out, what)
                self.emitted += 1
                self.ems[(v, em.number)] = (i, em, len(self.o.lookback.log[v][em.number % (2 * self.L)].boxes))

    def drain(self, video, nums, douts):
        want = self.o.drain(video)
        if self.mo:
            self.mo.reset(video)
        assert list(nums) == [e.number for e in want], (self.tag, list(nums))
        canary = np.full(douts[0].shape, 0x5A, np.uint8)
        for e, o in zip(want, douts):
            self._out(canary, e, o.cpu().numpy(), "drain")

    def reset(self, video):
        self.o.reset(video)
        if self.mo:
            self.mo.reset(video)


def _state_equal(trk, o, video=0):
    hdr, rows = trk.debug_state(video)
    assert np.array_equal(np.r_[hdr, rows.reshape(-1)].view(np.uint64), o.tracker.debug_state(video).view(np.uint64))


@pytest.mark.parametrize("prec,st,layout,L,k,motion,search,video", [
    ("fp16", ("blur", "ellipse"), "nv12", 15, 3, False, False, "planted"),
    ("fp32", ("mosaic", "rect"), "i420", 1, 2, True, False, "planted"),
    ("int8", ("blur", "rect"), "i420", 15, 5, True, True, "shaking"),
    ("fp16", ("mosaic", "ellipse"), "nv12", 4, 5, False, True, "planted")])
def test_out_frames_equal_the_oracle(planted, shaking, prec, st, layout, L, k, motion, search, video):
    frames = planted[0] if video == "planted" else shaking
    matrix = "bt601" if layout == "nv12" else "bt709"
    dev, host = _in_frames(frames, layout)
    outs = _out_frames(len(frames), layout)
    eng = _engine(prec)
    trk = eng.tracker(motion=motion or None, lookback=dict(frames=L), lookback_search=search or None, lookback_follow=True, **TCFG)
    vids = [0] * len(frames)
    order, got = _drive(eng, trk, _views(dev, layout), _views(outs, layout), vids, k, min(4, L), layout, matrix, st)
    tag = f"{prec} {layout} L{L} k{k} motion={motion} search={search} {video}"
    ck = _Check(layout, st, L, motion, search, tag=tag)
    ck.frames(order, got, host, vids, outs)
    _state_equal(trk, ck.o)
    douts = _out_frames(min(L, len(frames)), layout)
    nums = trk.drain(0, _views(douts, layout), layout=layout, style=st[0], shape=st[1])
    eng.synchronize()
    ck.drain(0, nums, douts)
    assert ck.emitted == max(0, len(frames) - L) and ck.followed > 0, (tag, ck.emitted, ck.followed)
    assert not search or video == "shaking" or ck.chains > 0, tag      # the shaking video's faces are all born on frame 0
    if video == "shaking":
        assert any(int(g[5]["status"]) == 0 for g in got.values() if g[0] == "follow"), tag
    trk.close()
    eng.close()


def _region_mask(boxes, m, b):
    """The NV12 samples (luma rows, then interleaved chroma rows, W bytes each) inside the rectangles of the boxes' regions."""
    mask = np.zeros((H + H // 2, W), bool)
    for X0, Y0, X1, Y1, _ in regions(boxes, m, b):
        x0, y0, x1, y1 = max(X0, 0), max(Y0, 0), min(X1, W), min(Y1, H)
        if x1 > x0 and y1 > y0:
            mask[y0:y1, x0:x1] = True
            mask[H + y0 // 2:H + y1 // 2, x0:x1] = True
    return mask


def test_tracking_and_bytes_equal_the_undelayed_follow_tracker(planted):
    """The same calls on a follow tracker (rf_detect_yuv_redact_device_style / rf_track_follow_redact_device, in place): lists and FP64
    state bit for bit, and every byte of each emitted frame outside its (c) regions equals what the undelayed call wrote on it."""
    import torch
    frames = planted[0]
    L, k = 6, 5
    dev, host = _in_frames(frames, "nv12")
    outs = _out_frames(len(frames), "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(motion=True, lookback=dict(frames=L), lookback_follow=True, **TCFG)
    vids = [0] * len(frames)
    order, got = _drive(eng, trk, _views(dev, "nv12"), _views(outs, "nv12"), vids, k, 4, st="mosaic")
    ref = eng.tracker(motion=True, follow=True, **TCFG)
    inplace = [d.clone() for d in dev]
    torch.cuda.synchronize()
    views = _views(inplace, "nv12")
    lists = {}
    for det, idx in _calls(vids, k, 4):
        fr = [views[i] for i in idx]
        if det:
            tp, tc = ref.detect_yuv_redact_device(fr, [0] * len(idx), THR, NMS, style="mosaic", shape="rect")[:2]
        else:
            tp, tc = ref.follow_redact_device(fr, [0] * len(idx), style="mosaic", shape="rect")
        for j, tr in enumerate(ref.read(tp, tc, len(idx))):
            lists[idx[j]] = tr
    eng.synchronize()
    for i in order:
        assert got[i][2].tobytes() == lists[i].tobytes(), i
    a, b = trk.debug_state(0), ref.debug_state(0)
    assert all(np.array_equal(x.view(np.uint64), y.view(np.uint64)) for x, y in zip(a, b))
    ck = _Check("nv12", "mosaic", L, True, False, tag="undelayed")
    ck.frames(order, got, host, vids, outs)
    bb, mm = params(0, 0.0)
    checked = 0
    for (_, e), (i, em, own) in sorted(ck.ems.items()):
        keep = ~_region_mask(em.boxes[own:], mm, bb)
        out, und = outs[i].cpu().numpy()[:, :W], inplace[e].cpu().numpy()[:, :W]
        assert np.array_equal(out[keep], und[keep]), (i, e)
        checked += 1
    assert checked == len(frames) - L
    trk.close()
    ref.close()
    eng.close()


def test_k1_equals_a_plain_lookback_tracker(planted):
    """With every frame a detect frame the following look-back tracker's out frames, numbers and lists are a plain look-back tracker's."""
    import torch
    frames = planted[0][:20]
    L = 4
    res = []
    eng = _engine("fp16")
    for follow in (True, False):
        dev, _ = _in_frames(frames, "nv12")
        outs = _out_frames(len(frames), "nv12")
        trk = eng.tracker(lookback=dict(frames=L), lookback_follow=follow or None, lookback_search=True)
        order, got = _drive(eng, trk, _views(dev, "nv12"), _views(outs, "nv12"), [0] * len(frames), 1, 4, st="blur")
        res.append(([o.cpu() for o in outs], [(got[i][1], got[i][2].tobytes()) for i in order]))
        trk.close()
    assert all(torch.equal(a, b) for a, b in zip(res[0][0], res[1][0])) and res[0][1] == res[1][1]
    eng.close()


def test_a_face_revealed_on_a_follow_frame_is_covered(planted):
    """The occluded face is revealed on frame 12, a follow frame at k = 5: f16's redaction alone leaves its true box untouched on some
    frame before the next key frame; the following look-back tracker at L = k - 1 covers it with a region rectangle on every frame
    from the reveal to the key frame after its first detection, blurred below f14's Laplacian bound."""
    import torch
    frames, truth = planted
    L, k = 4, 5
    dev, host = _in_frames(frames, "nv12")
    outs = _out_frames(len(frames), "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(lookback=dict(frames=L), lookback_follow=True, **TCFG)
    vids = [0] * len(frames)
    order, got = _drive(eng, trk, _views(dev, "nv12"), _views(outs, "nv12"), vids, k, 4, st=("blur", "rect"))
    gt0 = truth[REVEAL]["occluded"]
    born = [t for t in sorted(got) if got[t][0] == "detect" and any(
        int(r["age"]) == 1 and gt0[0] <= (r["face"][1] + r["face"][3]) / 2 <= gt0[2] for r in got[t][2])]
    assert born and born[0] >= REVEAL and born[0] - REVEAL <= L, born
    b = born[0]
    # f16 alone: the same calls on a follow tracker, redacting in place
    ref = eng.tracker(follow=True, **TCFG)
    f16 = [d.clone() for d in dev]
    torch.cuda.synchronize()
    v16 = _views(f16, "nv12")
    for det, idx in _calls(vids, k, 4):
        fr = [v16[i] for i in idx]
        if det:
            ref.detect_yuv_redact_device(fr, [0] * len(idx), THR, NMS, style="blur", shape="rect")
        else:
            ref.follow_redact_device(fr, [0] * len(idx), style="blur", shape="rect")
    eng.synchronize()
    x1, y1, x2, y2 = gt0
    leaked = [e for e in range(REVEAL, b) if np.array_equal(f16[e].cpu().numpy()[y1:y2, x1:x2], host[e][y1:y2, x1:x2])]
    assert leaked, "f16 covers the revealed face before its first detection: the test shows nothing"
    ck = _Check("nv12", ("blur", "rect"), L, False, False, tag="reveal")
    ck.frames(order, got, host, vids, outs)
    bb, mm = params(0, 0.0)
    bad = []
    for e in range(REVEAL, min(b + k + 1, len(frames) - L)):
        i, em, _ = ck.ems[(0, e)]
        inside = any(X0 <= x1 and Y0 <= y1 and X1 >= x2 and Y1 >= y2 for X0, Y0, X1, Y1, _ in regions(em.boxes, mm, bb))
        v = _lap_var(outs[i].cpu().numpy()[:H, :W], gt0)
        if not (inside and v < 2.5):
            bad.append((e, inside, round(float(v), 3)))
    assert not bad, (b, leaked, bad)
    trk.close()
    ref.close()
    eng.close()


def test_call_shapes_contexts_and_in_flight(planted):
    """1, 4 and 8 frames per call, in place and into out frames, on one and two contexts: the emitted frames are bit-equal; two videos
    interleaved in every call equal each video alone; 2 streams + 1 calls in flight equal the same calls read back one by one."""
    import torch
    frames = planted[0][:24]
    L, k = 8, 3
    ref = None
    for per_call, inplace, streams in ((1, False, 1), (4, False, 1), (8, False, 1), (4, True, 1), (8, True, 2)):
        dev, _ = _in_frames(frames, "nv12")
        eng = _engine("fp16", streams=streams)
        trk = eng.tracker(lookback=dict(frames=L), lookback_follow=True)
        outs = dev if inplace else _out_frames(len(frames), "nv12")
        _drive(eng, trk, _views(dev, "nv12"), _views(outs, "nv12"), [0] * 24, k, per_call)
        planes = [o[:H + H // 2, :W].cpu() for o in outs[L:]]
        if ref is None:
            ref = planes
        assert all(torch.equal(a, b) for a, b in zip(ref, planes)), (per_call, inplace, streams)
        trk.close()
        eng.close()
    eng = _engine("fp16", streams=2)
    trk = eng.tracker(max_videos=2, lookback=dict(frames=L), lookback_follow=True)
    dev, _ = _in_frames(frames[:12] + frames[:12], "nv12")
    order = [i // 2 + 12 * (i % 2) for i in range(24)]
    outs = _out_frames(24, "nv12")
    _drive(eng, trk, _views([dev[i] for i in order], "nv12"), _views(outs, "nv12"), [i % 2 for i in range(24)], k, 4)
    for i in range(24):
        if i // 2 >= L:
            assert torch.equal(outs[i][:H + H // 2, :W].cpu(), ref[i // 2 - L]), i
    trk.close()
    eng.close()
    for streams in (2, 8):
        n = 2 * streams + 1
        eng = _engine("fp16", streams=streams)
        res = []
        for sync in (True, False):
            trk = eng.tracker(lookback=dict(frames=4), lookback_follow=True)
            dev, _ = _in_frames(planted[0][:n], "nv12")
            outs = _out_frames(n, "nv12")
            _drive(eng, trk, _views(dev, "nv12"), _views(outs, "nv12"), [0] * n, k, 1, sync=sync)
            res.append([o.cpu() for o in outs])
            trk.close()
        assert all(torch.equal(x, y) for x, y in zip(*res)), streams
        eng.close()


def test_drain_and_reset_mid_interval(planted):
    """A drain after a follow frame emits the buffered frames (follow frames among them) as the oracle does and restarts the count and
    the templates; a reset mid-interval emits nothing and the next frame is number 0 -- against the oracle throughout."""
    frames = planted[0][:22]
    L, k = 4, 3
    dev, host = _in_frames(frames, "nv12")
    outs = _out_frames(len(frames), "nv12")
    views, ov = _views(dev, "nv12"), _views(outs, "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(lookback=dict(frames=L), lookback_follow=True, **TCFG)
    ck = _Check("nv12", "mosaic", L, False, False, tag="drain/reset")
    segs = (range(0, 8), range(8, 15), range(15, 22))     # 8 frames, drain; 7 frames, reset; 7 frames, drain
    for n_seg, seg in enumerate(segs):
        idx = list(seg)
        order, got = _drive(eng, trk, [views[i] for i in idx], [ov[i] for i in idx], [0] * len(idx), k, 4)
        ck.frames(order, got, [host[i] for i in idx], [0] * len(idx), [outs[i] for i in idx])
        if n_seg == 1:
            trk.reset(0)
            ck.reset(0)
            continue
        douts = _out_frames(L, "nv12")
        nums = trk.drain(0, _views(douts, "nv12"))
        eng.synchronize()
        assert len(nums) == min(L, len(idx))
        ck.drain(0, nums, douts)
    _state_equal(trk, ck.o)
    trk.close()
    eng.close()


def test_detector_redact_frames_lookback_detect_every(planted):
    """RetinaFace.redactFrames(lookback=L, detect_every=k, out=...) issues the calls a following look-back tracker takes and returns
    every frame's number in input order; drainVideo restarts the video's numbering, so the next frame is a key frame again."""
    import os
    import torch
    from conftest import GOLDEN
    from retinaface_b200.detector import RetinaFace
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    eng = det.engine
    frames = planted[0][:14]
    dev, _ = _in_frames(frames, "nv12")
    views = _views(dev, "nv12")
    a, b = _out_frames(14, "nv12"), _out_frames(14, "nv12")
    va, vb = _views(a, "nv12"), _views(b, "nv12")
    L, k = 3, 3
    trk = eng.tracker(max_videos=64, lookback=dict(frames=L), lookback_follow=True)
    nums = []
    for s in (0, 5):
        nums += list(det.redactFrames(views[s:s + 5], [0] * 5, threshold=THR, lookback=L, detect_every=k, out=va[s:s + 5]))
    assert det._tracker.lookback_follow_on and not det._tracker.follow_on
    ref = []
    for d, idx in _calls([0] * 10, k, 5):
        fr, oo = [views[i] for i in idx], [vb[i] for i in idx]
        if d:
            got = trk.detect_yuv_redact_lookback_device(fr, [0] * len(idx), oo, THR, det.nms_threshold)[0]
        else:
            got = trk.follow_redact_lookback_device(fr, [0] * len(idx), oo)[0]
        ref += list(zip(idx, got))
    assert nums == [int(n) for _, n in sorted(ref)] == [-1] * L + list(range(10 - L))
    da, db = _out_frames(L, "nv12"), _out_frames(L, "nv12")
    assert list(det.drainVideo(0, _views(da, "nv12"))) == list(range(10 - L, 10)) == list(trk.drain(0, _views(db, "nv12")))
    # after the drain frame 10 is number 0: a key frame for both
    n2 = det.redactFrames(views[10:14], [0] * 4, threshold=THR, lookback=L, detect_every=k, out=va[10:14])
    ref2 = {}
    for d, idx in _calls([0] * 4, k, 4):
        fr, oo = [views[10 + i] for i in idx], [vb[10 + i] for i in idx]
        got = (trk.detect_yuv_redact_lookback_device(fr, [0] * len(idx), oo, THR, det.nms_threshold) if d else
               trk.follow_redact_lookback_device(fr, [0] * len(idx), oo))[0]
        ref2.update(zip(idx, got))
    assert list(n2) == [int(ref2[i]) for i in range(4)] == [-1, -1, -1, 0]
    eng.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a + da, b + db))
    with pytest.raises(ValueError):
        det.redactFrames(views[:1], [0], detect_every=2)            # no lookback: this tracker is not a follow tracker
    trk.close()


# ---- admission ---------------------------------------------------------------------------------------------------------------------
NEW_KINDS = {
    "lbfollow": dict(lookback=2, lookback_follow=True), "lbfollow+motion": dict(lookback=2, lookback_follow=True, motion=True),
    "lbfollow+search": dict(lookback=2, lookback_follow=True, lookback_search=True),
}
ONLY_LBF = ("a following look-back tracker takes frames only through rf_detect_yuv_redact_lookback_device and "
            "rf_track_follow_redact_lookback_device")
NOT_LBF = "not a following look-back tracker (rf_tracker_set_lookback_follow)"


def _why_new(call, motion, search, updated):
    """The admission table of a following look-back tracker: None (taken) or the refusal's reason."""
    from test_gpu_tracker_kinds import UPDATED
    if call in ("update", "detect", "detect_redact", "follow", "follow_redact"):
        return ONLY_LBF
    if call in ("best", "finish"):
        return "not a best-shot tracker (rf_tracker_create_best)"
    if call in ("lookback", "drain", "follow_lookback", "q_follow"):
        return None
    if call == "q_motion":
        return None if motion else "motion is off (rf_tracker_set_motion)"
    if call == "q_search":
        return None if search else "not a searching look-back tracker (rf_tracker_set_lookback_search)"
    why = {"set_motion": "motion is already on" if motion else None, "set_follow": "a look-back tracker cannot follow",
           "set_lookback": "look-back is already on", "set_lookback_search": "the look-back search is already on" if search else None,
           "set_lookback_follow": "look-back following is already on"}[call]
    return why or (UPDATED if updated else None)


def _call(rig, name, t):
    lib = rig.lib
    p, q = C.c_void_p(), C.c_void_p()
    if name == "follow_lookback":
        vids = (C.c_int * 1)(0)
        return lib.rf_track_follow_redact_lookback_device(t, rig.frames, vids, 1, C.byref(rig.style), rig.outs, rig.nums.ctypes.data,
                                                          C.byref(p), C.byref(q))
    if name == "set_lookback_follow":
        return lib.rf_tracker_set_lookback_follow(t, C.byref(rig.capi.FollowConfig(0, 0.0)))
    return rig.call(name, t)


@pytest.fixture(scope="module")
def rig():
    from test_gpu_tracker_kinds import _Rig
    r = _Rig()
    yield r
    r.eng.close()


@pytest.mark.parametrize("updated", [False, True], ids=["fresh", "updated"])
@pytest.mark.parametrize("kind", list(NEW_KINDS) + ["plain", "best", "follow+motion", "lookback", "lookback+search"])
def test_admission_table(rig, kind, updated):
    """Every call on a following look-back tracker, and the two new calls on the existing kinds: status and message; a refused call
    leaves the state, the frames and the follow records untouched."""
    import torch
    from test_gpu_tracker_kinds import KINDS, MAX_TRACKS, WHO, _snapshot, _why
    who = dict(WHO, follow_lookback="rf_track_follow_redact_lookback_device", set_lookback_follow="rf_tracker_set_lookback_follow")
    new = kind in NEW_KINDS
    base = kind.split("+")[0]
    motion, search = "motion" in kind, "search" in kind
    for call in who:
        trk = rig.eng.tracker(max_tracks=MAX_TRACKS, **(NEW_KINDS[kind] if new else KINDS[kind]))
        if updated:
            assert _call(rig, rig.first_call("lookback" if new else kind), trk.t) == 0, (kind, call)
        before = _snapshot(rig, trk)
        if new:
            why = _why_new(call, motion, search, updated)
        elif call == "follow_lookback":
            why = NOT_LBF
        elif call == "set_lookback_follow":
            from test_gpu_tracker_kinds import UPDATED
            why = "not a look-back tracker (rf_tracker_set_lookback)" if base != "lookback" else UPDATED if updated else None
        else:
            why = _why(call, base, motion, search, updated)
        rc = _call(rig, call, trk.t)
        if why is None:
            assert rc == 0, (kind, updated, call, rig.lib.rf_last_error(rig.eng.h))
        else:
            assert rc == -1, (kind, updated, call, rc)
            assert rig.lib.rf_last_error(rig.eng.h).decode() == f"{who[call]}: {why}", (kind, updated, call)
            after = _snapshot(rig, trk)
            assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1]), (kind, updated, call)
            assert torch.equal(before[2], after[2]) and torch.equal(before[3], after[3]), (kind, updated, call)
        trk.close()


def test_setter_order_and_bad_configs():
    """rf_tracker_set_lookback_follow before rf_tracker_set_motion and rf_tracker_set_lookback_search is taken; bad values are refused
    and leave a look-back tracker that then takes no follow call."""
    from retinaface_b200 import capi
    eng = _engine("fp16", max_batch=2)
    lib = eng.lib
    t = eng.tracker(lookback=2)
    for bad in ((17, 0.0), (-1, 0.0), (0, 256.0), (0, -1.0), (0, float("nan"))):
        assert lib.rf_tracker_set_lookback_follow(t.t, C.byref(capi.FollowConfig(*bad))) == -1, bad
    assert lib.rf_tracker_set_lookback_follow(t.t, None) == -1
    assert lib.rf_tracker_follow(t.t, C.byref(C.c_void_p())) == -1          # still a look-back tracker without following
    t.set_lookback_follow()
    t.set_motion()
    t.set_lookback_search()
    assert lib.rf_tracker_follow(t.t, C.byref(C.c_void_p())) == 0
    t.close()
    with pytest.raises(capi.RfError):
        eng.tracker(follow=True, lookback=2)
    with pytest.raises(capi.RfError):
        eng.tracker(lookback_follow=True)                                      # not a look-back tracker
    eng.close()
