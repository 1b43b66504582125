"""GPU (-m gpu): f15 look-back redaction -- every out frame of rf_detect_yuv_redact_lookback_device and rf_tracker_drain against
oracle/lookback.py byte for byte (every plane byte, pitch padding included), fed the device's records and scales and the tracks and
motions of oracle/track.py / oracle/motion.py (checked bit for bit against the device's); that faces are covered on the frames before
their first detection where the undelayed call leaves them; grouping, contexts and calls in flight; drain and reset; the refusals."""
import ctypes as C

import cv2
import numpy as np
import pytest

from oracle.lookback import Frame, LookbackOracle, births, emit_into, frame_boxes, regions
from oracle.motion import MotionOracle, MotionTrackerOracle, applied
from oracle.redact import params
from oracle.redact_style import redact_yuv, style
from oracle.track import TrackerOracle
from oracle.yuv import bgr_to_frame
from test_gpu_motion import _same, _same_motion, _scene, _shake
from test_gpu_redact import _engine

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
W, H, NF = 1920, 1080, 40
PITCH, OPITCH = 2048, 1984              # input surfaces (NVDEC-like) and out surfaces: pitches are free
STYLES = {"blur": ("blur", "ellipse"), "mosaic": ("mosaic", "rect")}
# the planted face: the golden photo's face [462, 267, 573, 416] with half its size of context, scaled 2x; FACE is its box in the patch
CROP = (407, 192, 628, 491)
FACE = (110, 150, 332, 448)
PY = 240
REVEAL, SHARP, SPEED = 12, 20, 6        # occluder lifted on frame 12, blur (sigma 4) ends on frame 20, entering at 6 px per frame


def _patch(golden):
    x0, y0, x1, y1 = CROP
    return cv2.resize(golden[y0:y1, x0:x1], None, fx=2, fy=2, interpolation=cv2.INTER_LINEAR)


def _enter_x(t):
    return 1830 - SPEED * t


def _planted(golden):
    """NF BGR frames: a textured scene with four copies of the face -- still at x 20, revealed from behind a textured occluder on frame
    REVEAL at x 480, blurred with sigma 4 until frame SHARP at x 940, and entering from the right edge at SPEED px per frame -- and
    each copy's ground-truth face box per frame."""
    S = _scene(3, 2400, 1400)
    p = _patch(golden)
    ph, pw = p.shape[:2]
    blurred = cv2.GaussianBlur(p, (0, 0), 4)
    occ = S[900:900 + FACE[3] - FACE[1] + 40, 100:100 + FACE[2] - FACE[0] + 40]
    frames, truth = [], []
    for t in range(NF):
        f = S[:H, :W].copy()
        f[PY:PY + ph, 20:20 + pw] = p
        f[PY:PY + ph, 480:480 + pw] = p
        if t < REVEAL:
            f[PY + FACE[1] - 20:PY + FACE[3] + 20, 480 + FACE[0] - 20:480 + FACE[2] + 20] = occ
        f[PY:PY + ph, 940:940 + pw] = blurred if t < SHARP else p
        x = _enter_x(t)
        if x < W:
            f[PY:PY + ph, x:min(W, x + pw)] = p[:, :min(W, x + pw) - x]
        frames.append(f)
        truth.append({k: (x0 + FACE[0], PY + FACE[1], x0 + FACE[2], PY + FACE[3]) for k, x0 in
                      (("still", 20), ("occluded", 480), ("blurred", 940), ("entering", x))})
    return frames, truth


@pytest.fixture(scope="module")
def planted(golden_image):
    return _planted(golden_image)


@pytest.fixture(scope="module")
def shaking(golden_image):
    return _shake(golden_image)[0]


def _in_frames(frames, layout):
    """Device input frames and their host buffers: NV12 in pitched surfaces (0xEE padding), or packed I420."""
    import torch
    dev, host = [], []
    for f in frames:
        buf = bgr_to_frame(f, layout)
        if layout == "nv12":
            surf = np.full((H + H // 2, PITCH), 0xEE, np.uint8)
            surf[:, :W] = buf
            buf = surf
        host.append(buf)
        dev.append(torch.from_numpy(buf).cuda())
    torch.cuda.synchronize()
    return dev, host


def _views(dev, layout):
    return [(d[:H, :W], d[H:, :W]) for d in dev] if layout == "nv12" else dev


def _surface(layout, pitch):
    if layout == "nv12":
        return dict(width=W, height=H, y_pitch=pitch, uv_offset=pitch * H, uv_pitch=pitch)
    return dict(width=W, height=H)


def _out_frames(n, layout):
    """n device out frames with 0x5A canaries: NV12 surfaces of pitch OPITCH, or packed I420 buffers."""
    import torch
    shape = (H + H // 2, OPITCH) if layout == "nv12" else (H + H // 2, W)
    outs = [torch.full(shape, 0x5A, dtype=torch.uint8, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    return outs


def _run(eng, trk, dev, layout, matrix, per_call, st, outs=None, videos=None, **kw):
    """The frames through the look-back call, per_call per call; returns (per frame: number, tracks, records, scale, motion) and the
    out frames."""
    outs = outs if outs is not None else _out_frames(len(dev), layout)
    views, oviews = _views(dev, layout), _views(outs, layout)
    got = []
    for s in range(0, len(dev), per_call):
        m = min(per_call, len(dev) - s)
        vids = [0] * m if videos is None else videos[s:s + m]
        nums, tp, tc, d, c, sc = trk.detect_yuv_redact_lookback_device(views[s:s + m], vids, oviews[s:s + m], THR, NMS, layout=layout,
                                                                       matrix=matrix, style=st[0], shape=st[1], **kw)
        recs = eng.read_dets(d, c, m)[0]
        tr = trk.read(tp, tc, m)
        mo = trk.motion(m) if trk.motion_on else [None] * m
        got += [(int(nums[i]), tr[i], recs[i], sc[i], mo[i]) for i in range(m)]
    eng.synchronize()
    return got, outs


def _check_oracle(got, host, outs, layout, st, L, motion, drained=None, tag=""):
    """Every emitted out frame (and the drained ones) against the look-back oracle over the oracle trackers' lists."""
    b, m = params(0, 0.0)
    sty = style(*(1 if st[0] == "mosaic" else 2, 1 if st[1] == "rect" else 2))
    lo = LookbackOracle(L)
    to = MotionTrackerOracle(1) if motion else TrackerOracle(1)
    mo = MotionOracle(1) if motion else None
    isurf, osurf = _surface(layout, PITCH), _surface(layout, OPITCH)
    canary = np.full(outs[0].shape, 0x5A, np.uint8)
    emitted = 0
    for t, (num, tracks, recs, sc, mrec) in enumerate(got):
        if motion:
            luma = host[t][:H, :W]
            want_m = mo.update(0, luma, recs, len(recs), float(sc))
            _same_motion(mrec, want_m, f"{tag} frame {t}")
            want = to.update(0, recs, sc, motion=applied(want_m))
        else:
            want = to.update(0, recs, sc)
        _same(tracks, want, f"{tag} frame {t}")
        fr = Frame(host[t], frame_boxes(recs, len(recs), float(sc), want), births(want),
                   (int(mrec["status"]), tuple(mrec["m"])) if motion else None)
        em = lo.push(0, fr)
        assert num == (-1 if em is None else em.number), (tag, t, num)
        got_out = outs[t].cpu().numpy()
        if em is None:
            assert np.array_equal(got_out, canary), (tag, t)
            continue
        exp = emit_into(canary, em.data, layout, data_surface=isurf, **osurf)
        exp = redact_yuv(exp, layout, regions(em.boxes, m, b), sty, **osurf)
        assert np.array_equal(got_out, exp), (tag, t, em.number)
        emitted += 1
    if drained is not None:
        nums, douts = drained
        want = lo.drain(0)
        assert list(nums) == [e.number for e in want], (tag, list(nums))
        for e, o in zip(want, douts):
            exp = emit_into(canary, e.data, layout, data_surface=isurf, **osurf)
            exp = redact_yuv(exp, layout, regions(e.boxes, m, b), sty, **osurf)
            assert np.array_equal(o.cpu().numpy(), exp), (tag, "drain", e.number)
    return emitted


@pytest.mark.parametrize("prec,st,layout,L,motion,video", [("fp16", "blur", "nv12", 15, False, "planted"),
                                                            ("fp32", "mosaic", "i420", 1, True, "planted"),
                                                            ("int8", "blur", "i420", 64, True, "shaking"),
                                                            ("fp16", "mosaic", "nv12", 15, True, "shaking")])
def test_out_frames_equal_the_oracle(planted, shaking, prec, st, layout, L, motion, video):
    frames = planted[0] if video == "planted" else shaking
    matrix = "bt601" if layout == "nv12" else "bt709"
    dev, host = _in_frames(frames, layout)
    eng = _engine(prec)
    trk = eng.tracker(motion=motion or None, lookback=dict(frames=L))
    got, outs = _run(eng, trk, dev, layout, matrix, min(4, L), STYLES[st])       # a video appears at most L times per call
    k = min(L, len(frames))
    douts = _out_frames(k, layout)
    nums = trk.drain(0, _views(douts, layout), layout=layout, style=STYLES[st][0], shape=STYLES[st][1])
    eng.synchronize()
    n = _check_oracle(got, host, outs, layout, STYLES[st], L, motion, (nums, douts), f"{prec} {st} {layout} L{L} {video}")
    assert n == max(0, len(frames) - L) and len(nums) == k
    trk.close()
    eng.close()


def _lap_var(luma, box):
    x1, y1, x2, y2 = (int(round(v)) for v in box)
    x1, y1, x2, y2 = max(x1, 0), max(y1, 0), min(x2, W), min(y2, H)
    lap = cv2.Laplacian(luma[y1:y2, x1:x2].astype(np.float64), cv2.CV_64F)
    return lap[1:-1, 1:-1].var()


def test_faces_are_covered_before_their_first_detection(planted):
    """For each planted face, first born on frame b: on frames max(0, b - L) .. b - 1 its ground-truth box (clipped to the frame) lies
    inside a look-back region's rectangle for every k -- grow * w >= SPEED for these ~220 px faces, so the bound is k <= L -- and the
    blurred Laplacian variance inside it is below f14's bound of 2.5; through rf_detect_yuv_redact_device_style the same frames keep the
    face's original pixels."""
    import torch
    frames, truth = planted
    L = 15
    dev, host = _in_frames(frames, "nv12")
    eng = _engine("fp16")
    trk = eng.tracker(high_thresh=THR, new_thresh=THR, lookback=dict(frames=L))
    got, outs = _run(eng, trk, dev, "nv12", "bt601", 4, STYLES["blur"])
    plain = eng.tracker(high_thresh=THR, new_thresh=THR)
    f12 = [d.clone() for d in dev]
    torch.cuda.synchronize()
    for s in range(0, NF, 4):
        plain.detect_yuv_redact_device(_views(f12[s:s + 4], "nv12"), [0] * 4, THR, NMS, style="blur", shape="ellipse")
    eng.synchronize()
    b_, m_ = params(0, 0.0)
    first = {}
    for t, (_, tracks, _, _, _) in enumerate(got):
        for r in tracks:
            if int(r["age"]) == 1:
                cx, cy = (r["face"][1] + r["face"][3]) / 2, (r["face"][2] + r["face"][4]) / 2
                for name, (x1, y1, x2, y2) in truth[t].items():
                    if max(x1, 0) <= cx <= min(x2, W) and y1 <= cy <= y2:
                        first.setdefault(name, (t, r))
    assert set(first) == {"still", "occluded", "blurred", "entering"}, {k: v[0] for k, v in first.items()}
    assert first["occluded"][0] >= REVEAL and first["entering"][0] >= L, {k: v[0] for k, v in first.items()}
    bad, checked = [], 0
    for name, (b, rec) in first.items():
        for e in range(max(0, b - L), b):
            em_frame = e + L                       # the call frame that emitted frame e
            out = outs[em_frame].cpu().numpy()
            luma = out[:H, :W]
            gt = truth[e][name]
            gt = (max(gt[0], 0), max(gt[1], 0), min(gt[2], W), min(gt[3], H))
            if gt[2] - gt[0] < 8:
                continue
            boxes = regions(_lookback_boxes(got, e, L), m_, b_)
            inside = any(X0 <= gt[0] and Y0 <= gt[1] and X1 >= gt[2] and Y1 >= gt[3] for X0, Y0, X1, Y1, _ in boxes)
            v = _lap_var(luma, gt)
            orig = host[e][:H, :W]
            kept = np.array_equal(f12[e].cpu().numpy()[:H, :W][gt[1]:gt[3], gt[0]:gt[2]], orig[gt[1]:gt[3], gt[0]:gt[2]])
            if not (inside and v < 2.5 and kept):
                bad.append((name, b, e, gt, inside, round(float(v), 3), kept))
            checked += 1
    assert checked >= L and not bad, (checked, bad)
    trk.close()
    plain.close()
    eng.close()


def _lookback_boxes(got, e, L):
    """The (c) boxes of frame e from the device's own track lists (the oracle equality test checks them against the tracker oracle)."""
    from oracle.lookback import lookback_box
    out = []
    for b in range(e + 1, min(e + L, len(got) - 1) + 1):
        for _, face in births(got[b][1]):
            out.append(lookback_box(face, b - e, float(np.float32(0.1))))
    return out


def _run_outs(eng, trk, dev, per_call, inplace=False, videos=None):
    import torch
    if inplace:
        outs = dev
        views = _views(dev, "nv12")
        for s in range(0, len(dev), per_call):
            m = min(per_call, len(dev) - s)
            trk.detect_yuv_redact_lookback_device(views[s:s + m], [0] * m if videos is None else videos[s:s + m], views[s:s + m], THR, NMS,
                                                  style="mosaic", shape="ellipse")
        eng.synchronize()
        return outs
    return _run(eng, trk, dev, "nv12", "bt601", per_call, ("mosaic", "ellipse"), videos=videos)[1]


def test_grouping_contexts_and_in_place(planted):
    """1, 4 and 8 frames per call, in place and into separate out frames, and two interleaved videos over two contexts: the emitted
    frames are bit-equal (an in-place call leaves frame num - L in frame num's surface)."""
    import torch
    frames = planted[0][:24]
    L = 8
    ref = None
    for per_call, inplace, streams in ((1, False, 1), (4, False, 1), (8, False, 1), (4, True, 1), (8, True, 2)):
        dev, _ = _in_frames(frames, "nv12")
        eng = _engine("fp16", streams=streams)
        trk = eng.tracker(lookback=dict(frames=L))
        outs = _run_outs(eng, trk, dev, per_call, inplace)
        planes = [o[:H + H // 2, :W].cpu() for o in outs[L:]]
        if ref is None:
            ref = planes
        assert all(torch.equal(a, b) for a, b in zip(ref, planes)), (per_call, inplace, streams)
        trk.close()
        eng.close()
    # two videos interleaved one frame each per call over two contexts, against each video alone
    eng = _engine("fp16", streams=2)
    trk = eng.tracker(max_videos=2, lookback=dict(frames=L))
    dev, _ = _in_frames(frames[:12] + frames[:12], "nv12")
    order = [i // 2 + 12 * (i % 2) for i in range(24)]
    outs = _run(eng, trk, [dev[i] for i in order], "nv12", "bt601", 2, ("mosaic", "ellipse"), videos=[i % 2 for i in range(24)])[1]
    for i in range(24):
        if i // 2 >= L:
            assert torch.equal(outs[i][:H + H // 2, :W].cpu(), ref[i // 2 - L]), i
    trk.close()
    eng.close()


def test_eight_videos_in_one_call_and_in_flight(planted):
    """Eight videos one frame each per call against eight calls of one video; 2 streams + 1 calls in flight (2 and 8 streams) against
    the same calls synchronised one by one: bit-equal."""
    import torch
    frames = planted[0][:12]
    L = 4
    eng = _engine("fp16")
    a = eng.tracker(max_videos=8, lookback=dict(frames=L))
    dev, _ = _in_frames(frames, "nv12")
    outs8 = _out_frames(8 * 12, "nv12")
    views, ov = _views(dev, "nv12"), _views(outs8, "nv12")
    for t in range(12):
        a.detect_yuv_redact_lookback_device([views[t]] * 1 + [views[(t + v) % 12] for v in range(1, 8)], list(range(8)),
                                            ov[8 * t:8 * t + 8], THR, NMS, style="blur", shape="ellipse")
    eng.synchronize()
    for v in range(8):
        b = eng.tracker(lookback=dict(frames=L))
        seq = [dev[(t + v) % 12] for t in range(12)]
        single = _run(eng, b, seq, "nv12", "bt601", 1, ("blur", "ellipse"))[1]
        for t in range(L, 12):
            assert torch.equal(single[t], outs8[8 * t + v]), (v, t)
        b.close()
    a.close()
    eng.close()
    for streams in (2, 8):
        k = 2 * streams + 1
        eng = _engine("fp16", streams=streams)
        res = []
        for sync in (False, True):
            trk = eng.tracker(lookback=dict(frames=L))
            dev, _ = _in_frames(planted[0][:k], "nv12")
            outs = _out_frames(k, "nv12")
            views, ov = _views(dev, "nv12"), _views(outs, "nv12")
            for s in range(k):
                trk.detect_yuv_redact_lookback_device([views[s]], [0], [ov[s]], THR, NMS, style="blur", shape="ellipse")
                if sync:
                    eng.synchronize()
            eng.synchronize()
            res.append([o.cpu() for o in outs])
            trk.close()
        assert all(torch.equal(x, y) for x, y in zip(*res)), streams
        eng.close()


def test_drain_and_reset(planted):
    """A drain after fewer than L frames emits them all and restarts the ids at 1; a reset emits nothing and the next L frames emit
    nothing either."""
    import torch
    frames = planted[0][:10]
    L = 6
    eng = _engine("fp16")
    trk = eng.tracker(lookback=dict(frames=L))
    dev, _ = _in_frames(frames, "nv12")
    views = _views(dev, "nv12")
    outs = _out_frames(10, "nv12")
    ov = _views(outs, "nv12")
    nums = trk.detect_yuv_redact_lookback_device(views[:4], [0] * 4, ov[:4], THR, NMS)[0]
    assert list(nums) == [-1] * 4
    douts = _out_frames(L, "nv12")
    got = trk.drain(0, _views(douts, "nv12"))
    assert list(got) == [0, 1, 2, 3]
    eng.synchronize()
    r = trk.detect_yuv_redact_lookback_device(views[4:5], [0], ov[4:5], THR, NMS)
    tracks = trk.read(r[1], r[2], 1)[0]
    assert len(tracks) and sorted(int(x["id"]) for x in tracks)[0] == 1
    trk.reset(0)
    canary = outs[5].cpu()
    nums = trk.detect_yuv_redact_lookback_device(views[5:5 + 4], [0] * 4, ov[5:9], THR, NMS)[0]
    eng.synchronize()
    assert list(nums) == [-1] * 4 and torch.equal(outs[5].cpu(), canary)
    assert list(trk.drain(0, _views(_out_frames(L, "nv12"), "nv12"))) == [0, 1, 2, 3]
    trk.close()
    eng.close()


def test_refusals_launch_nothing(planted):
    """Each refusal returns its status with nothing launched: input and out canaries untouched, the tracker's frame numbers unchanged;
    rf_detect_batch, rf_detect_yuv_redact_device_style and launches per batch are the same before and after look-back calls."""
    import torch
    from retinaface_b200 import capi
    frames = planted[0][:3]
    eng = _engine("fp16", max_batch=4)
    lib = eng.lib
    inp = cv2.resize(frames[0], (448, 448))
    before = (eng.detect_batch([inp], THR, NMS), eng.launches_per_batch(4))
    trk = eng.tracker(max_videos=2, lookback=dict(frames=2))
    dev, _ = _in_frames(frames, "nv12")
    outs = _out_frames(3, "nv12")
    v, o = _views(dev, "nv12"), _views(outs, "nv12")
    ins0, outs0 = [d.clone() for d in dev], [x.clone() for x in outs]
    torch.cuda.synchronize()
    arr = eng._frames(v, "nv12", True)
    oarr = eng._frames(o, "nv12", True)
    st = capi.RedactStyle(0, 0, 0, 0, 0.0)
    nums = np.zeros(4, np.int32)

    def call(frames_arr, vids, n, out_arr, style=C.byref(st), t=trk.t):
        vv = (C.c_int * max(4, len(vids)))(*vids)
        return lib.rf_detect_yuv_redact_lookback_device(eng.h, t, frames_arr, vv, n, 0, THR, NMS, style, out_arr, nums.ctypes.data,
                                                        None, None, None, None, None)

    bad_style = capi.RedactStyle(9, 0, 0, 0, 0.0)
    assert call(arr, [0, 0, 0], 3, oarr) == -1                       # video 0 three times at L = 2
    assert call(arr, [0, 1], 2, oarr, style=C.byref(bad_style)) == -1
    assert call(arr, [0, 5], 2, oarr) == -1                          # video out of range
    assert call(arr, [0, 1], 2, None) == -1
    overl = eng._frames([v[0], v[0]], "nv12", True)
    assert call(arr, [0, 1], 2, overl) == -1                         # out frame 1 is input frame 0
    small = [(outs[0][:540, :960], outs[0][540:810, :960])]
    assert call(arr, [0], 1, eng._frames(small, "nv12", True)) == -1   # out frame of another size
    i420 = _out_frames(1, "i420")
    assert call(arr, [0], 1, eng._frames(i420, "i420", True)) == -1   # another layout
    nv21 = eng._frames([o[0]], "nv21", True)
    assert call(arr, [0], 1, nv21) == -1                             # another chroma order
    assert call(arr, [0, 1, 0, 1, 0], 5, oarr) == -6                 # n > max_batch
    plain = eng.tracker()
    assert call(arr, [0], 1, oarr, t=plain.t) == -1                  # not a look-back tracker
    for fn in (lambda: trk.detect_yuv_device(v[:1], [0], THR, NMS), lambda: trk.update([0], 0, 0),
               lambda: trk.detect_yuv_redact_device(v[:1], [0], THR, NMS), lambda: trk.detect_yuv_redact_device(v[:1], [0], THR, NMS, style="blur")):
        with pytest.raises(capi.RfError):
            fn()
    cfg = capi.LookbackConfig(0, 0.0)
    for bad in ((65, 0.0), (-1, 0.0), (0, 1.5), (0, float("nan"))):
        assert lib.rf_tracker_set_lookback(plain.t, C.byref(capi.LookbackConfig(*bad))) == -1, bad
    assert lib.rf_tracker_set_lookback(trk.t, C.byref(cfg)) == -1     # twice
    best = eng.tracker(best={})
    assert lib.rf_tracker_set_lookback(best.t, C.byref(cfg)) == -1
    n_out = C.c_int(7)
    assert lib.rf_tracker_drain(plain.t, 0, None, None, 0, C.byref(n_out), None) == -1
    eng.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(dev, ins0)) and all(torch.equal(a, b) for a, b in zip(outs, outs0))
    # the tracker saw no frame: the first two frames of a valid call emit nothing, and its drain has exactly those two
    assert call(arr, [0, 1], 2, oarr) == 0 and list(nums[:2]) == [-1, -1]
    assert call(arr, [0, 1], 2, oarr) == 0 and list(nums[:2]) == [-1, -1]
    assert lib.rf_tracker_drain(trk.t, 0, None, oarr, 1, C.byref(n_out), nums.ctypes.data) == -6   # cap below 2
    assert lib.rf_tracker_drain(trk.t, 0, None, oarr, 2, C.byref(n_out), nums.ctypes.data) == 0 and n_out.value == 2
    eng.synchronize()
    after = (eng.detect_batch([inp], THR, NMS), eng.launches_per_batch(4))
    assert after[1] == before[1] and all(np.array_equal(x, y) for x, y in zip(before[0], after[0]))
    d1 = [x.clone() for x in ins0[:2]]
    d2 = [x.clone() for x in ins0[:2]]
    torch.cuda.synchronize()
    eng.detect_yuv_redact_device(_views(d1, "nv12"), THR, NMS, style="blur", shape="ellipse")
    trk2 = eng.tracker(lookback=True)
    trk2.close()
    eng.detect_yuv_redact_device(_views(d2, "nv12"), THR, NMS, style="blur", shape="ellipse")
    eng.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(d1, d2))
    for x in (trk, plain, best):
        x.close()
    eng.close()


def test_detector_redact_frames_lookback(planted):
    """RetinaFace.redactFrames(lookback=L, out=...) and drainVideo are the look-back call and the drain."""
    import os
    import torch
    from conftest import GOLDEN
    from retinaface_b200.detector import RetinaFace
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    eng = det.engine
    dev, _ = _in_frames(planted[0][:6], "nv12")
    views = _views(dev, "nv12")
    a, b = _out_frames(6, "nv12"), _out_frames(6, "nv12")
    trk = eng.tracker(max_videos=64, lookback=dict(frames=3))
    nums = []
    for t in range(6):
        nums.append(int(det.redactFrames([views[t]], [0], threshold=THR, lookback=3, out=_views(a[t:t + 1], "nv12"))[0]))
        trk.detect_yuv_redact_lookback_device([views[t]], [0], _views(b[t:t + 1], "nv12"), THR, det.nms_threshold)
    assert nums == [-1, -1, -1, 0, 1, 2]
    da, db = _out_frames(3, "nv12"), _out_frames(3, "nv12")
    assert list(det.drainVideo(0, _views(da, "nv12"))) == [3, 4, 5] == list(trk.drain(0, _views(db, "nv12")))
    eng.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a + da, b + db))
    trk.close()
