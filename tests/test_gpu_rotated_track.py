"""GPU (-m gpu): f25 rotated views as the detector of every tracker call (rf_tracker_set_views).  A views tracker's detect calls must
return rf_detect_yuv_views_rotated_device's records bit for bit and do with them what the same call does with records at scale 1:
checked against a separate rotated call and a twin tracker fed those records (the twin is the tracker the oracles already hold bit for
bit), on oriented videos against materialised displayed frames, on a 45-degree tilted video whose faces the letter-box cannot see, with
one upright view against a plain tracker, with calls in flight over the rotated ring, on every refusal, and through the Python and C++
drivers."""
import ctypes as C
import math
import os
import subprocess

import cv2
import numpy as np
import pytest

from conftest import ROOT, caffemodel
from oracle.align import ARCFACE_112, umeyama
from oracle.bestshot import BestShotOracle
from oracle.orient import unorient_planes
from oracle.track import TrackerOracle
from oracle.yuv import bgr_to_frame
from test_gpu_bestshot import _same_shot
from test_gpu_follow import _check_oracle, _drive

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
INVALID_ARG, CAPACITY, UNSUPPORTED = -1, -6, -7     # RF_ERR_*
W, H = 1920, 1080
SWEEP = [(45.0 * k, 1.0) for k in range(8)]
MIXED = [(0.0, 1.0), (45.0, 0.75), (90.0, 0.5), (200.0, 1.0), (-30.0, 0.6)]


def _engine(prec="fp16", max_image=(1920, 1920), **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    from conftest import GOLDEN
    kw.setdefault("max_batch", 8)
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8, max_image=max_image,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, max_image=max_image, **kw)


def _tilted(golden, placement=False):
    """The golden photo turned 45 degrees counter-clockwise at its own scale, rows 180 .. 1259 (its six faces), centred on black; with
    `placement`, also the 2 x 3 matrix that maps upright photo pixels into the canvas."""
    h, w = golden.shape[:2]
    R = cv2.getRotationMatrix2D((w / 2, h / 2), 45.0, 1.0)
    c, s = abs(R[0, 0]), abs(R[0, 1])
    tw, th = int(h * s + w * c), int(h * c + w * s)
    R[0, 2] += tw / 2 - w / 2
    R[1, 2] += th / 2 - h / 2
    tilted = cv2.warpAffine(golden, R, (tw, th))[180:180 + H]
    canvas = np.zeros((H, W, 3), np.uint8)
    x0 = (W - tilted.shape[1]) // 2
    canvas[:, x0:x0 + tilted.shape[1]] = tilted
    if placement:
        R[0, 2] += x0
        R[1, 2] -= 180
        return canvas, R
    return canvas


def _video(golden, n, video=0, layout="nv12"):
    """n frames of a tilted video drifting 4 columns a frame (video v starts 16 v columns on)."""
    base = _tilted(golden)
    return [bgr_to_frame(np.roll(base, 16 * video + 4 * k, axis=1), layout) for k in range(n)]


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _clone(dev):
    import torch
    torch.cuda.synchronize()
    out = [d.clone() for d in dev]
    torch.cuda.synchronize()
    return out


def _host(dev):
    import torch
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dev]


def _same_lists(a, b, what):
    assert len(a) == len(b), what
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.tobytes() == y.tobytes(), (what, i, len(x), len(y))


def _same_state(t1, t2, nvideos, what):
    for v in range(nvideos):
        h1, r1 = t1.debug_state(v)
        h2, r2 = t2.debug_state(v)
        assert np.array_equal(h1, h2) and r1.tobytes() == r2.tobytes(), (what, v)


# ---- 1 / 2. records equal the rotated detector; every kind does what its twin does with them ------------------------------------------
KINDS = {
    "plain": {}, "redact": {}, "motion": {"motion": True}, "best": {"best": {}}, "follow": {"follow": True},
    "lookback": {"lookback": 2}, "lookback+search": {"lookback": 2, "lookback_search": True},
}
STYLES = [("mosaic", "rect"), ("blur", "ellipse")]


def _call(trk, kind, dev, vids, layout, matrix, style, outs=None, crops=None):
    if kind == "redact":
        tp, tc, d, c, sc = trk.detect_yuv_redact_device(dev, vids, THR, NMS, layout=layout, matrix=matrix, style=style[0], shape=style[1])
        return d, c, sc, tp, tc
    if kind == "best":
        _, _, tp, tc, d, c, sc = trk.detect_yuv_best_device(dev, vids, THR, NMS, crops.data_ptr(), layout=layout, matrix=matrix)
        return d, c, sc, tp, tc
    if kind.startswith("lookback"):
        _, tp, tc, d, c, sc = trk.detect_yuv_redact_lookback_device(dev, vids, outs, THR, NMS, layout=layout, matrix=matrix, style=style[0],
                                                                    shape=style[1])
        return d, c, sc, tp, tc
    tp, tc, d, c, sc = trk.detect_yuv_device(dev, vids, THR, NMS, layout=layout, matrix=matrix)
    return d, c, sc, tp, tc


CASES = [("fp32", "nv12", "bt601", 1, 1, "sweep"), ("fp16", "i420", "bt709", 3, 3, "mixed"), ("fp16", "nv12", "bt601", 3, 3, "sweep"),
         ("int8", "nv12", "bt601", 1, 1, "mixed"), ("int8", "i420", "bt709", 3, 3, "sweep")]


@pytest.mark.parametrize("prec,layout,matrix,per_call,nvideos,views", CASES)
def test_records_equal_the_rotated_detector(golden_image, prec, layout, matrix, per_call, nvideos, views):
    """Every kind's records and counts are a separate rf_detect_yuv_views_rotated_device's on the same frames, bit for bit, scales all
    1; a plain tracker's lists and FP64 state equal a twin plain tracker fed those records through rf_track_update, and a redacting
    tracker's bytes equal that twin's rf_redact_yuv_device_style of them."""
    import torch
    vset = SWEEP if views == "sweep" else MIXED
    nframes = 4
    order = [(k, v) for k in range(nframes) for v in range(nvideos)]
    per_video = [_video(golden_image, nframes, v, layout) for v in range(nvideos)]
    host = [per_video[v][k] for k, v in order]
    vids = [v for _, v in order]
    eng = _engine(prec)
    try:
        for kind, opts in KINDS.items():
            style = STYLES[len(kind) % 2]
            trk = eng.tracker(max_videos=nvideos, max_tracks=128, views=vset, **opts)
            twin = eng.tracker(max_videos=nvideos, max_tracks=128) if kind in ("plain", "redact") else None
            crops = torch.zeros((per_call, 128, 112, 112, 3), dtype=torch.uint8, device="cuda") if kind == "best" else None
            found = 0
            for s in range(0, len(host), per_call):
                m = min(per_call, len(host) - s)
                dev = [_cuda(f) for f in host[s:s + m]]
                pristine = _clone(dev)
                outs = _clone(dev) if kind.startswith("lookback") else None
                d, c, sc, tp, tc = _call(trk, kind, dev, vids[s:s + m], layout, matrix, style, outs=outs, crops=crops)
                assert np.array_equal(sc, np.ones(m, np.float32)), (kind, sc)
                got = eng.read_dets(d, c, m)
                lists = trk.read(tp, tc, m)
                d2, c2, _, _ = eng.detect_yuv_views_rotated_device(pristine, vset, THR, NMS, layout=layout, matrix=matrix)
                want = eng.read_dets(d2, c2, m)
                for i in range(m):
                    assert got[0][i].tobytes() == want[0][i].tobytes() and np.array_equal(got[1][i], want[1][i]), (kind, s + i)
                    found += len(want[0][i])
                if twin is not None:
                    tp2, tc2 = twin.update(vids[s:s + m], d2, c2, scales=None)
                    _same_lists(lists, twin.read(tp2, tc2, m), (kind, s))
                    if kind == "redact":
                        eng.redact_yuv_device(pristine, d2, c2, scales=None, layout=layout, tracker=twin, tracks_ptr=tp2, track_counts_ptr=tc2,
                                              style=style[0], shape=style[1])
                        for i, (a, b) in enumerate(zip(_host(dev), _host(pristine))):
                            assert np.array_equal(a, b), (kind, s + i)
            # the 45-degree sweep finds the tilted faces; the mixed set (one shrunk 45-degree view) some of them
            assert found >= (3 * len(host) if views == "sweep" else 1), (kind, found)
            if twin is not None:
                _same_state(trk, twin, nvideos, kind)
                twin.close()
            trk.close()
    finally:
        eng.close()


# ---- 3. display orientations -------------------------------------------------------------------------------------------------------
def _flat(x):
    if isinstance(x, (list, tuple)):
        return [y for e in x for y in _flat(e)]
    return [np.asarray(x).tobytes()]


def _oriented_run(eng, trk, kind, dev, style):
    """Every frame of one video through trk, two frames a call: records, lists, best shots and crops, the state, and the frames."""
    import torch
    out = []
    crops = torch.zeros((2, 128, 112, 112, 3), dtype=torch.uint8, device="cuda") if kind == "best" else None
    for s in range(0, len(dev), 2):
        views, vids = dev[s:s + 2], [0] * len(dev[s:s + 2])
        m = len(views)
        if kind == "best":
            bp, bc, tp, tc, d, c, sc = trk.detect_yuv_best_device(views, vids, THR, NMS, crops.data_ptr())
            eng.synchronize()
            out += [trk.read_best(bp, bc, m), crops[:m].cpu().numpy()]
        elif kind == "redact":
            tp, tc, d, c, sc = trk.detect_yuv_redact_device(views, vids, THR, NMS, style=style[0], shape=style[1])
        else:
            tp, tc, d, c, sc = trk.detect_yuv_device(views, vids, THR, NMS)
        out += [eng.read_dets(d, c, m), trk.read(tp, tc, m)]
    out.append(trk.debug_state(0))
    return out


@pytest.mark.parametrize("o", [3, 5, 6, 8])
def test_oriented_videos_equal_materialised_frames(golden_image, o):
    """A views tracker on stored frames S shown at orientation o equals the same tracker on orient_planes(S, o) at orientation 1:
    records, lists, best shots and crops, state, and the written bytes mapped back -- pitch padding never written."""
    import torch
    eng = _engine("fp16")
    try:
        disp = _video(golden_image, 4, 0, "nv12")
        stored = [unorient_planes(f, "nv12", o) for f in disp]
        for kind in ("plain", "redact", "best"):
            style = STYLES[1]
            opts = {"best": {}} if kind == "best" else {}
            t1 = eng.tracker(max_tracks=128, views=SWEEP, **opts)
            t1.set_orientation(0, o)
            # the stored NV12 surfaces with rows 64 bytes wider than the frame and chroma in its own allocation: the padding holds
            # a canary
            sw, sh = stored[0].shape[1], stored[0].shape[0] * 2 // 3
            surfs = []
            for f in stored:
                y, uv = np.full((sh, sw + 64), 0xA5, np.uint8), np.full((sh // 2, sw + 64), 0xA5, np.uint8)
                y[:, :sw], uv[:, :sw] = f[:sh], f[sh:]
                surfs.append((_cuda(y), _cuda(uv)))
            got = _oriented_run(eng, t1, kind, [(y[:, :sw], uv[:, :sw]) for y, uv in surfs], style)
            t1.close()
            t2 = eng.tracker(max_tracks=128, views=SWEEP, **opts)
            mat = [_cuda(f) for f in disp]
            want = _oriented_run(eng, t2, kind, mat, style)
            t2.close()
            a, b = _flat(got), _flat(want)
            assert len(a) == len(b), (o, kind)
            for i, (x, y) in enumerate(zip(a, b)):
                assert x == y, (o, kind, i)
            for (y, uv), m in zip(surfs, _host(mat)):
                yh, uvh = y.cpu().numpy(), uv.cpu().numpy()
                assert (yh[:, sw:] == 0xA5).all() and (uvh[:, sw:] == 0xA5).all(), (o, kind)
                assert np.array_equal(np.concatenate([yh[:, :sw], uvh[:, :sw]]), unorient_planes(m, "nv12", o)), (o, kind)
    finally:
        eng.close()


# ---- 4. the gap is closed ---------------------------------------------------------------------------------------------------------
def _confirmed_runs(lists_per_frame):
    """For each id confirmed at some frame: the number of frames it is listed as confirmed."""
    from retinaface_b200 import capi
    runs = {}
    for lst in lists_per_frame:
        for r in lst:
            if r["state"] == capi.TRACK_CONFIRMED:
                runs[int(r["id"])] = runs.get(int(r["id"]), 0) + 1
    return runs


def test_tilted_video_is_tracked_and_redacted(golden_image):
    """On the 45-degree tilted drifting video a plain tracker confirms at most one track; a views tracker confirms at least four, each
    one id over >= 20 frames; a redacting views tracker covers every landmark of those faces on every frame at the default margin.  A
    landmark counts as covered when its 3 x 3 block was written: a single redacted sample may equal the original (a blur of a flat
    patch, a mosaic cell whose mean it is)."""
    nframes = 24
    frames = _video(golden_image, nframes)
    eng = _engine("fp16")
    try:
        res = {}
        for name, kw in (("plain", {}), ("views", {"views": SWEEP})):
            trk = eng.tracker(max_tracks=128, **kw)
            lists, dets = [], []
            for k in range(nframes):
                tp, tc, d, c, _ = trk.detect_yuv_device([_cuda(frames[k])], [0], THR, NMS)
                lists += trk.read(tp, tc, 1)
                dets.append(eng.read_dets(d, c, 1)[0][0])
            res[name] = (lists, dets)
            trk.close()
        assert sum(n >= 1 for n in _confirmed_runs(res["plain"][0]).values()) <= 1
        runs = _confirmed_runs(res["views"][0])
        long = [i for i, n in runs.items() if n >= 20]
        assert len(long) >= 4, runs
        # every landmark of the views tracker's faces, frame by frame, lies in a written sample
        trk = eng.tracker(max_tracks=128, views=SWEEP)
        dev = [_cuda(f) for f in frames]
        for k in range(nframes):
            trk.detect_yuv_redact_device(dev[k:k + 1], [0], THR, NMS, style="blur", shape="ellipse")
        got = _host(dev)
        trk.close()
        faces = res["views"][1]
        for k in range(nframes):
            for f in faces[k]:
                for j in range(5):
                    x, y = int(f[5 + j]), int(f[10 + j])
                    assert _written(got[k], frames[k], x, y), (k, j)
    finally:
        eng.close()


def _written(out, orig, x, y):
    return out[y - 1:y + 2, x - 1:x + 2].tobytes() != orig[y - 1:y + 2, x - 1:x + 2].tobytes()


@pytest.mark.parametrize("L", [1, 4])
def test_lookback_covers_the_frames_before_the_first_detection(golden_image, L):
    """Seeded noise on the first frames (no face is detected there, and no 3 x 3 block is flat), then the tilted scene from frame `start`
    on: the faces are first detected at `start`, and a look-back views tracker covers every landmark of those records on each of the L
    frames before it, as well as on `start` itself."""
    start, nframes = 6, 6 + 2 * 4
    base = _tilted(golden_image)
    noise = np.random.default_rng(25).integers(0, 256, base.shape, dtype=np.uint8)
    bgr = [noise if k < start else base for k in range(nframes)]
    frames = [bgr_to_frame(b, "nv12") for b in bgr]
    eng = _engine("fp16")
    try:
        trk = eng.tracker(max_tracks=128, views=SWEEP, lookback=L)
        dev = [_cuda(f) for f in frames]
        outs = [_cuda(np.zeros_like(f)) for f in frames]
        recs = []
        for k in range(nframes):
            _, _, _, d, c, _ = trk.detect_yuv_redact_lookback_device(dev[k:k + 1], [0], outs[k:k + 1], THR, NMS)
            recs.append(eng.read_dets(d, c, 1)[0][0])
        emitted = _host(outs)          # frame e was emitted into the out frame of frame e + L
        trk.close()
        assert all(len(recs[k]) == 0 for k in range(start)), [len(r) for r in recs]
        assert len(recs[start]) >= 4, len(recs[start])
        for e in range(start - L, start + 1):
            for f in recs[start]:
                for j in range(5):
                    x, y = int(f[5 + j]), int(f[10 + j])
                    assert _written(emitted[e + L], frames[e], x, y), (L, e, j)
    finally:
        eng.close()


# ---- 5. one upright view ---------------------------------------------------------------------------------------------------------
ONE_VIEW_KINDS = {
    "plain": {}, "crops": {}, "redact": {}, "motion": {"motion": True}, "best": {"best": {}}, "best+live": {"best": {}, "best_live": True},
    "best+follow": {"best": {}, "best_follow": True}, "follow": {"follow": True}, "follow+motion": {"follow": True, "motion": True},
    "lookback": {"lookback": 2}, "lookback15+motion": {"lookback": 15, "motion": True},
    "lookback+search": {"lookback": 2, "lookback_search": True}, "lookback+follow": {"lookback": 3, "lookback_follow": True},
}


def _kind_run(eng, trk, kind, dev, style):
    """Every frame of one 1080p video through trk, two frames a call; following kinds detect every third call and follow the others.
    Returns everything the calls output -- lists, motions, follow records, shots and their crops, new-identity crops, look-back
    numbers, search steps, the drained and the written frames, finish shots and the FP64 state -- on the host."""
    import torch
    out = []
    best = kind.startswith("best")
    crops = torch.zeros((2, 128, 112, 112, 3), dtype=torch.uint8, device="cuda") if best or kind == "crops" else None
    for s in range(0, len(dev), 2):
        views, vids = dev[s:s + 2], [0] * len(dev[s:s + 2])
        m = len(views)
        follow = "follow" in kind and (s // 2) % 3 != 0
        if crops is not None:
            crops.zero_()
        extra = []
        if follow and kind.startswith("lookback"):
            nums, tp, tc = trk.follow_redact_lookback_device(views, vids, views, style=style[0], shape=style[1])
            extra = [nums]
        elif follow and best:
            bp, bc, tp, tc = trk.follow_best_device(views, vids, crops.data_ptr())
            eng.synchronize()
            extra = [trk.read_best(bp, bc, m), crops[:m].cpu().numpy()]
        elif follow:
            tp, tc = trk.follow_device(views, vids)
        elif kind == "crops":
            tp, tc, _, _, _ = trk.detect_yuv_device(views, vids, THR, NMS, align={"max_faces": 128}, dev_crops_ptr=crops.data_ptr())
            eng.synchronize()
            extra = [crops[:m].cpu().numpy()]
        elif best:
            bp, bc, tp, tc, _, _, _ = trk.detect_yuv_best_device(views, vids, THR, NMS, crops.data_ptr())
            eng.synchronize()
            extra = [trk.read_best(bp, bc, m), crops[:m].cpu().numpy()]
        elif kind.startswith("lookback"):
            nums, tp, tc, _, _, _ = trk.detect_yuv_redact_lookback_device(views, vids, views, THR, NMS, style=style[0], shape=style[1])
            extra = [nums]
            if trk.lookback_search_on:
                steps, lengths = trk.lookback_search(m)
                extra += [lengths] + [steps[i, r, :lengths[i, r]] for i in range(m) for r in range(steps.shape[1])]
        elif kind == "redact":
            tp, tc, _, _, _ = trk.detect_yuv_redact_device(views, vids, THR, NMS, style=style[0], shape=style[1])
        else:
            tp, tc, _, _, _ = trk.detect_yuv_device(views, vids, THR, NMS)
        lists = trk.read(tp, tc, m)
        out += [lists] + extra
        if follow:
            fo = trk.follow(m)
            out += [fo[i, :len(lists[i])] for i in range(m)]
        if trk.motion_on:
            out.append(trk.motion(m))
    if kind.startswith("lookback"):
        outs = _clone(dev[:trk.lookback])
        out.append(trk.drain(0, outs, style=style[0], shape=style[1]))
        out += _host(outs)
    if best:
        fc = torch.zeros((128, 112, 112, 3), dtype=torch.uint8, device="cuda")
        bp, bc = trk.finish(0, fc.data_ptr())
        out += [trk.read_best(bp, bc, 1), fc.cpu().numpy()]
    out += _host(dev)
    out.append(trk.debug_state(0))
    return out


@pytest.mark.parametrize("prec", ["fp16", "int8"])
def test_one_upright_view_equals_a_plain_tracker(golden_image, prec):
    """views = [(0, 1)] on untilted 1920 x 1080 frames: every kind's lists, state, motions, follow records, best shots (live and
    following included) and their crops, new-identity crops, look-back numbers, search steps, drained, redacted and written bytes
    equal a tracker without views, bit for bit.  The one view is the letter-box, and its merge maps each record to frame pixels with
    the same float product the tracker's update applies to the letter-box records, so no rounding step differs."""
    big = cv2.resize(golden_image, (1600, 1108))
    bgr = []
    for k in range(12):
        c = np.full((H, W, 3), 40, np.uint8)
        x, y = 40 + 9 * k, 6 * (k % 3)
        c[y:y + 1060, x:x + 1600] = big[:1060]
        bgr.append(c)
    frames = [bgr_to_frame(b, "nv12") for b in bgr]
    eng = _engine(prec, max_image=(1080, 1920))
    try:
        for kind, opts in ONE_VIEW_KINDS.items():
            style = STYLES[len(kind) % 2]
            got = []
            for views in ([(0.0, 1.0)], None):
                trk = eng.tracker(max_tracks=128, views=views, **opts)
                got.append(_flat(_kind_run(eng, trk, kind, [_cuda(f) for f in frames], style)))
                trk.close()
            assert len(got[0]) == len(got[1]), kind
            for i, (a, b) in enumerate(zip(*got)):
                assert a == b, (prec, kind, i)
    finally:
        eng.close()


# ---- 2. the oracles on the tilted video's records --------------------------------------------------------------------------------
def _angle(M):
    return math.degrees(math.atan2(M[1, 0], M[0, 0]))


def test_best_shots_equal_the_oracle_and_come_out_upright(golden_image):
    """A views best-shot tracker on the tilted video: every shot, crop and matrix equals oracle/bestshot.py fed oracle/track.py on the
    rotated call's records and the crops / matrices that call cuts for them, bit for bit; each shot's crop is upright -- its fitted
    angle is the upright photo's crop of the same face turned by the 45-degree tilt, within f23's 20 degrees."""
    import torch
    nframes, max_lost = 12, 3
    frames = _video(golden_image, nframes)
    _, R = _tilted(golden_image, placement=True)
    dev = [_cuda(f) for f in frames]
    eng = _engine("fp16")
    try:
        mf = eng.max_faces
        to, bo = TrackerOracle(1, max_lost=max_lost), BestShotOracle()
        want = []
        for t in range(nframes):
            crops = torch.zeros((1, mf, 112, 112, 3), dtype=torch.uint8, device="cuda")
            mats = torch.zeros((1, mf, 6), dtype=torch.float64, device="cuda")
            d, c, _, _ = eng.detect_yuv_views_rotated_device([dev[t]], SWEEP, THR, NMS, align=dict(), dev_crops_ptr=crops.data_ptr(),
                                                             dev_mats_ptr=mats.data_ptr())
            tracks = to.update(0, eng.read_dets(d, c, 1)[0][0], 1.0)
            want.append(bo.update(0, tracks, crops[0].cpu().numpy(), mats[0].cpu().numpy(), W, H))
        want_fin = bo.finish(0)
        trk = eng.tracker(max_lost=max_lost, best=dict(), views=SWEEP)
        T = trk.max_tracks
        crops = torch.zeros((nframes, T, 112, 112, 3), dtype=torch.uint8, device="cuda")
        mats = torch.zeros((nframes, T, 6), dtype=torch.float64, device="cuda")
        shots = []
        for t in range(nframes):
            bp, bc, _, _, _, _, sc = trk.detect_yuv_best_device([dev[t]], [0], THR, NMS, crops[t].data_ptr(), mats[t].data_ptr())
            assert sc[0] == 1.0
            shots.append(trk.read_best(bp, bc, 1)[0])
        fc = torch.zeros((T, 112, 112, 3), dtype=torch.uint8, device="cuda")
        fm = torch.zeros((T, 6), dtype=torch.float64, device="cuda")
        bp, bc = trk.finish(0, fc.data_ptr(), fm.data_ptr())
        fin = trk.read_best(bp, bc, 1)[0]
        trk.close()
        ch, mh = crops.cpu().numpy(), mats.cpu().numpy()
        got = [(s, ch[t, k], mh[t, k]) for t in range(nframes) for k, s in enumerate(shots[t])]
        got += [(s, fc[k].cpu().numpy(), fm[k].cpu().numpy()) for k, s in enumerate(fin)]
        wanted = [w for t in range(nframes) for w in want[t]] + list(want_fin)
        assert len(got) == len(wanted) >= 4, (len(got), len(wanted))
        for (s, cr, m), w in zip(got, wanted):
            _same_shot(s, w, "tilted")
            assert np.array_equal(cr, w["crop"]) and m.tobytes() == w["M"].reshape(6).tobytes()
        # upright: the upright photo's faces mapped into the canvas of the shot's frame, matched by centre
        ref = eng.detect_views_rotated(golden_image, [(0.0, 1.0)], THR, NMS)[0]
        for s, _, m in got:
            shift = 4 * int(s["frame"])
            ctr = np.stack([R @ np.array([(r[1] + r[3]) / 2, (r[2] + r[4]) / 2, 1.0]) + [shift, 0] for r in ref])
            f = s["face"]
            d = np.hypot(*(ctr - [(f[1] + f[3]) / 2, (f[2] + f[4]) / 2]).T)
            i = int(np.argmin(d))
            assert d[i] < 0.25 * (ref[i, 3] - ref[i, 1]), (int(s["id"]), d[i])
            Mu = umeyama(np.stack([ref[i, 5:10], ref[i, 10:15]], 1).astype(np.float64), ARCFACE_112)[:2]
            dd = (_angle(m.reshape(2, 3)) - 45.0 - _angle(Mu) + 180.0) % 360.0 - 180.0
            assert abs(dd) < 20.0, (int(s["id"]), dd)
    finally:
        eng.close()


@pytest.mark.parametrize("k", [2, 3])
def test_follow_equals_the_oracle(golden_image, k):
    """A views follow tracker on the tilted video, detecting every k-th frame: its lists on every frame and its follow records equal
    oracle/follow.py fed the detect frames' records (scale 1) and the frames' luma, bit for bit."""
    host = _video(golden_image, 12)
    eng = _engine("fp16")
    try:
        trk = eng.tracker(follow=True, views=SWEEP)
        got = _drive(eng, trk, [_cuda(f) for f in host], host, k, 4, "nv12")
        trk.close()
        assert all(sc == 1.0 for kind, _, _, sc in got if kind == "detect")
        assert sum(len(tr) for kind, tr, _, _ in got if kind == "follow") >= 4
        _check_oracle(got, host, f"views k={k}")
    finally:
        eng.close()


# ---- 6. rings and refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("streams", [2, 4])
def test_calls_in_flight_equal_blocking(golden_image, streams):
    """2 streams + 1 redacting views-tracker calls in flight, each after a standalone rotated and a tiled device call: every redacted
    frame and every video's state equal the same calls made one at a time, and the records of the standalone calls issued
    ceil(streams / 2) iterations before the end -- followed by as many views-tracker calls and streams - 1 or fewer further rotated
    calls in all, within the ring's validity rule -- read after the run, equal the blocking run's."""
    ncalls = 2 * streams + 1
    keep = ncalls - (streams + 1) // 2
    host = [_video(golden_image, 1, v)[0] for v in range(ncalls)]
    results = []
    for blocking in (True, False):
        eng = _engine("fp16", streams=streams)
        try:
            trk = eng.tracker(max_videos=ncalls, max_tracks=128, views=SWEEP)
            dev = [_cuda(f) for f in host]
            side = [_cuda(f) for f in host]
            for i in range(ncalls):
                rd, rc, _, _ = eng.detect_yuv_views_rotated_device([side[(i + 1) % ncalls]], SWEEP, THR, NMS)
                td, tc = eng.detect_yuv_tiled_device([side[i]], THR, NMS)
                if i == keep:
                    kept = (rd, rc, td, tc)
                trk.detect_yuv_redact_device([dev[i]], [i], THR, NMS)
                if blocking:
                    eng.synchronize()
            recs = (eng.read_dets(kept[0], kept[1], 1), eng.read_dets(kept[2], kept[3], 1))
            results.append((_host(dev), [trk.debug_state(v) for v in range(ncalls)], recs))
            trk.close()
        finally:
            eng.close()
    (a, sa, ra), (b, sb, rb) = results
    for i in range(ncalls):
        assert np.array_equal(a[i], b[i]), (streams, i)
        assert np.array_equal(sa[i][0], sb[i][0]) and sa[i][1].tobytes() == sb[i][1].tobytes(), (streams, i)
    assert len(ra[0][0][0]) >= 1 and _flat(ra) == _flat(rb)
    assert any(not np.array_equal(a[i], host[i]) for i in range(ncalls))


def _status(eng, fn, *args):
    rc = fn(*args)
    return rc, (eng.lib.rf_last_error(eng.h) or b"").decode()


def test_setter_refusals(golden_image):
    """Every refusal of rf_tracker_set_views with its status and message; after each the tracker is still a plain one (its next
    setter is taken) and its first frame call is the plain tracker's."""
    from retinaface_b200 import capi
    eng = _engine("fp16")
    lib = eng.lib
    try:
        def setter(trk, views, n=None):
            arr = (capi._RotatedView * max(len(views), 1))(*[capi._RotatedView(a, s) for a, s in views])
            return _status(eng, lib.rf_tracker_set_views, trk.t, arr if views is not None else None, len(views) if n is None else n)

        trk = eng.tracker()
        rc, err = _status(eng, lib.rf_tracker_set_views, trk.t, None, 4)
        assert rc == INVALID_ARG and err == "rf_tracker_set_views: views is NULL", err
        for n in (0, 17, -1):
            rc, err = setter(trk, SWEEP, n)
            assert rc == CAPACITY and err == f"rf_tracker_set_views: {n} views, limit RF_MAX_VIEWS = 16", err
        for views, msg in (([(0.0, 1.0), (float("nan"), 1.0)], "view 1: the angle must be finite"),
                           ([(float("inf"), 1.0)], "view 0: the angle must be finite"),
                           ([(10.0, 0.0)], "view 0: shrink must be in (0, 1]"), ([(10.0, 1.5)], "view 0: shrink must be in (0, 1]")):
            rc, err = setter(trk, views)
            assert rc == INVALID_ARG and err == "rf_tracker_set_views: " + msg, (views, err)
        assert setter(trk, SWEEP)[0] == 0
        rc, err = setter(trk, SWEEP)
        assert rc == INVALID_ARG and err == "rf_tracker_set_views: rotated views are already on", err
        rc, err = _status(eng, lib.rf_tracker_set_tiling, trk.t, None)
        assert rc == UNSUPPORTED and err.startswith("rf_tracker_set_tiling: this tracker detects through rotated views"), err
        trk.close()
        trk = eng.tracker(tiling=True)
        rc, err = setter(trk, SWEEP)
        assert rc == UNSUPPORTED and err.startswith("rf_tracker_set_views: a tiling tracker"), err
        trk.close()
        # after a frame call: refused, and nothing was launched or written by the refusal
        trk = eng.tracker()
        dev = [_cuda(_video(golden_image, 1)[0])]
        trk.detect_yuv_device(dev, [0], THR, NMS)
        eng.synchronize()
        before = trk.debug_state(0)
        rc, err = setter(trk, SWEEP)
        assert rc == INVALID_ARG and err == "rf_tracker_set_views: the tracker has already been updated", err
        after = trk.debug_state(0)
        assert np.array_equal(before[0], after[0]) and before[1].tobytes() == after[1].tobytes()
        trk.close()
        # orientations: a views tracker takes them, a tiling tracker still refuses them
        trk = eng.tracker(views=SWEEP)
        trk.set_orientation(-1, 6)
        trk.close()
    finally:
        eng.close()


@pytest.mark.parametrize("kind", ["plain", "best", "best+live", "best+follow", "follow", "lookback", "lookback+search",
                                  "lookback+follow", "motion"])
def test_setter_admission_rows(golden_image, kind):
    """Every kind takes the setter before its first frame call, in either order with the other setters."""
    eng = _engine("fp16")
    opts = {"plain": {}, "best": {"best": {}}, "best+live": {"best": {}, "best_live": True}, "best+follow": {"best": {}, "best_follow": True},
            "follow": {"follow": True}, "lookback": {"lookback": 2}, "lookback+search": {"lookback": 2, "lookback_search": True},
            "lookback+follow": {"lookback": 2, "lookback_follow": True}, "motion": {"motion": True}}[kind]
    try:
        trk = eng.tracker(views=SWEEP, **opts)
        if kind == "plain":
            trk.set_motion()           # a setter after the views
        trk.close()
    finally:
        eng.close()


# ---- 7. the drivers --------------------------------------------------------------------------------------------------------------
def test_detector_surfaces_equal_hand_calls(golden_image):
    """RetinaFace.trackFrames / redactFrames with any_angle (and lookback, detect_every) equal the same tracker calls made by hand."""
    from retinaface_b200.detector import RetinaFace
    host = _video(golden_image, 6)
    eng = _engine("fp16")
    try:
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        dev = [_cuda(f) for f in host]
        lists = [rf.trackFrames(dev[s:s + 3], [0, 0, 0], THR, max_videos=1, any_angle=45)[0] for s in (0, 3)]
        trk = eng.tracker(max_videos=1, views=SWEEP)
        for s, got in zip((0, 3), lists):
            tp, tc, _, _, _ = trk.detect_yuv_device(dev[s:s + 3], [0, 0, 0], THR, NMS)
            assert got == RetinaFace._lists(trk.read(tp, tc, 3))
        trk.close()
        rf._tracker.close()
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        a = [_cuda(f) for f in host]
        b = [_cuda(f) for f in host]
        nums = [rf.redactFrames(a[s:s + 3], [0, 0, 0], THR, lookback=2, detect_every=3, max_videos=1, any_angle=45) for s in (0, 3)]
        trk = eng.tracker(max_videos=1, lookback=2, lookback_follow=True, views=SWEEP)
        for s, want in zip((0, 3), nums):
            got = trk.detect_yuv_redact_lookback_device(b[s:s + 1], [0], b[s:s + 1], THR, NMS)[0]
            got = np.concatenate([got, trk.follow_redact_lookback_device(b[s + 1:s + 3], [0, 0], b[s + 1:s + 3])[0]])
            assert np.array_equal(got, want)
        for x, y in zip(_host(a), _host(b)):
            assert np.array_equal(x, y)
        trk.close()
        rf._tracker.close()
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        rf.trackFrames(a[:1], [0], THR, max_videos=1)
        with pytest.raises(ValueError):
            rf.trackFrames(a[1:2], [0], THR, any_angle=45)
        rf._tracker.close()
    finally:
        eng.close()


CPP_PROGRAM = r'''
#include "RetinaFace.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <fstream>
// argv: model directory, frames file (n NV12 1920x1080 frames), out file, n.  redactYUV with track_any_angle_step 45, three frames a
// call, then the bytes.
int main(int argc, char **argv) {
    string model = argv[1];
    const int n = atoi(argv[4]), w = 1920, h = 1080;
    const size_t bytes = (size_t)w * h * 3 / 2;
    std::vector<unsigned char> buf(bytes * n);
    std::ifstream(argv[2], std::ios::binary).read((char *)buf.data(), buf.size());
    RetinaFaceOptions opt;
    opt.net_w = opt.net_h = 448;
    opt.model_file = "mnet25.caffemodel";
    opt.track_any_angle_step = 45.f;
    RetinaFace rf(model, "net3", 0.4f, opt);
    unsigned char *d = nullptr;
    if (cudaMalloc(&d, buf.size()) != cudaSuccess) return 2;
    cudaMemcpy(d, buf.data(), buf.size(), cudaMemcpyHostToDevice);
    RedactOptions ro;
    for (int s = 0; s < n; s += 3) {
        std::vector<rf_yuv_frame> frames;
        std::vector<int> videos;
        for (int i = s; i < s + 3 && i < n; i++) {
            unsigned char *y = d + bytes * i, *uv = y + (size_t)w * h;
            frames.push_back(rf_yuv_frame{y, uv, uv + 1, w, w, 2, w, h});
            videos.push_back(0);
        }
        rf.redactYUV(frames, &videos, 0.5f, ro);
    }
    cudaDeviceSynchronize();
    cudaMemcpy(buf.data(), d, buf.size(), cudaMemcpyDeviceToHost);
    std::ofstream(argv[3], std::ios::binary).write((const char *)buf.data(), buf.size());
    return 0;
}
'''


def test_host_shell_redact_any_angle_equals_c_calls(golden_image, tmp_path):
    """The C++ RetinaFace::redactYUV with RetinaFaceOptions::track_any_angle_step gives the bytes of the same C calls."""
    from retinaface_b200.build import HERE, build_host
    from retinaface_b200 import Engine, RF_PREC_FP16
    build_host()
    host = _video(golden_image, 6)
    (tmp_path / "in.bin").write_bytes(b"".join(f.tobytes() for f in host))
    src = tmp_path / "user.cpp"
    src.write_text(CPP_PROGRAM)
    exe = tmp_path / "user"
    cuda = "/usr/local/cuda"
    hostdir = os.path.join(HERE, "host")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", hostdir, "-I", os.path.join(ROOT, "include"), "-I", cuda + "/include", str(src),
                           os.path.join(hostdir, "RetinaFace.cpp"), "-o", str(exe), "-L", HERE, "-lrf_b200", "-L", cuda + "/lib64", "-lcudart",
                           "-Wl,-rpath," + HERE + ":" + cuda + "/lib64"])
    subprocess.check_call([str(exe), os.path.dirname(caffemodel("mnet25")), str(tmp_path / "in.bin"), str(tmp_path / "out.bin"), str(len(host))])
    got = np.frombuffer((tmp_path / "out.bin").read_bytes(), np.uint8).reshape(len(host), *host[0].shape)
    eng = Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP16, max_batch=8, max_faces=256, max_image=(3072, 4096), network="net3")
    try:
        trk = eng.tracker(max_videos=16, views=SWEEP)
        dev = [_cuda(f) for f in host]
        for s in (0, 3):
            trk.detect_yuv_redact_device(dev[s:s + 3], [0, 0, 0], 0.5, 0.4)
        want = _host(dev)
        trk.close()
    finally:
        eng.close()
    assert any(not np.array_equal(g, f) for g, f in zip(got, host))
    for i in range(len(host)):
        assert np.array_equal(got[i], want[i]), i
