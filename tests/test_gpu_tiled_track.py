"""GPU (-m gpu): f19 tiled detection as the detector of every tracker call (rf_tracker_set_tiling).  A tiling tracker's detect calls
must return rf_detect_yuv_tiled_device's records bit for bit, and do with them what the same call does with records at scale 1: checked
against a separate tiled call and a twin tracker fed those records, against a twin tracker without tiling where the fitted level alone
equals the letter-box, on 4K frames whose faces the letter-box cannot see, with calls in flight over the tiled ring, on every refusal,
and through the Python and C++ drivers."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, ROOT, caffemodel
from oracle.yuv import bgr_to_frame

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
INVALID_ARG, CAPACITY, UNSUPPORTED = -1, -6, -7     # RF_ERR_*
STYLES = [("mosaic", "rect"), ("blur", "ellipse")]


def _engine(prec="fp16", max_image=(1440, 2560), **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    if prec == "int8":
        eng = Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8, max_image=max_image,
                     int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    else:
        eng = Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, max_image=max_image, **kw)
    # every tracker made on the engine (RetinaFace's included) is closed before the engine, however the test ends
    made, tracker, close = [], eng.tracker, eng.close

    def track(*a, **kw):
        made.append(tracker(*a, **kw))
        return made[-1]

    def close_all():
        for t in made:
            t.close()
        close()
    eng.tracker, eng.close = track, close_all
    return eng


def _half(golden):
    """The golden photo at half size (640 x 443, faces about 50 x 70 px): far below the smallest anchor of a 4K letter-box."""
    return cv2.resize(golden, (640, 443), interpolation=cv2.INTER_AREA)


def _scene(golden, w, h, n, spots, video=0, step=(3, 2)):
    """n BGR frames of a w x h video: the half photo (mirrored on odd videos) at each spot, moving `step` pixels per frame."""
    half = _half(golden)
    if video % 2:
        half = half[:, ::-1].copy()
    frames = []
    for k in range(n):
        c = np.full((h, w, 3), 16 + 8 * video, np.uint8)
        for x, y in spots:
            x, y = x + step[0] * k, y + step[1] * k
            c[y:y + 443, x:x + 640] = half
        frames.append(c)
    return frames


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _device(bgrs, layout):
    return [_cuda(bgr_to_frame(b, layout)) for b in bgrs]


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


# ---- 1. exact against the tiled detector ------------------------------------------------------------------------------------------
KINDS = {
    "plain": {}, "redact": {}, "motion": {"motion": True}, "best": {"best": {}}, "follow": {"follow": True},
    "lookback": {"lookback": 2}, "lookback+search": {"lookback": 2, "lookback_search": True},
}


def _call(eng, trk, kind, views, vids, layout, matrix, style, outs=None, crops=None):
    """One detect call of `kind` on the views; returns (dets_ptr, counts_ptr, scales, tracks_ptr, track_counts_ptr, extra)."""
    if kind == "redact":
        tp, tc, d, c, sc = trk.detect_yuv_redact_device(views, vids, THR, NMS, layout=layout, matrix=matrix, style=style[0], shape=style[1])
        return d, c, sc, tp, tc, None
    if kind == "best":
        bp, bc, tp, tc, d, c, sc = trk.detect_yuv_best_device(views, vids, THR, NMS, crops.data_ptr(), layout=layout, matrix=matrix)
        return d, c, sc, tp, tc, (bp, bc)
    if kind.startswith("lookback"):
        nums, tp, tc, d, c, sc = trk.detect_yuv_redact_lookback_device(views, vids, outs, THR, NMS, layout=layout, matrix=matrix,
                                                                       style=style[0], shape=style[1])
        return d, c, sc, tp, tc, nums
    tp, tc, d, c, sc = trk.detect_yuv_device(views, vids, THR, NMS, layout=layout, matrix=matrix)
    return d, c, sc, tp, tc, None


CASES = [("fp32", "nv12", "bt601", 1, 1), ("fp16", "i420", "bt709", 4, 2), ("fp16", "nv12", "bt601", 8, 1), ("int8", "nv12", "bt709", 4, 1),
         ("int8", "i420", "bt601", 8, 2)]


@pytest.mark.parametrize("prec,layout,matrix,per_call,nvideos", CASES)
def test_records_equal_the_tiled_detector(golden_image, prec, layout, matrix, per_call, nvideos):
    """2560 x 1440 videos with small moving faces: every kind's records and counts are a separate rf_detect_yuv_tiled_device's on the
    same frames, bit for bit, scales all 1; a plain tracker's lists and FP64 state equal a twin plain tracker fed those records through
    rf_track_update, and a redacting tracker's bytes equal that twin's rf_redact_yuv_device_style of them."""
    nframes = 8 if nvideos == 1 else 4
    spots = [(32, 16), (1376, 16), (704, 976)]
    bgr = [_scene(golden_image, 2560, 1440, nframes, spots, video=v) for v in range(nvideos)]
    order = [(k, v) for k in range(nframes) for v in range(nvideos)]
    host = [bgr_to_frame(bgr[v][k], layout) for k, v in order]
    vids = [v for _, v in order]
    eng = _engine(prec)
    import torch
    try:
        for kind, opts in KINDS.items():
            style = STYLES[len(kind) % 2]
            trk = eng.tracker(max_videos=nvideos, max_tracks=128, tiling=True, **opts)
            twin = eng.tracker(max_videos=nvideos, max_tracks=128) if kind in ("plain", "redact") else None
            per = min(per_call, 2 * nvideos) if kind.startswith("lookback") else per_call
            crops = torch.zeros((per, 128, 112, 112, 3), dtype=torch.uint8, device="cuda") if kind == "best" else None
            found = 0
            for s in range(0, len(host), per):
                m = min(per, len(host) - s)
                dev = [_cuda(f) for f in host[s:s + m]]
                pristine = _clone(dev)
                outs = _clone(dev) if kind.startswith("lookback") else None
                d, c, sc, tp, tc, _ = _call(eng, trk, kind, dev, vids[s:s + m], layout, matrix, style, outs=outs, crops=crops)
                assert np.array_equal(sc, np.ones(m, np.float32)), (kind, sc)
                got = eng.read_dets(d, c, m)
                lists = trk.read(tp, tc, m)
                d2, c2 = eng.detect_yuv_tiled_device(pristine, THR, NMS, layout=layout, matrix=matrix)
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
            assert found >= len(spots) * len(host), (kind, found)      # the small faces are found
            if twin is not None:
                _same_state(trk, twin, nvideos, kind)
                twin.close()
            trk.close()
    finally:
        eng.close()


# ---- 2. the fitted level alone is the letter-box --------------------------------------------------------------------------------
FITTED_KINDS = {
    "plain": {}, "crops": {}, "redact": {}, "motion": {"motion": True}, "best": {"best": {}}, "follow": {"follow": True},
    "follow+motion": {"follow": True, "motion": True}, "lookback": {"lookback": 2}, "lookback15+motion": {"lookback": 15, "motion": True},
    "lookback+search": {"lookback": 2, "lookback_search": True}, "lookback+follow": {"lookback": 3, "lookback_follow": True},
}


def _fitted_run(eng, trk, kind, dev, style):
    """Every frame of one 1080p video through trk, two frames a call; follow kinds detect every other call.  Returns everything the
    calls output, on the host."""
    import torch
    out = []
    crops = torch.zeros((2, 128, 112, 112, 3), dtype=torch.uint8, device="cuda") if kind in ("best", "crops") else None
    for s in range(0, len(dev), 2):
        views, vids = dev[s:s + 2], [0] * len(dev[s:s + 2])
        m = len(views)
        follow = "follow" in kind and (s // 2) % 2 == 1
        if follow and kind.startswith("lookback"):
            nums, tp, tc = trk.follow_redact_lookback_device(views, vids, views, style=style[0], shape=style[1])
            extra = [nums, "follow"]
        elif follow:
            tp, tc = trk.follow_device(views, vids)
            extra = ["follow"]
        elif kind == "crops":
            crops.zero_()
            tp, tc, d, c, sc = trk.detect_yuv_device(views, vids, THR, NMS, align={"max_faces": 128}, dev_crops_ptr=crops.data_ptr())
            eng.synchronize()
            extra = [crops[:m].cpu().numpy()]
        elif kind.startswith("lookback"):
            nums, tp, tc, d, c, sc = trk.detect_yuv_redact_lookback_device(views, vids, views, THR, NMS, style=style[0], shape=style[1])
            extra = [nums]
            if trk.lookback_search_on:      # the step records of each birth's steps taken; rows past them are not written
                steps, lengths = trk.lookback_search(m)
                extra += [lengths] + [steps[i, r, :lengths[i, r]] for i in range(m) for r in range(steps.shape[1])]
        else:
            d, c, sc, tp, tc, bx = _call(eng, trk, kind, views, vids, "nv12", "bt601", style, crops=crops)
            eng.synchronize()
            extra = [] if bx is None else [trk.read_best(bx[0], bx[1], m), crops[:m].cpu().numpy()]
        lists = trk.read(tp, tc, m)
        out.append(lists)
        if any(isinstance(x, str) for x in extra):      # each frame's follow records, in its list order
            fo = trk.follow(m)
            extra = [x for x in extra if not isinstance(x, str)] + [fo[i, :len(lists[i])] for i in range(m)]
        if trk.motion_on:
            out.append(trk.motion(m))
        out += extra
    if kind.startswith("lookback"):
        outs = _clone(dev[:trk.lookback])
        out.append(trk.drain(0, outs, style=style[0], shape=style[1]))
        out += _host(outs)
    out += _host(dev)
    out.append(trk.debug_state(0))
    return out


def _flat(x):
    if isinstance(x, (list, tuple)):
        return [y for e in x for y in _flat(e)]
    return [np.asarray(x).tobytes()]


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_fitted_level_alone_equals_no_tiling(golden_image, prec):
    """levels = {{0, 0}} on 1920 x 1080 frames: every kind's lists, state, motions, follow records, redacted and look-back bytes, best
    shots and crops equal a twin tracker without tiling, bit for bit."""
    big = cv2.resize(golden_image, (1600, 1108))
    bgr = []
    for k in range(8):
        c = np.full((1080, 1920, 3), 40, np.uint8)
        x, y = 40 + 9 * k, 6 * (k % 3)
        c[y:y + 1060, x:x + 1600] = big[:1060]
        bgr.append(c)
    eng = _engine(prec, max_image=(1080, 1920))
    try:
        for kind, opts in FITTED_KINDS.items():
            style = STYLES[len(kind) % 2]
            got = []
            for tiling in ({"levels": [(0.0, 0)]}, None):
                trk = eng.tracker(max_tracks=128, tiling=tiling, **opts)
                got.append(_flat(_fitted_run(eng, trk, kind, _device(bgr, "nv12"), style)))
                trk.close()
            assert len(got[0]) == len(got[1]), kind
            for i, (a, b) in enumerate(zip(*got)):
                assert a == b, (prec, kind, i)
    finally:
        eng.close()


# ---- 3. the gap is closed ---------------------------------------------------------------------------------------------------------
SPOTS_4K = [(32, 32), (1376, 32), (2720, 32), (32, 992), (1376, 1536), (2720, 992)]


def _planted(eng, golden, nframes):
    """The 4K video and every planted face's box on every frame: the faces the tiled detector finds in the half photo alone."""
    half = _half(golden)
    faces = eng.detect_tiled([half], THR, NMS)[0][0]
    assert len(faces) >= 3
    bgr = _scene(golden, 3840, 2160, nframes, SPOTS_4K)
    boxes = [[(f[1] + x + 3 * k, f[2] + y + 2 * k, f[3] + x + 3 * k, f[4] + y + 2 * k) for f in faces for x, y in SPOTS_4K] for k in range(nframes)]
    return bgr, boxes


def _inner(box, w, h):
    x1, y1, x2, y2 = box
    dx, dy = 0.2 * (x2 - x1), 0.2 * (y2 - y1)
    return int(max(0, x1 + dx)), int(max(0, y1 + dy)), int(min(w, x2 - dx)), int(min(h, y2 - dy))


def _covered(out, orig, box, w=3840, h=2160):
    """More than half the luma samples of the box's inner 60 % were written."""
    x1, y1, x2, y2 = _inner(box, w, h)
    return (out[y1:y2, x1:x2] != orig[y1:y2, x1:x2]).mean() > 0.5


def _untouched(out, orig, box, w=3840, h=2160):
    x1, y1, x2, y2 = _inner(box, w, h)
    return np.array_equal(out[y1:y2, x1:x2], orig[y1:y2, x1:x2])


@pytest.mark.parametrize("k", [1, 3])
def test_small_faces_are_redacted_on_every_frame(golden_image, k):
    """3840 x 2160, faces 30-60 px moving a few pixels per frame: a look-back tracker without tiling leaves every face untouched on
    every frame; with tiling every planted face lies inside a written region on every emitted frame, also at detect_every = 3."""
    from retinaface_b200.detector import RetinaFace
    L, nframes = 2, 9
    eng = _engine("fp16", max_image=(2160, 3840), max_faces=512)
    try:
        bgr, boxes = _planted(eng, golden_image, nframes)
        orig = [bgr_to_frame(b, "nv12") for b in bgr]
        for tiling in (None, True):
            if k > 1 and not tiling:
                continue
            rf = RetinaFace.__new__(RetinaFace)
            rf.engine, rf.nms_threshold = eng, NMS
            dev = [_cuda(f) for f in orig]
            for s in range(0, nframes, L):
                rf.redactFrames(dev[s:s + L], [0] * len(dev[s:s + L]), THR, lookback=L, detect_every=k, max_videos=1, tiling=tiling)
            outs = _clone(dev[:L])
            drained = rf.drainVideo(0, outs)
            assert list(drained) == list(range(nframes - L, nframes))
            got = _host(dev[L:nframes]) + _host(outs)      # frame e was emitted into the input of frame e + L, then the drain
            for e in range(nframes):
                for b in boxes[e]:
                    if tiling:
                        assert _covered(got[e][:2160], orig[e][:2160], b), (k, e, b)
                    else:
                        assert _untouched(got[e][:2160], orig[e][:2160], b), (e, b)
    finally:
        eng.close()


# ---- 4. ordering over the tiled ring --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("streams", [2, 8])
def test_calls_in_flight_equal_blocking(golden_image, streams):
    """2 streams + 1 redacting tiling-tracker calls in flight, interleaved with standalone tiled device calls and letter-box detect
    calls on the same handle: every redacted frame and every video's state equal the same calls made one at a time."""
    ncalls = 2 * streams + 1
    spots = [(32, 16), (1376, 16), (704, 976)]
    host = [bgr_to_frame(_scene(golden_image, 2560, 1440, 1, spots, video=v, step=(0, 0))[0], "nv12") for v in range(ncalls)]
    results = []
    for blocking in (True, False):
        eng = _engine("fp16", streams=streams)
        try:
            trk = eng.tracker(max_videos=ncalls, max_tracks=128, tiling=True)
            dev = [_cuda(f) for f in host]
            side = [_cuda(f) for f in host]
            for i in range(ncalls):
                trk.detect_yuv_redact_device([dev[i]], [i], THR, NMS)
                if blocking:
                    eng.synchronize()
                eng.detect_yuv_tiled_device([side[(i + 1) % ncalls]], THR, NMS)
                eng.detect_yuv_device([side[i]], THR, NMS)
                if blocking:
                    eng.synchronize()
            results.append((_host(dev), [trk.debug_state(v) for v in range(ncalls)]))
            trk.close()
        finally:
            eng.close()
    (a, sa), (b, sb) = results
    for i in range(ncalls):
        assert np.array_equal(a[i], b[i]), (streams, i)
        assert np.array_equal(sa[i][0], sb[i][0]) and sa[i][1].tobytes() == sb[i][1].tobytes(), (streams, i)
    assert any(not np.array_equal(a[i], host[i]) for i in range(ncalls))      # something was redacted


# ---- 5. refusals ------------------------------------------------------------------------------------------------------------------
def _status(eng, fn, *args):
    rc = fn(*args)
    return rc, (eng.lib.rf_last_error(eng.h) or b"").decode()


def test_setter_refusals(golden_image):
    from retinaface_b200 import capi
    eng = _engine("fp16")
    lib = eng.lib
    try:
        def setter(trk, levels=None, nlevels=None, overlap=0):
            t = capi.tiling(levels, overlap)
            if nlevels is not None:
                t.nlevels = nlevels
            return _status(eng, lib.rf_tracker_set_tiling, trk.t, C.byref(t))

        trk = eng.tracker()
        bad = [({"nlevels": 9}, "nlevels 9, must be in [0, 8]"), ({"nlevels": -1}, "nlevels -1, must be in [0, 8]"),
               ({"levels": [(1.0, 0), (-0.5, 0)]}, "level 1: scale -0.5, must be finite and >= 0"),
               ({"levels": [(float("nan"), 0)]}, "level 0: scale nan, must be finite and >= 0"),
               ({"levels": [(float("inf"), 0)]}, "level 0: scale inf, must be finite and >= 0"),
               ({"overlap": 8}, "overlap 8, must be 0 (64) or in [16, 224]"), ({"overlap": 225}, "overlap 225, must be 0 (64) or in [16, 224]")]
        for kw, msg in bad:
            rc, err = setter(trk, **kw)
            assert rc == INVALID_ARG and err == "rf_tracker_set_tiling: " + msg, (kw, rc, err)
        # NULL tiling, NULL levels with a count and a copied array are all fine; a second call is refused
        assert _status(eng, lib.rf_tracker_set_tiling, trk.t, None)[0] == 0
        rc, err = setter(trk)
        assert rc == INVALID_ARG and err == "rf_tracker_set_tiling: tiling is already on", err
        trk.close()
        trk = eng.tracker()
        t = capi.Tiling(None, 3, 0)
        assert _status(eng, lib.rf_tracker_set_tiling, trk.t, C.byref(t))[0] == 0
        trk.close()
        # after an update
        trk = eng.tracker()
        dev = _device(_scene(golden_image, 2560, 1440, 1, [(32, 16)]), "nv12")
        trk.detect_yuv_device(dev, [0], THR, NMS)
        rc, err = setter(trk)
        assert rc == INVALID_ARG and err == "rf_tracker_set_tiling: the tracker has already been updated", err
        trk.close()
    finally:
        eng.close()
    npp = _engine("fp16", flags=capi.RF_FLAG_NPP_RESIZE)
    try:
        trk = npp.tracker()
        rc, err = _status(npp, npp.lib.rf_tracker_set_tiling, trk.t, None)
        assert rc == UNSUPPORTED and err.startswith("rf_tracker_set_tiling: tiles are levels of cv::resize"), err
        trk.close()
    finally:
        npp.close()


@pytest.mark.parametrize("kind", ["plain", "best", "follow", "lookback", "lookback+follow", "motion"])
def test_setter_admission_rows(golden_image, kind):
    """test_admission_table's rows for the new setter: every kind takes it before its first frame call, in any order with the other
    setters, and refuses it after one."""
    eng = _engine("fp16")
    opts = {"plain": {}, "best": {"best": {}}, "follow": {"follow": True}, "lookback": {"lookback": 2},
            "lookback+follow": {"lookback": 2, "lookback_follow": True}, "motion": {"motion": True}}[kind]
    try:
        trk = eng.tracker(**opts)
        trk.set_tiling()
        if kind == "plain":
            trk.set_motion()           # a setter after tiling
        trk.close()
    finally:
        eng.close()


def test_frame_size_statuses_launch_nothing(golden_image):
    """A level side above 16384 or of 0 and more than RF_MAX_TILES tiles are the frame call's own statuses, before anything is
    launched or allocated: output canaries stay, frames stay untouched and the look-back buffers are not allocated."""
    import torch
    from retinaface_b200 import capi
    eng = _engine("fp16")
    lib = eng.lib
    try:
        cases = [([(7.0, 0)], INVALID_ARG, "level 0: scale 7 resizes 2560x1440 to 17920x10080; each side must be in [1, 16384]"),
                 ([(1e-4, 0)], INVALID_ARG, "level 0: scale 0.0001 resizes 2560x1440 to 0x0; each side must be in [1, 16384]"),
                 ([(4.0, 0)], CAPACITY, "the layout of a 2560x1440 image has more than RF_MAX_TILES = 256 tiles")]
        frame = bgr_to_frame(_scene(golden_image, 2560, 1440, 1, [(32, 16)])[0], "nv12")
        for levels, want, msg in cases:
            trk = eng.tracker(lookback=15, tiling={"levels": levels})
            dev = [_cuda(frame)]
            outs = [_cuda(np.full_like(frame, 0x5A))]
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            arr, oarr = eng._frames(dev, "nv12", True), eng._frames(outs, "nv12", True)
            vids = (C.c_int * 1)(0)
            canary = [C.c_void_p(0xDEAD) for _ in range(4)]
            sc = np.full(1, 7.0, np.float32)
            nums = np.full(1, 77, np.int32)
            st = capi.redact_style("blur", "ellipse")
            rc, err = _status(eng, lib.rf_detect_yuv_redact_lookback_device, eng.h, trk.t, arr, vids, 1, 0, THR, NMS, C.byref(st), oarr,
                              nums.ctypes.data, *[C.byref(p) for p in canary], sc.ctypes.data)
            assert rc == want and err == "rf_detect_yuv_redact_lookback_device: image 0: " + msg, (levels, rc, err)
            assert [p.value for p in canary] == [0xDEAD] * 4 and sc[0] == 7.0 and nums[0] == 77
            torch.cuda.synchronize()
            assert free0 - torch.cuda.mem_get_info()[0] < 32 << 20          # an allocated look-back buffer would take 83 MB
            assert np.array_equal(_host(dev)[0], frame) and (_host(outs)[0] == 0x5A).all()
            trk.close()
            # the plain detect call reports the same status
            trk = eng.tracker(tiling={"levels": levels})
            sc2 = np.full(1, 7.0, np.float32)
            rc, err = _status(eng, lib.rf_detect_yuv_track_device, eng.h, trk.t, arr, vids, 1, 0, THR, NMS, None, None, None,
                              *[C.byref(p) for p in canary], sc2.ctypes.data)
            assert rc == want and err == "rf_detect_yuv_track_device: image 0: " + msg, (levels, rc, err)
            trk.close()
        # a frame above max_image is the frame check's refusal, as before
        trk = eng.tracker(tiling=True)
        big = [_cuda(np.zeros((2160 * 3 // 2, 3840), np.uint8))]
        rc, err = _status(eng, lib.rf_detect_yuv_track_device, eng.h, trk.t, eng._frames(big, "nv12", True), (C.c_int * 1)(0), 1, 0, THR,
                          NMS, None, None, None, None, None, None, None, None)
        assert rc == CAPACITY and "larger than max_image" in err, err
        trk.close()
    finally:
        eng.close()


# ---- 6. the drivers ------------------------------------------------------------------------------------------------------------------
def test_detector_surfaces_equal_hand_calls(golden_image):
    """RetinaFace.trackFrames / redactFrames with tiling (and lookback, detect_every) equal the same tracker calls made by hand."""
    from retinaface_b200.detector import RetinaFace
    spots = [(32, 16), (1376, 16), (704, 976)]
    host = [bgr_to_frame(b, "nv12") for b in _scene(golden_image, 2560, 1440, 6, spots)]
    eng = _engine("fp16")
    try:
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        dev = [_cuda(f) for f in host]
        lists = [rf.trackFrames(dev[s:s + 3], [0, 0, 0], THR, max_videos=1, tiling=True)[0] for s in (0, 3)]
        trk = eng.tracker(max_videos=1, tiling=True)
        for s, got in zip((0, 3), lists):
            tp, tc, _, _, _ = trk.detect_yuv_device(dev[s:s + 3], [0, 0, 0], THR, NMS)
            assert got == RetinaFace._lists(trk.read(tp, tc, 3))
        trk.close()
        rf._tracker.close()
        # redactFrames(lookback=2, detect_every=3, tiling=...) against the following look-back tracker's calls
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        a = [_cuda(f) for f in host]
        b = [_cuda(f) for f in host]
        nums = [rf.redactFrames(a[s:s + 3], [0, 0, 0], THR, lookback=2, detect_every=3, max_videos=1, tiling={"overlap": 48})
                for s in (0, 3)]
        trk = eng.tracker(max_videos=1, lookback=2, lookback_follow=True, tiling={"overlap": 48})
        for s, want in zip((0, 3), nums):
            got = trk.detect_yuv_redact_lookback_device(b[s:s + 1], [0], b[s:s + 1], THR, NMS)[0]
            got = np.concatenate([got, trk.follow_redact_lookback_device(b[s + 1:s + 3], [0, 0], b[s + 1:s + 3])[0]])
            assert np.array_equal(got, want)
        for x, y in zip(_host(a), _host(b)):
            assert np.array_equal(x, y)
        trk.close()
        rf._tracker.close()
        # asking for tiling on a detector whose tracker was made without it
        rf = RetinaFace.__new__(RetinaFace)
        rf.engine, rf.nms_threshold = eng, NMS
        rf.trackFrames(a[:1], [0], THR, max_videos=1)
        with pytest.raises(ValueError):
            rf.trackFrames(a[1:2], [0], THR, tiling=True)
        with pytest.raises(ValueError):
            rf.redactFrames(a[1:2], [0], THR, tiling={"overlap": 48})
        rf._tracker.close()
    finally:
        eng.close()


CPP_PROGRAM = r'''
#include "RetinaFace.h"
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <fstream>
// argv: model directory, frames file (n NV12 2560x1440 frames), out file, n.  redactYUV with tiling, three frames a call, then the bytes.
int main(int argc, char **argv) {
    string model = argv[1];
    const int n = atoi(argv[4]), w = 2560, h = 1440;
    const size_t bytes = (size_t)w * h * 3 / 2;
    std::vector<unsigned char> buf(bytes * n);
    std::ifstream(argv[2], std::ios::binary).read((char *)buf.data(), buf.size());
    RetinaFaceOptions opt;
    opt.net_w = opt.net_h = 448;
    opt.model_file = "mnet25.caffemodel";
    opt.track_tiling = true;
    opt.track_tile_scales = {1.f, 0.5f, 0.f};
    opt.track_tile_overlap = 48;
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


def test_host_shell_redact_with_tiling_equals_c_calls(golden_image, tmp_path):
    """The C++ RetinaFace::redactYUV with RetinaFaceOptions::track_tiling gives the bytes of the same C calls."""
    from retinaface_b200.build import HERE, build_host
    from retinaface_b200 import Engine, RF_PREC_FP16
    build_host()
    yf = [f for f in YuvFrameFields()]
    assert yf == ["y", "u", "v", "y_pitch", "uv_pitch", "uv_step", "width", "height"]
    spots = [(32, 16), (1376, 16), (704, 976)]
    host = [bgr_to_frame(b, "nv12") for b in _scene(golden_image, 2560, 1440, 6, spots)]
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
        trk = eng.tracker(max_videos=16, tiling={"levels": [(1.0, 0), (0.5, 0), (0.0, 0)], "overlap": 48})
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


def YuvFrameFields():
    from retinaface_b200 import capi
    return [f for f, _ in capi.YuvFrame._fields_]
