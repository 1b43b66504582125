"""GPU (-m gpu): f10 tracking -- rf_detect_yuv_track_device and rf_track_update against oracle/track.py bit for bit (ids, states,
every float field and the FP64 Kalman state), the behaviour on a synthetic 40-frame 1080p video, the new-identity crops, the ordering
rules (videos and frames in one call, calls in flight over the contexts, reset) and that nothing else changes."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.track import CONFIRMED, TENTATIVE, TrackerOracle
from oracle.yuv import bgr_to_frame

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
W, H, NF = 1920, 1080, 40
X0, Y0 = 100, 40
FIELDS = ("id", "state", "det", "crop_slot", "hits", "age", "lost_frames")


def _engine(prec="fp16", **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (H, W))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


@pytest.fixture(scope="module")
def video(golden_image):
    """40 NV12 frames: the golden photo moving (7, 3) px per frame on grey, a grey occluder over its best face on frames 12-17, and a
    2x copy of that face entering from the right at frame 25 (moving left 4 px per frame).  Returns (nv12 frames, occluded face box
    at frame 0)."""
    eng = _engine("fp32")
    faces = eng.detect_batch([golden_image], 0.8, NMS)[0]
    eng.close()
    sc = max(golden_image.shape[1] / 448, golden_image.shape[0] / 448, 1.0)     # network-input pixels -> photo pixels
    occ = (faces[0, 1:5] * sc).astype(int)
    x1, y1, x2, y2 = occ
    face = golden_image[max(y1 - 20, 0):y2 + 20, max(x1 - 20, 0):x2 + 20]
    face = cv2.resize(face, (face.shape[1] * 2, face.shape[0] * 2))
    frames = []
    for t in range(NF):
        img = np.full((H, W, 3), 128, np.uint8)
        ox, oy = X0 + 7 * t, Y0 + 3 * t
        img[oy:oy + golden_image.shape[0], ox:ox + golden_image.shape[1]] = golden_image
        if 12 <= t <= 17:
            img[oy + y1 - 10:oy + y2 + 10, ox + x1 - 10:ox + x2 + 10] = 128
        if t >= 25:
            fx = W - face.shape[1] - 10 - 4 * (t - 25)
            img[300:300 + face.shape[0], fx:fx + face.shape[1]] = face
        frames.append(bgr_to_frame(img, "nv12"))
    return frames, occ


def _cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _same(dev, want, what):
    assert len(dev) == len(want), (what, [int(r["id"]) for r in dev], [w["id"] for w in want])
    for r, w in zip(dev, want):
        for f in FIELDS:
            assert int(r[f]) == w[f], (what, f, int(r[f]), w[f])
        for f in ("kx1", "ky1", "kx2", "ky2", "vx", "vy"):
            assert np.float32(r[f]).tobytes() == np.float32(w[f]).tobytes(), (what, f, r[f], w[f])
        assert np.array_equal(r["face"].view(np.uint32), w["face"].view(np.uint32)), what


def _track_video(eng, trk, frames, per_call=1, align=None, crops=None):
    """The video through rf_detect_yuv_track_device, per_call frames of video 0 per call; per frame (tracks, records, scale)."""
    out = []
    for s in range(0, len(frames), per_call):
        chunk = frames[s:s + per_call]
        tp, tc, d, c, sc = trk.detect_yuv_device(chunk, [0] * len(chunk), THR, NMS, align=align,
                                                  dev_crops_ptr=crops[s:s + per_call].data_ptr() if crops is not None else None)
        recs = eng.read_dets(d, c, len(chunk))[0]
        tr = trk.read(tp, tc, len(chunk))
        out += [(tr[i], recs[i], sc[i]) for i in range(len(chunk))]
    return out


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_tracks_equal_the_oracle(video, prec):
    """Ids, states, det, hits, lost_frames, every float field and the FP64 Kalman state equal oracle/track.py fed the records of
    rf_detect_yuv_batch_device, on every frame; the records themselves equal rf_detect_yuv_batch_device's."""
    frames, _ = video
    eng = _engine(prec)
    trk = eng.tracker()
    dev = [_cuda(f) for f in frames]
    o = TrackerOracle(1)
    got = _track_video(eng, trk, dev, per_call=8)
    for t, (tracks, recs, sc) in enumerate(got):
        d, c, sc2 = eng.detect_yuv_device([dev[t]], THR, NMS)
        ref = eng.read_dets(d, c, 1)[0][0]
        assert np.array_equal(ref, recs) and sc2[0] == sc, t
        _same(tracks, o.update(0, ref, sc), f"{prec} frame {t}")
    hdr, rows = trk.debug_state(0)
    want = o.debug_state(0)
    assert np.array_equal(np.r_[hdr, rows.reshape(-1)].view(np.uint64), want.view(np.uint64))
    trk.close()
    eng.close()


def test_behaviour_on_the_synthetic_video(video):
    frames, _ = video
    eng = _engine("fp16")
    trk = eng.tracker()
    got = _track_video(eng, trk, [_cuda(f) for f in frames], per_call=4)
    first = [int(r["id"]) for r in got[0][0]]
    assert len(first) >= 3 and all(r["state"] == CONFIRMED for r in got[0][0])
    for t, (tracks, _, _) in enumerate(got):
        ids = {int(r["id"]): r for r in tracks}
        assert set(first) <= set(ids), t                                  # one id each over all 40 frames
        if t > 10:
            for i in first:
                r = ids[i]
                if r["det"] >= 0:
                    assert abs(r["vx"] - 7) <= 1 and abs(r["vy"] - 3) <= 1, (t, i, r["vx"], r["vy"])
    occluded = [i for i in first if any(int(r["id"]) == i and r["det"] < 0 for r in got[14][0])]
    assert occluded, "the occluder hid no tracked face"
    for i in occluded:      # it comes back with its old id once the occluder is gone
        assert any(r["det"] >= 0 and r["state"] == CONFIRMED for tracks, _, _ in got[18:26] for r in tracks if int(r["id"]) == i), i
    # the entering copy: a new id whose face lies right of the photo (a face of the photo first found on a later frame is new too)
    new = [(t, r) for t, (tracks, _, _) in enumerate(got) for r in tracks if r["id"] > max(first) and r["face"][1] > X0 + 7 * t + 1280]
    assert new and new[0][0] >= 25, new[:1]
    t0, r0 = new[0]
    assert r0["state"] == TENTATIVE and r0["hits"] == 1
    later = [r for t, r in new if r["id"] == r0["id"] and r["hits"] == 2]
    assert later and later[0]["state"] == CONFIRMED
    trk.close()
    eng.close()


def test_crops_only_for_new_identities(video):
    """A crop is cut only on the frame its track is confirmed, and equals the crop rf_detect_yuv_batch_device cuts for the matched
    record; the other slots keep their canary."""
    import torch
    frames, _ = video
    eng = _engine("fp16")
    trk = eng.tracker()
    A, mf = 4, eng.max_faces
    dev = [_cuda(f) for f in frames]
    crops = torch.full((NF, A, 112, 112, 3), 0xA5, dtype=torch.uint8, device="cuda")
    got = _track_video(eng, trk, dev, per_call=1, align=dict(max_faces=A), crops=crops)
    eng.synchronize()
    cut = 0
    prev = {}
    for t, (tracks, recs, _) in enumerate(got):
        ref = torch.full((1, mf, 112, 112, 3), 0x5A, dtype=torch.uint8, device="cuda")
        eng.detect_yuv_device([dev[t]], THR, NMS, align=dict(), dev_crops_ptr=ref.data_ptr())
        eng.synchronize()
        used = set()
        newly_ids = [int(r["id"]) for r in tracks if r["state"] == CONFIRMED and (t == 0 or prev.get(int(r["id"])) == TENTATIVE)]
        assert [int(r["id"]) for r in tracks if r["crop_slot"] >= 0] == newly_ids[:A], t
        for r in tracks:
            newly = int(r["id"]) in newly_ids
            if r["crop_slot"] >= 0:
                assert newly
                used.add(int(r["crop_slot"]))
                assert torch.equal(crops[t, r["crop_slot"]], ref[0, r["det"]]), (t, r["id"])
                cut += 1
        for j in set(range(A)) - used:
            assert bool((crops[t, j] == 0xA5).all()), (t, j)
        prev = {int(r["id"]): int(r["state"]) for r in tracks}
    assert cut >= 4
    trk.close()
    eng.close()


def _all(trk, tp, tc, n):
    return [a.tobytes() for a in trk.read(tp, tc, n)]


def test_ordering_rules(video, golden_image):
    frames, _ = video
    dev = [_cuda(f) for f in frames]
    eng = _engine("fp16")
    # eight videos in one call == eight separate calls; 8 consecutive frames of one video in one call == 8 single-frame calls
    a, b = eng.tracker(max_videos=8), eng.tracker(max_videos=8)
    for s in range(4):
        fr = [dev[v + s] for v in range(8)]
        tp, tc, _, _, _ = a.detect_yuv_device(fr, list(range(8)), THR, NMS)
        one = _all(a, tp, tc, 8)
        sep = []
        for v in range(8):
            tp, tc, _, _, _ = b.detect_yuv_device([fr[v]], [v], THR, NMS)
            sep += _all(b, tp, tc, 1)
        assert one == sep, s
    c, d = eng.tracker(), eng.tracker()
    tp, tc, _, _, _ = c.detect_yuv_device(dev[:8], [0] * 8, THR, NMS)
    one = _all(c, tp, tc, 8)
    sep = []
    for t in range(8):
        tp, tc, _, _, _ = d.detect_yuv_device([dev[t]], [0], THR, NMS)
        sep += _all(d, tp, tc, 1)
    assert one == sep
    # reset mid-sequence restarts ids at 1 for that video only
    for t in range(8, 12):
        tp, tc, _, _, _ = a.detect_yuv_device([dev[t], dev[t]], [0, 1], THR, NMS)
    before = a.read(tp, tc, 2)
    a.reset(1)
    tp, tc, _, _, _ = a.detect_yuv_device([dev[12], dev[12]], [0, 1], THR, NMS)
    after = a.read(tp, tc, 2)
    assert [int(r["id"]) for r in after[1]] == list(range(1, len(after[1]) + 1))
    assert set(int(r["id"]) for r in before[0]) <= set(int(r["id"]) for r in after[0]) | {0}
    assert max(int(r["id"]) for r in after[0]) == max(int(r["id"]) for r in before[0])
    for t in (a, b, c, d):
        t.close()
    eng.close()
    # 2 * streams + 1 calls in flight on streams 2 and 8 equal the same calls one at a time, bit for bit (a streams = 1 handle runs
    # the latency-oriented layer plan, whose records are not the same bits, so the reference is a handle of the same plan with a
    # synchronize after every call)
    res = {}
    for streams in (2, 8):
        e = _engine("fp16", streams=streams)
        k = e.tracker(max_videos=2)
        n_calls = 2 * max(streams, 2) + 1
        for i in range(n_calls):
            tp, tc, _, _, _ = k.detect_yuv_device([dev[i], dev[NF - 1 - i]], [0, 1], THR, NMS)
        res[streams] = (_all(k, tp, tc, 2), [np.r_[x[0], x[1].reshape(-1)].tobytes() for x in (k.debug_state(0), k.debug_state(1))], n_calls)
        k.close()
        e.close()
    for s in (2, 8):
        e = _engine("fp16", streams=s)
        k = e.tracker(max_videos=2)
        for i in range(res[s][2]):
            tp, tc, _, _, _ = k.detect_yuv_device([dev[i], dev[NF - 1 - i]], [0, 1], THR, NMS)
            e.synchronize()
        ref = (_all(k, tp, tc, 2), [np.r_[x[0], x[1].reshape(-1)].tobytes() for x in (k.debug_state(0), k.debug_state(1))])
        assert res[s][:2] == ref, s
        k.close()
        e.close()


def test_update_on_tiled_device_records(video):
    """rf_track_update on rf_detect_tiled_device records (already in image pixels: scales NULL) equals the oracle."""
    import torch
    frames, _ = video
    eng = _engine("fp16")
    trk = eng.tracker()
    o = TrackerOracle(1)
    from oracle.yuv import frame_to_bgr
    for t in range(0, 12, 3):
        img = torch.from_numpy(frame_to_bgr(frames[t], "nv12")).cuda()
        d, c = eng.detect_tiled_device([img], THR, NMS)
        tp, tc = trk.update([0], d, c)
        recs = eng.read_dets(d, c, 1)[0][0]
        _same(trk.read(tp, tc, 1)[0], o.update(0, recs, None), f"tiled {t}")
    trk.close()
    eng.close()


def test_nothing_else_changes_and_bad_calls_launch_nothing(video, golden_image):
    from retinaface_b200 import capi
    frames, _ = video
    dev = [_cuda(f) for f in frames[:2]]
    eng = _engine("fp16")
    base = eng.detect_batch([golden_image], THR, NMS)[0]
    d, c, _ = eng.detect_yuv_device(dev, THR, NMS)
    yuv = eng.read_dets(d, c, 2)[0]
    launches = eng.launches_per_batch(2)
    trk = eng.tracker(max_videos=2)
    tp, tc, d2, c2, _ = trk.detect_yuv_device(dev, [0, 1], THR, NMS)
    assert [np.array_equal(a, b) for a, b in zip(eng.read_dets(d2, c2, 2)[0], yuv)] == [True, True]
    state = [trk.debug_state(v)[0].tobytes() for v in (0, 1)]
    lib, t = eng.lib, trk.t
    can_t, can_c = C.c_void_p(0x1234), C.c_void_p(0x5678)
    vids = (C.c_int * 2)(0, 1)
    bad_v = (C.c_int * 2)(0, 2)
    sc = (C.c_float * 2)(1.0, 1.0)
    for args, status in (((t, bad_v, 2, d2, c2, sc), -1), ((t, None, 2, d2, c2, sc), -1), ((t, vids, 2, None, c2, sc), -1),
                         ((t, vids, 9, d2, c2, sc), -6), ((t, vids, 2, d2, c2, (C.c_float * 2)(1.0, float("nan"))), -1),
                         ((t, vids, 2, d2, c2, (C.c_float * 2)(1.0, 0.0)), -1), ((t, vids, 2, d2, c2, (C.c_float * 2)(1.0, -2.0)), -1)):
        assert lib.rf_track_update(*args, C.byref(can_t), C.byref(can_c)) == status, args
        assert (can_t.value, can_c.value) == (0x1234, 0x5678)
    arr = eng._frames(dev, "nv12", True)
    bad_align = capi.align_params(crop=(4, 4))
    good_align = capi.align_params()
    for args, status in (((bad_v, 2, 0, None, None), -1), ((vids, 2, 5, None, None), -1), ((vids, 2, 0, C.byref(bad_align), 1), -1),
                         ((vids, 2, 0, C.byref(good_align), None), -1), ((vids, 9, 0, None, None), -6)):
        v, n, m, al, cr = args
        assert lib.rf_detect_yuv_track_device(eng.h, t, arr, v, n, m, THR, NMS, al, cr, None, C.byref(can_t), C.byref(can_c), None, None,
                                              None) == status, args
        assert (can_t.value, can_c.value) == (0x1234, 0x5678)
    assert lib.rf_tracker_reset(t, 2) == -1 and lib.rf_tracker_reset(t, -2) == -1
    bad_cfg = [capi.TrackConfig(0, 0, 0, 0, 0, 0, 0, 0), capi.TrackConfig(1, 1025, 0, 0, 0, 0, 0, 0), capi.TrackConfig(1, 0, 1.5, 0, 0, 0, 0, 0),
               capi.TrackConfig(1, 0, 0, 0, float("nan"), 0, 0, 0), capi.TrackConfig(1, 0, 0, 0, 0, 0, 0, -1)]
    for cfg in bad_cfg:
        out = C.c_void_p(0x42)
        assert lib.rf_tracker_create(eng.h, C.byref(cfg), C.byref(out)) == -1
    assert [trk.debug_state(v)[0].tobytes() for v in (0, 1)] == state     # nothing was applied
    assert np.array_equal(eng.detect_batch([golden_image], THR, NMS)[0], base)
    d, c, _ = eng.detect_yuv_device(dev, THR, NMS)
    assert all(np.array_equal(a, b) for a, b in zip(eng.read_dets(d, c, 2)[0], yuv))
    assert eng.launches_per_batch(2) == launches
    trk.close()
    eng.close()


def test_detector_track_frames(video):
    from retinaface_b200 import RetinaFace
    frames, _ = video
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(H, W))
    dev = [_cuda(f) for f in frames[:3]]
    tracks, new = rf.trackFrames(dev, [0, 0, 0], THR, align=dict(max_faces=8))
    assert len(tracks) == 3 and len(tracks[0]) >= 3 and len(new[0]) == min(len(tracks[0]), 8) and new[1] == []
    assert [i for i, _, _ in tracks[2]] == sorted(i for i, _, _ in tracks[2])
