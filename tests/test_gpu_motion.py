"""GPU (-m gpu): f13 camera-motion compensation -- every rf_motion against oracle/motion.py and every track list and the FP64 Kalman
state against oracle/motion.py's MotionTrackerOracle, bit for bit, on a shaking 1080p video built from the golden photo (FP32, FP16, INT8; NV12
in a pitched surface and I420; 1, 4 and 8 frames per call); that the video breaks a plain tracker and not a motion tracker; LOST
tracks' redaction boxes following the camera; best-shot trackers; ordering; and the refusals."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.motion import FIRST, OK, MotionOracle, MotionTrackerOracle, applied
from oracle.redact import frame_regions, params, redact_yuv
from oracle.track import LOST
from oracle.yuv import bgr_to_frame

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
W, H, NF = 1920, 1080, 36
PITCH = 2048
FIELDS = ("id", "state", "det", "crop_slot", "hits", "age", "lost_frames")


def _engine(prec="fp16", **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (H, W))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


def _scene(seed=7, w=3000, h=2000):
    r = np.random.default_rng(seed)
    a = cv2.resize(r.integers(0, 256, (h // 24, w // 24, 3)).astype(np.uint8), (w, h), interpolation=cv2.INTER_CUBIC).astype(np.float32)
    b = cv2.resize(r.integers(0, 256, (h // 6, w // 6, 3)).astype(np.uint8), (w, h), interpolation=cv2.INTER_CUBIC).astype(np.float32)
    return np.clip(0.6 * a + 0.4 * b, 0, 255).astype(np.uint8)


def _shake(golden_image, lo=40, hi=70, reach=280):
    """NF BGR frames: the golden photo inside a textured scene, seen through a 1920 x 1080 window that moves by seeded steps of lo-hi
    px with changing signs (within reach of the start), holds still on frames 10-13 and zooms in 3 % per frame on frames 20-24.
    Returns (frames, per-frame scene -> frame matrices)."""
    S = _scene()
    gh, gw = golden_image.shape[:2]
    cx0, cy0 = S.shape[1] // 2, S.shape[0] // 2
    S[cy0 - gh // 2:cy0 - gh // 2 + gh, cx0 - gw // 2:cx0 - gw // 2 + gw] = golden_image
    rng = np.random.default_rng(11)
    cx, cy, z, sign = float(cx0), float(cy0), 1.0, 1.0
    frames, mats = [], []
    for t in range(NF):
        if t > 0 and not 10 <= t <= 13:
            if 20 <= t <= 24:
                z *= 1.03
            else:
                step = rng.uniform(lo, hi)
                if abs(cx + sign * step / z - cx0) > reach:
                    sign = -sign
                cx += sign * step / z
                cy += rng.uniform(-12, 12) / z
                cy = min(max(cy, cy0 - 25), cy0 + 25)
                sign = -sign if rng.uniform() < 0.5 else sign
        M = np.array([[z, 0, W / 2 - z * cx], [0, z, H / 2 - z * cy]])
        frames.append(cv2.warpAffine(S, M, (W, H), flags=cv2.INTER_LINEAR))
        mats.append(M)
    return frames, mats


@pytest.fixture(scope="module")
def shake(golden_image):
    return _shake(golden_image)


def _surfaces(frames):
    """NV12 device frames in NVDEC-like pitched surfaces: (y, uv) plane views, and the host luma planes."""
    import torch
    out, lumas = [], []
    for f in frames:
        buf = bgr_to_frame(f, "nv12")
        surf = np.full((H + 2 + H // 2, PITCH), 0xEE, np.uint8)
        surf[:H, :W] = buf[:H]
        surf[H + 2:, :W] = buf[H:]
        d = torch.from_numpy(surf).cuda()
        out.append((d[:H, :W], d[H + 2:, :W]))
        lumas.append(buf[:H].copy())
    torch.cuda.synchronize()
    return out, lumas


def _i420(frames):
    import torch
    out, lumas = [], []
    for f in frames:
        buf = bgr_to_frame(f, "i420")
        out.append(torch.from_numpy(buf).cuda())
        lumas.append(buf[:H].copy())
    torch.cuda.synchronize()
    return out, lumas


def _same(dev, want, what):
    assert len(dev) == len(want), (what, [int(r["id"]) for r in dev], [w["id"] for w in want])
    for r, w in zip(dev, want):
        for f in FIELDS:
            assert int(r[f]) == w[f], (what, f, int(r[f]), w[f])
        for f in ("kx1", "ky1", "kx2", "ky2", "vx", "vy"):
            assert np.float32(r[f]).tobytes() == np.float32(w[f]).tobytes(), (what, f, r[f], w[f])
        assert np.array_equal(r["face"].view(np.uint32), w["face"].view(np.uint32)), what


def _same_motion(got, want, what):
    assert (int(got["status"]), int(got["blocks"]), int(got["inliers"])) == (want["status"], want["blocks"], want["inliers"]), (what, got, want)
    assert np.array_equal(np.asarray(got["m"], np.float64).view(np.uint64), np.asarray(want["m"], np.float64).view(np.uint64)), (what, got, want)


def _run(eng, trk, dev, per_call, layout="nv12", videos=None):
    """The frames through rf_detect_yuv_track_device, per_call per call; per frame (tracks, records, scale, motion)."""
    out = []
    for s in range(0, len(dev), per_call):
        chunk = dev[s:s + per_call]
        vids = [0] * len(chunk) if videos is None else videos[s:s + per_call]
        tp, tc, d, c, sc = trk.detect_yuv_device(chunk, vids, THR, NMS, layout=layout)
        recs = eng.read_dets(d, c, len(chunk))[0]
        tr = trk.read(tp, tc, len(chunk))
        mo = trk.motion(len(chunk)) if trk.motion_on else [None] * len(chunk)
        out += [(tr[i], recs[i], sc[i], mo[i]) for i in range(len(chunk))]
    return out


@pytest.mark.parametrize("prec,per_call,layout", [("fp32", 8, "nv12"), ("fp16", 8, "nv12"), ("int8", 8, "nv12"), ("fp16", 1, "nv12"),
                                                  ("fp16", 4, "nv12"), ("fp16", 4, "i420")])
def test_motion_and_tracks_equal_the_oracles(shake, prec, per_call, layout):
    frames, _ = shake
    dev, lumas = _surfaces(frames) if layout == "nv12" else _i420(frames)
    eng = _engine(prec)
    trk = eng.tracker(motion=True)
    got = _run(eng, trk, dev, per_call, layout)
    mo, to = MotionOracle(1), MotionTrackerOracle(1)
    statuses = []
    for t, (tracks, recs, sc, m) in enumerate(got):
        want = mo.update(0, lumas[t], recs, len(recs), float(sc))
        _same_motion(m, want, f"{prec} {layout} frame {t}")
        statuses.append(want["status"])
        _same(tracks, to.update(0, recs, sc, motion=applied(want)), f"{prec} {layout} frame {t}")
    assert statuses[0] == FIRST and statuses.count(OK) >= NF - 3, statuses
    hdr, rows = trk.debug_state(0)
    assert np.array_equal(np.r_[hdr, rows.reshape(-1)].view(np.uint64), to.debug_state(0).view(np.uint64))
    trk.close()
    eng.close()


def test_estimates_follow_the_camera(shake):
    """The estimate maps the frame centre within 3 px (half a thumbnail pixel) of the true frame-to-frame transform."""
    frames, mats = shake
    dev, _ = _surfaces(frames)
    eng = _engine("fp16")
    trk = eng.tracker(motion=True)
    got = _run(eng, trk, dev, 8)
    for t in range(1, NF):
        A0 = np.r_[mats[t - 1], [[0, 0, 1]]]
        T = (np.r_[mats[t], [[0, 0, 1]]] @ np.linalg.inv(A0))[:2]
        m = got[t][3]["m"]
        c = np.array([W / 2, H / 2, 1.0])
        e = np.abs(np.array([m[0] * c[0] + m[1] * c[1] + m[2], m[3] * c[0] + m[4] * c[1] + m[5]]) - T @ c).max()
        assert int(got[t][3]["status"]) == OK and e <= 3.0, (t, e, m, T)
    trk.close()
    eng.close()


def test_plain_tracker_breaks_and_motion_tracker_keeps_ids(golden_image):
    """The photo's faces are about 100 px wide, so 40-70 px steps keep them inside a plain tracker's IoU gate; steps of 100-140 px
    (with the search radius at 24 thumbnail pixels, 144 px) take every face out of it."""
    frames, _ = _shake(golden_image, 100, 140, 260)
    dev, _ = _surfaces(frames)
    eng = _engine("fp16")
    kept, seen = {}, {}
    for motion in (False, dict(search=24)):
        trk = eng.tracker(motion=motion)
        got = _run(eng, trk, dev, 4)
        first = [int(r["id"]) for r in got[0][0]]
        assert len(first) >= 3
        # kept: each first-frame id is matched to a record (det >= 0) on at least 90 % of the frames -- a LOST track stays listed,
        # so presence alone proves nothing; a broken identity is LOST from its break on, and its face continues under a new id
        matched = {i: sum(any(int(r["id"]) == i and int(r["det"]) >= 0 for r in g[0]) for g in got) for i in first}
        seen[bool(motion)] = matched
        kept[bool(motion)] = min(matched.values()) >= 0.9 * len(got)
        trk.close()
    assert not kept[False], ("the video does not discriminate: a plain tracker keeps every identity", seen)
    assert kept[True], seen
    eng.close()


def test_best_shot_tracker_with_motion_tracks_as_the_plain_one(shake):
    import torch
    frames, _ = shake
    dev, _ = _surfaces(frames[:16])
    eng = _engine("fp16")
    plain = eng.tracker(motion=True)
    best = eng.tracker(best={}, motion=True)
    crops = torch.empty((8, best.max_tracks, 112, 112, 3), dtype=torch.uint8, device="cuda")
    for s in range(0, 16, 8):
        chunk = dev[s:s + 8]
        tp, tc, _, _, _ = plain.detect_yuv_device(chunk, [0] * 8, THR, NMS)
        a = plain.read(tp, tc, 8)
        ma = plain.motion(8)
        _, _, tp2, tc2, _, _, _ = best.detect_yuv_best_device(chunk, [0] * 8, THR, NMS, crops.data_ptr())
        b = best.read(tp2, tc2, 8)
        mb = best.motion(8)
        assert ma.tobytes() == mb.tobytes()
        for i in range(8):
            assert a[i].tobytes() == b[i].tobytes(), (s, i)
    plain.close()
    best.close()
    eng.close()


def test_redaction_follows_the_camera(shake, golden_image):
    """One face blanked on two frames during a step: a motion tracker's LOST box covers its true box (IoU >= 0.5), a plain tracker's
    does not; every plane byte equals oracle/redact.py applied to the records and the compensated tracks."""
    import torch
    frames, mats = shake
    frames = [f.copy() for f in frames[:12]]
    eng = _engine("fp16")
    d, c, sc = eng.detect_yuv_device([torch.from_numpy(bgr_to_frame(frames[5], "nv12")).cuda()], THR, NMS)
    torch.cuda.synchronize()
    rec = eng.read_dets(d, c, 1)[0][0]
    j = int(np.argmax((rec[:, 3] - rec[:, 1]) * (rec[:, 0] > 0.8)))
    box5 = rec[j, 1:5] * sc[0]
    truth = {}
    for t in (6, 7):                                  # the face's true box on the blanked frames: frame 5's moved by the camera
        T = (np.r_[mats[t], [[0, 0, 1]]] @ np.linalg.inv(np.r_[mats[5], [[0, 0, 1]]]))[:2]
        p = T @ np.array([[box5[0], box5[2]], [box5[1], box5[3]], [1, 1]])
        truth[t] = (p[0, 0], p[1, 0], p[0, 1], p[1, 1])
        x1, y1, x2, y2 = (int(v) for v in truth[t])
        frames[t][y1 - 6:y2 + 6, x1 - 6:x2 + 6] = 128
    nv12 = [bgr_to_frame(f, "nv12") for f in frames]

    def iou(a, b):
        x1, y1, x2, y2 = max(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2]), min(a[3], b[3])
        inter = max(x2 - x1, 0) * max(y2 - y1, 0)
        return inter / ((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)

    best_iou = {}
    for motion in (False, True):
        trk = eng.tracker(motion=motion)
        dev = [torch.from_numpy(f).cuda() for f in nv12]
        torch.cuda.synchronize()
        ious = []
        b, m = params(0, 0.0)
        for s in range(0, 12, 4):
            chunk = dev[s:s + 4]
            tp, tc, dd, cc, scs = trk.detect_yuv_redact_device(chunk, [0] * 4, THR, NMS)
            recs = eng.read_dets(dd, cc, 4)[0]
            tr = trk.read(tp, tc, 4)
            for i in range(4):
                t = s + i
                want = redact_yuv(nv12[t], "nv12", frame_regions(recs[i], len(recs[i]), scs[i], m, b, tracks=tr[i]))
                if motion:
                    assert np.array_equal(chunk[i].cpu().numpy(), want), t
                if t in truth:
                    lost = [r for r in tr[i] if int(r["state"]) == LOST]
                    ious.append(max([iou((r["kx1"], r["ky1"], r["kx2"], r["ky2"]), truth[t]) for r in lost], default=0.0))
        best_iou[motion] = min(ious)
        trk.close()
    assert best_iou[True] >= 0.5 and best_iou[False] < 0.5, best_iou
    eng.close()


def test_interleaved_videos_calls_in_flight_and_reset(shake):
    frames, _ = shake
    dev, lumas = _surfaces(frames[:16])
    eng = _engine("fp16", streams=2)
    trk = eng.tracker(max_videos=2, motion=True)
    inter = [f for f in dev[:8] for _ in range(2)]                    # frame k of video 0, frame k of video 1, ...
    got = _run(eng, trk, inter, 8, videos=[0, 1] * 8)
    mo = MotionOracle(2)
    for k, g in enumerate(got):
        _same_motion(g[3], mo.update(k % 2, lumas[k // 2], g[1], len(g[1]), float(g[2])), f"interleaved {k}")
    trk.reset(1)
    tp, tc, d, c, sc = trk.detect_yuv_device([dev[8], dev[8]], [0, 1], THR, NMS)
    m = trk.motion(2)
    assert int(m[0]["status"]) == OK and int(m[1]["status"]) == FIRST
    trk.close()
    eng.close()


def test_refusals_launch_nothing(shake):
    from retinaface_b200.capi import RfError, motion_config
    frames, _ = shake
    dev, _ = _surfaces(frames[:2])
    eng = _engine("fp16")
    for bad in (dict(search=33), dict(search=-1), dict(min_inliers=2), dict(min_inliers=400)):
        trk = eng.tracker()
        with pytest.raises(RfError):
            trk.set_motion(**bad)
        trk.close()
    trk = eng.tracker(motion=True)
    with pytest.raises(RfError):
        trk.set_motion()                               # already on
    d, c, _ = eng.detect_yuv_device(dev[:1], THR, NMS)
    with pytest.raises(RfError):
        trk.update([0], d, c, [1.0])                   # no pixels
    with pytest.raises(RuntimeError):
        trk.motion(1)                                  # no frame call yet: nothing to read
    trk.detect_yuv_device(dev[:1], [0], THR, NMS)
    assert int(trk.motion(1)[0]["status"]) == FIRST
    trk.close()
    plain = eng.tracker()
    plain.detect_yuv_device(dev[:1], [0], THR, NMS)
    with pytest.raises(RfError):
        plain.set_motion()                             # after an update
    with pytest.raises(RfError):
        plain.motion(1)                                # motion is off
    cfg = motion_config()
    assert eng.lib.rf_tracker_set_motion(plain.t, C.byref(cfg)) == -1
    plain.close()
    eng.close()


def test_detector_track_frames_with_motion(shake):
    from retinaface_b200 import RetinaFace
    frames, _ = shake
    dev, _ = _surfaces(frames[:8])
    det = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_batch=8, max_image=(H, W))
    tracks, _ = det.trackFrames(dev, [0] * 8, motion=True)
    assert len(tracks) == 8 and det._tracker.motion_on
    assert int(det._tracker.motion(8)[1]["status"]) == OK
