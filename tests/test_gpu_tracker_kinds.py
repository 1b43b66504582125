"""GPU (-m gpu): which calls each kind of tracker takes.  A tracker is plain, best-shot (f11), follow (f16) or look-back (f15); camera
motion (f13) is an option of any kind and the look-back search (f17) one of a look-back tracker.  Every frame entry point, finish,
drain, each setter and each query of the latest call's records is called on every kind, before and after its first frame call, and
returns the status (and, refused, the message) of the table below.  A refused call leaves the tracker's state and the frames untouched."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_redact import _engine

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
FW, FH = 320, 240
L = 2
MAX_TRACKS = 8
OK, INVALID = 0, -1

KINDS = {
    "plain": {}, "plain+motion": dict(motion=True),
    "best": dict(best={}), "best+motion": dict(best={}, motion=True),
    "follow": dict(follow=True), "follow+motion": dict(follow=True, motion=True),
    "lookback": dict(lookback=L), "lookback+motion": dict(lookback=L, motion=True),
    "lookback+search": dict(lookback=L, lookback_search=True),
}

ONLY_BEST = "a best-shot tracker takes frames only through rf_detect_yuv_track_best_device"
ONLY_LOOKBACK = "a look-back tracker takes frames only through rf_detect_yuv_redact_lookback_device"
UPDATED = "the tracker has already been updated"


def _why(call, kind, motion, search, updated):
    """The admission table: None (taken) or the refusal's reason."""
    frames_only = {"best": ONLY_BEST, "lookback": ONLY_LOOKBACK}
    name = {"best": "best-shot", "follow": "follow", "lookback": "look-back"}
    if call == "update":
        if kind == "best":
            return ONLY_BEST
        if motion:
            return "a motion tracker needs the frames (rf_detect_yuv_track_device)"
        if kind == "follow":
            return "a follow tracker needs the frames (rf_detect_yuv_track_device)"
        return frames_only.get(kind)
    if call in ("detect", "detect_redact"):
        return frames_only.get(kind)
    if call in ("best", "finish"):
        return None if kind == "best" else "not a best-shot tracker (rf_tracker_create_best)"
    if call in ("follow", "follow_redact", "q_follow"):
        return None if kind == "follow" else "not a follow tracker (rf_tracker_set_follow)"
    if call in ("lookback", "drain"):
        return None if kind == "lookback" else "not a look-back tracker (rf_tracker_set_lookback)"
    if call == "q_motion":
        return None if motion else "motion is off (rf_tracker_set_motion)"
    if call == "q_search":
        return None if search else "not a searching look-back tracker (rf_tracker_set_lookback_search)"
    if call == "set_motion":
        why = "motion is already on" if motion else None
    elif call == "set_follow":
        why = None if kind == "plain" else "following is already on" if kind == "follow" else f"a {name[kind]} tracker cannot follow"
    elif call == "set_lookback":
        why = None if kind == "plain" else "look-back is already on" if kind == "lookback" else f"a {name[kind]} tracker cannot look back"
    else:
        assert call == "set_lookback_search"
        why = "not a look-back tracker (rf_tracker_set_lookback)" if kind != "lookback" else "the look-back search is already on" if search else None
    return why or (UPDATED if updated else None)


WHO = {
    "update": "rf_track_update", "detect": "rf_detect_yuv_track_device", "detect_redact": "rf_detect_yuv_redact_device_style",
    "best": "rf_detect_yuv_track_best_device", "finish": "rf_tracker_finish", "follow": "rf_track_follow_device",
    "follow_redact": "rf_track_follow_redact_device", "lookback": "rf_detect_yuv_redact_lookback_device", "drain": "rf_tracker_drain",
    "set_motion": "rf_tracker_set_motion", "set_follow": "rf_tracker_set_follow", "set_lookback": "rf_tracker_set_lookback",
    "set_lookback_search": "rf_tracker_set_lookback_search", "q_motion": "rf_tracker_motion", "q_follow": "rf_tracker_follow",
    "q_search": "rf_tracker_lookback_search",
}


class _Rig:
    """One engine, an NV12 input frame and an out frame (both canaries), and every call's arguments, valid but for the tracker."""

    def __init__(self):
        import torch
        from retinaface_b200 import capi
        self.capi = capi
        self.eng = _engine("fp16", max_batch=2)
        self.lib = self.eng.lib
        g = np.add.outer(np.arange(FH + FH // 2), 3 * np.arange(FW)).astype(np.uint8)
        self.inp = torch.from_numpy(g).cuda()
        self.out = torch.full((FH + FH // 2, FW), 0x5A, dtype=torch.uint8, device="cuda")
        self.frames = self.eng._frames([(self.inp[:FH], self.inp[FH:])], "nv12", True)
        self.outs = self.eng._frames([(self.out[:FH], self.out[FH:])], "nv12", True)
        self.dets = torch.zeros(self.eng.max_faces * 256, dtype=torch.uint8, device="cuda")
        self.counts = torch.zeros(2, dtype=torch.int32, device="cuda")
        self.crops = torch.zeros(MAX_TRACKS * 112 * 112 * 3 * 4 * 2, dtype=torch.uint8, device="cuda")
        self.style = capi.RedactStyle(0, 0, 0, 0, 0.0)
        self.nums = np.zeros(4, np.int32)
        torch.cuda.synchronize()

    def tracker(self, kind):
        return self.eng.tracker(max_tracks=MAX_TRACKS, **KINDS[kind])

    def call(self, name, t):
        lib, h, capi = self.lib, self.eng.h, self.capi
        vids = (C.c_int * 1)(0)
        p, q, r, s = (C.c_void_p() for _ in range(4))
        sc = np.zeros(1, np.float32)
        if name == "update":
            return lib.rf_track_update(t, vids, 1, self.dets.data_ptr(), self.counts.data_ptr(), None, C.byref(p), C.byref(q))
        if name == "detect":
            return lib.rf_detect_yuv_track_device(h, t, self.frames, vids, 1, 0, THR, NMS, None, None, None, C.byref(p), C.byref(q),
                                                  C.byref(r), C.byref(s), sc.ctypes.data)
        if name == "detect_redact":
            return lib.rf_detect_yuv_redact_device_style(h, t, self.frames, vids, 1, 0, THR, NMS, C.byref(self.style), C.byref(p), C.byref(q),
                                                         C.byref(r), C.byref(s), sc.ctypes.data)
        if name == "best":
            a, b = C.c_void_p(), C.c_void_p()
            return lib.rf_detect_yuv_track_best_device(h, t, self.frames, vids, 1, 0, THR, NMS, self.crops.data_ptr(), None, C.byref(a), C.byref(b),
                                                       C.byref(p), C.byref(q), C.byref(r), C.byref(s), sc.ctypes.data)
        if name == "finish":
            return lib.rf_tracker_finish(t, 0, self.crops.data_ptr(), None, C.byref(p), C.byref(q))
        if name == "follow":
            return lib.rf_track_follow_device(t, self.frames, vids, 1, C.byref(p), C.byref(q))
        if name == "follow_redact":
            return lib.rf_track_follow_redact_device(t, self.frames, vids, 1, C.byref(self.style), C.byref(p), C.byref(q))
        if name == "lookback":
            return lib.rf_detect_yuv_redact_lookback_device(h, t, self.frames, vids, 1, 0, THR, NMS, C.byref(self.style), self.outs,
                                                            self.nums.ctypes.data, C.byref(p), C.byref(q), C.byref(r), C.byref(s), sc.ctypes.data)
        if name == "drain":
            n_out = C.c_int(0)
            return lib.rf_tracker_drain(t, 0, C.byref(self.style), self.outs, L, C.byref(n_out), self.nums.ctypes.data)
        if name == "set_motion":
            return lib.rf_tracker_set_motion(t, C.byref(capi.MotionConfig(0, 0)))
        if name == "set_follow":
            return lib.rf_tracker_set_follow(t, C.byref(capi.FollowConfig(0, 0.0)))
        if name == "set_lookback":
            return lib.rf_tracker_set_lookback(t, C.byref(capi.LookbackConfig(L, 0.0)))
        if name == "set_lookback_search":
            return lib.rf_tracker_set_lookback_search(t, C.byref(capi.FollowConfig(0, 0.0)))
        if name == "q_motion":
            return lib.rf_tracker_motion(t, C.byref(p))
        if name == "q_follow":
            return lib.rf_tracker_follow(t, C.byref(p))
        assert name == "q_search"
        return lib.rf_tracker_lookback_search(t, C.byref(p), C.byref(q))

    def first_call(self, kind):
        return {"best": "best", "lookback": "lookback"}.get(kind.split("+")[0], "detect")


@pytest.fixture(scope="module")
def rig():
    r = _Rig()
    yield r
    r.eng.close()


def _snapshot(rig, trk):
    rig.eng.synchronize()
    head, rows = trk.debug_state(0)
    return head, rows, rig.inp.cpu(), rig.out.cpu()


@pytest.mark.parametrize("updated", [False, True], ids=["fresh", "updated"])
@pytest.mark.parametrize("kind", list(KINDS))
def test_admission_table(rig, kind, updated):
    import torch
    base = kind.split("+")[0]
    motion, search = "motion" in kind, "search" in kind
    for call in WHO:
        trk = rig.tracker(kind)
        if updated:
            assert rig.call(rig.first_call(kind), trk.t) == OK, (kind, call)
        before = _snapshot(rig, trk)
        why = _why(call, base, motion, search, updated)
        rc = rig.call(call, trk.t)
        if why is None:
            assert rc == OK, (kind, updated, call, rig.lib.rf_last_error(rig.eng.h))
        else:
            assert rc == INVALID, (kind, updated, call, rc)
            assert rig.lib.rf_last_error(rig.eng.h).decode() == f"{WHO[call]}: {why}", (kind, updated, call)
            after = _snapshot(rig, trk)
            assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1]), (kind, updated, call)
            assert torch.equal(before[2], after[2]) and torch.equal(before[3], after[3]), (kind, updated, call)
        trk.close()
