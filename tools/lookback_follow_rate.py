#!/usr/bin/env python
"""Cost of f18 following look-back redaction on device-resident video: lookback_rate.py's eight 1920x1080 NV12 BT.601 videos, one
frame of each per call, batch 8, a 448x448 mnet25 FP16 handle, mosaic + rect, L = --frames.  Call n of a following look-back tracker
detects (rf_detect_yuv_redact_lookback_device) when n % k == 0 and follows (rf_track_follow_redact_lookback_device) otherwise, both
into separate out surfaces.  Prints one JSON line with
  frames_per_s  per k in --every: "lbfollow k" (the following look-back tracker), "f16 k" (a follow tracker's undelayed
                rf_detect_yuv_redact_device / rf_track_follow_redact_device; they redact in place, so each call first copies the call's
                pristine frames into working frames, 24 MB, as follow_rate.py does), and "lookback" (a plain look-back tracker, every
                frame detected): warmed up, --rounds alternated rounds of at least --min-seconds of back-to-back calls, the host clock
                ended by rf_synchronize;  speedup: "lbfollow k" over "lookback";
  kernel_us     mean microseconds per launch, on follow calls and on detect calls apart, of k_lookback_log, k_lookback_swap,
                k_lookback_boxes and the redaction kernels, and of f16's k_follow_search / k_follow_update / k_follow_cut, at k = 3 in a
                separate torch.profiler run (one k_lookback_log launch per call: the j-th is call j's);
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/lookback_follow_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--frames L] [--every 1,3,5]
"""
import json
import os

import numpy as np

import rates
from rates import bench

B, FRAMES = 8, 16
KERNELS = ("k_lookback_log", "k_lookback_swap", "k_lookback_boxes", "k_redact", "k_follow_search", "k_follow_update", "k_follow_cut",
           "k_track_update")


def main():
    ap = rates.args(warmup=20)
    ap.add_argument("--frames", type=int, default=15)
    ap.add_argument("--every", default="1,3,5")
    args = ap.parse_args()
    every = [int(k) for k in args.every.split(",")]
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    out = [f.clone() for f in frames[0]]
    work = [f.clone() for f in frames[0]]
    torch.cuda.synchronize()
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(1080, 1920))
    L = args.frames
    modes = [("lookback", 1)] + [(kind, k) for k in every for kind in ("lbfollow", "f16")]
    trackers = {}
    for m in modes:
        kind = m[0]
        trackers[m] = eng.tracker(max_videos=B, lookback=dict(frames=L) if kind != "f16" else None, lookback_follow=kind == "lbfollow" or None,
                                  follow=kind == "f16" or None)
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = {m: 0 for m in modes}

    def call(mode):
        kind, k = mode
        n = step[mode]
        step[mode] += 1
        f, trk = frames[n % FRAMES], trackers[mode]
        if kind == "f16":
            for w, src in zip(work, f):
                w.copy_(src)
            if n % k == 0:
                trk.detect_yuv_redact_device(work, vids, thr, nms)
            else:
                trk.follow_redact_device(work, vids)
        elif n % k == 0:
            trk.detect_yuv_redact_lookback_device(f, vids, out, thr, nms)
        else:
            trk.follow_redact_lookback_device(f, vids, out)
    label = {m: m[0] if m[0] == "lookback" else f"{m[0]} {m[1]}" for m in modes}
    warmup = max(args.warmup, L + 2)
    med, per_round, _ = rates.alternate({label[m]: lambda m=m: call(m) for m in modes}, args.rounds,
                                        lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, warmup, B))
    kp = ("lbfollow", 3 if 3 in every else every[-1])
    step[kp] += -step[kp] % kp[1]          # the profiled run starts on a detect call
    ncalls = 20 * kp[1]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ncalls):
            call(kp)
        eng.synchronize()
    evs = sorted((e for e in prof.events() if e.device_time > 0), key=lambda e: e.time_range.start)
    logs = [e for e in evs if "k_lookback_log" in e.name]
    assert len(logs) == ncalls, (len(logs), ncalls)
    # each kernel launch belongs to the call whose k_lookback_log precedes it, or, before it in that call, follows the previous one
    starts = [e.time_range.start for e in logs]
    kernel_us = {}
    for name in KERNELS:
        per = {"follow": [], "detect": []}
        for e in evs:
            if name not in e.name:
                continue
            j = int(np.searchsorted(starts, e.time_range.start, side="right")) - 1
            if name in ("k_follow_search", "k_follow_update", "k_follow_cut", "k_track_update"):
                j += 1                     # the tracking runs before the call's log
            j = min(max(j, 0), ncalls - 1)
            per["detect" if j % kp[1] == 0 else "follow"].append(e.device_time)
        kernel_us[name] = {c: dict(mean_us=round(float(np.mean(v)), 2), launches=len(v)) for c, v in per.items() if v}
    med = {k: round(v, 1) for k, v in med.items()}
    speed = {label[m]: round(med[label[m]] / med["lookback"], 3) for m in modes if m[0] == "lbfollow"}
    print(json.dumps(dict(frames_per_s=med, speedup_over_lookback=speed, rounds=per_round, L=L,
                          profiled_every=kp[1], kernel_us=kernel_us, gpu=rates.card())))
    for t in trackers.values():
        t.close()
    eng.close()


if __name__ == "__main__":
    main()
