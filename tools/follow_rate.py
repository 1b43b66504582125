#!/usr/bin/env python
"""Cost of f16 following on device-resident video: track_rate.py's eight 1920x1080 NV12 BT.601 videos (the golden photo resized to
1080p, video i rolled by 8 i columns and moved 7 px per frame), one frame of each per call, batch 8, a 448x448 mnet25 FP16 handle with
the default execution contexts, a follow tracker.  Call n detects (rf_detect_yuv_track_device) when n % k == 0 and follows
(rf_track_follow_device) otherwise.  Prints one JSON line with
  frames_per_s  per detect_every k in --every, tracking alone ("track k") and tracking + the default mosaic redaction of every
                call (rf_detect_yuv_redact_device / rf_track_follow_redact_device, "redact k"; both redact in place, so each
                redact call first copies the call's pristine frames into working frames -- 24 MB, in every redact rate alike):
                warmed up, --rounds alternated rounds of at least --min-seconds of back-to-back calls, the host clock ended by
                rf_synchronize;
  kernel_us     mean microseconds per launch of k_follow_cut, k_follow_search, k_follow_update and k_track_update at k = 3 in a
                separate torch.profiler run, and the kernels' sum per 8-frame follow call;
and the mean faces per frame and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/follow_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--every 1,2,3,5]
"""
import json
import os

import numpy as np

import rates
from rates import bench

B, FRAMES = 8, 16
KERNELS = ("k_follow_cut", "k_follow_search", "k_follow_update", "k_track_update")


def main():
    ap = rates.args(warmup=10)
    ap.add_argument("--every", default="1,2,3,5")
    args = ap.parse_args()
    every = [int(k) for k in args.every.split(",")]
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(1080, 1920))
    work = [f.clone() for f in frames[0]]
    modes = [(k, r) for r in (False, True) for k in every]
    trackers = {m: eng.tracker(max_videos=B, follow=True) for m in modes}
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = {m: 0 for m in modes}

    def call(mode):
        k, red = mode
        n = step[mode]
        step[mode] += 1
        f, trk = frames[n % FRAMES], trackers[mode]
        if red:
            for w, src in zip(work, f):
                w.copy_(src)
            f = work
        if n % k == 0:
            (trk.detect_yuv_redact_device if red else trk.detect_yuv_device)(f, vids, thr, nms)
        else:
            (trk.follow_redact_device if red else trk.follow_device)(f, vids)
    name = {m: f"{'redact' if m[1] else 'track'} {m[0]}" for m in modes}
    med, per_round, _ = rates.alternate({name[m]: lambda m=m: call(m) for m in modes}, args.rounds,
                                        lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    d, c, _ = eng.detect_yuv_device(frames[0], thr, nms)
    faces = float(np.mean([len(f) for f in eng.read_dets(d, c, B)[0]]))
    kp = (3 if 3 in every else every[-1], False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(60):
            call(kp)
        eng.synchronize()
    us, launches = rates.kernel_us(prof, KERNELS)
    us = {k: None if t is None else dict(mean_us=t, launches=launches[k]) for k, t in us.items()}
    follow_call_us = sum(us[n]["mean_us"] for n in ("k_follow_search", "k_follow_update") if us[n]) + \
        (us["k_follow_cut"]["mean_us"] if us["k_follow_cut"] else 0.0)
    med = {k: round(v, 1) for k, v in med.items()}
    speed = {name[m]: round(med[name[m]] / med[name[(every[0], m[1])]], 3) for m in modes}
    print(json.dumps(dict(frames_per_s=med, speedup=speed, rounds=per_round, kernel_us=us,
                          follow_kernels_us_per_call=follow_call_us, profiled_every=kp[0], faces_per_frame=faces, gpu=rates.card())))
    for t in trackers.values():
        t.close()
    eng.close()


if __name__ == "__main__":
    main()
