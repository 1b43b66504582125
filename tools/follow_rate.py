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
and the mean faces per frame and the card's name and power limit, read in the same command.

    python tools/follow_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--every 1,2,3,5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

W, H, B, FRAMES = 1920, 1080, 8, 16
KERNELS = ("k_follow_cut", "k_follow_search", "k_follow_update", "k_track_update")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--every", default="1,2,3,5")
    args = ap.parse_args()
    every = [int(k) for k in args.every.split(",")]
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W - 7 * FRAMES, H))
    frames = []
    for t in range(FRAMES):
        img = np.full((H, W, 3), 128, np.uint8)
        img[:, 7 * t:7 * t + base.shape[1]] = base
        frames.append([torch.from_numpy(bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12")).cuda() for i in range(B)])
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H, W))
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
    for k in modes:
        for _ in range(args.warmup):
            call(k)
    eng.synchronize()
    rates = {k: [] for k in modes}
    for _ in range(args.rounds):
        for k in modes:
            n, t0 = 0, time.perf_counter()
            while True:
                call(k)
                n += 1
                if time.perf_counter() - t0 >= args.min_seconds:
                    break
            eng.synchronize()
            rates[k].append(B * n / (time.perf_counter() - t0))
    d, c, _ = eng.detect_yuv_device(frames[0], thr, nms)
    faces = float(np.mean([len(f) for f in eng.read_dets(d, c, B)[0]]))
    kp = (3 if 3 in every else every[-1], False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(60):
            call(kp)
        eng.synchronize()
    us = {}
    for name in KERNELS:
        ks = [e for e in prof.events() if name in e.name]
        us[name] = dict(mean_us=sum(e.device_time for e in ks) / len(ks), launches=len(ks)) if ks else None
    follow_call_us = sum(us[n]["mean_us"] for n in ("k_follow_search", "k_follow_update") if us[n]) + \
        (us["k_follow_cut"]["mean_us"] if us["k_follow_cut"] else 0.0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name = {m: f"{'redact' if m[1] else 'track'} {m[0]}" for m in modes}
    med = {name[m]: round(float(np.median(v)), 1) for m, v in rates.items()}
    speed = {name[m]: round(med[name[m]] / med[name[(every[0], m[1])]], 3) for m in modes}
    print(json.dumps(dict(frames_per_s=med, speedup=speed, rounds={name[m]: v for m, v in rates.items()}, kernel_us=us,
                          follow_kernels_us_per_call=follow_call_us, profiled_every=kp[0], faces_per_frame=faces, gpu=smi.stdout.strip())))
    for t in trackers.values():
        t.close()
    eng.close()


if __name__ == "__main__":
    main()
