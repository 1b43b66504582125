#!/usr/bin/env python
"""Cost of f13 camera-motion compensation: track_rate.py's eight 1920x1080 NV12 BT.601 device videos (the golden photo resized to
1080p, video i rolled by 8 i columns), with the camera shaking -- each frame the photo's window moves by a seeded step of 40-70 px
with changing signs -- one frame of each per call, batch 8, a 448x448 mnet25 FP16 handle with the default execution contexts.  Prints
one JSON line with
  frames/s    of rf_detect_yuv_track_device on a plain tracker (detect+track) and on a motion tracker (detect+track+motion): warmed
              up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended by
              rf_synchronize;
  kernel_us   microseconds per launch of k_motion_thumb, k_motion_match, k_motion_fit and k_motion_commit (and k_track_update) in a
              separate torch.profiler run, and their sum per 8-frame call;
and the card's name and power limit, read in the same command.

    python tools/motion_rate.py [--min-seconds S] [--warmup W] [--rounds R]
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
KERNELS = ("k_motion_thumb", "k_motion_match", "k_motion_fit", "k_motion_commit", "k_track_update")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    pad = 200
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W + 2 * pad, H + 2 * pad))
    rng = np.random.default_rng(3)
    x, sign, frames = pad, 1, []
    for t in range(FRAMES):
        step = int(rng.integers(40, 71))
        if not 0 <= x + sign * step <= 2 * pad:
            sign = -sign
        x += sign * step
        sign = -sign if rng.uniform() < 0.5 else sign
        img = np.ascontiguousarray(base[pad:pad + H, x:x + W])
        frames.append([torch.from_numpy(bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12")).cuda() for i in range(B)])
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H, W))
    plain = eng.tracker(max_videos=B)
    moving = eng.tracker(max_videos=B, motion=True)
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]
    runs = {
        "detect+track": lambda: plain.detect_yuv_device(nxt(), vids, thr, nms),
        "detect+track+motion": lambda: moving.detect_yuv_device(nxt(), vids, thr, nms),
    }
    for fn in runs.values():
        for _ in range(args.warmup):
            fn()
    eng.synchronize()
    rates = {k: [] for k in runs}
    for _ in range(args.rounds):
        for k, fn in runs.items():
            n, t0 = 0, time.perf_counter()
            while True:
                fn()
                n += 1
                if time.perf_counter() - t0 >= args.min_seconds:
                    break
            eng.synchronize()
            rates[k].append(B * n / (time.perf_counter() - t0))
    calls = 50
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            runs["detect+track+motion"]()
        eng.synchronize()
    us, launches = {}, {}
    for k in KERNELS:
        ev = [e for e in prof.events() if k in e.name]
        launches[k] = len(ev)
        us[k] = sum(e.device_time for e in ev) / max(len(ev), 1) if ev else None
    per_call = sum(us[k] * launches[k] for k in KERNELS[:4] if us[k]) / calls
    status = moving.motion(B)["status"].tolist()
    med = {k: round(float(np.median(v)), 1) for k, v in rates.items()}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(frames_per_s=med, rounds=rates, motion_cost=round(1 - med["detect+track+motion"] / med["detect+track"], 4),
                          kernel_us=us, launches=launches, motion_us_per_call=per_call, last_status=status, gpu=smi.stdout.strip())))
    plain.close()
    moving.close()
    eng.close()


if __name__ == "__main__":
    main()
