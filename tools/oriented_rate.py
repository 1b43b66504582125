#!/usr/bin/env python
"""Cost of f9 orientations on device-resident video frames: eight S-real 1920x1080 NV12 BT.601 frames on the device (the golden photo
resized to 1080p, frame i rolled by 8 i columns), batch 8, a 448x448 mnet25 FP16 handle with the default execution contexts.  Prints
one JSON line with
  frames/s      of rf_detect_yuv_batch_device (orientation 1) and of rf_detect_yuv_oriented_device at orientations 3 and 6: warmed up,
                --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended by rf_synchronize;
  letterbox_us  microseconds per letter-box launch (k_letterbox_batch, or k_letterbox_transposed for orientation 6), in a separate
                torch.profiler run of each variant;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/oriented_rate.py [--min-seconds S] [--warmup W] [--rounds R]
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

W, H, B = 1920, 1080, 8


def rate(fn, sync, min_s, warmup):
    """Frames per second of fn() (one call = B frames), host clock over >= min_s of calls ended by sync()."""
    for _ in range(warmup):
        fn()
    sync()
    k, t0 = 0, time.perf_counter()
    while True:
        fn()
        k += 1
        if time.perf_counter() - t0 >= min_s:
            break
    sync()
    return B * k / (time.perf_counter() - t0), k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W, H))
    dev = [torch.from_numpy(bgr_to_frame(np.roll(base, 8 * i, axis=1), "nv12")).cuda() for i in range(B)]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H, W))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    runs = {
        "o1_yuv_batch_device": lambda: eng.detect_yuv_device(dev, thr, nms),
        "o3_oriented_device": lambda: eng.detect_yuv_oriented_device(dev, [3] * B, thr, nms),
        "o6_oriented_device": lambda: eng.detect_yuv_oriented_device(dev, [6] * B, thr, nms),
    }
    got = {k: [] for k in runs}
    for _ in range(args.rounds):              # alternated: every round runs each variant once
        for name, fn in runs.items():
            got[name].append(rate(fn, eng.synchronize, args.min_seconds, args.warmup))
    lb = {}
    for name, fn in runs.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                fn()
            eng.synchronize()
        t = [e.device_time for e in prof.events() if "k_letterbox" in e.name]
        lb[name] = dict(us_per_launch=float(np.mean(t)) if t else None, launches=len(t))
    eng.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {name: dict(frames_per_s_median=float(np.median([r for r, _ in v])), frames_per_s=[round(r, 1) for r, _ in v],
                      calls=[k for _, k in v], letterbox=lb[name]) for name, v in got.items()}
    print(json.dumps(dict(frames=f"{B} x {W}x{H} NV12 BT.601 S-real, device", model="mnet25 FP16 448x448, batch 8, default contexts",
                          gpu=gpu, **out)))


if __name__ == "__main__":
    main()
