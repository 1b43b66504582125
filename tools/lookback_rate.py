#!/usr/bin/env python
"""Cost of f15 look-back redaction on device-resident video: redact_rate.py's eight 1920x1080 NV12 BT.601 videos, one frame of each
per call, batch 8, a 448x448 mnet25 FP16 handle.  Prints one JSON line with
  frames/s    track+redact (rf_detect_yuv_track_device, then rf_redact_yuv_device_style of its records and tracks into a second set of
              surfaces: what rf_detect_yuv_redact_device_style launches, without writing the frames the detector reads again) against
              lookback (rf_detect_yuv_redact_lookback_device at L = --frames into separate out surfaces), both mosaic + rect: warmed
              up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended by
              rf_synchronize;
  kernel_us   microseconds per launch of k_lookback_log, k_lookback_swap and k_lookback_boxes in a separate torch.profiler run, and
              k_lookback_swap's effective bandwidth: 4 x w h 3 / 2 bytes per frame (buffer and input read, out and buffer written);
and the card's name and power limit, read in the same command.

    python tools/lookback_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--frames L]
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
KERNELS = ("k_lookback_log", "k_lookback_swap", "k_lookback_boxes")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=15)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    photo = cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg"))
    base = cv2.resize(photo, (W - 7 * FRAMES, H))
    frames = []
    for t in range(FRAMES):
        img = np.full((H, W, 3), 128, np.uint8)
        img[:, 7 * t:7 * t + base.shape[1]] = base
        frames.append([torch.from_numpy(bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12")).cuda() for i in range(B)])
    out = [f.clone() for f in frames[0]]
    torch.cuda.synchronize()
    weights = os.path.join(bench.GOLD, "weights", "mnet25.caffemodel")
    eng = Engine(weights, 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(H, W))
    trk = eng.tracker(max_videos=B)
    lbt = eng.tracker(max_videos=B, lookback=dict(frames=args.frames))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]

    def track_redact():
        tp, tc, d, c, sc = trk.detect_yuv_device(nxt(), vids, thr, nms)
        eng.redact_yuv_device(out, d, c, sc, tracker=trk, tracks_ptr=tp, track_counts_ptr=tc)

    def lookback():
        lbt.detect_yuv_redact_lookback_device(nxt(), vids, out, thr, nms)

    runs = {"track+redact": track_redact, "lookback": lookback}
    for fn in runs.values():
        for _ in range(max(args.warmup, args.frames + 2)):
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
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            lookback()
        eng.synchronize()
    kernel_us = {}
    for k in KERNELS:
        ks = [ev for ev in prof.events() if k in ev.name]
        kernel_us[k] = sum(ev.device_time for ev in ks) / len(ks) if ks else None
    swap_bytes = B * 4 * W * H * 3 // 2
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    med = {k: round(float(np.median(v)), 1) for k, v in rates.items()}
    print(json.dumps(dict(frames_per_s=med, rounds=rates, lookback_share=round(med["lookback"] / med["track+redact"], 4), L=args.frames,
                          kernel_us=kernel_us, log_plus_boxes_us=(kernel_us["k_lookback_log"] or 0) + (kernel_us["k_lookback_boxes"] or 0),
                          swap_bytes_per_call=swap_bytes,
                          swap_tb_per_s=swap_bytes / (kernel_us["k_lookback_swap"] * 1e-6) / 1e12 if kernel_us["k_lookback_swap"] else None,
                          swap_floor_us=swap_bytes / 3.35e12 * 1e6, gpu=smi.stdout.strip())))
    trk.close()
    lbt.close()
    eng.close()


if __name__ == "__main__":
    main()
