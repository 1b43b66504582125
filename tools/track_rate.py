#!/usr/bin/env python
"""Cost of f10 tracking on device-resident video: eight 1920x1080 NV12 BT.601 videos on the device (the golden photo resized to 1080p,
video i rolled by 8 i columns and moved 7 px per frame), one frame of each per call, batch 8, a 448x448 mnet25 FP16 handle with the
default execution contexts.  Prints one JSON line with
  frames/s    of rf_detect_yuv_batch_device (detect), rf_detect_yuv_track_device (detect + track) and rf_detect_yuv_track_device with
              112x112 crops of the new identities (detect + track + crops): warmed up, --rounds alternated rounds of at least
              --min-seconds of back-to-back calls each, the host clock ended by rf_synchronize;
  track_us    microseconds per k_track_update launch, in a separate torch.profiler run, and the mean faces per frame;
and the card's name and power limit, read in the same command.

    python tools/track_rate.py [--min-seconds S] [--warmup W] [--rounds R]
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
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W - 7 * FRAMES, H))
    frames = []
    for t in range(FRAMES):
        img = np.full((H, W, 3), 128, np.uint8)
        img[:, 7 * t:7 * t + base.shape[1]] = base
        frames.append([torch.from_numpy(bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12")).cuda() for i in range(B)])
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H, W))
    trk = eng.tracker(max_videos=B)
    crops = torch.empty((B, 8, 112, 112, 3), dtype=torch.uint8, device="cuda")
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]
    runs = {
        "detect": lambda: eng.detect_yuv_device(nxt(), thr, nms),
        "detect+track": lambda: trk.detect_yuv_device(nxt(), vids, thr, nms),
        "detect+track+crops": lambda: trk.detect_yuv_device(nxt(), vids, thr, nms, align=dict(max_faces=8), dev_crops_ptr=crops.data_ptr()),
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
    d, c, _ = eng.detect_yuv_device(frames[0], thr, nms)
    faces = float(np.mean([len(f) for f in eng.read_dets(d, c, B)[0]]))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            runs["detect+track"]()
        eng.synchronize()
    ks = [e for e in prof.events() if "k_track_update" in e.name]
    track_us = sum(e.device_time for e in ks) / max(len(ks), 1) if ks else None
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps(dict(frames_per_s={k: round(float(np.median(v)), 1) for k, v in rates.items()}, rounds=rates, track_us=track_us,
                          track_launches=len(ks), faces_per_frame=faces, gpu=smi.stdout.strip())))
    trk.close()
    eng.close()


if __name__ == "__main__":
    main()
