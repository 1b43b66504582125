#!/usr/bin/env python
"""Cost of f11 best shots on device-resident video: tools/track_rate.py's workload (eight 1920x1080 NV12 BT.601 videos on the device,
the golden photo resized to 1080p, video i rolled by 8 i columns and moved 7 px per frame; one frame of each per call, batch 8, a
448x448 mnet25 FP16 handle with the default execution contexts).  Prints one JSON line with
  frames/s    of rf_detect_yuv_batch_device (detect), rf_detect_yuv_track_device (detect + track), the same with 112x112 crops of the
              new identities (detect + track + crops) and rf_detect_yuv_track_best_device with 112x112 u8 best shots (detect + track
              + best): warmed up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended
              by rf_synchronize;
  kernel_us   microseconds per launch of k_track_update and of each k_best_* kernel, in a separate torch.profiler run (CUPTI's
              device timestamps), and the mean faces per frame;
and the card's name and power limit, read in the same command.  The videos loop over 16 frames, so tracks live on and the best-shot
store is exercised on every frame; best_cost is 1 - (detect + track + best) / (detect + track).

    python tools/bestshot_rate.py [--min-seconds S] [--warmup W] [--rounds R]
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
    best = eng.tracker(max_videos=B, best=dict())
    crops = torch.empty((B, 8, 112, 112, 3), dtype=torch.uint8, device="cuda")
    shots = torch.empty((B, best.max_tracks, 112, 112, 3), dtype=torch.uint8, device="cuda")
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
        "detect+track+best": lambda: best.detect_yuv_best_device(nxt(), vids, thr, nms, shots.data_ptr()),
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
            runs["detect+track+best"]()
        eng.synchronize()
    kernel_us, launches = {}, {}
    for name in ("k_track_update", "k_best_measure", "k_best_select", "k_best_emit", "k_best_commit"):
        ks = [e for e in prof.events() if name in e.name]
        kernel_us[name] = round(sum(e.device_time for e in ks) / len(ks), 2) if ks else None
        launches[name] = len(ks)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    med = {k: round(float(np.median(v)), 1) for k, v in rates.items()}
    print(json.dumps(dict(frames_per_s=med, rounds=rates, best_cost=round(1 - med["detect+track+best"] / med["detect+track"], 4),
                          kernel_us=kernel_us, launches=launches, faces_per_frame=faces, gpu=smi.stdout.strip())))
    best.close()
    trk.close()
    eng.close()


if __name__ == "__main__":
    main()
