#!/usr/bin/env python
"""Cost of f8 tiled detection on device-resident video frames: eight S-real 3840x2160 NV12 BT.601 frames on the device (the golden
photo resized to 4K, frame i rolled by 8 i columns), the default pyramid (overlap 64), a 448x448 mnet25 FP16 handle with the default
execution contexts.  Prints one JSON line with
  device        frames/s of rf_detect_yuv_tiled_device, without crops and with 112x112 F16 crops: warmed up, at least --min-seconds
                of back-to-back calls, the host clock ended by rf_synchronize;
  host_pinned   frames/s of the blocking rf_detect_yuv_tiled on the same frames in pinned host memory, its runs alternated with the
                device runs;
  align_kernel  microseconds per launch of k_align_faces, in a separate torch.profiler run of the device calls with crops;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/tiled_device_rate.py [--min-seconds S] [--warmup W] [--rounds R]
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

W4K, H4K, B = 3840, 2160, 8


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
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W4K, H4K))
    frames = [bgr_to_frame(np.roll(base, 8 * i, axis=1), "nv12") for i in range(B)]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    pinned = [torch.from_numpy(f).pin_memory().numpy() for f in frames]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H4K, W4K))
    crops = torch.empty((B, eng.max_faces, 3, 112, 112), dtype=torch.float16, device="cuda")
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    runs = {
        "device": lambda: eng.detect_yuv_tiled_device(dev, thr, nms),
        "device_crops_f16": lambda: eng.detect_yuv_tiled_device(dev, thr, nms, align=dict(fmt="rgb_f16"), dev_crops_ptr=crops.data_ptr()),
        "host_pinned": lambda: eng.detect_yuv_tiled(pinned, thr, nms),
    }
    got = {k: [] for k in runs}
    for _ in range(args.rounds):              # alternated: every round runs each variant once
        for name, fn in runs.items():
            got[name].append(rate(fn, eng.synchronize, args.min_seconds, args.warmup))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            runs["device_crops_f16"]()
        eng.synchronize()
    al = [e.device_time for e in prof.events() if "k_align_faces" in e.name]
    faces, _ = eng.detect_yuv_tiled(pinned, thr, nms)
    eng.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {name: dict(frames_per_s_median=float(np.median([r for r, _ in v])), frames_per_s=[round(r, 1) for r, _ in v],
                      calls=[k for _, k in v]) for name, v in got.items()}
    print(json.dumps(dict(frames=f"{B} x {W4K}x{H4K} NV12 BT.601 S-real", pyramid="default, overlap 64",
                          tiles_per_frame=len(capi.tile_layout(448, 448, W4K, H4K)), model="mnet25 FP16 448x448, default contexts",
                          faces_per_frame=float(np.mean([len(f) for f in faces])), gpu=gpu, **out,
                          align_kernel=dict(us_per_launch=float(np.mean(al)) if al else None, launches=len(al)))))


if __name__ == "__main__":
    main()
