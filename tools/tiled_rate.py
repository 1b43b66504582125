#!/usr/bin/env python
"""Cost of f7 tiled detection: batches of 8 S-real 3840x2160 BGR images (the golden photo resized to 4K, element i rolled by 8 i
columns), the default pyramid (overlap 64), through rf_detect_tiled on
  - a 448x448 mnet25 FP16 handle with the default execution contexts,
  - the same with streams = 1 (one context, the latency plan),
  - a 1280x896 mnet25 FP16 handle.
Prints one JSON line with, per handle:
  tiled       blocking calls timed with the host clock after warm-up, enough calls for about 0.5 s: images/s and tiles/s;
  batch       the same images through rf_detect_batch (one letter-box each), and the cost ratio tiled / batch;
  kernels     in a separate torch.profiler run: microseconds per launch of the tile letter-box and of the merge kernel;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/tiled_rate.py [--min-seconds S] [--warmup W]
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


def timed(fn, min_s, warmup):
    for _ in range(warmup):
        fn()
    t = time.perf_counter()
    fn()
    one = time.perf_counter() - t
    k = max(3, int(np.ceil(min_s / max(one, 1e-6))))
    t = time.perf_counter()
    for _ in range(k):
        fn()
    return (time.perf_counter() - t) / k, k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W4K, H4K))
    imgs = [np.roll(base, 8 * i, axis=1) for i in range(B)]
    model = os.path.join(bench.GOLD, "weights", "mnet25.caffemodel")
    out = {}
    for name, (nw, nh, streams) in {"448x448": (448, 448, 0), "448x448_streams1": (448, 448, 1), "1280x896": (1280, 896, 0)}.items():
        eng = Engine(model, nh, nw, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(H4K, W4K), streams=streams)
        tiles = len(capi.tile_layout(nw, nh, W4K, H4K))
        s_tiled, k_tiled = timed(lambda: eng.detect_tiled(imgs, bench.SCORE_THR, bench.NMS_THR), args.min_seconds, args.warmup)
        s_batch, k_batch = timed(lambda: eng.detect_batch(imgs, bench.SCORE_THR, bench.NMS_THR), args.min_seconds, args.warmup)
        faces, _ = eng.detect_tiled(imgs, bench.SCORE_THR, bench.NMS_THR)
        plain = eng.detect_batch(imgs, bench.SCORE_THR, bench.NMS_THR)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                eng.detect_tiled(imgs, bench.SCORE_THR, bench.NMS_THR)
            eng.synchronize()
        lb = [e.device_time for e in prof.events() if "k_letterbox_batch" in e.name]
        mg = [e.device_time for e in prof.events() if "k_merge" in e.name]
        out[name] = dict(
            net=f"{nw}x{nh}", streams=streams, tiles_per_image=tiles,
            tiled=dict(calls=k_tiled, ms_per_call=s_tiled * 1e3, images_per_s=B / s_tiled, tiles_per_s=B * tiles / s_tiled,
                       faces_per_image=float(np.mean([len(f) for f in faces]))),
            batch=dict(calls=k_batch, ms_per_call=s_batch * 1e3, images_per_s=B / s_batch,
                       faces_per_image=float(np.mean([len(f) for f in plain]))),
            cost_ratio_tiled_over_batch=s_tiled / s_batch,
            kernels=dict(tile_letterbox_us_per_launch=float(np.mean(lb)) if lb else None, letterbox_launches=len(lb),
                         merge_us_per_launch=float(np.mean(mg)) if mg else None, merge_launches=len(mg)))
        eng.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps(dict(images=f"{B} x {W4K}x{H4K} S-real BGR, pageable", pyramid="default, overlap 64", model="mnet25 FP16", gpu=gpu,
                          **out)))


if __name__ == "__main__":
    main()
