#!/usr/bin/env python
"""Cost of f21 oriented tiled detection on portrait 4K video: eight 3840x2160 NV12 BT.601 device frames (the golden photo resized to
4K, frame i rolled by 8 i columns) shown at orientation 6 through rf_detect_yuv_tiled_oriented_device, against the same frames
materialised as 2160x3840 portrait surfaces through rf_detect_yuv_tiled_device (the same tiles, records bit for bit), default
pyramid (84 tiles per frame), a 448x448 mnet25 FP16 handle with the default execution contexts.  Prints one JSON line with
  frames/s       of each: warmed up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock
                 ended by rf_synchronize; their medians and ratio;
  letterbox_us   microseconds per tile letter-box launch (k_letterbox_transposed for the stored frames, k_letterbox_batch for the
                 portrait surfaces), in a separate torch.profiler run of each, and their ratio;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/oriented_tiled_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402

W, H, B, O = 3840, 2160, 8, 6


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
    from retinaface_b200 import RF_PREC_FP16, Engine
    from test_oriented_cpu import orient_planes
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W, H))
    stored = [bgr_to_frame(np.roll(base, 8 * i, axis=1), "nv12") for i in range(B)]
    dev = [torch.from_numpy(f).cuda() for f in stored]
    portrait = [torch.from_numpy(orient_planes(f, "nv12", O)).cuda() for f in stored]
    torch.cuda.synchronize()
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(W, W))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    runs = {
        "oriented_stored": lambda: eng.detect_yuv_tiled_oriented_device(dev, [O] * B, thr, nms),
        "portrait_surfaces": lambda: eng.detect_yuv_tiled_device(portrait, thr, nms),
    }
    # the two calls compute the same records
    recs = {}
    for name, fn in runs.items():
        d, c = fn()
        eng.synchronize()
        recs[name] = [np.ascontiguousarray(a).tobytes() for part in eng.read_dets(d, c, B) for a in part]
    same = recs["oriented_stored"] == recs["portrait_surfaces"]
    got = {k: [] for k in runs}
    for _ in range(args.rounds):              # alternated: every round runs each variant once
        for name, fn in runs.items():
            got[name].append(rate(fn, eng.synchronize, args.min_seconds, args.warmup))
    lb = {}
    for name, fn in runs.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            eng.synchronize()
        t = [e.device_time for e in prof.events() if "k_letterbox" in e.name]
        kinds = sorted({re.search(r"k_letterbox_\w+", e.name).group(0) for e in prof.events() if "k_letterbox" in e.name})
        lb[name] = dict(us_per_launch=float(np.mean(t)) if t else None, launches=len(t), kernels=kinds)
    eng.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {name: dict(frames_per_s_median=float(np.median([r for r, _ in v])), frames_per_s=[round(r, 1) for r, _ in v],
                      calls=[k for _, k in v], letterbox=lb[name]) for name, v in got.items()}
    o, p = out["oriented_stored"], out["portrait_surfaces"]
    print(json.dumps(dict(frames=f"{B} x {W}x{H} NV12 BT.601 S-real, device, shown at {O}", model="mnet25 FP16 448x448, batch 8, default contexts",
                          gpu=gpu, records_equal=same, rate_ratio=o["frames_per_s_median"] / p["frames_per_s_median"],
                          letterbox_ratio=(o["letterbox"]["us_per_launch"] / p["letterbox"]["us_per_launch"]
                                           if o["letterbox"]["us_per_launch"] and p["letterbox"]["us_per_launch"] else None),
                          **out)))


if __name__ == "__main__":
    main()
