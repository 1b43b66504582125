#!/usr/bin/env python
"""Cost of f23 rotated views: one S-real 1920x1080 BGR host image (the golden photo resized), a 448x448 mnet25 FP16 handle with
max_batch 8.  Prints one JSON line with
  calls/s     of rf_detect_views_rotated with 8 views at 45-degree steps (4 quarter turns, 4 warp views), of rf_detect_views_oriented with
              8 views ({1, 6, 3, 8} at shrink 1 and 0.75) and of the 12-view 30-degree sweep (two batches): warmed up, --rounds
              alternated rounds of at least --min-seconds of back-to-back blocking calls each;
  kernels     microseconds per launch of k_letterbox_warp and k_merge_rotated (45-degree run), and of the oriented letter-box kernels
              (k_letterbox_batch, k_letterbox_transposed) in the oriented run, where each launch covers 4 views as the warp launch does;
              in a separate torch.profiler run of each variant;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/rotated_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import rates
from rates import bench

W, H = 1920, 1080
# name -> the regular expression that picks its launches out of the profile (k_merge<...> without k_merge_rotated)
KERNELS = {"k_letterbox_warp": "k_letterbox_warp", "k_merge_rotated": "k_merge_rotated", "k_letterbox_batch": "k_letterbox_batch",
           "k_letterbox_transposed": "k_letterbox_transposed", "k_merge": "k_merge<"}


def main():
    args = rates.args(warmup=5).parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    img = rates.golden_4k(1, W, H)[0]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=8, max_image=(H, W))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    runs = {
        "rotated_45deg_8views": lambda: eng.detect_views_rotated(img, [(45.0 * k, 1.0) for k in range(8)], thr, nms),
        "oriented_8views": lambda: eng.detect_views_oriented(img, [(s, o) for s in (1.0, 0.75) for o in (1, 6, 3, 8)], thr, nms),
        "rotated_30deg_12views": lambda: eng.detect_views_rotated(img, [(30.0 * k, 1.0) for k in range(12)], thr, nms),
    }
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, 1))
    kern = {}
    for name, fn in runs.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                fn()
            eng.synchronize()
        us, launches = rates.kernel_us(prof, list(KERNELS.values()))
        kern[name] = {k: dict(us_per_launch=us[r], launches=launches[r]) for k, r in KERNELS.items() if launches[r]}
    eng.close()
    ratio = med["rotated_45deg_8views"] / med["oriented_8views"]
    warp = kern["rotated_45deg_8views"]["k_letterbox_warp"]["us_per_launch"]
    lb = [kern["oriented_8views"][k]["us_per_launch"] for k in ("k_letterbox_batch", "k_letterbox_transposed")]
    out = {name: dict(calls_per_s_median=med[name], calls_per_s=[round(r, 1) for r in v], calls=calls[name], kernels=kern[name])
           for name, v in per_round.items()}
    print(json.dumps(dict(image=f"{W}x{H} BGR S-real, host", model="mnet25 FP16 448x448, max_batch 8",
                          rotated_over_oriented_calls=ratio, warp_over_oriented_letterbox=warp / max(lb), gpu=rates.card(), **out)))


if __name__ == "__main__":
    main()
