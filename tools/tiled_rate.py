#!/usr/bin/env python
"""Cost of f7 tiled detection: batches of 8 S-real 3840x2160 BGR images (the golden photo resized to 4K, element i rolled by 8 i
columns), the default pyramid (overlap 64), through rf_detect_tiled on
  - a 448x448 mnet25 FP16 handle with the default execution contexts,
  - the same with streams = 1 (one context, the latency plan),
  - a 1280x896 mnet25 FP16 handle.
Prints one JSON line with, per handle:
  tiled       blocking calls timed with the host clock after warm-up, at least --min-seconds of calls: images/s and tiles/s;
  batch       the same images through rf_detect_batch (one letter-box each), and the cost ratio tiled / batch;
  kernels     in a separate torch.profiler run: microseconds per launch of the tile letter-box and of the merge kernel;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/tiled_rate.py [--min-seconds S] [--warmup W]
"""
import argparse
import json
import os

import numpy as np

import rates
from rates import bench

W4K, H4K, B = 3840, 2160, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    imgs = rates.golden_4k(B)
    model = os.path.join(bench.GOLD, "weights", "mnet25.caffemodel")
    out = {}
    for name, (nw, nh, streams) in {"448x448": (448, 448, 0), "448x448_streams1": (448, 448, 1), "1280x896": (1280, 896, 0)}.items():
        eng = Engine(model, nh, nw, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(H4K, W4K), streams=streams)
        tiles = len(capi.tile_layout(nw, nh, W4K, H4K))
        # blocking calls: seconds per call is the inverse of host_rate's calls per second
        r_tiled, k_tiled = rates.host_rate(lambda: eng.detect_tiled(imgs, bench.SCORE_THR, bench.NMS_THR), eng.synchronize, args.min_seconds,
                                           args.warmup, 1)
        r_batch, k_batch = rates.host_rate(lambda: eng.detect_batch(imgs, bench.SCORE_THR, bench.NMS_THR), eng.synchronize, args.min_seconds,
                                           args.warmup, 1)
        s_tiled, s_batch = 1 / r_tiled, 1 / r_batch
        faces, _ = eng.detect_tiled(imgs, bench.SCORE_THR, bench.NMS_THR)
        plain = eng.detect_batch(imgs, bench.SCORE_THR, bench.NMS_THR)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                eng.detect_tiled(imgs, bench.SCORE_THR, bench.NMS_THR)
            eng.synchronize()
        us, launches = rates.kernel_us(prof, ["k_letterbox_batch", "k_merge"])
        out[name] = dict(
            net=f"{nw}x{nh}", streams=streams, tiles_per_image=tiles,
            tiled=dict(calls=k_tiled, ms_per_call=s_tiled * 1e3, images_per_s=B / s_tiled, tiles_per_s=B * tiles / s_tiled,
                       faces_per_image=float(np.mean([len(f) for f in faces]))),
            batch=dict(calls=k_batch, ms_per_call=s_batch * 1e3, images_per_s=B / s_batch,
                       faces_per_image=float(np.mean([len(f) for f in plain]))),
            cost_ratio_tiled_over_batch=s_tiled / s_batch,
            kernels=dict(tile_letterbox_us_per_launch=us["k_letterbox_batch"], letterbox_launches=launches["k_letterbox_batch"],
                         merge_us_per_launch=us["k_merge"], merge_launches=launches["k_merge"]))
        eng.close()
    print(json.dumps(dict(images=f"{B} x {W4K}x{H4K} S-real BGR, pageable", pyramid="default, overlap 64", model="mnet25 FP16", gpu=rates.card(),
                          **out)))


if __name__ == "__main__":
    main()
