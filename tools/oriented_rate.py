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
import json
import os

import rates
from rates import bench

W, H, B = 1920, 1080, 8


def main():
    args = rates.args(warmup=5).parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    dev = [torch.from_numpy(bgr_to_frame(im, "nv12")).cuda() for im in rates.golden_4k(B, W, H)]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H, W))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    runs = {
        "o1_yuv_batch_device": lambda: eng.detect_yuv_device(dev, thr, nms),
        "o3_oriented_device": lambda: eng.detect_yuv_oriented_device(dev, [3] * B, thr, nms),
        "o6_oriented_device": lambda: eng.detect_yuv_oriented_device(dev, [6] * B, thr, nms),
    }
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    lb = {}
    for name, fn in runs.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                fn()
            eng.synchronize()
        us, launches = rates.kernel_us(prof, ["k_letterbox"])
        lb[name] = dict(us_per_launch=us["k_letterbox"], launches=launches["k_letterbox"])
    eng.close()
    out = {name: dict(frames_per_s_median=med[name], frames_per_s=[round(r, 1) for r in v], calls=calls[name], letterbox=lb[name])
           for name, v in per_round.items()}
    print(json.dumps(dict(frames=f"{B} x {W}x{H} NV12 BT.601 S-real, device", model="mnet25 FP16 448x448, batch 8, default contexts",
                          gpu=rates.card(), **out)))


if __name__ == "__main__":
    main()
