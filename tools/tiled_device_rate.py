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
import json
import os

import numpy as np

import rates
from rates import bench

W4K, H4K, B = 3840, 2160, 8


def main():
    args = rates.args().parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    frames = [bgr_to_frame(im, "nv12") for im in rates.golden_4k(B)]
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
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            runs["device_crops_f16"]()
        eng.synchronize()
    us, launches = rates.kernel_us(prof, ["k_align_faces"])
    faces, _ = eng.detect_yuv_tiled(pinned, thr, nms)
    eng.close()
    out = {name: dict(frames_per_s_median=med[name], frames_per_s=[round(r, 1) for r in v], calls=calls[name]) for name, v in per_round.items()}
    print(json.dumps(dict(frames=f"{B} x {W4K}x{H4K} NV12 BT.601 S-real", pyramid="default, overlap 64",
                          tiles_per_frame=len(capi.tile_layout(448, 448, W4K, H4K)), model="mnet25 FP16 448x448, default contexts",
                          faces_per_frame=float(np.mean([len(f) for f in faces])), gpu=rates.card(), **out,
                          align_kernel=dict(us_per_launch=us["k_align_faces"], launches=launches["k_align_faces"]))))


if __name__ == "__main__":
    main()
