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
import json
import os
import re

import numpy as np

import rates
from rates import bench

W, H, B, O = 3840, 2160, 8, 6


def main():
    args = rates.args().parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from oracle.orient import orient_planes
    from retinaface_b200 import RF_PREC_FP16, Engine
    stored = [bgr_to_frame(im, "nv12") for im in rates.golden_4k(B, W, H)]
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
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    lb = {}
    for name, fn in runs.items():
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                fn()
            eng.synchronize()
        us, launches = rates.kernel_us(prof, ["k_letterbox"])
        kinds = sorted({re.search(r"k_letterbox_\w+", e.name).group(0) for e in prof.events() if "k_letterbox" in e.name})
        lb[name] = dict(us_per_launch=us["k_letterbox"], launches=launches["k_letterbox"], kernels=kinds)
    eng.close()
    out = {name: dict(frames_per_s_median=med[name], frames_per_s=[round(r, 1) for r in v], calls=calls[name], letterbox=lb[name])
           for name, v in per_round.items()}
    o, p = out["oriented_stored"], out["portrait_surfaces"]
    print(json.dumps(dict(frames=f"{B} x {W}x{H} NV12 BT.601 S-real, device, shown at {O}", model="mnet25 FP16 448x448, batch 8, default contexts",
                          gpu=rates.card(), records_equal=same, rate_ratio=o["frames_per_s_median"] / p["frames_per_s_median"],
                          letterbox_ratio=(o["letterbox"]["us_per_launch"] / p["letterbox"]["us_per_launch"]
                                           if o["letterbox"]["us_per_launch"] and p["letterbox"]["us_per_launch"] else None),
                          **out)))


if __name__ == "__main__":
    main()
