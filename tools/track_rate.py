#!/usr/bin/env python
"""Cost of f10 tracking on device-resident video: eight 1920x1080 NV12 BT.601 videos on the device (the golden photo resized to 1080p,
video i rolled by 8 i columns and moved 7 px per frame), one frame of each per call, batch 8, a 448x448 mnet25 FP16 handle with the
default execution contexts.  Prints one JSON line with
  frames/s    of rf_detect_yuv_batch_device (detect), rf_detect_yuv_track_device (detect + track) and rf_detect_yuv_track_device with
              112x112 crops of the new identities (detect + track + crops): warmed up, --rounds alternated rounds of at least
              --min-seconds of back-to-back calls each, the host clock ended by rf_synchronize;
  track_us    microseconds per k_track_update launch, in a separate torch.profiler run, and the mean faces per frame;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/track_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rates import bench

B, FRAMES = 8, 16


def main():
    args = rates.args(warmup=10).parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(1080, 1920))
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
    med, per_round, _ = rates.alternate(runs, args.rounds, lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    d, c, _ = eng.detect_yuv_device(frames[0], thr, nms)
    faces = float(np.mean([len(f) for f in eng.read_dets(d, c, B)[0]]))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            runs["detect+track"]()
        eng.synchronize()
    us, launches = rates.kernel_us(prof, ["k_track_update"])
    print(json.dumps(dict(frames_per_s={k: round(v, 1) for k, v in med.items()}, rounds=per_round, track_us=us["k_track_update"],
                          track_launches=launches["k_track_update"], faces_per_frame=faces, gpu=rates.card())))
    trk.close()
    eng.close()


if __name__ == "__main__":
    main()
