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
and the card's name, power limit and maximum SM clock, read in the same command.  The videos loop over 16 frames, so tracks live on
and the best-shot store is exercised on every frame; best_cost is 1 - (detect + track + best) / (detect + track).

    python tools/bestshot_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rates import bench

B, FRAMES = 8, 16
KERNELS = ("k_track_update", "k_best_measure", "k_best_select", "k_best_emit", "k_best_commit")


def main():
    args = rates.args(warmup=10).parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(1080, 1920))
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
    med, per_round, _ = rates.alternate(runs, args.rounds, lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    d, c, _ = eng.detect_yuv_device(frames[0], thr, nms)
    faces = float(np.mean([len(f) for f in eng.read_dets(d, c, B)[0]]))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            runs["detect+track+best"]()
        eng.synchronize()
    us, launches = rates.kernel_us(prof, KERNELS)
    med = {k: round(v, 1) for k, v in med.items()}
    print(json.dumps(dict(frames_per_s=med, rounds=per_round, best_cost=round(1 - med["detect+track+best"] / med["detect+track"], 4),
                          kernel_us={k: None if t is None else round(t, 2) for k, t in us.items()}, launches=launches, faces_per_frame=faces, gpu=rates.card())))
    best.close()
    trk.close()
    eng.close()


if __name__ == "__main__":
    main()
