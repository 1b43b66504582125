#!/usr/bin/env python
"""Cost of f13 camera-motion compensation: track_rate.py's eight 1920x1080 NV12 BT.601 device videos (the golden photo resized to
1080p, video i rolled by 8 i columns), with the camera shaking -- each frame the photo's window moves by a seeded step of 40-70 px
with changing signs -- one frame of each per call, batch 8, a 448x448 mnet25 FP16 handle with the default execution contexts.  Prints
one JSON line with
  frames/s    of rf_detect_yuv_track_device on a plain tracker (detect+track) and on a motion tracker (detect+track+motion): warmed
              up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended by
              rf_synchronize;
  kernel_us   microseconds per launch of k_motion_thumb, k_motion_match, k_motion_fit and k_motion_commit (and k_track_update) in a
              separate torch.profiler run, and their sum per 8-frame call;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/motion_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rates import bench

W, H, B, FRAMES = 1920, 1080, 8, 16
KERNELS = ("k_motion_thumb", "k_motion_match", "k_motion_fit", "k_motion_commit", "k_track_update")


def main():
    args = rates.args(warmup=10).parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    pad = 200
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W + 2 * pad, H + 2 * pad))
    rng = np.random.default_rng(3)
    x, sign, frames = pad, 1, []
    for t in range(FRAMES):
        step = int(rng.integers(40, 71))
        if not 0 <= x + sign * step <= 2 * pad:
            sign = -sign
        x += sign * step
        sign = -sign if rng.uniform() < 0.5 else sign
        img = np.ascontiguousarray(base[pad:pad + H, x:x + W])
        frames.append([torch.from_numpy(bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12")).cuda() for i in range(B)])
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H, W))
    plain = eng.tracker(max_videos=B)
    moving = eng.tracker(max_videos=B, motion=True)
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]
    runs = {
        "detect+track": lambda: plain.detect_yuv_device(nxt(), vids, thr, nms),
        "detect+track+motion": lambda: moving.detect_yuv_device(nxt(), vids, thr, nms),
    }
    med, per_round, _ = rates.alternate(runs, args.rounds, lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    calls = 50
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            runs["detect+track+motion"]()
        eng.synchronize()
    us, launches = rates.kernel_us(prof, KERNELS)
    per_call = sum(us[k] * launches[k] for k in KERNELS[:4] if us[k]) / calls
    status = moving.motion(B)["status"].tolist()
    med = {k: round(v, 1) for k, v in med.items()}
    print(json.dumps(dict(frames_per_s=med, rounds=per_round, motion_cost=round(1 - med["detect+track+motion"] / med["detect+track"], 4),
                          kernel_us=us, launches=launches, motion_us_per_call=per_call, last_status=status, gpu=rates.card())))
    plain.close()
    moving.close()
    eng.close()


if __name__ == "__main__":
    main()
