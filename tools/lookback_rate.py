#!/usr/bin/env python
"""Cost of f15 look-back redaction on device-resident video: redact_rate.py's eight 1920x1080 NV12 BT.601 videos, one frame of each
per call, batch 8, a 448x448 mnet25 FP16 handle.  Prints one JSON line with
  frames/s    track+redact (rf_detect_yuv_track_device, then rf_redact_yuv_device_style of its records and tracks into a second set of
              surfaces: what rf_detect_yuv_redact_device_style launches, without writing the frames the detector reads again) against
              lookback (rf_detect_yuv_redact_lookback_device at L = --frames into separate out surfaces), both mosaic + rect: warmed
              up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended by
              rf_synchronize;
  kernel_us   microseconds per launch of k_lookback_log, k_lookback_swap and k_lookback_boxes in a separate torch.profiler run, and
              k_lookback_swap's effective bandwidth: 4 x w h 3 / 2 bytes per frame (buffer and input read, out and buffer written);
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/lookback_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--frames L]
"""
import json
import os

import rates
from rates import bench

W, H, B, FRAMES = 1920, 1080, 8, 16
KERNELS = ("k_lookback_log", "k_lookback_swap", "k_lookback_boxes")


def main():
    ap = rates.args(warmup=20)
    ap.add_argument("--frames", type=int, default=15)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    out = [f.clone() for f in frames[0]]
    torch.cuda.synchronize()
    weights = os.path.join(bench.GOLD, "weights", "mnet25.caffemodel")
    eng = Engine(weights, 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(H, W))
    trk = eng.tracker(max_videos=B)
    lbt = eng.tracker(max_videos=B, lookback=dict(frames=args.frames))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]

    def track_redact():
        tp, tc, d, c, sc = trk.detect_yuv_device(nxt(), vids, thr, nms)
        eng.redact_yuv_device(out, d, c, sc, tracker=trk, tracks_ptr=tp, track_counts_ptr=tc)

    def lookback():
        lbt.detect_yuv_redact_lookback_device(nxt(), vids, out, thr, nms)

    runs = {"track+redact": track_redact, "lookback": lookback}
    warmup = max(args.warmup, args.frames + 2)
    med, per_round, _ = rates.alternate(runs, args.rounds, lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, warmup, B))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            lookback()
        eng.synchronize()
    kernel_us, _ = rates.kernel_us(prof, KERNELS)
    swap_bytes = B * 4 * W * H * 3 // 2
    med = {k: round(v, 1) for k, v in med.items()}
    print(json.dumps(dict(frames_per_s=med, rounds=per_round, lookback_share=round(med["lookback"] / med["track+redact"], 4), L=args.frames,
                          kernel_us=kernel_us, log_plus_boxes_us=(kernel_us["k_lookback_log"] or 0) + (kernel_us["k_lookback_boxes"] or 0),
                          swap_bytes_per_call=swap_bytes,
                          swap_tb_per_s=swap_bytes / (kernel_us["k_lookback_swap"] * 1e-6) / 1e12 if kernel_us["k_lookback_swap"] else None,
                          swap_floor_us=swap_bytes / 3.35e12 * 1e6, gpu=rates.card())))
    trk.close()
    lbt.close()
    eng.close()


if __name__ == "__main__":
    main()
