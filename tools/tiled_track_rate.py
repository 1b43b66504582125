#!/usr/bin/env python
"""Cost of f19 tiling trackers on 4K video: eight 3840x2160 NV12 BT.601 device videos (the golden photo resized to 4K, video i rolled
by 8 i columns), one frame of each per call, a 448x448 mnet25 FP16 handle with the default pyramid (84 tiles per frame) and the
default execution contexts.  Prints one JSON line with frames/s (warmed up, at least --min-seconds of back-to-back calls ended by
rf_synchronize, --rounds rounds with the modes alternated) of
  detect          rf_detect_yuv_tiled_device alone;
  track           a tiling tracker's rf_detect_yuv_track_device;
  motion          the same with camera motion;
  redact          rf_detect_yuv_redact_device (mosaic) with a tiling tracker, in place (later calls see mosaicked faces);
  lookback15      rf_detect_yuv_redact_lookback_device at L = 15 (mosaic) into separate out frames;
  follow_k3/k5    a tiling follow tracker that detects every 3rd / 5th call and follows the others (rf_track_follow_device);
  lookback15_k3   a following look-back tracker at L = 15, detecting every 3rd call (rf_track_follow_redact_lookback_device between);
each mode's ratio to detect (follow: to track), the device time per call of detect and track from a separate torch.profiler run, and
the card's name and power limit, read in the same command.

    python tools/tiled_track_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

W4K, H4K, B = 3840, 2160, 8


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


def cycle(k, detect, follow):
    """A call function that detects on every k-th call and follows on the others."""
    n = [0]

    def fn():
        (detect if n[0] % k == 0 else follow)()
        n[0] += 1
    return fn


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
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W4K, H4K))
    frames = [bgr_to_frame(np.roll(base, 8 * i, axis=1), "nv12") for i in range(B)]
    dev = [torch.from_numpy(f).cuda() for f in frames]
    red = [d.clone() for d in dev]
    outs = [d.clone() for d in dev]
    vids = list(range(B))
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(H4K, W4K))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    trk = {name: eng.tracker(max_videos=B, tiling=True, **kw) for name, kw in {
        "track": {}, "motion": {"motion": True}, "redact": {}, "lookback15": {"lookback": 15}, "follow_k3": {"follow": True},
        "follow_k5": {"follow": True}, "lookback15_k3": {"lookback": 15, "lookback_follow": True}}.items()}
    runs = {
        "detect": lambda: eng.detect_yuv_tiled_device(dev, thr, nms),
        "track": lambda: trk["track"].detect_yuv_device(dev, vids, thr, nms),
        "motion": lambda: trk["motion"].detect_yuv_device(dev, vids, thr, nms),
        "redact": lambda: trk["redact"].detect_yuv_redact_device(red, vids, thr, nms),
        "lookback15": lambda: trk["lookback15"].detect_yuv_redact_lookback_device(dev, vids, outs, thr, nms),
        "follow_k3": cycle(3, lambda: trk["follow_k3"].detect_yuv_device(dev, vids, thr, nms), lambda: trk["follow_k3"].follow_device(dev, vids)),
        "follow_k5": cycle(5, lambda: trk["follow_k5"].detect_yuv_device(dev, vids, thr, nms), lambda: trk["follow_k5"].follow_device(dev, vids)),
        "lookback15_k3": cycle(3, lambda: trk["lookback15_k3"].detect_yuv_redact_lookback_device(dev, vids, outs, thr, nms),
                               lambda: trk["lookback15_k3"].follow_redact_lookback_device(dev, vids, outs)),
    }
    got = {k: [] for k in runs}
    for _ in range(args.rounds):              # alternated: every round runs each mode once
        for name, fn in runs.items():
            got[name].append(rate(fn, eng.synchronize, args.min_seconds, args.warmup))
    eng.synchronize()
    per_call = {}
    for name in ("detect", "track"):          # a separate profiled run: device time of every kernel per call
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                runs[name]()
            eng.synchronize()
        per_call[name] = sum(e.device_time for e in prof.events() if e.device_type.name == "CUDA") / 5
    faces = eng.read_dets(*eng.detect_yuv_tiled_device(dev, thr, nms), B)[0]
    for t in trk.values():
        t.close()
    eng.close()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                         text=True).stdout.strip()
    med = {name: float(np.median([r for r, _ in v])) for name, v in got.items()}
    out = {name: dict(frames_per_s_median=round(med[name], 1), frames_per_s=[round(r, 1) for r, _ in v], calls=[k for _, k in v])
           for name, v in got.items()}
    ratios = {f"{name}_over_detect": round(med[name] / med["detect"], 4) for name in ("track", "motion", "redact", "lookback15")}
    ratios.update({f"{name}_over_track": round(med[name] / med["track"], 3) for name in ("follow_k3", "follow_k5", "lookback15_k3")})
    print(json.dumps(dict(frames=f"{B} videos x {W4K}x{H4K} NV12 BT.601 S-real, one frame of each per call", pyramid="default, overlap 64",
                          tiles_per_frame=len(capi.tile_layout(448, 448, W4K, H4K)), model="mnet25 FP16 448x448, default contexts",
                          faces_per_frame=float(np.mean([len(f) for f in faces])), gpu=gpu, **out, ratios=ratios,
                          profiled_us_per_call={k: round(v, 1) for k, v in per_call.items()})))


if __name__ == "__main__":
    main()
