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
the card's name, power limit and maximum SM clock, read in the same command.

    python tools/tiled_track_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rates import bench

W4K, H4K, B = 3840, 2160, 8


def cycle(k, detect, follow):
    """A call function that detects on every k-th call and follows on the others."""
    n = [0]

    def fn():
        (detect if n[0] % k == 0 else follow)()
        n[0] += 1
    return fn


def main():
    args = rates.args().parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    dev = [torch.from_numpy(bgr_to_frame(im, "nv12")).cuda() for im in rates.golden_4k(B)]
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
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
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
    out = {name: dict(frames_per_s_median=round(med[name], 1), frames_per_s=[round(r, 1) for r in v], calls=calls[name])
           for name, v in per_round.items()}
    ratios = {f"{name}_over_detect": round(med[name] / med["detect"], 4) for name in ("track", "motion", "redact", "lookback15")}
    ratios.update({f"{name}_over_track": round(med[name] / med["track"], 3) for name in ("follow_k3", "follow_k5", "lookback15_k3")})
    print(json.dumps(dict(frames=f"{B} videos x {W4K}x{H4K} NV12 BT.601 S-real, one frame of each per call", pyramid="default, overlap 64",
                          tiles_per_frame=len(capi.tile_layout(448, 448, W4K, H4K)), model="mnet25 FP16 448x448, default contexts",
                          faces_per_frame=float(np.mean([len(f) for f in faces])), gpu=rates.card(), **out, ratios=ratios,
                          profiled_us_per_call={k: round(v, 1) for k, v in per_call.items()})))


if __name__ == "__main__":
    main()
