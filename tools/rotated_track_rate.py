#!/usr/bin/env python
"""Cost of f25 rotated views as a tracker's detector: eight 1920x1080 NV12 BT.601 device videos of the golden photo tilted 45 degrees
(rotated_device_rate.py's scene; video v rolled by 8 v columns, drifting 4 columns a frame), a 448x448 mnet25 FP16 handle with
max_batch 8, the 8-view 45-degree sweep, score threshold 0.5 and NMS 0.4.  One call takes one frame of each video.  Prints one JSON
line with frames/s, warmed up, --rounds alternated rounds of at least --min-seconds each, of
  rotated_detect      rf_detect_yuv_views_rotated_device alone,
  views_tracker       rf_detect_yuv_track_device on a views tracker,
  views_blur          rf_detect_yuv_redact_device_style (blur, ellipse) on a views tracker,
  views_lookback15    rf_detect_yuv_redact_lookback_device on a views look-back tracker, L = 15,
  views_follow_k1     a views follow tracker detecting every frame (k = 1: every call a detect call),
  views_follow_k3     the same detecting every third call and following the two between (rf_track_follow_device);
the ratios the targets name (views_tracker / rotated_detect >= 0.97, follow k = 3 / k = 1 >= 2), confirmed tracks after the warm-up
run, and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/rotated_track_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rotated_device_rate import B, H, W, tilted_scene

VIEWS = [(45.0 * k, 1.0) for k in range(8)]
THR, NMS = 0.5, 0.4
FRAMES = 24          # distinct frames of each video, cycled


def main():
    args = rates.args(warmup=6).parse_args()
    import torch
    from retinaface_b200 import RF_PREC_FP16, Engine, capi
    from oracle.yuv import bgr_to_frame, frame_to_bgr
    base = frame_to_bgr(tilted_scene()[0][0], "nv12")
    # frame k of video v: the scene rolled by 8 v + 4 k columns
    dev = [[torch.from_numpy(bgr_to_frame(np.roll(base, 8 * v + 4 * k, axis=1), "nv12")).cuda() for v in range(B)] for k in range(FRAMES)]
    vids = list(range(B))
    eng = Engine(os.path.join(rates.bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B,
                 max_image=(H, W))
    trk = {name: eng.tracker(max_videos=B, views=VIEWS, **kw) for name, kw in
           (("track", {}), ("blur", {}), ("lookback", {"lookback": 15}), ("follow1", {"follow": True}), ("follow3", {"follow": True}))}
    outs = [torch.empty_like(f) for f in dev[0]]
    step = {name: 0 for name in ("detect",) + tuple(trk)}

    def nxt(name):
        k = step[name]
        step[name] += 1
        return k

    def follow(name, every):
        k = nxt(name)
        frames = dev[k % FRAMES]
        if k % every == 0:
            return trk[name].detect_yuv_device(frames, vids, THR, NMS)
        return trk[name].follow_device(frames, vids)

    runs = {
        "rotated_detect": lambda: eng.detect_yuv_views_rotated_device(dev[nxt("detect") % FRAMES], VIEWS, THR, NMS),
        "views_tracker": lambda: trk["track"].detect_yuv_device(dev[nxt("track") % FRAMES], vids, THR, NMS),
        "views_blur": lambda: trk["blur"].detect_yuv_redact_device(dev[nxt("blur") % FRAMES], vids, THR, NMS, style="blur", shape="ellipse"),
        "views_lookback15": lambda: trk["lookback"].detect_yuv_redact_lookback_device(dev[nxt("lookback") % FRAMES], vids, outs, THR, NMS),
        "views_follow_k1": lambda: follow("follow1", 1),
        "views_follow_k3": lambda: follow("follow3", 3),
    }
    for name, fn in runs.items():     # the warm-up run: every tracker sees its faces before the clock starts
        for _ in range(FRAMES):
            last = fn()
        if name == "views_tracker":
            tp, tc = last[0], last[1]
            confirmed = [int((lst["state"] == capi.TRACK_CONFIRMED).sum()) for lst in trk["track"].read(tp, tc, B)]
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    for t in trk.values():
        t.close()
    eng.close()
    out = {name: dict(frames_per_s_median=med[name], frames_per_s=[round(r, 1) for r in v], calls=calls[name])
           for name, v in per_round.items()}
    print(json.dumps(dict(
        frames=f"{B} videos x {W}x{H} NV12 BT.601 device, golden photo tilted 45 degrees, drifting", model=f"mnet25 FP16 448x448, max_batch {B}",
        views="8 at 45-degree steps", views_tracker_over_rotated_detect=med["views_tracker"] / med["rotated_detect"],
        follow_k3_over_k1=med["views_follow_k3"] / med["views_follow_k1"], confirmed_tracks_per_video=confirmed, gpu=rates.card(), **out)))


if __name__ == "__main__":
    main()
