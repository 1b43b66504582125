#!/usr/bin/env python
"""Cost of f20 oriented videos in tracker calls: eight 1920x1080 NV12 BT.601 device videos stored as landscape surfaces and shown at
orientation 6 (the golden photo on a portrait canvas, video i rolled by 8 i rows), one frame of each per call, a 448x448 mnet25 FP16
handle with the default execution contexts, against the same frames materialised as 1080x1920 portrait surfaces at orientation 1.
Both sides detect the same faces and draw the same regions; only the addressing differs.  Prints one JSON line with frames/s
(warmed up, at least --min-seconds of back-to-back calls ended by rf_synchronize, --rounds rounds with the modes and the two sides
alternated) of
  track          rf_detect_yuv_track_device;
  mosaic         rf_detect_yuv_redact_device, mosaic / rect, in place (later calls see the mosaicked faces, on both sides);
  blur           the same with the blur / ellipse style;
  motion         a motion tracker's rf_detect_yuv_track_device;
  lookback15     rf_detect_yuv_redact_lookback_device at L = 15 (mosaic) into separate out frames;
  follow_k3      a follow tracker detecting every 3rd call and following the others (rf_track_follow_device);
each mode's oriented / portrait ratio, the card's name, power limit and maximum SM clock read in the same command, and, from a separate torch.profiler
run, the device time per launch of the redaction apply and blur, motion thumbnail and follow search kernels in their oriented and
upright instantiations.

    python tools/oriented_track_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os
from collections import defaultdict

import numpy as np

import rates
from rates import bench

W, H, B, O = 1920, 1080, 8, 6


def cycle(k, detect, follow):
    """A call function that detects on every k-th call and follows on the others."""
    n = [0]

    def fn():
        (detect if n[0] % k == 0 else follow)()
        n[0] += 1
    return fn


def main():
    args = rates.args().parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from oracle.orient import unorient_planes
    from retinaface_b200 import RF_PREC_FP16, Engine
    canvas = np.full((W, H, 3), 128, np.uint8)          # displayed: H wide, W tall
    g = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), None, fx=0.8, fy=0.8)
    canvas[200:200 + g.shape[0], :g.shape[1]] = g[:, :H]
    shown = [bgr_to_frame(np.roll(canvas, 8 * i, axis=0), "nv12") for i in range(B)]
    stored = [unorient_planes(f, "nv12", O) for f in shown]
    dev = {"oriented": [torch.from_numpy(f).cuda() for f in stored], "portrait": [torch.from_numpy(f).cuda() for f in shown]}
    torch.cuda.synchronize()
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(W, W))
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    kinds = {"track": {}, "mosaic": {}, "blur": {}, "motion": {"motion": True}, "lookback15": {"lookback": 15}, "follow_k3": {"follow": True}}
    runs, trackers = {}, []
    for side in ("oriented", "portrait"):
        for mode, kw in kinds.items():
            t = eng.tracker(max_videos=B, **kw)
            if side == "oriented":
                t.set_orientation(-1, O)
            trackers.append(t)
            fr = dev[side] if mode in ("track", "motion", "follow_k3") else [d.clone() for d in dev[side]]
            outs = [d.clone() for d in dev[side]]
            torch.cuda.synchronize()
            runs[(mode, side)] = {
                "track": lambda t=t, fr=fr: t.detect_yuv_device(fr, vids, thr, nms),
                "mosaic": lambda t=t, fr=fr: t.detect_yuv_redact_device(fr, vids, thr, nms),
                "blur": lambda t=t, fr=fr: t.detect_yuv_redact_device(fr, vids, thr, nms, style="blur", shape="ellipse"),
                "motion": lambda t=t, fr=fr: t.detect_yuv_device(fr, vids, thr, nms),
                "lookback15": lambda t=t, fr=fr, outs=outs: t.detect_yuv_redact_lookback_device(fr, vids, outs, thr, nms),
                "follow_k3": cycle(3, lambda t=t, fr=fr: t.detect_yuv_device(fr, vids, thr, nms), lambda t=t, fr=fr: t.follow_device(fr, vids)),
            }[mode]
    got = defaultdict(list)
    for r in range(args.rounds):              # alternated: every round runs each mode on both sides, the side order swapped per round
        for mode in kinds:
            for side in (("oriented", "portrait") if r % 2 == 0 else ("portrait", "oriented")):
                got[(mode, side)].append(rates.host_rate(runs[(mode, side)], eng.synchronize, args.min_seconds, args.warmup, B)[0])
    eng.synchronize()
    # a separate profiled run: device time per launch of the kernels whose addressing differs
    per_launch = defaultdict(lambda: [0.0, 0])
    for mode in ("mosaic", "blur", "motion", "follow_k3"):
        for side in ("oriented", "portrait"):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(6):
                    runs[(mode, side)]()
                eng.synchronize()
            for e in prof.events():
                if e.device_type.name != "CUDA":
                    continue
                name = e.name
                for k in ("k_redact_apply", "k_redact_blur", "k_redact_measure", "k_motion_thumb", "k_follow_search", "k_follow_cut"):
                    if k in name:
                        inst = "oriented" if ("YuvPlanesWO" in name or "_oriented" in name or "<true>" in name) else "upright"
                        key = f"{k}{'<ellipse>' if k == 'k_redact_apply' and mode == 'blur' else ''} {inst}"
                        per_launch[key][0] += e.device_time
                        per_launch[key][1] += 1
    for t in trackers:
        t.close()
    eng.close()
    med = {k: float(np.median(v)) for k, v in got.items()}
    out = {mode: dict(oriented_frames_per_s=round(med[(mode, "oriented")], 1), portrait_frames_per_s=round(med[(mode, "portrait")], 1),
                      ratio=round(med[(mode, "oriented")] / med[(mode, "portrait")], 4),
                      oriented_runs=[round(x, 1) for x in got[(mode, "oriented")]], portrait_runs=[round(x, 1) for x in got[(mode, "portrait")]])
           for mode in kinds}
    print(json.dumps(dict(frames=f"{B} videos x {W}x{H} NV12 BT.601 stored, shown at orientation {O}, vs {H}x{W} portrait surfaces at 1; "
                                 "one frame of each per call", model="mnet25 FP16 448x448, default contexts", gpu=rates.card(), modes=out,
                          profiled_us_per_launch={k: round(v[0] / v[1], 2) for k, v in sorted(per_launch.items())},
                          profiled_launches={k: v[1] for k, v in sorted(per_launch.items())})))


if __name__ == "__main__":
    main()
