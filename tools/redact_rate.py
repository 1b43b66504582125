#!/usr/bin/env python
"""Cost of f12 redaction on device-resident video: track_rate.py's eight 1920x1080 NV12 BT.601 videos, one frame of each per call, batch 8,
a 448x448 mnet25 FP16 handle with the default execution contexts, plus a tiled case: eight 3840x2160 NV12 frames (the photo at half
scale, four times) through rf_detect_yuv_tiled_device, then rf_redact_yuv_device.  Prints one JSON line with
  frames/s    detect (rf_detect_yuv_batch_device), detect+redact, track (rf_detect_yuv_track_device), track+redact, tiled and
              tiled+redact: warmed up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock
              ended by rf_synchronize.  The detector always reads the same unredacted frames, so that every call sees the same faces;
              the redaction writes a second set of surfaces with that call's records (and tracks) -- the launches
              rf_detect_yuv_redact_device issues after the forward;
  kernel_us   microseconds per launch of each k_redact_* kernel (and their sum per 8-frame call) in a separate torch.profiler run, the mean
              faces per frame, and the byte floor of one call: the region pixels (1.5 bytes each) read twice and written once, over
              3.35 TB/s;
and the card's name, power limit and maximum SM clock, read in the same command.  --style / --shape / --detail (f14) redact with that style instead
of f12's rectangular mosaic; the runs then add detect+mosaic (the f12 call on the same records), the style's rate against it, and
k_redact_blur's time per launch.

    python tools/redact_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--style mosaic|blur] [--shape rect|ellipse] [--detail D]
"""
import json
import os

import numpy as np

import rates
from rates import bench

W, H, B, FRAMES = 1920, 1080, 8, 16
KERNELS = ("k_redact_regions", "k_redact_measure", "k_redact_apply")


def _floor_bytes(recs, scales, w, h):
    """Region pixels of one call (the union of each frame's rectangles inside the frame), 1.5 bytes each, read twice, written once."""
    from oracle.redact import frame_regions, params
    b, m = params()
    px = 0
    for i, r in enumerate(recs):
        mask = np.zeros((h, w), bool)
        for X0, Y0, X1, Y1, _ in frame_regions(r, len(r), None if scales is None else scales[i], m, b):
            mask[max(Y0, 0):Y1, max(X0, 0):X1] = True
        px += int(mask.sum())
    return 3 * 1.5 * px


def main():
    ap = rates.args(warmup=10)
    ap.add_argument("--style", default="mosaic", choices=("mosaic", "blur"))
    ap.add_argument("--shape", default="rect", choices=("rect", "ellipse"))
    ap.add_argument("--detail", type=int, default=0)
    args = ap.parse_args()
    rk = dict(style=args.style, shape=args.shape, detail=args.detail)
    styled = (args.style, args.shape, args.detail) != ("mosaic", "rect", 0)
    kernels = KERNELS + (("k_redact_blur",) if styled else ())
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    photo = cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg"))
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    out = [f.clone() for f in frames[0]]
    half = cv2.resize(photo, None, fx=0.5, fy=0.5)
    big = np.full((2160, 3840, 3), 128, np.uint8)
    for x, y in ((200, 150), (2000, 300), (900, 1300), (2900, 1500)):
        big[y:y + half.shape[0], x:x + half.shape[1]] = half
    tiled_in = [torch.from_numpy(bgr_to_frame(np.roll(big, 16 * i, axis=1), "nv12")).cuda() for i in range(B)]
    tiled_out = [f.clone() for f in tiled_in]
    torch.cuda.synchronize()
    weights = os.path.join(bench.GOLD, "weights", "mnet25.caffemodel")
    eng = Engine(weights, 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(H, W))
    eng4k = Engine(weights, 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(2160, 3840))
    trk = eng.tracker(max_videos=B)
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]

    def detect_redact():
        d, c, sc = eng.detect_yuv_device(nxt(), thr, nms)
        eng.redact_yuv_device(out, d, c, sc, **rk)

    def detect_mosaic():
        d, c, sc = eng.detect_yuv_device(nxt(), thr, nms)
        eng.redact_yuv_device(out, d, c, sc)

    def track_redact():
        tp, tc, d, c, sc = trk.detect_yuv_device(nxt(), vids, thr, nms)
        eng.redact_yuv_device(out, d, c, sc, tracker=trk, tracks_ptr=tp, track_counts_ptr=tc, **rk)

    def tiled_redact():
        d, c = eng4k.detect_yuv_tiled_device(tiled_in, thr, nms)
        eng4k.redact_yuv_device(tiled_out, d, c, None, **rk)

    runs = {
        "detect": (eng, lambda: eng.detect_yuv_device(nxt(), thr, nms)),
        "detect+redact": (eng, detect_redact),
        "track": (eng, lambda: trk.detect_yuv_device(nxt(), vids, thr, nms)),
        "track+redact": (eng, track_redact),
        "tiled": (eng4k, lambda: eng4k.detect_yuv_tiled_device(tiled_in, thr, nms)),
        "tiled+redact": (eng4k, tiled_redact),
    }
    if styled:
        runs["detect+mosaic"] = (eng, detect_mosaic)
    med, per_round, _ = rates.alternate(runs, args.rounds,
                                        lambda run: rates.host_rate(run[1], run[0].synchronize, args.min_seconds, args.warmup, B))
    d, c, sc = eng.detect_yuv_device(frames[0], thr, nms)
    recs = eng.read_dets(d, c, B)[0]
    faces = float(np.mean([len(r) for r in recs]))
    floor_bytes = _floor_bytes(recs, sc, W, H)
    d, c = eng4k.detect_yuv_tiled_device(tiled_in, thr, nms)
    recs4k = eng4k.read_dets(d, c, B)[0]
    kernel_us = {}
    for name in ("detect+redact", "tiled+redact") + (("detect+mosaic",) if styled else ()):
        e, fn = runs[name]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(50):
                fn()
            e.synchronize()
        per, _ = rates.kernel_us(prof, kernels)
        per["per_call"] = sum(v for v in per.values() if v is not None)
        kernel_us[name] = per
    med = {k: round(v, 1) for k, v in med.items()}
    res = dict(frames_per_s=med, rounds=per_round, redact_share={k: round(med[k + "+redact"] / med[k], 4) for k in ("detect", "track", "tiled")},
               kernel_us=kernel_us, faces_per_frame=faces, faces_per_frame_4k=float(np.mean([len(r) for r in recs4k])),
               floor_bytes_per_call=floor_bytes, floor_us_per_call=floor_bytes / 3.35e12 * 1e6,
               floor_bytes_per_call_4k=_floor_bytes(recs4k, None, 3840, 2160), gpu=rates.card())
    if styled:
        res["style"] = rk
        res["style_vs_mosaic"] = dict(frames=round(med["detect+redact"] / med["detect+mosaic"], 4),
                                      kernels=round(kernel_us["detect+redact"]["per_call"] / kernel_us["detect+mosaic"]["per_call"], 4))
    print(json.dumps(res))
    trk.close()
    eng.close()
    eng4k.close()


if __name__ == "__main__":
    main()
