#!/usr/bin/env python
"""Cost of f24 rotated views on device-resident video: eight 1920x1080 NV12 BT.601 device frames of a tilted scene (the golden photo
turned 45 degrees counter-clockwise at its own scale, rows 180 .. 1259 of the 1531 x 1531 result -- the band that holds its six faces --
centred on black, frame i rolled by 8 i columns), a 448x448 mnet25 FP16 handle with max_batch 8, score threshold 0.5 (the tests'; at
bench.py's 0.9 faces this small are not kept) and NMS 0.4.  Prints one JSON line with
  frames/s     and network inputs/s, warmed up, --rounds alternated rounds of at least --min-seconds each, of
                 rf_detect_yuv_views_rotated_device with 8 views at 45-degree steps (64 network inputs a call),
                 the same with the four quarter turns only,
                 rf_detect_yuv_batch_device on the same frames,
                 rf_detect_views_rotated on the 8 host BGR copies (cv2.cvtColor of the frames), one blocking call each (8 views at 45 degrees);
  recall       faces found per frame by each variant, over the 6 faces of the upright photo;
  kernels      microseconds per launch of k_letterbox_warp<YuvPlanes> against k_letterbox_warp<BgrRows> on the same views of the same
               pixels (rf_detect_views_rotated_device on BGR device copies), and of k_merge_rotated, in a separate torch.profiler run;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/rotated_device_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rates import bench

W, H, B = 1920, 1080, 8
FACES = 6           # the golden photo's faces
KERNELS = {"warp_yuv": r"k_letterbox_warp<.*YuvPlanes", "warp_bgr": r"k_letterbox_warp<.*BgrRows", "k_merge_rotated": "k_merge_rotated"}


def tilted_scene():
    import cv2
    from oracle.yuv import bgr_to_frame, frame_to_bgr
    img = cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg"))
    h, w = img.shape[:2]
    R = cv2.getRotationMatrix2D((w / 2, h / 2), 45.0, 1.0)
    c, s = abs(R[0, 0]), abs(R[0, 1])
    tw, th = int(h * s + w * c), int(h * c + w * s)
    R[0, 2] += tw / 2 - w / 2
    R[1, 2] += th / 2 - h / 2
    tilted = cv2.warpAffine(img, R, (tw, th))[180:180 + H]
    canvas = np.zeros((H, W, 3), np.uint8)
    x0 = (W - tilted.shape[1]) // 2
    canvas[:, x0:x0 + tilted.shape[1]] = tilted
    frames = [bgr_to_frame(np.roll(canvas, 8 * i, axis=1), "nv12") for i in range(B)]
    return frames, [frame_to_bgr(f, "nv12") for f in frames]


def main():
    args = rates.args(warmup=5).parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames, bgr = tilted_scene()
    dev = [torch.from_numpy(f).cuda() for f in frames]
    dev_bgr = [torch.from_numpy(b).cuda() for b in bgr]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_image=(H, W))
    thr, nms = 0.5, 0.4
    v8 = [(45.0 * k, 1.0) for k in range(8)]
    v4 = [(90.0 * k, 1.0) for k in range(4)]
    runs = {
        "yuv_rotated_8views": lambda: eng.detect_yuv_views_rotated_device(dev, v8, thr, nms)[:2],
        "yuv_rotated_4quarters": lambda: eng.detect_yuv_views_rotated_device(dev, v4, thr, nms)[:2],
        "yuv_batch_device": lambda: eng.detect_yuv_device(dev, thr, nms)[:2],
        "host_rotated_loop": lambda: [eng.detect_views_rotated(b, v8, thr, nms) for b in bgr],
    }
    inputs = {"yuv_rotated_8views": 8, "yuv_rotated_4quarters": 4, "yuv_batch_device": 1, "host_rotated_loop": 8}
    recall = {}
    for name, fn in runs.items():
        out = fn()
        per = [len(r[0]) for r in out] if name == "host_rotated_loop" else [len(f) for f in eng.read_dets(out[0], out[1], B)[0]]
        recall[name] = dict(faces_per_frame=per, recall=sum(per) / (FACES * B))
    med, per_round, calls = rates.alternate(runs, args.rounds,
                                            lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            eng.detect_yuv_views_rotated_device(dev, v8, thr, nms)
            eng.detect_views_rotated_device(dev_bgr, v8, thr, nms)
        eng.synchronize()
    us, launches = rates.kernel_us(prof, list(KERNELS.values()))
    eng.close()
    kern = {k: dict(us_per_launch=us[r], launches=launches[r]) for k, r in KERNELS.items()}
    out = {name: dict(frames_per_s_median=med[name], inputs_per_s_median=med[name] * inputs[name],
                      frames_per_s=[round(r, 1) for r in v], calls=calls[name], **recall[name]) for name, v in per_round.items()}
    batch = med["yuv_batch_device"]
    print(json.dumps(dict(
        frames=f"{B} x {W}x{H} NV12 BT.601 device, golden photo tilted 45 degrees", model=f"mnet25 FP16 448x448, max_batch {B}",
        inputs_8views_over_batch_frames=med["yuv_rotated_8views"] * 8 / batch,
        rotated_8views_over_host_loop=med["yuv_rotated_8views"] / med["host_rotated_loop"],
        warp_yuv_over_bgr=(kern["warp_yuv"]["us_per_launch"] or 0) / max(kern["warp_bgr"]["us_per_launch"] or 1e-9, 1e-9),
        kernels=kern, gpu=rates.card(), **out)))


if __name__ == "__main__":
    main()
