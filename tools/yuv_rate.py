#!/usr/bin/env python
"""Cost of f6 video frames: bench.py's headline configuration (mnet25 FP16, batch 8, 448x448) on S-real 1920x1080 frames (the golden
photo resized to 1080p, element i rolled by 8 i columns, cv2.cvtColor(BGR2YUV_I420), also re-laid out as NV12) in a device ring
larger than twice the H100's L2, as bench.py.  Prints one JSON line:

  device      one device-timed block (CUDA events, rf_fence) of K steps each, the same K, calibrated as align_rate.py:
              rf_detect_yuv_batch_device on NV12 without and with 112x112 RGB F16 crops, and rf_detect_batch_device on the same
              frames pre-letter-boxed to BGR; the difference is the conversion + letter-box per step.
  host        blocking calls, host clock over at least --host-seconds of calls: I420 host frames through rf_detect_yuv_batch vs 1080p
              BGR host images through rf_detect_batch (pinned and pageable), and the CPU cv2.cvtColor a BGR caller pays first, timed
              on its own.
  kernel      in a separate torch.profiler run: the YUV letter-box kernel's microseconds per launch (batch 8) against its byte
              floor -- the luma / chroma rows its taps touch plus the output, at the data-sheet 3.35 TB/s (not measured).

    python tools/yuv_rate.py [--steps K] [--warmup W] [--host-seconds S]
"""
import argparse
import itertools
import json
import os

import numpy as np

import rates
from rates import bench

FW, FH = 1920, 1080


def tap_rows(d_rows, src_rows, scale):
    """Source rows the bilinear vertical taps of output rows [0, d_rows) read (preprocess.cu tap_of<false>)."""
    rows = set()
    for d in range(d_rows):
        s = int(np.floor(np.float32((d + 0.5) * scale - 0.5)))
        rows.update({min(max(s, 0), src_rows - 1), min(max(s + 1, 0), src_rows - 1)})
    return rows


def letterbox_floor_bytes(net_h, net_w):
    """Bytes one 1080p NV12 frame's letter-box must move: every touched luma row and chroma row in whole 32-byte sectors (at a
    4.3x shrink every sector of a touched row holds a tap), plus the net_h x net_w x 3 output."""
    f = np.float32(1) / max(np.float32(FW / net_w), np.float32(FH / net_h))
    scale = 1.0 / float(f)
    dh = int(np.rint(FH * float(f)))
    luma = tap_rows(min(dh, net_h), FH, scale)
    chroma = {r >> 1 for r in luma}
    row = -(-FW // 32) * 32
    return (len(luma) + len(chroma)) * row, net_h * net_w * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=0, help="timed device steps (0: calibrate to about 0.5 s)")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--host-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import cv2
    import torch
    from oracle.inputs import letterbox_bgr_u8
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    w = bench.WORKLOADS[bench.DEFAULT_WORKLOAD]
    B, H, Wd = w["batch"], w["h"], w["w"]
    eng = Engine(os.path.join(bench.GOLD, "weights", w["model"] + ".caffemodel"), H, Wd, precision=RF_PREC_FP16, max_batch=B, max_faces=128,
                 max_image=(FH, FW))
    stream = torch.cuda.ExternalStream(eng.stream_ptr())
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (FW, FH))
    frame_bytes = FW * FH * 3 // 2
    ring = max(2, -(-2 * 50 * 2**20 // (B * frame_bytes)) + 1)
    bgr = [[np.roll(base, 8 * (i + B * s), axis=1) for i in range(B)] for s in range(ring)]
    i420 = [[cv2.cvtColor(im, cv2.COLOR_BGR2YUV_I420) for im in b] for b in bgr]
    nv12 = [[bgr_to_frame(im, "nv12") for im in b] for b in bgr]
    dev = [[torch.from_numpy(f).cuda() for f in b] for b in nv12]
    net = torch.from_numpy(np.stack([np.stack([letterbox_bgr_u8(im, H, Wd) for im in b]) for b in bgr])).cuda()
    nctx = 8
    crops = [torch.empty((B, eng.max_faces, 3, 112, 112), dtype=torch.float16, device="cuda") for _ in range(nctx)]
    pos = [0]

    def step(mode):
        s = pos[0] % ring
        if mode == "yuv":
            eng.detect_yuv_device(dev[s], bench.SCORE_THR, bench.NMS_THR, "nv12")
        elif mode == "yuv_align":
            eng.detect_yuv_device(dev[s], bench.SCORE_THR, bench.NMS_THR, "nv12", align=dict(fmt="rgb_f16"),
                                  dev_crops_ptr=crops[pos[0] % nctx].data_ptr())
        else:
            eng.detect_device(B, bench.SCORE_THR, bench.NMS_THR, net[s].data_ptr())
        pos[0] += 1

    def block(k, mode):
        return rates.device_ms(lambda: step(mode), k, stream, eng.fence, torch.cuda.synchronize)

    modes = ("yuv", "yuv_align", "bgr_net")
    for _ in range(args.warmup):
        for m in modes:
            block(1, m)
    K = args.steps
    if K <= 0:
        K = int(max(bench.CAL_STEPS, np.ceil(bench.MIN_TIMED_S * 1e3 / max(block(bench.CAL_STEPS, "yuv_align") / bench.CAL_STEPS, 1e-4))))
    ms = {}
    for m in modes:
        block(K, m)
        pos[0] = 0
        ms[m] = block(K, m)
    device = {m: dict(ms_per_step=ms[m] / K, frames_per_s=K * B / (ms[m] * 1e-3)) for m in modes}
    device["convert_letterbox_us_per_step"] = (ms["yuv"] - ms["bgr_net"]) / K * 1e3

    # host ingest: blocking calls, so seconds per call is the inverse of host_rate's calls per second
    def host_s(fn, batches):
        it = itertools.cycle(batches)
        return 1 / rates.host_rate(lambda: fn(next(it)), eng.synchronize, args.host_seconds, 1, 1)[0]

    pin = lambda b: [torch.from_numpy(x).pin_memory().numpy() for x in b]  # noqa: E731
    hb = bgr[:2]
    hy = i420[:2]
    host = dict(
        i420_pageable_ms=host_s(lambda b: eng.detect_yuv(b, bench.SCORE_THR, bench.NMS_THR, "i420"), hy) * 1e3,
        i420_pinned_ms=host_s(lambda b: eng.detect_yuv(b, bench.SCORE_THR, bench.NMS_THR, "i420"), [pin(b) for b in hy]) * 1e3,
        bgr_pageable_ms=host_s(lambda b: eng.detect_batch(b, bench.SCORE_THR, bench.NMS_THR), hb) * 1e3,
        bgr_pinned_ms=host_s(lambda b: eng.detect_batch(b, bench.SCORE_THR, bench.NMS_THR), [pin(b) for b in hb]) * 1e3,
        cpu_cvtcolor_i420_to_bgr_ms_per_batch=host_s(lambda b: [cv2.cvtColor(f, cv2.COLOR_YUV2BGR_I420) for f in b], hy) * 1e3)

    # kernel time, profiler on, its own run
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(50):
            eng.detect_yuv_device(dev[i % ring], bench.SCORE_THR, bench.NMS_THR, "nv12")
        eng.synchronize()
    kernel = "k_letterbox_batch<.*YuvPlanes"          # the letter-box instantiated for YUV planes
    us, launches = rates.kernel_us(prof, [kernel])
    us, launches = us[kernel], launches[kernel]
    rd, wr = letterbox_floor_bytes(H, Wd)
    floor_us = B * (rd + wr) / 3.35e12 * 1e6
    eng.close()
    print(json.dumps(dict(workload=bench.DEFAULT_WORKLOAD, frames=f"{FW}x{FH} S-real, NV12 device / I420 host", gpu=rates.card(), steps=K, ring=ring,
                          device=device, host=host,
                          kernel=dict(yuv_letterbox_us_per_launch=us, launches=launches, batch=B, read_bytes_per_frame=rd, write_bytes_per_frame=wr,
                                      floor_us_at_3_35_TBps=floor_us, share_of_floor=floor_us / us if us else None))))


if __name__ == "__main__":
    main()
