#!/usr/bin/env python
"""Cost of face alignment on the device path: bench.py's headline workload (mnet25 FP16, batch 8, 448x448, the same S-real input
ring) through rf_detect_align_batch_device -- detect, then a 112x112 RGB float16 ArcFace crop of every kept face written into a
torch device tensor -- against rf_detect_batch_device on the same inputs.  Each rate is one device-timed block (CUDA events,
rf_fence) of K steps, the same K for both, after W warm-up steps and one warm-up block.  Prints one JSON line.

    python tools/align_rate.py [--steps K] [--warmup W] [--streams S]
"""
import argparse
import json
import os

import numpy as np

import rates
from rates import bench


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=0, help="timed steps (0: calibrate to about 0.5 s)")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--streams", type=int, default=0, help="execution contexts (0 = library default)")
    args = ap.parse_args()
    import torch
    from retinaface_b200 import RF_PREC_FP16, Engine
    w = bench.WORKLOADS[bench.DEFAULT_WORKLOAD]
    B, H, Wd = w["batch"], w["h"], w["w"]
    eng = Engine(os.path.join(bench.GOLD, "weights", w["model"] + ".caffemodel"), H, Wd, precision=RF_PREC_FP16, max_batch=B, max_faces=128,
                 streams=args.streams)
    stream = torch.cuda.ExternalStream(eng.stream_ptr())
    ring = max(4, min(256, -(-2 * 50 * 2**20 // (B * H * Wd * 3))))       # input ring > 2 x the H100's L2, as bench.py
    host = bench.make_batches(w, ring, 0)
    dev = torch.from_numpy(host).cuda()
    crops_per_slot = [sum(len(f) for f in eng.detect_batch(list(host[s]), bench.SCORE_THR, bench.NMS_THR)) for s in range(ring)]
    nctx = args.streams or 8
    # one crop tensor per execution context: consecutive (overlapping) steps never write the same buffer
    crops = [torch.empty((B, eng.max_faces, 3, 112, 112), dtype=torch.float16, device="cuda") for _ in range(nctx)]
    pos = [0]

    def step(align):
        s = pos[0] % ring
        if align:
            eng.detect_align_device(B, bench.SCORE_THR, bench.NMS_THR, crops[pos[0] % nctx].data_ptr(), fmt="rgb_f16", dev_ptr=dev[s].data_ptr())
        else:
            eng.detect_device(B, bench.SCORE_THR, bench.NMS_THR, dev[s].data_ptr())
        pos[0] += 1

    def block(k, align):
        return rates.device_ms(lambda: step(align), k, stream, eng.fence, torch.cuda.synchronize)

    for _ in range(args.warmup):
        block(1, True)
        block(1, False)
    K = args.steps
    if K <= 0:
        K = int(max(bench.CAL_STEPS, np.ceil(bench.MIN_TIMED_S * 1e3 / max(block(bench.CAL_STEPS, True) / bench.CAL_STEPS, 1e-4))))
    block(K, True)
    pos[0] = 0
    a_ms = block(K, True)
    pos[0] = 0
    d_ms = block(K, False)
    crops_step = float(np.mean([crops_per_slot[i % ring] for i in range(K)]))
    eng.close()
    print(json.dumps(dict(workload=bench.DEFAULT_WORKLOAD, crop="112x112 RGB float16 (ArcFace template), written to a torch device tensor",
                          gpu=rates.card(), steps=K, images_per_s=K * B / (a_ms * 1e-3), crops_per_s=crops_step * K / (a_ms * 1e-3),
                          ms_per_step=a_ms / K, detect_only=dict(images_per_s=K * B / (d_ms * 1e-3), ms_per_step=d_ms / K),
                          align_us_per_step=(a_ms - d_ms) / K * 1e3,
                          timing="device-timed (CUDA events, rf_fence), rf_detect_align_batch_device vs rf_detect_batch_device, same inputs and K")))


if __name__ == "__main__":
    main()
