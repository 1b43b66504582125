#!/usr/bin/env python
"""Device-timed step time of the FP16 engine's own plan against RF_FLAG_LEGACY_TC (per-layer kernels only) (development tool):
4 execution contexts (throughput mode) and 1 context (single-step latency: the tile chains), batch 8 and 32.  One process per
configuration."""
import argparse, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def child(legacy, batch, streams):
    import cv2, torch
    from oracle.inputs import letterbox_bgr_u8
    from retinaface_b200 import RF_PREC_FP16, Engine
    from retinaface_b200.capi import RF_FLAG_LEGACY_TC
    img = cv2.imread(os.path.join(ROOT, "tests/golden/data/img.jpg"))
    inp = letterbox_bgr_u8(img, 448, 448)
    ring = 56 if batch <= 8 else 16
    host = np.stack([np.stack([np.roll(inp, 8 * (i + batch * s), axis=1) for i in range(batch)]) for s in range(ring)])
    dev = torch.from_numpy(host).cuda()
    eng = Engine(os.path.join(ROOT, "tests/golden/weights/mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=batch, max_faces=128, streams=streams,
                 flags=RF_FLAG_LEGACY_TC if legacy else 0)
    stream = torch.cuda.ExternalStream(eng.stream_ptr())
    for i in range(30):
        eng.detect_device(batch, 0.9, 0.4, dev[i % ring].data_ptr())
    eng.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    K = 100
    for rep in range(7):
        torch.cuda.synchronize()
        ev0.record(stream)
        for i in range(K):
            eng.detect_device(batch, 0.9, 0.4, dev[(rep * K + i) % ring].data_ptr())
        eng.fence()
        ev1.record(stream)
        torch.cuda.synchronize()
        times.append(ev0.elapsed_time(ev1) / K)
    print(json.dumps(dict(plan="legacy_tc" if legacy else "default", batch=batch, streams=streams, us_per_step=round(float(np.median(times)) * 1e3, 2), launches=eng.launches_per_batch(batch),
                          img_per_s=round(batch / (float(np.median(times)) * 1e-3)))), flush=True)
    eng.close()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--child", default=None)
    ap.add_argument("--batches", default="8,32")
    ap.add_argument("--streams", default="4,1")
    args = ap.parse_args()
    if args.child:
        m, b, s = (int(x) for x in args.child.split(","))
        child(m, b, s)
        sys.exit(0)
    for b in [int(x) for x in args.batches.split(",")]:
        for s in [int(x) for x in args.streams.split(",")]:
            for legacy in (1, 0):
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", f"{legacy},{b},{s}"], capture_output=True, text=True, timeout=300)
                print(r.stdout.strip() or ("ERR " + r.stderr[-400:]), flush=True)
