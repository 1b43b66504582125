#!/usr/bin/env python
"""Rate of the arbitrary-size-image path (the reference's RetinaFace::detect on camera frames): 8 x 1280x886 BGR photos per
call through rf_detect_batch (GPU letter-box), from pageable and from pinned caller memory.  Blocking calls, host clock over at
least 0.5 s of calls after warm-up.  Prints one JSON line with the card's name, power limit and maximum SM clock."""
import json
import os
import sys

import numpy as np

import rates
from rates import bench

MIN_S = 0.5


def main():
    import cv2
    import torch
    from retinaface_b200 import RF_PREC_FP16, Engine
    img = cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg"))
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=8, max_faces=128,
                 max_image=(1024, 1280))

    def timed(fn, warmup):
        """Seconds per blocking call of fn() and its last result."""
        last = [None]

        def call():
            last[0] = fn()
        return 1 / rates.host_rate(call, eng.synchronize, MIN_S, warmup, 1)[0], last[0]
    out = {"image": "%dx%d" % (img.shape[1], img.shape[0]), "batch": 8}
    pins = [torch.empty(img.shape, dtype=torch.uint8).pin_memory() for _ in range(8)]
    for t in pins:
        t.numpy()[:] = img
    for name, imgs in (() if "--jpeg-only" in sys.argv else (("pageable", [img.copy() for _ in range(8)]), ("pinned", [t.numpy() for t in pins]))):
        dt, r = timed(lambda: eng.detect_batch(imgs, 0.9, 0.4), 5)
        out[name] = {"ms_per_batch": dt * 1e3, "images_per_s": 8 / dt, "faces_in_image0": int(len(r[0]))}
    # compressed ingest: the same photo as JPEG bitstreams (baseline 4:2:0, quality 90), decoded on the GPU by nvJPEG
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
    streams = [enc.tobytes()] * 8
    try:
        dt, (r, _sz) = timed(lambda: eng.detect_jpeg(streams, 0.9, 0.4), 5)
        out["jpeg"] = {"ms_per_batch": dt * 1e3, "images_per_s": 8 / dt, "faces_in_image0": int(len(r[0])), "bytes_per_image": len(streams[0]),
                       "backend": eng.jpeg_backend()}
        dt, _ = timed(lambda: eng.detect_batch([cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR) for s in streams], 0.9, 0.4), 0)
        out["jpeg_host_decode"] = {"ms_per_batch": dt * 1e3, "images_per_s": 8 / dt, "note": "cv2.imdecode on one host thread + the pixel path (what main.cpp does)"}
    except Exception as e:  # noqa: BLE001
        out["jpeg"] = {"error": str(e)[:200]}
    out["gpu"] = rates.card()
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
