#!/usr/bin/env python
"""Cost of f17 searching look-back: lookback_rate.py's eight 1920x1080 NV12 videos, one frame of each per call, batch 8, a 448x448
mnet25 FP16 handle, mosaic + rect, L = --frames.  Prints one JSON line with
  frames/s    plain look-back against searching look-back, alternated rounds of at least --min-seconds each (host clock ended by
              rf_synchronize), on two workloads:
                steady        lookback_rate.py's calls at the benchmark's threshold: faces are born once, then tracked;
                birth_heavy   trackers with max_lost = 2; spans of 3 calls at a threshold no face reaches (1.0) alternate with spans
                              of 3 calls at 0.5, so every face is born again every 6 calls with L buffered frames in which it is visible;
  kernel_us   microseconds per launch, averaged over every launch, of k_lookback_search (and k_lookback_log, _swap, _boxes) over
              the birth-heavy calls, and of k_follow_search on the same frames through a follow tracker, in a separate torch.profiler
              run; search_launches pairs each k_lookback_search launch with its call's chains, its longest chain and whether every
              step of that chain is OK (these frames jump back every 16 calls, so chains stop early); one_chain_us is the launch of
              a call on one video whose faces are born after L frames of 3 px steps, with at least one chain of L OK steps (its
              chains run side by side, so this bounds one such chain from above), against L x k_follow_search;
and the card's name, power limit and maximum SM clock, read in the same command.

    python tools/lookback_search_rate.py [--min-seconds S] [--warmup W] [--rounds R] [--frames L]
"""
import json
import os

import numpy as np

import rates
from rates import bench

W, H, B, FRAMES = 1920, 1080, 8, 16
KERNELS = ("k_lookback_search", "k_lookback_log", "k_lookback_swap", "k_lookback_boxes", "k_follow_search")
SPAN, MAX_LOST = 3, 2
REPEATS = 5


def main():
    ap = rates.args(warmup=20)
    ap.add_argument("--frames", type=int, default=15)
    args = ap.parse_args()
    import cv2
    import torch
    from torch.profiler import ProfilerActivity, profile
    from oracle.yuv import bgr_to_frame
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    out = [f.clone() for f in frames[0]]
    torch.cuda.synchronize()
    weights = os.path.join(bench.GOLD, "weights", "mnet25.caffemodel")
    eng = Engine(weights, 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256, max_image=(H, W))
    L, thr, nms, vids = args.frames, bench.SCORE_THR, bench.NMS_THR, list(range(B))
    trackers = {
        ("steady", "plain"): eng.tracker(max_videos=B, lookback=dict(frames=L)),
        ("steady", "search"): eng.tracker(max_videos=B, lookback=dict(frames=L), lookback_search=True),
        ("birth_heavy", "plain"): eng.tracker(max_videos=B, max_lost=MAX_LOST, lookback=dict(frames=L)),
        ("birth_heavy", "search"): eng.tracker(max_videos=B, max_lost=MAX_LOST, lookback=dict(frames=L), lookback_search=True),
    }
    step = {k: 0 for k in trackers}

    def call(key):
        s = step[key] = step[key] + 1
        t = thr if key[0] == "steady" else (1.0 if (s // SPAN) % 2 == 0 else 0.5)
        trackers[key].detect_yuv_redact_lookback_device(frames[s % FRAMES], vids, out, t, nms)

    def cycle(key):         # the timed unit is one threshold cycle of 2 SPAN calls, so every rate spans whole cycles
        for _ in range(2 * SPAN):
            call(key)
    warmup = -(-max(args.warmup, L + 2 * SPAN + 2) // (2 * SPAN))
    med, per_round, _ = rates.alternate({f"{w}/{k}": lambda key=(w, k): cycle(key) for w, k in trackers}, args.rounds,
                                        lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, warmup, 2 * SPAN * B))
    fol = eng.tracker(max_videos=B, follow=True)
    fol.detect_yuv_device(frames[0], vids, thr, nms)
    key = ("birth_heavy", "search")
    calls = []              # per profiled call: (chains, longest chain, its steps all OK)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(8 * SPAN):
            call(key)
            steps, lens = trackers[key].lookback_search(B)
            i, r = np.unravel_index(int(np.argmax(lens)), lens.shape)
            n = int(lens[i, r])
            calls.append((int((lens > 0).sum()), n, bool(n) and bool((steps[i, r, :n]["status"] == 0).all())))
        for s in range(4 * SPAN):
            fol.follow_device(frames[(s + 1) % FRAMES], vids)
        eng.synchronize()
    kernel_us, _ = rates.kernel_us(prof, KERNELS)
    # one k_lookback_search launch per call (8 frames <= LOOKBACK_SEARCH_FRAMES), in issue order
    search = sorted((ev for ev in prof.events() if "k_lookback_search" in ev.name), key=lambda ev: ev.time_range.start)
    assert len(search) == len(calls), (len(search), len(calls))
    launches = [dict(us=ev.device_time, chains=c, longest=n, longest_all_ok=ok) for ev, (c, n, ok) in zip(search, calls)]
    with_births = [x["us"] for x in launches if x["chains"]]
    # one video whose faces move 3 px per frame, records withheld on its first L frames: each face is born on frame L and its
    # chain has L steps; the launch of that call, repeated after a reset, is the one-chain measurement
    lin_base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W - 3 * (L + 1), H))
    lin = []
    for t in range(L + 1):
        img = np.full((H, W, 3), 128, np.uint8)
        img[:, 3 * t:3 * t + lin_base.shape[1]] = lin_base
        lin.append(torch.from_numpy(bgr_to_frame(img, "nv12")).cuda())
    one = eng.tracker(max_videos=1, lookback=dict(frames=L), lookback_search=True)
    single = []
    for rep in range(REPEATS + 1):           # the first repetition warms up
        one.reset(0)
        for t in range(L):
            one.detect_yuv_redact_lookback_device([lin[t]], [0], [out[0]], 1.0, nms)
        eng.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof1:
            one.detect_yuv_redact_lookback_device([lin[L]], [0], [out[0]], 0.5, nms)
            eng.synchronize()
        steps, lens = one.lookback_search(1)
        full = [r for r in range(lens.shape[1]) if lens[0, r] == L and (steps[0, r, :L]["status"] == 0).all()]
        ev = [e for e in prof1.events() if "k_lookback_search" in e.name]
        if rep:
            single.append(dict(us=ev[0].device_time, chains=int((lens > 0).sum()), full_ok_chains=len(full)))
    one.close()
    full_us = [x["us"] for x in single if x["full_ok_chains"]]
    med = {k: round(v, 1) for k, v in med.items()}
    share = {w: round(med[f"{w}/search"] / med[f"{w}/plain"], 4) for w in ("steady", "birth_heavy")}
    follow_L = L * kernel_us["k_follow_search"] if kernel_us["k_follow_search"] else None
    print(json.dumps(dict(frames_per_s=med, rounds=per_round, search_share=share, L=L, kernel_us=kernel_us, search_launches=launches,
                          search_us_with_births=float(np.mean(with_births)) if with_births else None, one_chain_launches=single,
                          one_chain_us=float(np.mean(full_us)) if full_us else None, L_x_follow_search_us=follow_L,
                          one_chain_over_L_follow=float(np.mean(full_us)) / follow_L if full_us and follow_L else None,
                          gpu=rates.card())))
    for t in list(trackers.values()) + [fol]:
        t.close()
    eng.close()


if __name__ == "__main__":
    main()
