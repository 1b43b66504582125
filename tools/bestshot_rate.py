#!/usr/bin/env python
"""Cost of f11 best shots on device-resident video: tools/track_rate.py's workload (eight 1920x1080 NV12 BT.601 videos on the device,
the golden photo resized to 1080p, video i rolled by 8 i columns and moved 7 px per frame; one frame of each per call, batch 8, a
448x448 mnet25 FP16 handle with the default execution contexts).  Prints one JSON line with
  frames/s    of rf_detect_yuv_batch_device (detect), rf_detect_yuv_track_device (detect + track), the same with 112x112 crops of the
              new identities (detect + track + crops) and rf_detect_yuv_track_best_device with 112x112 u8 best shots (detect + track
              + best): warmed up, --rounds alternated rounds of at least --min-seconds of back-to-back calls each, the host clock ended
              by rf_synchronize;
  kernel_us   microseconds per launch of k_track_update and of each k_best_* kernel, in a separate torch.profiler run (CUPTI's
              device timestamps), and the mean faces per frame;
and the card's name, power limit and maximum SM clock, read in the same command.  The videos loop over 16 frames, so tracks live on
and the best-shot store is exercised on every frame; best_cost is 1 - (detect + track + best) / (detect + track).
f22 adds the modes best+live (live shots at their defaults), best k=3 and best k=5 (a following best-shot tracker: every video's
frames detected every k-th call, followed by rf_track_follow_best_device in between) and follow k=3 (f16's follow tracker on the same
split); live_ratio (best+live over best), interval_speedup (best k=3 over best); and kernel_us_live / kernel_us_follow, the
microseconds per launch of k_best_select on the live tracker and of k_best_select / k_follow_update on the k = 3 following one, each
in its own profiler run.

    python tools/bestshot_rate.py [--min-seconds S] [--warmup W] [--rounds R]
"""
import json
import os

import numpy as np

import rates
from rates import bench

B, FRAMES = 8, 16
KERNELS = ("k_track_update", "k_best_measure", "k_best_select", "k_best_emit", "k_best_commit")
FOLLOW_KERNELS = ("k_best_select", "k_follow_update", "k_follow_search")


def main():
    args = rates.args(warmup=10).parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from retinaface_b200 import RF_PREC_FP16, Engine
    frames = [[torch.from_numpy(f).cuda() for f in fr] for fr in rates.videos_1080p(B, FRAMES)]
    eng = Engine(os.path.join(bench.GOLD, "weights", "mnet25.caffemodel"), 448, 448, precision=RF_PREC_FP16, max_batch=B, max_faces=256,
                 max_image=(1080, 1920))
    trk = eng.tracker(max_videos=B)
    best = eng.tracker(max_videos=B, best=dict())
    live = eng.tracker(max_videos=B, best=dict(), best_live=True)
    bf = {k: eng.tracker(max_videos=B, best=dict(), best_follow=True) for k in (3, 5)}
    fol = eng.tracker(max_videos=B, follow=True)
    crops = torch.empty((B, 8, 112, 112, 3), dtype=torch.uint8, device="cuda")
    shots = torch.empty((B, best.max_tracks, 112, 112, 3), dtype=torch.uint8, device="cuda")
    thr, nms = bench.SCORE_THR, bench.NMS_THR
    vids = list(range(B))
    step = [0]

    def nxt():
        step[0] += 1
        return frames[step[0] % FRAMES]

    def interval(t, k, with_best):
        """One call of tracker t's own count: every video's next frame, detected on every k-th call and followed otherwise."""
        n = [0]

        def call():
            det = n[0] % k == 0
            n[0] += 1
            if with_best:
                return t.detect_yuv_best_device(nxt(), vids, thr, nms, shots.data_ptr()) if det else t.follow_best_device(nxt(), vids, shots.data_ptr())
            return t.detect_yuv_device(nxt(), vids, thr, nms) if det else t.follow_device(nxt(), vids)
        return call
    runs = {
        "detect": lambda: eng.detect_yuv_device(nxt(), thr, nms),
        "detect+track": lambda: trk.detect_yuv_device(nxt(), vids, thr, nms),
        "detect+track+crops": lambda: trk.detect_yuv_device(nxt(), vids, thr, nms, align=dict(max_faces=8), dev_crops_ptr=crops.data_ptr()),
        "detect+track+best": lambda: best.detect_yuv_best_device(nxt(), vids, thr, nms, shots.data_ptr()),
        "best+live": lambda: live.detect_yuv_best_device(nxt(), vids, thr, nms, shots.data_ptr()),
        "best k=3": interval(bf[3], 3, True),
        "best k=5": interval(bf[5], 5, True),
        "follow k=3": interval(fol, 3, False),
    }
    med, per_round, _ = rates.alternate(runs, args.rounds, lambda fn: rates.host_rate(fn, eng.synchronize, args.min_seconds, args.warmup, B))
    d, c, _ = eng.detect_yuv_device(frames[0], thr, nms)
    faces = float(np.mean([len(f) for f in eng.read_dets(d, c, B)[0]]))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            runs["detect+track+best"]()
        eng.synchronize()
    us, launches = rates.kernel_us(prof, KERNELS)
    extra = {}
    for name, mode, kernels in (("live", "best+live", ("k_best_select",)), ("follow", "best k=3", FOLLOW_KERNELS)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(60):
                runs[mode]()
            eng.synchronize()
        extra[name] = rates.kernel_us(prof, kernels)
    med = {k: round(v, 1) for k, v in med.items()}
    r2 = lambda d: {k: None if t is None else round(t, 2) for k, t in d.items()}     # noqa: E731
    print(json.dumps(dict(frames_per_s=med, rounds=per_round, best_cost=round(1 - med["detect+track+best"] / med["detect+track"], 4),
                          kernel_us=r2(us), launches=launches, faces_per_frame=faces,
                          live_ratio=round(med["best+live"] / med["detect+track+best"], 4),
                          interval_speedup=round(med["best k=3"] / med["detect+track+best"], 4),
                          kernel_us_live=r2(extra["live"][0]), kernel_us_follow=r2(extra["follow"][0]), gpu=rates.card())))
    for t in (live, fol, *bf.values()):
        t.close()
    best.close()
    trk.close()
    eng.close()


if __name__ == "__main__":
    main()
