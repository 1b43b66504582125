"""The measurement harness of the rate tools (tools/*_rate.py): their common options, the host-clock rate loop, alternated rounds
and their medians, the CUDA-event block timer, the torch.profiler reduction per kernel, the card line printed beside every number,
and the two S-real workloads several tools share.  Importing it puts the repository root on sys.path."""
import argparse
import os
import re
import subprocess
import sys
from time import perf_counter

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def args(parser=None, *, warmup=3, rounds=3, min_seconds=0.5):
    """`parser` (a new one by default) with --min-seconds, --warmup and --rounds at the tool's defaults."""
    parser = parser or argparse.ArgumentParser()
    parser.add_argument("--min-seconds", type=float, default=min_seconds)
    parser.add_argument("--warmup", type=int, default=warmup)
    parser.add_argument("--rounds", type=int, default=rounds)
    return parser


def host_rate(fn, sync, min_s, warmup, per_call):
    """(items per second, calls) of fn(), per_call items a call: `warmup` calls, sync(), then calls until min_s has passed on the
    host clock, ended by sync().  A launch returns before its work ends, so the clock stops after the closing sync()."""
    for _ in range(warmup):
        fn()
    sync()
    calls, t0 = 0, perf_counter()
    while True:
        fn()
        calls += 1
        if perf_counter() - t0 >= min_s:
            break
    sync()
    return per_call * calls / (perf_counter() - t0), calls


def alternate(runs, rounds, rate):
    """Times every variant of `runs` (name -> call) once per round, in dict order, with rate(call) -> (rate, calls), so that
    drift on a shared host falls on every variant alike.  Returns three dicts by name: the median rate, the per-round rates and
    the per-round call counts."""
    got = {name: [] for name in runs}
    for _ in range(rounds):
        for name, fn in runs.items():
            got[name].append(rate(fn))
    per_round = {name: [r for r, _ in v] for name, v in got.items()}
    return ({name: float(np.median(v)) for name, v in per_round.items()}, per_round,
            {name: [k for _, k in v] for name, v in got.items()})


def device_ms(fn, k, stream, fence, sync):
    """Device milliseconds of k calls of fn(): sync(), an event on `stream`, the calls, fence() (which orders the library's
    execution contexts onto its stream), a second event, sync()."""
    import torch
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sync()
    ev0.record(stream)
    for _ in range(k):
        fn()
    fence()
    ev1.record(stream)
    sync()
    return ev0.elapsed_time(ev1)


def kernel_us(prof, names):
    """Two dicts by name, over the kernels of a torch.profiler run whose name it matches (re.search: a plain kernel name matches
    every instantiation): the mean device microseconds per launch (None for a kernel that did not run) and the number of launches."""
    us, launches = {}, {}
    for name in names:
        t = [e.device_time for e in prof.events() if re.search(name, e.name)]
        us[name], launches[name] = float(np.mean(t)) if t else None, len(t)
    return us, launches


def card():
    """One CSV line, `name, power.limit, clocks.max.sm`, of the device the run used.  nvidia-smi numbers the physical GPUs and
    ignores CUDA_VISIBLE_DEVICES, so the query names torch's device 0 by its UUID; if that query fails it falls back to index 0
    and the line says so."""
    import torch
    query = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i"]
    r = subprocess.run(query + [f"GPU-{torch.cuda.get_device_properties(0).uuid}"], capture_output=True, text=True)
    if r.returncode == 0 and r.stdout.strip():
        return r.stdout.strip()
    r = subprocess.run(query + ["0"], capture_output=True, text=True)
    return f"{r.stdout.strip()} (physical GPU 0: the query by UUID failed)"


def videos_1080p(B, frames):
    """The S-real video of the tracker tools, host NV12 BT.601 arrays indexed [frame][video]: B 1920x1080 videos of `frames`
    frames, the golden photo resized to (1920 - 7 frames) x 1080 on a grey canvas and moved 7 px right per frame, video i rolled
    by 8 i columns."""
    import cv2
    from oracle.yuv import bgr_to_frame
    W, H = 1920, 1080
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W - 7 * frames, H))
    out = []
    for t in range(frames):
        img = np.full((H, W, 3), 128, np.uint8)
        img[:, 7 * t:7 * t + base.shape[1]] = base
        out.append([bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12") for i in range(B)])
    return out


def golden_4k(B, W=3840, H=2160):
    """The S-real batch of the tiled tools, host BGR arrays: the golden photo resized to W x H, image i rolled by 8 i columns."""
    import cv2
    base = cv2.resize(cv2.imread(os.path.join(bench.GOLD, "data", "img.jpg")), (W, H))
    return [np.roll(base, 8 * i, axis=1) for i in range(B)]
