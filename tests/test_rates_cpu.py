"""CPU: the rate tools' measurement harness (tools/rates.py) with fakes -- host_rate's order of warm-up, synchronisation and clock,
alternate's round-robin and medians, kernel_us on fake profiler events, card()'s UUID-addressed nvidia-smi query (subprocess.run
patched, nothing run), and the two shared S-real workloads against the inline builders the tools used before."""
import os
import subprocess
from types import SimpleNamespace

import cv2
import numpy as np

from conftest import GOLDEN
from oracle.yuv import bgr_to_frame
from tools import rates


def test_host_rate_syncs_around_the_timed_calls(monkeypatch):
    log, clock = [], [0.0]

    def fake_clock():
        log.append("clock")
        return clock[0]

    def fn():
        log.append("call")
        clock[0] += 0.25
    monkeypatch.setattr(rates, "perf_counter", fake_clock)
    rate, calls = rates.host_rate(fn, lambda: log.append("sync"), 1.0, 2, 8)
    assert calls == 4
    assert rate == 8 * 4 / 1.0
    # warm-up, sync, start the clock; calls until min_s has passed; sync, stop the clock
    assert log == ["call", "call", "sync", "clock"] + ["call", "clock"] * 4 + ["sync", "clock"]


def test_alternate_runs_round_robin_and_takes_medians():
    order, results = [], {"a": iter([(10.0, 1), (30.0, 3), (20.0, 2)]), "b": iter([(5.0, 7), (1.0, 8), (3.0, 9)])}

    def rate(fn):
        order.append(fn)
        return next(results[fn])
    med, per_round, calls = rates.alternate({"a": "a", "b": "b"}, 3, rate)
    assert order == ["a", "b"] * 3
    assert med == {"a": 20.0, "b": 3.0}
    assert per_round == {"a": [10.0, 30.0, 20.0], "b": [5.0, 1.0, 3.0]}
    assert calls == {"a": [1, 3, 2], "b": [7, 8, 9]}


def test_kernel_us_reduces_fake_events():
    ev = lambda name, t: SimpleNamespace(name=name, device_time=t)  # noqa: E731
    prof = SimpleNamespace(events=lambda: [ev("void rf::k_track_update<0>(int)", 2.0), ev("void rf::k_track_update<1>(int)", 4.0),
                                           ev("void rf::k_letterbox_batch<rf::YuvPlanes>(rf::LbBatch<rf::YuvPlanes>)", 7.0),
                                           ev("void rf::k_letterbox_batch<rf::Bgr>(rf::LbBatch<rf::Bgr>)", 1.0)])
    us, launches = rates.kernel_us(prof, ["k_track_update", "k_letterbox_batch<.*YuvPlanes", "k_best_emit"])
    assert us == {"k_track_update": 3.0, "k_letterbox_batch<.*YuvPlanes": 7.0, "k_best_emit": None}
    assert launches == {"k_track_update": 2, "k_letterbox_batch<.*YuvPlanes": 1, "k_best_emit": 0}


def _fake_device(monkeypatch, uuid):
    import torch
    monkeypatch.setattr(torch.cuda, "get_device_properties", lambda i: SimpleNamespace(uuid=uuid))


def test_card_queries_the_device_by_uuid(monkeypatch):
    _fake_device(monkeypatch, "5f0c6a2e-1d3b-4c8e-9a7f-0123456789ab")
    calls = []

    def run(cmd, **kw):
        calls.append(cmd)
        return SimpleNamespace(returncode=0, stdout="NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n")
    monkeypatch.setattr(subprocess, "run", run)
    assert rates.card() == "NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz"
    assert calls == [["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                      "GPU-5f0c6a2e-1d3b-4c8e-9a7f-0123456789ab"]]


def test_card_falls_back_to_index_0_and_says_so(monkeypatch):
    _fake_device(monkeypatch, "5f0c6a2e-1d3b-4c8e-9a7f-0123456789ab")
    calls = []

    def run(cmd, **kw):
        calls.append(cmd)
        if cmd[-1].startswith("GPU-"):
            return SimpleNamespace(returncode=6, stdout="No devices were found\n")
        return SimpleNamespace(returncode=0, stdout="NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz\n")
    monkeypatch.setattr(subprocess, "run", run)
    line = rates.card()
    assert line.startswith("NVIDIA H100 80GB HBM3, 700.00 W, 1980 MHz") and "GPU 0" in line and "UUID" in line
    assert [c[-1] for c in calls] == ["GPU-5f0c6a2e-1d3b-4c8e-9a7f-0123456789ab", "0"]


def test_videos_1080p_is_the_tools_inline_video():
    B, FRAMES, W, H = 3, 4, 1920, 1080
    base = cv2.resize(cv2.imread(os.path.join(GOLDEN, "data", "img.jpg")), (W - 7 * FRAMES, H))
    want = []
    for t in range(FRAMES):
        img = np.full((H, W, 3), 128, np.uint8)
        img[:, 7 * t:7 * t + base.shape[1]] = base
        want.append([bgr_to_frame(np.roll(img, 8 * i, axis=1), "nv12") for i in range(B)])
    got = rates.videos_1080p(B, FRAMES)
    assert len(got) == FRAMES and all(len(f) == B for f in got)
    for gf, wf in zip(got, want):
        for g, w in zip(gf, wf):
            assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes()


def test_golden_4k_is_the_tools_inline_batch():
    B = 2
    for W, H in ((3840, 2160), (1920, 1080)):
        base = cv2.resize(cv2.imread(os.path.join(GOLDEN, "data", "img.jpg")), (W, H))
        got = rates.golden_4k(B, W, H)
        assert len(got) == B
        for i, g in enumerate(got):
            w = np.roll(base, 8 * i, axis=1)
            assert g.dtype == w.dtype and g.shape == w.shape and g.tobytes() == w.tobytes()
    assert rates.golden_4k(1)[0].shape == (2160, 3840, 3)
