"""Host-only guards of the NMS load sweep (tests/test_gpu_nms_load.py): its candidate-count targets straddle every branch
boundary of nms_image as compiled, its plans still hold each NMS instantiation they are there for (rf_plan_describe), and the threshold
picker lands on exact counts through ties."""
import os

import numpy as np
import pytest

from conftest import caffemodel
from nms_load import ALL, MAX_FACES, PLANS, nms_constants, nms_variant, pick_threshold, regime, regimes, targets

TABLE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "weights", "mnet-deconv-0517.table.int8")


def test_targets_straddle_every_branch_boundary():
    c = nms_constants()
    assert c["NMS_MASK_MAX"] < c["NMS_RANK_MAX"] < c["NMS_SMEM_CAP"]
    ts = targets()
    assert ts[-1] is ALL
    for name in ("NMS_MASK_MAX", "NMS_RANK_MAX", "NMS_SMEM_CAP"):
        v = c[name]
        assert v in ts and v + 1 in ts and regime(v) != regime(v + 1), name
    assert [regime(t) for t in ts[:-1]] == ["rows", "rank+rounds", "rank+rounds", "bitonic", "bitonic", "bitonic-global"]
    # the 64-bit rows of the smallest branch: one bit per later candidate
    assert c["NMS_MASK_MAX"] == 64
    # every plan's anchor count reaches the global-scratch branch at "every anchor"
    for name, p in PLANS.items():
        assert regime(p.anchors) == "bitonic-global", name


def _describe(plan, max_faces):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8
    from retinaface_b200.capi import plan_describe
    prec = {"fp32": RF_PREC_FP32, "fp16": RF_PREC_FP16, "int8": RF_PREC_INT8}[plan.prec]
    return plan_describe(caffemodel(plan.model), plan.hw[0], plan.hw[1], precision=prec, max_batch=plan.max_batch,
                         int8_table=TABLE if plan.prec == "int8" else None, streams=plan.streams, max_faces=max_faces)


@pytest.mark.parametrize("name", list(PLANS))
def test_sweep_plans_hold_their_nms_instantiation(name):
    """Each plan of the sweep holds the NMS instantiation it is there for, at the default max_faces and the small one.  The sweep
    also runs max_faces 8192: there a latency plan's SSH chains may no longer have room for the last-block NMS's kept list; the
    GPU test asserts whatever this reports."""
    plan = PLANS[name]
    text = _describe(plan, 256)
    assert nms_variant(text) == plan.nms, (name, text)
    steps = [ln.split(": ", 1)[1] for ln in text.splitlines() if ln.startswith("step lane")]
    if plan.nms == "fused":
        tail = steps[-1]
        assert tail == ("i8_" if plan.prec == "int8" else "") + "heads_1x1+softmax+decode+nms_all_levels", steps
    assert nms_variant(_describe(plan, 4)) == plan.nms, name
    print(f"{name}: max_faces 8192 -> {nms_variant(_describe(plan, 8192))}")


def test_sweep_covers_the_three_instantiations():
    """k_nms (rf_postprocess, which every plan of the sweep runs), the last block of k_head_decode for float, half and int8
    features, and the last CTA of the SSH tile chains, at 448^2 and at a size with partial chain tiles and the global scratch."""
    kinds = {(p.nms, p.prec) for p in PLANS.values()}
    assert {("fused", "fp32"), ("fused", "fp16"), ("fused", "int8"), ("chain", "fp16")} <= kinds
    assert {p.hw for p in PLANS.values() if p.nms == "chain"} >= {(448, 448), (416, 288)}
    assert {p.hw for p in PLANS.values() if p.nms == "fused" and p.prec == "fp16"} >= {(448, 448), (896, 1280)}
    assert {p.max_batch for p in PLANS.values() if p.nms == "chain" and p.hw == (448, 448)} == {2, 8}


def test_latency_plan_keeps_its_fused_nms_up_to():
    """The largest max_faces (powers of two up to 8192) at which the 448^2 latency plan still runs its NMS in the SSH chains:
    the chains reserve sizeof(NmsSmem) + 4 max_faces bytes of shared memory for it.  Recorded here so that a change to the
    chains' shared-memory layout that moves it shows up."""
    plan = PLANS["fp16_448_latency_b8"]
    fused = [mf for mf in (256, 512, 1024, 2048, 4096, 8192) if nms_variant(_describe(plan, mf)) == "chain"]
    print(f"448^2 latency plan: NMS in the SSH chains up to max_faces {max(fused)}")
    assert fused and fused == [256, 512, 1024, 2048, 4096, 8192][:len(fused)]
    assert max(fused) >= 256


def test_threshold_picker_through_ties():
    p = np.array([0.9, 0.8, 0.8, 0.8, 0.5, 0.3, 0.3, 0.1], np.float32)
    assert pick_threshold(p, 1) == (np.float32(0.8), 1)
    assert pick_threshold(p, 0) == (np.float32(0.9), 0)
    # 2 and 3 sit inside the tie at 0.8: the nearest untied counts are 1 and 4; 2 steps down, 3 up
    assert pick_threshold(p, 2) == (np.float32(0.8), 1)
    assert pick_threshold(p, 3) == (np.float32(0.5), 4)
    # kept inside a range: 2 within [2, 8] must go up to 4
    assert pick_threshold(p, 2, 2, 8) == (np.float32(0.5), 4)
    assert pick_threshold(p, 6, 6, 7) == (np.float32(0.1), 7)
    assert pick_threshold(p, 8) == (np.float32(-1.0), 8)
    assert pick_threshold(p, ALL) == (np.float32(-1.0), 8)
    with pytest.raises(ValueError):
        pick_threshold(p, 2, 2, 3)
    # a flat image: every score equal -> only 0 or all
    flat = np.full(100, 0.25, np.float32)
    assert pick_threshold(flat, 60) == (np.float32(-1.0), 100)
    assert pick_threshold(flat, 40) == (np.float32(0.25), 0)
    with pytest.raises(ValueError):
        pick_threshold(flat, 10, 1, 64)
    # random scores with many exact duplicates: the count is exact and the picked k is the nearest untied one
    rng = np.random.default_rng(3)
    q = rng.integers(0, 50, 3000).astype(np.float32) / 64
    for k in (64, 65, 256, 257, 1024, 1025):
        thr, kk = pick_threshold(q, k)
        assert (q > thr).sum() == kk
        s = np.sort(q)[::-1]
        untied = [j for j in range(len(q) + 1) if j in (0, len(q)) or s[j - 1] > s[j]]
        assert abs(kk - k) == min(abs(j - k) for j in untied)
    assert [name for name, _, _ in regimes()] == ["rows", "rank+rounds", "bitonic", "bitonic-global"]
