"""The FP16 tensor-core engine (RF_PREC_FP16) step by step against its own rounding (oracle/fp16_steps.py), on every kind of
per-layer plan it builds: the benchmarked batch-8 plan, batch 32 with both FPN merges stand-alone, batch 1 with both
fused, 2-D depthwise tiles at stride 1 and 2, the 1-D kernels' geometries on large and tiny maps, the CUDA-core stem, the
second model's weights and the production buffer placement.

Each case forwards a batch of dissimilar neighbours on a handle that keeps every tensor.  Every materialised tensor is
recomputed from its nearest materialised ancestors (the engine's own values) as an interval per element -- one FP16 value
where the kernels spell their arithmetic out, a derived tensor-core bound elsewhere -- and every element must lie inside,
with no allowance for outliers.  The heads' regression and landmark deltas must be bit-exact, the class probabilities
inside their interval, and the detections equal to the oracle post-process of the engine's own heads.
"""
import time
from typing import NamedTuple

import numpy as np
import pytest

from conftest import caffemodel
from oracle import fp16_steps as fs
from oracle.inputs import mixed_batch
from retinaface_b200.capi import RF_FLAG_DW_1D, RF_FLAG_SIMT_STEM

THR, NMS = 0.5, 0.4


class Case(NamedTuple):
    hw: tuple               # network (H, W)
    max_batch: int
    runs: tuple             # batch sizes forwarded one after the other on the same handle
    model: str = "mnet25"
    flags: int = 0
    placement: bool = False  # also run a handle with the production (liveness) buffer placement
    mutate: bool = False     # also apply the mutations of oracle.fp16_steps to one step's engine output
    streams: int = 0         # 1: the latency plans (tile chains for SSH + heads + NMS, and merge + aggr at max_batch <= 2)


CASES = {
    # the benchmarked plan: fused c2 merge, stand-alone c1 merge, 2-D dw3 / dw5, k_head_decode with fused NMS
    "448_mb8": Case((448, 448), 8, (8,), placement=True, mutate=True),
    "448_mb32": Case((448, 448), 32, (32, 5)),                    # both merges stand-alone; persistent runs over many images
    "448_mb1": Case((448, 448), 1, (1,)),                         # both merges fused, smallest grids
    "896x1280_mb3": Case((896, 1280), 3, (3,), placement=True),   # 2-D tiles at stride 2 on C = 16, 32, 64
    "896x1280_mb3_dw1d": Case((896, 1280), 3, (3,), flags=RF_FLAG_DW_1D),   # 1-D geometries on large maps
    "288x416_mb3": Case((288, 416), 3, (3,)),                     # partial 2-D tiles (104 wide)
    "96x160_mb3": Case((96, 160), 3, (3,)),                       # every layer 1-D, SSH taps mostly in the padding
    "32x224_mb4": Case((32, 224), 4, (4,)),                       # 1 x 7 stride-32 map (32 x 32 does not fit the planner)
    "448_mb3_simt_stem": Case((448, 448), 3, (3,), flags=RF_FLAG_SIMT_STEM),
    "deconv_448_mb8": Case((448, 448), 8, (8,), model="mnet-deconv-0517"),
    "latency_448_mb8": Case((448, 448), 8, (8,), streams=1),        # SSH + heads + NMS chains
    "latency_448_mb2": Case((448, 448), 2, (2,), streams=1),        # + merge + aggr chains
    "latency_896x1280_mb8": Case((896, 1280), 8, (3,), streams=1),   # SSH chains without the predictors, streamed weights
}


def plan_steps(case):
    """The case's plan (rf_plan_describe, host-only): its step names and the tile-chain lines."""
    from retinaface_b200.capi import plan_describe
    text = plan_describe(caffemodel(case.model), case.hw[0], case.hw[1], max_batch=case.max_batch, flags=case.flags,
                         streams=case.streams)
    steps = [ln.split(": ", 1)[1] for ln in text.splitlines() if ln.startswith("step lane")]
    chains = [ln for ln in text.splitlines() if ln.startswith("tile_")]
    return steps, chains


def walk_options(steps):
    """What the walk must know of a plan: whether the predictors run in the SSH chains, and the tensors the chains keep in
    shared memory."""
    inner = {"_plus0", "_plus1"}
    for lv in ("c3", "c2", "c1"):
        if any(s.startswith(f"tile_ssh_{lv}") for s in steps):
            inner.update({f"rf_{lv}_det_context_conv1_relu", f"rf_{lv}_det_context_conv3_1_relu"})
    heads = [s.endswith("+heads+decode") for s in steps if s.startswith("tile_ssh_")]
    return len(heads) == 3 and all(heads), inner


def _engine(case, keep_all):
    from retinaface_b200 import RF_PREC_FP16, Engine
    eng = Engine(caffemodel(case.model), case.hw[0], case.hw[1], precision=RF_PREC_FP16, max_batch=case.max_batch,
                 flags=case.flags, streams=case.streams)
    if keep_all:
        eng.debug_keep_all()
    return eng


def first_outside(name, step, got, lo, hi):
    bad = (got < lo) | (got > hi)
    b, c, y, x = np.argwhere(bad)[0]
    return (f"{name} ({step}): first element outside at (image {b}, channel {c}, y {y}, x {x}): engine {got[b, c, y, x]!r}, "
            f"interval [{lo[b, c, y, x]!r}, {hi[b, c, y, x]!r}]; {int(bad.sum())} of {bad.size} elements outside")


def _fetcher(eng, n):
    from retinaface_b200 import RfError

    def fetch(name, _):
        try:
            return eng.debug_tensor(name, n).astype(np.float64)
        except RfError:
            return None
    return fetch


def check_case(case, eng, batch, steps, post, label, options):
    """Every step of one forward inside its interval; returns the per-tensor report lines and the engine's heads."""
    n = len(batch)
    heads = eng.forward_heads(batch)
    compared, missing, diffs, report = [], [], [], []
    chain_heads, inner = options
    for name, step, iv, got in steps.walk(batch, _fetcher(eng, n), simt_stem=bool(case.flags & RF_FLAG_SIMT_STEM),
                                          chain_heads=chain_heads):
        if name.startswith("heads"):
            cls, bbox, lm = iv
            l = {"heads_stride32": 0, "heads_stride16": 1, "heads_stride8": 2}[name]
            one = []
            for what, e, want in (("class probabilities", heads[3 * l], cls), ("bbox", heads[3 * l + 1], bbox),
                                  ("landmarks", heads[3 * l + 2], lm)):
                lo, hi = want if isinstance(want, tuple) else (want, want)     # k_head_decode's deltas: one value
                e = e.astype(float)
                if ((e < lo) | (e > hi)).any():
                    diffs.append(first_outside(f"{name} {what}", step, e, lo, hi))
                one.append(f"{what} {np.mean(lo == hi):.1%}")
            report.append(f"{name} ({step}): inside; one-value intervals: " + ", ".join(one))
            continue
        if got is None:
            missing.append(name)
            continue
        compared.append(name)
        if ((got < iv.lo) | (got > iv.hi)).any():
            diffs.append(first_outside(name, step, got, iv.lo, iv.hi))
            continue
        width = int((fs.f16_ordinal(iv.hi) - fs.f16_ordinal(iv.lo)).max())
        report.append(f"{name}: {np.mean(got == iv.mid):.2%} equal RN16(float64 midpoint), widest interval {width} ulp")
    assert not diffs, (label, diffs)
    # only the FPN sums (fused into the aggr conv's staging) and the tensors inside tile chains may be left unmaterialised
    assert set(missing) <= inner, (label, missing)
    assert len(compared) >= 29 - len(inner), (label, compared)
    found = post.check_engine(eng, batch, heads, THR, NMS, label)
    return report, compared, heads, found


@pytest.fixture(scope="module")
def post_oracle():
    from oracle.postproc import PostprocOracle
    return PostprocOracle()


@pytest.mark.gpu
@pytest.mark.parametrize("case_id", list(CASES))
def test_fp16_engine_inside_its_rounding_intervals(case_id, golden_image, post_oracle):
    case = CASES[case_id]
    h, w = case.hw
    options = walk_options(plan_steps(case)[0])
    steps = fs.Fp16Steps(caffemodel(case.model))
    keep = _engine(case, keep_all=True)
    prod = _engine(case, keep_all=False) if case.placement else None
    try:
        for run, n in enumerate(case.runs):
            label = f"{case_id} n={n}"
            t0 = time.perf_counter()
            batch = mixed_batch(golden_image, n, h, w, start=3 * run)
            report, compared, heads, found = check_case(case, keep, batch, steps, post_oracle, label, options)
            merges = ", ".join(f"_plus{k} {'stand-alone' if f'_plus{k}' in compared else 'fused'}" for k in (0, 1))
            print(f"\n{label}: {len(compared)} tensors inside their intervals ({merges}), {found} faces, "
                  f"{time.perf_counter() - t0:.1f} s")
            for line in report:
                print("   " + line)
            if prod is not None:
                # production placement: tensors share memory across the three lanes; heads bit-equal to the kept handle's
                heads_p = prod.forward_heads(batch)
                for k in range(9):
                    assert np.array_equal(heads_p[k], heads[k]), (label, "liveness placement", k)
            if case.mutate and run == 0:
                _mutations_rejected(keep, batch, steps, n)
    finally:
        keep.close()
        if prod is not None:
            prod.close()


def _mutations_rejected(eng, batch, steps, n):
    """The mutations of oracle.fp16_steps applied to the engine's dw5+pw6 output: the check rejects each on real data."""
    from oracle.fp16_steps import mutations, outside
    x = fs.Iv.exact(eng.debug_tensor("mobilenet0_relu4_fwd", n).astype(np.float64))
    got = eng.debug_tensor("mobilenet0_relu6_fwd", n).astype(np.float64)
    iv = steps.pair(x, 5)
    assert not outside(got, iv).any()
    for name, bad in mutations(x, steps.p["mobilenet0_conv5_fwd"], steps.p["mobilenet0_conv6_fwd"], 1, got):
        assert outside(bad, iv).any(), name
        rel = float(np.abs(bad - got).max() / np.abs(got).max())
        print(f"   mutation '{name}' on the engine's relu6: rejected; the 2e-2-of-max bar "
              f"{'would' if rel >= 2e-2 else 'would NOT'} have caught it ({rel:.2e})")


# ---- host side ----------------------------------------------------------------------------------------------------------
def test_fp16_sweep_covers_every_planner_branch():
    """rf_plan_describe (host-only, 132 SMs assumed) for every case of the sweep: together they must run the tensor-core and
    the CUDA-core stem, the 2-D depthwise+pointwise kernel at stride 2 on C = 16, 32 and 64 and at stride 1, a 1-D depthwise
    step on a map above 56x56, a fused and a stand-alone FPN merge, the fused heads, the SSH chains with and without their
    predictors, and the merge + aggr chains, with both resident and streamed chain weights.  A planner change that moves a
    branch out of the sweep fails here, without a GPU."""
    import re
    stems, s2_channels, s1_2d, big_1d, fused, alone, heads = set(), set(), [], [], [], [], []
    ssh_heads, ssh_alone, merge_chain, weights = [], [], [], set()
    for case_id, case in CASES.items():
        h, w = case.hw
        steps, chains = plan_steps(case)
        for s in steps:
            if "stem_conv0" in s:
                stems.add(s.split("stem")[0])
            if re.fullmatch(r"tc_c\d_upsample\+add\+aggr_.*", s):
                fused.append(case_id)
            if re.fullmatch(r"fpn_merge_plus\d_upsample\+add_h2", s):
                alone.append(case_id)
            if s == "heads_1x1+softmax+decode+nms_all_levels":
                heads.append(case_id)
            if re.fullmatch(r"tile_ssh_c\d\+heads\+decode", s):
                ssh_heads.append(case_id)
            if re.fullmatch(r"tile_ssh_c\d", s):
                ssh_alone.append(case_id)
            if re.fullmatch(r"tile_c\d_merge\+aggr", s):
                merge_chain.append(case_id)
            m = re.fullmatch(r"tc(2d)?_dw(\d+)\+pw\d+_s(\d)_(\d+)to\d+", s)
            if not m:
                continue
            layer, stride, c = int(m.group(2)), int(m.group(3)), int(m.group(4))
            if m.group(1):
                (s2_channels.add(c) if stride == 2 else s1_2d.append(case_id))
            else:
                down = 2 ** (1 + sum(1 for i in (3, 7, 11, 23) if i <= layer))
                if (h // down) * (w // down) > 56 * 56:
                    big_1d.append(case_id)
        for ln in chains:
            m = re.match(r"tile_(ssh_c\d|c\d_merge\+aggr)\S*:.*\((resident|streamed) weights\)", ln)
            if m:
                weights.add(m.group(2))
    assert stems == {"tc_", ""}, stems
    assert {16, 32, 64} <= s2_channels, s2_channels
    assert s1_2d and big_1d and fused and alone and heads, (s1_2d, big_1d, fused, alone, heads)
    assert ssh_heads and ssh_alone and merge_chain, (ssh_heads, ssh_alone, merge_chain)
    assert weights == {"resident", "streamed"}, weights
