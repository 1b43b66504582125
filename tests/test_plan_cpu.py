"""rf_plan_describe (host-only) over a grid of configurations, against the plans the per-precision builders made before the
layer plans were built from one walk of the network (tests/golden/plans/describe.json.gz).  Every step name, lane, launch count,
activation-arena size and tile-chain line must stay as it was, except for the changes that came with the single walk:

- the per-layer fallback of the FP16 tile-chain plan names its lateral convolutions as the other per-layer plans do;
- the SIMT plans (FP32, FP16 with RF_FLAG_NO_TENSORCORE) run rf_c1_red_conv and rf_c2_lateral right after the pointwise layer
  that produces their input (pw10, pw22) instead of after the backbone;
- RF_FLAG_LEGACY_TC builds the FP16 plan with no tile chains.

The fixture was written by running this module as a script against a library built from commit 23f7863, the last one with
a builder per precision: RF_B200_LIB=<that library> python tests/test_plan_cpu.py --write.  Its grid then also held the
plans selected by the RF_TILE_* environment variables, which no longer exist; a one-off filter has since dropped those
configurations (and the texts only they referenced) and the key suffix that named the variables' values."""
import gzip
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
FIXTURE = os.path.join(ROOT, "tests", "golden", "plans", "describe.json.gz")
WEIGHTS = os.path.join(ROOT, "tests", "golden", "weights")
TABLE = os.path.join(WEIGHTS, "mnet-deconv-0517.table.int8")

FP32, FP16, INT8 = 0, 1, 2
NO_TC, SIMT_STEM, DW_1D, LEGACY_TC = 0x2, 0x4, 0x8, 0x10
MODELS = ("mnet25", "mnet-deconv-0517")
SIZES = ((448, 448), (896, 1280), (288, 416), (320, 320), (96, 160))      # (net_h, net_w)
BATCHES = (1, 3, 8, 32)


def grid():
    """(key, model, precision, h, w, batch, flags, streams).  Streams matter only to the FP16 tensor-core plan; the flags
    only where a plan reads them."""
    for model in MODELS:
        for h, w in SIZES:
            for b in BATCHES:
                cases = [(FP32, 0, 0)]
                cases += [(FP16, f, 0) for f in (NO_TC, SIMT_STEM, DW_1D)]
                cases += [(FP16, 0, s) for s in (1, 0)]
                cases += [(INT8, f, 0) for f in (0, SIMT_STEM, DW_1D)]
                for prec, flags, streams in cases:
                    yield f"{model} p{prec} {h}x{w} b{b} f{flags} s{streams}", model, prec, h, w, b, flags, streams


def describe(model, prec, h, w, b, flags, streams):
    from retinaface_b200.capi import RfError, plan_describe
    try:
        return plan_describe(os.path.join(WEIGHTS, model + ".caffemodel"), h, w, precision=prec, max_batch=b, flags=flags,
                             int8_table=TABLE if prec == INT8 else None, streams=streams)
    except RfError as e:
        return f"error {e.status}"


def move_after(lines, name, producer):
    """moves the step line ending in `name` to just after the step line starting with the pointwise step `producer`"""
    i = next(k for k, ln in enumerate(lines) if ln.endswith(": " + name))
    line = lines.pop(i)
    j = next(k for k, ln in enumerate(lines) if ln.startswith("step lane 0: " + producer))
    lines.insert(j + 1, line)


def expected(text, prec, flags):
    """the parent's text with the intended changes applied"""
    for old, new in (("tc_rf_c1_red_conv_1x1", "tc_c1_red_1x1_64to64"), ("tc_rf_c2_lateral_1x1", "tc_c2_lateral_1x1_128to64"),
                     ("tc_rf_c3_lateral_1x1", "tc_c3_lateral_1x1_256to64")):
        text = text.replace(": " + old + "\n", ": " + new + "\n")
    if prec == FP32 or (prec == FP16 and flags & NO_TC):
        lines = text.split("\n")
        move_after(lines, "c1_red_1x1_64to64", "pw10_")
        move_after(lines, "c2_lateral_1x1_128to64", "pw22_")
        text = "\n".join(lines)
    return text


@pytest.fixture(scope="module")
def fixture(built_lib):
    with gzip.open(FIXTURE, "rt") as f:
        return json.load(f)


def test_plans_equal_the_parent_builders_but_for_the_intended_changes(fixture):
    texts, plans = fixture["texts"], fixture["plans"]
    assert len(plans) == sum(1 for _ in grid())
    for key, model, prec, h, w, b, flags, streams in grid():
        got = describe(model, prec, h, w, b, flags, streams)
        assert got == expected(texts[plans[key]], prec, flags), key
    # the grid reaches every builder and every merge rule
    joined = "\n".join(texts[plans[key]] for key, *_ in grid())
    for step in ("upsample_add_plus1", "tc_c1_upsample+add+aggr", "fpn_merge_plus1_upsample+add_h2", "fpn_merge_plus0_upsample+add_h2",
                 "i8_c1_upsample+add+aggr", "i8_fpn_merge_c1_upsample+add", "tile_c1_merge+aggr", "tile_ssh_c1+heads+decode",
                 "i8_2d_dw3", "tc2d_dw3", "stem_conv0+dw1+pw2_u8_to_16ch_i8", "tc_rf_c1_red_conv_1x1"):
        assert step in joined, step


def test_legacy_tc_is_the_fp16_plan_without_tile_chains(built_lib):
    """RF_FLAG_LEGACY_TC on a one-context handle (where the chains would run) builds the several-context plan."""
    for model in MODELS:
        for h, w in SIZES:
            for b in BATCHES:
                assert describe(model, FP16, h, w, b, LEGACY_TC, 1) == describe(model, FP16, h, w, b, 0, 0), (model, h, w, b)


if __name__ == "__main__" and "--write" in sys.argv:
    texts, index, plans = [], {}, {}
    for key, *cfg in grid():
        text = describe(*cfg)
        plans[key] = index.setdefault(text, len(texts))
        if plans[key] == len(texts):
            texts.append(text)
    os.makedirs(os.path.dirname(FIXTURE), exist_ok=True)
    with open(FIXTURE, "wb") as f:
        f.write(gzip.compress(json.dumps({"texts": texts, "plans": plans}, indent=0).encode() + b"\n", 9, mtime=0))
    print(f"{len(plans)} configurations, {len(texts)} distinct plans -> {FIXTURE}")
