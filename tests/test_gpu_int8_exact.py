"""The INT8 engine (RF_PREC_INT8) bit for bit against its integer oracle (oracle/mnet_int8.py), on every kind of plan
build_plan_i8 makes: the benchmarked batch-32 plan with its stand-alone FPN merge, the fused merge, 2-D depthwise tiles at
stride 1 and 2, the 1-D kernels' geometries on large and tiny maps, the CUDA-core stem, a table that saturates every
epilogue's clamp, the second model's weights, and the production buffer placement.

Each GPU case forwards a batch of dissimilar neighbours on a handle that keeps every tensor, checks the FP32 stem within
1 LSB, continues the oracle from the engine's own stem and compares every int8 tensor the handle materialises with
np.array_equal, the nine head blobs within 1e-4, and the detections (selection and order exact) with the oracle
post-process of the engine's own heads.  The host-side guard at the end checks that the sweep's plans still cover every
branch of the planner it was written for.
"""
import os
import re
import struct
import time
from typing import NamedTuple

import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle import topology
from oracle.inputs import letterbox_bgr_u8, mixed_batch
from oracle.mnet_int8 import Int8Oracle, int_gemm, read_table
from retinaface_b200.capi import RF_FLAG_DW_1D, RF_FLAG_SIMT_STEM, RF_PREC_INT8

MODEL = "mnet-deconv-0517"
SHIPPED_TABLE = os.path.join(GOLDEN, "weights", MODEL + ".table.int8")
STEM = "mobilenet0_relu2_fwd"
THR, NMS = 0.5, 0.4


class Case(NamedTuple):
    hw: tuple               # network (H, W)
    max_batch: int
    runs: tuple             # batch sizes forwarded one after the other on the same handle
    model: str = MODEL
    table: str = "shipped"  # "shipped", "saturating" (every scale x 0.25) or "absmax" (made from the FP32 oracle)
    flags: int = 0
    placement: bool = False  # also run a handle with the production (liveness) buffer placement
    faces: bool = True      # the batch yields faces at THR (none when saturated, nor at 96x160)


CASES = {
    # the benchmarked plan: stand-alone k_fpn_merge_i8, persistent stem runs across many image boundaries, then n < max_batch
    "448_mb32": Case((448, 448), 32, (32, 5), placement=True),
    "448_mb8_saturating": Case((448, 448), 8, (8,), table="saturating", faces=False),
    "448_mb1": Case((448, 448), 1, (1,)),                         # fused merge, smallest grid
    "896x1280_mb3": Case((896, 1280), 3, (3,), placement=True),   # 2-D tiles at stride 2 on C = 16, 32, 64
    "896x1280_mb3_dw1d": Case((896, 1280), 3, (3,), flags=RF_FLAG_DW_1D),   # 1-D row / N-split geometries on large maps
    "288x416_mb3": Case((288, 416), 3, (3,)),                     # partial 2-D tiles (104 wide), 9x13 stride-32 map
    "96x160_mb3": Case((96, 160), 3, (3,), faces=False),          # every layer 1-D, SSH taps mostly in the padding
    "32_mb4": Case((32, 32), 4, (4,), faces=False),               # smallest network: 1 x 1 stride-32 map
    "320_mb32": Case((320, 320), 32, (3,)),                       # stand-alone merge at a second geometry
    "448_mb3_simt_stem": Case((448, 448), 3, (3,), flags=RF_FLAG_SIMT_STEM),
    "mnet25_448_mb8": Case((448, 448), 8, (8,), model="mnet25", table="absmax"),
}

# The saturating case's proof that the clamps ran: the fraction of each named oracle tensor at +127 on its batch must reach
# the floor (measured on the CPU with the oracle's own stem: relu2 26 %, concats 8.7 / 18 / 23 %, _plus1 6.1 %, _plus0
# 1.4 %), and at least SATURATED_TENSORS of the 29 quantised tensors must reach +127 somewhere (26 do; relu24, c2_lateral and
# c3 context_conv3_1 stay below).  Every tensor is post-ReLU, so -127 is never reached and is not claimed.
SATURATION_FLOOR = {STEM: 0.15, "rf_c3_det_concat_relu": 0.04, "rf_c2_det_concat_relu": 0.1, "rf_c1_det_concat_relu": 0.1,
                    "_plus1": 0.03, "_plus0": 0.007}
SATURATED_TENSORS = 24


# ---- tables -------------------------------------------------------------------------------------------------------------
def write_table(path, scales):
    """TensorRT's EntropyCalibration2 cache format: '<tensor>: <big-endian float32 hex>' per line."""
    with open(path, "w") as f:
        f.write("TRT-5102-EntropyCalibration2\n")
        for k, v in scales.items():
            f.write(f"{k}: {struct.pack('>f', v).hex()}\n")
    return path


def quantised_tensor_names():
    """Every tensor the INT8 plan quantises (and so looks up in the table): each ReLU output and each FPN sum."""
    names = []
    for op in topology.ops():
        if op["op"] == "conv" and op["relu"]:
            names.append(op["relu"])
        elif op["op"] in ("relu", "add"):
            names.append(op["name"])
    return names


def absmax_table(path, model, photo, h=448, w=448):
    """A table for a model without a shipped one, deterministic and independent of rf_calibrate_int8: absmax / 127 of each
    quantised tensor of the FP32 oracle on the golden photo."""
    from oracle.mnet_numpy import MnetOracle, preprocess_bgr_u8
    names = quantised_tensor_names()
    act = MnetOracle(caffemodel(model)).forward(preprocess_bgr_u8(letterbox_bgr_u8(photo, h, w)), want=names)
    scales = {"data": float(np.float32(255.0 / 127.0))}
    scales.update({k: float(np.float32(np.abs(act[k]).max()) / np.float32(127)) for k in names})
    return write_table(path, scales)


@pytest.fixture(scope="module")
def tables(tmp_path_factory, golden_image):
    d = tmp_path_factory.mktemp("int8_tables")
    shipped = read_table(SHIPPED_TABLE)
    return {"shipped": SHIPPED_TABLE,
            "saturating": write_table(str(d / "saturating.table.int8"), {k: v * 0.25 for k, v in shipped.items()}),
            "absmax": absmax_table(str(d / "mnet25.table.int8"), "mnet25", golden_image)}


def _engine(case, table, keep_all):
    from retinaface_b200 import Engine
    eng = Engine(caffemodel(case.model), case.hw[0], case.hw[1], precision=RF_PREC_INT8, max_batch=case.max_batch,
                 int8_table=table, flags=case.flags)
    if keep_all:
        eng.debug_keep_all()
    return eng


# ---- comparisons ------------------------------------------------------------------------------------------------------
def first_difference(name, got, want):
    bad = got != want
    b, c, y, x = np.argwhere(bad)[0]
    return (f"{name}: first difference at (image {b}, channel {c}, y {y}, x {x}): engine {got[b, c, y, x]:.0f}, oracle "
            f"{want[b, c, y, x]}; {bad.mean():.4%} of the bytes differ")


_ATTEMPTED, _MERGE = set(), {}


@pytest.fixture(scope="module")
def post_oracle():
    from oracle.postproc import PostprocOracle
    return PostprocOracle()


def check_forward(keep, oracle, batch, post, label):
    """One forward of `batch` on the keep-all handle against the integer oracle: the FP32 stem within 1 LSB, every
    materialised int8 tensor bit-identical (continued from the engine's own stem), the heads within 1e-4 and the detections
    equal to the oracle post-process of the engine's own heads.  Returns (heads, oracle tensors, tensors compared, faces)."""
    from retinaface_b200 import RfError
    n = len(batch)
    heads = keep.forward_heads(batch)
    # FP32 stem: within 1 LSB of the oracle's quantised stem (summation order), on fewer than 1e-3 of the elements
    stem = keep.debug_tensor(STEM, n)
    d = np.abs(stem - oracle.stem(batch)[0])
    assert d.max() <= 1 and (d > 0).mean() < 1e-3, (label, d.max(), (d > 0).mean())
    # the integer part, continued from the engine's own stem: every materialised int8 tensor bit-identical
    o_heads, o_t = oracle.forward(batch, want_tensors=True, q_stem=stem)
    compared, missing, diffs = [], [], []
    for name, (q, _) in o_t.items():
        if name == STEM:
            continue
        try:
            got = keep.debug_tensor(name, n)
        except RfError:
            missing.append(name)
            continue
        compared.append(name)
        if not np.array_equal(got, q):
            diffs.append(first_difference(name, got, q))
    assert not diffs, (label, diffs)
    # only the FPN sums may be left unmaterialised (fused into the aggr conv's staging)
    assert set(missing) <= {"_plus0", "_plus1"}, (label, missing)
    assert len(compared) >= 26, (label, compared)
    for k in range(9):
        assert np.abs(heads[k] - o_heads[k]).max() < 1e-4, (label, k, np.abs(heads[k] - o_heads[k]).max())
    found = post.check_engine(keep, batch, heads, THR, NMS, label)
    return heads, o_t, compared, found


@pytest.mark.gpu
@pytest.mark.parametrize("case_id", list(CASES))
def test_int8_engine_bit_exact_vs_integer_oracle(case_id, golden_image, tables, post_oracle):
    case = CASES[case_id]
    _ATTEMPTED.add(case_id)
    h, w = case.hw
    table = tables[case.table]
    oracle = Int8Oracle(caffemodel(case.model), table)
    keep = _engine(case, table, keep_all=True)
    prod = _engine(case, table, keep_all=False) if case.placement else None
    try:
        for run, n in enumerate(case.runs):
            label = f"{case_id} n={n}"
            t0 = time.perf_counter()
            batch = mixed_batch(golden_image, n, h, w, start=3 * run)
            heads, o_t, compared, found = check_forward(keep, oracle, batch, post_oracle, label)
            _MERGE[case_id] = "stand-alone" if "_plus1" in compared else "fused"
            if case.table == "saturating":
                frac = {name: float((q == 127).mean()) for name, (q, _) in o_t.items()}
                for name, floor in SATURATION_FLOOR.items():
                    assert frac[name] >= floor, (label, name, frac[name])
                assert sum(f > 0 for f in frac.values()) >= SATURATED_TENSORS, (label, frac)
            assert found > 0 or not case.faces, label       # the selection and order compared are not empty
            if prod is not None:
                # production placement: tensors share memory across the three lanes; heads bit-equal, detections exact
                heads_p = prod.forward_heads(batch)
                faces_p = post_oracle.check_engine(prod, batch, heads_p, THR, NMS, label + " (liveness placement)")
                for k in range(9):
                    assert np.array_equal(heads_p[k], heads[k]), (label, "liveness placement", k)
                assert faces_p == found, label
            print(f"{label}: {len(compared)} int8 tensors bit-identical, {_MERGE[case_id]} c1 merge, {found} faces, "
                  f"{time.perf_counter() - t0:.1f} s")
    finally:
        keep.close()
        if prod is not None:
            prod.close()


@pytest.mark.gpu
def test_int8_sweep_compared_both_fpn_merges():
    """The c1 FPN merge is fused into the aggr conv when its tiles fit in one wave (c1_tiles <= SM count), else it runs
    stand-alone: 448x448 at max_batch 1 and 32 bracket that threshold for any SM count from 26 to 826, so the sweep must
    have compared both on this device."""
    if not {"448_mb1", "448_mb32"} <= _ATTEMPTED:
        pytest.skip("the bracketing cases of the sweep were not run")
    assert set(_MERGE.values()) == {"fused", "stand-alone"}, _MERGE


# ---- host side ----------------------------------------------------------------------------------------------------------
def test_int8_gemm_in_float64_equals_the_integer_product():
    """The oracle's integer GEMM, multiplied in float64, against the int64 product: random operands and the extremes, at
    the widest K of the network (3x3 over 64 channels, 1x1 over 256)."""
    rng = np.random.default_rng(3)
    for k in (576, 256, 2304):
        a = rng.integers(-127, 128, (300, k), dtype=np.int32)
        b = rng.integers(-127, 128, (k, 70), dtype=np.int32)
        a[0], a[1], b[:, 0], b[:, 1] = 127, -127, 127, -127
        got = int_gemm(a, b)
        assert got.dtype == np.int64 and np.array_equal(got, a.astype(np.int64) @ b.astype(np.int64)), k


def test_int8_sweep_covers_every_planner_branch(tables):
    """rf_plan_describe (host-only, 132 SMs assumed) for every case of the sweep: together they must run the stand-alone c1
    FPN merge and plans without it, the 2-D INT8 depthwise+pointwise kernel at stride 2 on C = 16, 32 and 64 and at stride
    1, and a 1-D depthwise step on a map larger than 56x56.  A planner change that moves a branch out of the sweep fails
    here, without a GPU."""
    from retinaface_b200.capi import plan_describe
    merge, no_merge, s2_channels, s1_2d, big_1d = [], [], set(), [], []
    for case_id, case in CASES.items():
        h, w = case.hw
        steps = [ln.split(": ", 1)[1] for ln in plan_describe(caffemodel(case.model), h, w, precision=RF_PREC_INT8,
                                                               max_batch=case.max_batch, flags=case.flags,
                                                               int8_table=tables[case.table]).splitlines()
                 if ln.startswith("step lane")]
        (merge if "i8_fpn_merge_c1_upsample+add" in steps else no_merge).append(case_id)
        for s in steps:
            m = re.fullmatch(r"i8_(2d_)?dw(\d+)\+pw\d+_s(\d)_(\d+)to\d+", s)
            if not m:
                continue
            layer, stride, c = int(m.group(2)), int(m.group(3)), int(m.group(4))
            if m.group(1) and stride == 2:
                s2_channels.add(c)
            elif m.group(1):
                s1_2d.append(case_id)
            else:
                down = 2 ** (1 + sum(1 for i in (3, 7, 11, 23) if i <= layer))     # the stem halves; stride-2 dw layers
                if (h // down) * (w // down) > 56 * 56:
                    big_1d.append(case_id)
    assert merge and no_merge, (merge, no_merge)
    assert {16, 32, 64} <= s2_channels, s2_channels
    assert s1_2d, "no i8_2d_*_s1_* step in the sweep"
    assert big_1d, "no 1-D INT8 depthwise step on a map above 56x56 in the sweep"
