"""The SIMT plans -- the FP32 engine (RF_PREC_FP32) and FP16 with RF_FLAG_NO_TENSORCORE -- bit for bit against their exact
restatement (oracle/fp32_steps.py), and the INT8 calibrator's table against a numpy rebuild from the same FP32 tensors.

Each case forwards a batch of dissimilar neighbours (oracle.inputs.mixed_batch) on a handle that keeps every tensor.  Every
one of the 43 tensors the SIMT plan materialises is recomputed from the engine's own inputs and must be equal element for
element (np.array_equal); the bbox and landmark deltas must be equal, the class probabilities inside softmax_pair's expf
interval, and the detections equal to the oracle post-process of the engine's own heads.  The benchmarked plan (448^2,
max_batch 8) and the 1280x896 plan also run a handle with the production (liveness) buffer placement, whose heads must be
bit-equal to the keep-all handle's.  Every image of every case is checked: on an H100 80GB HBM3 (700 W) the whole file
took 137 s, 51 s each for 448^2 max_batch 8 (13 images) and 1280x896 (2 images), nearly all of it the host restatement.

The calibrator: rf_calibrate_int8 on an FP32 handle, then the same chunks forwarded on a keep-all FP32 handle of the same
configuration and the table rebuilt in numpy exactly as rf_calibrate_int8 builds it (engine.cu:1582-1616): float32 absmax
over all chunks, float32 bin width, truncated float32 bins clamped to the last, the library's own KL search
(capi.kl_threshold_bins, checked separately in tests/test_host_side.py), float64 threshold, float32 scale.  The written file
must equal the rebuilt one byte for byte, which checks k_absmax and k_hist.  The branch for a tensor that is zero on every
calibration image (scale 1/127) needs an input no real batch gives; it is not tested, and the test asserts it was not taken.
"""
import re
import struct
import time
from typing import NamedTuple

import numpy as np
import pytest

from conftest import caffemodel
from oracle import fp16_steps as fs
from oracle import fp32_steps as f3
from oracle.inputs import mixed_batch
from retinaface_b200.capi import RF_FLAG_NO_TENSORCORE, RF_PREC_FP16, RF_PREC_FP32

THR, NMS = 0.5, 0.4
DECONV = "mnet-deconv-0517"


class Case(NamedTuple):
    hw: tuple               # network (H, W)
    max_batch: int
    runs: tuple             # batch sizes forwarded one after the other on the same handle
    model: str = "mnet25"
    fp16: bool = False      # RF_PREC_FP16 with RF_FLAG_NO_TENSORCORE (FP16 storage) instead of RF_PREC_FP32
    placement: bool = False  # also run a handle with the production (liveness) buffer placement


CASES = {
    "448_mb8": Case((448, 448), 8, (8, 5), placement=True),      # the benchmarked plan, then a partial batch
    "deconv_448_mb2": Case((448, 448), 2, (2,), model=DECONV),
    "896x1280_mb2": Case((896, 1280), 2, (2,), placement=True),  # large maps
    "288x416_mb3": Case((288, 416), 3, (3,), model=DECONV),      # shipped size, 9 x 13 stride-32 map
    "96x160_mb3": Case((96, 160), 3, (3,)),                      # every GEMM tile spans images; taps mostly padding
    "32_mb4": Case((32, 32), 4, (4,)),                           # 1 x 1 stride-32 map: merges from one coarse pixel
    "32x224_mb2": Case((32, 224), 2, (2,)),                      # one-row maps
    "simt16_448_mb3": Case((448, 448), 3, (3,), fp16=True),      # the second reference of test_fp16_tensor_core_layers_vs_oracle
    "simt16_96x160_mb3": Case((96, 160), 3, (3,), model=DECONV, fp16=True),
}


def _precision(case):
    return (RF_PREC_FP16, RF_FLAG_NO_TENSORCORE) if case.fp16 else (RF_PREC_FP32, 0)


def _engine(case, keep_all):
    from retinaface_b200 import Engine
    prec, flags = _precision(case)
    eng = Engine(caffemodel(case.model), case.hw[0], case.hw[1], precision=prec, max_batch=case.max_batch, flags=flags)
    if keep_all:
        eng.debug_keep_all()
    return eng


def first_difference(name, step, got, want):
    bad = got != want
    b, c, y, x = np.argwhere(bad)[0]
    return (f"{name} ({step}): first difference at (image {b}, channel {c}, y {y}, x {x}): engine {got[b, c, y, x]!r}, "
            f"oracle {want[b, c, y, x]!r}; {int(bad.sum())} of {bad.size} elements differ")


def _fetcher(eng, n):
    def fetch(name, _):
        return eng.debug_tensor(name, n).astype(np.float64)
    return fetch


def check_forward(eng, batch, steps, post, label):
    """Every tensor of one forward equal to its restatement, the heads exact (class probabilities inside their interval),
    the detections equal to the oracle post-process.  Returns (tensors compared, heads, faces found)."""
    n = len(batch)
    heads = eng.forward_heads(batch)
    compared, diffs = [], []
    for name, step, want, got in steps.walk(batch, _fetcher(eng, n)):
        if name.startswith("heads"):
            (lo, hi), bbox, lm = want
            l = {"heads_stride32": 0, "heads_stride16": 1, "heads_stride8": 2}[name]
            cls = heads[3 * l].astype(np.float64)
            if ((cls < lo) | (cls > hi)).any():
                bad = (cls < lo) | (cls > hi)
                b, c, y, x = np.argwhere(bad)[0]
                diffs.append(f"{name} class probabilities: first outside at (image {b}, channel {c}, y {y}, x {x}): engine "
                             f"{cls[b, c, y, x]!r}, interval [{lo[b, c, y, x]!r}, {hi[b, c, y, x]!r}]")
            for what, e, w in (("bbox", heads[3 * l + 1], bbox), ("landmarks", heads[3 * l + 2], lm)):
                if not np.array_equal(e.astype(np.float64), w):
                    diffs.append(first_difference(f"{name} {what}", step, e.astype(np.float64), w))
            continue
        compared.append(name)
        if not np.array_equal(got, want):
            diffs.append(first_difference(name, step, got, want))
    assert not diffs, (label, diffs)
    assert len(compared) == len(set(compared)) == f3.TENSORS, (label, compared)
    found = post.check_engine(eng, batch, heads, THR, NMS, label)
    return len(compared), heads, found


@pytest.fixture(scope="module")
def post_oracle():
    from oracle.postproc import PostprocOracle
    return PostprocOracle()


@pytest.mark.gpu
@pytest.mark.parametrize("case_id", list(CASES))
def test_simt_engine_bit_exact_vs_its_restatement(case_id, golden_image, post_oracle):
    case = CASES[case_id]
    h, w = case.hw
    steps = f3.SimtSteps(caffemodel(case.model), fs.rn16 if case.fp16 else fs.rn32)
    keep = _engine(case, keep_all=True)
    prod = _engine(case, keep_all=False) if case.placement else None
    t_case = time.perf_counter()
    try:
        for run, n in enumerate(case.runs):
            label = f"{case_id} n={n}"
            t0 = time.perf_counter()
            batch = mixed_batch(golden_image, n, h, w, start=3 * run)
            compared, heads, found = check_forward(keep, batch, steps, post_oracle, label)
            if prod is not None:
                heads_p = prod.forward_heads(batch)
                for k in range(9):
                    assert np.array_equal(heads_p[k], heads[k]), (label, "liveness placement", k)
            print(f"\n{label}: {compared} tensors bit-equal, heads exact, {found} faces, {time.perf_counter() - t0:.1f} s")
    finally:
        keep.close()
        if prod is not None:
            prod.close()
    print(f"{case_id}: {time.perf_counter() - t_case:.1f} s")


# ---- the calibrator -----------------------------------------------------------------------------------------------------
def library_tensor_order():
    """h->tensors of the SIMT plan in creation order (plan_net.cu walk_network with SimtOps): the stem's conv0 and pair, the
    pairs and each segment's lateral after them, then per FPN level the concat before its two context tensors (ssh) and the
    aggr output before its FPN sum (merge_aggr)."""
    names = [f"mobilenet0_relu{i}_fwd" for i in range(3)]
    for pairs, lat in (((3, 5), None), ((7, 9), "rf_c1_red_conv"), ((11, 13, 15), None), ((17, 19, 21), "rf_c2_lateral"),
                       ((23,), None), ((25,), "rf_c3_lateral")):
        for i in pairs:
            names += [f"mobilenet0_relu{i}_fwd", f"mobilenet0_relu{i + 1}_fwd"]
        if lat:
            names.append(lat + "_relu")
    for lv in ("c3", "c2", "c1"):
        if lv != "c3":
            names += [f"rf_{lv}_aggr_relu", "_plus0" if lv == "c2" else "_plus1"]
        names += [f"rf_{lv}_det_concat_relu", f"rf_{lv}_det_context_conv1_relu", f"rf_{lv}_det_context_conv3_1_relu"]
    return names


def rebuild_table(eng, images, max_batch, names):
    """rf_calibrate_int8's table from the keep-all handle's tensors, in numpy.  Returns (text, {name: (hmax, bins)})."""
    from retinaface_b200.capi import kl_threshold_bins
    absx = {nm: [] for nm in names}
    for i0 in range(0, len(images), max_batch):
        chunk = images[i0:i0 + max_batch]
        eng.forward_heads(chunk)
        for nm in names:
            absx[nm].append(np.abs(eng.debug_tensor(nm, len(chunk)).astype(np.float32)).ravel())
    lines = ["TRT-5102-EntropyCalibration2", f"data: {struct.pack('>f', np.float32(255) / np.float32(127)).hex()}"]
    info = {}
    for nm in names:
        hmax = np.float32(max(a.max() for a in absx[nm]))
        assert hmax > 0, (nm, "zero on every calibration image: the untested branch")
        inv = np.float32(2048) / hmax
        hist = sum(np.bincount(np.minimum((a * inv).astype(np.int64), 2047), minlength=2048) for a in absx[nm])
        bins = kl_threshold_bins(hist.astype(np.uint32))
        scale = np.float32(bins * float(hmax) / 2048 / 127.0)
        lines.append(f"{nm}: {struct.pack('>f', scale).hex()}")
        info[nm] = (float(hmax), bins)
    return "\n".join(lines) + "\n", info


CALIBRATIONS = {"mnet25_96x160_mb3": ("mnet25", (96, 160), 3, 7), "deconv_448_mb4": (DECONV, (448, 448), 4, 9)}


@pytest.mark.gpu
@pytest.mark.parametrize("cal_id", list(CALIBRATIONS))
def test_calibrator_table_equals_its_numpy_rebuild(cal_id, golden_image, tmp_path):
    """The written table byte for byte equal to the numpy rebuild from the same chunks (3 + 3 + 1 and 4 + 4 + 1 images)."""
    from retinaface_b200 import Engine
    model, (h, w), mb, n = CALIBRATIONS[cal_id]
    t0 = time.perf_counter()
    images = mixed_batch(golden_image, n, h, w)
    table = str(tmp_path / "calib.table.int8")
    cal = Engine(caffemodel(model), h, w, precision=RF_PREC_FP32, max_batch=mb)
    try:
        cal.calibrate_int8(images, table)
    finally:
        cal.close()
    keep = Engine(caffemodel(model), h, w, precision=RF_PREC_FP32, max_batch=mb)
    try:
        keep.debug_keep_all()
        names = library_tensor_order()
        want, info = rebuild_table(keep, images, mb, names)
    finally:
        keep.close()
    with open(table, "rb") as f:
        got = f.read().decode()
    if got != want:
        g, r = got.splitlines(), want.splitlines()
        bad = [(a, b) for a, b in zip(g, r) if a != b]
        nm = (bad[0][1].split(":")[0] if bad else "")
        pytest.fail(f"{cal_id}: {len(bad)} lines differ ({len(g)} written, {len(r)} rebuilt); first: written {bad[:1]}, "
                    f"rebuilt hmax / bins {info.get(nm)}")
    print(f"\n{cal_id}: {len(names)} tensors + data, table byte-identical, {time.perf_counter() - t0:.1f} s")


# ---- host side ----------------------------------------------------------------------------------------------------------
def test_library_tensor_order_is_the_walk():
    """The calibrator rebuild's order names the 43 tensors the step walk checks, each once."""
    names = library_tensor_order()
    steps = f3.SimtSteps(caffemodel("mnet25"))
    img = np.zeros((1, 32, 32, 3), np.uint8)
    walked = [name for name, *_ in steps.walk(img, lambda name, want: None) if not name.startswith("heads")]
    assert len(names) == len(set(names)) == f3.TENSORS and set(names) == set(walked)


def test_fp32_sweep_reaches_every_simt_kernel():
    """rf_plan_describe (host-only) for every case of the sweep: each is the SIMT plan (k_conv0, no tensor-core stem), and
    together they run the depthwise kernel at stride 1 and 2, 1x1 and 3x3 GEMMs with N = 16, 32, 48 and 64 or more (every
    BN of launch_gemm: 64, 32 and 16), both FPN merges and the fused heads.  A planner change that moves a kernel out of the
    sweep fails here, without a GPU."""
    from retinaface_b200.capi import plan_describe
    seen, bns = set(), set()
    for case_id, case in CASES.items():
        prec, flags = _precision(case)
        steps = [ln.split(": ", 1)[1] for ln in plan_describe(caffemodel(case.model), case.hw[0], case.hw[1], precision=prec,
                                                               max_batch=case.max_batch, flags=flags).splitlines()
                 if ln.startswith("step lane")]
        assert steps[0] == "conv0_u8_3x3s2_bn_relu" and not any("stem" in s for s in steps), (case_id, steps[:2])
        for s in steps:
            if m := re.fullmatch(r"dw\d+_3x3s(\d)_c\d+", s):
                seen.add(f"dw s{m.group(1)}")
            elif m := re.fullmatch(r".*_(1x1|3x3)_(\d+)to(\d+)", s):
                seen.add(f"gemm {m.group(1)}")
                N = int(m.group(3))
                bns.add(64 if N % 64 == 0 else (32 if N % 32 == 0 else 16))
            elif s in ("upsample_add_plus0", "upsample_add_plus1", "heads_1x1+softmax+decode+nms_all_levels"):
                seen.add(s)
    assert seen == {"dw s1", "dw s2", "gemm 1x1", "gemm 3x3", "upsample_add_plus0", "upsample_add_plus1",
                    "heads_1x1+softmax+decode+nms_all_levels"}, seen
    assert bns == {16, 32, 64}, bns
