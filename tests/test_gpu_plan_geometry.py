"""The three engines on every tile geometry the planner builds (tests/plan_geometry.py), portrait networks included.

Each case of plan_geometry.CASES forwards a batch of dissimilar neighbours (oracle.inputs.mixed_batch) on a handle that
keeps every tensor, and runs the step sweep of its precision on it: FP32 bit for bit against its FMA order
(test_gpu_fp32_steps), FP16 inside every element's rounding interval (test_gpu_fp16_steps), INT8 bit for bit against the
integer oracle continued from the engine's own stem (test_gpu_int8_exact); in each, the heads and the detections against
the post-process oracle.  tests/test_plan_geometry_cpu.py checks, without a GPU, that the cases reach every class.

The end-to-end check runs rf_detect_batch on a landscape and a portrait photo on a 640 x 352 (9:16 portrait) handle of each
precision: the detections, anchor indices and order included, equal the post-process oracle on the engine's own heads of
the same letter-boxed inputs.  Every map of that network is taller than it is wide.

On an H100 80GB HBM3 (700 W) the whole file took 70 s, nearly all of it the host oracles of the largest FP16 cases.
"""
import time

import numpy as np
import pytest

import plan_geometry as pg
import test_gpu_fp16_steps as f16
import test_gpu_fp32_steps as f32
import test_gpu_int8_exact as i8
from conftest import caffemodel
from oracle import fp16_steps as fs
from oracle import fp32_steps as f3
from oracle.inputs import letterbox_bgr_u8, mixed_batch
from oracle.mnet_int8 import Int8Oracle
from oracle.postproc import compare_dets

THR, NMS = 0.5, 0.4


@pytest.fixture(scope="module")
def post_oracle():
    from oracle.postproc import PostprocOracle
    return PostprocOracle()


def _check_fp32(c, batch, post, label):
    case = f32.Case(c.hw, c.max_batch, (c.n,), c.model)
    eng = f32._engine(case, keep_all=True)
    try:
        compared, _, found = f32.check_forward(eng, batch, f3.SimtSteps(caffemodel(c.model), fs.rn32), post, label)
    finally:
        eng.close()
    return f"{compared} tensors bit-equal, heads exact, {found} faces"


def _check_fp16(c, batch, post, label):
    case = f16.Case(c.hw, c.max_batch, (c.n,), c.model, streams=c.streams)
    options = f16.walk_options(f16.plan_steps(case)[0])
    eng = f16._engine(case, keep_all=True)
    try:
        _, compared, _, found = f16.check_case(case, eng, batch, fs.Fp16Steps(caffemodel(c.model)), post, label, options)
    finally:
        eng.close()
    return f"{len(compared)} tensors inside their intervals, {found} faces"


def _check_int8(c, batch, post, label):
    assert c.model == i8.MODEL, "the shipped calibration table is the deconv model's"
    case = i8.Case(c.hw, c.max_batch, (c.n,))
    eng = i8._engine(case, i8.SHIPPED_TABLE, keep_all=True)
    try:
        _, _, compared, found = i8.check_forward(eng, Int8Oracle(caffemodel(c.model), i8.SHIPPED_TABLE), batch, post, label)
    finally:
        eng.close()
    return f"{len(compared)} int8 tensors bit-identical, {found} faces"


CHECKS = {pg.FP32: _check_fp32, pg.FP16: _check_fp16, pg.INT8: _check_int8}


@pytest.mark.gpu
@pytest.mark.parametrize("case_id", list(pg.CASES))
def test_engine_on_every_tile_geometry(case_id, golden_image, post_oracle):
    c = pg.CASES[case_id]
    t0 = time.perf_counter()
    batch = mixed_batch(golden_image, c.n, c.hw[0], c.hw[1])
    result = CHECKS[c.prec](c, batch, post_oracle, case_id)
    print(f"\n{case_id}: {result}, {time.perf_counter() - t0:.1f} s")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [pg.FP32, pg.FP16, pg.INT8], ids=lambda p: pg.PREC_NAMES[p])
def test_detect_batch_on_a_portrait_network(prec, golden_image, post_oracle):
    from retinaface_b200 import Engine
    h, w = pg.PORTRAIT
    model = i8.MODEL if prec == pg.INT8 else "mnet25"
    images = [golden_image, np.ascontiguousarray(golden_image[:, 330:830])]       # 1280 x 886 and 500 x 886
    inputs = np.stack([letterbox_bgr_u8(im, h, w) for im in images])
    eng = Engine(caffemodel(model), h, w, precision=prec, max_batch=2, max_image=golden_image.shape[:2],
                 int8_table=i8.SHIPPED_TABLE if prec == pg.INT8 else None)
    try:
        for im, x in zip(images, inputs):
            assert np.array_equal(eng.preprocess(im), x), im.shape
        faces, idx = eng.detect_batch(images, THR, NMS, want_index=True)
        heads = eng.forward_heads(inputs)
        for i, im in enumerate(images):
            ref = post_oracle.postprocess([x[i] for x in heads], h, w, THR, NMS)
            compare_dets(faces[i], idx[i], ref, f"{pg.PREC_NAMES[prec]} {im.shape[1]}x{im.shape[0]}", eng.max_faces)
            assert len(faces[i]) >= 1, im.shape
        print(f"\n{pg.PREC_NAMES[prec]} {h}x{w} network: {[len(f) for f in faces]} faces, anchor indices and order "
              "equal the oracle's")
    finally:
        eng.close()
