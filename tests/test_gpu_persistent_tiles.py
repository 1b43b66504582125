"""GPU (-m gpu): the persistent front-end kernels -- k_stem_tc and k_tc_dwpw_2d take a run of consecutive tiles per CTA, with
the next tile's input staged while the current one computes.  These tests cover what a one-tile-per-CTA grid never exercised:
several tiles per CTA, runs that cross from one image into the next, and a grid smaller than the tile count."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.inputs import mixed_batch

pytestmark = pytest.mark.gpu

HEAD_NAMES = ("mobilenet0_relu4_fwd", "mobilenet0_relu6_fwd", "mobilenet0_relu8_fwd", "mobilenet0_relu10_fwd")


def _engine(prec, h, w, batch, flags=0):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_INT8, Engine
    if prec == "fp16":
        return Engine(caffemodel("mnet25"), h, w, precision=RF_PREC_FP16, max_batch=batch, flags=flags)
    model = "mnet-deconv-0517"
    return Engine(caffemodel(model), h, w, precision=RF_PREC_INT8, max_batch=batch, flags=flags,
                  int8_table=os.path.join(GOLDEN, "weights", model + ".table.int8"))


@pytest.mark.parametrize("hw, batch", [((448, 448), 8), ((448, 448), 1), ((896, 1280), 8), ((288, 416), 5)])
def test_persistent_2d_tiles_equal_the_1d_kernels(hw, batch, golden_image):
    """FP16 default plan (persistent k_tc_dwpw_2d on every map above 56x56) against RF_FLAG_DW_1D (the one-tile-per-CTA
    linear kernels): same arithmetic, so relu4..relu10 and all nine head blobs are identical.  1280x896 runs the 2-D tiles on
    dw3..dw11; 416x288 leaves partial 2-D tiles on its 104-wide map."""
    from retinaface_b200.capi import RF_FLAG_DW_1D
    h, w = hw
    batch_u8 = mixed_batch(golden_image, batch, h, w)
    a, b = _engine("fp16", h, w, batch), _engine("fp16", h, w, batch, flags=RF_FLAG_DW_1D)
    try:
        a.debug_keep_all()
        b.debug_keep_all()
        ha, hb = a.forward_heads(batch_u8), b.forward_heads(batch_u8)
        for name in HEAD_NAMES:
            assert np.array_equal(a.debug_tensor(name, batch), b.debug_tensor(name, batch)), name
        for k in range(9):
            assert np.array_equal(ha[k], hb[k]), k
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("prec", ["fp16", "int8"])
@pytest.mark.parametrize("hw", [(448, 448), (288, 416)])
def test_persistent_tiles_batch_equals_each_image_alone(prec, hw, golden_image):
    """Each image of a batch of 8 dissimilar images gives, in relu2 (k_stem_tc) and -- FP16 -- relu6 (k_tc_dwpw_2d), exactly
    what it gives forwarded alone: a CTA's run of tiles crosses image boundaries in the batch, never alone."""
    h, w = hw
    n = 8
    batch_u8 = mixed_batch(golden_image, n, h, w)
    names = ["mobilenet0_relu2_fwd"] + (["mobilenet0_relu6_fwd"] if prec == "fp16" else [])
    eng = _engine(prec, h, w, n)
    try:
        eng.debug_keep_all()
        eng.forward_heads(batch_u8)
        together = {name: eng.debug_tensor(name, n) for name in names}
        for i in range(n):
            eng.forward_heads(batch_u8[i:i + 1])
            for name in names:
                assert np.array_equal(eng.debug_tensor(name, 1)[0], together[name][i]), (name, i)
    finally:
        eng.close()
