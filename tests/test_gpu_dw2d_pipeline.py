"""GPU (-m gpu): the pipelined k_tc_dwpw_2d -- a ring of staged windows ahead of the tile that computes, the output tile
written through shared memory and stored as whole lines, single-output stencil items at C = 16.  Each case compares the
default plan with RF_FLAG_DW_1D (the one-tile-per-CTA linear kernels, same arithmetic) bit for bit, at run lengths from one
tile to more than the ring holds."""
import numpy as np
import pytest

from conftest import caffemodel
from oracle.inputs import mixed_batch

pytestmark = pytest.mark.gpu


def _engine(h, w, batch, flags=0):
    from retinaface_b200 import RF_PREC_FP16, Engine
    return Engine(caffemodel("mnet25"), h, w, precision=RF_PREC_FP16, max_batch=batch, flags=flags)


# (input h, w), batch, the 2-D layers' outputs.  On 132 SMs, one CTA each, 448x448 gives runs of one tile at batch 1, two at
# batch 2, six at 8 and 24 at 32 (98 tiles per image); six and 24 do not divide 98, so runs cross images.  416x288 ends each
# tile row with a half-empty tile; 1280x896 runs dw3..dw11 on 2-D tiles, dw11 with a ring of two windows.
CASES = [
    ((448, 448), 1, ("relu4", "relu6")),
    ((448, 448), 2, ("relu4", "relu6")),
    ((448, 448), 8, ("relu4", "relu6")),
    ((448, 448), 32, ("relu4", "relu6")),
    ((288, 416), 3, ("relu4", "relu6")),
    ((896, 1280), 8, ("relu4", "relu6", "relu8", "relu10", "relu12")),
]


@pytest.mark.parametrize("hw, batch, relus", CASES, ids=[f"{hw[1]}x{hw[0]}_b{b}" for hw, b, _ in CASES])
def test_pipelined_2d_tiles_equal_the_1d_kernels(hw, batch, relus, golden_image):
    from retinaface_b200.capi import RF_FLAG_DW_1D
    h, w = hw
    batch_u8 = mixed_batch(golden_image, batch, h, w)
    a, b = _engine(h, w, batch), _engine(h, w, batch, flags=RF_FLAG_DW_1D)
    try:
        a.debug_keep_all()
        b.debug_keep_all()
        ha, hb = a.forward_heads(batch_u8), b.forward_heads(batch_u8)
        for r in relus:
            name = f"mobilenet0_{r}_fwd"
            assert np.array_equal(a.debug_tensor(name, batch), b.debug_tensor(name, batch)), name
        for k in range(9):
            assert np.array_equal(ha[k], hb[k]), k
    finally:
        a.close()
        b.close()
