"""Exact restatement of every step of the SIMT plans: the FP32 engine (RF_PREC_FP32) and FP16 with RF_FLAG_NO_TENSORCORE.
Test infrastructure -- see ``oracle/__init__.py``.

Both plans are ``build_plan<T>`` (plan_fp.cu ``SimtOps``): every layer its own CUDA-core kernel of ``kernels_simt.cuh``,
each spelling its arithmetic out as ``fmaf`` chains in a fixed order, with no atomics and no reduction across threads.  So
each step is one value per element, and a test holds the engine to "every element equal".  The two plans differ only in
how a step stores its FP32 result: ``store`` is ``rn32`` (T = float: the identity on FP32 values) or ``rn16`` (T = __half:
``from_f<__half>`` / ``Vec8<__half>::from_float``, ``common.cuh:31-35, 53``, round to nearest even).  The primitives
(``fma32``, ``add32``, ``head_dots``, ``cls_prob``) are those of ``oracle/fp16_steps.py``.  Rounding points, per kernel:

* ``k_conv0`` (``kernels_simt.cuh:20-63``): acc = FP32 bias (:39), ``fmaf`` over the taps in (ky, kx, c_bgr) order (:41-57;
  a tap outside the image is skipped, the same value as adding 0 * w), ``fmaxf`` ReLU (:59), store (:60-62).
* ``k_dw3x3`` (:70-113): acc = FP32 bias (:89), ``fmaf`` over the taps in (ky, kx) order with the FP32 weights (:92-107,
  ``pack_dw``: not rounded to FP16, unlike the tensor-core plans), ReLU (:109), store (:110-112).
* ``k_conv_gemm`` (:132-216, ``launch_gemm`` plan_fp.cu:34-44): acc = 0 (:157), ``fmaf`` for k = tap * Cin + c in order
  (:160-196; the ``kc`` chunks and the 64-pixel tiles change nothing in that order; an out-of-map tap adds 0 * w), then
  one FP32 add of the bias (:206), ReLU per ``OutSplit`` half (:207-212), store.
* ``k_upsample_add`` (:225-268): acc = the lateral value (:244), ``fmaf`` with the FP32 deconvolution weights over the taps
  (i_hi, j_hi), (i_hi, j_hi - 1), (i_hi - 1, j_hi), (i_hi - 1, j_hi - 1), a tap outside the coarse map skipped (:246-264),
  no ReLU, store.
* ``k_head_decode<T>`` (postproc.cu:73-92): ``__fmaf_rn`` from the bias over the 64 channels (``fs.head_dots``): the bbox
  and landmark deltas are exact; the class probabilities are ``softmax_pair``'s ``expf`` interval (``fs.cls_prob``).

Signed zeros are not restated (a skipped tap and an added 0 * w can differ in the sign of a zero); the comparisons are of
values (``np.array_equal``), for which -0 == +0.

Speed: ``fma32`` rounds every sum to odd (TwoSum), about 40 ns per multiply-add.  ``fma32_fast`` evaluates the float64 sum
once -- the product of two FP32 values is exact in float64 -- and rounds it to FP32: that is the correctly rounded fmaf
unless the float64 rounding landed exactly on an FP32 midpoint (no other FP32 midpoint lies between the exact sum and its
float64 rounding, midpoints being float64 values), or the sum is below the FP32 normal range where the midpoint pattern
differs.  Those elements are recomputed with ``fma32``.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np

from . import fp16_steps as fs
from .fp16_steps import F64, STRIDE2, nchw, nhwc, rn16, rn32
from .mnet_numpy import folded_params

_MID_MASK, _MID_BIT = 0x1FFFFFFF, 0x10000000        # float64 bits below FP32 precision: exactly half an FP32 ulp
_EXP_MASK = 0x7FF0000000000000
_EXP_TINY = (1023 - 125) << 52                       # |s| < 2**-125: FP32 subnormal range (and one binade of margin)


def _risky(s):
    """Where rn32(s) may differ from the correctly rounded exact sum that s is the float64 rounding of."""
    bits = s.view(np.int64)
    r = (bits & _MID_MASK) == _MID_BIT
    r |= ((bits & _EXP_MASK) < _EXP_TINY) & (s != 0)
    return r


def fma32_fast(x, w, acc):
    """fmaf(x, w, acc) of FP32 values (float64 arrays, broadcast): equal to fs.fma32, one float64 sum per element."""
    s = np.multiply(x, w, dtype=F64) + np.asarray(acc, F64)
    risky = _risky(s)
    r = rn32(s)
    if risky.any():
        xb, wb, ab = np.broadcast_arrays(np.asarray(x, F64), np.asarray(w, F64), np.asarray(acc, F64))
        r[risky] = fs.fma32(xb[risky], wb[risky], ab[risky])
    return r


def fma_chain(acc, pairs):
    """acc (M, N) float64 FP32 values, updated by fmaf(a_k[:, None], w_k[None, :], acc) for each (a_k, w_k) in order: the
    inner loop of a GEMM, with in-place buffers (the accumulator is held as float32)."""
    acc32 = np.asarray(acc, np.float32).copy()
    s = np.empty(acc32.shape, F64)
    for a, w in pairs:
        np.multiply(a[:, None], w[None, :], out=s)
        s += acc32
        risky = _risky(s)
        if risky.any():
            rows, cols = np.nonzero(risky)
            fix = fs.fma32(a[rows], w[cols], acc32[rows, cols].astype(F64))
            acc32[...] = s                                               # RN to FP32
            acc32[rows, cols] = fix
        else:
            acc32[...] = s
    return acc32.astype(F64)


# ---- steps --------------------------------------------------------------------------------------------------------------
def conv0(img, c0, store=rn32):
    """k_conv0: u8 BGR (n, H, W, 3) -> (n, 8, H/2, W/2)."""
    n, H, W, _ = img.shape
    cols = fs._stem_image_cols(img).astype(F64)                             # k = (ky * 3 + kx) * 3 + c_bgr
    w0 = fs._conv0_matrix(c0["w"])
    acc = np.broadcast_to(np.asarray(c0["b"], F64), (cols.shape[0], 8))
    acc = fma_chain(acc, ((cols[:, k].copy(), w0[k]) for k in range(27)))
    return store(nchw(np.maximum(acc, 0).reshape(n, H // 2, W // 2, 8)))


def depthwise(x, w, b, stride, store=rn32, weights16=False):
    """k_dw3x3<T, stride>: NCHW x, FP32 bias, fmaf over the taps in (ky, kx) order, ReLU.  weights16: the tensor-core plans'
    FP16-rounded weights instead (a mistake here: the SIMT kernel reads pack_dw's FP32 weights)."""
    wt = fs.dw_weights16(w) if weights16 else np.asarray(w, F64).reshape(w.shape[0], 9)
    n, c, h, wd = x.shape
    oh, ow = h // stride, wd // stride
    xp = np.pad(np.asarray(x, F64), ((0, 0), (0, 0), (1, 1), (1, 1)))
    acc = np.broadcast_to(np.asarray(b, F64)[None, :, None, None], (n, c, oh, ow))
    for t in range(9):
        dy, dx = t // 3, t % 3
        acc = fma32_fast(xp[:, :, dy:dy + stride * oh:stride, dx:dx + stride * ow:stride], wt[None, :, t, None, None], acc)
    return store(np.maximum(acc, 0))


def gemm_matrix(ws):
    """pack_gemm (plan_fp.cu:15-32): convs sharing an input, concatenated along N, as [K = (tap, cin)][N] FP32 values."""
    return np.concatenate([np.asarray(w, F64).transpose(2, 3, 1, 0).reshape(-1, w.shape[0]) for w in ws], axis=1)


def gemm_acc(x, wk, ks):
    """The accumulator of k_conv_gemm before its epilogue: x NCHW (n, Cin, h, w), wk [ks*ks*Cin][N]; returns (M, N)."""
    n, cin, h, wd = x.shape
    xh = nhwc(np.asarray(x, F64))
    xp = np.pad(xh, ((0, 0), (1, 1), (1, 1), (0, 0))) if ks == 3 else xh

    def pairs():
        for t in range(ks * ks):
            dy, dx = (t // 3, t % 3) if ks == 3 else (0, 0)
            at = np.ascontiguousarray(xp[:, dy:dy + h, dx:dx + wd].reshape(-1, cin).T)      # (Cin, M)
            for c in range(cin):
                yield at[c], wk[t * cin + c]
    return fma_chain(np.zeros((n * h * wd, wk.shape[1])), pairs())


def gemm_epilogue(acc, bias, outs, shape, store=rn32):
    """+ FP32 bias (one add), ReLU per OutSplit half, store; outs = [(channels, relu)].  Returns one NCHW array per half."""
    n, h, wd = shape
    v = fs.add32(acc, np.asarray(bias, F64)[None])
    res, o0 = [], 0
    for cn, relu in outs:
        seg = v[:, o0:o0 + cn]
        res.append(store(nchw((np.maximum(seg, 0) if relu else seg).reshape(n, h, wd, cn))))
        o0 += cn
    return res


def gemm_conv(x, ws, bs, outs, store=rn32):
    """k_conv_gemm: the convs of ws (1x1 or 3x3, pad 1) sharing the input x (NCHW), split over outs = [(channels, relu)]."""
    acc = gemm_acc(x, gemm_matrix(ws), ws[0].shape[2])
    return gemm_epilogue(acc, np.concatenate([np.asarray(b, F64) for b in bs]), outs, (x.shape[0],) + x.shape[2:], store)


def upsample_add(lat, up, up_w, store=rn32):
    """k_upsample_add: lateral + crop(deconv k4 s2 p1 of up) with the FP32 weights up_w (C, 1, 4, 4), fmaf from the
    lateral over the taps (i_hi, j_hi), (i_hi, j_hi - 1), (i_hi - 1, j_hi), (i_hi - 1, j_hi - 1), skipping those outside."""
    w = np.asarray(up_w, F64).reshape(-1, 4, 4)
    n, c, h, wd = lat.shape
    uh, uw = up.shape[2:]
    y, x = np.arange(h), np.arange(wd)
    acc = np.asarray(lat, F64)
    for di in range(2):
        i = (y + 1) // 2 - di
        ky = y - 2 * i + 1
        for dj in range(2):
            j = (x + 1) // 2 - dj
            kx = x - 2 * j + 1
            ok = ((i >= 0) & (i < uh))[:, None] & ((j >= 0) & (j < uw))[None, :]
            u = np.asarray(up, F64)[:, :, np.clip(i, 0, uh - 1)][:, :, :, np.clip(j, 0, uw - 1)]
            acc = np.where(ok, fma32_fast(u, w[:, ky][:, :, kx][None], acc), acc)
    return store(acc)


# ---- the network, continued from the engine's own tensors ---------------------------------------------------------------
LATERALS = {10: "rf_c1_red_conv", 22: "rf_c2_lateral", 26: "rf_c3_lateral"}     # after the pointwise conv producing relu{k}


class SimtSteps:
    """The SIMT plan of one caffemodel, step by step.  store: rn32 (RF_PREC_FP32) or rn16 (FP16, RF_FLAG_NO_TENSORCORE)."""

    def __init__(self, caffemodel: str, store=rn32):
        self.p = folded_params(caffemodel)
        self.store = store

    def conv(self, x, names, outs):
        return gemm_conv(x, [self.p[n]["w"] for n in names], [self.p[n]["b"] for n in names], outs, self.store)

    def heads(self, cat, stride):
        """-> (cls interval (lo, hi), bbox deltas, landmark deltas) of one level, NCHW (k_head_decode<T>)."""
        names = [f"face_rpn_{k}_stride{stride}" for k in ("cls_score", "bbox_pred", "landmark_pred")]
        w = np.concatenate([self.p[n]["w"][:, :, 0, 0] for n in names])
        b = np.concatenate([self.p[n]["b"] for n in names])
        s = fs.head_dots(cat, w, b)
        return fs.cls_prob(s[:, :4]), s[:, 4:12], s[:, 12:32]

    def walk(self, img, fetch: Callable[[str, np.ndarray], Optional[np.ndarray]]):
        """Every tensor of the SIMT plan in step order (plan_net.cu walk_network with SimtOps), each computed from the engine's
        own inputs: fetch(name, want) returns the engine's tensor (NCHW) or None.  Yields (tensor, step, want, engine value
        or None); the three levels' heads come last as ("heads_stride{s}", "k_head_decode", (cls (lo, hi), bbox, lm), cat)."""
        cur: Dict[str, np.ndarray] = {}
        p = self.p

        def emit(name, step, want):
            got = fetch(name, want)
            cur[name] = want if got is None else np.asarray(got, F64)
            return name, step, want, got

        yield emit("mobilenet0_relu0_fwd", "k_conv0", conv0(img, p["mobilenet0_conv0_fwd"], self.store))
        for i in range(1, 27, 2):
            dw, pw = p[f"mobilenet0_conv{i}_fwd"], p[f"mobilenet0_conv{i + 1}_fwd"]
            s = 2 if i in STRIDE2 else 1
            yield emit(f"mobilenet0_relu{i}_fwd", f"k_dw3x3 s{s} dw{i}",
                       depthwise(cur[f"mobilenet0_relu{i - 1}_fwd"], dw["w"], dw["b"], s, self.store))
            yield emit(f"mobilenet0_relu{i + 1}_fwd", f"k_conv_gemm 1x1 pw{i + 1}",
                       self.conv(cur[f"mobilenet0_relu{i}_fwd"], [f"mobilenet0_conv{i + 1}_fwd"], [(pw["w"].shape[0], True)])[0])
            if i + 1 in LATERALS:
                nm = LATERALS[i + 1]
                yield emit(nm + "_relu", f"k_conv_gemm 1x1 {nm}", self.conv(cur[f"mobilenet0_relu{i + 1}_fwd"], [nm], [(64, True)])[0])
        for lv, ssh_in in (("c3", "rf_c3_lateral_relu"), ("c2", "rf_c2_aggr_relu"), ("c1", "rf_c1_aggr_relu")):
            if lv != "c3":
                level = 0 if lv == "c2" else 1
                lat_t = "rf_c2_lateral_relu" if lv == "c2" else "rf_c1_red_conv_relu"
                up_t = "rf_c3_lateral_relu" if lv == "c2" else "rf_c2_aggr_relu"
                up_w = p["rf_c3_upsampling" if level == 0 else "rf_c2_upsampling"]["w"]
                yield emit(f"_plus{level}", "k_upsample_add", upsample_add(cur[lat_t], cur[up_t], up_w, self.store))
                yield emit(ssh_in, f"k_conv_gemm 3x3 rf_{lv}_aggr", self.conv(cur[f"_plus{level}"], [f"rf_{lv}_aggr"], [(64, True)])[0])
            d = f"rf_{lv}_det"
            det, ctx1 = self.conv(cur[ssh_in], [d + "_conv1", d + "_context_conv1"], [(32, True), (16, True)])
            yield emit(d + "_context_conv1_relu", f"k_conv_gemm 3x3 {d}_conv1+context_conv1", ctx1)
            c2, c31 = self.conv(cur[d + "_context_conv1_relu"], [d + "_context_conv2", d + "_context_conv3_1"], [(16, True), (16, True)])
            yield emit(d + "_context_conv3_1_relu", f"k_conv_gemm 3x3 {d}_context_conv2+context_conv3_1", c31)
            c32, = self.conv(cur[d + "_context_conv3_1_relu"], [d + "_context_conv3_2"], [(16, True)])
            yield emit(d + "_concat_relu", f"k_conv_gemm 3x3 {d} (three launches into the concat)", np.concatenate([det, c2, c32], axis=1))
        for lv, stride in (("c3", 32), ("c2", 16), ("c1", 8)):
            cat = cur[f"rf_{lv}_det_concat_relu"]
            yield f"heads_stride{stride}", "k_head_decode", self.heads(cat, stride), cat


TENSORS = 43        # the tensors walk() yields before the heads: relu0, 13 depthwise + 13 pointwise, 3 laterals, 2 FPN sums,
                    # 2 aggr convs, and per SSH level the two context tensors and the concat
