"""Float64 restatement of the rounding of every step of the FP16 tensor-core engine (RF_PREC_FP16).  Test infrastructure --
see ``oracle/__init__.py``.

Each step is restated from its inputs to its FP16 output, so that a test can continue from the engine's own materialised
tensors: error never builds up over the network, and a wrong tap, halo row, bias or ReLU shows at the step that made it.
Every value is held in float64; a tensor is an interval ``Iv(lo, hi, mid)`` of FP16 (or, inside the stem, FP32) values per
element: ``lo == hi`` where the kernel spells its arithmetic out, a few values wide after a tensor-core GEMM.  ``mid`` is
the float64 midpoint of the exact sum carried through the same epilogue (for statistics only).

Exact steps (the result is one value, restated operation by operation):

* FP32 ``fmaf``: the product of two FP32 values is exact in float64 (48 bits), the sum is rounded to odd in float64, then
  to nearest FP32 -- exact because 53 >= 24 + 2.  ``__hfma2`` the same way to FP16.  An FP32 add, subtract or divide of
  two FP32 values is computed in float64 and rounded to FP32: double rounding is innocuous for 53 >= 2 * 24 + 2.
* depthwise 3x3 of the per-layer kernels (``common.cuh:61-107``: ``dw_bias8`` FP32 bias first, ``fmaf`` over the taps in
  (ky, kx) order with the FP16-rounded weights of ``dw_weight_f16``, ``dw_relu_h8`` ReLU and RN to FP16);
* the FPN merge with HFMA2 (``kernels_simt.cuh`` ``k_fpn_merge_h2``, ``tc_conv.cuh:276-296`` the UPADD staging): lateral,
  then the up-to-four deconvolution taps (i, j) = (i_hi, j_hi), (i_hi, j_hi - 1), (i_hi - 1, j_hi), (i_hi - 1, j_hi - 1);
* the CUDA-core stem ``k_stem`` (``kernels_simt.cuh:288-420``, ``RF_FLAG_SIMT_STEM``): FP32 ``fmaf`` chains throughout;
* the predictor dots of ``k_head_decode`` (``postproc.cu:73-85``): ``__fmaf_rn`` from the bias over the 64 channels.

The tensor-core model (the only arithmetic the code does not spell out: the PTX ISA leaves the order and the intermediate
rounding of ``wgmma``'s FP32 accumulation unspecified):

* every ``wgmma`` K step adds its 16 exact FP16 x FP16 products to the FP32 accumulator: 17 addends.  Its error is at most
  ``17 * 2**-22 * (the largest addend's magnitude)``: each addend truncated 23 bits below the largest one's leading bit,
  with one bit of slack, plus a final rounding in any direction.  The first step of a GEMM starts from zero (16 addends).
* the largest addend is bounded by ``max(|S| + E, P)``: S the exact partial sum of the earlier steps, E their error bound,
  P the sum of this step's |products| (an upper bound of the largest product).
* a GEMM's error is the sum of its steps' errors; the hi + lo weight pieces of conv0 are two steps per K step, in the
  order the kernel issues them (``stem_tc.cuh:193-200``).  Float64 evaluation adds ``(K + 2 T) * 2**-53 * sum|a w|``.
* then the epilogue (``tc_conv.cuh:131-149``, ``stem_tc.cuh:209-222, 315-330``): the accumulator is an FP32 value inside
  the interval, the FP32 bias add, ReLU and RN to FP16 are monotone, so the output is an interval of FP16 values.

This model is not a measurement of the hardware: nobody has measured how the H100 orders and rounds ``wgmma``'s
accumulation.  A test that finds an engine value outside its interval has found either a kernel bug or an H100 whose
accumulation exceeds the model; the first difference tells which.

Class probabilities: ``expf`` within its documented 2 ulp (CUDA C Programming Guide, mathematical functions), then RN
subtract, add and divide (``postproc_dev.cuh:22-28``); the regression and landmark deltas are exact.

Tile chains (``tile_chain.cuh``: the latency plans): the conv stages are the same GEMMs as ``k_tc_conv_staged``
(``tile_chain.cuh:233-252``, epilogue ``:197-230``), the FPN merge pre-stage is the same HFMA2 sum (``:352-386``); the
predictors differ (``:423-446``): one N = 32 GEMM with hi + lo FP16 weight pieces issued hi, lo per K step
(``plan_tile.cu:104-125``), then an FP32 add of the bias: every head value, deltas included, is an interval.

The FP32 engine and FP16 with ``RF_FLAG_NO_TENSORCORE`` (the SIMT plans, every step exact) are restated in
``oracle/fp32_steps.py``, from the primitives and head functions of this file.
"""
from __future__ import annotations

from typing import Callable, Dict, NamedTuple, Optional

import numpy as np

from .mnet_numpy import folded_params

F64 = np.float64
TC_STEP = 17 * 2.0 ** -22      # error of one wgmma K step, relative to its largest addend
STRIDE2 = (3, 7, 11, 23)       # depthwise layers of stride 2 (prototxt)


# ---- exact primitives ---------------------------------------------------------------------------------------------------
def rn32(x):
    """Round float64 to nearest FP32 (ties to even, subnormals included), as float64."""
    with np.errstate(over="ignore"):
        return np.asarray(x, F64).astype(np.float32).astype(F64)


def rn16(x):
    """Round float64 to nearest FP16 (ties to even, subnormals, overflow to inf), as float64: numpy rounds once, from the
    float64 bits."""
    with np.errstate(over="ignore"):
        return np.asarray(x, F64).astype(np.float16).astype(F64)


def odd_sum(a, b):
    """a + b rounded to odd in float64 (TwoSum, then the odd neighbour where the sum is inexact): rounding this to a format
    of p <= 51 bits gives the correctly rounded sum."""
    a, b = np.asarray(a, F64), np.asarray(b, F64)
    s = a + b
    bp = s - a
    err = (a - (s - bp)) + (b - bp)
    fix = (err != 0) & ((s.view(np.int64) & 1) == 0)
    return np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)


def fma32(x, w, acc):
    """fmaf(x, w, acc) of FP32 values: one rounding."""
    return rn32(odd_sum(np.asarray(x, F64) * w, acc))


def hfma16(u, w, acc):
    """__hfma2 lane: u * w + acc of FP16 values, one rounding to FP16."""
    return rn16(odd_sum(np.asarray(u, F64) * w, acc))


def add32(a, b):
    return rn32(np.asarray(a, F64) + b)


def floor32(x):
    """Largest FP32 value <= x."""
    x = np.asarray(x, F64)
    r = rn32(x)
    return np.where(r > x, np.nextafter(r.astype(np.float32), np.float32(-np.inf)).astype(F64), r)


def ceil32(x):
    """Smallest FP32 value >= x."""
    x = np.asarray(x, F64)
    r = rn32(x)
    return np.where(r < x, np.nextafter(r.astype(np.float32), np.float32(np.inf)).astype(F64), r)


def f16_ordinal(x):
    """Position of each FP16 value on the number line (consecutive values differ by 1): widths in ulps."""
    bits = rn16(x).astype(np.float16).view(np.int16).astype(np.int32)
    return np.where(bits < 0, -(bits & 0x7FFF), bits)


class Iv(NamedTuple):
    lo: np.ndarray
    hi: np.ndarray
    mid: np.ndarray

    @staticmethod
    def exact(x):
        x = np.asarray(x, F64)
        return Iv(x, x, x)


# ---- weight images, as the plans pack them ------------------------------------------------------------------------------
def tc_weights(w):
    """pack_tc_weights (plan_fp.cu:50-74): FP16 RN of the folded FP32 weights, as a GEMM matrix [K = (tap, cin)][cout]."""
    o, ci, k, _ = w.shape
    return rn16(w.transpose(2, 3, 1, 0).reshape(k * k * ci, o))


def hi_lo(w):
    """The two FP16 pieces of an FP32 weight (plan_fp.cu:144-150): hi = RN16(w), lo = RN16(w - hi) with the difference in
    FP32."""
    hi = rn16(w)
    return hi, rn16(rn32(np.asarray(w, F64) - hi))


def dw_weights16(w):
    """dw_weight_f16 (common.cuh:69): the FP32 depthwise weights [C][9] rounded to FP16, used as FP32 values."""
    return rn16(w.reshape(w.shape[0], 9))


def up_weights16(w):
    """The FPN deconvolution weights [C][4][4] as FP16 (plan_fp.cu:271-273, tc_conv.cuh:189)."""
    return rn16(w.reshape(-1, 4, 4))


# ---- the tensor-core GEMM -----------------------------------------------------------------------------------------------
def tc_gemm(a: Iv, steps, rows=1 << 15):
    """a: (M, K) interval of FP16 A operands; steps: [(k0, k1, W[k1-k0][N])] in the order the kernel issues its wgmma, each
    16 K wide.  Returns the interval (lo, hi) of the FP32 accumulator in float64, and the exact midpoint."""
    M = a.lo.shape[0]
    N = steps[0][2].shape[1]
    lo, hi, mid = (np.empty((M, N)) for _ in range(3))
    ksum = sum(k1 - k0 for k0, k1, _ in steps)
    exact = a.lo is a.hi
    for r0 in range(0, M, rows):
        al_all = a.lo[r0:r0 + rows].astype(F64)
        ah_all = al_all if exact else a.hi[r0:r0 + rows].astype(F64)
        m = al_all.shape[0]
        s_lo, e, tot = np.zeros((m, N)), np.zeros((m, N)), np.zeros((m, N))
        s_hi = s_lo if exact else np.zeros((m, N))
        for t, (k0, k1, w) in enumerate(steps):
            al, ah = al_all[:, k0:k1], ah_all[:, k0:k1]
            p = (np.abs(al) if exact else np.maximum(np.abs(al), np.abs(ah))) @ np.abs(w)
            big = p if t == 0 else np.maximum(np.maximum(np.abs(s_lo), np.abs(s_hi)) + e, p)
            e += TC_STEP * big
            if exact:
                s_lo += al @ w
            else:
                wp, wn = np.maximum(w, 0), np.minimum(w, 0)
                s_lo += al @ wp + ah @ wn
                s_hi += ah @ wp + al @ wn
            tot += p
        e += (ksum + 2 * len(steps)) * 2.0 ** -53 * tot
        lo[r0:r0 + m], hi[r0:r0 + m], mid[r0:r0 + m] = s_lo - e, s_hi + e, 0.5 * (s_lo + s_hi)
    return lo, hi, mid


def k_steps(w16):
    """The wgmma K steps of a GEMM whose B image is w16 [K][N] (K a multiple of 16), in K order."""
    return [(k, k + 16, w16[k:k + 16]) for k in range(0, w16.shape[0], 16)]


def pad_k(x, axis):
    """Zero-pad K (the given axis) to a multiple of 16 (the kernels' K padding)."""
    k = x.shape[axis]
    pad = [(0, 0)] * x.ndim
    pad[axis] = (0, (k + 15) // 16 * 16 - k)
    return np.pad(x, pad) if pad[axis][1] else x


def epilogue(lo, hi, mid, bias, relu, out=rn16):
    """FP32 accumulator interval -> + FP32 bias, ReLU, RN (tc_conv.cuh:144-146): monotone, so endpoints map to endpoints."""
    lo, hi = add32(floor32(lo), bias), add32(ceil32(hi), bias)
    mid = np.asarray(mid, F64) + bias
    if relu:
        lo, hi, mid = np.maximum(lo, 0), np.maximum(hi, 0), np.maximum(mid, 0)
    return Iv(out(lo), out(hi), out(mid))


# ---- layouts -------------------------------------------------------------------------------------------------------------
def nhwc(x):
    return np.ascontiguousarray(np.moveaxis(x, 1, -1))


def nchw(x):
    return np.ascontiguousarray(np.moveaxis(x, -1, 1))


def im2col3(x):
    """x: (n, h, w, c) -> (n*h*w, 9*c), K ordered (tap, channel), zero padding 1, stride 1 (the shifted descriptors of
    k_tc_conv_staged)."""
    n, h, w, c = x.shape
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0)))
    cols = np.empty((n, h, w, 9, c), x.dtype)
    for t in range(9):
        cols[:, :, :, t] = xp[:, t // 3:t // 3 + h, t % 3:t % 3 + w]
    return cols.reshape(n * h * w, 9 * c)


def _both(f, x: Iv):
    """Apply a layout function to lo and hi (and mid), sharing the work where the interval is one value."""
    lo = f(x.lo)
    return Iv(lo, lo, lo) if x.lo is x.hi else Iv(lo, f(x.hi), f(x.mid))


# ---- steps ---------------------------------------------------------------------------------------------------------------
def depthwise(x: Iv, w, b, stride, weights16=True):
    """Depthwise 3x3 (pad 1) of NCHW x: FP32 bias, fmaf over the taps in (ky, kx) order, ReLU (common.cuh:61-107, stem_tc.cuh
    224-245 and kernels_simt.cuh:369-382).  weights16: the FP16-rounded weights of the per-layer kernels; the stems use the
    FP32 ones.  Returns the FP32 result after ReLU (exact; an interval only where x is one)."""
    wt = dw_weights16(w) if weights16 else np.asarray(w, F64).reshape(w.shape[0], 9)
    n, c, h, wd = x.lo.shape
    oh, ow = h // stride, wd // stride
    pad = lambda a: np.pad(a, ((0, 0), (0, 0), (1, 1), (1, 1)))
    xl = pad(x.lo)
    xh = xl if x.lo is x.hi else pad(x.hi)
    lo = np.broadcast_to(np.asarray(b, F64)[None, :, None, None], (n, c, oh, ow)).copy()
    hi = lo.copy() if xh is not xl else lo
    for t in range(9):
        dy, dx = t // 3, t % 3
        wv = wt[None, :, t, None, None]
        sl = lambda a: a[:, :, dy:dy + stride * oh:stride, dx:dx + stride * ow:stride]
        if xh is xl:
            lo = fma32(sl(xl), wv, lo)
            hi = lo
        else:
            pos = wv >= 0
            lo, hi = fma32(np.where(pos, sl(xl), sl(xh)), wv, lo), fma32(np.where(pos, sl(xh), sl(xl)), wv, hi)
    lo, hi = np.maximum(lo, 0), np.maximum(hi, 0)
    return Iv(lo, hi, 0.5 * (lo + hi)) if hi is not lo else Iv(lo, lo, lo)


def gemm_conv(x: Iv, ws, bs, outs):
    """k_tc_conv_staged (and the pointwise GEMM of the depthwise+pointwise kernels): the convs of `ws` (1x1 or 3x3, pad 1,
    stride 1, sharing the input) concatenated along N, FP16 weights, one wgmma K step per 16 of K = (tap, cin); the output
    channels split into `outs` = [(n_channels, relu)] (TcOut's two destinations).  Returns one Iv (NCHW) per segment."""
    n, c, h, wd = x.lo.shape
    k = ws[0].shape[2]
    w16 = np.concatenate([tc_weights(w) for w in ws], axis=1)
    bias = np.concatenate([np.asarray(b, F64) for b in bs])
    lay = (lambda a: im2col3(nhwc(a).astype(np.float32))) if k == 3 else (lambda a: nhwc(a).reshape(-1, c))
    a = _both(lambda v: pad_k(lay(v), 1), x)
    lo, hi, mid = tc_gemm(a, k_steps(pad_k(w16, 0)))
    res, o0 = [], 0
    for cn, relu in outs:
        sl = slice(o0, o0 + cn)
        r = epilogue(lo[:, sl], hi[:, sl], mid[:, sl], bias[sl], relu)
        res.append(Iv(*(nchw(v.reshape(n, h, wd, cn)) for v in r)))
        o0 += cn
    return res


def dw_pw(x: Iv, dw, pw, stride):
    """k_tc_dwpw_staged / k_tc_dwpw_2d: the depthwise exactly, its FP16 output as the A operand, the pointwise GEMM."""
    d = depthwise(x, dw["w"], dw["b"], stride)
    a = Iv(rn16(d.lo), rn16(d.hi), rn16(d.mid))
    return gemm_conv(a, [pw["w"]], [pw["b"]], [(pw["w"].shape[0], True)])[0]


def merge_h2(lat: Iv, up: Iv, up_w):
    """k_fpn_merge_h2 (and the UPADD staging of k_tc_conv_staged): lateral + crop(deconv k4 s2 p1 of up), HFMA2 on FP16
    lanes, taps (i_hi, j_hi), (i_hi, j_hi - 1), (i_hi - 1, j_hi), (i_hi - 1, j_hi - 1); a tap outside the coarse map adds 0."""
    w = up_weights16(up_w)
    n, c, h, wd = lat.lo.shape
    uh, uw = up.lo.shape[2:]
    y, x = np.arange(h), np.arange(wd)
    lo, hi = lat.lo.astype(F64), lat.hi.astype(F64)
    for di in range(2):
        i = (y + 1) // 2 - di
        ky = y - 2 * i + 1
        for dj in range(2):
            j = (x + 1) // 2 - dj
            kx = x - 2 * j + 1
            ok = ((i >= 0) & (i < uh))[:, None] & ((j >= 0) & (j < uw))[None, :]
            ic, jc = np.clip(i, 0, uh - 1), np.clip(j, 0, uw - 1)
            ul = np.where(ok, up.lo[:, :, ic][:, :, :, jc], 0.0)
            uhh = ul if up.lo is up.hi else np.where(ok, up.hi[:, :, ic][:, :, :, jc], 0.0)
            wv = w[:, ky][:, :, kx][None]
            pos = wv >= 0
            lo = hfma16(np.where(pos, ul, uhh), wv, lo)
            hi = lo if (up.lo is up.hi and lat.lo is lat.hi) else hfma16(np.where(pos, uhh, ul), wv, hi)
    return Iv(lo, lo, lo) if hi is lo else Iv(lo, hi, 0.5 * (lo + hi))


def _stem_image_cols(img):
    """u8 BGR (n, H, W, 3) -> conv0 im2col (n*H/2*W/2, 27), k = (ky*3 + kx)*3 + c_bgr, stride 2, pad 1 (stem_tc.cuh:139-177)."""
    n, H, W, _ = img.shape
    oh, ow = H // 2, W // 2
    xp = np.pad(img.astype(np.float32), ((0, 0), (1, 1), (1, 1), (0, 0)))
    cols = np.empty((n, oh, ow, 9, 3), np.float32)
    for t in range(9):
        cols[:, :, :, t] = xp[:, t // 3:t // 3 + 2 * oh:2, t % 3:t % 3 + 2 * ow:2]
    return cols.reshape(n * oh * ow, 27)


def _conv0_matrix(w):
    """conv0 weights (8, 3 RGB, 3, 3) -> [27][8] with k = tap*3 + c_bgr (plan_net.cu:122-124)."""
    return np.asarray(w, F64)[:, ::-1].transpose(2, 3, 1, 0).reshape(27, 8)


def stem_tc(img, c0, dw, pw):
    """k_stem_tc<__half> (stem_tc.cuh): conv0 on tensor cores with hi + lo weights (an interval), + bias and ReLU in FP32,
    the FP32 depthwise (FP32 weights), FP16 A operand, the pointwise GEMM.  img: u8 (n, H, W, 3) BGR.  Returns NCHW."""
    n, H, W, _ = img.shape
    oh, ow = H // 2, W // 2
    a = pad_k(_stem_image_cols(img), 1)
    hi, lo = (pad_k(v, 0) for v in hi_lo(_conv0_matrix(c0["w"])))
    steps = [(0, 16, hi[:16]), (16, 32, hi[16:]), (0, 16, lo[:16]), (16, 32, lo[16:])]     # part outer, K step inner
    s_lo, s_hi, s_mid = tc_gemm(Iv(a, a, None), steps)
    r = epilogue(s_lo, s_hi, s_mid, np.asarray(c0["b"], F64), True, out=lambda v: v)      # conv0 output stays FP32
    x = Iv(*(nchw(v.reshape(n, oh, ow, 8)) for v in r))
    d = depthwise(x, dw["w"], dw["b"], 1, weights16=False)
    d = Iv(rn16(d.lo), rn16(d.hi), rn16(d.mid))
    return gemm_conv(d, [pw["w"]], [pw["b"]], [(16, True)])[0]


def stem_simt(img, c0, dw, pw):
    """k_stem<__half> (kernels_simt.cuh:288-420, RF_FLAG_SIMT_STEM): every layer an FP32 fmaf chain, exact.  Returns NCHW."""
    n, H, W, _ = img.shape
    oh, ow = H // 2, W // 2
    cols = _stem_image_cols(img).astype(F64)
    w0 = _conv0_matrix(c0["w"])
    acc = np.broadcast_to(np.asarray(c0["b"], F64), (cols.shape[0], 8)).copy()
    for k in range(27):                   # ky outer, then the 9 bytes kx * 3 + c_bgr of the row (kernels_simt.cuh:347-356)
        acc = fma32(cols[:, k:k + 1], w0[k][None], acc)
    x = Iv.exact(nchw(np.maximum(acc, 0).reshape(n, oh, ow, 8)))
    d = depthwise(x, dw["w"], dw["b"], 1, weights16=False).lo
    wp = np.asarray(pw["w"], F64)[:, :, 0, 0]                              # (16, 8)
    o = np.broadcast_to(np.asarray(pw["b"], F64)[None, :, None, None], (n, 16, oh, ow)).copy()
    for c in range(8):
        o = fma32(d[:, c:c + 1], wp[None, :, c, None, None], o)
    return Iv.exact(rn16(np.maximum(o, 0)))


def head_dots(cat, w, b):
    """The 32 predictor outputs of one level (k_head_decode's dot): acc = bias, __fmaf_rn over the 64 channels in order.
    cat: NCHW FP16 values; w: (32, 64) FP32; returns (n, 32, h, w) exact."""
    x = np.asarray(cat, F64)
    acc = np.broadcast_to(np.asarray(b, F64)[None, :, None, None], (x.shape[0], 32) + x.shape[2:]).copy()
    for c in range(64):
        acc = fma32(x[:, c:c + 1], np.asarray(w, F64)[None, :, c, None, None], acc)
    return acc


def _expf(d):
    """The FP32 interval holding expf(d) (CUDA: at most 2 ulp from exp(d))."""
    r = np.exp(np.asarray(d, F64))
    _, e = np.frexp(r)
    ulp = np.ldexp(1.0, np.maximum(e - 24, -149))
    return np.maximum(floor32(r * (1 - 2.0 ** -50) - 2 * ulp), 0), ceil32(r * (1 + 2.0 ** -50) + 2 * ulp)


def cls_prob(s):
    """softmax_pair (postproc_dev.cuh:22-28) over the (bg, face) score pairs (a, a + 2) of s (n, 4, h, w): the interval of
    each of the 4 probabilities [bg0, bg1, face0, face1]."""
    lo, hi = np.empty_like(s), np.empty_like(s)
    for a in range(2):
        sb, sf = s[:, a], s[:, a + 2]
        m = np.maximum(sb, sf)
        e0, e1 = _expf(add32(sb, -m)), _expf(add32(sf, -m))
        s_lo, s_hi = add32(e0[0], e1[0]), add32(e0[1], e1[1])
        for ch, e in ((a, e0), (a + 2, e1)):
            lo[:, ch], hi[:, ch] = rn32(e[0] / s_hi), rn32(e[1] / s_lo)
    return lo, hi


def cls_prob_iv(s_lo, s_hi):
    """cls_prob over interval scores: each probability of a pair rises with its own score and falls with the other's, and the
    rounded softmax_pair keeps that order (RN and the expf interval are monotone), so the corners bound it."""
    a = s_hi.copy(); a[:, 2:] = s_lo[:, 2:]          # background high, face low
    b = s_lo.copy(); b[:, 2:] = s_hi[:, 2:]          # background low, face high
    (a_lo, a_hi), (b_lo, b_hi) = cls_prob(a), cls_prob(b)
    lo, hi = b_lo.copy(), a_hi.copy()                # background: lowest at b, highest at a
    lo[:, 2:], hi[:, 2:] = a_lo[:, 2:], b_hi[:, 2:]  # face: lowest at a, highest at b
    return lo, hi


def chain_heads(cat, w, b):
    """A tile chain's TCH_HEAD stage (tile_chain.cuh:423-459): cat (NCHW FP16 values) times the hi + lo FP16 pieces of the
    FP32 predictor weights w (32, 64), issued hi, lo per 16-channel K step (tile_chain.cuh:241-248), + FP32 bias (__fadd_rn),
    softmax_pair.  Returns (cls (lo, hi), bbox (lo, hi), landmarks (lo, hi)), NCHW."""
    n, c, h, wd = cat.shape
    hi, lo = hi_lo(np.asarray(w, F64).T)                                   # (64, 32)
    steps = []
    for k0 in range(0, 64, 16):
        steps += [(k0, k0 + 16, hi[k0:k0 + 16]), (k0, k0 + 16, lo[k0:k0 + 16])]
    a = nhwc(np.asarray(cat, F64)).reshape(-1, c)
    s_lo, s_hi, s_mid = tc_gemm(Iv(a, a, None), steps)
    v = epilogue(s_lo, s_hi, s_mid, np.asarray(b, F64), False, out=lambda x: x)
    v_lo, v_hi = (nchw(t.reshape(n, h, wd, 32)) for t in (v.lo, v.hi))
    return cls_prob_iv(v_lo[:, :4], v_hi[:, :4]), (v_lo[:, 4:12], v_hi[:, 4:12]), (v_lo[:, 12:], v_hi[:, 12:])


# ---- the network, continued from the engine's own tensors ---------------------------------------------------------------
class Fp16Steps:
    """The FP16 tensor-core plan of one caffemodel, step by step.  ``walk`` computes the interval of every tensor of the
    per-layer (throughput) plans from its nearest materialised ancestors."""

    def __init__(self, caffemodel: str):
        self.p = folded_params(caffemodel)

    def stem(self, img, simt=False):
        c0, dw, pw = (self.p[f"mobilenet0_conv{i}_fwd"] for i in range(3))
        return (stem_simt if simt else stem_tc)(img, c0, dw, pw)

    def pair(self, x: Iv, i):
        return dw_pw(x, self.p[f"mobilenet0_conv{i}_fwd"], self.p[f"mobilenet0_conv{i + 1}_fwd"], 2 if i in STRIDE2 else 1)

    def conv(self, x: Iv, names, outs):
        return gemm_conv(x, [self.p[n]["w"] for n in names], [self.p[n]["b"] for n in names], outs)

    def merge(self, lat: Iv, up: Iv, level):
        return merge_h2(lat, up, self.p["rf_c3_upsampling" if level == 0 else "rf_c2_upsampling"]["w"])

    def heads(self, cat, stride, chain=False):
        """-> (cls interval (lo, hi), bbox deltas, landmark deltas) of one level, NCHW: k_head_decode's exact deltas, or
        (chain) the intervals of a tile chain's predictor stage."""
        names = [f"face_rpn_{k}_stride{stride}" for k in ("cls_score", "bbox_pred", "landmark_pred")]
        w = np.concatenate([self.p[n]["w"][:, :, 0, 0] for n in names])
        b = np.concatenate([self.p[n]["b"] for n in names])
        if chain:
            return chain_heads(cat, w, b)
        s = head_dots(cat, w, b)
        return cls_prob(s[:, :4]), s[:, 4:12], s[:, 12:32]

    def walk(self, img, fetch: Callable[[str, Iv], Optional[np.ndarray]], simt_stem=False, tc_dw=(), chain_heads=False):
        """Every step of the plan, each continued from the engine's materialised tensors: fetch(name, interval) returns the
        engine's tensor (NCHW) or None where the plan does not materialise it.  Yields (tensor, step, Iv, engine value or None) in
        step order; the three levels' heads come last as ("heads_stride{s}", step, (cls (lo, hi), bbox, lm), cat).
        tc_dw: the depthwise layers the plan runs on tensor cores inside a tile chain -- no plan does, so any layer named here
        is an error rather than a step checked against the wrong arithmetic; chain_heads: the predictors run in the SSH chains."""
        if tc_dw:
            raise ValueError(f"no plan runs depthwise layers {sorted(tc_dw)} on tensor cores; their steps have no restatement")
        cur: Dict[str, Iv] = {}

        def emit(name, step, iv):
            got = fetch(name, iv)
            cur[name] = iv if got is None else Iv.exact(got)
            return name, step, iv, got

        yield emit("mobilenet0_relu2_fwd", "k_stem" if simt_stem else "k_stem_tc", self.stem(img, simt_stem))
        for i in range(3, 27, 2):
            yield emit(f"mobilenet0_relu{i + 1}_fwd", f"k_tc_dwpw dw{i}+pw{i + 1}", self.pair(cur[f"mobilenet0_relu{i - 1}_fwd"], i))
        lat = {"c3": ("rf_c3_lateral", 26), "c2": ("rf_c2_lateral", 22), "c1": ("rf_c1_red_conv", 10)}
        for lv, (nm, src) in lat.items():
            yield emit(nm + "_relu", f"k_tc_conv {nm}", self.conv(cur[f"mobilenet0_relu{src}_fwd"], [nm], [(64, True)])[0])
        for lv, ssh_in in (("c3", "rf_c3_lateral_relu"), ("c2", "rf_c2_aggr_relu"), ("c1", "rf_c1_aggr_relu")):
            if lv != "c3":
                level = 0 if lv == "c2" else 1
                lat_t = "rf_c2_lateral_relu" if lv == "c2" else "rf_c1_red_conv_relu"
                up_t = "rf_c3_lateral_relu" if lv == "c2" else "rf_c2_aggr_relu"
                yield emit(f"_plus{level}", "fpn merge (HFMA2)", self.merge(cur[lat_t], cur[up_t], level))
                yield emit(ssh_in, f"k_tc_conv rf_{lv}_aggr", self.conv(cur[f"_plus{level}"], [f"rf_{lv}_aggr"], [(64, True)])[0])
            p = f"rf_{lv}_det"
            det, ctx1 = self.conv(cur[ssh_in], [p + "_conv1", p + "_context_conv1"], [(32, True), (16, True)])
            yield emit(p + "_context_conv1_relu", f"k_tc_conv {p}_conv1+context_conv1", ctx1)
            c2, c31 = self.conv(cur[p + "_context_conv1_relu"], [p + "_context_conv2", p + "_context_conv3_1"], [(16, True), (16, True)])
            yield emit(p + "_context_conv3_1_relu", f"k_tc_conv {p}_context_conv2+context_conv3_1", c31)
            c32, = self.conv(cur[p + "_context_conv3_1_relu"], [p + "_context_conv3_2"], [(16, True)])
            cat = Iv(*(np.concatenate(v, axis=1) for v in zip(det, c2, c32)))
            yield emit(p + "_concat_relu", f"k_tc_conv {p} (concat + ReLU)", cat)
        for lv, stride in (("c3", 32), ("c2", 16), ("c1", 8)):
            c = cur[f"rf_{lv}_det_concat_relu"]
            assert c.lo is c.hi, "the heads are checked from a materialised concat"
            yield (f"heads_stride{stride}", "k_tile_chain TCH_HEAD" if chain_heads else "k_head_decode",
                   self.heads(c.lo, stride, chain_heads), c.lo)


# ---- teeth: what the check must reject ---------------------------------------------------------------------------------
def outside(got, iv: Iv):
    return (got < iv.lo) | (got > iv.hi)


def mutations(x: Iv, dw, pw, stride, good):
    """Realistic kernel mistakes on one depthwise+pointwise step whose correct FP16 output is `good` (NCHW), as (name, mutated
    output): large ones (a whole column, row, chunk or tile) and small ones that move a few elements a little (one output
    of one tile, one channel's bias)."""
    n, c, h, w = good.shape
    out = []
    dw_m = dict(dw, w=dw["w"].copy())
    dw_m["w"][:, 0, 2, 2] = 0                                       # tap (2, 2) dropped ...
    no22 = dw_pw(x, dw_m, pw, stride).mid
    t = good.copy()
    t[:, :, :, w // 2] = no22[:, :, :, w // 2]                       # ... in one output column
    out.append((f"tap (2, 2) dropped in column {w // 2}", t))
    dw_g = dict(dw, w=dw["w"].copy())
    dw_g["w"][:8, 0, 2, 2] = 0                                      # one thread's 8-channel group (dw_stencil_block) ...
    t = good.copy()
    t[1, :, h // 2, w // 2] = dw_pw(x, dw_g, pw, stride).mid[1, :, h // 2, w // 2]     # ... at one output of one tile
    out.append((f"tap (2, 2) of channels 0..7 dropped at one output (image 1, y {h // 2}, x {w // 2})", t))
    t = good.copy()
    t[:, :, h // 2] = good[:, :, h // 2 - 1]
    out.append(("one output row from the row above (stale halo)", t))
    pw_m = dict(pw, b=pw["b"].copy())
    pw_m["b"][16:32] = pw["b"][17:33] if len(pw["b"]) > 32 else np.roll(pw["b"][16:32], -1)
    out.append(("bias of channel n + 1 in channels 16..31", dw_pw(x, dw, pw_m, stride).mid))
    pw_m = dict(pw, b=pw["b"].copy())
    d = np.abs(pw["b"][1:16] - pw["b"][:15])
    ch = int(np.argmin(np.where(d > 0, d, np.inf)))                  # the channel whose neighbour's bias is closest
    pw_m["b"][ch] = pw["b"][ch + 1]
    out.append((f"bias of channel {ch + 1} used for channel {ch} only", dw_pw(x, dw, pw_m, stride).mid))
    dd = depthwise(x, dw["w"], dw["b"], stride)
    a = Iv(rn16(dd.lo), rn16(dd.hi), rn16(dd.mid))
    pre = gemm_conv(a, [pw["w"]], [pw["b"]], [(len(pw["b"]), False)])[0].mid
    ch = int(np.argmin(pre.min(axis=(0, 2, 3))))
    t = good.copy()
    t[:, ch] = pre[:, ch]
    out.append((f"ReLU missing on channel {ch}", t))
    t = good.copy()
    t[1, :, :8, :16] = good[0, :, :8, :16]
    out.append(("image 1's first 8x16 tile computed from image 0", t))
    return out
