"""Host side of the SIMT step check (oracle/fp32_steps.py): its fast fmaf against the exact one, each step against a literal
scalar transcription of its kernel (thread mapping, tiles, chunks, bounds, packing) and against a plain float64 convolution
within an order-free error bound, its teeth (kernel mistakes the check must reject), and a walk of the whole network.  The
guard that the GPU sweep still reaches every SIMT kernel is host-only too; it sits with the sweep's case table in
tests/test_gpu_fp32_steps.py."""
import math
import struct

import numpy as np
import pytest

from conftest import caffemodel
from oracle import fp16_steps as fs
from oracle import fp32_steps as f3
from oracle.mnet_numpy import folded_params

U32 = 2.0 ** -24


# ---- scalar arithmetic: Python floats, no numpy ------------------------------------------------------------------------
def fmaf(x, w, a):
    """fmaf of FP32 values: the exact product (48 bits) plus a, rounded to odd in float64 (TwoSum), then to FP32."""
    p = x * w
    s = p + a
    bp = s - p
    err = (p - (s - bp)) + (a - bp)
    if err != 0 and not struct.unpack("<q", struct.pack("<d", s))[0] & 1:
        s = math.nextafter(s, math.inf if err > 0 else -math.inf)
    return struct.unpack("<f", struct.pack("<f", s))[0]


def f32(x):
    return struct.unpack("<f", struct.pack("<f", x))[0]


def f16(x):
    return struct.unpack("<e", struct.pack("<e", x))[0]


STORES = {"float": (fs.rn32, f32), "half": (fs.rn16, f16)}


def _rand32(rng, shape, scale=1.0):
    return fs.rn32(rng.standard_normal(shape) * scale)


def _act(rng, shape, store=fs.rn32, signed=False):
    """Activations as a stored tensor holds them: post-ReLU (or signed), a third of them zero."""
    v = rng.standard_normal(shape) * 2
    return store(fs.rn32(v if signed else np.abs(v) * (rng.random(shape) < 0.67)))


# ---- the fast path ------------------------------------------------------------------------------------------------------
def test_fma32_fast_and_fma_chain_equal_fma32():
    """fma32_fast and fma_chain (float64 sum once, fma32 where it is an FP32 midpoint or below the normal range) against
    fma32 on random, cancelling, midpoint and subnormal operands, and the scalar fmaf of this file against fma32."""
    rng = np.random.default_rng(11)
    n = 200_000
    x, w = _rand32(rng, n) * 2.0 ** rng.integers(-20, 20, n), _rand32(rng, n)
    acc = fs.rn32(rng.standard_normal(n) * 2.0 ** rng.integers(-40, 40, n))
    near = rng.random(n) < 0.3                                    # cancelling sums
    acc[near] = fs.rn32(-x[near] * w[near] * (1 + rng.integers(-3, 4, near.sum()) * 2.0 ** -23))
    # float64 sums that land exactly on an FP32 midpoint while the exact sum does not (the double-rounding cases):
    # x * w = +-2^-24 (1 - 2^-46), 2^-70 short of half an ulp of acc = 1 + k 2^-23, below float64's resolution there
    k = rng.integers(0, 1 << 20, 2000)
    mid_acc = 1 + k * 2.0 ** -23
    mid_x = np.full(2000, 2.0 ** -24 * (1 - 2.0 ** -23))
    mid_w = rng.choice([-1.0, 1.0], 2000) * (1 + 2.0 ** -23)
    tiny = [(2.0 ** -100, 1.5 * 2.0 ** -49, 0.0), (2.0 ** -126, -0.5, 2.0 ** -126), (2.0 ** -75, 2.0 ** -75, -(2.0 ** -149)),
            (3 * 2.0 ** -76, 2.0 ** -74, 2.0 ** -149), (-0.0, 1.0, -0.0), (1.0, -1.0, 1.0)]
    x = np.concatenate([x, mid_x, [t[0] for t in tiny]])
    w = np.concatenate([w, mid_w, [t[1] for t in tiny]])
    acc = np.concatenate([acc, mid_acc, [t[2] for t in tiny]])
    want = fs.fma32(x, w, acc)
    assert np.array_equal(f3.fma32_fast(x, w, acc), want)
    assert f3._risky(x * w + acc).sum() >= 2000                         # the midpoint cases took the exact path
    assert not np.array_equal(fs.rn32(x * w + acc), want)               # ... which plain float64 gets wrong
    # the GEMM chain: one (M, N) accumulator, every step an outer product
    m = 257
    a = np.concatenate([x[:m], mid_x[:1]])
    wv = np.concatenate([w[:m], mid_w[:1]])
    acc2 = acc[:(m + 1)][:, None] * np.ones((1, m + 1))
    acc2[-1, -1] = mid_acc[0]
    got = f3.fma_chain(acc2, [(a, wv)])
    assert np.array_equal(got, fs.fma32(a[:, None], wv[None, :], acc2))
    for i in range(0, len(x), 997):
        assert fmaf(float(x[i]), float(w[i]), float(acc[i])) == want[i], i


# ---- literal scalar transcriptions of the kernels ---------------------------------------------------------------------
def k_conv0_scalar(img, c0, store):
    """kernels_simt.cuh k_conv0 with pack_stem's w0 (plan_net.cu:119-124), one output pixel per thread index."""
    wsrc, bias = c0["w"].ravel().tolist(), c0["b"].tolist()
    wk = [0.0] * 216
    for o in range(8):
        for cb in range(3):
            for t in range(9):
                wk[(t * 3 + cb) * 8 + o] = wsrc[(o * 3 + (2 - cb)) * 9 + t]
    n, H, W, _ = img.shape
    OH, OW = H >> 1, W >> 1
    out = np.zeros((n * OH * OW, 8))
    im = img.tolist()
    for idx in range(n * OH * OW):
        ox, oy, b = idx % OW, (idx // OW) % OH, idx // (OW * OH)
        acc = list(bias)
        for ky in range(3):
            iy = oy * 2 + ky - 1
            if iy < 0 or iy >= H:
                continue
            for kx in range(3):
                ix = ox * 2 + kx - 1
                if ix < 0 or ix >= W:
                    continue
                for c in range(3):
                    v = float(im[b][iy][ix][c])
                    for o in range(8):
                        acc[o] = fmaf(v, wk[((ky * 3 + kx) * 3 + c) * 8 + o], acc[o])
        out[idx] = [store(max(a, 0.0)) for a in acc]
    return fs.nchw(out.reshape(n, OH, OW, 8))


def k_dw3x3_scalar(x, dw, stride, store):
    """k_dw3x3<T, STRIDE> with pack_dw's [9][C] weights (plan_net.cu:132-138): one thread per (pixel, 8 channels)."""
    n, C, H, W = x.shape
    wd = [0.0] * (9 * C)
    wsrc = dw["w"].ravel().tolist()
    for c in range(C):
        for t in range(9):
            wd[t * C + c] = wsrc[c * 9 + t]
    bias = dw["b"].tolist()
    xin = fs.nhwc(x).tolist()
    OH, OW, cg = H // stride, W // stride, C >> 3
    out = np.zeros((n * OH * OW, C))
    for idx in range(n * OH * OW * cg):
        g, pix = idx % cg, idx // cg
        ox, oy, b = pix % OW, (pix // OW) % OH, pix // (OW * OH)
        c0 = g * 8
        acc = [bias[c0 + i] for i in range(8)]
        for ky in range(3):
            iy = oy * stride + ky - 1
            if iy < 0 or iy >= H:
                continue
            for kx in range(3):
                ix = ox * stride + kx - 1
                if ix < 0 or ix >= W:
                    continue
                f = xin[b][iy][ix][c0:c0 + 8]
                for i in range(8):
                    acc[i] = fmaf(f[i], wd[(ky * 3 + kx) * C + c0 + i], acc[i])
        out[pix, c0:c0 + 8] = [store(max(a, 0.0)) for a in acc]
    return fs.nchw(out.reshape(n, OH, OW, C))


def k_conv_gemm_scalar(x, ws, bs, outs, store):
    """launch_gemm + k_conv_gemm<T, BN, KS> with pack_gemm's weights (plan_fp.cu:15-44): 64-pixel x BN tiles, 256 threads
    (16 x 16, 4 x TN outputs each), K chunks of kc = min(Cin, 16) staged through As / Bs, epilogue with the OutSplit.
    outs = [(channels, relu)], at most two halves."""
    nimg, Cin, H, W = x.shape
    KS = ws[0].shape[2]
    N = sum(w.shape[0] for w in ws)
    wk, bias, n0 = [0.0] * (KS * KS * Cin * N), [], 0
    for w, b in zip(ws, bs):
        src = w.ravel().tolist()
        for o in range(w.shape[0]):
            bias.append(float(b[o]))
            for ci in range(Cin):
                for t in range(KS * KS):
                    wk[(t * Cin + ci) * N + n0 + o] = src[(o * Cin + ci) * KS * KS + t]
        n0 += w.shape[0]
    BN = 64 if N % 64 == 0 else (32 if N % 32 == 0 else 16)
    TN, BM, BK = BN // 16, 64, 16
    split_n0, relu0 = outs[0]
    relu1 = outs[1][1] if len(outs) > 1 else False
    xin = fs.nhwc(x).reshape(-1, Cin).tolist()
    M = nimg * H * W
    out = np.full((M, N), np.nan)
    kc = Cin if Cin < BK else BK
    for bx in range((M + BM - 1) // BM):
        m0 = bx * BM
        for by in range((N + BN - 1) // BN):
            nb0 = by * BN
            acc = [[[0.0] * TN for _ in range(4)] for _ in range(256)]
            for tap in range(KS * KS):
                dy, dx = (tap // 3 - 1, tap % 3 - 1) if KS == 3 else (0, 0)
                for c0 in range(0, Cin, kc):
                    As = [[0.0] * BM for _ in range(BK)]
                    for tid in range(256):                                   # the A-load role
                        lm, lk = tid >> 2, (tid & 3) * 4
                        gm = m0 + lm
                        if lk >= kc:
                            continue
                        v = [0.0] * 4
                        if gm < M:
                            px, py, pb = gm % W, (gm // W) % H, gm // (W * H)
                            iy, ix = py + dy, px + dx
                            if 0 <= iy < H and 0 <= ix < W:
                                v = xin[(pb * H + iy) * W + ix][c0 + lk:c0 + lk + 4]
                        for i in range(4):
                            As[lk + i][lm] = v[i]
                    Bs = [[wk[(tap * Cin + c0 + k) * N + nb0 + nn] if nb0 + nn < N else 0.0 for nn in range(BN)] for k in range(kc)]
                    for tid in range(256):
                        tx, ty = tid & 15, tid >> 4
                        a_t = acc[tid]
                        for k in range(kc):
                            for i in range(4):
                                a = As[k][ty + 16 * i]
                                for j in range(TN):
                                    a_t[i][j] = fmaf(a, Bs[k][tx * TN + j], a_t[i][j])
            for tid in range(256):                                           # epilogue
                tx, ty = tid & 15, tid >> 4
                for i in range(4):
                    m = m0 + ty + 16 * i
                    if m >= M:
                        continue
                    for j in range(TN):
                        nn = nb0 + tx * TN + j
                        if nn >= N:
                            continue
                        v = f32(acc[tid][i][j] + bias[nn])
                        if (relu0 if nn < split_n0 else relu1):
                            v = max(v, 0.0)
                        out[m, nn] = store(v)
    assert not np.isnan(out).any()
    res, o0 = [], 0
    for cn, _ in outs:
        res.append(fs.nchw(out[:, o0:o0 + cn].reshape(nimg, H, W, cn)))
        o0 += cn
    return res


def k_upsample_add_scalar(lat, up, up_w, store):
    """k_upsample_add<T>: one thread per (pixel, 8 channels), uw = the caffemodel's [C][4][4] deconvolution weights."""
    n, C, H, W = lat.shape
    UH, UW = up.shape[2:]
    uw = up_w.ravel().tolist()
    lt, ut = fs.nhwc(lat).tolist(), fs.nhwc(up).tolist()
    out = np.zeros((n, H, W, C))
    cg = C >> 3
    for idx in range(n * H * W * cg):
        g, pix = idx % cg, idx // cg
        x, y, b = pix % W, (pix // W) % H, pix // (W * H)
        c0 = g * 8
        acc = lt[b][y][x][c0:c0 + 8]
        i_hi, j_hi = (y + 1) >> 1, (x + 1) >> 1
        for di in range(2):
            i = i_hi - di
            ky = y - 2 * i + 1
            if i < 0 or i >= UH or ky < 0 or ky > 3:
                continue
            for dj in range(2):
                j = j_hi - dj
                kx = x - 2 * j + 1
                if j < 0 or j >= UW or kx < 0 or kx > 3:
                    continue
                f = ut[b][i][j][c0:c0 + 8]
                for c in range(8):
                    acc[c] = fmaf(f[c], uw[(c0 + c) * 16 + ky * 4 + kx], acc[c])
        out[b, y, x, c0:c0 + 8] = [store(a) for a in acc]
    return fs.nchw(out)


# ---- plain float64 convolutions and the order-free bound ----------------------------------------------------------------
def gamma(k):
    return k * U32 / (1 - k * U32)


def conv64(x, w, b, stride=1, groups=1):
    """Cross-correlation, zero padding (k - 1) / 2, in float64: (value, sum of |products| + |bias|)."""
    n, c, h, wd = x.shape
    o, ci, k, _ = w.shape
    p = (k - 1) // 2
    xp = np.pad(np.asarray(x, float), ((0, 0), (0, 0), (p, p), (p, p)))
    oh, ow = (h + 2 * p - k) // stride + 1, (wd + 2 * p - k) // stride + 1
    val = np.broadcast_to(np.asarray(b, float)[None, :, None, None], (n, o, oh, ow)).copy()
    mag = np.abs(val)
    for dy in range(k):
        for dx in range(k):
            win = xp[:, :, dy:dy + stride * oh:stride, dx:dx + stride * ow:stride]
            wt = np.asarray(w, float)[:, :, dy, dx]
            if groups == 1:
                val += np.einsum("nchw,oc->nohw", win, wt)
                mag += np.einsum("nchw,oc->nohw", np.abs(win), np.abs(wt))
            else:
                val += win * wt[None, :, 0, None, None]
                mag += np.abs(win * wt[None, :, 0, None, None])
    return val, mag


def within(got, val, mag, k, store, relu=True):
    """|got - (ReLU) val| <= gamma_k * mag, widened by the storage rounding where the store is FP16."""
    want = np.maximum(val, 0) if relu else val
    tol = gamma(k) * mag * (1 + 2.0 ** -10)
    if store is fs.rn16:
        tol = tol + 2.0 ** -11 * np.abs(got) + 2.0 ** -24
    return np.all(np.abs(got - want) <= tol)


# ---- each step: scalar transcription, float64 bound ---------------------------------------------------------------------
@pytest.mark.parametrize("T", list(STORES))
@pytest.mark.parametrize("shape", [(2, 6, 10), (1, 2, 2), (1, 2, 8), (2, 8, 2)])
def test_conv0_step(T, shape):
    store, store1 = STORES[T]
    rng = np.random.default_rng(sum(shape))
    c0 = dict(w=_rand32(rng, (8, 3, 3, 3), 0.05), b=_rand32(rng, 8, 0.5))
    img = rng.integers(0, 256, shape + (3,), dtype=np.uint8)
    got = f3.conv0(img, c0, store)
    assert np.array_equal(got, k_conv0_scalar(img, c0, store1))
    x = np.ascontiguousarray(img[..., ::-1].transpose(0, 3, 1, 2)).astype(float)       # BGR u8 -> RGB NCHW
    val, mag = conv64(x, c0["w"], c0["b"], stride=2)
    assert within(got, val, mag, 28, store)


@pytest.mark.parametrize("T", list(STORES))
@pytest.mark.parametrize("shape,stride", [((2, 8, 1, 1), 1), ((2, 16, 1, 5), 1), ((3, 8, 6, 1), 1), ((2, 16, 5, 7), 1),
                                          ((2, 8, 2, 2), 2), ((2, 16, 4, 6), 2), ((1, 8, 2, 8), 2), ((1, 8, 8, 2), 2)])
def test_depthwise_step(T, shape, stride):
    store, store1 = STORES[T]
    rng = np.random.default_rng(shape[1] * 7 + shape[2] * 3 + shape[3] + stride)
    c = shape[1]
    dw = dict(w=_rand32(rng, (c, 1, 3, 3), 0.4), b=_rand32(rng, c, 0.3))
    x = _act(rng, shape, store, signed=True)
    got = f3.depthwise(x, dw["w"], dw["b"], stride, store)
    assert np.array_equal(got, k_dw3x3_scalar(x, dw, stride, store1))
    val, mag = conv64(x, dw["w"], dw["b"], stride=stride, groups=c)
    assert within(got, val, mag, 10, store)


# (images, H, W, Cin, ks, OutSplit halves): M not a multiple of 64 (tiles across images), Cin = 8 (kc = 8 chunks), 16, 32
# and 64 (four chunks), N = 16 / 32 / 48 / 64 (BN 16, 32, 16, 64), one- and two-half splits with ReLU on either half,
# 1 x 1, 1 x n and n x 1 maps (3x3 taps mostly padding)
GEMMS = [(3, 5, 7, 8, 3, ((32, True), (16, True))), (2, 1, 1, 16, 3, ((16, True), (16, False))), (2, 1, 6, 16, 3, ((16, True),)),
         (3, 7, 1, 8, 1, ((64, True),)), (2, 9, 8, 32, 1, ((32, False), (32, True))), (1, 3, 3, 64, 3, ((32, True), (16, False)))]


@pytest.mark.parametrize("T", list(STORES))
@pytest.mark.parametrize("case", GEMMS, ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}_cin{c[3]}_k{c[4]}_n{sum(o[0] for o in c[5])}")
def test_gemm_step(T, case):
    store, store1 = STORES[T]
    n, h, w, cin, ks, outs = case
    rng = np.random.default_rng(n * 1000 + h * 100 + w * 10 + cin)
    ws = [_rand32(rng, (cn, cin, ks, ks), 0.3) for cn, _ in outs]
    bs = [_rand32(rng, cn, 0.5) for cn, _ in outs]
    x = _act(rng, (n, cin, h, w), store)
    got = f3.gemm_conv(x, ws, bs, list(outs), store)
    want = k_conv_gemm_scalar(x, ws, bs, list(outs), store1)
    for g, s in zip(got, want):
        assert np.array_equal(g, s)
    for g, wt, b, (_, relu) in zip(got, ws, bs, outs):
        val, mag = conv64(x, wt, b)
        assert within(g, val, mag, ks * ks * cin + 1, store, relu)


def deconv64(up, w, h, wd):
    """Caffe Deconvolution k4 s2 p1, grouped: the full transposed output, cropped to h x wd (float64)."""
    n, c, uh, uw = up.shape
    full, mag = np.zeros((n, c, 2 * uh + 2, 2 * uw + 2)), np.zeros((n, c, 2 * uh + 2, 2 * uw + 2))
    for ky in range(4):
        for kx in range(4):
            t = up * np.asarray(w, float)[None, :, 0, ky, kx, None, None]
            full[:, :, ky:ky + 2 * uh:2, kx:kx + 2 * uw:2] += t
            mag[:, :, ky:ky + 2 * uh:2, kx:kx + 2 * uw:2] += np.abs(t)
    return full[:, :, 1:1 + h, 1:1 + wd], mag[:, :, 1:1 + h, 1:1 + wd]


@pytest.mark.parametrize("T", list(STORES))
@pytest.mark.parametrize("lat_hw", [(2, 2), (2, 6), (4, 2), (6, 10)])
def test_upsample_add_step(T, lat_hw):
    store, store1 = STORES[T]
    rng = np.random.default_rng(lat_hw[0] * 10 + lat_hw[1])
    h, w = lat_hw
    lat, up = _act(rng, (2, 16, h, w), store), _act(rng, (2, 16, h // 2, w // 2), store)
    uw = _rand32(rng, (16, 1, 4, 4), 0.4)
    got = f3.upsample_add(lat, up, uw, store)
    assert np.array_equal(got, k_upsample_add_scalar(lat, up, uw, store1))
    val, mag = deconv64(up, uw, h, w)
    assert within(got, val + lat, mag + np.abs(lat), 5, store, relu=False)


# ---- teeth ----------------------------------------------------------------------------------------------------------------
def _chain_mul_add(x, wk):
    """The GEMM accumulator with a multiply, a rounding, then an add: what a kernel without fmaf computes."""
    n, cin, h, wd = x.shape
    a = fs.nhwc(x).reshape(-1, cin)
    acc = np.zeros((a.shape[0], wk.shape[1]))
    for c in range(cin):
        acc = fs.add32(fs.rn32(a[:, c:c + 1] * wk[c][None]), acc)
    return acc


def _chain_bias_first(x, wk, bias):
    n, cin, h, wd = x.shape
    a = fs.nhwc(x).reshape(-1, cin)
    return f3.fma_chain(np.broadcast_to(bias[None], (a.shape[0], wk.shape[1])), ((a[:, c].copy(), wk[c]) for c in range(cin)))


def mutations(p, rng):
    """(name, correct output, mutated output, float64 reference) of realistic kernel mistakes on the network's own weights
    and post-ReLU inputs of its scale."""
    out = []
    pw = p["mobilenet0_conv6_fwd"]
    x = _act(rng, (2, 32, 12, 20))
    good = f3.gemm_conv(x, [pw["w"]], [pw["b"]], [(32, True)])[0]
    wk, b = f3.gemm_matrix([pw["w"]]), np.asarray(pw["b"], float)
    shp = (2, 12, 20)
    bad = f3.gemm_epilogue(_chain_mul_add(x, wk), b, [(32, True)], shp)[0]
    out.append(("k_conv_gemm: multiply, round, add instead of fmaf", good, bad))
    bad = fs.nchw(np.maximum(_chain_bias_first(x, wk, b), 0).reshape(2, 12, 20, 32))
    out.append(("k_conv_gemm: bias as the accumulator's start instead of one add at the end", good, bad))
    d = np.abs(b[1:] - b[:-1])
    ch = int(np.argmin(np.where(d > 0, d, np.inf)))
    b2 = b.copy()
    b2[ch] = b[ch + 1]
    bad = f3.gemm_conv(x, [pw["w"]], [b2], [(32, True)])[0]
    out.append((f"k_conv_gemm: bias of channel {ch + 1} used for channel {ch}", good, bad))
    dw = p["mobilenet0_conv5_fwd"]
    xd = _act(rng, (2, 32, 12, 20))
    good = f3.depthwise(xd, dw["w"], dw["b"], 1)
    xm = xd.copy()
    xm[:, :, :, -1] = 0
    bad = good.copy()
    bad[:, :, 6] = f3.depthwise(xm, dw["w"], dw["b"], 1)[:, :, 6]
    out.append(("k_dw3x3: taps on the last input column skipped on output row 6", good, bad))
    ssh = [p["rf_c1_det_conv1"], p["rf_c1_det_context_conv1"]]
    xs = _act(rng, (1, 64, 6, 10))
    good = np.concatenate(f3.gemm_conv(xs, [c["w"] for c in ssh], [c["b"] for c in ssh], [(32, True), (16, False)]), axis=1)
    bad = np.concatenate(f3.gemm_conv(xs, [c["w"] for c in ssh], [c["b"] for c in ssh], [(32, False), (16, True)]), axis=1)
    out.append(("k_conv_gemm: ReLU applied to the other OutSplit half", good, bad))
    x16 = _act(rng, (2, 32, 12, 20), fs.rn16)
    good = f3.depthwise(x16, dw["w"], dw["b"], 1, fs.rn16)
    bad = f3.depthwise(x16, dw["w"], dw["b"], 1, fs.rn16, weights16=True)
    out.append(("FP16 k_dw3x3 with FP16-rounded weights (the tensor-core plans' rule)", good, bad))
    return out


def test_the_check_rejects_realistic_kernel_mistakes():
    """Each mutation changes at least one element, so "every element equal" rejects it; the old FP32 bar (2e-4 of the
    tensor's max, at least 1) misses the rounding-order ones."""
    p = folded_params(caffemodel("mnet25"))
    print()
    missed = []
    for name, good, bad in mutations(p, np.random.default_rng(17)):
        diff = int((good != bad).sum())
        assert diff > 0 and not np.array_equal(good, bad), name
        rel = float(np.abs(bad - good).max() / max(1.0, np.abs(good).max()))
        if rel < 2e-4:
            missed.append(name)
        print(f"  {name}: rejected ({diff} of {good.size} elements differ); the 2e-4-of-max bar "
              f"{'would' if rel >= 2e-4 else 'would NOT'} have caught it (max change {rel:.2e} of max)")
    assert len(missed) >= 2, missed


# ---- the walk -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", list(STORES))
def test_walk_yields_every_simt_tensor(T):
    """The whole walk on two 32 x 64 images (1 x 2 stride-32 map), the 'engine' materialising nothing: 43 tensors with the
    shapes of the network, stored values (FP32 or FP16), class probabilities within [0, 1], finite deltas."""
    store = STORES[T][0]
    steps = f3.SimtSteps(caffemodel("mnet25"), store)
    img = np.random.default_rng(5).integers(0, 256, (2, 32, 64, 3), dtype=np.uint8)
    seen = []
    for name, step, want, got in steps.walk(img, lambda name, want: None):
        if name.startswith("heads"):
            (lo, hi), bbox, lm = want
            assert np.all(0 <= lo) and np.all(lo <= hi) and np.all(hi <= 1), name
            assert np.all(np.isfinite(bbox)) and np.all(np.isfinite(lm)), name
            continue
        assert got is None and np.array_equal(store(want), want), name
        seen.append(name)
    assert len(seen) == len(set(seen)) == f3.TENSORS
    assert seen[:3] == ["mobilenet0_relu0_fwd", "mobilenet0_relu1_fwd", "mobilenet0_relu2_fwd"]
