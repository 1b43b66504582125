"""Host side of the FP16 step check (oracle/fp16_steps.py): its exact primitives against rational arithmetic, its tensor-core
bound against simulated accumulations, its teeth (mutations a kernel could make must be rejected), and a walk of the whole
network.  The guard that the GPU sweep still reaches every branch of the planner is host-only too; it sits with the sweep's
case table in tests/test_gpu_fp16_steps.py."""
from fractions import Fraction

import numpy as np
import pytest

from conftest import caffemodel
from oracle import fp16_steps as fs
from oracle.mnet_numpy import folded_params

FP32 = (24, -126, 127)          # significand bits, emin, emax
FP16 = (11, -14, 15)


def round_frac(q: Fraction, fmt):
    """Round-to-nearest-even of a rational into a binary format, subnormals and overflow included: the reference."""
    p, emin, emax = fmt
    if q == 0:
        return 0.0
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    quantum = Fraction(2) ** (max(e, emin) - p + 1)
    m = a / quantum
    r = int(m)
    if m - r > Fraction(1, 2) or (m - r == Fraction(1, 2) and r % 2):
        r += 1
    v = r * quantum
    if v > (2 - Fraction(2) ** (1 - p)) * Fraction(2) ** emax:
        return float(np.copysign(np.inf, float(q)))
    return float(v) if q > 0 else -float(v)


def _same(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.array_equal(a, b) and np.array_equal(np.signbit(a), np.signbit(b))


def _random_values(rng, n, fmt_round, lo_exp, hi_exp):
    return fmt_round(rng.choice([-1, 1], n) * rng.uniform(1, 2, n) * 2.0 ** rng.integers(lo_exp, hi_exp, n))


# ---- exact primitives ---------------------------------------------------------------------------------------------------
def test_rounding_to_fp16_and_fp32_against_fractions():
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.standard_normal(2000) * 2.0 ** rng.integers(-30, 20, 2000),
                        [1 + 2 ** -11, 1 + 3 * 2 ** -11, 1 + 2 ** -11 + 2 ** -40,       # FP16 midpoints and just above one
                         1 + 2 ** -24, 1 + 3 * 2 ** -24, 1 + 2 ** -24 + 2 ** -52,       # FP32 midpoints and just above one
                         2 ** -25, 3 * 2 ** -26, 2 ** -25 + 2 ** -40, 2 ** -150, 2 ** -150 + 2 ** -170,   # subnormals
                         65504, 65519.99, 65520, -65520, 0.0, -0.0, 2.0 ** 128]])
    for rn, fmt in ((fs.rn16, FP16), (fs.rn32, FP32)):
        got = rn(x)
        want = [np.copysign(round_frac(Fraction(float(v)), fmt), v) if np.isfinite(v) else v for v in x]
        assert _same(got, want), [(v, g, w) for v, g, w in zip(x, got, want) if not _same(g, w)][:5]
    # through float32, the FP16 rounding of 1 + 2^-11 + 2^-40 would be a tie (and go down): numpy rounds from the float64 bits
    assert fs.rn16(1 + 2 ** -11 + 2 ** -40) == 1 + 2 ** -10


def test_fma32_hfma16_and_add32_against_fractions():
    rng = np.random.default_rng(2)
    n = 3000
    x, w = _random_values(rng, n, fs.rn32, -40, 40), _random_values(rng, n, fs.rn32, -40, 40)
    acc = _random_values(rng, n, fs.rn32, -80, 80)
    near = rng.random(n) < 0.5                     # cancelling: acc = -RN32(x * w) + a few ulps
    acc[near] = fs.rn32(-x[near] * w[near] * (1 + rng.integers(-3, 4, near.sum()) * 2.0 ** -23))
    # hard cases: naive float64 rounds 1 + 3 * 2^-24 - 2^-70 to a tie, then to the even FP32 value 1 + 2^-22 (wrong);
    # subnormal results; signed zeros
    hard = [(1 + 2 ** -23, 2 ** -24 * (1 - 2 ** -23), 1 + 2 ** -23), (2.0 ** -100, 1.5 * 2.0 ** -49, 0.0),
            (-0.0, 1.0, -0.0), (1.0, -1.0, 1.0), (0.0, -5.0, -0.0), (2.0 ** -126, -0.5, 2.0 ** -126)]
    x, w, acc = (np.concatenate([v, [h[i] for h in hard]]) for i, v in enumerate((x, w, acc)))
    got = fs.fma32(x, w, acc)
    want = [round_frac(Fraction(a) * Fraction(b) + Fraction(c), FP32) for a, b, c in zip(x, w, acc)]
    for i, (a, b, c) in enumerate(zip(x, w, acc)):
        if a * b + c == 0 and not (a * b == 0 and c == 0):
            want[i] = 0.0                           # an exact zero sum of non-zero terms is +0 in round-to-nearest
        elif a * b == 0 and c == 0:
            want[i] = float(np.float64(a * b) + np.float64(c))     # IEEE signed-zero sum
    assert _same(got, want), [(a, b, c, g, v) for a, b, c, g, v in zip(x, w, acc, got, want) if not _same(g, v)][:5]
    assert fs.rn32(np.float64(hard[0][0]) * hard[0][1] + hard[0][2]) != got[n]     # the case defeats plain float64
    # FP16: random operands over the whole range, products that overflow, subnormal sums
    u, v = _random_values(rng, n, fs.rn16, -14, 9), _random_values(rng, n, fs.rn16, -14, 9)
    a16 = _random_values(rng, n, fs.rn16, -24, 16)
    extra = [(255.0, 255.0, 0.0), (256.0, 256.0, 0.0), (256.0, 256.0, -65504.0), (2.0 ** -14, 2.0 ** -10, 2.0 ** -24),
             (3.0, 683 * 2.0 ** -11, -(2.0 ** -24)), (1.0, -1.0, 1.0)]
    u, v, a16 = (np.concatenate([t, [e[i] for e in extra]]) for i, t in enumerate((u, v, a16)))
    got = fs.hfma16(u, v, a16)
    want = [round_frac(Fraction(a) * Fraction(b) + Fraction(c), FP16) for a, b, c in zip(u, v, a16)]
    assert _same(got, want), [(a, b, c, g, t) for a, b, c, g, t in zip(u, v, a16, got, want) if not _same(g, t)][:5]
    assert got[n] == 65024 and np.isinf(got[n + 1]) and got[n + 2] == 32
    got = fs.add32(x, acc)
    want = [round_frac(Fraction(a) + Fraction(c), FP32) if a + c != 0 else float(np.float64(a) + c) for a, c in zip(x, acc)]
    assert _same(got, want)


def test_directed_roundings_to_fp32():
    rng = np.random.default_rng(4)
    x = rng.standard_normal(5000) * 2.0 ** rng.integers(-60, 60, 5000)
    lo, hi = fs.floor32(x), fs.ceil32(x)
    assert np.all(lo <= x) and np.all(hi >= x) and np.all(fs.rn32(lo) == lo) and np.all(fs.rn32(hi) == hi)
    gap = hi - lo
    assert np.all((gap == 0) == (fs.rn32(x) == x))
    ulp = np.spacing(np.abs(lo).astype(np.float32)).astype(float)
    assert np.all((gap == 0) | (gap <= ulp * 1.0000001) | (gap <= np.spacing(np.abs(hi).astype(np.float32)).astype(float)))


# ---- the tensor-core bound ----------------------------------------------------------------------------------------------
def _trunc(x, quantum):
    return np.trunc(x / quantum) * quantum


def _trunc32(x):
    """Round toward zero to FP32."""
    r = fs.rn32(x)
    return np.where(np.abs(r) > np.abs(x), np.nextafter(r.astype(np.float32), np.float32(0)).astype(float), r)


def _accumulations(a, w_steps):
    """FP32 results of one GEMM under several accumulation orders: sequential forward, reverse and shuffled, pairwise per K
    step, and a block model (each K step's 16 products and the accumulator aligned to the largest exponent, truncated 23
    bits below it, summed exactly, truncated to FP32).  w_steps: [(k0, k1, W)] as oracle.fp16_steps.tc_gemm takes them."""
    prods = [a[:, k0:k1, None] * w[None] for k0, k1, w in w_steps]          # exact in float64 (FP16 x FP16)
    flat = np.concatenate(prods, axis=1)                                     # (M, K', N) in issue order
    out = []
    rng = np.random.default_rng(5)
    for order in (np.arange(flat.shape[1]), np.arange(flat.shape[1])[::-1], rng.permutation(flat.shape[1])):
        acc = np.zeros((a.shape[0], flat.shape[2]), np.float32)
        for k in order:
            acc = acc + flat[:, k].astype(np.float32)
        out.append(acc.astype(float))
    acc = np.zeros((a.shape[0], flat.shape[2]), np.float32)
    for p in prods:                                                          # pairwise tree inside each step
        v = p.astype(np.float32)
        while v.shape[1] > 1:
            v = v[:, 0::2] + v[:, 1::2]
        acc = acc + v[:, 0]
    out.append(acc.astype(float))
    acc = np.zeros((a.shape[0], flat.shape[2]))
    for p in prods:
        terms = np.concatenate([acc[:, None], p], axis=1)
        big = np.abs(terms).max(axis=1)
        _, e = np.frexp(np.where(big > 0, big, 1.0))
        q = np.ldexp(1.0, e - 24)[:, None]
        acc = _trunc32(_trunc(terms, q).sum(axis=1))
    out.append(acc)
    return out


@pytest.mark.parametrize("k", [8, 16, 27, 32, 64, 128, 256, 576])
@pytest.mark.parametrize("hilo", [False, True])
def test_tc_bound_contains_every_accumulation(k, hilo):
    rng = np.random.default_rng(k + 1000 * hilo)
    m, n = 96, 24
    kp = (k + 15) // 16 * 16
    a = fs.rn16(np.abs(rng.standard_normal((m, k))) * 4 * (rng.random((m, k)) < 0.7))       # post-ReLU activations
    a[m // 3:2 * m // 3] = fs.rn16(rng.standard_normal((m // 3, k)) * 2.0 ** rng.integers(-8, 6, (m // 3, k)))   # signed, wide
    w = rng.standard_normal((k, n)) * 0.3
    w[:, n // 2:] = np.concatenate([w[:k // 2, :n // 2], -w[:k - k // 2, :n // 2]])[:, :n - n // 2]     # cancelling columns
    a[2 * m // 3:, k // 2:] = a[2 * m // 3:, :k - k // 2]
    a, w = fs.pad_k(a, 1), fs.pad_k(w, 0)
    if hilo:
        hi, lo = fs.hi_lo(w)
        steps = fs.k_steps(hi) + [(k0, k1, lo[k0:k1]) for k0, k1, _ in fs.k_steps(lo)]
    else:
        steps = fs.k_steps(fs.rn16(w))
    lo_b, hi_b, _ = fs.tc_gemm(fs.Iv(a, a, None), steps)
    sums = _accumulations(a, steps)
    exact = sum(a[:, k0:k1] @ ws for k0, k1, ws in steps)
    assert np.all((lo_b <= exact) & (exact <= hi_b))
    for i, s in enumerate(sums):
        assert np.all((lo_b <= s) & (s <= hi_b)), (k, hilo, i, np.max(np.maximum(lo_b - s, s - hi_b)))
    assert len(steps) == (2 if hilo else 1) * kp // 16


# ---- teeth: mutations a kernel could make -------------------------------------------------------------------------------
def test_the_check_rejects_realistic_kernel_mistakes():
    """Every mutation of oracle.fp16_steps.mutations is rejected, including the small ones (one output of one tile missing a
    tap in one 8-channel group, one channel's bias taken from its neighbour); the last passes the 2e-2-of-max bar of the
    older FP16 tests."""
    p = folded_params(caffemodel("mnet25"))
    rng = np.random.default_rng(7)
    x = fs.Iv.exact(fs.rn16(np.abs(rng.standard_normal((2, 32, 12, 20))) * 3 * (rng.random((2, 32, 12, 20)) < 0.7)))
    dw, pw = p["mobilenet0_conv5_fwd"], p["mobilenet0_conv6_fwd"]
    iv = fs.dw_pw(x, dw, pw, 1)
    good = iv.mid
    assert not fs.outside(good, iv).any()               # the control: RN16 of the float64 midpoint is accepted
    print()
    missed_by_old_bar = []
    for name, bad in fs.mutations(x, dw, pw, 1, good):
        assert fs.outside(bad, iv).any(), name
        rel = float(np.abs(bad - good).max() / np.abs(good).max())
        if rel < 2e-2:
            missed_by_old_bar.append(name)
        print(f"  {name}: rejected ({int(fs.outside(bad, iv).sum())} elements outside); the 2e-2-of-max bar "
              f"{'would' if rel >= 2e-2 else 'would NOT'} have caught it (max change {rel:.2e} of max)")
    assert any("only" in m for m in missed_by_old_bar), missed_by_old_bar


@pytest.mark.parametrize("chains", [False, True])
def test_every_step_accepts_its_own_midpoint(chains):
    """The whole walk on a tiny batch, the 'engine' materialising every tensor as the oracle's own midpoint rounding: every
    midpoint inside its interval, the class probabilities within [0, 1]; per layer, and (chains) with the SSH tile chains'
    predictor stages."""
    steps = fs.Fp16Steps(caffemodel("mnet25"))
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, (2, 64, 96, 3), dtype=np.uint8)
    seen = []
    for name, step, iv, _ in steps.walk(img, lambda name, iv: iv.mid, chain_heads=chains):
        if name.startswith("heads"):
            (lo, hi), bbox, lm = iv
            assert np.all(lo <= hi) and np.all(hi <= 1) and np.all(lo >= 0), name
            for d in (bbox, lm):
                assert np.all(d[0] <= d[1]) if chains else np.all(np.isfinite(d)), name
            continue
        assert np.all(iv.lo <= iv.mid) and np.all(iv.mid <= iv.hi), (name, step)
        seen.append(name)
    assert len(seen) == 1 + 12 + 3 + 2 + 2 + 3 * 3
    # no plan runs a depthwise layer on tensor cores: naming one is an error, not a walk with the wrong arithmetic
    with pytest.raises(ValueError):
        next(steps.walk(img, lambda name, iv: iv.mid, tc_dw=(3,)))
