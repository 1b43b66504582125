// tc_conv_i8.cuh -- INT8 twins of the tensor-core convolution kernels of tc_conv.cuh (RF_PREC_INT8).
//
// Same design -- staged range + shifted descriptors, weights by one TMA bulk copy, wgmma with the accumulator in
// registers, programmatic dependent launch -- with 8-bit operands:
//   * activations: int8 NHWC, per-tensor scale from the reference's TensorRT calibration table
//     (model/mnet-deconv-0517.table.int8: symmetric, range = 127 * scale); a 16-byte group holds 16 channels;
//   * weights: int8, per-output-channel scale, packed [K/16][N][16] (K-major, no swizzle);
//   * MMA: wgmma.mma_async m64nNCk32 .s32.s8.s8 per warpgroup (K = 32 per instruction: two 16-channel groups),
//     S32 accumulator in registers;
//   * epilogue: v = float(acc) * mult[n] + bq[n] (two roundings: __fmul_rn, __fadd_rn -- bit-identical to the
//     integer oracle oracle/mnet_int8.py), ReLU, round-to-nearest-even, clamp +-127, int8 pairs;
//   * depthwise stage (k_tc_dwpw_staged_i8): FP32 stencil on the dequantised int8 input (input scale folded into
//     the depthwise weights), requantised with the table's scale of the depthwise output into the A operand.
// The exact integer scheme is restated in oracle/mnet_int8.py; TensorRT's own INT8 kernels are closed source.
#pragma once
#include "tc_conv.cuh"

namespace rf {

struct TcOutI8 {
    int8_t *p0; int ld0; int n0; int relu0;    // channels [0, n0)  -> p0[m*ld0 + n]
    int8_t *p1; int ld1; int relu1;            // channels [n0, N)  -> p1[m*ld1 + n - n0]
};

namespace tc {
__device__ __forceinline__ int q8(float v) {            // round to nearest even, clamp to the symmetric int8 range
    int q = __float2int_rn(v);
    return max(-127, min(127, q));
}
__device__ __forceinline__ uint32_t pack4(int a, int b, int c, int d) {
    return (uint32_t)(a & 0xff) | ((uint32_t)(b & 0xff) << 8) | ((uint32_t)(c & 0xff) << 16) | ((uint32_t)(d & 0xff) << 24);
}
__device__ __forceinline__ void unpack16(const uint4 &v, float f[16]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
        f[4 * i + 0] = (float)(int8_t)(w[i] & 0xff);
        f[4 * i + 1] = (float)(int8_t)((w[i] >> 8) & 0xff);
        f[4 * i + 2] = (float)(int8_t)((w[i] >> 16) & 0xff);
        f[4 * i + 3] = (float)(int8_t)(w[i] >> 24);
    }
}
__device__ __forceinline__ void unpack8(const uint2 &v, float f[8]) {
    const uint32_t w[2] = {v.x, v.y};
#pragma unroll
    for (int i = 0; i < 2; i++) {
        f[4 * i + 0] = (float)(int8_t)(w[i] & 0xff);
        f[4 * i + 1] = (float)(int8_t)((w[i] >> 8) & 0xff);
        f[4 * i + 2] = (float)(int8_t)((w[i] >> 16) & 0xff);
        f[4 * i + 3] = (float)(int8_t)(w[i] >> 24);
    }
}
}  // namespace tc

// Epilogue of one accumulator chunk (columns [n0, n0 + NC)), rows out_row[e] < 0 are not stored (see tc_epilogue).
template <int NC>
__device__ __forceinline__ void tc_epilogue_i8(const int (&d)[NC / 2], int n0, const float *s_mult, const float *s_bq, const TcOutI8 &o,
                                               const long (&out_row)[2], int n_off) {
    const int c2 = 2 * (threadIdx.x & 3);
#pragma unroll
    for (int e = 0; e < 2; e++) {
        if (out_row[e] < 0) continue;
#pragma unroll
        for (int i = 0; i < NC / 8; i++) {
            const int n = n0 + 8 * i + c2;
            const int gn = n_off + n;
            const bool first = gn < o.n0;
            const int relu = first ? o.relu0 : o.relu1;
            int8_t *dst = first ? o.p0 + (size_t)out_row[e] * o.ld0 + gn : o.p1 + (size_t)out_row[e] * o.ld1 + (gn - o.n0);
            float v0 = __fadd_rn(__fmul_rn((float)d[4 * i + 2 * e], s_mult[n]), s_bq[n]);
            float v1 = __fadd_rn(__fmul_rn((float)d[4 * i + 2 * e + 1], s_mult[n + 1]), s_bq[n + 1]);
            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
            *reinterpret_cast<uint16_t *>(dst) = (uint16_t)((tc::q8(v0) & 0xff) | ((tc::q8(v1) & 0xff) << 8));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
struct TcConvArgsI8 {
    const int8_t *in;       // NHWC dense [nimg][H][W][Cin]
    int Cin, nimg, H, W;
    int taps;               // 1 | 9
    int N;
    int Wp, Hp, R;          // as TcConvArgs
    uint32_t mul_Wp, mul_Hp, mul_H;   // fast_div multipliers (set by the launch helper)
    const int8_t *wimg;     // [taps * GS][N][16] int8, GS = max(Cin/16, 2) groups per tap (zero padded)
    const float *mult, *bq; // [N]: s_in*s_w[n]/s_out(n), b'[n]/s_out(n)
    TcOutI8 out;
    const int8_t *up;       // UPADD: coarse map [nimg][H/2][W/2][Cin]
    const float *up_wq;     // UPADD: [16 taps][Cin] = w[c][tap] * s_up / s_out
    float lat_mul;          // UPADD: s_lat / s_out
    int Cmax;
};

inline int tc_i8_gs(int Cin) { int g = Cin / 16; return g < 2 ? 2 : g; }
inline size_t tc_conv_i8_smem_bytes(const TcConvArgsI8 &a) {
    const int GS = tc_i8_gs(a.Cin);
    return (size_t)GS * a.R * 16 + (size_t)a.taps * GS * 16 * a.N + (a.up ? (size_t)(a.Cin / 16) * a.Cmax * 16 : 0) +
           (size_t)a.R * 4 * (a.up ? 2 : 1) + 128;      // + position tables (s_pix, UPADD: s_yx)
}

template <int NT, bool UPADD>
__global__ void __launch_bounds__(TC_THREADS) k_tc_conv_staged_i8(const TcConvArgsI8 a) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_b;
    __shared__ float s_mult[256], s_bq[256];
    __shared__ __align__(16) float s_uw[UPADD ? 64 * 16 : 4];   // [tap][channel]
    __shared__ int s_crow[2];

    const int tid = threadIdx.x, warp = tid >> 5;
    const int pad = a.taps == 9 ? 1 : 0;
    const int G = a.Cin >> 4;
    const int GS = G < 2 ? 2 : G;
    const uint32_t lbo_s = (uint32_t)a.R * 16;
    unsigned char *sS = smem;
    unsigned char *sB = smem + (size_t)GS * lbo_s;
    // position tables behind the operands: s_pix: staged position -> pixel index in `in`, -1 = zero padding; UPADD: s_yx
    int *s_pix = reinterpret_cast<int *>(sB + (size_t)a.taps * GS * 16 * a.N + (UPADD ? (size_t)G * a.Cmax * 16 : 0));
    int *s_yx = s_pix + a.R;
    const int m0 = blockIdx.x * 128;
    const int lo = m0 - (a.Wp + 1) * pad;

    if (tid == 0) {
        s_crow[0] = 0x7fffffff; s_crow[1] = -1;
        tc::mbar_init(&bar_b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)((size_t)a.taps * GS * 16 * a.N);
        tc::mbar_expect_tx(&bar_b, bytes);
        tc::bulk_g2s(sB, a.wimg, bytes, &bar_b);
    }
    pdl_trigger();
    if (tid < a.N) { s_mult[tid] = a.mult[tid]; s_bq[tid] = a.bq[tid]; }
    if (UPADD) for (int i = tid; i < a.Cin * 16; i += TC_THREADS) s_uw[i] = a.up_wq[i];
    {
        const int lane = tid & 31;
        const int prow0 = fast_floor_div(lo, a.Wp, a.mul_Wp);
        const int prow1 = fast_div(lo + a.R - 1, a.mul_Wp);
        for (int prow = prow0 + warp; prow <= prow1; prow += TC_THREADS / 32) {
            const int b = prow >= 0 ? fast_div(prow, a.mul_Hp) : -1;
            const int yy = prow >= 0 ? (int)(prow - b * a.Hp) : 0;
            const bool rowok = prow >= 0 && b < a.nimg && yy < a.H;
            for (int xx = lane; xx < a.Wp; xx += 32) {
                const int pl = prow * a.Wp + xx - lo;
                if (pl < 0 || pl >= a.R) continue;
                int pix = -1;
                if (rowok && xx >= pad && xx < a.W + pad) {
                    pix = (b * a.H + yy) * a.W + (xx - pad);
                    if (UPADD) {
                        s_yx[pl] = ((b * a.H + yy) << 12) | (xx - pad);
                        const int UH = a.H >> 1, ih = (yy + 1) >> 1;
                        atomicMin(&s_crow[0], b * UH + max(ih - 1, 0));
                        atomicMax(&s_crow[1], b * UH + min(ih, UH - 1));
                    }
                }
                s_pix[pl] = pix;
            }
        }
    }
    __syncthreads();
    pdl_wait();
    const int lgs = 31 - __clz(GS);
    const int UH = a.H >> 1, UW = a.W >> 1;
    const int lg = 31 - __clz(G);
    unsigned char *sC = sB + (size_t)a.taps * GS * 16 * a.N;      // UPADD: coarse rows, pixel-major [coarse position][Cin]
    const int crow_lo = UPADD ? s_crow[0] : 0, crow_hi = UPADD ? s_crow[1] : -1;
    if (UPADD && crow_hi >= crow_lo) {       // coarse rows first: asynchronous plain copy (see k_tc_conv_staged)
        const int ncp = (crow_hi - crow_lo + 1) * UW;
        if (ncp > a.Cmax) __trap();
        const int8_t *csrc = a.up + (size_t)crow_lo * UW * a.Cin;
        for (int it = tid; it < ncp * G; it += TC_THREADS) cp_async16_zfill(sC + (size_t)it * 16, csrc + (size_t)it * 16, true);
    }
    {   // the range itself through registers: coalesced LDG.128, conflict-free STS.128 into the K-major operand (R is odd)
        constexpr int UNR = 4;
        for (int it0 = tid; it0 < a.R * GS; it0 += TC_THREADS * UNR) {
            uint4 v[UNR];
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int it = it0 + u * TC_THREADS;
                v[u] = make_uint4(0, 0, 0, 0);
                if (it < a.R * GS) {
                    const int g = it & (GS - 1), pix = s_pix[it >> lgs];
                    if (pix >= 0 && g < G) v[u] = __ldcg(reinterpret_cast<const uint4 *>(a.in + (size_t)pix * a.Cin + g * 16));
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int it = it0 + u * TC_THREADS;
                if (it < a.R * GS) *reinterpret_cast<uint4 *>(sS + (size_t)(it & (GS - 1)) * lbo_s + (size_t)(it >> lgs) * 16) = v[u];
            }
        }
    }
    if (UPADD) {
        cp_async_wait_all();
        __syncthreads();
        for (int it = tid; it < a.R * G; it += TC_THREADS) {
            const int g = it & (G - 1), pl = it >> lg;
            if (s_pix[pl] < 0) continue;
            const int c0 = g * 16;
            const int yx = s_yx[pl];
            const int x = yx & 0xfff, gy = yx >> 12;
            const int b = fast_div(gy, a.mul_H), y = gy - b * a.H;
            unsigned char *slot = sS + (size_t)g * lbo_s + (size_t)pl * 16;
            float acc[16];
            tc::unpack16(*reinterpret_cast<const uint4 *>(slot), acc);
#pragma unroll
            for (int c = 0; c < 16; c++) acc[c] = __fmul_rn(acc[c], a.lat_mul);
            const int i_hi = (y + 1) >> 1, j_hi = (x + 1) >> 1;
#pragma unroll
            for (int di = 0; di < 2; di++) {
                const int i = i_hi - di, ky = y - 2 * i + 1;
                if (i < 0 || i >= UH || ky < 0 || ky > 3) continue;
#pragma unroll
                for (int dj = 0; dj < 2; dj++) {
                    const int j = j_hi - dj, kx = x - 2 * j + 1;
                    if (j < 0 || j >= UW || kx < 0 || kx > 3) continue;
                    float u[16];
                    tc::unpack16(*reinterpret_cast<const uint4 *>(sC + ((size_t)((b * UH + i - crow_lo) * UW + j) * G + g) * 16), u);
                    const float *w = &s_uw[(ky * 4 + kx) * a.Cin + c0];
#pragma unroll
                    for (int c = 0; c < 16; c++) acc[c] = __fadd_rn(acc[c], __fmul_rn(u[c], w[c]));   // no FMA: matches the oracle bit for bit
                }
            }
            int q[16];
#pragma unroll
            for (int c = 0; c < 16; c++) q[c] = tc::q8(acc[c]);
            uint4 pk;
            pk.x = tc::pack4(q[0], q[1], q[2], q[3]);   pk.y = tc::pack4(q[4], q[5], q[6], q[7]);
            pk.z = tc::pack4(q[8], q[9], q[10], q[11]); pk.w = tc::pack4(q[12], q[13], q[14], q[15]);
            *reinterpret_cast<uint4 *>(slot) = pk;
        }
    } else {
        cp_async_wait_all();
    }
    tc::fence_async_smem();
    __syncthreads();
    tc::mbar_wait(&bar_b, 0);
    const int row_base = (int)(m0 - lo);
    long orow[2];
#pragma unroll
    for (int e = 0; e < 2; e++) orow[e] = s_pix[row_base + tc_frag_row() + 8 * e];
    const uint32_t s_addr = tc::smem_u32(sS) + (uint32_t)(row_base + 64 * (warp >> 2)) * 16u, b_addr = tc::smem_u32(sB);
    const uint32_t lbo_b = (uint32_t)a.N * 16;
    wg::for_chunks<(NT < 64 ? NT : 64)>(a.N, [&](auto nc, int n0) {
        constexpr int NC = decltype(nc)::value;
        int d[NC / 2];                   // not zeroed: the first MMA runs with scale-d = 0 (see wg::fence)
        wg::fence();
        int acc = 0;
        for (int t = 0; t < a.taps; t++) {
            const int shift = pad ? (t / 3 - 1) * a.Wp + (t % 3 - 1) : 0;
            for (int cs = 0; cs < (GS >> 1); cs++) {
                const uint64_t ad = wg::desc(s_addr + (uint32_t)(2 * cs) * lbo_s + (uint32_t)(shift * 16), lbo_s, 128);
                const uint64_t bd = wg::desc(b_addr + (uint32_t)(t * GS + 2 * cs) * lbo_b + (uint32_t)n0 * 16u, lbo_b, 128);
                wg::mma_s8<NC>(d, ad, bd, acc);
                acc = 1;
            }
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(d);
        tc_epilogue_i8<NC>(d, n0, s_mult, s_bq, a.out, orow, 0);
    });
}

// ---------------------------------------------------------------------------------------------------------
struct TcDwArgsI8 {
    const int8_t *in;       // NHWC dense [nimg][IH][IW][C]
    int C, nimg, IH, IW, OH, OW, S;
    int N, Ntotal, Kpad;    // Kpad = C rounded up to 32
    int rows, Wp, Hp, Rmax;
    uint32_t mul_Wp, mul_Hp, mul_OW, mul_OH;   // fast_div multipliers (set by the launch helper)
    const int8_t *wimg;     // slice s at s * Kpad * N bytes: [Kpad/16][N][16]
    const float *mult, *bq; // [Ntotal]
    const float *dw_w;      // [9][C] folded depthwise weights * s_in
    const float *dw_b;      // [C]
    float inv_mid;          // 1 / scale of the depthwise output tensor
    int8_t *out;            // [nimg][OH][OW][Ntotal]
};

inline size_t tc_dw_i8_smem_bytes(const TcDwArgsI8 &a) {
    return (size_t)(a.C / 16) * a.Rmax * 16 + (size_t)(a.Kpad / 16) * tc_dw_lbo_a(a.rows) + (size_t)a.Kpad * a.N +
           (size_t)a.Rmax * 4 + 128;
}

// WREG (C >= 64): the stencil's work item is 8 channels (half of a 16-byte group); a thread owns ONE half for all its rows, so
// its 72 folded depthwise weights + 8 biases live in registers (with the weights in shared memory the 16-byte weight reads
// of the 8 groups of a warp are 4-way bank conflicted and the kernel is shared-memory-wavefront bound).  Same arithmetic.
template <int NT, bool WREG>
__global__ void __launch_bounds__(TC_THREADS, 2) k_tc_dwpw_staged_i8(const TcDwArgsI8 a) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_b;
    __shared__ int s_cpos[128];
    __shared__ float s_mult[256], s_bq[256];
    __shared__ __align__(16) float s_dw[WREG ? 4 : 10 * 64];   // !WREG: [tap][C] (input scale folded in), [9] = bias (C < 64)

    const int tid = threadIdx.x, warp = tid >> 5;
    const int G = a.C >> 4;
    const int GA = a.Kpad >> 4;
    const int g_own = tid % GA;
    const int pix = a.C;                 // staged range is pixel-major, [position][C] int8 (see k_tc_dwpw_staged)
    unsigned char *sS = smem;
    unsigned char *sA = smem + (size_t)a.Rmax * pix;
    const uint32_t lbo_a = tc_dw_lbo_a(a.rows);
    unsigned char *sB = sA + (size_t)GA * lbo_a;
    int *s_pix = reinterpret_cast<int *>(sB + (size_t)a.Kpad * a.N);
    const int M = a.nimg * a.OH * a.OW;
    const int m0 = blockIdx.x * a.rows;
    const int mlast = min(m0 + a.rows, M) - 1;
    auto centre = [&](int m) -> int {
        const int q = fast_div(m, a.mul_OW), ox = m - q * a.OW, b = fast_div(q, a.mul_OH), oy = q - b * a.OH;
        return (b * a.Hp + oy * a.S) * a.Wp + ox * a.S + 1;
    };
    const int lo = centre(m0) - a.Wp - 1;
    const int R = (int)(centre(mlast) + a.Wp + 1 - lo) + 1;
    if (R > a.Rmax) __trap();

    if (tid == 0) {
        tc::mbar_init(&bar_b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)((size_t)a.Kpad * a.N);
        tc::mbar_expect_tx(&bar_b, bytes);
        tc::bulk_g2s(sB, a.wimg + (size_t)blockIdx.y * a.Kpad * a.N, bytes, &bar_b);
    }
    pdl_trigger();
    if (tid < a.N) { s_mult[tid] = a.mult[blockIdx.y * a.N + tid]; s_bq[tid] = a.bq[blockIdx.y * a.N + tid]; }
    const int H8 = a.C >> 3, h_own = tid % H8;          // WREG: this thread's 8-channel half
    float wreg[WREG ? 10 : 1][8];
    if (WREG) {
#pragma unroll
        for (int t = 0; t < (WREG ? 10 : 1); t++) {
            const float *src = (t < 9 ? a.dw_w + t * a.C : a.dw_b) + h_own * 8;
            const float4 w0 = __ldg(reinterpret_cast<const float4 *>(src)), w1 = __ldg(reinterpret_cast<const float4 *>(src) + 1);
            wreg[t][0] = w0.x; wreg[t][1] = w0.y; wreg[t][2] = w0.z; wreg[t][3] = w0.w;
            wreg[t][4] = w1.x; wreg[t][5] = w1.y; wreg[t][6] = w1.z; wreg[t][7] = w1.w;
        }
    } else {
        for (int i = tid; i < 10 * a.C; i += TC_THREADS) s_dw[i] = i < 9 * a.C ? a.dw_w[i] : a.dw_b[i - 9 * a.C];
    }
    {
        const int lane = tid & 31;
        const int prow0 = fast_floor_div(lo, a.Wp, a.mul_Wp);
        const int prow1 = fast_div(lo + R - 1, a.mul_Wp);
        for (int prow = prow0 + warp; prow <= prow1; prow += TC_THREADS / 32) {
            const int b = prow >= 0 ? fast_div(prow, a.mul_Hp) : -1;
            const int yy = prow >= 0 ? (int)(prow - b * a.Hp) : 0;
            const bool rowok = prow >= 0 && b < a.nimg && yy < a.IH;
            for (int xx = lane; xx < a.Wp; xx += 32) {
                const int pl = prow * a.Wp + xx - lo;
                if (pl < 0 || pl >= R) continue;
                s_pix[pl] = (rowok && xx >= 1 && xx <= a.IW) ? (b * a.IH + yy) * a.IW + (xx - 1) : -1;
            }
        }
    }
    if (tid < 128) {
        const int m = m0 + tid;
        s_cpos[tid] = (tid < a.rows && m < M) ? (int)(centre(m) - lo) : -1;
    }
    __syncthreads();
    pdl_wait();
    const int lg = 31 - __clz(G);
    for (int it = tid; it < R * G; it += TC_THREADS) {
        const int g = it & (G - 1), pl = it >> lg;
        const int src_pix = s_pix[pl];
        cp_async16_zfill(sS + (size_t)it * 16, a.in + (src_pix >= 0 ? (size_t)src_pix * a.C + g * 16 : 0), src_pix >= 0);
    }
    cp_async_wait_all();
    __syncthreads();
    // ---- depthwise stencil (FP32 on the int8 input; the input scale lives in the weights) -> int8 A operand ----
    if (WREG) {
        for (int r = tid / H8; r < a.rows; r += TC_THREADS / H8) {
            const int cp = s_cpos[r];
            if (cp < 0) continue;
            float acc[8];
#pragma unroll
            for (int i = 0; i < 8; i++) acc[i] = wreg[WREG ? 9 : 0][i];
            const unsigned char *base = sS + cp * pix + h_own * 8;
#pragma unroll
            for (int t = 0; t < 9; t++) {
                const int shift = (t / 3 - 1) * a.Wp + (t % 3 - 1);
                float f[8];
                tc::unpack8(*reinterpret_cast<const uint2 *>(base + shift * pix), f);
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] = __fadd_rn(acc[i], __fmul_rn(f[i], wreg[WREG ? t : 0][i]));     // no FMA, see below
            }
            int q[8];
#pragma unroll
            for (int i = 0; i < 8; i++) q[i] = tc::q8(__fmul_rn(fmaxf(acc[i], 0.f), a.inv_mid));
            *reinterpret_cast<uint2 *>(sA + (size_t)(h_own >> 1) * lbo_a + (size_t)r * 16 + (h_own & 1) * 8) =
                make_uint2(tc::pack4(q[0], q[1], q[2], q[3]), tc::pack4(q[4], q[5], q[6], q[7]));
        }
    } else if (g_own < G) {
        const int c0 = g_own * 16;
        for (int r = tid / GA; r < a.rows; r += TC_THREADS / GA) {
            const int cp = s_cpos[r];
            if (cp < 0) continue;
            float acc[16];
#pragma unroll
            for (int i = 0; i < 16; i++) acc[i] = s_dw[9 * a.C + c0 + i];
            const unsigned char *base = sS + cp * pix + g_own * 16;
#pragma unroll
            for (int t = 0; t < 9; t++) {
                const int shift = (t / 3 - 1) * a.Wp + (t % 3 - 1);
                float f[16];
                tc::unpack16(*reinterpret_cast<const uint4 *>(base + shift * pix), f);
                const float *w = &s_dw[t * a.C + c0];
                // separate multiply and add (no FMA): bit-identical to the integer oracle's float32 arithmetic, so a
                // rounding flip here cannot be amplified by the following integer GEMM into a multi-LSB difference
#pragma unroll
                for (int i = 0; i < 16; i++) acc[i] = __fadd_rn(acc[i], __fmul_rn(f[i], w[i]));
            }
            int q[16];
#pragma unroll
            for (int i = 0; i < 16; i++) q[i] = tc::q8(__fmul_rn(fmaxf(acc[i], 0.f), a.inv_mid));
            uint4 pk;
            pk.x = tc::pack4(q[0], q[1], q[2], q[3]);   pk.y = tc::pack4(q[4], q[5], q[6], q[7]);
            pk.z = tc::pack4(q[8], q[9], q[10], q[11]); pk.w = tc::pack4(q[12], q[13], q[14], q[15]);
            *reinterpret_cast<uint4 *>(sA + (size_t)g_own * lbo_a + (size_t)r * 16) = pk;
        }
    } else {                                  // K padding group (C = 16): zeros
        for (int r = tid / GA; r < a.rows; r += TC_THREADS / GA)
            *reinterpret_cast<uint4 *>(sA + (size_t)g_own * lbo_a + (size_t)r * 16) = make_uint4(0, 0, 0, 0);
    }
    tc::fence_async_smem();
    __syncthreads();
    if (64 * (warp >> 2) >= a.rows) return;       // rows = 64: the second warpgroup has no GEMM rows
    tc::mbar_wait(&bar_b, 0);
    long orow[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int r = tc_frag_row() + 8 * e, m = m0 + r;
        orow[e] = (r < a.rows && m < M) ? m : -1;
    }
    const uint32_t a_addr = tc::smem_u32(sA) + (uint32_t)(64 * (warp >> 2)) * 16u, b_addr = tc::smem_u32(sB);
    const uint32_t lbo_b = (uint32_t)a.N * 16;
    const TcOutI8 o{a.out, a.Ntotal, a.Ntotal, 1, nullptr, 0, 0};
    wg::for_chunks<(NT < 64 ? NT : 64)>(a.N, [&](auto nc, int n0) {
        constexpr int NC = decltype(nc)::value;
        int d[NC / 2];                   // not zeroed: the first MMA runs with scale-d = 0 (see wg::fence)
        wg::fence();
        for (int ks = 0; ks < (GA >> 1); ks++) {
            const uint64_t ad = wg::desc(a_addr + (uint32_t)(2 * ks) * lbo_a, lbo_a, 128);
            const uint64_t bd = wg::desc(b_addr + (uint32_t)(2 * ks) * lbo_b + (uint32_t)n0 * 16u, lbo_b, 128);
            wg::mma_s8<NC>(d, ad, bd, ks > 0);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(d);
        tc_epilogue_i8<NC>(d, n0, s_mult, s_bq, o, orow, (int)blockIdx.y * a.N);
    });
}

}  // namespace rf
