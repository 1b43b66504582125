// tc_dwpw2d_i8.cuh -- INT8 twin of k_tc_dwpw_2d (tc_dwpw2d.cuh): fused depthwise 3x3 + pointwise 1x1 on the large feature
// maps, 2-D tiles, int8 activations.  Arithmetic is that of k_tc_dwpw_staged_i8 (tc_conv_i8.cuh), operation by operation:
// FP32 depthwise stencil on the int8 input with the input scale folded into the weights, taps in (ky, kx) order, separate
// multiply and add (no FMA), ReLU, requantisation with the depthwise tensor's scale into the int8 A operand;
// wgmma .s32.s8.s8 with an S32 accumulator; epilogue rint(acc * mult[n] + bq[n]) -- so every output byte equals the
// 1-D kernel's and the integer oracle's (oracle/mnet_int8.py).
// Work item of the stencil: 8 channels (half of a 16-byte group) x one column x a PAIR of output rows at stride 1.
#pragma once
#include "tc_conv_i8.cuh"
#include "tc_dwpw2d.cuh"

namespace rf {

struct TcDw2dArgsI8 {
    const int8_t *in;       // NHWC dense [nimg][IH][IW][C], C in {16, 32, 64}
    int C, nimg, IH, IW, OH, OW, S;
    int N, Kpad;            // Kpad = C rounded up to 32
    int TH, TW, tiles_x, tiles_y, PH, PW;
    uint32_t lbo_a;
    uint32_t mul_TW;        // fast_div multiplier (tc_dw2d_i8_finish)
    const int8_t *wimg;     // [Kpad/16][N][16]
    const float *mult, *bq; // [N]
    const float *dw_w;      // [9][C] folded depthwise weights * s_in
    const float *dw_b;      // [C]
    float inv_mid;          // 1 / scale of the depthwise output tensor
    int8_t *out;            // [nimg][OH][OW][N]
};

inline void tc_dw2d_i8_finish(TcDw2dArgsI8 &a) {
    a.PH = (a.TH - 1) * a.S + 3;
    a.PW = (a.TW - 1) * a.S + 3;
    a.tiles_x = (a.OW + a.TW - 1) / a.TW;
    a.tiles_y = (a.OH + a.TH - 1) / a.TH;
    a.lbo_a = 129 * 16;
    a.mul_TW = fast_div_mul((uint32_t)a.TW);
}
inline size_t tc_dw2d_i8_smem_bytes(const TcDw2dArgsI8 &a) {
    return (size_t)a.PH * a.PW * a.C + (size_t)(a.Kpad / 16) * a.lbo_a + (size_t)a.Kpad * a.N + 128 + 16;
}

template <int NT>
__global__ void __launch_bounds__(TC_THREADS, 3) k_tc_dwpw_2d_i8(const TcDw2dArgsI8 a) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_b;
    __shared__ float s_mult[256], s_bq[256];
    __shared__ __align__(16) float s_dw[10 * 64];     // [tap][C] (input scale folded in), [9] = bias

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = a.C >> 4, lg = 31 - __clz(G);       // 16-byte groups per pixel
    const int GA = a.Kpad >> 4;
    const int H8 = a.C >> 3, lh = 31 - __clz(H8);     // 8-channel halves per pixel
    const int PH = a.PH, PW = a.PW;
    const uint32_t lbo_a = a.lbo_a;
    const int pix = a.C;                              // bytes per staged pixel
    unsigned char *sS = smem;
    unsigned char *sA = smem + (((size_t)PH * PW * pix + 15) & ~(size_t)15);
    unsigned char *sB = sA + (size_t)GA * lbo_a;
    const int b = blockIdx.z;
    const int oy0 = blockIdx.y * a.TH, ox0 = blockIdx.x * a.TW;
    const int iy0 = oy0 * a.S - 1, ix0 = ox0 * a.S - 1;

    if (tid == 0) {
        tc::mbar_init(&bar_b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)((size_t)a.Kpad * a.N);
        tc::mbar_expect_tx(&bar_b, bytes);
        tc::bulk_g2s(sB, a.wimg, bytes, &bar_b);
    }
    pdl_trigger();
    if (tid < a.N) { s_mult[tid] = a.mult[tid]; s_bq[tid] = a.bq[tid]; }
    for (int i = tid; i < 10 * a.C; i += TC_THREADS) s_dw[i] = i < 9 * a.C ? a.dw_w[i] : a.dw_b[i - 9 * a.C];
    if (GA > G)                                       // K padding group (C = 16): zeros
        for (int r = tid; r < 128; r += TC_THREADS) *reinterpret_cast<uint4 *>(sA + (size_t)G * lbo_a + (size_t)r * 16) = make_uint4(0, 0, 0, 0);
    pdl_wait();
    {   // stage the window: a byte-for-byte copy of the NHWC rows (see tc_dwpw2d.cuh)
        const int per_row = PW << lg;
        const int px_lo = max(0, -ix0), px_hi = min(PW, a.IW - ix0);
        for (int py = warp; py < PH; py += TC_THREADS / 32) {
            const int iy = iy0 + py;
            const bool rowok = iy >= 0 && iy < a.IH;
            const int8_t *src_row = a.in + (ptrdiff_t)(((b * a.IH + (rowok ? iy : 0)) * a.IW + ix0) * a.C);
            unsigned char *dst_row = sS + py * PW * pix;
            for (int i = lane; i < per_row; i += 32) {
                const int px = i >> lg;
                const bool ok = rowok && px >= px_lo && px < px_hi;
                cp_async16_zfill(dst_row + i * 16, src_row + (ok ? i * 16 : -ix0 * a.C), ok);
            }
        }
    }
    cp_async_wait_all();
    __syncthreads();
    const int rows = a.TH * a.TW;
    if (a.S == 1) {
        const int items = (a.TH >> 1) * a.TW << lh;
        for (int it = tid; it < items; it += TC_THREADS) {
            const int hg = it & (H8 - 1), rest = it >> lh;
            const int typ = fast_div(rest, a.mul_TW), tx = rest - typ * a.TW;
            const int ty = typ * 2, c0 = hg * 8;
            float acc0[8], acc1[8];
#pragma unroll
            for (int i = 0; i < 8; i++) acc0[i] = acc1[i] = s_dw[9 * a.C + c0 + i];
            const unsigned char *base = sS + (ty * PW + tx) * pix + hg * 8;
#pragma unroll 1
            for (int ry = 0; ry < 4; ry++) {
#pragma unroll
                for (int kx = 0; kx < 3; kx++) {
                    float f[8];
                    tc::unpack8(*reinterpret_cast<const uint2 *>(base + (ry * PW + kx) * pix), f);
                    if (ry < 3) {
                        const float *w = &s_dw[(ry * 3 + kx) * a.C + c0];
#pragma unroll
                        for (int i = 0; i < 8; i++) acc0[i] = __fadd_rn(acc0[i], __fmul_rn(f[i], w[i]));
                    }
                    if (ry > 0) {
                        const float *w = &s_dw[((ry - 1) * 3 + kx) * a.C + c0];
#pragma unroll
                        for (int i = 0; i < 8; i++) acc1[i] = __fadd_rn(acc1[i], __fmul_rn(f[i], w[i]));
                    }
                }
            }
            int q0[8], q1[8];
#pragma unroll
            for (int i = 0; i < 8; i++) {
                q0[i] = tc::q8(__fmul_rn(fmaxf(acc0[i], 0.f), a.inv_mid));
                q1[i] = tc::q8(__fmul_rn(fmaxf(acc1[i], 0.f), a.inv_mid));
            }
            const int r = ty * a.TW + tx;
            unsigned char *dst = sA + (size_t)(hg >> 1) * lbo_a + (size_t)r * 16 + (hg & 1) * 8;
            *reinterpret_cast<uint2 *>(dst) = make_uint2(tc::pack4(q0[0], q0[1], q0[2], q0[3]), tc::pack4(q0[4], q0[5], q0[6], q0[7]));
            *reinterpret_cast<uint2 *>(dst + (size_t)a.TW * 16) = make_uint2(tc::pack4(q1[0], q1[1], q1[2], q1[3]), tc::pack4(q1[4], q1[5], q1[6], q1[7]));
        }
    } else {
        const int items = rows << lh;
        for (int it = tid; it < items; it += TC_THREADS) {
            const int hg = it & (H8 - 1), r = it >> lh;
            const int ty = fast_div(r, a.mul_TW), tx = r - ty * a.TW;
            const int c0 = hg * 8;
            float acc[8];
#pragma unroll
            for (int i = 0; i < 8; i++) acc[i] = s_dw[9 * a.C + c0 + i];
            const unsigned char *base = sS + (ty * a.S * PW + tx * a.S) * pix + hg * 8;
#pragma unroll
            for (int t = 0; t < 9; t++) {
                float f[8];
                tc::unpack8(*reinterpret_cast<const uint2 *>(base + ((t / 3) * PW + (t % 3)) * pix), f);
                const float *w = &s_dw[t * a.C + c0];
#pragma unroll
                for (int i = 0; i < 8; i++) acc[i] = __fadd_rn(acc[i], __fmul_rn(f[i], w[i]));
            }
            int q[8];
#pragma unroll
            for (int i = 0; i < 8; i++) q[i] = tc::q8(__fmul_rn(fmaxf(acc[i], 0.f), a.inv_mid));
            *reinterpret_cast<uint2 *>(sA + (size_t)(hg >> 1) * lbo_a + (size_t)r * 16 + (hg & 1) * 8) =
                make_uint2(tc::pack4(q[0], q[1], q[2], q[3]), tc::pack4(q[4], q[5], q[6], q[7]));
        }
    }
    tc::fence_async_smem();
    __syncthreads();
    if (64 * (warp >> 2) >= rows) return;         // the second warpgroup has no GEMM rows
    tc::mbar_wait(&bar_b, 0);
    long orow[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int r = tc_frag_row() + 8 * e;
        const int ty = fast_div(r, a.mul_TW), tx = r - ty * a.TW;
        const int oy = oy0 + ty, ox = ox0 + tx;
        orow[e] = (r < rows && oy < a.OH && ox < a.OW) ? (long)((b * a.OH + oy) * a.OW + ox) : -1;
    }
    const uint32_t a_addr = tc::smem_u32(sA) + (uint32_t)(64 * (warp >> 2)) * 16u, b_addr = tc::smem_u32(sB);
    const uint32_t lbo_b = (uint32_t)a.N * 16;
    const TcOutI8 o{a.out, a.N, a.N, 1, nullptr, 0, 0};
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
        tc_epilogue_i8<NC>(d, n0, s_mult, s_bq, o, orow, 0);
    });
}

}  // namespace rf
