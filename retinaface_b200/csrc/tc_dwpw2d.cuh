// tc_dwpw2d.cuh -- fused depthwise 3x3 (stride 1|2) + BN + ReLU -> pointwise 1x1 + BN + ReLU for the LARGE feature maps
// (112x112, 56x56 at 448x448 input: conv3..conv10, prototxt:143-488), 2-D tiles.
//
// Same arithmetic, rounding points and GEMM as k_tc_dwpw_staged (tc_conv.cuh): the depthwise stencil runs on CUDA cores
// from staged shared memory (FP32 accumulate, FP16 round) straight into the MMA A operand, the pointwise GEMM on wgmma
// with the accumulator in registers.  What differs is the tile: TH x TW output pixels of ONE image (TH*TW <= 128) instead of
// 128 consecutive pixels of the linearised map.  On a wide map the 1-D tile stages 128 + 2*(W+3) input positions for 128
// outputs (2.8x at W = 112); the 2-D tile stages ((TH-1)*S+3) x ((TW-1)*S+3) (1.4x), needs no position table (a staged
// row is a contiguous run of the NHWC input: the cp.async addresses are affine in the lane), and a pair of horizontally
// adjacent outputs sits in one thread: each staged activation it reads is converted once for both (dw_stencil_block).
#pragma once
#include "tc_conv.cuh"

namespace rf {

struct TcDw2dArgs {
    const __half *in;       // NHWC dense [nimg][IH][IW][C], C in {16, 32, 64}
    int C, nimg, IH, IW, OH, OW, S;
    int N;                  // output channels (multiple of 16, <= 256)
    int TH, TW;             // output tile, TH * TW <= 128, TH even
    int tiles_x, tiles_y;
    int run;                // consecutive tiles per CTA (tiles of all images numbered image-major); grid = ceil(tiles / run)
    int stages;             // staged windows in the ring: 2 or 3 (plan_pair_tc)
    int PH, PW;             // staged window: (TH-1)*S+3 x (TW-1)*S+3   (tc_dw2d_finish)
    uint32_t lbo_a;         // group stride of the A operand, bytes (tc_dw2d_finish)
    uint32_t mul_TW, mul_tiles_x, mul_tiles, mul_cpp;   // fast_div multipliers (tc_dw2d_finish)
    const __half *wimg;     // [C/8][N][8]
    const float *bias;      // [N]
    const float *dw_w, *dw_b;   // [9][C], [C]
    __half *out;            // [nimg][OH][OW][N]
};

// Derived geometry, computed once on the host.  The staged window is PIXEL-major, [PH][PW][C] -- a byte-for-byte copy of the
// NHWC rows it comes from: consecutive cp.async lanes write consecutive shared addresses (one wavefront per 128 bytes; a
// channel-group-major layout scatters every 16-byte piece into its own wavefront), and the stencil's lanes -- (group, column)
// with the group fastest -- read consecutive 16-byte pieces.  The A operand's group stride in 16-byte units is 8/G mod 8, so
// that the 8 lanes of a quarter warp hit 8 different bank groups.
inline void tc_dw2d_finish(TcDw2dArgs &a) {
    const int G = a.C >> 3;
    a.PH = (a.TH - 1) * a.S + 3;
    a.PW = (a.TW - 1) * a.S + 3;
    a.tiles_x = (a.OW + a.TW - 1) / a.TW;
    a.tiles_y = (a.OH + a.TH - 1) / a.TH;
    a.lbo_a = (uint32_t)(128 + 8 / G) * 16;
    a.mul_TW = fast_div_mul((uint32_t)a.TW);
    a.mul_tiles_x = fast_div_mul((uint32_t)a.tiles_x);
    a.mul_tiles = fast_div_mul((uint32_t)(a.tiles_x * a.tiles_y));
    a.mul_cpp = fast_div_mul((uint32_t)(a.N >> 3));
}
inline size_t tc_dw2d_stage_bytes(const TcDw2dArgs &a) { return (size_t)a.PH * a.PW * a.C * 2; }
// The output tile, [128 rows][N + 8 halfs]: the 16-byte pad per row puts the 8 rows of an accumulator fragment's store in 8
// different bank groups.  It is written into the staged window the tile has just consumed.
inline size_t tc_dw2d_out_bytes(const TcDw2dArgs &a) { return (size_t)128 * (a.N * 2 + 16); }
inline bool tc_dw2d_out_fits(const TcDw2dArgs &a) { return tc_dw2d_out_bytes(a) <= tc_dw2d_stage_bytes(a); }
inline size_t tc_dw2d_smem_bytes(const TcDw2dArgs &a) {
    return (size_t)a.stages * tc_dw2d_stage_bytes(a) + (size_t)(a.C / 8) * a.lbo_a + (size_t)a.C * a.N * 2 + 128;
}

// resident CTAs per SM the register allocation aims at (75 registers at 3; at 4 -- 64 registers -- the persistent loop
// spills).  The pointwise accumulator is taken in chunks of at most 32 columns.
#ifndef RF_DW2D_OCC
#define RF_DW2D_OCC 3
#endif
template <int NT>
__global__ void __launch_bounds__(TC_THREADS, RF_DW2D_OCC) k_tc_dwpw_2d(const TcDw2dArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_b;
    __shared__ float s_bias[256];
    __shared__ __align__(16) float s_dww[9 * 64];     // [tap][C] folded depthwise weights, FP16-rounded, as FP32 (dw_stencil_block)
    __shared__ __align__(16) float s_dwb[64];         // [C] bias

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = a.C >> 3, lg = 31 - __clz(G);
    const int PH = a.PH, PW = a.PW, ns = a.stages;
    const uint32_t lbo_a = a.lbo_a;
    const int pix = a.C * 2;             // bytes per staged pixel
    const uint32_t stage_bytes = (uint32_t)(PH * PW * pix);
    unsigned char *sA = smem + (size_t)ns * stage_bytes;         // behind the staging ring
    unsigned char *sB = sA + (size_t)G * lbo_a;
    const int tiles = a.tiles_x * a.tiles_y;
    const int t_begin = (int)blockIdx.x * a.run;
    const int t_end = min(t_begin + a.run, tiles * a.nimg);
    // tile t -> image b, output origin (oy0, ox0); a CTA's run of tiles may cross from one image into the next
    auto decode = [&](int t, int &b, int &oy0, int &ox0) {
        b = fast_div(t, a.mul_tiles);
        const int trem = t - b * tiles, ty0 = fast_div(trem, a.mul_tiles_x);
        oy0 = ty0 * a.TH; ox0 = (trem - ty0 * a.tiles_x) * a.TW;
    };

    if (tid == 0) {
        tc::mbar_init(&bar_b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)((size_t)a.C * a.N * 2);
        tc::mbar_expect_tx(&bar_b, bytes);
        tc::bulk_g2s(sB, a.wimg, bytes, &bar_b);
    }
    pdl_trigger();
    if (tid < a.N) s_bias[tid] = a.bias[tid];
    for (int i = tid; i < 9 * a.C; i += TC_THREADS) s_dww[i] = dw_weight_f16(a.dw_w[i]);
    if (tid < a.C) s_dwb[tid] = a.dw_b[tid];
    pdl_wait();
    // ---- stage tile t's (PH x PW) input window into buffer buf: one warp per staged row, lanes over (column, channel
    // group) -- a staged row is PW*C contiguous halfs of the input (16 B per lane, fully coalesced); outside the map: zero
    // fill.  Every call commits one cp.async group, an empty one past the end of the run, so that the window of tile t is
    // always the group issued ns - 1 calls before the latest
    const uint32_t sS_s = tc::smem_u32(smem);
    auto stage = [&](int t, int buf) {
        if (t < t_end) {
            int b, oy0, ox0;
            decode(t, b, oy0, ox0);
            const int iy0 = oy0 * a.S - 1, ix0 = ox0 * a.S - 1;      // input coordinates of staged (0, 0)
            // item i of a row = (column px = i / G, group g = i % G): with C = 8 G its source is src_row + 8 i halfs -- affine in i
            const int per_row = PW << lg;
            const int px_lo = max(0, -ix0), px_hi = min(PW, a.IW - ix0);       // columns inside the map
            const unsigned px_n = (unsigned)max(px_hi - px_lo, 0);
            for (int py = warp; py < PH; py += TC_THREADS / 32) {
                const int iy = iy0 + py;
                const bool rowok = iy >= 0 && iy < a.IH;
                const __half *src_row = a.in + (ptrdiff_t)(((b * a.IH + (rowok ? iy : 0)) * a.IW + ix0) * a.C);
                const uint32_t dst_row = sS_s + (uint32_t)buf * stage_bytes + (uint32_t)(py * PW * pix);
                const __half *zsrc = a.in;      // any valid address: zero bytes are read from it
                for (int i = lane; i < per_row; i += 32) {
                    const bool ok = rowok && (unsigned)((i >> lg) - px_lo) < px_n;
                    cp_async16_zfill_s(dst_row + (uint32_t)i * 16u, ok ? src_row + i * 8 : zsrc, ok);
                }
            }
        }
        cp_async_commit();
    };
    // ---- depthwise stencil of the window at sS -> A operand.  GEMM row r = ty * TW + tx ------------------------------------
    // item = (channel group, NX horizontally adjacent outputs).  A pair (NX = 2) at stride 1 reads a 3x4 window for 2 outputs
    // (12 conversions for 18 taps), at stride 2 a 3x5 window (15 for 18); TW is even.  Where pairs are fewer than the threads
    // (C = 16: 64 pairs x 2 groups) every thread takes one output instead (9 conversions for 9 taps), so that none waits at
    // the barrier while the others compute.  A 2x2 block (16 / 25 conversions for 36 taps) has half as many items again.
    auto stencil = [&](auto s_, auto nx_, const unsigned char *sS) {
        constexpr int S = decltype(s_)::value, NX = decltype(nx_)::value;
        const int items = (a.TH * a.TW / NX) << lg;
        for (int it = tid; it < items; it += TC_THREADS) {
            const int g = it & (G - 1), rest = it >> lg;
            const int ty = fast_div(NX * rest, a.mul_TW), tx = NX * rest - ty * a.TW;
            float acc[1][NX][8];
            dw_bias8(acc[0][0], &s_dwb[g * 8]);
#pragma unroll
            for (int q = 1; q < NX; q++)
#pragma unroll
                for (int i = 0; i < 8; i++) acc[0][q][i] = acc[0][0][i];
            dw_stencil_block<S, 1, NX>(acc, sS + (ty * S * PW + tx * S) * pix + g * 16, PW * pix, pix, &s_dww[g * 8], a.C);
            unsigned char *dst = sA + (size_t)g * lbo_a + (size_t)(ty * a.TW + tx) * 16;
#pragma unroll
            for (int q = 0; q < NX; q++) *reinterpret_cast<uint4 *>(dst + 16 * q) = dw_relu_h8(acc[0][q]);
        }
    };
    const bool singles = ((a.TH * a.TW / 2) << lg) < TC_THREADS;
    const int rows = a.TH * a.TW;
    const bool has_gemm = 64 * (warp >> 2) < rows;      // the second warpgroup has no GEMM rows when TH * TW <= 64
    const uint32_t ostride = (uint32_t)a.N * 2 + 16;     // bytes per row of the output tile (tc_dw2d_out_bytes)
    const int cpp = a.N >> 3;                             // 16-byte pieces per output pixel
    for (int j = 0; j < ns - 1; j++) stage(t_begin + j, j);
    // ---- persistent loop over the CTA's run of tiles: the windows of tiles t + 1 .. t + ns - 1 are in flight while tile t
    // computes.  Three barriers per tile: X (window t landed; tile t - 1's output tile read), Y (A operand written), Z
    // (output tile written)
    for (int t = t_begin, buf = 0; t < t_end; t++, buf = buf + 1 == ns ? 0 : buf + 1) {
        if (ns == 3) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_group 0;" ::: "memory");
        // X: every thread's pieces of window t have landed, and every thread is done with tile t - 1: its stencil read the
        // buffer the next window goes into, its stores read that buffer's output tile
        __syncthreads();
        stage(t + ns - 1, buf == 0 ? ns - 1 : buf - 1);
        unsigned char *sS = smem + (size_t)buf * stage_bytes;
        if (a.S == 1) {
            if (singles) stencil(std::integral_constant<int, 1>{}, std::integral_constant<int, 1>{}, sS);
            else stencil(std::integral_constant<int, 1>{}, std::integral_constant<int, 2>{}, sS);
        } else {
            if (singles) stencil(std::integral_constant<int, 2>{}, std::integral_constant<int, 1>{}, sS);
            else stencil(std::integral_constant<int, 2>{}, std::integral_constant<int, 2>{}, sS);
        }
        tc::fence_async_smem();
        __syncthreads();                             // Y: the A operand is complete; window t has been read
        if (has_gemm) {
            tc::mbar_wait(&bar_b, 0);
            const uint32_t a_addr = tc::smem_u32(sA) + (uint32_t)(64 * (warp >> 2)) * 16u, b_addr = tc::smem_u32(sB);
            const uint32_t lbo_b = (uint32_t)a.N * 16;
            // rows of this thread's fragment in the output tile, which takes the place of window t
            unsigned char *orow0 = sS + (uint32_t)tc_frag_row() * ostride + 4 * (lane & 3);
            wg::for_chunks<(NT < 32 ? NT : 32)>(a.N, [&](auto nc, int n0) {
                constexpr int NC = decltype(nc)::value;
                float d[NC / 2];                 // not zeroed: the first MMA runs with scale-d = 0 (see wg::fence)
                wg::fence();
                wg::mma_ss<NC>(d, wg::desc(a_addr, lbo_a, 128), wg::desc(b_addr + (uint32_t)n0 * 16u, lbo_b, 128), 0);
                for (int ks = 1; ks < (a.C >> 4); ks++) {
                    const uint64_t ad = wg::desc(a_addr + (uint32_t)(2 * ks) * lbo_a, lbo_a, 128);
                    const uint64_t bd = wg::desc(b_addr + (uint32_t)(2 * ks) * lbo_b + (uint32_t)n0 * 16u, lbo_b, 128);
                    wg::mma_ss<NC>(d, ad, bd, 1);
                }
                wg::commit();
                wg::wait<0>();
                wg::fence_regs(d);
                // bias, ReLU and FP16 round as tc_epilogue, into the output tile
                const int c2 = 2 * (lane & 3);
#pragma unroll
                for (int e = 0; e < 2; e++) {
#pragma unroll
                    for (int i = 0; i < NC / 8; i++) {
                        const int n = n0 + 8 * i + c2;
                        const float f0 = fmaxf(d[4 * i + 2 * e] + s_bias[n], 0.f), f1 = fmaxf(d[4 * i + 2 * e + 1] + s_bias[n + 1], 0.f);
                        *reinterpret_cast<__half2 *>(orow0 + 8 * e * ostride + (n0 + 8 * i) * 2) = __floats2half2_rn(f0, f1);
                    }
                }
            });
        }
        __syncthreads();                             // Z: the output tile is complete
        // ---- the output tile -> global memory: an output row of the tile is TW * N contiguous halfs of the NHWC output,
        // stored as 16-byte pieces, consecutive lanes on consecutive pieces; pixels outside the map are not stored
        int b, oy0, ox0;
        decode(t, b, oy0, ox0);
        for (int it = tid; it < rows * cpp; it += TC_THREADS) {
            const int r = fast_div(it, a.mul_cpp), j = it - r * cpp;
            const int ty = fast_div(r, a.mul_TW), tx = r - ty * a.TW;
            const int oy = oy0 + ty, ox = ox0 + tx;
            if (oy >= a.OH || ox >= a.OW) continue;
            const uint4 v = *reinterpret_cast<const uint4 *>(sS + (uint32_t)r * ostride + 16 * j);
            *reinterpret_cast<uint4 *>(a.out + (size_t)((b * a.OH + oy) * a.OW + ox) * a.N + 8 * j) = v;
        }
    }
}

}  // namespace rf
