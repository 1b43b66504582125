// tc_conv.cuh -- tensor-core convolution kernels of librf_b200: FP16 operands in shared memory, FP32 accumulators in
// registers.  sm_90a (wgmma.mma_async, cp.async.bulk, mbarrier, griddepcontrol).
//
// Two kernels cover every GEMM-shaped layer of the network (model/mnet-deconv-0517.prototxt):
//   k_tc_conv_staged : 1x1 and 3x3 (pad 1) convolutions -- rf_c*_lateral / rf_c1_red_conv, rf_c*_aggr, the SSH
//                      det/context convs (branches that share an input run as one conv, outputs split);
//                      UPADD variant: the FPN merge (deconv-upsample + crop + add) fused into the staging.
//   k_tc_dwpw_staged : depthwise 3x3 (stride 1|2) + BN + ReLU fused with the following pointwise 1x1 + BN +
//                      ReLU (mobilenet0_conv3..conv26): the stencil runs on CUDA cores from shared memory
//                      straight into the A operand of the tensor-core GEMM.
// GEMM view: D[128 rows][N] (+)= A[128][K] * W[N][K]^T, one CTA (256 threads) per 128-row tile.
//   Operand layout : canonical K-major, no swizzle: 8x8 core matrices (8 rows x 16 B), SBO = 128 B between
//                    8-row groups, LBO between 8-channel groups (odd multiple of 16 B, so 16-byte shared stores of
//                    a quarter-warp never conflict).  Descriptors: wgmma.cuh.
//   A operand      : "staged range + shifted descriptors", see below -- no im2col, not even in shared memory.
//   B operand      : weights pre-packed on the host as the exact shared-memory image, fetched by ONE TMA bulk
//                    copy (cp.async.bulk ... mbarrier::complete_tx) per CTA, issued before griddepcontrol.wait so
//                    it overlaps the previous kernel (programmatic dependent launch).
//   MMA            : wgmma.mma_async m64nNCk16, warpgroup w (128 threads) computes GEMM rows [64 w, 64 w + 64); N = Cout
//                    (16..256) in column chunks of NC <= 64, so the accumulator is at most 32 registers per thread.
//   Epilogue       : straight from the accumulator fragment: + folded-BN bias (shared memory), ReLU, FP16 pairs; the
//                    output channels may be split over two destinations with their own pixel stride (Concat + ReLU fusion).
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace rf {

constexpr int TC_LBO_A = 128 * 16 + 16;        // bytes between 8-channel groups of the A tile

struct TcOut {
    __half *p0; int ld0; int n0; int relu0;    // channels [0, n0)  -> p0[m*ld0 + n]
    __half *p1; int ld1; int relu1;            // channels [n0, N)  -> p1[m*ld1 + n - n0]
};

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
    unsigned done = 0;
    unsigned spins = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (!done && ++spins > (1u << 24)) __trap();   // a lost arrive must fail loudly, never hang the GPU
    }
}
// TMA bulk copy global -> shared, completion counted on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace tc

// kernel template bucket of a layer's N: the kernels instantiate accumulator chunks up to min(bucket, 64) columns
constexpr int tc_n_bucket(int n) { return n <= 32 ? 32 : (n <= 64 ? 64 : (n <= 128 ? 128 : 256)); }

// =============================================================================================
// v2 kernels: "staged range + shifted descriptors".
//
// The input pixels a 128-row tile needs form ONE contiguous range of a zero-padded linear
// position space: position p <-> (image b, row yy in [0,H], column xx in [0,W+1]) with
// p = (b*(H+1) + yy)*(W+2) + xx; xx = 0 / W+1 and yy = H are zero padding (one shared zero row
// between consecutive images).  The range is staged ONCE into shared memory as
// [channel group g][position][8 halfs] (16 B per item, cp.async with zero-fill for padding), which
// is exactly the canonical K-major no-swizzle layout with SBO = 128 B and LBO = R*16 B.  In
// this space a 3x3 tap is a constant position shift dy*(W+2)+dx, so the A operand of every tap is
// the SAME staged buffer with the descriptor start address moved by shift*16 bytes: the im2col
// matrix is never materialised, not even in shared memory.  GEMM rows enumerate padded positions
// (W/(W+2) of them are real pixels; results of padding rows are discarded).
// =============================================================================================
constexpr int TC_THREADS = 256;
constexpr int TC_MAX_R = 2048;     // staged positions per tile (table size)

struct TcConvArgs {
    const __half *in;       // NHWC dense [nimg][H][W][Cin]
    int Cin, nimg, H, W;
    int taps;               // 1 (pointwise) or 9 (3x3, pad 1)
    int N;                  // output channels (multiple of 16, <= 256)
    int Wp, Hp;             // padded geometry: taps==9 ? (W+2, H+1) : (W, H)
    int R;                  // staged positions per tile (odd): 128 + 2*(Wp+1) for 3x3, 129 for 1x1
    uint32_t mul_Wp, mul_Hp, mul_H;   // fast_div multipliers (set by the launch helper)
    const __half *wimg;     // B image [K/8][N][8] halfs, K = taps*Cin ordered (tap, cin)
    const float *bias;      // [N]
    TcOut out;
    // FPN merge fused into the staging (template UPADD): in := in + crop(deconv_k4s2p1(up)) -- the
    // Eltwise SUM of prototxt:1585 / :1980 never exists as a tensor.  up: [nimg][H/2][W/2][Cin], up_w: [Cin][16].
    const __half *up;
    const float *up_w;
    int Cmax;               // UPADD: staged coarse positions per tile, upper bound (odd)
};

__device__ __forceinline__ void cp_async16_zfill(void *smem_dst, const void *gsrc, bool valid) {
    const unsigned sz = valid ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(tc::smem_u32(smem_dst)), "l"(gsrc), "r"(sz) : "memory");
}
// same with the destination given as a shared-window address (tc::smem_u32 hoisted out of the caller's loop)
__device__ __forceinline__ void cp_async16_zfill_s(uint32_t smem_dst, const void *gsrc, bool valid) {
    const unsigned sz = valid ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gsrc) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(tc::smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

// GEMM rows of this thread in the accumulator fragment of its warpgroup (wgmma.cuh): tc_frag_row() and tc_frag_row() + 8
__device__ __forceinline__ int tc_frag_row() { return 64 * (threadIdx.x >> 7) + 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2); }

// Epilogue of one accumulator chunk (columns [n0, n0 + NC) of the CTA's N), shared by both kernels: rows out_row[e] < 0 are
// not stored.
template <int NC>
__device__ __forceinline__ void tc_epilogue(const float (&d)[NC / 2], int n0, const float *s_bias /* smem, this CTA's N channels */,
                                            const TcOut &o, const long (&out_row)[2], int n_off) {
    const int c2 = 2 * (threadIdx.x & 3);
#pragma unroll
    for (int e = 0; e < 2; e++) {
        if (out_row[e] < 0) continue;
#pragma unroll
        for (int i = 0; i < NC / 8; i++) {
            const int n = n0 + 8 * i + c2;
            const int gn = n_off + n;             // channel index in the layer's full output
            const bool first = gn < o.n0;
            const int relu = first ? o.relu0 : o.relu1;
            __half *dst = first ? o.p0 + (size_t)out_row[e] * o.ld0 + gn : o.p1 + (size_t)out_row[e] * o.ld1 + (gn - o.n0);
            float f0 = d[4 * i + 2 * e] + s_bias[n], f1 = d[4 * i + 2 * e + 1] + s_bias[n + 1];
            if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
            *reinterpret_cast<__half2 *>(dst) = __floats2half2_rn(f0, f1);
        }
    }
}

inline size_t tc_conv_smem_bytes(const TcConvArgs &a) {
    // staged range + weight image (+ UPADD: staged coarse rows) + the position tables (s_off, UPADD: s_yx)
    return (size_t)(a.Cin / 8) * a.R * 16 + (size_t)a.taps * a.Cin * a.N * 2 + (a.up ? (size_t)(a.Cin / 8) * a.Cmax * 16 : 0) +
           (size_t)a.R * 4 * (a.up ? 2 : 1) + 128;
}

template <int NT, bool UPADD>
__global__ void __launch_bounds__(TC_THREADS) k_tc_conv_staged(const TcConvArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_b;
    __shared__ float s_bias[256];
    __shared__ __align__(16) __half s_uw[UPADD ? 64 * 16 : 8];   // [tap][channel] deconv weights as FP16 (bilinear taps are exact)
    __shared__ int s_crow[2];            // UPADD: [lo, hi] global coarse rows (b*UH + i) the tile reads

    const int tid = threadIdx.x, warp = tid >> 5;
    const int pad = a.taps == 9 ? 1 : 0;
    const int G = a.Cin >> 3;
    const uint32_t lbo_s = (uint32_t)a.R * 16;
    unsigned char *sS = smem;
    unsigned char *sB = smem + (size_t)G * lbo_s;
    // position tables behind the operands (sized by R, so that the footprint -- and with it the number of co-resident
    // CTAs -- follows the layer): s_off: staged position -> element offset of its pixel in `in`, -1 = zero padding;
    // UPADD: s_yx: staged position -> (global fine row b*H+y) << 12 | x
    int *s_off = reinterpret_cast<int *>(sB + (size_t)a.taps * a.Cin * a.N * 2 + (UPADD ? (size_t)G * a.Cmax * 16 : 0));
    int *s_yx = s_off + a.R;
    const int m0 = blockIdx.x * 128;
    const int lo = m0 - (a.Wp + 1) * pad;

    if (tid == 0) {
        s_crow[0] = 0x7fffffff; s_crow[1] = -1;
        tc::mbar_init(&bar_b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)((size_t)a.taps * a.Cin * a.N * 2);
        tc::mbar_expect_tx(&bar_b, bytes);
        tc::bulk_g2s(sB, a.wimg, bytes, &bar_b);     // all taps' weights: one TMA bulk copy
    }
    pdl_trigger();
    if (tid < a.N) s_bias[tid] = a.bias[tid];
    if (UPADD) for (int i = tid; i < a.Cin * 16; i += TC_THREADS) s_uw[(i & 15) * 64 + (i >> 4)] = __float2half_rn(a.up_w[i]);
    // position table, one warp per padded row (no per-position divisions): p = prow * Wp + xx
    {
        const int lane = tid & 31;
        const int prow0 = fast_floor_div(lo, a.Wp, a.mul_Wp);          // floor
        const int prow1 = fast_div(lo + a.R - 1, a.mul_Wp);
        for (int prow = prow0 + warp; prow <= prow1; prow += TC_THREADS / 32) {
            const int b = prow >= 0 ? fast_div(prow, a.mul_Hp) : -1;
            const int yy = prow >= 0 ? (int)(prow - b * a.Hp) : 0;
            const bool rowok = prow >= 0 && b < a.nimg && yy < a.H;
            for (int xx = lane; xx < a.Wp; xx += 32) {
                const int pl = prow * a.Wp + xx - lo;
                if (pl < 0 || pl >= a.R) continue;
                int off = -1;
                if (rowok && xx >= pad && xx < a.W + pad) {
                    off = ((b * a.H + yy) * a.W + (xx - pad)) * a.Cin;
                    if (UPADD) {
                        s_yx[pl] = ((b * a.H + yy) << 12) | (xx - pad);
                        const int UH = a.H >> 1, ih = (yy + 1) >> 1;
                        atomicMin(&s_crow[0], b * UH + max(ih - 1, 0));
                        atomicMax(&s_crow[1], b * UH + min(ih, UH - 1));
                    }
                }
                s_off[pl] = off;
            }
        }
    }
    __syncthreads();
    pdl_wait();                          // everything above is independent of the previous kernel's output
    // ---- stage the range: item = (position, 8-channel group), 16 B each --------------------------------
    const int lg = 31 - __clz(G);        // G is a power of two (Cin in {16, 64, 128, 256})
    // lanes run over the channel groups of one pixel first: the 16-byte pieces of a pixel are contiguous in global memory
    // (fully used L2 sectors) and land in G different group planes of the K-major operand.  (Positions fastest -- 16-byte
    // reads at pixel stride -- measured up to 1.6x slower on the 1x1 convs with Cin = 256.)
    const int UH = a.H >> 1, UW = a.W >> 1;
    unsigned char *sC = sB + (size_t)a.taps * a.Cin * a.N * 2;      // UPADD: coarse rows, pixel-major [coarse position][Cin]
    const int crow_lo = UPADD ? s_crow[0] : 0, crow_hi = UPADD ? s_crow[1] : -1;
    if (UPADD && crow_hi >= crow_lo) {
        // FPN merge: staged := lateral + crop(deconv_k4s2p1(up)).  The coarse rows the tile needs (one contiguous range of the
        // coarse map: global coarse rows [crow_lo, crow_hi]) go first, asynchronously and as a plain copy (contiguous shared
        // stores), so that all global traffic of the tile is in flight at once
        const int ncp = (crow_hi - crow_lo + 1) * UW;
        if (ncp > a.Cmax) __trap();
        const __half *csrc = a.up + (size_t)crow_lo * UW * a.Cin;
        for (int it = tid; it < ncp * G; it += TC_THREADS) cp_async16_zfill(sC + (size_t)it * 16, csrc + (size_t)it * 8, true);
    }
    {
        // through registers: LDG.128 (coalesced) then STS.128 -- with R odd the 8 lanes of a quarter warp (8 groups of one
        // pixel) hit 8 different bank groups, so the store costs the ideal 4 wavefronts per warp instead of cp.async's 32
        // TC_THREADS is a multiple of G: a thread keeps ONE channel group and walks positions p0, p0 + pstep, ... -- source and
        // destination addresses are a per-thread base plus a multiple of the position (32-bit adds only)
        constexpr int UNR = 4;
        const int g = tid & (G - 1), p0 = tid >> lg, pstep = TC_THREADS >> lg;
        const __half *src_g = a.in + g * 8;
        unsigned char *dst_g = sS + (uint32_t)g * lbo_s;
        for (int pb = p0; pb < a.R; pb += pstep * UNR) {
            uint4 v[UNR];
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int p = pb + u * pstep;
                v[u] = make_uint4(0, 0, 0, 0);
                if (p < a.R) {
                    const int off = s_off[p];
                    if (off >= 0) v[u] = __ldcg(reinterpret_cast<const uint4 *>(src_g + off));     // L2 only, like cp.async.cg
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; u++) {
                const int p = pb + u * pstep;
                if (p < a.R) *reinterpret_cast<uint4 *>(dst_g + (uint32_t)p * 16u) = v[u];
            }
        }
    }
    if (UPADD) {
        // the add runs shared -> shared, in the same operation order as k_upsample_add (kernels_simt.cuh): the staged FP16
        // values equal the unfused Eltwise tensor
        cp_async_wait_all();
        __syncthreads();
        for (int it = tid; it < a.R * G; it += TC_THREADS) {
            const int g = it & (G - 1), pl = it >> lg;
            const int off = s_off[pl];
            if (off < 0) continue;
            const int c0 = g * 8;
            const int yx = s_yx[pl];
            const int x = yx & 0xfff, gy = yx >> 12;             // gy = b*H + y
            const int b = fast_div(gy, a.mul_H), y = gy - b * a.H;            // one division (vs three): b changes at most once per tile
            unsigned char *slot = sS + (size_t)g * lbo_s + (size_t)pl * 16;
            // packed FP16 arithmetic (HFMA2): the sum of <= 5 terms is stored as FP16 anyway; the reference's
            // deconvolution weights (1/16, 3/16, 9/16) are exact in FP16
            uint4 accv = *reinterpret_cast<const uint4 *>(slot);
            __half2 *acc = reinterpret_cast<__half2 *>(&accv);
            const int i_hi = (y + 1) >> 1, j_hi = (x + 1) >> 1;
#pragma unroll
            for (int di = 0; di < 2; di++) {
                const int i = i_hi - di, ky = y - 2 * i + 1;
                if (i < 0 || i >= UH || ky < 0 || ky > 3) continue;
#pragma unroll
                for (int dj = 0; dj < 2; dj++) {
                    const int j = j_hi - dj, kx = x - 2 * j + 1;
                    if (j < 0 || j >= UW || kx < 0 || kx > 3) continue;
                    const uint4 uv = *reinterpret_cast<const uint4 *>(sC + ((size_t)((b * UH + i - crow_lo) * UW + j) * G + g) * 16);
                    const uint4 wv = *reinterpret_cast<const uint4 *>(&s_uw[(ky * 4 + kx) * 64 + c0]);
                    const __half2 *u2 = reinterpret_cast<const __half2 *>(&uv), *w2 = reinterpret_cast<const __half2 *>(&wv);
#pragma unroll
                    for (int c = 0; c < 4; c++) acc[c] = __hfma2(u2[c], w2[c], acc[c]);
                }
            }
            *reinterpret_cast<uint4 *>(slot) = accv;
        }
    } else {
        cp_async_wait_all();
    }
    tc::fence_async_smem();
    __syncthreads();
    tc::mbar_wait(&bar_b, 0);
    // ---- MMA: taps * Cin/16 instructions per column chunk, A = shifted views of the one staged buffer ------------------
    const int row_base = (int)(m0 - lo);
    long orow[2];
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int off = s_off[row_base + tc_frag_row() + 8 * e];      // element offset / Cin == output pixel index
        orow[e] = off >= 0 ? (off >> (31 - __clz(a.Cin))) : -1;      // Cin is a power of two (plan_conv_legacy checks)
    }
    const uint32_t s_addr = tc::smem_u32(sS) + (uint32_t)(row_base + 64 * (warp >> 2)) * 16u, b_addr = tc::smem_u32(sB);
    const uint32_t lbo_b = (uint32_t)a.N * 16;
    wg::for_chunks<(NT < 64 ? NT : 64)>(a.N, [&](auto nc, int n0) {
        constexpr int NC = decltype(nc)::value;
        float d[NC / 2];                 // not zeroed: the first MMA runs with scale-d = 0 (see wg::fence)
        wg::fence();
        int acc = 0;
        for (int t = 0; t < a.taps; t++) {
            const int shift = pad ? (t / 3 - 1) * a.Wp + (t % 3 - 1) : 0;
            for (int cs = 0; cs < (a.Cin >> 4); cs++) {
                const uint64_t ad = wg::desc(s_addr + (uint32_t)(2 * cs) * lbo_s + (uint32_t)(shift * 16), lbo_s, 128);
                const uint64_t bd = wg::desc(b_addr + (uint32_t)(t * G + 2 * cs) * lbo_b + (uint32_t)n0 * 16u, lbo_b, 128);
                wg::mma_ss<NC>(d, ad, bd, acc);
                acc = 1;
            }
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(d);
        tc_epilogue<NC>(d, n0, s_bias, a.out, orow, 0);
    });
}

// ---------------------------------------------------------------------------------------------
// Fused depthwise 3x3 (stride 1|2) + BN + ReLU -> pointwise 1x1 + BN + ReLU.
// The input range of the tile is staged as above; the depthwise stencil is evaluated from shared
// memory on CUDA cores (FP32 accumulate, FP16 round -- the same rounding point as the unfused
// layer pair) straight into the tensor-core A operand; the pointwise GEMM runs on wgmma.
// rows: 64 or 128 output pixels per CTA (one or both warpgroups run the GEMM);
// blockIdx.y selects a slice of N output channels (keeps the weight image within shared memory).
// ---------------------------------------------------------------------------------------------
struct TcDwArgs {
    const __half *in;       // NHWC dense [nimg][IH][IW][C]
    int C, nimg, IH, IW, OH, OW, S;
    int N;                  // output channels of this CTA slice
    int Ntotal;             // layer output channels (pixel stride of out)
    int Kpad;               // C rounded up to 16
    int rows;               // output pixels per CTA (64 | 128)
    int Wp, Hp;             // IW + 2, IH + 1
    int Rmax;               // staged positions, upper bound over tiles (odd)
    uint32_t mul_Wp, mul_Hp, mul_OW, mul_OH;   // fast_div multipliers (set by the launch helper)
    const __half *wimg;     // slice s at s * Kpad * N halfs: [Kpad/8][N][8]
    const float *bias;      // [Ntotal]
    const float *dw_w, *dw_b;   // [9][C], [C]
    __half *out;            // [nimg][OH][OW][Ntotal]
};

// A operand of the pointwise GEMM: [Kpad/8 groups][rows][16 B], group stride rows*16 + 16.
__host__ __device__ inline uint32_t tc_dw_lbo_a(int rows) { return (uint32_t)rows * 16 + 16; }
inline size_t tc_dw_smem_bytes(const TcDwArgs &a) {
    return (size_t)((a.C + 7) / 8) * a.Rmax * 16 + (size_t)(a.Kpad / 8) * tc_dw_lbo_a(a.rows) + (size_t)a.Kpad * a.N * 2 +
           (size_t)10 * a.C * 4 + (size_t)a.Rmax * 4 + 128;
}

// The depthwise weights and biases sit in shared memory as FP32 (all lanes of a warp read the same few addresses, so the reads
// are broadcasts); a thread computes up to 4 consecutive outputs of one output row (dw_stencil_block).
template <int NT>
__global__ void __launch_bounds__(TC_THREADS, 3) k_tc_dwpw_staged(const TcDwArgs a) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ __align__(8) uint64_t bar_b;
    __shared__ int s_cpos[128];          // GEMM row -> staged index of its stencil centre, -1 = no output
    __shared__ float s_bias[256];

    const int tid = threadIdx.x, warp = tid >> 5;
    const int G = a.C >> 3;
    const int GA = a.Kpad >> 3;          // A groups (== G except the Cin = 8 layer: 2, second one zero)
    const int lgGA = 31 - __clz(GA);          // Kpad / 8 (16) is a power of two
    const int g_own = tid & (GA - 1);
    // the staged range is PIXEL-major, [position][C] (a copy of the NHWC pixels): consecutive cp.async lanes write consecutive
    // shared addresses, and the stencil's lanes -- channel group fastest -- read consecutive 16-byte pieces
    const int pix = a.C * 2;
    unsigned char *sS = smem;
    unsigned char *sA = smem + (size_t)a.Rmax * pix;
    const uint32_t lbo_a = tc_dw_lbo_a(a.rows);
    unsigned char *sB = sA + (size_t)(a.Kpad / 8) * lbo_a;
    float *s_dww = reinterpret_cast<float *>(sB + (size_t)a.Kpad * a.N * 2);  // [tap][C] FP16-rounded depthwise weights as FP32
    float *s_dwb = s_dww + 9 * a.C;                                             // [C] depthwise bias
    int *s_off = reinterpret_cast<int *>(s_dwb + a.C);                          // staged position -> element offset, -1 = padding
    const int M = a.nimg * a.OH * a.OW;
    const int m0 = blockIdx.x * a.rows;
    const int mlast = min(m0 + a.rows, M) - 1;
    auto centre = [&](int m) -> int {
        const int q = fast_div(m, a.mul_OW), ox = m - q * a.OW, b = fast_div(q, a.mul_OH), oy = q - b * a.OH;
        return (b * a.Hp + oy * a.S) * a.Wp + ox * a.S + 1;
    };
    const int lo = centre(m0) - a.Wp - 1;
    const int R = (int)(centre(mlast) + a.Wp + 1 - lo) + 1;
    if (R > a.Rmax) __trap();            // host-side geometry (plan_fp.cu dw_geometry) must bound every tile

    if (tid == 0) {
        tc::mbar_init(&bar_b, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const unsigned bytes = (unsigned)((size_t)a.Kpad * a.N * 2);
        tc::mbar_expect_tx(&bar_b, bytes);
        tc::bulk_g2s(sB, a.wimg + (size_t)blockIdx.y * a.Kpad * a.N, bytes, &bar_b);
    }
    pdl_trigger();
    if (tid < a.N) s_bias[tid] = a.bias[blockIdx.y * a.N + tid];
    for (int i = tid; i < 9 * a.C; i += TC_THREADS) s_dww[i] = dw_weight_f16(a.dw_w[i]);
    for (int i = tid; i < a.C; i += TC_THREADS) s_dwb[i] = a.dw_b[i];
    {
        const int lane = tid & 31;
        const int prow0 = fast_floor_div(lo, a.Wp, a.mul_Wp);          // floor
        const int prow1 = fast_div(lo + R - 1, a.mul_Wp);
        for (int prow = prow0 + warp; prow <= prow1; prow += TC_THREADS / 32) {
            const int b = prow >= 0 ? fast_div(prow, a.mul_Hp) : -1;
            const int yy = prow >= 0 ? (int)(prow - b * a.Hp) : 0;
            const bool rowok = prow >= 0 && b < a.nimg && yy < a.IH;
            for (int xx = lane; xx < a.Wp; xx += 32) {
                const int pl = prow * a.Wp + xx - lo;
                if (pl < 0 || pl >= R) continue;
                s_off[pl] = (rowok && xx >= 1 && xx <= a.IW) ? ((b * a.IH + yy) * a.IW + (xx - 1)) * a.C : -1;
            }
        }
    }
    if (tid < 128) {
        const int m = m0 + tid;
        s_cpos[tid] = (tid < a.rows && m < M) ? (int)(centre(m) - lo) : -1;
    }
    __syncthreads();
    pdl_wait();
    const int lg = 31 - __clz(G);        // C / 8 is a power of two
    {
        // TC_THREADS is a multiple of G: a thread keeps its channel group; item `it` lands at sS + it * 16
        const uint32_t sS_s = tc::smem_u32(sS);
        const __half *src_g = a.in + (tid & (G - 1)) * 8;
        for (int it = tid; it < R * G; it += TC_THREADS) {
            const int off = s_off[it >> lg];
            cp_async16_zfill_s(sS_s + (uint32_t)it * 16u, off >= 0 ? src_g + off : a.in, off >= 0);
        }
    }
    cp_async_wait_all();
    __syncthreads();
    // ---- depthwise stencil from shared memory -> A operand (canonical K-major layout) -------------------
    // Each thread owns ONE 8-channel group (TC_THREADS % GA == 0) and walks the tile's rows four at a time.  Four consecutive
    // outputs of one output row have their stencil centres S staged positions apart and share window columns: 3 x (3S + 3)
    // loads and conversions for 36 taps.  A quad that crosses the end of an output row, of an image or of M takes its rows
    // one by one (within an output row the centres step by exactly S, across one by more).
    if (g_own < G) {
        auto stencil = [&](auto s_) {
            constexpr int S = decltype(s_)::value;
            const float *w = s_dww + g_own * 8;
            const int win = g_own * 16 - (a.Wp + 1) * pix;     // sS + win + centre * pix: window pixel (0, 0)
            for (int r0 = 4 * (tid >> lgGA); r0 < a.rows; r0 += 4 * (TC_THREADS >> lgGA)) {
                const int cp0 = s_cpos[r0];
                if (cp0 < 0) continue;       // rows beyond M (last tile): never read back
                unsigned char *dst = sA + (size_t)g_own * lbo_a + (size_t)r0 * 16;
                if (s_cpos[r0 + 3] == cp0 + 3 * S) {
                    float acc[1][4][8];
                    dw_bias8(acc[0][0], s_dwb + g_own * 8);
#pragma unroll
                    for (int i = 0; i < 8; i++) { acc[0][1][i] = acc[0][0][i]; acc[0][2][i] = acc[0][0][i]; acc[0][3][i] = acc[0][0][i]; }
                    dw_stencil_block<S, 1, 4>(acc, sS + win + cp0 * pix, a.Wp * pix, pix, w, a.C);
#pragma unroll
                    for (int q = 0; q < 4; q++) *reinterpret_cast<uint4 *>(dst + q * 16) = dw_relu_h8(acc[0][q]);
                } else {
                    for (int q = 0; q < 4; q++) {
                        const int cp = s_cpos[r0 + q];
                        if (cp < 0) continue;
                        float acc[1][1][8];
                        dw_bias8(acc[0][0], s_dwb + g_own * 8);
                        dw_stencil_block<S, 1, 1>(acc, sS + win + cp * pix, a.Wp * pix, pix, w, a.C);
                        *reinterpret_cast<uint4 *>(dst + q * 16) = dw_relu_h8(acc[0][0]);
                    }
                }
            }
        };
        if (a.S == 1) stencil(std::integral_constant<int, 1>{});
        else stencil(std::integral_constant<int, 2>{});
    } else {                                  // K padding group of the Cin = 8 layer: zeros
        for (int r = tid >> lgGA; r < a.rows; r += TC_THREADS >> lgGA)
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
    const TcOut o{a.out, a.Ntotal, a.Ntotal, 1, nullptr, 0, 0};
    wg::for_chunks<(NT < 64 ? NT : 64)>(a.N, [&](auto nc, int n0) {
        constexpr int NC = decltype(nc)::value;
        float d[NC / 2];                 // not zeroed: the first MMA runs with scale-d = 0 (see wg::fence)
        wg::fence();
        wg::mma_ss<NC>(d, wg::desc(a_addr, lbo_a, 128), wg::desc(b_addr + (uint32_t)n0 * 16u, lbo_b, 128), 0);
        for (int ks = 1; ks < (a.Kpad >> 4); ks++) {
            const uint64_t ad = wg::desc(a_addr + (uint32_t)(2 * ks) * lbo_a, lbo_a, 128);
            const uint64_t bd = wg::desc(b_addr + (uint32_t)(2 * ks) * lbo_b + (uint32_t)n0 * 16u, lbo_b, 128);
            wg::mma_ss<NC>(d, ad, bd, 1);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs(d);
        tc_epilogue<NC>(d, n0, s_bias, o, orow, (int)blockIdx.y * a.N);
    });
}

}  // namespace rf
