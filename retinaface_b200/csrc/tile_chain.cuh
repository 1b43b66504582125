// tile_chain.cuh -- persistent, warp-specialised wgmma "tile chain" kernel of librf_b200 (FP16 operands, FP32 accumulate).
// sm_90a: cp.async.bulk.tensor (TMA tensor maps), wgmma.mma_async (A from shared memory or registers), mbarrier hand-offs,
// griddepcontrol.
//
// One CTA owns a tile = TH full-width rows of one image and runs a CHAIN of layers on it without leaving the SM:
// every intermediate activation stays in shared memory, only the tensors other kernels need are written
// back, by TMA stores.  Layers the reference's graph (model/mnet-deconv-0517.prototxt) runs one by one inside TensorRT
// (retinaface/tensorrt/trtretinafacenet.cpp:60) become STAGES of one launch:
//   TCH_CONV : 1x1 or 3x3 (pad 1) convolution + BN (+ ReLU)                                (rf_c*_aggr, SSH convs)
//   TCH_HEAD : the three predictor 1x1 convs of a level as ONE N = 32 GEMM (FP32-grade: hi + lo FP16 weight pieces) whose
//              epilogue is the post-process: 2-way softmax, threshold, anchor decode, clip, candidate append
//              (RetinaFace.cpp:666-723) -- and, in the last CTA that finishes an image, sort + greedy NMS (:434-492).
//   (pre-stage) FPN merge: lateral + crop(deconv_k4s2p1(coarser level)) (prototxt:1553-1592, :1948-1987) into the input tile.
//
// Geometry.  Local position space of a tile: width Wl = W + 2 (one zero column either side), rows = tile rows plus the
// halo the chain needs; position p = ly * Wl + lx.  In this space a 3x3 tap is the constant shift dy * Wl + dx, so the A
// operand of every tap is the SAME shared-memory buffer with the descriptor start address moved by shift * ROW bytes (the
// swizzle is anchored on absolute address bits of the 1024-aligned buffers, so the descriptor's base offset stays 0).  A
// stage computes whole local rows, 128 consecutive positions per MMA tile (two 64-row wgmma blocks); positions outside
// the image are written as zeros (they are the next stage's padding).  Halo rows are recomputed per tile.
//
// Data movement.  Activations enter by TMA tiled loads (4-D NHWC tensor map, box {<=64 channels, Wl, rows}, out-of-bounds
// fill = the zero padding) in SWIZZLE_128B / 64B / 32B mode (64 / 32 / 16 channels per row), which is exactly the wgmma
// K-major swizzled operand layout.  Epilogue threads write stage outputs into shared memory in the same swizzled layout.
//
// Roles (288 threads): warps 0-3 / 4-7 = two compute warpgroups that take the MMA tiles of a stage in turn, each issuing
// its own MMAs and running the epilogue from its accumulators; warp 8 = TMA producer (tiles, per-stage weights, TMA
// stores).  All hand-offs between the producer and the warpgroups are mbarriers; the CTA loops over tiles (persistent).
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "postproc_dev.cuh"
#include "tc_conv.cuh"
#include "wgmma.cuh"

namespace rf {

constexpr int TCH_THREADS = 288;
constexpr int TCH_MAX_STAGES = 8;
constexpr int TCH_MAX_BUFS = 8;
constexpr int TCH_EPI_THREADS = 256;
enum { TCH_CONV = 0, TCH_HEAD = 1 };

struct TchBuf {
    int off;            // byte offset in dynamic shared memory (1024-aligned); position index 0 lives here
    int row;            // bytes per position per slab: 32 | 64 | 128 (16 | 32 | >= 64 channels)
    int slabs;          // 64-channel slabs (1 unless channels >= 128)
    int slab_stride;    // bytes between slabs
    int rows_lo;        // local row held at position index `slack`
    int nrows;          // rows held
    int slack;          // positions in front of row rows_lo (>= 1: the (-1, -1) tap of the first computed position reads one back)
};

struct TchStage {
    int type;
    int Cin, N;               // input / output channels
    int taps;                 // CONV: 1 | 9;  HEAD: 1
    int in_buf;
    int rows_lo, nrows;       // local rows this stage computes
    int wp_off, wp_bytes;     // B image [K/8][N][8] (HEAD: hi image then lo image)
    int wp_smem;              // resident weights: this stage's own region in shared memory
    int bias_pw;              // float offset into the bias arena
    int store_buf, store_map; // -1 | buffer whose owned rows [HT, HT + TH) are TMA-stored once the stage is complete
    unsigned char ob_buf[16], ob_c16[16], ob_relu[16];   // per 16-column output block: buffer, channel offset / 16, ReLU
};

struct TchHead {              // TCH_HEAD epilogue + last-block NMS
    LevelDesc lv;
    PostBuffers pb;
    const PostParams *params;
    int net_w, net_h;
    int *done;                // [max_batch] tiles finished per image (all levels); the last one runs the NMS
    int expected;             // tiles per image over all levels; 0: no fused NMS
    int nms_smem;             // byte offset of the NMS scratch in dynamic shared memory (never a TMA-stored buffer)
    float *blobs[3];          // rf_forward_heads: cls_prob / bbox_pred / landmark_pred of this level (NCHW f32) or NULL
};

struct TchArgs {
    int nstages, nbufs;
    TchStage st[TCH_MAX_STAGES];
    TchBuf buf[TCH_MAX_BUFS];
    int Wl, HT, TH;
    int W, H, nimg, tiles_per_img, ntiles;
    int wp_smem, bias_smem, smem_bytes;              // byte offsets in dynamic shared memory / total
    int resident;             // 1: the weights of ALL stages stay in shared memory for the CTA's lifetime (loaded once, before
                              // griddepcontrol.wait); 0: streamed per stage through the wp buffer
    unsigned *dbg;            // host-mapped word: code of the hand-off a timed-out wait was stuck on (0: none)
    unsigned long long *trace;   // -DRF_TCH_TRACE builds: timeline of CTA 0 (count, then (code, ns) pairs)
    const unsigned char *warena;
    const float *bias;
    int bias_floats;
    int in_C;
    unsigned in_bytes;
    // FPN merge pre-stage (merge_C > 0): buffer 0 += crop(deconv(coarse)); coarse tile in buffer `merge_buf`
    int merge_C, merge_buf, merge_rows, merge_w_bias;   // merge_w_bias: float offset of the [16 taps][C] FP16 weights in the bias arena
    unsigned merge_bytes;
    TchHead head;
};

struct TchMaps {
    CUtensorMap in;           // chain input
    CUtensorMap aux;          // FPN merge: the coarser level
    CUtensorMap st[3];        // TMA stores
};

namespace tch {

__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *map, uint64_t *bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(map), "r"(tc::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *map, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
// mbarrier wait that reports WHICH hand-off was lost before trapping (code -> host-mapped debug word): a lost arrive must
// fail loudly and say where, never hang the GPU
__device__ __forceinline__ void wait(uint64_t *bar, unsigned parity, unsigned *dbg, unsigned code) {
    unsigned done = 0, spins = 0;
    while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(tc::smem_u32(bar)), "r"(parity)
            : "memory");
        if (!done && ++spins > (1u << 22)) {
            if (dbg) { *reinterpret_cast<volatile unsigned *>(dbg) = code | (blockIdx.x << 20); __threadfence_system(); __nanosleep(2000000); }
            __trap();
        }
    }
}
// the same for a whole warp: lanes may leave the polling loop in different iterations; the warpgroup-collective
// (.sync.aligned) wgmma instructions that follow need it converged again
__device__ __forceinline__ void wait_warp(uint64_t *bar, unsigned parity, unsigned *dbg, unsigned code) {
    wait(bar, parity, dbg, code);
    __syncwarp();
}
// Optional timeline of CTA 0 (build with -DRF_TCH_TRACE; launch_chain prints the last launch's events of each chain to stderr):
// (event code, globaltimer ns) pairs
#ifdef RF_TCH_TRACE
__device__ __forceinline__ void trace(unsigned long long *t, unsigned code) {
    if (t && blockIdx.x == 0) {
        unsigned long long now;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        const unsigned i = atomicAdd(reinterpret_cast<unsigned *>(t), 1u);
        if (i < 500) { t[1 + 2 * i] = code; t[2 + 2 * i] = now; }
    }
}
#define TCH_TRACE(code) tch::trace(a.trace, (code))
#else
#define TCH_TRACE(code)
#endif
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void prefetch_map(const CUtensorMap *map) { asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(tc::smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_g2s_u32(uint32_t dst, const void *src, unsigned bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes),
                 "r"(tc::smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void epi_bar() { asm volatile("bar.sync 1, %0;" ::"n"(TCH_EPI_THREADS) : "memory"); }
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
// byte offset of 16-byte chunk j of position p inside a buffer (swizzle on address bits [4,7) ^ [7,10), buffers are 1024-aligned)
__device__ __forceinline__ uint32_t chunk_off(int row, int p, int j) {
    const int sh = row == 128 ? 0 : (row == 64 ? 1 : 2), m = (row >> 4) - 1;
    return (uint32_t)p * row + (uint32_t)((j ^ ((p >> sh) & m)) << 4);
}

// ---- compute warpgroups: one 64-row block of a stage (rows = stage positions q0 .. q0 + 63) ---------------------------------
// Shared-memory offsets are bytes.  K step k of an input buffer with kpr = row / 32 steps per row: slab k >> lkpr, 32 bytes
// per step inside the row.
__device__ __forceinline__ uint32_t k_off(int k, int lkpr, int kpr, uint32_t slab) {
    return (uint32_t)(k >> lkpr) * slab + (uint32_t)(k & (kpr - 1)) * 32u;
}
struct BlkGeo {
    uint32_t abase;           // A operand: position q0 of the stage, tap (0, 0), K step 0
    uint32_t row, slab;       // input buffer: bytes per position per slab, bytes between slabs
    int lkpr, kpr;
    uint32_t wp;              // weight image
    int q0, npos, Y0;
};

// stage output of one accumulator chunk (columns [n0, n0 + NC)) -> destination buffers in the swizzled operand layout;
// positions outside the image are written as zeros (the next stage's padding)
template <int NC>
__device__ __forceinline__ void store_chunk(const float (&d)[NC / 2], int n0, const TchArgs &a, const TchStage &st, unsigned char *smem,
                                            const float *bp, const BlkGeo &k) {
    const int lane = threadIdx.x & 31, t4 = lane & 3;
    const int rl = 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);
#pragma unroll
    for (int e = 0; e < 2; e++) {
        const int q = k.q0 + rl + 8 * e;
        if (q >= k.npos) continue;
        const int qy = q / a.Wl;
        const int ly = st.rows_lo + qy, lx = q - qy * a.Wl;
        const int gy = k.Y0 + ly, gx = lx - 1;
        const bool inimg = gx >= 0 && gx < a.W && gy >= 0 && gy < a.H;
#pragma unroll
        for (int jj = 0; jj < NC / 16; jj++) {
            const int jb = (n0 >> 4) + jj;
            const TchBuf &BO = a.buf[st.ob_buf[jb]];
            const int prow = ly - BO.rows_lo;
            if (prow < 0 || prow >= BO.nrows) continue;
            const bool relu = st.ob_relu[jb] != 0;
            const int p = BO.slack + prow * a.Wl + lx;
            const int c16 = st.ob_c16[jb];
            unsigned char *base = smem + BO.off + (c16 >> 2) * BO.slab_stride;
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int i = 2 * jj + h;
                const float2 bb = *reinterpret_cast<const float2 *>(bp + jb * 16 + 8 * h + 2 * t4);
                float f0 = d[4 * i + 2 * e] + bb.x, f1 = d[4 * i + 2 * e + 1] + bb.y;
                if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
                *reinterpret_cast<uint32_t *>(base + chunk_off(BO.row, p, (c16 & 3) * 2 + h) + 4 * t4) = inimg ? pack_h2(f0, f1) : 0u;
            }
        }
    }
}

// convolution / predictors: columns [n0, n0 + NC) of taps x K steps x weight pieces into one accumulator
template <int NC>
__device__ __forceinline__ void conv_chunk(float (&d)[NC / 2], int n0, const TchStage &st, const uint32_t (&tapb)[9], const BlkGeo &k, int pieces) {
#pragma unroll
    for (int i = 0; i < NC / 2; i++) d[i] = 0.f;
    const int nk = st.Cin >> 4;
    const uint32_t lbo = (uint32_t)st.N * 16, kb = 2u * lbo, tap_bytes = (uint32_t)st.Cin * st.N * 2, piece_bytes = (uint32_t)st.taps * tap_bytes;
    wg::fence();
    int acc = 0;
    for (int t = 0; t < st.taps; t++)
        for (int kk = 0; kk < nk; kk++) {
            const uint64_t ad = wg::desc_sw(k.abase + (st.taps == 9 ? tapb[t] : 0u) + k_off(kk, k.lkpr, k.kpr, k.slab), k.row);
            for (int pc = 0; pc < pieces; pc++) {
                wg::mma_ss<NC>(d, ad, wg::desc(k.wp + (uint32_t)pc * piece_bytes + (uint32_t)t * tap_bytes + (uint32_t)kk * kb + (uint32_t)n0 * 16u, lbo, 128), acc);
                acc = 1;
            }
        }
    wg::commit();
    wg::wait<0>();
    wg::fence_regs(d);
}

}  // namespace tch

template <int UNUSED>
__global__ void __launch_bounds__(TCH_THREADS, 1) k_tile_chain(const __grid_constant__ TchMaps maps, const __grid_constant__ TchArgs a) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t bar_in, bar_bias, bar_stage, bar_tile, bar_wp_full;
    __shared__ int s_last;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t sbase = (tc::smem_u32(smem_raw) + 1023u) & ~1023u;
    unsigned char *const smem = smem_raw + (sbase - tc::smem_u32(smem_raw));
    const int Wl = a.Wl;

    if (tid == 0) {
        tc::mbar_init(&bar_in, 1); tc::mbar_init(&bar_bias, 1); tc::mbar_init(&bar_stage, 8); tc::mbar_init(&bar_tile, 8);
        tc::mbar_init(&bar_wp_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_trigger();
    __syncthreads();
    if (tid == 0) TCH_TRACE(1);

    if (warp == 8) {
        // =========================================== TMA producer ===========================================
        if (lane == 0) {
            const unsigned bias_bytes = (unsigned)a.bias_floats * 4u;
            unsigned const_bytes = bias_bytes;
            if (a.resident) for (int s = 0; s < a.nstages; s++) const_bytes += (unsigned)a.st[s].wp_bytes;
            tc::mbar_expect_tx(&bar_bias, const_bytes);
            tch::bulk_g2s_u32(sbase + a.bias_smem, a.bias, bias_bytes, &bar_bias);       // constants: independent of earlier kernels
            if (a.resident)
                for (int s = 0; s < a.nstages; s++)
                    tch::bulk_g2s_u32(sbase + a.st[s].wp_smem, a.warena + a.st[s].wp_off, (unsigned)a.st[s].wp_bytes, &bar_bias);
            tch::prefetch_map(&maps.in);
            pdl_wait();                                                                   // activations of earlier kernels from here on
            unsigned sc = 0;
            const TchBuf &B0 = a.buf[0];
            // owned rows of a finished buffer -> global, one box {<= 64 channels, W, 1} per row and slab starting at image column 0
            // (TMA stores reject negative coordinates, so the zero column at lx = 0 stays behind)
            auto store_rows = [&](const TchBuf &BS, int map, int ty, int b) {
                for (int rr = 0; rr < a.TH; rr++) {
                    const int y = ty * a.TH + rr;
                    if (y >= a.H) break;
                    for (int k = 0; k < BS.slabs; k++)
                        tch::tma_store_4d(&maps.st[map], sbase + BS.off + k * BS.slab_stride + (BS.slack + (a.HT - BS.rows_lo + rr) * Wl + 1) * BS.row, k * 64, 0, y, b);
                }
                tch::bulk_commit();
            };
            for (int tile = blockIdx.x, it = 0; tile < a.ntiles; tile += gridDim.x, it++) {
                const int b = tile / a.tiles_per_img, ty = tile - b * a.tiles_per_img;
                const int Y0 = ty * a.TH - a.HT;                 // image row of local row 0; image column of local column 0 is -1
                if (it > 0) { tch::wait(&bar_tile, (it - 1) & 1, a.dbg, __LINE__); tch::bulk_wait_read0(); }   // buffers free, stores have read them
                tc::mbar_expect_tx(&bar_in, a.in_bytes + a.merge_bytes);
                const int in_slabs = (a.in_C + 63) >> 6;
                for (int s = 0; s < in_slabs; s++)
                    tch::tma_load_4d(sbase + B0.off + s * B0.slab_stride + B0.slack * B0.row, &maps.in, &bar_in, s * 64, -1, Y0 + B0.rows_lo, b);
                if (a.merge_C) {
                    const TchBuf &BM = a.buf[a.merge_buf];
                    // coarse rows ((Y0 + rows_lo + 1) >> 1) - 1 ..., coarse columns -1 .. W/2
                    const int cy0 = ((Y0 + B0.rows_lo + 1) >> 1) - 1;
                    tch::tma_load_4d(sbase + BM.off, &maps.aux, &bar_in, 0, -1, cy0, b);
                }
                for (int s = 0; s < a.nstages; s++, sc++) {
                    const TchStage &st = a.st[s];
                    // every phase of bar_stage is observed in order; stage s-1 is complete -> its TMA store, and (streamed
                    // weights) the single weight buffer is free for stage s
                    if (s > 0) {
                        tch::wait(&bar_stage, (sc - 1) & 1, a.dbg, __LINE__);
                        const TchStage &sp = a.st[s - 1];
                        if (sp.store_buf >= 0) store_rows(a.buf[sp.store_buf], sp.store_map, ty, b);
                    }
                    if (!a.resident) {
                        tc::mbar_expect_tx(&bar_wp_full, (unsigned)st.wp_bytes);
                        tch::bulk_g2s_u32(sbase + a.wp_smem, a.warena + st.wp_off, (unsigned)st.wp_bytes, &bar_wp_full);
                    }
                }
                tch::wait(&bar_stage, (sc - 1) & 1, a.dbg, __LINE__);
                {
                    const TchStage &sp = a.st[a.nstages - 1];
                    if (sp.store_buf >= 0) store_rows(a.buf[sp.store_buf], sp.store_map, ty, b);
                }
            }
            tch::bulk_wait0();       // global writes of the last stores are complete before the CTA exits
        }
    } else {
        // =========================================== compute warpgroups =====================================
        const int wgi = warp >> 2, t4 = lane & 3;
        const int rl = 16 * (warp & 3) + (lane >> 2);           // fragment rows rl, rl + 8 of a 64-row block (wgmma.cuh)
        const int etid = tid;                                   // 0..255 over both warpgroups
        const float *s_bias = reinterpret_cast<const float *>(smem + a.bias_smem);
        tch::wait_warp(&bar_bias, 0, a.dbg, __LINE__);
        pdl_wait();
        unsigned g = 0, sc = 0, wpc = 0;
        for (int tile = blockIdx.x, it = 0; tile < a.ntiles; tile += gridDim.x, it++) {
            const int b = tile / a.tiles_per_img, ty = tile - b * a.tiles_per_img;
            const int Y0 = ty * a.TH - a.HT;
            tch::wait_warp(&bar_in, it & 1, a.dbg, __LINE__);
            if (lane == 0) TCH_TRACE(3);
            if (a.merge_C) {
                // ---- FPN merge: buffer 0 (lateral) += crop(deconv_k4s2p1(coarse)) at in-image positions; packed HFMA2, the
                //      sum of <= 5 terms is stored as FP16 anyway (same operation order as k_fpn_merge_h2)
                const TchBuf &B0 = a.buf[0], &BM = a.buf[a.merge_buf];
                const int UH = a.H >> 1, UW = a.W >> 1, CW = UW + 2;
                const int cy0 = ((Y0 + B0.rows_lo + 1) >> 1) - 1;
                const __half *uw = reinterpret_cast<const __half *>(s_bias + a.merge_w_bias);     // [16 taps][64]
                const int items = B0.nrows * Wl * 8;
                for (int i = etid; i < items; i += TCH_EPI_THREADS) {
                    const int j = i & 7, p = i >> 3;
                    const int ly = p / Wl, lx = p - ly * Wl;
                    const int y = Y0 + B0.rows_lo + ly, x = lx - 1;
                    if (x < 0 || x >= a.W || y < 0 || y >= a.H) continue;
                    unsigned char *slot = smem + B0.off + tch::chunk_off(128, B0.slack + p, j);
                    uint4 accv = *reinterpret_cast<const uint4 *>(slot);
                    __half2 *acc = reinterpret_cast<__half2 *>(&accv);
                    const int i_hi = (y + 1) >> 1, j_hi = (x + 1) >> 1;
#pragma unroll
                    for (int di = 0; di < 2; di++) {
                        const int ci = i_hi - di, ky = y - 2 * ci + 1;
                        if (ci < 0 || ci >= UH) continue;
#pragma unroll
                        for (int dj = 0; dj < 2; dj++) {
                            const int cj = j_hi - dj, kx = x - 2 * cj + 1;
                            if (cj < 0 || cj >= UW) continue;
                            const int cp = (ci - cy0) * CW + (cj + 1);
                            const uint4 uv = *reinterpret_cast<const uint4 *>(smem + BM.off + tch::chunk_off(128, cp, j));
                            const uint4 wv = *reinterpret_cast<const uint4 *>(uw + (ky * 4 + kx) * 64 + j * 8);
                            const __half2 *u2 = reinterpret_cast<const __half2 *>(&uv), *w2 = reinterpret_cast<const __half2 *>(&wv);
#pragma unroll
                            for (int c = 0; c < 4; c++) acc[c] = __hfma2(u2[c], w2[c], acc[c]);
                        }
                    }
                    *reinterpret_cast<uint4 *>(slot) = accv;
                }
                tc::fence_async_smem();
                tch::epi_bar();
            }
            for (int s = 0; s < a.nstages; s++, sc++) {
                const TchStage &st = a.st[s];
                const TchBuf &BI = a.buf[st.in_buf];
                if (sc > 0) tch::wait_warp(&bar_stage, (sc - 1) & 1, a.dbg, __LINE__);      // inputs of this stage are in shared memory
                if (!a.resident) { tch::wait_warp(&bar_wp_full, wpc & 1, a.dbg, __LINE__); wpc++; }
                if (lane == 0) TCH_TRACE(100 + s);
                const int npos = st.nrows * Wl, ntile = (npos + 127) >> 7;
                const int kpr = BI.row >> 5;                             // 16-channel K steps per row: 1 | 2 | 4
                // position index (in the input buffer) of this stage's position 0
                const int pos0 = BI.slack + (st.rows_lo - BI.rows_lo) * Wl;
                tch::BlkGeo k;
                k.row = (uint32_t)BI.row; k.slab = (uint32_t)BI.slab_stride;
                k.kpr = kpr; k.lkpr = kpr == 4 ? 2 : (kpr == 2 ? 1 : 0);
                k.wp = sbase + (a.resident ? st.wp_smem : a.wp_smem);
                k.npos = npos; k.Y0 = Y0;
                // per tap: operand shift, bytes
                uint32_t tapb[9];
#pragma unroll
                for (int t = 0; t < 9; t++) tapb[t] = (uint32_t)(((t / 3 - 1) * Wl + t % 3 - 1) * BI.row);
                const float *bp = s_bias + st.bias_pw;
                for (int m = 0; m < ntile; m++) {
                    if ((int)((g + m) & 1) != wgi) continue;             // the warpgroups take the MMA tiles in turn
                    for (int hb = 0; hb < 2; hb++) {
                        k.q0 = m * 128 + hb * 64;
                        if (k.q0 >= npos) break;
                        k.abase = sbase + BI.off + (uint32_t)(pos0 + k.q0) * (uint32_t)BI.row;
                        if (st.type == TCH_CONV) {
                            wg::for_chunks<64>(st.N, [&](auto nc, int n0) {
                                constexpr int NC = decltype(nc)::value;
                                float d[NC / 2];
                                tch::conv_chunk<NC>(d, n0, st, tapb, k, 1);
                                tch::store_chunk<NC>(d, n0, a, st, smem, bp, k);
                            });
                        } else {
                            // ---- predictor GEMM (N = 32, hi + lo pieces) -> softmax, threshold, decode, candidate append
                            float d[16];
                            tch::conv_chunk<32>(d, 0, st, tapb, k, 2);
                            // the 32 columns of row rl + 8 * (t4 & 1) -> threads t4 = 0, 1 of the quad
                            float hv[32];
#pragma unroll
                            for (int sl = 0; sl < 4; sl++)
#pragma unroll
                                for (int j = 0; j < 16; j++) {
                                    const float v = __shfl_sync(0xffffffffu, d[j], (lane & ~3) | sl);
                                    if (((j >> 1) & 1) == (t4 & 1)) hv[8 * (j >> 2) + 2 * sl + (j & 1)] = v;
                                }
                            const TchHead &hd = a.head;
                            const int q = k.q0 + rl + 8 * (t4 & 1);
                            const bool valid = t4 < 2 && q < npos;
                            const int qy = q / Wl;
                            const int ly = st.rows_lo + qy, lx = q - qy * Wl;
                            const int gy = Y0 + ly, gx = lx - 1;
                            const bool inimg = valid && gx >= 0 && gx < a.W && gy >= 0 && gy < a.H;
                            const bool owned = inimg && ly >= a.HT && ly < a.HT + a.TH;
                            float sc4[4], pf[2], pbg[2];
#pragma unroll
                            for (int i = 0; i < 4; i++) sc4[i] = __fadd_rn(hv[i], bp[i]);
#pragma unroll
                            for (int an = 0; an < 2; an++) softmax_pair(sc4[an], sc4[an + 2], pbg[an], pf[an]);
                            const float thr = hd.params->score_thr;
                            const bool wb = hd.blobs[0] != nullptr;
                            const bool pass0 = owned && !(pf[0] <= thr), pass1 = owned && !(pf[1] <= thr);
                            const bool need = __any_sync(0xffffffffu, pass0 || pass1 || (wb && owned));
                            if (need) {
                                const int hw = hd.lv.h * hd.lv.w, jpix = gy * hd.lv.w + gx;
                                float reg[8], lm[20];
#pragma unroll
                                for (int i = 0; i < 8; i++) reg[i] = __fadd_rn(hv[4 + i], bp[4 + i]);
#pragma unroll
                                for (int i = 0; i < 20; i++) lm[i] = __fadd_rn(hv[12 + i], bp[12 + i]);
                                if (wb && owned) {
                                    float *cls = hd.blobs[0] + (size_t)b * 4 * hw, *bb = hd.blobs[1] + (size_t)b * 8 * hw, *lb = hd.blobs[2] + (size_t)b * 20 * hw;
                                    cls[0 * hw + jpix] = pbg[0]; cls[1 * hw + jpix] = pbg[1]; cls[2 * hw + jpix] = pf[0]; cls[3 * hw + jpix] = pf[1];
#pragma unroll
                                    for (int i = 0; i < 8; i++) bb[i * hw + jpix] = reg[i];
#pragma unroll
                                    for (int i = 0; i < 20; i++) lb[i * hw + jpix] = lm[i];
                                }
#pragma unroll
                                for (int an = 0; an < 2; an++) {
                                    if (!(an ? pass1 : pass0)) continue;
                                    rf_det det;
                                    decode_one(pf[an], reg + 4 * an, lm + 10 * an, hd.lv, an, gy, gx, hd.net_w, hd.net_h, hd.lv.anchor_base + an * hw + jpix, det);
                                    append_candidate(hd.pb, b, det);
                                }
                            }
                        }
                    }
                }
                g += ntile;
                if (lane == 0) TCH_TRACE(200 + s);
                tc::fence_async_smem();          // this stage's shared-memory writes -> visible to wgmma / TMA (async proxy)
                __syncwarp();
                if (lane == 0) tch::mbar_arrive(&bar_stage);
            }
            if (a.head.expected > 0) {
                // ---- last-block NMS: the CTA that completes an image's last tile (over all three levels) sorts and suppresses it
                __threadfence();
                tch::epi_bar();
                if (etid == 0) s_last = atomicAdd(&a.head.done[b], 1) == a.head.expected - 1;
                tch::epi_bar();
                if (s_last) {
                    __threadfence();
                    NmsSmem &S = *reinterpret_cast<NmsSmem *>(smem + a.head.nms_smem);
                    int *s_kept = reinterpret_cast<int *>(smem + a.head.nms_smem + ((sizeof(NmsSmem) + 15) & ~15));
                    nms_image<TCH_EPI_THREADS, true>(b, etid, a.head.params->nms_thr, a.head.params, a.head.pb, S, s_kept, [] { tch::epi_bar(); });
                    if (etid == 0) a.head.done[b] = 0;           // self-cleaning for the next forward
                }
            }
            __syncwarp();
            if (lane == 0) tch::mbar_arrive(&bar_tile);
        }
    }
    if (tid == 0) TCH_TRACE(9);
}

}  // namespace rf
