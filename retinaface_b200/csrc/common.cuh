// common.cuh -- shared device/host helpers of librf_b200 (sm_90a).
#pragma once
#include <cstdint>
#include <cstdlib>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rf_b200.h"

namespace rf {

// ---- element type helpers (activations are NHWC in T = float or __half) --------------------
template <typename T> struct Vec8;  // 8 consecutive channels
template <> struct Vec8<float> {
    float4 a, b;
    __device__ __forceinline__ void load(const float *p) { a = *reinterpret_cast<const float4 *>(p); b = *reinterpret_cast<const float4 *>(p + 4); }
    __device__ __forceinline__ void store(float *p) const { *reinterpret_cast<float4 *>(p) = a; *reinterpret_cast<float4 *>(p + 4) = b; }
    __device__ __forceinline__ void to_float(float f[8]) const { f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w; }
    __device__ __forceinline__ void from_float(const float f[8]) { a = make_float4(f[0], f[1], f[2], f[3]); b = make_float4(f[4], f[5], f[6], f[7]); }
};
template <> struct Vec8<__half> {
    uint4 v;
    __device__ __forceinline__ void load(const __half *p) { v = *reinterpret_cast<const uint4 *>(p); }
    __device__ __forceinline__ void store(__half *p) const { *reinterpret_cast<uint4 *>(p) = v; }
    __device__ __forceinline__ void to_float(float f[8]) const {
        const __half2 *h = reinterpret_cast<const __half2 *>(&v);
#pragma unroll
        for (int i = 0; i < 4; i++) { float2 t = __half22float2(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
    }
    __device__ __forceinline__ void from_float(const float f[8]) {
        __half2 *h = reinterpret_cast<__half2 *>(&v);
#pragma unroll
        for (int i = 0; i < 4; i++) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
    }
};

// int8 activations (INT8 path): 8 consecutive channels = 8 bytes; to_float yields the raw integer values, the
// caller applies the tensor's scale.
template <> struct Vec8<int8_t> {
    uint2 v;
    __device__ __forceinline__ void load(const int8_t *p) { v = *reinterpret_cast<const uint2 *>(p); }
    __device__ __forceinline__ void to_float(float f[8]) const {
        f[0] = (float)(int8_t)(v.x & 0xff); f[1] = (float)(int8_t)((v.x >> 8) & 0xff); f[2] = (float)(int8_t)((v.x >> 16) & 0xff); f[3] = (float)(int8_t)(v.x >> 24);
        f[4] = (float)(int8_t)(v.y & 0xff); f[5] = (float)(int8_t)((v.y >> 8) & 0xff); f[6] = (float)(int8_t)((v.y >> 16) & 0xff); f[7] = (float)(int8_t)(v.y >> 24);
    }
};

__device__ __forceinline__ float to_f(float x) { return x; }
__device__ __forceinline__ float to_f(__half x) { return __half2float(x); }
template <typename T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ float from_f<float>(float x) { return x; }
template <> __device__ __forceinline__ __half from_f<__half>(float x) { return __float2half_rn(x); }

// ---- division by a launch constant: q = umulhi(n, ceil(2^32 / d)), exact while n * d < 2^32 (n, d >= 1; d == 1: mul = 0 marks
// the identity).  An integer division by a run-time value costs ~25 instructions; the 2-D depthwise kernels did five per thread.
inline uint32_t fast_div_mul(uint32_t d) { return d <= 1 ? 0u : (uint32_t)((((uint64_t)1 << 32) + d - 1) / d); }
__device__ __forceinline__ int fast_div(int n, uint32_t mul) { return mul ? (int)__umulhi((uint32_t)n, mul) : n; }
__device__ __forceinline__ int fast_floor_div(int n, int d, uint32_t mul) { return n >= 0 ? fast_div(n, mul) : -fast_div(-n + d - 1, mul); }

// ---- depthwise 3x3 stencil of the FP16 tensor-core kernels, 8 channels per thread, on an NY x NX block of outputs whose
// windows overlap (output (oy, ox) reads window row S*oy + ky, column S*ox + kx).  Each FP16 activation of the block's window
// is converted to FP32 once and feeds every output that reads it; the weights are FP32 values equal to the FP16-rounded
// depthwise weights (dw_weight_f16), so acc = fmaf(x, w, acc) rounds once, like a fused FP16 x FP16 + FP32 multiply-add.
// Every output starts from its FP32 bias and takes its taps in the order ky, kx ascending, whatever the block shape: the
// results do not depend on NY and NX.
//   base: window pixel (0, 0) of this thread's channel group; row / pix: bytes between window rows / pixels;
//   w: [9 taps][wstride] FP32 weights, at this thread's channel group
__device__ __forceinline__ float dw_weight_f16(float w) { return __half2float(__float2half_rn(w)); }
template <int S, int NY, int NX>
__device__ __forceinline__ void dw_stencil_block(float (&acc)[NY][NX][8], const unsigned char *base, int row, int pix, const float *w, int wstride) {
#pragma unroll 1                     // one window row at a time: unrolled, the loads of every row are hoisted and spill
    for (int ry = 0; ry < S * (NY - 1) + 3; ry++) {
#pragma unroll
        for (int cx = 0; cx < S * (NX - 1) + 3; cx++) {
            const uint4 raw = *reinterpret_cast<const uint4 *>(base + ry * row + cx * pix);
            const __half2 *h = reinterpret_cast<const __half2 *>(&raw);
            float x[8];
#pragma unroll
            for (int i = 0; i < 4; i++) { const float2 t = __half22float2(h[i]); x[2 * i] = t.x; x[2 * i + 1] = t.y; }
#pragma unroll
            for (int oy = 0; oy < NY; oy++) {
#pragma unroll
                for (int ox = 0; ox < NX; ox++) {
                    const int ky = ry - S * oy, kx = cx - S * ox;
                    if (ky < 0 || ky > 2 || kx < 0 || kx > 2) continue;
                    const float4 w0 = *reinterpret_cast<const float4 *>(w + (ky * 3 + kx) * wstride), w1 = *reinterpret_cast<const float4 *>(w + (ky * 3 + kx) * wstride + 4);
                    float *a = acc[oy][ox];
                    a[0] = fmaf(x[0], w0.x, a[0]); a[1] = fmaf(x[1], w0.y, a[1]); a[2] = fmaf(x[2], w0.z, a[2]); a[3] = fmaf(x[3], w0.w, a[3]);
                    a[4] = fmaf(x[4], w1.x, a[4]); a[5] = fmaf(x[5], w1.y, a[5]); a[6] = fmaf(x[6], w1.z, a[6]); a[7] = fmaf(x[7], w1.w, a[7]);
                }
            }
        }
    }
}
// bias in, ReLU and FP16 rounding out (the A operand of the pointwise GEMM)
__device__ __forceinline__ void dw_bias8(float (&acc)[8], const float *b) {
    const float4 b0 = *reinterpret_cast<const float4 *>(b), b1 = *reinterpret_cast<const float4 *>(b + 4);
    acc[0] = b0.x; acc[1] = b0.y; acc[2] = b0.z; acc[3] = b0.w; acc[4] = b1.x; acc[5] = b1.y; acc[6] = b1.z; acc[7] = b1.w;
}
__device__ __forceinline__ uint4 dw_relu_h8(float (&acc)[8]) {
    uint4 v;
    __half2 *h = reinterpret_cast<__half2 *>(&v);
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2half2_rn(fmaxf(acc[2 * i], 0.f), fmaxf(acc[2 * i + 1], 0.f));
    return v;
}

// ---- programmatic dependent launch (PDL) ------------------------------------------------------
// Every kernel of the forward pass is launched with cudaLaunchAttributeProgrammaticStreamSerialization:
// its CTAs may start while the previous kernel drains.  pdl_trigger() lets the NEXT kernel start its
// own prologue (barrier init, weight copies -- nothing that depends on activations);
// pdl_wait() blocks until the PREVIOUS kernel has completed and its global writes are visible, and
// must precede the first read of an activation and the first global write.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// RF_NO_PDL=1 (read once): launch without the attribute -- griddepcontrol.* are then no-ops (A/B measurements)
inline bool pdl_allowed() {
    static const bool on = [] { const char *e = getenv("RF_NO_PDL"); return !(e && e[0] == '1'); }();
    return on;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = pdl_allowed() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

// ---- post-process shared structures -------------------------------------------------------
struct LevelDesc {           // one FPN level of one launch
    int stride, h, w;        // feature map size
    int anchor_base;         // emission index of (num 0, j 0) of this level
    int pix_base;            // first pixel id of this level in the fused per-image pixel range
    float base[8];           // 2 base anchors x (x1,y1,x2,y2)
};
struct PostParams {          // device-resident: a replayed CUDA graph picks up new values without re-capture
    float score_thr;
    float nms_thr;
    const uint8_t *input;    // [n][net_h][net_w][3] u8 BGR images of this run (library buffer or caller's)
    unsigned comm_seq;       // multi-GPU exchange (comm.cu): sequence number of this step (0: no exchange) ...
    unsigned comm_slot;      // ... and its slot in every rank's gather window
};

}  // namespace rf
