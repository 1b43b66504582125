// yuv.cuh -- f6 video frames: 8-bit YUV 4:2:0 (NV12, NV21, I420, YV12) as a pixel source of the letter-box and the face-alignment
// kernels.  Every source tap those kernels read is converted on the fly; no BGR copy of a frame is ever materialised.
//
// Definition (OpenCV's COLOR_YUV2BGR_NV12 / NV21 / I420 / YV12, imgproc color_yuv.simd.hpp): nearest chroma -- each 2x2 luma
// block shares one (U, V) sample -- and 20-bit fixed point,
//   y' = max(Y - 16, 0) * CY, u' = U - 128, v' = V - 128, half = 1 << 19
//   B = clamp((y' + half + CUB u') >> 20), G = clamp((y' + half + CVG v' + CUG u') >> 20), R = clamp((y' + half + CVR v') >> 20)
// BT.601 uses OpenCV's own constants (bit-equal to cv2.cvtColor).  BT.709 (NVDEC's HD output) uses round(c * 2^20) of the
// limited-range BT.709 matrix (Kr = 0.2126, Kb = 0.0722, luma 255/219, chroma 255/224); OpenCV has no BT.709 4:2:0 conversion,
// so this formula is the definition (oracle/yuv.py restates it).  Every intermediate fits in int32.
#pragma once
#include "common.cuh"

namespace rf {

// One frame's planes as the kernels read them: luma sample (x, y) at y[y * y_pitch + x]; the chroma pair of (x, y) at
// u[c], v[c], c = (y / 2) * uv_pitch + (x / 2) * uv_step (uv_step 2: semi-planar, 1: planar).
struct YuvPlanes {
    const uint8_t *y, *u, *v;
    int y_pitch, uv_pitch, uv_step, matrix;   // matrix: RF_YUV_BT601 | RF_YUV_BT709
};

__host__ __device__ __forceinline__ void yuv_to_bgr(int Y, int U, int V, int matrix, int out[3]) {
    const bool bt709 = matrix != 0;
    const int cy = bt709 ? 1220945 : 1220542, cub = bt709 ? 2215014 : 2116026, cug = bt709 ? -223607 : -409993;
    const int cvg = bt709 ? -558796 : -852492, cvr = bt709 ? 1879825 : 1673527;
    const int y = (Y > 16 ? Y - 16 : 0) * cy + (1 << 19), u = U - 128, v = V - 128;
    const int b = (y + cub * u) >> 20, g = (y + cvg * v + cug * u) >> 20, r = (y + cvr * v) >> 20;
    out[0] = b < 0 ? 0 : b > 255 ? 255 : b;
    out[1] = g < 0 ? 0 : g > 255 ? 255 : g;
    out[2] = r < 0 ? 0 : r > 255 ? 255 : r;
}

// BGR of frame pixel (x, y) (inside the frame)
__device__ __forceinline__ void yuv_pixel(const YuvPlanes &p, int x, int y, int out[3]) {
    const int Y = p.y[(size_t)y * p.y_pitch + x];
    const size_t c = (size_t)(y >> 1) * p.uv_pitch + (size_t)(x >> 1) * p.uv_step;
    yuv_to_bgr(Y, p.u[c], p.v[c], p.matrix, out);
}

// f20: the stored address of a displayed plane sample.  A plane whose stored sample (c, r) lies at r * pitch + c * step, shown in
// orientation `bits` (preprocess.cuh's LB_* bits of f9's A_o) as a dw x dh plane, holds displayed sample (x, y) at
// off + x * xs + y * ys: A_o reflects then transposes integer addresses, so the map is affine with strides of +-step and +-pitch.
// Luma uses the displayed frame's size; chroma the halved size (even sides: the 2x2 blocks of the displayed frame are blocks of the
// stored one).  Bits 0 give off 0, xs step, ys pitch: the stored layout.
struct PlaneMap {
    long long off;
    int xs, ys;
};
__host__ __device__ inline PlaneMap plane_map(int bits, int dw, int dh, int pitch, int step) {
    const bool fx = bits & 1, fy = bits & 2, tr = bits & 4;      // LB_FLIP_X, LB_FLIP_Y, LB_TRANSPOSE
    const int a = tr ? pitch : step, b = tr ? step : pitch;      // the strides of the reflected x and y
    return PlaneMap{(fx ? (long long)a * (dw - 1) : 0) + (fy ? (long long)b * (dh - 1) : 0), fx ? -a : a, fy ? -b : b};
}

}  // namespace rf
