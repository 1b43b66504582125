// warp.cuh -- the device pieces of the f5 crop warp, shared by k_align_faces (align.cu) and the f11 best-shot kernels (best.cu):
// the similarity fit, cv::invertAffineTransform, one cv::warpAffine output pixel and the crop store.  Include it only from sources
// built with -fmad=false: OpenCV evaluates iM01 * y + iM02 (and the closed-form sums here mirror oracle/align.py) as a separate
// multiply and add, and a contracted FMA can move a coordinate across a 1/1024 rounding boundary.
#pragma once
#include "align.cuh"

namespace rf {

// Least-squares similarity from the five landmarks p (image pixels) to the template q, centred closed form:
// a = sum(p~ . q~) / sum |p~|^2, b = sum(p~x q~y - p~y q~x) / sum |p~|^2, M = [[a, -b, tx], [b, a, ty]] (the minimiser
// Umeyama's SVD form finds).  Returns false (M = 0) when the landmarks coincide.
__device__ inline bool fit_similarity(const rf_face &f, float scale, const double *q, double M[6]) {
    double px[5], py[5];
    double pmx = 0.0, pmy = 0.0, qmx = 0.0, qmy = 0.0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        px[k] = (double)__fmul_rn(f.lx[k], scale);      // the map-back of k_merge_views
        py[k] = (double)__fmul_rn(f.ly[k], scale);
        pmx += px[k]; pmy += py[k]; qmx += q[2 * k]; qmy += q[2 * k + 1];
    }
    pmx /= 5.0; pmy /= 5.0; qmx /= 5.0; qmy /= 5.0;
    double den = 0.0, sxx = 0.0, sxy = 0.0;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        const double ux = px[k] - pmx, uy = py[k] - pmy, vx = q[2 * k] - qmx, vy = q[2 * k + 1] - qmy;
        den += ux * ux + uy * uy;
        sxx += ux * vx + uy * vy;
        sxy += ux * vy - uy * vx;
    }
    if (den == 0.0) {
        for (int k = 0; k < 6; k++) M[k] = 0.0;
        return false;
    }
    const double a = sxx / den, b = sxy / den;
    M[0] = a; M[1] = -b; M[2] = qmx - a * pmx + b * pmy;
    M[3] = b; M[4] = a;  M[5] = qmy - b * pmx - a * pmy;
    return true;
}

// cv::invertAffineTransform (double); on the host for f23's rotated views
__host__ __device__ inline void invert_affine(const double m[6], double im[6]) {
    double D = m[0] * m[4] - m[1] * m[3];
    D = D != 0.0 ? 1.0 / D : 0.0;
    const double a11 = m[4] * D, a22 = m[0] * D, a12 = -m[1] * D, a21 = -m[3] * D;
    im[0] = a11; im[1] = a12; im[2] = -a11 * m[2] - a12 * m[5];
    im[3] = a21; im[4] = a22; im[5] = -a21 * m[2] - a22 * m[5];
}

// One output pixel of cv::warpAffine INTER_LINEAR / BORDER_CONSTANT 0 on 8UC3: X, Y in 1/32 source pixel (X0 + adelta >> 5),
// integer weights 32 (32 - fx) (32 - fy) ... summing to 32768, taps outside the image contribute 0, (sum + 16384) >> 15.
__device__ __forceinline__ void tap(const AlignImageT<BgrRows> &im, int x, int y, int p[3]) {
    const uint8_t *q = im.src.p + (size_t)y * im.src.pitch + (size_t)x * 3;
    p[0] = q[0]; p[1] = q[1]; p[2] = q[2];
}
__device__ __forceinline__ void tap(const AlignImageT<YuvPlanes> &im, int x, int y, int p[3]) { yuv_pixel(im.src, x, y, p); }
// displayed pixel (x, y) of an oriented image: reflected, then transposed, as the letter-box reads it (preprocess.cu)
template <typename Img>
__device__ __forceinline__ void oriented_tap(const Img &im, int x, int y, int p[3]) {
    if (im.orient & LB_FLIP_X) x = im.w - 1 - x;
    if (im.orient & LB_FLIP_Y) y = im.h - 1 - y;
    if (im.orient & LB_TRANSPOSE) tap(im, y, x, p);
    else tap(im, x, y, p);
}

// Returns whether all four taps lay in the image (f11's INSIDE test); the pixel does not depend on it.
template <bool ORIENTED, typename Img>
__device__ __forceinline__ bool sample(const Img &im, int X, int Y, int v[3]) {
    const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);   // saturate_cast<short>
    const int fx = X & 31, fy = Y & 31;
    const int wts[4] = {32 * (32 - fx) * (32 - fy), 32 * fx * (32 - fy), 32 * (32 - fx) * fy, 32 * fx * fy};
    int acc[3] = {16384, 16384, 16384};
    int inside = 0;
#pragma unroll
    for (int t = 0; t < 4; t++) {
        const int tx = sx + (t & 1), ty = sy + (t >> 1);
        if ((unsigned)tx < (unsigned)im.w && (unsigned)ty < (unsigned)im.h) {
            int p[3];
            if (ORIENTED) oriented_tap(im, tx, ty, p);
            else tap(im, tx, ty, p);
            acc[0] += wts[t] * p[0]; acc[1] += wts[t] * p[1]; acc[2] += wts[t] * p[2];
            inside++;
        }
    }
    v[0] = acc[0] >> 15; v[1] = acc[1] >> 15; v[2] = acc[2] >> 15;
    return inside == 4;
}

// Four consecutive pixels of one crop row (x4 .. x4 + 3, those < cw valid).  Vector stores where the address allows.
__device__ __forceinline__ void store_quad(const AlignArgs &a, unsigned char *crop, int y, int x4, const int v[4][3]) {
    const int cw = a.crop_w;
    const int nv = min(4, cw - x4);
    if (a.format == RF_CROP_BGR_U8) {
        unsigned char *d = crop + ((size_t)y * cw + x4) * 3;
        if (nv == 4 && ((uintptr_t)d & 3) == 0) {
            uint32_t *o = reinterpret_cast<uint32_t *>(d);
            o[0] = v[0][0] | (v[0][1] << 8) | (v[0][2] << 16) | ((uint32_t)v[1][0] << 24);
            o[1] = v[1][1] | (v[1][2] << 8) | (v[2][0] << 16) | ((uint32_t)v[2][1] << 24);
            o[2] = v[2][2] | (v[3][0] << 8) | (v[3][1] << 16) | ((uint32_t)v[3][2] << 24);
        } else {
            for (int k = 0; k < nv; k++)
                for (int c = 0; c < 3; c++) d[3 * k + c] = (unsigned char)v[k][c];
        }
        return;
    }
    const size_t plane = (size_t)a.crop_h * cw, off = (size_t)y * cw + x4;
#pragma unroll
    for (int c = 0; c < 3; c++) {                 // planes R, G, B = BGR channels 2, 1, 0
        float f[4];
#pragma unroll
        for (int k = 0; k < 4; k++) f[k] = __fmul_rn(__fsub_rn((float)v[k][2 - c], a.mean), a.inv_std);
        if (a.format == RF_CROP_RGB_F32) {
            float *d = reinterpret_cast<float *>(crop) + c * plane + off;
            if (nv == 4 && ((uintptr_t)d & 15) == 0) *reinterpret_cast<float4 *>(d) = make_float4(f[0], f[1], f[2], f[3]);
            else for (int k = 0; k < nv; k++) d[k] = f[k];
        } else {
            __half *d = reinterpret_cast<__half *>(crop) + c * plane + off;
            if (nv == 4 && ((uintptr_t)d & 7) == 0) {
                __half2 lo = __floats2half2_rn(f[0], f[1]), hi = __floats2half2_rn(f[2], f[3]);
                *reinterpret_cast<uint2 *>(d) = make_uint2(*reinterpret_cast<uint32_t *>(&lo), *reinterpret_cast<uint32_t *>(&hi));
            } else {
                for (int k = 0; k < nv; k++) d[k] = __float2half_rn(f[k]);
            }
        }
    }
}

}  // namespace rf
