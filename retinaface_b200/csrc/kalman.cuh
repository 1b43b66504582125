// kalman.cuh -- the f10 filter steps shared by k_track_update (track.cu) and the f16 follow kernels (follow.cu): z of a face, the
// box of a state, predict, f13's motion step and update, in the order track.cu's header states.  Include it only from sources built with -fmad=false.
#pragma once
#include "track.cuh"

namespace rf {

constexpr double kSp = 1.0 / 20.0, kSv = 1.0 / 160.0;

// z (cx, cy, a, h) of a face; false for an empty box
__device__ __forceinline__ bool measure(const rf_face &f, double z[4]) {
    const double x1 = f.x1, y1 = f.y1, w = (double)f.x2 - x1, h = (double)f.y2 - y1;
    if (!(w > 0.0) || !(h > 0.0)) return false;
    z[0] = x1 + w / 2.0;
    z[1] = y1 + h / 2.0;
    z[2] = w / h;
    z[3] = h;
    return true;
}

__device__ __forceinline__ void box_of(const double m[4], double b[4]) {
    const double w = m[2] * m[3];
    b[0] = m[0] - w / 2.0;
    b[1] = m[1] - m[3] / 2.0;
    b[2] = b[0] + w;
    b[3] = b[1] + m[3];
}

__device__ __forceinline__ void kalman_predict(TrackState &k) {
    if (k.state == RF_TRACK_LOST) k.u[3] = 0.0;
    const double h = k.m[3];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const double qp = c == 2 ? 1e-2 : kSp * h, qv = c == 2 ? 1e-5 : kSv * h;
        const double p00 = k.p00[c], p01 = k.p01[c], p11 = k.p11[c];
        k.p00[c] = ((p00 + p01) + (p01 + p11)) + qp * qp;
        k.p01[c] = p01 + p11;
        k.p11[c] = p11 + qv * qv;
        k.m[c] = k.m[c] + k.u[c];
    }
}

// m: rf_motion.m = {a, -b, tx, b, a, ty}
__device__ __forceinline__ void kalman_motion(TrackState &k, const double m[6]) {
    const double a = m[0], b = m[3], tx = m[2], ty = m[5];
    const double s = sqrt(a * a + b * b), ss = s * s;
    const double cx = k.m[0], cy = k.m[1], ux = k.u[0], uy = k.u[1];
    k.m[0] = (a * cx - b * cy) + tx;
    k.m[1] = (b * cx + a * cy) + ty;
    k.u[0] = a * ux - b * uy;
    k.u[1] = b * ux + a * uy;
    k.m[3] = s * k.m[3];
    k.u[3] = s * k.u[3];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        if (c == 2) continue;
        k.p00[c] = ss * k.p00[c];
        k.p01[c] = ss * k.p01[c];
        k.p11[c] = ss * k.p11[c];
    }
}

__device__ __forceinline__ void kalman_update(TrackState &k, const double z[4]) {
    const double h = k.m[3];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const double r = c == 2 ? 1e-1 : kSp * h;
        const double p00 = k.p00[c], p01 = k.p01[c], p11 = k.p11[c];
        const double S = p00 + r * r, K0 = p00 / S, K1 = p01 / S, y = z[c] - k.m[c];
        k.m[c] = k.m[c] + K0 * y;
        k.u[c] = k.u[c] + K1 * y;
        k.p00[c] = p00 - (K0 * S) * K0;
        k.p01[c] = p01 - (K0 * S) * K1;
        k.p11[c] = p11 - (K1 * S) * K1;
    }
}

}  // namespace rf
