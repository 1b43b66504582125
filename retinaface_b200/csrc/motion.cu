// motion.cu -- f13 camera-motion estimate (motion.cuh, rf_b200.h rf_tracker_set_motion).  Built with -fmad=false: every FP64 step
// below is one rounded operation in the order written, which oracle/motion.py restates operation by operation.
//
//   k_motion_thumb   one CTA per (thumbnail row, frame), one thread per thumbnail column: the rounded D x D luma box means.
//   k_motion_match   one CTA per (block, frame): texture and record tests, then the exhaustive SAD over (2R + 1)^2 offsets, one
//                    offset per thread at a time, the block in registers and the reference window in shared memory as four
//                    byte-shifted copies so that every row of a candidate is four aligned words (__vsadu4); the minimum key, the tie
//                    count and the sub-pixel parabola.
//   k_motion_fit     one CTA per frame: kept blocks compacted in block order, hypotheses over threads (shared-memory atomic max of
//                    (inliers, -index)), then two select + least-squares rounds in warp 0 (the header's 32-lane sums).
//   k_motion_commit  each video's last thumbnail of the call into its reference slot.
#include <algorithm>

#include "motion.cuh"

namespace rf {
namespace {

constexpr int MATCH_THREADS = 256;                        // one per block pixel, then per offset
constexpr int FIT_THREADS = 512;                          // >= MOTION_MAX_BLOCKS: one thread per block in the compactions
constexpr int WIN = MOTION_BLOCK + 2 * MOTION_MAX_R;      // reference window side at the largest R
constexpr int WIN_WORDS = 20;                             // words per row of one shifted copy: (2R >> 2) + 4 <= 20
constexpr int COPY_WORDS = WIN * WIN_WORDS + 8;           // the four copies start 8 banks apart
constexpr int MAX_OFFSETS = (2 * MOTION_MAX_R + 1) * (2 * MOTION_MAX_R + 1);
static_assert(FIT_THREADS >= MOTION_MAX_BLOCKS, "one thread per block");

// f20: the ORIENTED instantiation sums the displayed D x D box through the frame's signed strides (the sum is order-free).  On a
// transposed frame the displayed columns are stored rows: there a CTA takes a thumbnail column and its threads the rows, so that a
// warp's loads stay on consecutive stored bytes, and each thread walks its stored rows innermost.
template <bool ORIENTED>
__global__ void __launch_bounds__(MOTION_THUMB) k_motion_thumb(const MotionArgs a, const __grid_constant__ MotionTable t) {
    const MotionFrame &f = t.f[blockIdx.y];
    const bool tr = ORIENTED && f.xs != 1 && f.xs != -1;
    const int y = tr ? threadIdx.x : blockIdx.x, x = tr ? blockIdx.x : threadIdx.x;
    if (y >= f.th || x >= f.tw) return;
    const int D = f.D;
    unsigned sum = 0;
    if constexpr (ORIENTED) {
        const long long inner = tr ? f.pitch : f.xs, outer = tr ? f.xs : f.pitch;
        const uint8_t *src = f.y + (long long)D * y * f.pitch + (long long)D * x * f.xs;
        for (int r = 0; r < D; r++, src += outer)
            for (int c = 0; c < D; c++) sum += src[c * inner];
    } else {
        const uint8_t *src = f.y + (size_t)D * y * f.pitch + (size_t)D * x;
        for (int r = 0; r < D; r++, src += f.pitch)
            for (int c = 0; c < D; c++) sum += src[c];
    }
    const unsigned DD = (unsigned)(D * D);
    a.thumbs[(size_t)(t.i0 + blockIdx.y) * MOTION_THUMB_BYTES + y * f.tw + x] = (uint8_t)((sum + DD / 2) / DD);
}

__global__ void __launch_bounds__(MATCH_THREADS) k_motion_match(const MotionArgs a, const __grid_constant__ MotionTable t) {
    __shared__ uint32_t s_win[4 * COPY_WORDS];
    __shared__ uint32_t s_cur[MOTION_BLOCK * MOTION_BLOCK / 4];
    __shared__ int s_sad[MAX_OFFSETS];
    __shared__ unsigned long long s_key[MATCH_THREADS / 32];
    __shared__ unsigned long long s_sum, s_sq;
    __shared__ int s_skip, s_ties;
    const MotionFrame &f = t.f[blockIdx.y];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    if (f.ref == MOTION_REF_FIRST || b >= f.nbx * f.nby) return;       // uniform
    const int fi = t.i0 + blockIdx.y, R = a.search, tw = f.tw, side = 2 * R + 1;
    MotionBlock *out = a.blocks + (size_t)fi * MOTION_MAX_BLOCKS + b;
    const int x0 = R + MOTION_BLOCK * (b % f.nbx), y0 = R + MOTION_BLOCK * (b / f.nbx);
    const uint8_t *cur = a.thumbs + (size_t)fi * MOTION_THUMB_BYTES;
    const uint8_t *ref = f.ref >= 0 ? a.thumbs + (size_t)f.ref * MOTION_THUMB_BYTES : a.store + (size_t)f.video * MOTION_THUMB_BYTES;
    if (tid == 0) { s_sum = 0; s_sq = 0; s_skip = 0; s_ties = 0; }
    __syncthreads();
    {   // the block's bytes and its texture (integer sums: order-free)
        const unsigned p = cur[(y0 + (tid >> 4)) * tw + x0 + (tid & 15)];
        reinterpret_cast<uint8_t *>(s_cur)[tid] = (uint8_t)p;
        unsigned s1 = p, s2 = p * p;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
        if (lane == 0) { atomicAdd(&s_sum, (unsigned long long)s1); atomicAdd(&s_sq, (unsigned long long)s2); }
    }
    {   // the records, grown by the margin, against the block's frame rectangle
        const int K = min(max(a.counts[fi], 0), a.max_faces);
        const double X0 = (double)(f.D * x0), X1 = (double)(f.D * (x0 + MOTION_BLOCK));
        const double Y0 = (double)(f.D * y0), Y1 = (double)(f.D * (y0 + MOTION_BLOCK));
        for (int j = tid; j < K; j += MATCH_THREADS) {
            const rf_face &r = a.dets[(size_t)fi * a.max_faces + j].face;
            const double x1 = __fmul_rn(r.x1, f.scale), y1 = __fmul_rn(r.y1, f.scale), x2 = __fmul_rn(r.x2, f.scale), y2 = __fmul_rn(r.y2, f.scale);
            const double w = x2 - x1, h = y2 - y1;
            const double gx1 = x1 - RF_MOTION_FACE_MARGIN * w, gx2 = x2 + RF_MOTION_FACE_MARGIN * w;
            const double gy1 = y1 - RF_MOTION_FACE_MARGIN * h, gy2 = y2 + RF_MOTION_FACE_MARGIN * h;
            if (gx1 < X1 && gx2 > X0 && gy1 < Y1 && gy2 > Y0) s_skip = 1;
        }
    }
    __syncthreads();
    const long long var = 256LL * (long long)s_sq - (long long)s_sum * (long long)s_sum;
    if (s_skip || var < (long long)RF_MOTION_MIN_VAR * 65536) {          // uniform
        if (tid == 0) out->kept = 0;
        return;
    }
    // the reference window (origin (x0 - R, y0 - R), side 16 + 2R) as four copies: word w of copy k holds window bytes 4w + k .. + 3
    const int ww = MOTION_BLOCK + 2 * R, nw = (2 * R >> 2) + 4;
    const uint8_t *wsrc = ref + (size_t)(y0 - R) * tw + (x0 - R);
    for (int i = tid; i < 4 * ww * nw; i += MATCH_THREADS) {
        const int k = i / (ww * nw), rem = i - k * ww * nw, r = rem / nw, w = rem - r * nw;
        uint32_t word = 0;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int col = 4 * w + k + e;
            word |= (uint32_t)(col < ww ? wsrc[(size_t)r * tw + col] : 0) << (8 * e);
        }
        s_win[k * COPY_WORDS + r * WIN_WORDS + w] = word;
    }
    __syncthreads();
    uint32_t cw[MOTION_BLOCK * MOTION_BLOCK / 4];
#pragma unroll
    for (int k = 0; k < MOTION_BLOCK * MOTION_BLOCK / 4; k++) cw[k] = s_cur[k];
    unsigned long long best = ~0ull;
    for (int o = tid; o < side * side; o += MATCH_THREADS) {
        const int sy = o / side, sx = o - sy * side;
        const uint32_t *wp = s_win + (sx & 3) * COPY_WORDS + sy * WIN_WORDS + (sx >> 2);
        unsigned sad = 0;
#pragma unroll
        for (int r = 0; r < MOTION_BLOCK; r++)
#pragma unroll
            for (int w = 0; w < 4; w++) sad += __vsadu4(cw[r * 4 + w], wp[r * WIN_WORDS + w]);
        s_sad[o] = (int)sad;
        const int dy = sy - R, dx = sx - R;
        const unsigned long long key = ((unsigned long long)sad << 21) | ((unsigned long long)(abs(dy) + abs(dx)) << 14) |
                                       ((unsigned long long)sy << 7) | (unsigned long long)sx;
        best = min(best, key);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) s_key[tid >> 5] = best;
    __syncthreads();
    best = s_key[0];
#pragma unroll
    for (int w = 1; w < MATCH_THREADS / 32; w++) best = min(best, s_key[w]);
    const int smin = (int)(best >> 21);
    int ties = 0;
    for (int o = tid; o < side * side; o += MATCH_THREADS) ties += s_sad[o] == smin;
    if (ties) atomicAdd(&s_ties, ties);
    __syncthreads();
    if (tid != 0) return;
    const int sy = (int)(best >> 7) & 127, sx = (int)best & 127;
    if (s_ties > 1 || sx == 0 || sy == 0 || sx == 2 * R || sy == 2 * R) { out->kept = 0; return; }
    const int c = sy * side + sx;
    const int xm = s_sad[c - 1], xp = s_sad[c + 1], ym = s_sad[c - side], yp = s_sad[c + side];
    const double fx = (double)(xm - xp) / (double)(2 * (xm - 2 * smin + xp));
    const double fy = (double)(ym - yp) / (double)(2 * (ym - 2 * smin + yp));
    MotionBlock m;
    m.px = (double)x0 + 7.5;
    m.py = (double)y0 + 7.5;
    m.qx = (m.px + (double)(sx - R)) + fx;
    m.qy = (m.py + (double)(sy - R)) + fy;
    m.kept = 1;
    m.pad = 0;
    *out = m;
}

// Every thread of the CTA calls it: list[0..count) = the threads whose flag is set, in thread order; returns the count.
__device__ int ordered_compact(bool flag, short *list, int *s_warp) {
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    __syncthreads();
    if (lane == 0) s_warp[w] = __popc(bal);
    __syncthreads();
    int off = 0, total = 0;
#pragma unroll
    for (int k = 0; k < FIT_THREADS / 32; k++) {
        const int c = s_warp[k];
        off += k < w ? c : 0;
        total += c;
    }
    if (flag) list[off + __popc(bal & ((1u << lane) - 1u))] = (short)tid;
    __syncthreads();
    return total;
}

struct Points {
    const double *qx, *qy, *px, *py;
};

__device__ __forceinline__ bool inlier(const double m[4], const Points &P, int k) {
    const double ex = ((m[0] * P.qx[k] - m[1] * P.qy[k]) + m[2]) - P.px[k];
    const double ey = ((m[1] * P.qx[k] + m[0] * P.qy[k]) + m[3]) - P.py[k];
    return ex * ex + ey * ey <= RF_MOTION_TOL * RF_MOTION_TOL;
}

// hypothesis h of N points -> (a, b, tx, ty); false: a degenerate pair (no inliers)
__device__ __forceinline__ bool hypothesis(int h, int N, const Points &P, double m[4]) {
    if (h < N) {
        m[0] = 1.0; m[1] = 0.0; m[2] = P.px[h] - P.qx[h]; m[3] = P.py[h] - P.qy[h];
        return true;
    }
    const int k1 = h - N, k2 = k1 + N / 2;
    const double dqx = P.qx[k2] - P.qx[k1], dqy = P.qy[k2] - P.qy[k1], dpx = P.px[k2] - P.px[k1], dpy = P.py[k2] - P.py[k1];
    const double den = dqx * dqx + dqy * dqy;
    if (den == 0.0) return false;
    const double a = (dpx * dqx + dpy * dqy) / den, b = (dpy * dqx - dpx * dqy) / den;
    m[0] = a; m[1] = b;
    m[2] = P.px[k1] - (a * P.qx[k1] - b * P.qy[k1]);
    m[3] = P.py[k1] - (b * P.qx[k1] + a * P.qy[k1]);
    return true;
}

// the header's 32-lane sum: v is this lane's in-order partial
__device__ __forceinline__ double lane_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = v + __shfl_down_sync(0xffffffffu, v, o);
    return __shfl_sync(0xffffffffu, v, 0);
}

// least squares over list[0..n) (warp 0); false: the points coincide
__device__ bool ls_fit(const short *list, int n, const Points &P, double m[4]) {
    const int lane = threadIdx.x & 31;
    double sqx = 0.0, sqy = 0.0, spx = 0.0, spy = 0.0;
    for (int j = lane; j < n; j += 32) {
        const int k = list[j];
        sqx = sqx + P.qx[k]; sqy = sqy + P.qy[k]; spx = spx + P.px[k]; spy = spy + P.py[k];
    }
    const double dn = (double)n;
    const double mqx = lane_sum(sqx) / dn, mqy = lane_sum(sqy) / dn, mpx = lane_sum(spx) / dn, mpy = lane_sum(spy) / dn;
    double den = 0.0, sa = 0.0, sb = 0.0;
    for (int j = lane; j < n; j += 32) {
        const int k = list[j];
        const double ux = P.qx[k] - mqx, uy = P.qy[k] - mqy, vx = P.px[k] - mpx, vy = P.py[k] - mpy;
        den = den + (ux * ux + uy * uy);
        sa = sa + (ux * vx + uy * vy);
        sb = sb + (ux * vy - uy * vx);
    }
    den = lane_sum(den);
    sa = lane_sum(sa);
    sb = lane_sum(sb);
    if (den == 0.0) return false;
    const double a = sa / den, b = sb / den;
    m[0] = a; m[1] = b;
    m[2] = (mpx - a * mqx) + b * mqy;
    m[3] = (mpy - b * mqx) - a * mqy;
    return true;
}

__global__ void __launch_bounds__(FIT_THREADS) k_motion_fit(const MotionArgs a, const __grid_constant__ MotionTable t) {
    __shared__ double s_qx[MOTION_MAX_BLOCKS], s_qy[MOTION_MAX_BLOCKS], s_px[MOTION_MAX_BLOCKS], s_py[MOTION_MAX_BLOCKS];
    __shared__ short s_list[FIT_THREADS];
    __shared__ int s_warp[FIT_THREADS / 32];
    __shared__ unsigned s_best;
    __shared__ double s_m[4];
    __shared__ int s_ok;
    const MotionFrame &f = t.f[blockIdx.x];
    const int fi = t.i0 + blockIdx.x, tid = threadIdx.x;
    rf_motion *out = a.out + fi;
    rf_motion r{};
    r.m[0] = 1.0; r.m[4] = 1.0;       // the identity
    if (f.ref == MOTION_REF_FIRST) {   // uniform
        if (tid == 0) { r.status = RF_MOTION_FIRST; *out = r; }
        return;
    }
    r.status = RF_MOTION_LOST;
    const MotionBlock *blk = a.blocks + (size_t)fi * MOTION_MAX_BLOCKS;
    const int nb = f.nbx * f.nby;
    const int N = ordered_compact(tid < nb && blk[tid].kept, s_list, s_warp);
    r.blocks = N;
    if (tid < N) {
        const MotionBlock &b = blk[s_list[tid]];
        s_qx[tid] = b.qx; s_qy[tid] = b.qy; s_px[tid] = b.px; s_py[tid] = b.py;
    }
    if (tid == 0) s_best = 0;
    __syncthreads();
    if (N < a.min_inliers) {           // uniform
        if (tid == 0) *out = r;
        return;
    }
    const Points P{s_qx, s_qy, s_px, s_py};
    const int H = N + N / 2;
    for (int h = tid; h < H; h += FIT_THREADS) {
        double m[4];
        int cnt = 0;
        if (hypothesis(h, N, P, m))
            for (int k = 0; k < N; k++) cnt += inlier(m, P, k);
        atomicMax(&s_best, ((unsigned)cnt << 16) | (unsigned)(0xffff - h));
    }
    __syncthreads();
    double m[4];
    hypothesis(0xffff - (int)(s_best & 0xffff), N, P, m);
    for (int round = 0; round < 2; round++) {
        const int n = ordered_compact(tid < N && inlier(m, P, tid), s_list, s_warp);
        r.inliers = n;
        if (n < a.min_inliers) {       // uniform
            if (tid == 0) *out = r;
            return;
        }
        if (tid < 32) {
            double mm[4];
            const bool ok = ls_fit(s_list, n, P, mm);
            if (tid == 0) {
                s_ok = ok;
                for (int k = 0; k < 4; k++) s_m[k] = mm[k];
            }
        }
        __syncthreads();
        if (!s_ok) {                   // uniform
            if (tid == 0) *out = r;
            return;
        }
        for (int k = 0; k < 4; k++) m[k] = s_m[k];
        __syncthreads();               // s_m is rewritten by the next round
    }
    if (tid != 0) return;
    const double A = m[0], B = m[1], s = sqrt(A * A + B * B);
    if (s >= RF_MOTION_MIN_SCALE && s <= RF_MOTION_MAX_SCALE) {
        const double D = (double)f.D, c = (D - 1.0) / 2.0;
        r.status = RF_MOTION_OK;
        r.m[0] = A; r.m[1] = -B; r.m[3] = B; r.m[4] = A;
        r.m[2] = ((D * m[2]) + c) - ((A * c) - (B * c));
        r.m[5] = ((D * m[3]) + c) - ((B * c) + (A * c));
    }
    *out = r;
}

struct MotionCommit {
    int n;
    int frame[TRACK_MAX_FRAMES], video[TRACK_MAX_FRAMES], bytes[TRACK_MAX_FRAMES];
};

__global__ void __launch_bounds__(256) k_motion_commit(const MotionArgs a, const __grid_constant__ MotionCommit c) {
    const int k = blockIdx.y;
    const uint4 *src = reinterpret_cast<const uint4 *>(a.thumbs + (size_t)c.frame[k] * MOTION_THUMB_BYTES);
    uint4 *dst = reinterpret_cast<uint4 *>(a.store + (size_t)c.video[k] * MOTION_THUMB_BYTES);
    const int words = (c.bytes[k] + 15) / 16;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < words; i += gridDim.x * blockDim.x) dst[i] = src[i];
}

}  // namespace

cudaError_t launch_motion_estimate(const MotionArgs &a, const MotionTable *tables, int ntables, cudaStream_t s) {
    for (int k = 0; k < ntables; k++) {
        const MotionTable &t = tables[k];
        int th = 1;
        bool oriented = false;
        for (int i = 0; i < t.n; i++) {
            const bool tr = t.f[i].xs != 1 && t.f[i].xs != -1;        // f20: a transposed frame's CTAs take thumbnail columns
            th = std::max(th, tr ? t.f[i].tw : t.f[i].th);
            oriented |= t.f[i].xs != 1 || t.f[i].pitch < 0;
        }
        if (oriented) k_motion_thumb<true><<<dim3(th, t.n), MOTION_THUMB, 0, s>>>(a, t);
        else k_motion_thumb<false><<<dim3(th, t.n), MOTION_THUMB, 0, s>>>(a, t);
    }
    for (int k = 0; k < ntables; k++) {
        const MotionTable &t = tables[k];
        int nb = 1;
        for (int i = 0; i < t.n; i++) nb = std::max(nb, t.f[i].nbx * t.f[i].nby);
        k_motion_match<<<dim3(nb, t.n), MATCH_THREADS, 0, s>>>(a, t);
    }
    for (int k = 0; k < ntables; k++) k_motion_fit<<<tables[k].n, FIT_THREADS, 0, s>>>(a, tables[k]);
    return cudaGetLastError();
}

cudaError_t launch_motion_commit(const MotionArgs &a, const int *frames, const int *videos, const int *bytes, int n, cudaStream_t s) {
    for (int i0 = 0; i0 < n; i0 += TRACK_MAX_FRAMES) {
        MotionCommit c{};
        c.n = std::min(TRACK_MAX_FRAMES, n - i0);
        for (int i = 0; i < c.n; i++) { c.frame[i] = frames[i0 + i]; c.video[i] = videos[i0 + i]; c.bytes[i] = bytes[i0 + i]; }
        k_motion_commit<<<dim3(8, c.n), 256, 0, s>>>(a, c);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace rf
