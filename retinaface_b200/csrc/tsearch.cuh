// tsearch.cuh -- f16's template search (rf_b200.h rf_tracker_set_follow: Grid, Sampler, Cut, Windows, Match, Box, Status), shared by
// follow.cu's k_follow_cut / k_follow_search and f17's k_lookback_search (lookback_search.cu).  Every FP64 step is one rounding in the order
// written: include it only from sources built with -fmad=false.  The CTA is FOLLOW_THREADS threads; the functions marked "every
// thread" are called by all of them, the shared arrays are the caller's.
#pragma once
#include "follow.cuh"
#include "yuv.cuh"

namespace rf {

constexpr int FOLLOW_WIN = FOLLOW_T + 2 * FOLLOW_MAX_R;       // window side at the largest R
constexpr int FOLLOW_WWORDS = FOLLOW_WIN / 4 + 1;             // words per window row: a candidate row may read one word past its last
constexpr int FOLLOW_MAX_SIDE = 2 * FOLLOW_MAX_R + 1;
constexpr double kFollowGrow = 1.0 + 2.0 * RF_FOLLOW_MARGIN;
constexpr double FOLLOW_MAX_BOX = 65536.0;                    // predicted centre and size bound: keeps the fixed-point coordinates in int

struct Grid {
    double px, py, ox, oy;
};

__device__ __forceinline__ Grid grid_of(double cx, double cy, double w, double h, double c) {
    const double gw = (w * kFollowGrow) * c, gh = (h * kFollowGrow) * c;
    Grid g;
    g.px = gw / (double)FOLLOW_T;
    g.py = gh / (double)FOLLOW_T;
    g.ox = ((cx - gw / 2.0) + g.px / 2.0) - 0.5;
    g.oy = ((cy - gh / 2.0) + g.py / 2.0) - 0.5;
    return g;
}

// c_k: {1 / s, 1, s}
__device__ __forceinline__ double scale_of(int k) { return k == 0 ? 1.0 / RF_FOLLOW_SCALE : k == 1 ? 1.0 : RF_FOLLOW_SCALE; }

// A luma plane as the search reads it: sample (x, y) at y[y * pitch + x], w x h.
struct PitchedLuma {
    const uint8_t *y;
    int pitch, w, h;
};
// f20: a luma plane read as it is displayed: sample (x, y) at y[x * xs + y * ys] (yuv.cuh plane_map), w x h the displayed size.
struct OrientedLuma {
    const uint8_t *y;
    int xs, ys, w, h;
};
// A stored luma plane (pitch bytes a row) of a frame shown in orientation `bits` as w x h.
__device__ __forceinline__ OrientedLuma oriented_luma(const uint8_t *y, int pitch, int bits, int w, int h) {
    const PlaneMap m = plane_map(bits, w, h, pitch, 1);
    return OrientedLuma{y + m.off, m.xs, m.ys, w, h};
}
template <class P>
__device__ __forceinline__ int luma_px(const P &f, int x, int y) { return f.y[(size_t)y * f.pitch + x]; }
__device__ __forceinline__ int luma_px(const OrientedLuma &f, int x, int y) { return f.y[(long long)y * f.ys + (long long)x * f.xs]; }

// Pixel (i, j) of the map [[px, 0, X], [0, py, Y]]: cv::warpAffine's fixed-point coordinate and f5's integer bilinear on the luma
// plane (warp.cuh's sample() on one channel).  inside: all four taps lay in the frame.  P: a luma plane with y, w and h, read by
// luma_px (PitchedLuma, FollowFrame, or an OrientedLuma).
template <class P>
__device__ __forceinline__ int luma_at(const P &f, double px, double py, double X, double Y, int i, int j, bool &inside) {
    const int Xf = (__double2int_rn(X * 1024.0) + 16 + __double2int_rn((px * (double)i) * 1024.0)) >> 5;
    const int Yf = (__double2int_rn((py * (double)j + Y) * 1024.0) + 16) >> 5;
    const int sx = min(max(Xf >> 5, -32768), 32767), sy = min(max(Yf >> 5, -32768), 32767);
    const int fx = Xf & 31, fy = Yf & 31;
    const int wts[4] = {32 * (32 - fx) * (32 - fy), 32 * fx * (32 - fy), 32 * (32 - fx) * fy, 32 * fx * fy};
    int acc = 16384, in = 0;
#pragma unroll
    for (int t = 0; t < 4; t++) {
        const int tx = sx + (t & 1), ty = sy + (t >> 1);
        if ((unsigned)tx < (unsigned)f.w && (unsigned)ty < (unsigned)f.h) {
            acc += wts[t] * luma_px(f, tx, ty);
            in++;
        }
    }
    inside = in == 4;
    return acc >> 15;
}

// The Cut's grid of a face box (c = 1): g = {px, py, ox, oy}.
__device__ __forceinline__ void cut_grid(const rf_face &face, double g[4]) {
    const double x1 = face.x1, y1 = face.y1, w = (double)face.x2 - x1, h = (double)face.y2 - y1;
    const Grid q = grid_of(x1 + w / 2.0, y1 + h / 2.0, w, h, 1.0);
    g[0] = q.px; g[1] = q.py; g[2] = q.ox; g[3] = q.oy;
}

// Every thread: the T x T template at the grid s_g into dst (global or shared), its pixel sums added to *s_sum and *s_sq (zeroed
// before; read after a barrier).
template <class P, class D>
__device__ __forceinline__ void cut_template(const P &f, const double *s_g, D *dst, unsigned long long *s_sum, unsigned long long *s_sq) {
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned s1 = 0, s2 = 0;
    for (int p = tid; p < FOLLOW_BYTES; p += FOLLOW_THREADS) {
        bool in;
        const unsigned v = (unsigned)luma_at(f, s_g[0], s_g[1], s_g[2], s_g[3], p % FOLLOW_T, p / FOLLOW_T, in);
        dst[p] = (uint8_t)v;
        s1 += v;
        s2 += v * v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if (lane == 0) { atomicAdd(s_sum, (unsigned long long)s1); atomicAdd(s_sq, (unsigned long long)s2); }
}

// The FLAT test of a template's sums.
__device__ __forceinline__ bool template_flat(unsigned long long sum, unsigned long long sq) {
    const long long var = (long long)FOLLOW_BYTES * (long long)sq - (long long)sum * (long long)sum;
    return var < (long long)RF_FOLLOW_MIN_VAR * FOLLOW_BYTES * FOLLOW_BYTES;
}

// A predicted box the search may sample: ph, pw in (0, 65536], |pcx|, |pcy| <= 65536 (else MISMATCH, not searched).  An expression,
// not a function: k_follow_search then compiles as it did before the search moved here.
#define FOLLOW_SEARCH_BOUNDED(pcx, pcy, pw, ph)                                                                                      \
    ((ph) > 0.0 && (ph) <= FOLLOW_MAX_BOX && (pw) > 0.0 && (pw) <= FOLLOW_MAX_BOX && fabs(pcx) <= FOLLOW_MAX_BOX && fabs(pcy) <= FOLLOW_MAX_BOX)

// Threads 0..2: scale k's window grid, its origin moved back by R template pixels.
__device__ __forceinline__ void search_grid(double (*s_g)[4], int k, double pcx, double pcy, double pw, double ph, int R) {
    const Grid g = grid_of(pcx, pcy, pw, ph, scale_of(k));
    s_g[k][0] = g.px;
    s_g[k][1] = g.py;
    s_g[k][2] = g.ox - (double)R * g.px;
    s_g[k][3] = g.oy - (double)R * g.py;
}

// Every thread (tid: threadIdx.x): the three W x W windows and their INSIDE flags.
template <class P>
__device__ __forceinline__ void search_windows(const P &f, const double (*s_g)[4], int W, uint32_t (*s_win)[FOLLOW_WIN][FOLLOW_WWORDS],
                                               uint8_t (*s_in)[FOLLOW_WIN][FOLLOW_WIN], int tid) {
    for (int p = tid; p < 3 * W * W; p += FOLLOW_THREADS) {
        const int k = p / (W * W), rem = p - k * W * W, r = rem / W, c = rem - r * W;
        bool in;
        const int v = luma_at(f, s_g[k][0], s_g[k][1], s_g[k][2], s_g[k][3], c, r, in);
        reinterpret_cast<uint8_t *>(s_win[k][r])[c] = (uint8_t)v;
        s_in[k][r][c] = in;
    }
}

// Every thread, after the windows' barrier: every candidate's SAD into s_sad, and the minimum under (SAD, |dx| + |dy|, k, dy, dx) as
// one 64-bit key, returned to every thread.  side = 2 R + 1, nc = side^2 and lane = tid & 31 come from the caller, which computes them
// once for the whole kernel.
__device__ __forceinline__ unsigned long long search_min(const uint32_t (*s_win)[FOLLOW_WIN][FOLLOW_WWORDS], const uint32_t *s_tpl, int *s_sad,
                                                         unsigned long long *s_key, int R, int side, int nc, int tid, int lane) {
    unsigned long long best = ~0ull;
    for (int o = tid; o < 3 * nc; o += FOLLOW_THREADS) {
        const int k = o / nc, rem = o - k * nc, wy = rem / side, wx = rem - wy * side;
        const uint32_t *wp = &s_win[k][wy][wx >> 2];
        const unsigned sel = 0x3210u + 0x1111u * (unsigned)(wx & 3);
        unsigned sad = 0;
        for (int r = 0; r < FOLLOW_T; r++, wp += FOLLOW_WWORDS) {
            uint32_t w0 = wp[0];
#pragma unroll
            for (int q = 0; q < FOLLOW_T / 4; q++) {
                const uint32_t w1 = wp[q + 1];
                sad = __vsadu4(s_tpl[r * (FOLLOW_T / 4) + q], __byte_perm(w0, w1, sel)) + sad;
                w0 = w1;
            }
        }
        s_sad[o] = (int)sad;
        const int dx = wx - R, dy = wy - R;
        const unsigned long long key = ((unsigned long long)sad << 20) | ((unsigned long long)(abs(dx) + abs(dy)) << 14) |
                                       ((unsigned long long)k << 12) | ((unsigned long long)wy << 6) | (unsigned long long)wx;
        best = min(best, key);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) s_key[tid >> 5] = best;
    __syncthreads();
    best = s_key[0];
#pragma unroll
    for (int w = 1; w < FOLLOW_THREADS / 32; w++) best = min(best, s_key[w]);
    return best;
}

// The chosen candidate of a minimum key: scale k and window offset (wy, wx), dy = wy - R and dx = wx - R.
struct SearchPick {
    int k, wy, wx;
};
__device__ __forceinline__ SearchPick search_pick(unsigned long long best) {
    return SearchPick{(int)(best >> 12) & 3, (int)(best >> 6) & 63, (int)best & 63};
}

// Every thread: the chosen candidate's INSIDE pixels added to *s_inside (zeroed before; read after a barrier).
__device__ __forceinline__ void search_inside(const uint8_t (*s_in)[FOLLOW_WIN][FOLLOW_WIN], const SearchPick &c, int *s_inside, int tid) {
    int in = 0;
    for (int p = tid; p < FOLLOW_BYTES; p += FOLLOW_THREADS) in += s_in[c.k][c.wy + p / FOLLOW_T][c.wx + p % FOLLOW_T];
    if (in) atomicAdd(s_inside, in);
}

// The chosen candidate's offset, SAD, sub-pixel step and box (one thread).
struct SearchHit {
    int dx, dy, sad;
    bool border;
    double fx, fy, ncx, ncy, nw, nh;
};

__device__ __forceinline__ SearchHit search_hit(const int *s_sad, const double (*s_g)[4], const SearchPick &p, int R, int side, int nc, double pcx,
                                                double pcy, double pw, double ph) {
    SearchHit o;
    const int dx = p.wx - R, dy = p.wy - R, c = p.k * nc + p.wy * side + p.wx, s0 = s_sad[c];
    const bool border = abs(dx) == R || abs(dy) == R;
    double fx = 0.0, fy = 0.0;
    if (!border) {
        const int xm = s_sad[c - 1], xp = s_sad[c + 1], ym = s_sad[c - side], yp = s_sad[c + side];
        const int dnx = 2 * (xm - 2 * s0 + xp), dny = 2 * (ym - 2 * s0 + yp);
        if (dnx != 0) fx = (double)(xm - xp) / (double)dnx;
        if (dny != 0) fy = (double)(ym - yp) / (double)dny;
    }
    o.dx = dx;
    o.dy = dy;
    o.sad = s0;
    o.border = border;
    o.fx = fx;
    o.fy = fy;
    o.ncx = pcx + ((double)dx + fx) * s_g[p.k][0];
    o.ncy = pcy + ((double)dy + fy) * s_g[p.k][1];
    o.nw = pw * scale_of(p.k);
    o.nh = ph * scale_of(p.k);
    return o;
}

// The Status of a searched box.  flat: the template's FLAT test; empty: the box, rounded to float, has no positive width or height
// (the caller tests it where k_follow_search always has, so that kernel compiles as it did before the search moved here).
template <class Flat>
__device__ __forceinline__ int search_status(const Flat &flat, int inside, const SearchHit &s, float max_mad, bool empty) {
    return flat                                                               ? RF_FOLLOW_FLAT
           : 4 * inside < 3 * FOLLOW_BYTES                                    ? RF_FOLLOW_OUTSIDE
           : s.border                                                         ? RF_FOLLOW_BORDER
           : (double)s.sad > (double)max_mad * (double)FOLLOW_BYTES || empty ? RF_FOLLOW_MISMATCH
                                                                              : RF_FOLLOW_OK;
}

}  // namespace rf
