// redact.cu -- see redact.cuh.  Compiled with -fmad=false: the region geometry is FP64 with one rounding per step, as rf_b200.h and
// oracle/redact.py state it (margin * w, then the subtraction).
#include <algorithm>

#include "redact.cuh"

namespace rf {

namespace {

// Lower-index rectangles an apply item keeps in shared memory; an item overlapped by more of them scans the region table instead.
constexpr int REDACT_COVER = 512;

template <typename D>
struct RedactTable {
    using Dst = D;
    static constexpr int kMax = redact_table_limit<D>();
    RedactFrameT<D> f[kMax];
};
static_assert(sizeof(RedactArgs) + sizeof(RedactTable<YuvPlanesW>) + 32 <= 4096 && sizeof(RedactArgs) + sizeof(RedactTable<BgrRowsW>) + 32 <= 4096 &&
              sizeof(RedactArgs) + sizeof(RedactTable<YuvPlanesWO>) + 32 <= 4096,
              "redact launch exceeds the classic 4 KB kernel parameter space");

// f20: the oriented instantiation (YuvPlanesWO) addresses its planes with signed strides; the stored layouts keep size_t offsets.
template <typename Dst> constexpr bool kOrientedDst = std::is_same<Dst, YuvPlanesWO>::value;
template <typename Dst> using OffT = typename std::conditional<kOrientedDst<Dst>, long long, size_t>::type;
// Displayed luma / chroma sample (x, y): its byte offset from the plane pointer.
__device__ __forceinline__ size_t luma_off(const YuvPlanesW &p, int x, int y) { return (size_t)y * p.y_pitch + x; }
__device__ __forceinline__ long long luma_off(const YuvPlanesWO &p, int x, int y) { return (long long)y * p.y_ys + (long long)x * p.y_xs; }
__device__ __forceinline__ size_t chroma_off(const YuvPlanesW &p, int x, int y) { return (size_t)y * p.uv_pitch + (size_t)x * p.uv_step; }
__device__ __forceinline__ long long chroma_off(const YuvPlanesWO &p, int x, int y) { return (long long)y * p.c_ys + (long long)x * p.c_xs; }
// Whether displayed rows run down stored columns (a transposed orientation): the apply kernel then walks its bands column by column.
__device__ __forceinline__ bool transposed(const YuvPlanesW &) { return false; }
__device__ __forceinline__ bool transposed(const YuvPlanesWO &p) { return p.y_xs != 1 && p.y_xs != -1; }

// Exclusive block scan of v over REDACT_THREADS threads; *total receives the sum.  Every thread of the CTA calls it.
__device__ int block_scan(int v, int *total, int *s_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    int pre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < REDACT_THREADS / 32; w++) {
        if (w < warp) pre += s_w[w];
        tot += s_w[w];
    }
    __syncthreads();
    *total = tot;
    return pre + incl - v;
}

// Blur work items: strips of BLUR_W output columns x bands of BLUR_H rows.  s_v holds a band's vertical sums for its strip and the
// strip's 3a-column halo on each side at a <= 127; its row stride is odd, so that one thread per row reads it without bank conflicts.
constexpr int BLUR_W = 32, BLUR_H = 32, BLUR_STRIDE = BLUR_W + 6 * BLUR_MAX_RADIUS + 1, BLUR_COVER = 128;
constexpr size_t BLUR_SMEM = sizeof(uint32_t) * BLUR_H * BLUR_STRIDE;
constexpr int BLUR_UNROLL = 8;
__host__ __device__ __forceinline__ int blur_items(int cw, int ch) { return ((cw + BLUR_W - 1) / BLUR_W) * ((ch + BLUR_H - 1) / BLUR_H); }

// The header's ellipse test of plane sample (x, y) in [x0, x1) x [y0, y1): u^2 H^2 + v^2 W^2 <= W^2 H^2 in exact integers.  With the
// +-65536 clamp W^2 H^2 reaches about 3e20, so the products are 128-bit; |u| < W and |v| < H keep u^2 and v^2 in 64 bits.
__device__ __forceinline__ bool in_ellipse(int x0, int y0, int x1, int y1, int x, int y) {
    using u128 = unsigned __int128;
    const long long W = x1 - x0, H = y1 - y0, u = 2LL * x + 1 - x0 - x1, v = 2LL * y + 1 - y0 - y1;
    const unsigned long long W2 = W * W, H2 = H * H;
    return (u128)(unsigned long long)(u * u) * H2 + (u128)(unsigned long long)(v * v) * W2 <= (u128)W2 * H2;
}

// Whether the shape of a region with luma rectangle o = (x0, y0, x1, y1) covers sample (x, y) of a plane subsampled by 2^s (the
// rectangle halved for chroma; every bound is even).  RECT is f12's test, unchanged.
template <bool kEllipse>
__device__ __forceinline__ bool shape_covers(int4 o, int s, int x, int y) {
    if constexpr (!kEllipse) {
        const int X = x << s, Y = y << s;
        return X >= o.x && X < o.z && Y >= o.y && Y < o.w;
    } else {
        const int x0 = o.x >> s, y0 = o.y >> s, x1 = o.z >> s, y1 = o.w >> s;
        return x >= x0 && x < x1 && y >= y0 && y < y1 && in_ellipse(x0, y0, x1, y1, x, y);
    }
}

// The header's geometry of one box in frame pixels; false: the box is skipped.  mi / ai: the region's measure and apply items (0
// when its rectangle misses the frame).  The clamps beyond +-65536 keep the integers in range without changing any non-empty
// rectangle: a bound past them already makes the rectangle empty.
__device__ bool region_geometry(float fx1, float fy1, float fx2, float fy2, double margin, int blocks, int W, int H, RedactRegion &g, int &mi,
                                int &ai, int kind, int detail, bool yuv) {
    if (!(isfinite(fx1) && isfinite(fy1) && isfinite(fx2) && isfinite(fy2))) return false;
    const double x1 = fx1, y1 = fy1, x2 = fx2, y2 = fy2;
    const double w = x2 - x1, h = y2 - y1;
    if (!(w > 0.0) || !(h > 0.0)) return false;
    const double mx = margin * w, my = margin * h;
    g.x0 = (int)floor(fmin(fmax(x1 - mx, -65536.0), 65538.0)) & ~1;
    g.y0 = (int)floor(fmin(fmax(y1 - my, -65536.0), 65538.0)) & ~1;
    g.x1 = ((int)floor(fmax(fmin(x2 + mx, 65536.0), -65538.0)) + 2) & ~1;    // 2 ceil((floor(.) + 1) / 2)
    g.y1 = ((int)floor(fmax(fmin(y2 + my, 65536.0), -65538.0)) + 2) & ~1;
    const int D = max(g.x1 - g.x0, g.y1 - g.y0);
    g.c = D > 0 ? 2 * ((D + 2 * blocks - 1) / (2 * blocks)) : 2;
    g.nx = g.x1 > g.x0 ? (g.x1 - g.x0 + g.c - 1) / g.c : 0;
    g.cr0 = 0;
    mi = ai = 0;
    const int cx0 = max(g.x0, 0), cx1 = min(g.x1, W), cy0 = max(g.y0, 0), cy1 = min(g.y1, H);
    if (cx0 < cx1 && cy0 < cy1) {
        g.cr0 = (cy0 - g.y0) / g.c;
        mi = (cy1 - 1 - g.y0) / g.c - g.cr0 + 1;
        ai = (cy1 - cy0 + REDACT_BAND - 1) / REDACT_BAND;
        if (kind == REDACT_BLUR)      // blur items: every plane's strips x bands (YUV: luma, then U and V halved; BGR: one per channel)
            mi = yuv ? blur_items(cx1 - cx0, cy1 - cy0) + 2 * blur_items((cx1 - cx0) >> 1, (cy1 - cy0) >> 1) : 3 * blur_items(cx1 - cx0, cy1 - cy0);
    }
    g.rad = kind == REDACT_BLUR ? min(max(D > 0 ? (D + 2 * detail - 1) / (2 * detail) : 0, 1), BLUR_MAX_RADIUS) : 0;
    return true;
}

template <typename Table>
__global__ void __launch_bounds__(REDACT_THREADS) k_redact_regions(const RedactArgs a, const __grid_constant__ Table table) {
    __shared__ int s_w[3][REDACT_THREADS / 32];
    constexpr bool kYuv = kRedactYuv<typename Table::Dst>;
    const int i = blockIdx.x;
    const auto &fr = table.f[i];
    const int na = min(max(a.counts[i], 0), a.max_faces);
    const int nb = a.tracks ? min(max(a.track_counts[i], 0), a.max_tracks) : 0;
    int run_r = 0, run_m = 0, run_a = 0;
    for (int k0 = 0; k0 < na + nb; k0 += REDACT_THREADS) {
        const int k = k0 + threadIdx.x;
        bool ok = false;
        RedactRegion g{};
        int mi = 0, ai = 0;
        if (k < na) {
            const rf_face &f = a.dets[(size_t)i * a.max_faces + k].face;
            ok = region_geometry(__fmul_rn(f.x1, fr.scale), __fmul_rn(f.y1, fr.scale), __fmul_rn(f.x2, fr.scale), __fmul_rn(f.y2, fr.scale), a.margin,
                                 a.blocks, fr.w, fr.h, g, mi, ai, a.kind, a.detail, kYuv);
        } else if (k < na + nb) {
            const rf_track &t = a.tracks[(size_t)i * a.max_tracks + (k - na)];
            ok = t.state == RF_TRACK_LOST && region_geometry(t.kx1, t.ky1, t.kx2, t.ky2, a.margin, a.blocks, fr.w, fr.h, g, mi, ai, a.kind, a.detail, kYuv);
        }
        int tr, tm, ta;
        const int pr = block_scan(ok ? 1 : 0, &tr, s_w[0]);
        const int pm = block_scan(ok ? mi : 0, &tm, s_w[1]);
        const int pa = block_scan(ok ? ai : 0, &ta, s_w[2]);
        if (ok) {
            g.m_first = run_m + pm;
            g.a_first = run_a + pa;
            a.regions[(size_t)i * a.cap + run_r + pr] = g;
        }
        run_r += tr;
        run_m += tm;
        run_a += ta;
    }
    if (threadIdx.x == 0) *reinterpret_cast<int4 *>(a.totals + 4 * i) = make_int4(run_r, run_m, run_a, 0);
}

// s_first[0..n]: the first work item of each frame (column `col` of the totals), s_first[n] the total.
__device__ void frame_firsts(const RedactArgs &a, int col, int *s_first) {
    if (threadIdx.x == 0) {
        int run = 0;
        for (int i = 0; i < a.n; i++) {
            s_first[i] = run;
            run += a.totals[4 * i + col];
        }
        s_first[a.n] = run;
    }
    __syncthreads();
}

// The frame of work item `item` (the last frame whose first item is <= item) and, within it, the region (the last whose first
// item, field `first`, is <= k): regions without items share the next one's first item and are never chosen.
__device__ void locate(const RedactArgs &a, const int *s_first, int item, int RedactRegion::*first, int &i, int &r, int &k) {
    int lo = 0, hi = a.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_first[mid] <= item) lo = mid; else hi = mid - 1;
    }
    i = lo;
    k = item - s_first[i];
    const RedactRegion *R = a.regions + (size_t)i * a.cap;
    lo = 0;
    hi = a.totals[4 * i] - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (R[mid].*first <= k) lo = mid; else hi = mid - 1;
    }
    r = lo;
}

// Sum of the bytes q[y * pitch], y in [y0, y1): REDACT_UNROLL independent loads in flight per step, so that a column costs a few
// memory round trips rather than one per row.
constexpr int REDACT_UNROLL = 8;
template <typename Off>
__device__ __forceinline__ unsigned column_sum(const uint8_t *q, int pitch, int y0, int y1) {
    unsigned s = 0;
    int y = y0;
    for (; y + REDACT_UNROLL <= y1; y += REDACT_UNROLL) {
        unsigned v[REDACT_UNROLL];
#pragma unroll
        for (int k = 0; k < REDACT_UNROLL; k++) v[k] = q[(Off)(y + k) * pitch];
#pragma unroll
        for (int k = 0; k < REDACT_UNROLL; k++) s += v[k];
    }
    for (; y < y1; y++) s += q[(Off)y * pitch];
    return s;
}

// One cell row of one region per work item: every thread sums a column of the row's samples inside the frame and adds the sum to
// its cell's shared accumulator; then one thread per cell writes the rounded means.
template <typename Table>
__global__ void __launch_bounds__(REDACT_THREADS) k_redact_measure(const RedactArgs a, const __grid_constant__ Table table) {
    using Dst = typename Table::Dst;
    __shared__ int s_first[Table::kMax + 1];
    __shared__ unsigned long long s_sum[3][REDACT_MAX_BLOCKS];
    constexpr bool kYuv = kRedactYuv<Dst>;
    frame_firsts(a, 1, s_first);
    const int items = s_first[a.n], bb = a.blocks * a.blocks;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        int i, r, k;
        locate(a, s_first, item, &RedactRegion::m_first, i, r, k);
        const auto &fr = table.f[i];
        const RedactRegion g = a.regions[(size_t)i * a.cap + r];
        const int c = g.c, cr = g.cr0 + (k - g.m_first);
        for (int t = threadIdx.x; t < 3 * REDACT_MAX_BLOCKS; t += REDACT_THREADS) s_sum[t / REDACT_MAX_BLOCKS][t % REDACT_MAX_BLOCKS] = 0;
        __syncthreads();
        const int cx0 = max(g.x0, 0), cx1 = min(g.x1, fr.w);
        const int ry0 = max(g.y0 + cr * c, 0), ry1 = min(min(g.y0 + (cr + 1) * c, g.y1), fr.h);
        if constexpr (kOrientedDst<Dst>) {
            // f20: down a displayed column by y_ys / c_ys, across by y_xs / c_xs; the sums and cells are those of the upright frame
            const YuvPlanesWO &p = fr.dst;
            for (int x = cx0 + threadIdx.x; x < cx1; x += REDACT_THREADS) {
                const unsigned s = column_sum<long long>(p.y + (long long)x * p.y_xs, p.y_ys, ry0, ry1);
                atomicAdd(&s_sum[0][(x - g.x0) / c], (unsigned long long)s);
            }
            for (int x = (cx0 >> 1) + threadIdx.x; x < (cx1 >> 1); x += REDACT_THREADS) {
                const long long o = (long long)x * p.c_xs;
                const unsigned su = column_sum<long long>(p.u + o, p.c_ys, ry0 >> 1, ry1 >> 1), sv = column_sum<long long>(p.v + o, p.c_ys, ry0 >> 1, ry1 >> 1);
                const int cell = (2 * x - g.x0) / c;
                atomicAdd(&s_sum[1][cell], (unsigned long long)su);
                atomicAdd(&s_sum[2][cell], (unsigned long long)sv);
            }
        } else if constexpr (kYuv) {
            const YuvPlanesW &p = fr.dst;
            for (int x = cx0 + threadIdx.x; x < cx1; x += REDACT_THREADS) {
                const unsigned s = column_sum<size_t>(p.y + x, p.y_pitch, ry0, ry1);
                atomicAdd(&s_sum[0][(x - g.x0) / c], (unsigned long long)s);
            }
            // chroma: the rectangle and the row halved (every bound is even), cells of side c / 2 anchored at (x0 / 2, y0 / 2)
            for (int x = (cx0 >> 1) + threadIdx.x; x < (cx1 >> 1); x += REDACT_THREADS) {
                const size_t o = (size_t)x * p.uv_step;
                const unsigned su = column_sum<size_t>(p.u + o, p.uv_pitch, ry0 >> 1, ry1 >> 1), sv = column_sum<size_t>(p.v + o, p.uv_pitch, ry0 >> 1, ry1 >> 1);
                const int cell = (2 * x - g.x0) / c;
                atomicAdd(&s_sum[1][cell], (unsigned long long)su);
                atomicAdd(&s_sum[2][cell], (unsigned long long)sv);
            }
        } else {
            const BgrRowsW &p = fr.dst;
            for (int x = cx0 + threadIdx.x; x < cx1; x += REDACT_THREADS) {
                const uint8_t *q = p.p + 3 * (size_t)x;
                const unsigned s0 = column_sum<size_t>(q, p.pitch, ry0, ry1), s1 = column_sum<size_t>(q + 1, p.pitch, ry0, ry1),
                               s2 = column_sum<size_t>(q + 2, p.pitch, ry0, ry1);
                const int cell = (x - g.x0) / c;
                atomicAdd(&s_sum[0][cell], (unsigned long long)s0);
                atomicAdd(&s_sum[1][cell], (unsigned long long)s1);
                atomicAdd(&s_sum[2][cell], (unsigned long long)s2);
            }
        }
        __syncthreads();
        uint8_t *out = a.cells + ((size_t)i * a.cap + r) * bb * 3 + (size_t)cr * g.nx * 3;
        for (int cx = threadIdx.x; cx < g.nx; cx += REDACT_THREADS) {
            const int xa = max(g.x0 + cx * c, 0), xb = min(min(g.x0 + (cx + 1) * c, g.x1), fr.w);
            const unsigned long long cnt = xb > xa && ry1 > ry0 ? (unsigned long long)(xb - xa) * (ry1 - ry0) : 0;
            const unsigned long long cc = kYuv ? cnt / 4 : cnt;      // chroma: both sides halved
            out[3 * cx + 0] = cnt ? (uint8_t)((s_sum[0][cx] + cnt / 2) / cnt) : 0;
            out[3 * cx + 1] = cc ? (uint8_t)((s_sum[1][cx] + cc / 2) / cc) : 0;
            out[3 * cx + 2] = cc ? (uint8_t)((s_sum[2][cx] + cc / 2) / cc) : 0;
        }
        __syncthreads();     // the accumulators of the next item
    }
}

// The blur scratch planes of a YUV frame: plane p (0 Y, 1 U, 2 V), rows w >> s apart.
__device__ __forceinline__ uint8_t *blur_yuv_plane(uint8_t *b, int w, int h, int p) {
    return p == 0 ? b : b + (size_t)w * h + (size_t)(p - 1) * (w / 2) * (h / 2);
}

// One band of REDACT_BAND rows of one region per work item: the lower-index rectangles that reach the band go to shared memory, then
// every pixel of the band they do not cover takes its cell value -- luma first, then the band's chroma rows.  kEllipse: a sample is
// written only where the region's ellipse covers it, and only the lower-index ellipses take it away.  kBlur: the value is the
// sample's blurred value in the frame's scratch planes instead of its cell value.
template <typename Table, bool kEllipse = false, bool kBlur = false>
__global__ void __launch_bounds__(REDACT_THREADS) k_redact_apply(const RedactArgs a, const __grid_constant__ Table table) {
    using Dst = typename Table::Dst;
    __shared__ int s_first[Table::kMax + 1];
    __shared__ int4 s_rect[REDACT_COVER];
    __shared__ uint8_t s_cells[kBlur ? 1 : REDACT_MAX_BLOCKS * REDACT_MAX_BLOCKS * 3];
    __shared__ int s_nrect;
    constexpr bool kYuv = kRedactYuv<Dst>;
    frame_firsts(a, 2, s_first);
    const int items = s_first[a.n], bb = a.blocks * a.blocks;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        int i, r, k;
        locate(a, s_first, item, &RedactRegion::a_first, i, r, k);
        const auto &fr = table.f[i];
        const RedactRegion *R = a.regions + (size_t)i * a.cap;
        const RedactRegion g = R[r];
        const int c = g.c, nx = g.nx;
        const int cx0 = max(g.x0, 0), cx1 = min(g.x1, fr.w);
        const int by0 = max(g.y0, 0) + (k - g.a_first) * REDACT_BAND, by1 = min(by0 + REDACT_BAND, min(g.y1, fr.h));
        if (threadIdx.x == 0) s_nrect = 0;
        __syncthreads();
        for (int q = threadIdx.x; q < r; q += REDACT_THREADS) {
            const RedactRegion o = R[q];
            if (o.x0 < cx1 && o.x1 > cx0 && o.y0 < by1 && o.y1 > by0) {
                const int slot = atomicAdd(&s_nrect, 1);
                if (slot < REDACT_COVER) s_rect[slot] = make_int4(o.x0, o.y0, o.x1, o.y1);
            }
        }
        // the region's cell values: one round trip here instead of one per pixel below
        const uint8_t *cg = a.cells + ((size_t)i * a.cap + r) * bb * 3;
        const int ny = (g.y1 - g.y0 + c - 1) / c;
        if constexpr (!kBlur)
            for (int t = threadIdx.x; t < nx * ny * 3; t += REDACT_THREADS) s_cells[t] = cg[t];
        __syncthreads();
        const int nrect = s_nrect;
        const int4 own = make_int4(g.x0, g.y0, g.x1, g.y1);
        // (x, y): a sample of a plane subsampled by 2^s; true when the sample is not this region's to write
        auto covered = [&](int x, int y, int s) {
            if (kEllipse && !shape_covers<true>(own, s, x, y)) return true;
            if (nrect <= REDACT_COVER) {
                for (int j = 0; j < nrect; j++)
                    if (shape_covers<kEllipse>(s_rect[j], s, x, y)) return true;
                return false;
            }
            for (int q = 0; q < r; q++) {
                const RedactRegion &o = R[q];
                if (shape_covers<kEllipse>(make_int4(o.x0, o.y0, o.x1, o.y1), s, x, y)) return true;
            }
            return false;
        };
        const uint8_t *cv = s_cells;
        const int bw = cx1 - cx0, rows = by1 - by0;
        if constexpr (kYuv) {
            const Dst &p = fr.dst;
            // f20: down the band's columns when they are stored rows, so that consecutive threads write consecutive bytes
            const bool down = transposed(p);
            for (int t = threadIdx.x; t < rows * bw; t += REDACT_THREADS) {
                const int y = down ? by0 + t % rows : by0 + t / bw, x = down ? cx0 + t / rows : cx0 + t % bw;
                if (covered(x, y, 0)) continue;
                p.y[luma_off(p, x, y)] = kBlur ? fr.blur[(size_t)y * fr.w + x] : cv[((y - g.y0) / c * nx + (x - g.x0) / c) * 3];
            }
            const int hw = bw >> 1, hr = rows >> 1;
            for (int t = threadIdx.x; t < hr * hw; t += REDACT_THREADS) {
                const int y = (by0 >> 1) + (down ? t % hr : t / hw), x = (cx0 >> 1) + (down ? t / hr : t % hw);
                if (covered(x, y, 1)) continue;
                const auto o = chroma_off(p, x, y);
                if constexpr (kBlur) {
                    const size_t b = (size_t)y * (fr.w / 2) + x;
                    p.u[o] = blur_yuv_plane(fr.blur, fr.w, fr.h, 1)[b];
                    p.v[o] = blur_yuv_plane(fr.blur, fr.w, fr.h, 2)[b];
                } else {
                    const uint8_t *v = cv + ((2 * y - g.y0) / c * nx + (2 * x - g.x0) / c) * 3;
                    p.u[o] = v[1];
                    p.v[o] = v[2];
                }
            }
        } else {
            const BgrRowsW &p = fr.dst;
            for (int t = threadIdx.x; t < rows * bw; t += REDACT_THREADS) {
                const int y = by0 + t / bw, x = cx0 + t % bw;
                if (covered(x, y, 0)) continue;
                const uint8_t *v = kBlur ? fr.blur + (size_t)y * 3 * fr.w + 3 * (size_t)x : cv + ((y - g.y0) / c * nx + (x - g.x0) / c) * 3;
                uint8_t *q = p.p + (size_t)y * p.pitch + 3 * (size_t)x;
                q[0] = v[0];
                q[1] = v[1];
                q[2] = v[2];
            }
        }
        __syncthreads();     // s_rect / s_nrect of the next item
    }
}

// One (region, plane, strip, band) per work item: the blur of the strip's output columns [tx0, tx1) over the band's rows [ty0, ty1),
// from the ORIGINAL plane, into the frame's scratch planes at every sample the region owns.  The kernel k (6a + 1 taps) is three
// boxes of n = 2a + 1, so k = (1 - z^n)^3 / (1 - z)^3: each axis is the signed combination q(t) - 3 q(t - n) + 3 q(t - 2n) - q(t - 3n)
// of the clamped samples, summed three times.  Modular arithmetic makes every step exact -- u32 vertically (a column sum is at most
// 255^4 < 2^32), u64 horizontally (S is at most 255^7 < 2^63).  Vertical first, one thread per column of the strip and its 3a-column
// halo (coalesced reads across the warp), into s_v; then one thread per row of the band along s_v.
template <typename Table, bool kEllipse>
__global__ void __launch_bounds__(REDACT_THREADS, 2) k_redact_blur(const RedactArgs a, const __grid_constant__ Table table) {
    using Dst = typename Table::Dst;
    extern __shared__ uint32_t s_v[];           // [BLUR_H][BLUR_STRIDE]
    __shared__ int s_first[Table::kMax + 1];
    __shared__ int4 s_rect[BLUR_COVER];
    __shared__ int s_nrect;
    constexpr bool kYuv = kRedactYuv<Dst>;
    frame_firsts(a, 1, s_first);
    const int items = s_first[a.n];
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        int i, r, k;
        locate(a, s_first, item, &RedactRegion::m_first, i, r, k);
        const auto &fr = table.f[i];
        const RedactRegion *R = a.regions + (size_t)i * a.cap;
        const RedactRegion g = R[r];
        const int cx0 = max(g.x0, 0), cx1 = min(g.x1, fr.w), cy0 = max(g.y0, 0), cy1 = min(g.y1, fr.h);
        int j = k - g.m_first, p = 0, s = 0;
        const int n0 = blur_items(cx1 - cx0, cy1 - cy0);
        if (j >= n0) {
            if constexpr (kYuv) {
                const int n1 = blur_items((cx1 - cx0) >> 1, (cy1 - cy0) >> 1);
                s = 1;
                p = 1 + (j - n0) / n1;
                j = (j - n0) % n1;
            } else {
                p = j / n0;
                j %= n0;
            }
        }
        const uint8_t *src;
        uint8_t *dst;
        int pitch, step, pw, ph, dpitch, dstep;
        if constexpr (kYuv) {
            const Dst &d = fr.dst;
            src = p == 0 ? d.y : p == 1 ? d.u : d.v;
            if constexpr (kOrientedDst<Dst>) {
                pitch = p ? d.c_ys : d.y_ys;
                step = p ? d.c_xs : d.y_xs;
            } else {
                pitch = p ? d.uv_pitch : d.y_pitch;
                step = p ? d.uv_step : 1;
            }
            pw = fr.w >> s;
            ph = fr.h >> s;
            dst = blur_yuv_plane(fr.blur, fr.w, fr.h, p);
            dpitch = pw;
            dstep = 1;
        } else {
            src = fr.dst.p + p;
            pitch = fr.dst.pitch;
            step = 3;
            pw = fr.w;
            ph = fr.h;
            dst = fr.blur + p;
            dpitch = 3 * fr.w;
            dstep = 3;
        }
        const int ra = s ? (g.rad + 1) >> 1 : g.rad, n = 2 * ra + 1, h3 = 3 * ra;
        const int px0 = cx0 >> s, px1 = cx1 >> s, py0 = cy0 >> s, py1 = cy1 >> s;
        const int ns = (px1 - px0 + BLUR_W - 1) / BLUR_W;
        const int tx0 = px0 + (j % ns) * BLUR_W, tx1 = min(tx0 + BLUR_W, px1);
        const int ty0 = py0 + (j / ns) * BLUR_H, ty1 = min(ty0 + BLUR_H, py1);
        if (threadIdx.x == 0) s_nrect = 0;
        __syncthreads();
        const int lx0 = tx0 << s, lx1 = tx1 << s, ly0 = ty0 << s, ly1 = ty1 << s;
        for (int q = threadIdx.x; q < r; q += REDACT_THREADS) {
            const RedactRegion o = R[q];
            if (o.x0 < lx1 && o.x1 > lx0 && o.y0 < ly1 && o.y1 > ly0) {
                const int slot = atomicAdd(&s_nrect, 1);
                if (slot < BLUR_COVER) s_rect[slot] = make_int4(o.x0, o.y0, o.x1, o.y1);
            }
        }
        const int tw = tx1 - tx0, th = ty1 - ty0, cols = tw + 2 * h3, lv = th + 2 * h3;
        // vertical: s_v[y][c] = sum_j k[j] P[clampY(ty0 + y + j)][clampX(tx0 - 3a + c)]
        // BLUR_UNROLL steps' loads are issued before their sums (the row index is clamped, so every load is in the plane)
        for (int c = threadIdx.x; c < cols; c += REDACT_THREADS) {
            using Off = OffT<Dst>;
            const uint8_t *col = src + (Off)min(max(tx0 - h3 + c, 0), pw - 1) * step;
            const int ys = ty0 - h3;
            auto q = [&](int t) -> unsigned { return t >= 0 ? (unsigned)__ldg(col + (Off)min(max(ys + t, 0), ph - 1) * pitch) : 0u; };
            unsigned c1 = 0, c2 = 0, c3 = 0;
            for (int t0 = 0; t0 < lv; t0 += BLUR_UNROLL) {
                unsigned d[BLUR_UNROLL];
#pragma unroll
                for (int u = 0; u < BLUR_UNROLL; u++) d[u] = q(t0 + u) - 3u * q(t0 + u - n) + 3u * q(t0 + u - 2 * n) - q(t0 + u - 3 * n);
#pragma unroll
                for (int u = 0; u < BLUR_UNROLL; u++) {
                    const int t = t0 + u;
                    c1 += d[u];
                    c2 += c1;
                    c3 += c2;
                    if (t >= 2 * h3 && t < lv) s_v[(t - 2 * h3) * BLUR_STRIDE + c] = c3;
                }
            }
        }
        __syncthreads();
        const int nrect = s_nrect;
        const int4 own = make_int4(g.x0, g.y0, g.x1, g.y1);
        auto owned = [&](int x, int y) {
            if (kEllipse && !shape_covers<true>(own, s, x, y)) return false;
            if (nrect <= BLUR_COVER) {
                for (int e = 0; e < nrect; e++)
                    if (shape_covers<kEllipse>(s_rect[e], s, x, y)) return false;
                return true;
            }
            for (int q = 0; q < r; q++) {
                const RedactRegion &o = R[q];
                if (shape_covers<kEllipse>(make_int4(o.x0, o.y0, o.x1, o.y1), s, x, y)) return false;
            }
            return true;
        };
        // horizontal: S = sum_i k[i] s_v[y][3a + x - tx0 + i], rounded
        // The rounding (S + half) / n^6 as an FP64 estimate corrected in integers: the quotient is at most 255 and S + half < 2^63, so
        // the estimate is within one of the exact quotient, and the two corrections make it exact.
        const unsigned long long n2 = (unsigned long long)n * n, n6 = n2 * n2 * n2, half = (n6 - 1) / 2;
        const double inv6 = 1.0 / (double)n6;
        for (int yy = threadIdx.x; yy < th; yy += REDACT_THREADS) {
            const uint32_t *row = s_v + yy * BLUR_STRIDE;
            auto q = [&](int t) -> unsigned long long { return t >= 0 && t < cols ? (unsigned long long)row[t] : 0ull; };
            unsigned long long c1 = 0, c2 = 0, c3 = 0;
            const int y = ty0 + yy;
            for (int t0 = 0; t0 < cols; t0 += BLUR_UNROLL) {
                unsigned long long d[BLUR_UNROLL];
#pragma unroll
                for (int u = 0; u < BLUR_UNROLL; u++)
                    d[u] = q(t0 + u) - 3ull * q(t0 + u - n) + 3ull * q(t0 + u - 2 * n) - q(t0 + u - 3 * n);
#pragma unroll
                for (int u = 0; u < BLUR_UNROLL; u++) {
                    const int t = t0 + u;
                    c1 += d[u];
                    c2 += c1;
                    c3 += c2;
                    if (t >= 2 * h3 && t < cols) {
                        const int x = tx0 + t - 2 * h3;
                        if (owned(x, y)) {
                            const unsigned long long v = c3 + half;
                            unsigned long long r = (unsigned long long)((double)v * inv6);
                            if (r * n6 > v) r--;
                            if ((r + 1) * n6 <= v) r++;
                            dst[(size_t)y * dpitch + (size_t)x * dstep] = (uint8_t)r;
                        }
                    }
                }
            }
        }
        __syncthreads();     // s_v, s_rect and s_nrect of the next item
    }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace

size_t redact_scratch_bytes(int n, int cap, int blocks) {
    return align256(sizeof(RedactRegion) * n * cap) + align256(sizeof(int) * 4 * n) + (size_t)n * cap * blocks * blocks * 3;
}

void redact_carve(RedactArgs &a, void *scratch) {
    unsigned char *p = static_cast<unsigned char *>(scratch);
    a.regions = reinterpret_cast<RedactRegion *>(p);
    p += align256(sizeof(RedactRegion) * a.n * a.cap);
    a.totals = reinterpret_cast<int *>(p);
    p += align256(sizeof(int) * 4 * a.n);
    a.cells = p;
}

// Two CTAs per SM for measure and apply, as k_align_faces: a batch-8 call has a few hundred items of each.
template <typename Dst>
cudaError_t launch_redact(const RedactArgs &a, const RedactFrameT<Dst> *frames, int num_sms, cudaStream_t s) {
    constexpr int kMax = redact_table_limit<Dst>();
    const size_t cells = (size_t)a.blocks * a.blocks * 3;
    if (a.kind == REDACT_BLUR) {      // s_v: above the 48 KB default
        cudaError_t e = cudaFuncSetAttribute(k_redact_blur<RedactTable<Dst>, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BLUR_SMEM);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k_redact_blur<RedactTable<Dst>, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BLUR_SMEM);
        if (e != cudaSuccess) return e;
    }
    for (int i0 = 0; i0 < a.n; i0 += kMax) {
        const int m = std::min(kMax, a.n - i0);
        RedactArgs c = a;
        c.n = m;
        c.dets = a.dets + (size_t)i0 * a.max_faces;
        c.counts = a.counts + i0;
        if (a.tracks) {
            c.tracks = a.tracks + (size_t)i0 * a.max_tracks;
            c.track_counts = a.track_counts + i0;
        }
        c.regions = a.regions + (size_t)i0 * a.cap;
        c.totals = a.totals + 4 * i0;
        c.cells = a.cells + (size_t)i0 * a.cap * cells;
        RedactTable<Dst> t{};
        for (int i = 0; i < m; i++) t.f[i] = frames[i0 + i];
        k_redact_regions<<<m, REDACT_THREADS, 0, s>>>(c, t);
        const bool ell = a.shape == REDACT_ELLIPSE;
        if (a.kind == REDACT_BLUR) {
            if (ell) k_redact_blur<RedactTable<Dst>, true><<<2 * num_sms, REDACT_THREADS, BLUR_SMEM, s>>>(c, t);
            else k_redact_blur<RedactTable<Dst>, false><<<2 * num_sms, REDACT_THREADS, BLUR_SMEM, s>>>(c, t);
            if (ell) k_redact_apply<RedactTable<Dst>, true, true><<<2 * num_sms, REDACT_THREADS, 0, s>>>(c, t);
            else k_redact_apply<RedactTable<Dst>, false, true><<<2 * num_sms, REDACT_THREADS, 0, s>>>(c, t);
        } else {
            k_redact_measure<<<2 * num_sms, REDACT_THREADS, 0, s>>>(c, t);
            if (ell) k_redact_apply<RedactTable<Dst>, true><<<2 * num_sms, REDACT_THREADS, 0, s>>>(c, t);
            else k_redact_apply<<<2 * num_sms, REDACT_THREADS, 0, s>>>(c, t);
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

template cudaError_t launch_redact<YuvPlanesW>(const RedactArgs &, const RedactFrameT<YuvPlanesW> *, int, cudaStream_t);
template cudaError_t launch_redact<BgrRowsW>(const RedactArgs &, const RedactFrameT<BgrRowsW> *, int, cudaStream_t);
template cudaError_t launch_redact<YuvPlanesWO>(const RedactArgs &, const RedactFrameT<YuvPlanesWO> *, int, cudaStream_t);

}  // namespace rf
