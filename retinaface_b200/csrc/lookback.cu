// lookback.cu -- see lookback.cuh.  Compiled with -fmad=false: the look-back box is FP64 with one rounding per step, as rf_b200.h and
// oracle/lookback.py state it.
#include <algorithm>

#include "lookback.cuh"

namespace rf {

namespace {

static_assert(sizeof(LookbackArgs) + sizeof(LookbackLogTable) + 32 <= 4096, "k_lookback_log exceeds the classic 4 KB parameter space");
static_assert(sizeof(LookbackArgs) + sizeof(LookbackBoxTable) + 32 <= 4096, "k_lookback_boxes exceeds the classic 4 KB parameter space");
static_assert(sizeof(LookbackSwapTable) + 32 <= 4096, "k_lookback_swap exceeds the classic 4 KB parameter space");
static_assert(sizeof(LookbackHead) % 16 == 0, "the boxes after the head are float4");

constexpr int SWAP_ROWS = LOOKBACK_THREADS / 32;     // one warp per plane row
constexpr int SWAP_UNROLL = 4;                       // 16-byte chunks in flight per thread

__host__ __device__ __forceinline__ size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Exclusive block scan of a 0/1 flag over LOOKBACK_THREADS threads; *total receives the count.  Every thread of the CTA calls it.
__device__ int flag_scan(bool v, int *total, int *s_w) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned b = __ballot_sync(0xffffffffu, v);
    if (lane == 0) s_w[warp] = __popc(b);
    __syncthreads();
    int pre = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < LOOKBACK_THREADS / 32; w++) {
        if (w < warp) pre += s_w[w];
        tot += s_w[w];
    }
    __syncthreads();
    *total = tot;
    return pre + __popc(b & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(LOOKBACK_THREADS) k_lookback_log(const LookbackArgs a, const __grid_constant__ LookbackLogTable t) {
    __shared__ int s_w[2][LOOKBACK_THREADS / 32];
    const int k = blockIdx.x, i = t.i0 + k;
    uint8_t *slot = t.slot[k];
    float4 *ab = const_cast<float4 *>(slot_boxes(slot));
    LookbackBirth *births = const_cast<LookbackBirth *>(slot_births(slot, a.max_faces, a.max_tracks));
    const int bcap = min(a.max_faces, a.max_tracks);
    const int na = min(max(a.counts[i], 0), t.per_frame);
    const float sc = t.scale[k];
    for (int j = threadIdx.x; j < na; j += LOOKBACK_THREADS) {      // (a): f12's map-back
        const rf_face &f = a.dets[(size_t)i * t.per_frame + j].face;
        ab[j] = make_float4(__fmul_rn(f.x1, sc), __fmul_rn(f.y1, sc), __fmul_rn(f.x2, sc), __fmul_rn(f.y2, sc));
    }
    const int nt = min(max(a.track_counts[i], 0), a.max_tracks);
    int run_l = 0, run_b = 0;
    for (int q0 = 0; q0 < nt; q0 += LOOKBACK_THREADS) {           // (b) and the births, in list (id) order
        const int q = q0 + threadIdx.x;
        const rf_track *tr = q < nt ? a.tracks + (size_t)i * a.max_tracks + q : nullptr;
        const bool lost = tr && tr->state == RF_TRACK_LOST, born = tr && tr->age == 1;
        int tl, tb;
        const int pl = flag_scan(lost, &tl, s_w[0]), pb = flag_scan(born, &tb, s_w[1]);
        if (lost) ab[na + run_l + pl] = make_float4(tr->kx1, tr->ky1, tr->kx2, tr->ky2);
        if (born && run_b + pb < bcap) births[run_b + pb] = LookbackBirth{tr->id, tr->face.x1, tr->face.y1, tr->face.x2, tr->face.y2};
        run_l += tl;
        run_b += tb;
    }
    if (threadIdx.x == 0) {
        LookbackHead hd{};
        hd.nab = na + run_l;
        hd.nbirth = min(run_b, bcap);
        hd.status = a.motion ? a.motion[i].status : RF_MOTION_FIRST;
        for (int c = 0; c < 6; c++) hd.m[c] = a.motion ? a.motion[i].m[c] : 0.0;
        *reinterpret_cast<LookbackHead *>(slot) = hd;
    }
}

__global__ void __launch_bounds__(LOOKBACK_THREADS) k_lookback_boxes(const LookbackArgs a, const __grid_constant__ LookbackBoxTable t) {
    __shared__ int s_first[LOOKBACK_MAX_L + 1];
    const int k = blockIdx.x, span = t.span[k];
    const uint8_t *log = t.log[k];
    auto slot_of = [&](int d) { return log + (size_t)((t.e_slot[k] + d) % a.ring) * a.slot_bytes; };
    const uint8_t *se = slot_of(0);
    const int nab = reinterpret_cast<const LookbackHead *>(se)->nab;
    rf_det *out = a.out + (size_t)(t.j0 + k) * a.records;
    const float4 *ab = slot_boxes(se);
    for (int j = threadIdx.x; j < nab; j += LOOKBACK_THREADS) {
        const float4 b = ab[j];
        rf_det r{};
        r.face.score = 1.f;
        r.face.x1 = b.x;
        r.face.y1 = b.y;
        r.face.x2 = b.z;
        r.face.y2 = b.w;
        r.anchor_index = -1;
        out[j] = r;
    }
    // s_first[d - 1]: the first birth of frame e + d among the frame's (c) boxes; the heads are read in parallel, then summed
    if (threadIdx.x < span) s_first[threadIdx.x + 1] = reinterpret_cast<const LookbackHead *>(slot_of(threadIdx.x + 1))->nbirth;
    __syncthreads();
    if (threadIdx.x == 0) {
        s_first[0] = 0;
        for (int d = 1; d <= span; d++) s_first[d] += s_first[d - 1];
    }
    __syncthreads();
    const int nb = s_first[span];
    for (int q = threadIdx.x; q < nb; q += LOOKBACK_THREADS) {
        int d = 1;
        while (d < span && s_first[d] <= q) d++;
        const LookbackBirth bb = slot_births(slot_of(d), a.max_faces, a.max_tracks)[q - s_first[d - 1]];
        const double x1 = bb.x1, y1 = bb.y1, x2 = bb.x2, y2 = bb.y2;
        double w = x2 - x1, h = y2 - y1;
        double cx = x1 + w / 2.0, cy = y1 + h / 2.0;
        for (int f = d; f >= 1; f--) {     // frames b, b - 1, ..., e + 1: each motion undone
            const LookbackHead *m = reinterpret_cast<const LookbackHead *>(slot_of(f));
            if (m->status != RF_MOTION_OK) continue;
            const double A = m->m[0], B = m->m[3], tx = m->m[2], ty = m->m[5];
            const double s2 = A * A + B * B, dx = cx - tx, dy = cy - ty;
            cx = (A * dx + B * dy) / s2;
            cy = (A * dy - B * dx) / s2;
            const double s = sqrt(s2);
            w = w / s;
            h = h / s;
        }
        const double g = 0.5 + a.grow * (double)d, ex = g * w, ey = g * h;
        rf_det r{};
        r.face.score = 1.f;
        r.face.x1 = (float)(cx - ex);
        r.face.y1 = (float)(cy - ey);
        r.face.x2 = (float)(cx + ex);
        r.face.y2 = (float)(cy + ey);
        r.anchor_index = -1;
        out[nab + q] = r;
    }
    int nd = 0;
    if (a.search) {      // f17 (d): the same births in the same order, each with its step d's box when the chain reached it OK
        __shared__ int s_w[LOOKBACK_THREADS / 32];
        for (int q0 = 0; q0 < nb; q0 += LOOKBACK_THREADS) {
            const int q = q0 + threadIdx.x;
            int d = 1;
            while (d < span && s_first[d] <= q) d++;
            const uint8_t *sb = slot_of(d);
            const int rk = q - s_first[d - 1];
            const bool ok = q < nb && d <= slot_nok(sb, a.max_faces, a.max_tracks, a.L)[rk];
            int tot;
            const int pos = flag_scan(ok, &tot, s_w);
            if (ok) {
                const float4 b = slot_chain(sb, a.max_faces, a.max_tracks)[(size_t)rk * a.L + d - 1];
                rf_det r{};
                r.face.score = 1.f;
                r.face.x1 = b.x;
                r.face.y1 = b.y;
                r.face.x2 = b.z;
                r.face.y2 = b.w;
                r.anchor_index = -1;
                out[nab + nb + nd + pos] = r;
            }
            nd += tot;
        }
    }
    if (threadIdx.x == 0) a.out_counts[t.j0 + k] = nab + nb + nd;
}

// One warp per plane row (luma rows, then the chroma rows: one interleaved plane, or U then V).  A thread owns the same bytes of the
// slot, the input and the out frame: the slot's old bytes are loaded with the input's before either store.
__global__ void __launch_bounds__(LOOKBACK_THREADS) k_lookback_swap(const __grid_constant__ LookbackSwapTable t) {
    const LookbackSwapFrame &f = t.f[blockIdx.y];
    const int r = blockIdx.x * SWAP_ROWS + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    const int ch = f.h / 2;
    if (r >= f.h + (f.planar ? 2 * ch : ch)) return;
    const uint8_t *in;
    uint8_t *out, *buf;
    int len;
    if (r < f.h) {
        len = f.w;
        in = f.in[0] ? f.in[0] + (size_t)r * f.in_pitch[0] : nullptr;
        out = f.out[0] ? f.out[0] + (size_t)r * f.out_pitch[0] : nullptr;
        buf = f.slot + (size_t)r * f.w;
    } else if (!f.planar) {
        const int c = r - f.h;
        len = f.w;
        in = f.in[1] ? f.in[1] + (size_t)c * f.in_pitch[1] : nullptr;
        out = f.out[1] ? f.out[1] + (size_t)c * f.out_pitch[1] : nullptr;
        buf = f.slot + (size_t)f.w * f.h + (size_t)c * f.w;
    } else {
        const bool v = r - f.h >= ch;
        const int c = r - f.h - (v ? ch : 0), cw = f.w / 2;
        const uint8_t *ip = v ? f.in_v : f.in[1];
        uint8_t *op = v ? f.out_v : f.out[1];
        len = cw;
        in = ip ? ip + (size_t)c * f.in_pitch[1] : nullptr;
        out = op ? op + (size_t)c * f.out_pitch[1] : nullptr;
        buf = f.slot + (size_t)f.w * f.h + (v ? (size_t)cw * ch : 0) + (size_t)c * cw;
    }
    const bool vec = (((uintptr_t)in | (uintptr_t)out | (uintptr_t)buf) & 15) == 0;
    const int nchunks = (len + 15) >> 4;
    for (int c0 = lane; c0 < nchunks; c0 += 32 * SWAP_UNROLL) {
        uint4 old[SWAP_UNROLL], neu[SWAP_UNROLL];
#pragma unroll
        for (int u = 0; u < SWAP_UNROLL; u++) {
            const int c = c0 + 32 * u;
            if (vec && 16 * c + 16 <= len) {
                if (out) old[u] = *reinterpret_cast<const uint4 *>(buf + 16 * c);
                if (in) neu[u] = *reinterpret_cast<const uint4 *>(in + 16 * c);
            }
        }
#pragma unroll
        for (int u = 0; u < SWAP_UNROLL; u++) {
            const int c = c0 + 32 * u;
            if (c >= nchunks) continue;
            if (vec && 16 * c + 16 <= len) {
                if (out) *reinterpret_cast<uint4 *>(out + 16 * c) = old[u];
                if (in) *reinterpret_cast<uint4 *>(buf + 16 * c) = neu[u];
            } else {          // an unaligned row or its last partial chunk: byte by byte
                for (int b = 16 * c; b < min(16 * c + 16, len); b++) {
                    const uint8_t o = buf[b];
                    const uint8_t v = in ? in[b] : 0;
                    if (out) out[b] = o;
                    if (in) buf[b] = v;
                }
            }
        }
    }
}

}  // namespace

size_t lookback_slot_bytes(int max_faces, int max_tracks, int search_L) {
    const size_t bcap = std::min(max_faces, max_tracks);
    if (search_L) return align256(lookback_chain_offset(max_faces, max_tracks) + bcap * search_L * sizeof(float4) + bcap * sizeof(int));
    return align256(sizeof(LookbackHead) + sizeof(float4) * (max_faces + max_tracks) + sizeof(LookbackBirth) * bcap);
}

cudaError_t launch_lookback_log(const LookbackArgs &a, const LookbackLogTable &t, cudaStream_t s) {
    k_lookback_log<<<t.n, LOOKBACK_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

cudaError_t launch_lookback_swap(const LookbackSwapTable &t, int max_rows, cudaStream_t s) {
    k_lookback_swap<<<dim3((max_rows + SWAP_ROWS - 1) / SWAP_ROWS, t.n), LOOKBACK_THREADS, 0, s>>>(t);
    return cudaGetLastError();
}

cudaError_t launch_lookback_boxes(const LookbackArgs &a, const LookbackBoxTable &t, cudaStream_t s) {
    k_lookback_boxes<<<t.n, LOOKBACK_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

}  // namespace rf
