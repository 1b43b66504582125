// lookback_search.cu -- f17 k_lookback_search (lookback.cuh, rf_b200.h rf_tracker_set_lookback_search).  Built with -fmad=false: the
// steps are f16's template search (tsearch.cuh) and f15's motion undo, every FP64 step one rounding as oracle/lookback_search.py
// restates it.
#include <algorithm>

#include "lookback.cuh"
#include "tsearch.cuh"

namespace rf {
namespace {

static_assert(sizeof(LookbackArgs) + sizeof(LookbackSearchTable) + 32 <= 4096, "k_lookback_search exceeds the classic 4 KB parameter space");

// One CTA per (frame of the table, birth rank): the chain of the birth (rf_b200.h rf_tracker_set_lookback_search).  The template is
// cut once into shared memory; each step then runs f16's Windows, Match, Box and Status from the previous step's box, moved back by
// frame e + 1's camera motion when it is OK.
__global__ void __launch_bounds__(FOLLOW_THREADS) k_lookback_search(const LookbackArgs a, const __grid_constant__ LookbackSearchTable t) {
    __shared__ uint32_t s_win[3][FOLLOW_WIN][FOLLOW_WWORDS];
    __shared__ uint8_t s_in[3][FOLLOW_WIN][FOLLOW_WIN];
    __shared__ uint32_t s_tpl[FOLLOW_BYTES / 4];
    __shared__ int s_sad[3 * FOLLOW_MAX_SIDE * FOLLOW_MAX_SIDE];
    __shared__ unsigned long long s_key[FOLLOW_THREADS / 32];
    __shared__ double s_g[3][4];
    __shared__ unsigned long long s_sum, s_sq;
    __shared__ int s_inside;
    const LookbackSearchFrame &fr = t.f[blockIdx.y];
    const LookbackSearchVideo &v = t.v[fr.video];
    const int F = a.max_faces, T = a.max_tracks, bcap = min(F, T), L = a.L, rk = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const long long num = v.num0 + ((int)blockIdx.y - v.first);
    uint8_t *slot = const_cast<uint8_t *>(v.log) + (size_t)(num % a.ring) * a.slot_bytes;
    float4 *chain = const_cast<float4 *>(slot_chain(slot, F, T)) + (size_t)rk * L;
    int *nok = const_cast<int *>(slot_nok(slot, F, T, L)) + rk;
    rf_follow *steps = a.steps + ((size_t)fr.i * bcap + rk) * L;
    int *len = a.lengths + (size_t)fr.i * bcap + rk;
    const int K = rk < reinterpret_cast<const LookbackHead *>(slot)->nbirth ? (int)min((long long)L, num) : 0;
    if (K == 0) {                                                                 // uniform: no birth, or no frame before it
        if (tid == 0) { *len = 0; *nok = 0; }
        return;
    }
    const LookbackBirth b = slot_births(slot, F, T)[rk];
    const struct { const uint8_t *y; int pitch, w, h; } in{fr.y, fr.pitch, v.w, v.h};
    if (tid == 0) {
        rf_face face{};
        face.x1 = b.x1; face.y1 = b.y1; face.x2 = b.x2; face.y2 = b.y2;
        cut_grid(face, s_g[0]);
        s_sum = 0;
        s_sq = 0;
    }
    __syncthreads();
    cut_template(in, s_g[0], reinterpret_cast<uint8_t *>(s_tpl), &s_sum, &s_sq);
    __syncthreads();
    const bool flat = template_flat(s_sum, s_sq);
    const int R = a.search, W = FOLLOW_T + 2 * R, side = 2 * R + 1, nc = side * side;
    float x1 = b.x1, y1 = b.y1, x2 = b.x2, y2 = b.y2;
    int k = 1, ok = 0;
    for (; k <= K; k++) {
        const long long e = num - k;
        auto src = in;
        if (e >= v.num0) {
            const LookbackSearchFrame &g = t.f[v.first + (int)(e - v.num0)];
            src.y = g.y;
            src.pitch = g.pitch;
        } else {
            src.y = v.buf + (size_t)(e % L) * v.frame_bytes;
            src.pitch = v.w;
        }
        double w = (double)x2 - (double)x1, h = (double)y2 - (double)y1;
        double cx = (double)x1 + w / 2.0, cy = (double)y1 + h / 2.0;
        const LookbackHead *m = reinterpret_cast<const LookbackHead *>(v.log + (size_t)((e + 1) % a.ring) * a.slot_bytes);
        if (m->status == RF_MOTION_OK) {     // f15's step 2: frame e + 1's motion undone
            const double A = m->m[0], B = m->m[3], tx = m->m[2], ty = m->m[5];
            const double s2 = A * A + B * B, dx = cx - tx, dy = cy - ty;
            cx = (A * dx + B * dy) / s2;
            cy = (A * dy - B * dx) / s2;
            const double s = sqrt(s2);
            w = w / s;
            h = h / s;
        }
        const double pa = w / h, ph = h, pw = pa * ph;     // f10's z (cx, cy, w / h, h), searched as f16 searches a state
        rf_follow rec{};
        rec.id = b.id;
        if (!FOLLOW_SEARCH_BOUNDED(cx, cy, pw, ph)) {                             // uniform
            if (tid == 0) {
                rec.status = RF_FOLLOW_MISMATCH;
                steps[k - 1] = rec;
            }
            break;
        }
        __syncthreads();                      // the previous step's readers of s_g, s_win, s_sad and s_inside are done
        if (tid < 3) search_grid(s_g, tid, cx, cy, pw, ph, R);
        if (tid == 0) s_inside = 0;
        __syncthreads();
        search_windows(src, s_g, W, s_win, s_in, tid);
        __syncthreads();
        const unsigned long long best = search_min(s_win, s_tpl, s_sad, s_key, R, side, nc, tid, lane);
        const SearchPick pick = search_pick(best);
        search_inside(s_in, pick, &s_inside, tid);
        __syncthreads();
        const SearchHit hit = search_hit(s_sad, s_g, pick, R, side, nc, cx, cy, pw, ph);
        x1 = (float)(hit.ncx - hit.nw / 2.0);
        y1 = (float)(hit.ncy - hit.nh / 2.0);
        x2 = (float)(hit.ncx + hit.nw / 2.0);
        y2 = (float)(hit.ncy + hit.nh / 2.0);
        const bool empty = !((double)x2 - (double)x1 > 0.0) || !((double)y2 - (double)y1 > 0.0);
        rec.status = search_status(flat, s_inside, hit, a.max_mad, empty);
        if (tid == 0) {
            rec.dx = hit.dx;
            rec.dy = hit.dy;
            rec.scale = pick.k;
            rec.sad = hit.sad;
            rec.fx = (float)hit.fx;
            rec.fy = (float)hit.fy;
            rec.x1 = x1; rec.y1 = y1; rec.x2 = x2; rec.y2 = y2;
            steps[k - 1] = rec;
            if (rec.status == RF_FOLLOW_OK) chain[k - 1] = make_float4(x1, y1, x2, y2);
        }
        if (rec.status != RF_FOLLOW_OK) break;                                    // uniform
        ok = k;
    }
    if (tid == 0) {
        *len = min(k, K);
        *nok = ok;
    }
}

}  // namespace

cudaError_t launch_lookback_search(const LookbackArgs &a, const LookbackSearchTable &t, cudaStream_t s) {
    k_lookback_search<<<dim3(std::min(a.max_faces, a.max_tracks), t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

}  // namespace rf
