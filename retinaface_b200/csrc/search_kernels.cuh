// search_kernels.cuh -- the bodies of the kernels that search luma: f16's k_follow_cut and k_follow_search (follow.cu) and f17's
// k_lookback_search (lookback_search.cu), each a template on ORIENTED.  The upright kernels instantiate false in their own sources;
// f20's oriented twins (oriented_search.cu) instantiate true and read every frame as its video displays it (tsearch.cuh
// OrientedLuma).  Every FP64 step is one rounding in the order written: include it only from sources built with -fmad=false.
#pragma once
#include <type_traits>

#include "lookback.cuh"
#include "tsearch.cuh"

namespace rf {

// k_follow_cut (follow.cu) and, ORIENTED, its f20 twin (oriented_search.cu): the frame's luma read as stored, or as displayed.
template <bool ORIENTED>
__device__ __forceinline__ void follow_cut(const FollowArgs &a, const FollowTable &t) {
    __shared__ int s_slot;
    __shared__ double s_g[4];
    __shared__ unsigned long long s_sum, s_sq;
    const FollowFrame &f = t.f[blockIdx.y];
    const int T = a.p.max_tracks, tid = threadIdx.x;
    if ((int)blockIdx.x >= a.list_counts[f.frame]) return;                     // uniform
    const rf_track &tr = a.lists[(size_t)f.frame * T + blockIdx.x];
    if (tr.det < 0) return;                                                       // uniform
    if (tid == 0) {
        bool later = false;           // matched again on a later frame of the launch: that frame's cut is the one kept
        for (int g = blockIdx.y + 1; g < t.n && !later; g++) {
            if (t.f[g].video != f.video) continue;
            const rf_track *l = a.lists + (size_t)t.f[g].frame * T;
            for (int q = 0, cnt = a.list_counts[t.f[g].frame]; q < cnt; q++)
                if (l[q].id == tr.id) { later = l[q].det >= 0; break; }
        }
        int slot = -1;                // removed later in the launch: no slot
        for (int q = 0; !later && q < T; q++)
            if (a.state[(size_t)f.video * T + q].id == tr.id) { slot = q; break; }
        s_slot = slot;
        s_sum = 0;
        s_sq = 0;
        cut_grid(tr.face, s_g);
    }
    __syncthreads();
    const int slot = s_slot;
    if (slot < 0) return;                                                         // uniform
    const size_t e = (size_t)f.video * T + slot;
    if constexpr (ORIENTED) cut_template(oriented_luma(f.y, f.pitch, f.bits, f.w, f.h), s_g, a.store + e * FOLLOW_BYTES, &s_sum, &s_sq);
    else cut_template(f, s_g, a.store + e * FOLLOW_BYTES, &s_sum, &s_sq);
    __syncthreads();
    if (tid == 0) a.entries[e] = FollowEntry{tr.id, template_flat(s_sum, s_sq)};
}

// k_follow_search and its f20 twin.
template <bool ORIENTED>
__device__ __forceinline__ void follow_search(const FollowArgs &a, const FollowTable &t) {
    __shared__ uint32_t s_win[3][FOLLOW_WIN][FOLLOW_WWORDS];
    __shared__ uint8_t s_in[3][FOLLOW_WIN][FOLLOW_WIN];
    __shared__ uint32_t s_tpl[FOLLOW_BYTES / 4];
    __shared__ int s_sad[3 * FOLLOW_MAX_SIDE * FOLLOW_MAX_SIDE];
    __shared__ unsigned long long s_key[FOLLOW_THREADS / 32];
    __shared__ double s_g[3][4];
    __shared__ int s_inside;
    const FollowFrame &f = t.f[blockIdx.y];
    const int T = a.p.max_tracks, tid = threadIdx.x, lane = tid & 31;
    const size_t e = (size_t)f.video * T + blockIdx.x;
    const TrackState &S = a.state[e];
    const int id = S.id;
    if (!id || S.state == RF_TRACK_LOST) return;                                 // uniform: not searched
    FollowMeas *out = a.meas + (size_t)f.frame * T + blockIdx.x;
    // the predicted state's box: kalman_predict's mean step (the state is not LOST, so u_h stays), then kalman_motion's
    double pcx = S.m[0] + S.u[0], pcy = S.m[1] + S.u[1], ph = S.m[3] + S.u[3];
    const double pa = S.m[2] + S.u[2];
    if (a.motion && a.motion[f.frame].status == RF_MOTION_OK) {
        const double *m = a.motion[f.frame].m;
        const double ma = m[0], mb = m[3], cx = pcx, cy = pcy;
        pcx = (ma * cx - mb * cy) + m[2];
        pcy = (mb * cx + ma * cy) + m[5];
        ph = sqrt(ma * ma + mb * mb) * ph;
    }
    const double pw = pa * ph;
    const int R = a.search, W = FOLLOW_T + 2 * R, side = 2 * R + 1, nc = side * side;
    const bool bounded = FOLLOW_SEARCH_BOUNDED(pcx, pcy, pw, ph);
    if (a.entries[e].id != id || !bounded) {                                      // uniform: no template, or no search
        if (tid == 0) {
            rf_follow r{};
            r.id = id;
            r.status = bounded ? RF_FOLLOW_FLAT : RF_FOLLOW_MISMATCH;
            out->rec = r;
        }
        return;
    }
    if (tid < 3) search_grid(s_g, tid, pcx, pcy, pw, ph, R);
    if (tid == 0) s_inside = 0;
    const uint32_t *tsrc = reinterpret_cast<const uint32_t *>(a.store + e * FOLLOW_BYTES);
    for (int w = tid; w < FOLLOW_BYTES / 4; w += FOLLOW_THREADS) s_tpl[w] = tsrc[w];
    __syncthreads();
    if constexpr (ORIENTED) search_windows(oriented_luma(f.y, f.pitch, f.bits, f.w, f.h), s_g, W, s_win, s_in, tid);
    else search_windows(f, s_g, W, s_win, s_in, tid);
    __syncthreads();
    const unsigned long long best = search_min(s_win, s_tpl, s_sad, s_key, R, side, nc, tid, lane);
    const SearchPick pick = search_pick(best);
    search_inside(s_in, pick, &s_inside, tid);
    __syncthreads();
    if (tid != 0) return;
    const SearchHit h = search_hit(s_sad, s_g, pick, R, side, nc, pcx, pcy, pw, ph);
    const double ncx = h.ncx, ncy = h.ncy, nw = h.nw, nh = h.nh;
    const rf_face &o = S.face;
    rf_face nf;
    nf.score = o.score;
    nf.x1 = (float)(ncx - nw / 2.0);
    nf.y1 = (float)(ncy - nh / 2.0);
    nf.x2 = (float)(ncx + nw / 2.0);
    nf.y2 = (float)(ncy + nh / 2.0);
    const double ow = (double)o.x2 - (double)o.x1, oh = (double)o.y2 - (double)o.y1;
    const double ocx = (double)o.x1 + ow / 2.0, ocy = (double)o.y1 + oh / 2.0, sx = nw / ow, sy = nh / oh;
#pragma unroll
    for (int l = 0; l < 5; l++) {
        nf.lx[l] = (float)(ncx + ((double)o.lx[l] - ocx) * sx);
        nf.ly[l] = (float)(ncy + ((double)o.ly[l] - ocy) * sy);
    }
    rf_follow r;
    r.id = id;
    r.dx = h.dx;
    r.dy = h.dy;
    r.scale = pick.k;
    r.sad = h.sad;
    r.fx = (float)h.fx;
    r.fy = (float)h.fy;
    r.x1 = nf.x1; r.y1 = nf.y1; r.x2 = nf.x2; r.y2 = nf.y2;
    const bool empty = !((double)nf.x2 - (double)nf.x1 > 0.0) || !((double)nf.y2 - (double)nf.y1 > 0.0);
    r.status = search_status(a.entries[e].flat, s_inside, h, a.max_mad, empty);
    out->rec = r;
    out->face = nf;
}

// k_lookback_search (lookback_search.cu) and, ORIENTED, its f20 twin (oriented_search.cu), which reads every frame, input or buffered,
// as its video displays it.
template <bool ORIENTED>
__device__ __forceinline__ void lookback_search(const LookbackArgs &a, const LookbackSearchTable &t) {
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
    using Plane = typename std::conditional<ORIENTED, OrientedLuma, PitchedLuma>::type;
    Plane in;
    if constexpr (ORIENTED) in = oriented_luma(fr.y, fr.pitch, v.bits, v.w, v.h);
    else in = PitchedLuma{fr.y, fr.pitch, v.w, v.h};
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
        Plane src = in;
        if constexpr (ORIENTED) {      // a buffered frame is packed in stored geometry: rows of the stored width
            const int sw = v.bits & 4 ? v.h : v.w;
            src = e >= v.num0 ? oriented_luma(t.f[v.first + (int)(e - v.num0)].y, t.f[v.first + (int)(e - v.num0)].pitch, v.bits, v.w, v.h)
                              : oriented_luma(v.buf + (size_t)(e % L) * v.frame_bytes, sw, v.bits, v.w, v.h);
        } else if (e >= v.num0) {
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

}  // namespace rf
