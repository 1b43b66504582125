// follow.cu -- f16 following between detections (follow.cuh, rf_b200.h rf_tracker_set_follow).  Built with -fmad=false: every FP64
// step below is one rounded operation in the order written, which oracle/follow.py restates operation by operation.
//
//   k_follow_cut     one CTA per (list rank, frame) of a detect call, after the update: a track matched on the frame, and not again
//                    later in the launch, gets its T x T luma template (one pixel per thread at a time) and the FLAT test.
//   k_follow_search  one CTA per (track slot, frame) of a follow round: the three (T + 2R)^2 windows sampled into shared memory, the
//                    exhaustive SAD over 3 (2R + 1)^2 candidates (one candidate per thread at a time, the template rows broadcast
//                    from shared memory and each window row read as aligned words re-cut by __byte_perm for __vsadu4), the ordered
//                    minimum as one 64-bit key, then the parabola, the box and the status on one thread.
//   k_follow_update  one CTA per frame of the round (distinct videos): f10's predict (and f13's motion step), the follow rules, the
//                    list, the rf_follow records and the redaction regions in id order.
//   k_follow_mask    one CTA per frame of the round, with motion: the faces the estimate must not take for the scene.
#include <algorithm>

#include "follow.cuh"
#include "kalman.cuh"
#include "tsearch.cuh"

namespace rf {
namespace {

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_cut(const FollowArgs a, const __grid_constant__ FollowTable t) {
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
    cut_template(f, s_g, a.store + e * FOLLOW_BYTES, &s_sum, &s_sq);
    __syncthreads();
    if (tid == 0) a.entries[e] = FollowEntry{tr.id, template_flat(s_sum, s_sq)};
}

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_search(const FollowArgs a, const __grid_constant__ FollowTable t) {
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
    search_windows(f, s_g, W, s_win, s_in, tid);
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

__global__ void __launch_bounds__(TRACK_THREADS) k_follow_update(const FollowArgs a, const __grid_constant__ FollowTable t) {
    extern __shared__ int s_dyn[];
    __shared__ int s_live, s_regions;
    const FollowFrame &f = t.f[blockIdx.x];
    const int T = a.p.max_tracks, tid = threadIdx.x;
    int *s_id = s_dyn;
    unsigned char *s_ok = reinterpret_cast<unsigned char *>(s_id + T);      // 1: followed, 2: LOST at frame start
    TrackState *S = a.state + (size_t)f.video * T;
    const FollowMeas *meas = a.meas + (size_t)f.frame * T;
    const double *motion = a.motion && a.motion[f.frame].status == RF_MOTION_OK ? a.motion[f.frame].m : nullptr;
    if (tid == 0) { s_live = 0; s_regions = 0; }
    for (int i = tid; i < T; i += blockDim.x) {
        s_ok[i] = 0;
        s_id[i] = S[i].id;
        if (!s_id[i]) continue;
        TrackState &k = S[i];
        const int st0 = k.state;
        kalman_predict(k);
        if (motion) kalman_motion(k, motion);
        k.age++;
        k.det = -1;
        if (st0 != RF_TRACK_LOST && meas[i].rec.status == RF_FOLLOW_OK) {
            double z[4];
            measure(meas[i].face, z);
            kalman_update(k, z);
            k.lost = 0;
            k.face = meas[i].face;
            s_ok[i] = 1;
            continue;
        }
        s_ok[i] = st0 == RF_TRACK_LOST ? 2 : 0;
        bool remove = st0 == RF_TRACK_TENTATIVE;
        if (!remove) {
            if (st0 == RF_TRACK_CONFIRMED) { k.state = RF_TRACK_LOST; k.lost = 1; }
            else k.lost++;
            remove = k.lost > a.p.max_lost;
        }
        if (remove) {
            k.id = 0;
            s_id[i] = 0;
        }
    }
    __syncthreads();
    rf_track *out = a.tracks + (size_t)f.frame * T;
    rf_follow *fo = a.follow + (size_t)f.frame * T;
    for (int i = tid; i < T; i += blockDim.x) {
        const int id = s_id[i];
        if (!id) continue;
        int rank = 0, frank = 0;
        for (int q = 0; q < T; q++) {
            const int o = s_id[q];
            rank += o && o < id;
            frank += o && o < id && s_ok[q] == 1;
        }
        atomicAdd(&s_live, 1);
        const TrackState &k = S[i];
        rf_track r;
        r.id = id;
        r.state = k.state;
        r.det = -1;
        r.crop_slot = -1;
        r.hits = k.hits;
        r.age = k.age;
        r.lost_frames = k.lost;
        r.followed = s_ok[i] == 1;
        double b[4];
        box_of(k.m, b);
        r.kx1 = (float)b[0]; r.ky1 = (float)b[1]; r.kx2 = (float)b[2]; r.ky2 = (float)b[3];
        r.vx = (float)k.u[0];
        r.vy = (float)k.u[1];
        r.face = k.face;
        out[rank] = r;
        if (s_ok[i] == 1) {
            atomicAdd(&s_regions, 1);
            rf_det d;
            d.face = k.face;
            d.anchor_index = id;
            a.regions[(size_t)f.frame * T + frank] = d;
        }
        if (s_ok[i] == 2) {
            rf_follow l{};
            l.id = id;
            l.status = RF_FOLLOW_LOST;
            fo[rank] = l;
        } else {
            fo[rank] = meas[i].rec;
        }
    }
    __syncthreads();
    if (tid == 0) {
        a.track_counts[f.frame] = s_live;
        a.region_counts[f.frame] = s_regions;
        a.videos[f.video].frames++;
    }
}

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_mask(const FollowArgs a, const __grid_constant__ FollowTable t) {
    __shared__ int s_n;
    const FollowFrame &f = t.f[blockIdx.x];
    const int T = a.p.max_tracks;
    const TrackState *S = a.state + (size_t)f.video * T;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < T; i += blockDim.x) {     // any order: the mask only asks whether a block overlaps some face
        if (!S[i].id || S[i].state == RF_TRACK_LOST) continue;
        rf_det d;
        d.face = S[i].face;
        d.anchor_index = S[i].id;
        a.mask[(size_t)f.frame * T + atomicAdd(&s_n, 1)] = d;
    }
    __syncthreads();
    if (threadIdx.x == 0) a.mask_counts[f.frame] = s_n;
}

}  // namespace

cudaError_t launch_follow_mask(const FollowArgs &a, const FollowTable &t, cudaStream_t s) {
    k_follow_mask<<<t.n, FOLLOW_THREADS, 0, s>>>(a, t);
    return cudaGetLastError();
}

cudaError_t launch_follow_cut(const FollowArgs &a, const FollowFrame *frames, int n, cudaStream_t s) {
    for (int i0 = 0; i0 < n; i0 += TRACK_MAX_FRAMES) {
        FollowTable t{};
        t.n = std::min(TRACK_MAX_FRAMES, n - i0);
        std::copy(frames + i0, frames + i0 + t.n, t.f);
        k_follow_cut<<<dim3(a.p.max_tracks, t.n), FOLLOW_THREADS, 0, s>>>(a, t);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_follow_round(const FollowArgs &a, const FollowTable &t, cudaStream_t s) {
    const int T = a.p.max_tracks;
    k_follow_search<<<dim3(T, t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    k_follow_update<<<t.n, TRACK_THREADS, (size_t)T * (sizeof(int) + 1), s>>>(a, t);
    return cudaGetLastError();
}

}  // namespace rf
