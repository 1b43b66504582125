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
//                    list, the rf_follow records and the redaction regions in id order; f22, optionally, the removed tracks.
//   k_follow_mask    one CTA per frame of the round, with motion: the faces the estimate must not take for the scene.
// The bodies of k_follow_cut and k_follow_search live in search_kernels.cuh, shared with their f20 oriented twins (oriented_search.cu).
#include <algorithm>

#include "follow.cuh"
#include "kalman.cuh"
#include "search_kernels.cuh"

namespace rf {
namespace {

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_cut(const FollowArgs a, const __grid_constant__ FollowTable t) { follow_cut<false>(a, t); }

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_search(const FollowArgs a, const __grid_constant__ FollowTable t) {
    follow_search<false>(a, t);
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
    TrackGone *gone = a.gone ? a.gone + (size_t)f.frame * T : nullptr;
    if (tid == 0) { s_live = 0; s_regions = 0; }
    for (int i = tid; i < T; i += blockDim.x) {
        s_ok[i] = 0;
        if (gone) gone[i].id = 0;
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
            if (gone) gone[i] = TrackGone{k.id, k.hits, k.age, st0 != RF_TRACK_TENTATIVE};
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

cudaError_t launch_follow_cut(const FollowArgs &a, const FollowFrame *frames, int n, cudaStream_t s, bool oriented) {
    for (int i0 = 0; i0 < n; i0 += TRACK_MAX_FRAMES) {
        FollowTable t{};
        t.n = std::min(TRACK_MAX_FRAMES, n - i0);
        std::copy(frames + i0, frames + i0 + t.n, t.f);
        cudaError_t e;
        if (oriented) {
            e = launch_follow_cut_oriented(a, t, s);
        } else {
            k_follow_cut<<<dim3(a.p.max_tracks, t.n), FOLLOW_THREADS, 0, s>>>(a, t);
            e = cudaGetLastError();
        }
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_follow_round(const FollowArgs &a, const FollowTable &t, cudaStream_t s, bool oriented) {
    const int T = a.p.max_tracks;
    if (oriented) {
        const cudaError_t e = launch_follow_search_oriented(a, t, s);
        if (e != cudaSuccess) return e;
    } else {
        k_follow_search<<<dim3(T, t.n), FOLLOW_THREADS, 0, s>>>(a, t);
    }
    k_follow_update<<<t.n, TRACK_THREADS, (size_t)T * (sizeof(int) + 1), s>>>(a, t);
    return cudaGetLastError();
}

}  // namespace rf
