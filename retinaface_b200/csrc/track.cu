// track.cu -- f10 face tracking (track.cuh, rf_b200.h rf_track_update).  Built with -fmad=false: every FP64 step below is one
// rounded operation in the order written, which oracle/track.py restates operation by operation.
//
// Order of operations (c in cx, cy, a, h; h is the track's m_h before the step; sp = 1 / 20, sv = 1 / 160):
//   predict   LOST: u_h = 0.  q_pos = sp * h, q_vel = sv * h (a: 1e-2, 1e-5);
//             P00 = ((P00 + P01) + (P01 + P11)) + q_pos * q_pos;  P01 = P01 + P11;  P11 = P11 + q_vel * q_vel;  m = m + u
//   update    r = sp * h (a: 1e-1);  S = P00 + r * r;  K0 = P00 / S;  K1 = P01 / S;  y = z - m;  m = m + K0 * y;  u = u + K1 * y;
//             P00 = P00 - (K0 * S) * K0;  P01 = P01 - (K0 * S) * K1;  P11 = P11 - (K1 * S) * K1   (right-hand sides: old values)
//   birth     m = z;  u = 0;  P00 = ((2 * sp) * h) * ((2 * sp) * h) (a: 1e-2 * 1e-2);  P01 = 0;
//             P11 = ((10 * sv) * h) * ((10 * sv) * h) (a: 1e-5 * 1e-5)
//   z         x1..y2 = __fmul_rn(record coordinate, scale) widened to double;  w = x2 - x1;  h = y2 - y1;  cx = x1 + w / 2;
//             cy = y1 + h / 2;  a = w / h   (w <= 0 or h <= 0: the record is ignored)
//   box       w = a * h;  x1 = cx - w / 2;  y1 = cy - h / 2;  x2 = x1 + w;  y2 = y1 + h
//   IoU       x = max(x1), y = max(y1);  iw = (min(x2) - x) + 1;  ih = (min(y2) - y) + 1;  0 unless both > 0;
//             area = ((x2 - x1) + 1) * ((y2 - y1) + 1) of each;  inter = iw * ih;  IoU = inter / ((area_t + area_d) - inter)
//   motion    (f13, after predict, RF_MOTION_OK frames only; restated by oracle/motion.py compensate)  s = sqrt(a * a + b * b),
//             ss = s * s;  cx = ((a * cx) - (b * cy)) + tx;  cy = ((b * cx) + (a * cy)) + ty (old cx, cy);  u_cx, u_cy likewise
//             without t;  h = s * h;  u_h = s * u_h;  P00, P01, P11 = ss * P for cx, cy, h
#include <algorithm>

#include "kalman.cuh"

namespace rf {
namespace {

__device__ __forceinline__ rf_face mapped_face(const rf_det *dets, int j, float s) {
    rf_face f = dets[j].face;
    f.x1 = __fmul_rn(f.x1, s); f.y1 = __fmul_rn(f.y1, s); f.x2 = __fmul_rn(f.x2, s); f.y2 = __fmul_rn(f.y2, s);
#pragma unroll
    for (int l = 0; l < 5; l++) { f.lx[l] = __fmul_rn(f.lx[l], s); f.ly[l] = __fmul_rn(f.ly[l], s); }
    return f;
}

__device__ __forceinline__ double iou_of(const double a[4], const double b[4]) {
    const double x = fmax(a[0], b[0]), y = fmax(a[1], b[1]);
    const double w = (fmin(a[2], b[2]) - x) + 1.0, h = (fmin(a[3], b[3]) - y) + 1.0;
    if (!(w > 0.0) || !(h > 0.0)) return 0.0;
    const double area1 = ((a[2] - a[0]) + 1.0) * ((a[3] - a[1]) + 1.0);
    const double area2 = ((b[2] - b[0]) + 1.0) * ((b[3] - b[1]) + 1.0);
    const double inter = w * h;
    return inter / ((area1 + area2) - inter);
}

__device__ __forceinline__ void kalman_birth(TrackState &k, const double z[4]) {
    const double h = z[3];
#pragma unroll
    for (int c = 0; c < 4; c++) {
        const double sp = c == 2 ? 1e-2 : (2.0 * kSp) * h, sv = c == 2 ? 1e-5 : (10.0 * kSv) * h;
        k.m[c] = z[c];
        k.u[c] = 0.0;
        k.p00[c] = sp * sp;
        k.p01[c] = 0.0;
        k.p11[c] = sv * sv;
    }
}

// strict order of the greedy stages: IoU descending, then track id, then record index
__device__ __forceinline__ bool pair_before(const TrackPair &a, const TrackPair &b) {
    if (a.iou != b.iou) return a.iou > b.iou;
    if (a.id != b.id) return a.id < b.id;
    return a.det < b.det;
}

struct Shared {
    int *id;                 // [T] id of each slot, 0: free
    int *match;              // [T] record matched on this frame, -1
    unsigned char *st0;      // [T] state at frame start
    unsigned char *due;      // [T] confirmed on this frame (a new identity)
    unsigned char *used;     // [F] record matched
};

// One greedy stage: every (track, record) pair both free and eligible with IoU > thr into the CTA's scratch, rank-sorted, then
// matched by one thread in that order.
template <typename TrackOk, typename DetOk>
__device__ void greedy_stage(const Shared &sm, const TrackState *S, const rf_det *dets, float sc, int T, int K, double thr, TrackPair *pairs,
                             int *order, int *s_np, TrackOk track_ok, DetOk det_ok) {
    const int tid = threadIdx.x;
    if (tid == 0) *s_np = 0;
    __syncthreads();
    for (int q = tid; q < T * K; q += blockDim.x) {
        const int i = q / K, j = q - i * K;
        if (!sm.id[i] || sm.match[i] >= 0 || !track_ok(sm.st0[i]) || sm.used[j]) continue;
        const rf_face f = mapped_face(dets, j, sc);
        double z[4];
        if (!det_ok(f.score) || !measure(f, z)) continue;
        const double b[4] = {(double)f.x1, (double)f.y1, (double)f.x2, (double)f.y2};
        double p[4];
        box_of(S[i].m, p);
        const double iou = iou_of(p, b);
        if (iou > thr) pairs[atomicAdd(s_np, 1)] = TrackPair{iou, sm.id[i], (short)i, (short)j};
    }
    __syncthreads();
    const int np = *s_np;
    // rank sort: (id, record) is unique, so the order is total and the rank of a pair is the count of pairs before it
    for (int p = tid; p < np; p += blockDim.x) {
        const TrackPair me = pairs[p];
        int rank = 0;
        for (int q = 0; q < np; q++) rank += pair_before(pairs[q], me);
        order[rank] = p;
    }
    __syncthreads();
    if (tid == 0)
        for (int r = 0; r < np; r++) {
            const TrackPair pp = pairs[order[r]];
            if (sm.match[pp.slot] < 0 && !sm.used[pp.det]) {
                sm.match[pp.slot] = pp.det;
                sm.used[pp.det] = 1;
            }
        }
    __syncthreads();
}

// One CTA per distinct video of the launch; it applies that video's frames in call order.  Predict and the state changes run one
// thread per track slot, the stages as above, the births on one thread in record order, the output one thread per live track
// (its rank by id is its place).
__global__ void __launch_bounds__(TRACK_THREADS) k_track_update(const TrackArgs a, const __grid_constant__ TrackTable t) {
    extern __shared__ int s_dyn[];
    __shared__ int s_np, s_frames, s_issued, s_overflow, s_live, s_due;
    const int T = a.p.max_tracks, F = a.p.max_faces, tid = threadIdx.x;
    Shared sm;
    sm.id = s_dyn;
    sm.match = sm.id + T;
    sm.st0 = reinterpret_cast<unsigned char *>(sm.match + T);
    sm.due = sm.st0 + T;
    sm.used = sm.due + T;
    const int v = t.cta_video[blockIdx.x];
    TrackVideo *vid = a.videos + v;
    TrackState *S = a.state + (size_t)v * T;
    TrackPair *pairs = a.pairs + (size_t)blockIdx.x * T * F;
    int *order = a.order + (size_t)blockIdx.x * T * F;
    for (int i = tid; i < T; i += blockDim.x) sm.id[i] = S[i].id;
    if (tid == 0) { s_frames = vid->frames; s_issued = vid->issued; s_overflow = vid->overflow; }
    __syncthreads();
    const float high = a.p.high_thresh;
    for (int f = 0; f < t.n; f++) {
        if (t.video[f] != v) continue;       // uniform over the CTA
        const rf_det *dets = a.dets + (size_t)f * F;
        const int K = min(max(a.counts[f], 0), F);
        const float sc = t.scale[f];
        TrackSeen *seen = a.seen ? a.seen + (size_t)f * F : nullptr;
        TrackGone *gone = a.gone ? a.gone + (size_t)f * T : nullptr;
        const double *motion = a.motion && a.motion[f].status == RF_MOTION_OK ? a.motion[f].m : nullptr;
        if (seen)
            for (int j = tid; j < F; j += blockDim.x) seen[j].slot = -1;
        for (int i = tid; i < T; i += blockDim.x) {
            sm.match[i] = -1;
            sm.due[i] = 0;
            if (gone) gone[i].id = 0;
            if (!sm.id[i]) continue;
            TrackState &k = S[i];
            sm.st0[i] = (unsigned char)k.state;
            kalman_predict(k);
            if (motion) kalman_motion(k, motion);
            k.age++;
        }
        for (int j = tid; j < K; j += blockDim.x) sm.used[j] = 0;
        if (tid == 0) { s_live = 0; s_due = 0; }
        __syncthreads();
        greedy_stage(sm, S, dets, sc, T, K, (double)a.p.iou_high, pairs, order, &s_np,
                     [](int st) { return st == RF_TRACK_CONFIRMED || st == RF_TRACK_LOST; }, [&](float s) { return s >= high; });
        greedy_stage(sm, S, dets, sc, T, K, (double)a.p.iou_low, pairs, order, &s_np,
                     [](int st) { return st == RF_TRACK_CONFIRMED; }, [&](float s) { return !(s >= high); });
        greedy_stage(sm, S, dets, sc, T, K, (double)a.p.iou_tentative, pairs, order, &s_np,
                     [](int st) { return st == RF_TRACK_TENTATIVE; }, [&](float s) { return s >= high; });
        for (int i = tid; i < T; i += blockDim.x) {
            if (!sm.id[i]) continue;
            TrackState &k = S[i];
            const int j = sm.match[i], st0 = sm.st0[i];
            if (j >= 0) {
                const rf_face fj = mapped_face(dets, j, sc);
                double z[4];
                measure(fj, z);
                kalman_update(k, z);
                k.hits++;
                k.lost = 0;
                k.face = fj;
                k.det = j;
                k.state = RF_TRACK_CONFIRMED;
                sm.due[i] = st0 == RF_TRACK_TENTATIVE;
                if (seen) seen[j] = TrackSeen{i, k.id, fj};
                continue;
            }
            k.det = -1;
            bool remove = st0 == RF_TRACK_TENTATIVE;
            if (!remove) {
                if (st0 == RF_TRACK_CONFIRMED) { k.state = RF_TRACK_LOST; k.lost = 1; }
                else k.lost++;
                remove = k.lost > a.p.max_lost;
            }
            if (remove) {
                if (gone) gone[i] = TrackGone{k.id, k.hits, k.age, st0 != RF_TRACK_TENTATIVE};
                k.id = 0;
                sm.id[i] = 0;
            }
        }
        __syncthreads();
        if (tid == 0) {
            const bool first = s_frames == 0;
            int slot = 0;
            for (int j = 0; j < K; j++) {
                if (sm.used[j]) continue;
                const rf_face fj = mapped_face(dets, j, sc);
                double z[4];
                if (!(fj.score >= high) || !(fj.score >= a.p.new_thresh) || !measure(fj, z)) continue;
                while (slot < T && sm.id[slot]) slot++;
                if (slot == T) { s_overflow++; continue; }
                TrackState &k = S[slot];
                kalman_birth(k, z);
                k.face = fj;
                k.id = sm.id[slot] = ++s_issued;
                k.state = first ? RF_TRACK_CONFIRMED : RF_TRACK_TENTATIVE;
                k.hits = 1;
                k.age = 1;
                k.lost = 0;
                k.det = j;
                sm.due[slot] = first;
                if (seen) seen[j] = TrackSeen{slot, k.id, fj};
            }
            s_frames++;
        }
        __syncthreads();
        rf_track *out = a.tracks + (size_t)f * T;
        for (int i = tid; i < T; i += blockDim.x) {
            const int id = sm.id[i];
            if (!id) continue;
            int rank = 0, drank = 0;
            for (int q = 0; q < T; q++) {
                const int o = sm.id[q];
                if (o && o < id) { rank++; drank += sm.due[q]; }
            }
            atomicAdd(&s_live, 1);
            const TrackState &k = S[i];
            rf_track r;
            r.id = id;
            r.state = k.state;
            r.det = k.det;
            r.crop_slot = -1;
            if (sm.due[i]) {
                atomicAdd(&s_due, 1);
                if (drank < a.max_align) {
                    r.crop_slot = drank;
                    rf_det d;
                    d.face = k.face;
                    d.anchor_index = id;
                    a.due[(size_t)f * F + drank] = d;
                }
            }
            r.hits = k.hits;
            r.age = k.age;
            r.lost_frames = k.lost;
            r.followed = 0;
            if (a.life && k.det >= 0) a.life[(size_t)f * F + k.det] = TrackLife{k.hits, k.age, k.state, 0};
            double b[4];
            box_of(k.m, b);
            r.kx1 = (float)b[0]; r.ky1 = (float)b[1]; r.kx2 = (float)b[2]; r.ky2 = (float)b[3];
            r.vx = (float)k.u[0];
            r.vy = (float)k.u[1];
            r.face = k.face;
            out[rank] = r;
        }
        __syncthreads();
        if (tid == 0) {
            a.track_counts[f] = s_live;
            if (a.due_counts) a.due_counts[f] = min(s_due, a.max_align);
        }
    }
    if (tid == 0) { vid->frames = s_frames; vid->issued = s_issued; vid->overflow = s_overflow; }
}

}  // namespace

cudaError_t launch_track_update(const TrackArgs &a, const int *videos, const float *scales, int n, cudaStream_t s) {
    const int T = a.p.max_tracks, F = a.p.max_faces;
    const size_t smem = (size_t)T * (2 * sizeof(int) + 2) + F;
    for (int i0 = 0; i0 < n; i0 += TRACK_MAX_FRAMES) {
        const int m = std::min(TRACK_MAX_FRAMES, n - i0);
        TrackTable t{};
        t.n = m;
        for (int i = 0; i < m; i++) {
            t.video[i] = videos[i0 + i];
            t.scale[i] = scales ? scales[i0 + i] : 1.f;
            bool seen = false;
            for (int b = 0; b < t.nvideos; b++) seen |= t.cta_video[b] == t.video[i];
            if (!seen) t.cta_video[t.nvideos++] = t.video[i];
        }
        TrackArgs c = a;
        c.dets = a.dets + (size_t)i0 * F;
        c.counts = a.counts + i0;
        c.tracks = a.tracks + (size_t)i0 * T;
        c.track_counts = a.track_counts + i0;
        if (a.due) {
            c.due = a.due + (size_t)i0 * F;
            c.due_counts = a.due_counts + i0;
        }
        if (a.seen) c.seen = a.seen + (size_t)i0 * F;
        if (a.gone) c.gone = a.gone + (size_t)i0 * T;
        if (a.life) c.life = a.life + (size_t)i0 * F;
        if (a.motion) c.motion = a.motion + i0;
        k_track_update<<<t.nvideos, TRACK_THREADS, smem, s>>>(c, t);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace rf
