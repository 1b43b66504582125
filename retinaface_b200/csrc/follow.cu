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

namespace rf {
namespace {

constexpr int WIN = FOLLOW_T + 2 * FOLLOW_MAX_R;      // window side at the largest R
constexpr int WWORDS = WIN / 4 + 1;                    // words per window row: a candidate row may read one word past its last
constexpr int MAX_SIDE = 2 * FOLLOW_MAX_R + 1;
constexpr double kGrow = 1.0 + 2.0 * RF_FOLLOW_MARGIN;
constexpr double FOLLOW_MAX_BOX = 65536.0;             // predicted centre and size bound: keeps the fixed-point coordinates in int

struct Grid {
    double px, py, ox, oy;
};

__device__ __forceinline__ Grid grid_of(double cx, double cy, double w, double h, double c) {
    const double gw = (w * kGrow) * c, gh = (h * kGrow) * c;
    Grid g;
    g.px = gw / (double)FOLLOW_T;
    g.py = gh / (double)FOLLOW_T;
    g.ox = ((cx - gw / 2.0) + g.px / 2.0) - 0.5;
    g.oy = ((cy - gh / 2.0) + g.py / 2.0) - 0.5;
    return g;
}

// c_k: {1 / s, 1, s}
__device__ __forceinline__ double scale_of(int k) { return k == 0 ? 1.0 / RF_FOLLOW_SCALE : k == 1 ? 1.0 : RF_FOLLOW_SCALE; }

// Pixel (i, j) of the map [[px, 0, X], [0, py, Y]]: cv::warpAffine's fixed-point coordinate and f5's integer bilinear on the luma
// plane (warp.cuh's sample() on one channel).  inside: all four taps lay in the frame.
__device__ __forceinline__ int luma_at(const FollowFrame &f, double px, double py, double X, double Y, int i, int j, bool &inside) {
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
            acc += wts[t] * f.y[(size_t)ty * f.pitch + tx];
            in++;
        }
    }
    inside = in == 4;
    return acc >> 15;
}

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_cut(const FollowArgs a, const __grid_constant__ FollowTable t) {
    __shared__ int s_slot;
    __shared__ double s_g[4];
    __shared__ unsigned long long s_sum, s_sq;
    const FollowFrame &f = t.f[blockIdx.y];
    const int T = a.p.max_tracks, tid = threadIdx.x, lane = tid & 31;
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
        const double x1 = tr.face.x1, y1 = tr.face.y1, w = (double)tr.face.x2 - x1, h = (double)tr.face.y2 - y1;
        const Grid g = grid_of(x1 + w / 2.0, y1 + h / 2.0, w, h, 1.0);
        s_g[0] = g.px; s_g[1] = g.py; s_g[2] = g.ox; s_g[3] = g.oy;
    }
    __syncthreads();
    const int slot = s_slot;
    if (slot < 0) return;                                                         // uniform
    const size_t e = (size_t)f.video * T + slot;
    uint8_t *dst = a.store + e * FOLLOW_BYTES;
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
    if (lane == 0) { atomicAdd(&s_sum, (unsigned long long)s1); atomicAdd(&s_sq, (unsigned long long)s2); }
    __syncthreads();
    if (tid == 0) {
        const long long var = (long long)FOLLOW_BYTES * (long long)s_sq - (long long)s_sum * (long long)s_sum;
        a.entries[e] = FollowEntry{tr.id, var < (long long)RF_FOLLOW_MIN_VAR * FOLLOW_BYTES * FOLLOW_BYTES};
    }
}

__global__ void __launch_bounds__(FOLLOW_THREADS) k_follow_search(const FollowArgs a, const __grid_constant__ FollowTable t) {
    __shared__ uint32_t s_win[3][WIN][WWORDS];
    __shared__ uint8_t s_in[3][WIN][WIN];
    __shared__ uint32_t s_tpl[FOLLOW_BYTES / 4];
    __shared__ int s_sad[3 * MAX_SIDE * MAX_SIDE];
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
    const bool bounded = ph > 0.0 && ph <= FOLLOW_MAX_BOX && pw > 0.0 && pw <= FOLLOW_MAX_BOX && fabs(pcx) <= FOLLOW_MAX_BOX &&
                         fabs(pcy) <= FOLLOW_MAX_BOX;
    if (a.entries[e].id != id || !bounded) {                                      // uniform: no template, or no search
        if (tid == 0) {
            rf_follow r{};
            r.id = id;
            r.status = bounded ? RF_FOLLOW_FLAT : RF_FOLLOW_MISMATCH;
            out->rec = r;
        }
        return;
    }
    if (tid < 3) {
        const Grid g = grid_of(pcx, pcy, pw, ph, scale_of(tid));
        s_g[tid][0] = g.px;
        s_g[tid][1] = g.py;
        s_g[tid][2] = g.ox - (double)R * g.px;
        s_g[tid][3] = g.oy - (double)R * g.py;
    }
    if (tid == 0) s_inside = 0;
    const uint32_t *tsrc = reinterpret_cast<const uint32_t *>(a.store + e * FOLLOW_BYTES);
    for (int w = tid; w < FOLLOW_BYTES / 4; w += FOLLOW_THREADS) s_tpl[w] = tsrc[w];
    __syncthreads();
    for (int p = tid; p < 3 * W * W; p += FOLLOW_THREADS) {
        const int k = p / (W * W), rem = p - k * W * W, r = rem / W, c = rem - r * W;
        bool in;
        const int v = luma_at(f, s_g[k][0], s_g[k][1], s_g[k][2], s_g[k][3], c, r, in);
        reinterpret_cast<uint8_t *>(s_win[k][r])[c] = (uint8_t)v;
        s_in[k][r][c] = in;
    }
    __syncthreads();
    unsigned long long best = ~0ull;
    for (int o = tid; o < 3 * nc; o += FOLLOW_THREADS) {
        const int k = o / nc, rem = o - k * nc, wy = rem / side, wx = rem - wy * side;
        const uint32_t *wp = &s_win[k][wy][wx >> 2];
        const unsigned sel = 0x3210u + 0x1111u * (unsigned)(wx & 3);
        unsigned sad = 0;
        for (int r = 0; r < FOLLOW_T; r++, wp += WWORDS) {
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
    const int k = (int)(best >> 12) & 3, wy = (int)(best >> 6) & 63, wx = (int)best & 63;
    int in = 0;
    for (int p = tid; p < FOLLOW_BYTES; p += FOLLOW_THREADS) in += s_in[k][wy + p / FOLLOW_T][wx + p % FOLLOW_T];
    if (in) atomicAdd(&s_inside, in);
    __syncthreads();
    if (tid != 0) return;
    const int dx = wx - R, dy = wy - R, c = k * nc + wy * side + wx, s0 = s_sad[c];
    const bool border = abs(dx) == R || abs(dy) == R;
    double fx = 0.0, fy = 0.0;
    if (!border) {
        const int xm = s_sad[c - 1], xp = s_sad[c + 1], ym = s_sad[c - side], yp = s_sad[c + side];
        const int dnx = 2 * (xm - 2 * s0 + xp), dny = 2 * (ym - 2 * s0 + yp);
        if (dnx != 0) fx = (double)(xm - xp) / (double)dnx;
        if (dny != 0) fy = (double)(ym - yp) / (double)dny;
    }
    const double ncx = pcx + ((double)dx + fx) * s_g[k][0], ncy = pcy + ((double)dy + fy) * s_g[k][1];
    const double nw = pw * scale_of(k), nh = ph * scale_of(k);
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
    r.dx = dx;
    r.dy = dy;
    r.scale = k;
    r.sad = s0;
    r.fx = (float)fx;
    r.fy = (float)fy;
    r.x1 = nf.x1; r.y1 = nf.y1; r.x2 = nf.x2; r.y2 = nf.y2;
    const bool empty = !((double)nf.x2 - (double)nf.x1 > 0.0) || !((double)nf.y2 - (double)nf.y1 > 0.0);
    r.status = a.entries[e].flat                                 ? RF_FOLLOW_FLAT
               : 4 * s_inside < 3 * FOLLOW_BYTES                 ? RF_FOLLOW_OUTSIDE
               : border                                          ? RF_FOLLOW_BORDER
               : (double)s0 > (double)a.max_mad * (double)FOLLOW_BYTES || empty ? RF_FOLLOW_MISMATCH
                                                                 : RF_FOLLOW_OK;
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
