// best.cu -- see best.cuh.  Built with -fmad=false: the warp is align.cu's (warp.cuh), and every FP64 step of the quality is one
// rounded operation in the order rf_b200.h writes it, which oracle/bestshot.py restates.
#include "best.cuh"
#include "warp.cuh"

namespace rf {
namespace {

constexpr int EMIT_THREADS = 128;

template <typename V>
__device__ __forceinline__ V warp_sum(V v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// Records that may be seen, numbered frame by frame: s_first[f] is the number of frame f's first one (s_first[n]: the total).
__device__ __forceinline__ void record_prefix(const BestArgs &a, int n, int *s_first) {
    if (threadIdx.x < n) s_first[threadIdx.x + 1] = min(max(a.counts[threadIdx.x], 0), a.max_faces);     // the loads in parallel
    __syncthreads();
    if (threadIdx.x == 0) {
        s_first[0] = 0;
        for (int f = 1; f <= n; f++) s_first[f] += s_first[f - 1];
    }
    __syncthreads();
}

// the (frame, record) index of candidate c
__device__ __forceinline__ size_t record_of(const int *s_first, int c, int F) {
    int f = 0;
    while (s_first[f + 1] <= c) f++;
    return (size_t)f * F + (c - s_first[f]);
}

// Grid-stride over (record, band) items; records no track holds are skipped by the whole CTA.  A band's pixels are cut exactly as
// k_align_faces cuts them (same tables, same sample, same store); its grey values and INSIDE bits, with one halo row above and below,
// stay in shared memory for the Laplacian.
// f20: the ORIENTED instantiation samples each frame as displayed (warp.cuh sample<true>; im.w x im.h the displayed size).
template <bool ORIENTED>
__global__ void __launch_bounds__(BEST_THREADS) k_best_measure(const BestArgs a, const __grid_constant__ BestTable t) {
    constexpr int R = BEST_BAND + 2;
    __shared__ int s_first[TRACK_MAX_FRAMES + 1];
    __shared__ int s_ax[ALIGN_MAX_SIDE], s_bx[ALIGN_MAX_SIDE], s_x0[R], s_y0[R];
    __shared__ uint8_t s_g[R * ALIGN_MAX_SIDE];
    __shared__ uint32_t s_in[R * ALIGN_MAX_SIDE / 32];
    __shared__ double s_im[6];
    __shared__ long long s_red[4][BEST_THREADS / 32];
    __shared__ int s_zero;
    const int F = a.max_faces, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    record_prefix(a, t.n, s_first);
    const int cw = a.u8.crop_w, ch = a.u8.crop_h, qpr = (cw + 3) >> 2;
    const int bands = (ch + BEST_BAND - 1) / BEST_BAND, items = s_first[t.n] * bands;
    for (int item = blockIdx.x; item < items; item += gridDim.x) {
        const int c = item / bands, band = item - c * bands;
        const size_t fj = record_of(s_first, c, F);
        const int f = (int)(fj / F);
        const TrackSeen &sn = a.seen[fj];
        if (sn.slot < 0) continue;           // uniform over the CTA
        if (tid == 0) {
            double M[6], iM[6];
            s_zero = fit_similarity(sn.face, 1.f, a.u8.tmpl, M) ? 0 : 1;
            invert_affine(M, iM);
            for (int k = 0; k < 6; k++) s_im[k] = iM[k];
            if (band == 0)
                for (int k = 0; k < 6; k++) a.meas[fj].M[k] = M[k];
        }
        // row r of the tables is crop row y0 + r; rows outside the crop are not cut
        const int y0 = band * BEST_BAND - 1, rlo = y0 < 0 ? 1 : 0, rhi = min(R, ch - y0);
        for (int w = tid; w < (R * cw + 31) / 32; w += blockDim.x) s_in[w] = 0;
        __syncthreads();
        const double i0 = s_im[0], i1 = s_im[1], i2 = s_im[2], i3 = s_im[3], i4 = s_im[4], i5 = s_im[5];
        for (int x = tid; x < cw; x += blockDim.x) {
            s_ax[x] = __double2int_rn(i0 * x * 1024.0);
            s_bx[x] = __double2int_rn(i3 * x * 1024.0);
        }
        for (int r = rlo + tid; r < rhi; r += blockDim.x) {
            const int y = y0 + r;
            s_x0[r] = __double2int_rn((i1 * y + i2) * 1024.0) + 16;
            s_y0[r] = __double2int_rn((i4 * y + i5) * 1024.0) + 16;
        }
        __syncthreads();
        const bool zero = s_zero != 0;
        const AlignImageT<YuvPlanes> &im = t.img[f];
        unsigned char *crop = a.scratch + fj * a.u8.crop_bytes;
        int inside = 0;
        for (int qd = tid; qd < (rhi - rlo) * qpr; qd += blockDim.x) {
            const int rr = qd / qpr, r = rlo + rr, x4 = (qd - rr * qpr) * 4;
            int v[4][3];
            unsigned bits = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const int x = x4 + k;
                if (x < cw && !zero) {
                    if (sample<ORIENTED>(im, (s_x0[r] + s_ax[x]) >> 5, (s_y0[r] + s_bx[x]) >> 5, v[k])) bits |= 1u << k;
                } else {
                    v[k][0] = v[k][1] = v[k][2] = 0;
                }
                if (x < cw) s_g[r * cw + x] = (uint8_t)((3735 * v[k][0] + 19235 * v[k][1] + 9798 * v[k][2] + 16384) >> 15);   // BGR2GRAY
            }
            for (int k = 0; k < 4; k++)
                if (bits >> k & 1u) {
                    const int p = r * cw + x4 + k;
                    atomicOr(&s_in[p >> 5], 1u << (p & 31));
                }
            if (r >= 1 && r <= BEST_BAND) {      // the band's own rows
                store_quad(a.u8, crop, y0 + r, x4, v);
                inside += __popc(bits);
            }
        }
        __syncthreads();
        // the Laplacian on the band's rows of the interior where the pixel and its 4 neighbours are INSIDE
        long long s1 = 0, s2 = 0;
        int nl = 0;
        const int ylo = max(1, y0 + 1), yhi = min(ch - 2, y0 + BEST_BAND), iw = cw - 2;
        auto in = [&](int r, int x) { const int p = r * cw + x; return (s_in[p >> 5] >> (p & 31)) & 1u; };
        for (int p = tid; p < (yhi - ylo + 1) * iw; p += blockDim.x) {
            const int yy = p / iw, x = 1 + (p - yy * iw), r = ylo + yy - y0;
            if (!(in(r, x) && in(r, x - 1) && in(r, x + 1) && in(r - 1, x) && in(r + 1, x))) continue;
            const uint8_t *g = s_g + r * cw + x;
            const int L = (int)g[-1] + (int)g[1] + (int)g[-cw] + (int)g[cw] - 4 * (int)g[0];
            nl++;
            s1 += L;
            s2 += (long long)L * L;
        }
        const long long r0 = warp_sum((long long)inside), r1 = warp_sum((long long)nl), r2 = warp_sum(s1), r3 = warp_sum(s2);
        if (lane == 0) { s_red[0][warp] = r0; s_red[1][warp] = r1; s_red[2][warp] = r2; s_red[3][warp] = r3; }
        __syncthreads();
        if (tid == 0) {
            long long nin = 0, N = 0, S1 = 0, S2 = 0;
            for (int w = 0; w < BEST_THREADS / 32; w++) { nin += s_red[0][w]; N += s_red[1][w]; S1 += s_red[2][w]; S2 += s_red[3][w]; }
            BestAccum *acc = a.acc + fj;
            atomicAdd(&acc->inside, (unsigned long long)nin);
            atomicAdd(&acc->n, (unsigned long long)N);
            atomicAdd(&acc->s1, (unsigned long long)S1);
            atomicAdd(&acc->s2, (unsigned long long)S2);
            __threadfence();
            if (atomicAdd(&acc->done, 1u) == (unsigned)bands - 1) {      // the record's last band: every sum is in
                __threadfence();
                nin = (long long)atomicAdd(&acc->inside, 0ull);
                N = (long long)atomicAdd(&acc->n, 0ull);
                S1 = (long long)atomicAdd(&acc->s1, 0ull);
                S2 = (long long)atomicAdd(&acc->s2, 0ull);
                *acc = BestAccum{};
                const rf_face face = sn.face;
                BestMeasure *out = a.meas + fj;
                // the quality, in the header's order of operations
                const double lx0 = face.lx[0], ly0 = face.ly[0], lx1 = face.lx[1], ly1 = face.ly[1], lx2 = face.lx[2], ly2 = face.ly[2];
                const double ex = lx1 - lx0, ey = ly1 - ly0, d2 = ex * ex + ey * ey;
                double eye = 0.0, frontal = 0.0, sharpness = 0.0, coverage = 0.0, q = 0.0;
                if (!zero && d2 != 0.0) {
                    eye = sqrt(d2);
                    const double tt = ((lx2 - (lx0 + lx1) / 2.0) * ex + (ly2 - (ly0 + ly1) / 2.0) * ey) / d2;
                    frontal = fmax(0.0, 1.0 - 2.0 * fabs(tt));
                    const double *tm = a.u8.tmpl;
                    const double tx = tm[2] - tm[0], ty = tm[3] - tm[1];
                    const double eye_ref = sqrt(tx * tx + ty * ty);
                    const double size = eye_ref > 0.0 ? fmin(1.0, eye / eye_ref) : 1.0;
                    sharpness = N >= 2 ? (double)(N * S2 - S1 * S1) / ((double)N * (double)N) : 0.0;
                    const double sharp = sharpness / (sharpness + a.sharp_half);
                    coverage = (double)nin / (double)(cw * ch);
                    q = ((((double)face.score * frontal) * size) * sharp) * coverage;
                }
                out->q = q;
                out->score = face.score;
                out->eye = (float)eye;
                out->frontal = (float)frontal;
                out->sharpness = (float)sharpness;
                out->coverage = (float)coverage;
                out->pad = 0;
                out->face = face;
            }
        }
        __syncthreads();     // the tables of the next item overwrite these
    }
}

__device__ __forceinline__ const BestMeasure &source_measure(const BestArgs &a, int src) {
    return src >= 0 ? a.store[src].m : a.meas[-1 - src];
}

// Emission k of frame f: the record (its id rank is k), its crop's source and, optionally, M.
__device__ __forceinline__ void put_emission(const BestArgs &a, int f, int k, int src, int id, int video, int frame, int end_frame, int hits,
                                             int age, int reason) {
    const int T = a.max_tracks;
    const BestMeasure &m = source_measure(a, src);
    rf_best_shot r;
    r.id = id;
    r.video = video;
    r.frame = frame;
    r.end_frame = end_frame;
    r.hits = hits;
    r.age = age;
    r.reason = reason;
    r.reserved = 0;
    r.quality = (float)m.q;
    r.score = m.score;
    r.eye = m.eye;
    r.frontal = m.frontal;
    r.sharpness = m.sharpness;
    r.coverage = m.coverage;
    r.face = m.face;
    a.best[(size_t)f * T + k] = r;
    a.src[(size_t)f * T + k] = src;
    if (a.out.mats)
        for (int c = 0; c < 6; c++) a.out.mats[((size_t)f * T + k) * 6 + c] = m.M[c];
}

// rank of `id` among the non-zero ids of s_emit[0, T)
__device__ __forceinline__ int id_rank(const int *s_emit, int T, int id) {
    int rank = 0;
    for (int q = 0; q < T; q++) rank += s_emit[q] != 0 && s_emit[q] < id;
    return rank;
}

// One CTA per video of the call, thread i = track slot i (blockDim >= max_tracks).  Thread i carries the slot's best through the
// call's frames: id (0: none), q, source (>= 0: the store entry as it was before the call; < 0: a scratch crop of the call) and frame.
// f22: LIVE adds the live policy (rf_b200.h rf_tracker_set_best_live) after each frame's store step, and emits the frame's EXIT and
// LIVE shots together (a slot has at most one of them on a frame); SEEN false is a follow frame's launch: no records, removals only.
template <bool LIVE, bool SEEN>
__global__ void k_best_select(const BestArgs a, const __grid_constant__ BestTable t, const BestLiveArgs l) {
    extern __shared__ int s_dyn[];
    __shared__ int s_frame, s_count;
    const int T = a.max_tracks, F = a.max_faces, i = threadIdx.x, v = t.cta_video[blockIdx.x];
    int *s_j = s_dyn, *s_emit = s_dyn + T;
    const bool mine = i < T;
    const int si = v * T + i;
    int bid = 0, bsrc = si, bframe = 0;
    double bq = 0.0;
    BestLive lv{};
    if (mine) {
        const BestEntry &e = a.store[si];
        bid = e.id;
        bq = e.m.q;
        bframe = e.frame;
        if constexpr (LIVE) lv = l.live[si];
    }
    if (i == 0) s_frame = a.videos[v].frames;
    for (int f = 0; f < t.n; f++) {
        if (t.video[f] != v) continue;       // uniform over the CTA
        if (mine) { s_j[i] = -1; s_emit[i] = 0; }
        if constexpr (SEEN)
            for (int j = i; j < F; j += blockDim.x) a.commit[(size_t)f * F + j] = -1;
        if (i == 0) s_count = 0;
        __syncthreads();
        const int frame = s_frame;
        if constexpr (SEEN)
            for (int j = i; j < F; j += blockDim.x) {
                const int sl = a.seen[(size_t)f * F + j].slot;
                if (sl >= 0) s_j[sl] = j;
            }
        // removals first: an ever-confirmed track's best is emitted if it clears min_quality
        TrackGone g{};
        int esrc = 0, eframe = 0;
        if (mine) {
            g = a.gone[(size_t)f * T + i];
            if (g.id) {
                if (g.confirmed && bid == g.id && bq >= a.min_quality) {
                    s_emit[i] = g.id;
                    esrc = bsrc;
                    eframe = bframe;
                    atomicAdd(&s_count, 1);
                }
                bid = 0;
                bsrc = si;
            }
        }
        __syncthreads();
        if constexpr (!LIVE)
            if (mine && s_emit[i])
                put_emission(a, f, id_rank(s_emit, T, g.id), esrc, g.id, v, eframe, frame, g.hits, g.age, RF_BEST_EXIT);
        // then the tracks matched or born on the frame: a new track always stores, a known one only on a strictly better q
        if (SEEN && mine && s_j[i] >= 0) {
            const size_t fj = (size_t)f * F + s_j[i];
            const int id = a.seen[fj].id;
            const double q = a.meas[fj].q;
            if (bid != id || q > bq) {
                bid = id;
                bq = q;
                bsrc = -1 - (int)fj;
                bframe = frame;
            }
        }
        if constexpr (LIVE) {
            // a track CONFIRMED after the frame and matched on it: its first live shot once q clears first_quality and min_quality, a
            // further one once min_gap frames have passed and q beats the last one's by the factor 1 + improve
            TrackLife k{};
            bool live = false;
            if (mine && s_j[i] >= 0) {
                k = l.life[(size_t)f * F + s_j[i]];
                if (k.state == RF_TRACK_CONFIRMED) {
                    const int n = lv.id == bid ? lv.n : 0;
                    live = n == 0 ? bq >= l.first_quality && bq >= a.min_quality : frame - lv.e >= l.min_gap && bq > lv.q * l.ratio;
                    if (live) {
                        lv = BestLive{bid, n + 1, frame, 0, bq};
                        s_emit[i] = bid;
                        atomicAdd(&s_count, 1);
                    }
                }
            }
            __syncthreads();
            if (live) put_emission(a, f, id_rank(s_emit, T, bid), bsrc, bid, v, bframe, frame, k.hits, k.age, RF_BEST_LIVE);
            else if (mine && s_emit[i]) put_emission(a, f, id_rank(s_emit, T, g.id), esrc, g.id, v, eframe, frame, g.hits, g.age, RF_BEST_EXIT);
        }
        __syncthreads();
        if (i == 0) {
            a.best_counts[f] = s_count;
            s_frame = frame + 1;
        }
    }
    __syncthreads();
    if (mine) {
        if (bsrc < 0) {
            BestEntry &e = a.store[si];
            e.m = a.meas[-1 - bsrc];
            e.id = bid;
            e.frame = bframe;
            a.commit[-1 - bsrc] = si;
        } else if (!bid) {
            a.store[si].id = 0;
        }
        if constexpr (LIVE) l.live[si] = lv;
    }
    if (i == 0) a.videos[v].frames = s_frame;
}

// rf_tracker_finish: one CTA, thread i = slot i of the video.
__global__ void k_best_finish(const BestArgs a, int v, const TrackState *__restrict__ state) {
    extern __shared__ int s_dyn[];
    __shared__ int s_count;
    const int T = a.max_tracks, i = threadIdx.x, si = v * T + i;
    const bool mine = i < T;
    if (i == 0) s_count = 0;
    if (mine) s_dyn[i] = 0;
    __syncthreads();
    int id = 0;
    if (mine) {
        const TrackState &k = state[i];
        const BestEntry &e = a.store[si];
        if (k.id && k.state != RF_TRACK_TENTATIVE && e.id == k.id && e.m.q >= a.min_quality) {
            id = k.id;
            s_dyn[i] = id;
            atomicAdd(&s_count, 1);
        }
    }
    __syncthreads();
    if (id) {
        const TrackState &k = state[i];
        put_emission(a, 0, id_rank(s_dyn, T, id), si, id, v, a.store[si].frame, a.videos[v].frames - 1, k.hits, k.age, RF_BEST_FINISH);
    }
    if (i == 0) a.best_counts[0] = s_count;
}

// One CTA per (emission k, frame f): the u8 source crop into the caller's buffer, converted as k_align_faces converts it.
__global__ void __launch_bounds__(EMIT_THREADS) k_best_emit(const BestArgs a) {
    const int f = blockIdx.y, k = blockIdx.x, T = a.max_tracks;
    if (k >= a.best_counts[f]) return;
    const int src = a.src[(size_t)f * T + k];
    const unsigned char *from = src >= 0 ? a.store_crops + (size_t)src * a.u8.crop_bytes : a.scratch + (size_t)(-1 - src) * a.u8.crop_bytes;
    unsigned char *to = static_cast<unsigned char *>(a.out.crops) + ((size_t)f * T + k) * a.out.crop_bytes;
    const int cw = a.out.crop_w, ch = a.out.crop_h, qpr = (cw + 3) >> 2;
    for (int qd = threadIdx.x; qd < ch * qpr; qd += blockDim.x) {
        const int r = qd / qpr, x4 = (qd - r * qpr) * 4;
        int v[4][3];
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const int x = min(x4 + c, cw - 1);
            const unsigned char *p = from + ((size_t)r * cw + x) * 3;
            v[c][0] = p[0]; v[c][1] = p[1]; v[c][2] = p[2];
        }
        store_quad(a.out, to, r, x4, v);
    }
}

// Grid-stride over the records that may be seen: a scratch crop that became a slot's best goes to the store.
__global__ void __launch_bounds__(BEST_THREADS) k_best_commit(const BestArgs a, int n) {
    __shared__ int s_first[TRACK_MAX_FRAMES + 1];
    record_prefix(a, n, s_first);
    const size_t bytes = a.u8.crop_bytes;
    for (int c = blockIdx.x; c < s_first[n]; c += gridDim.x) {
        const size_t fj = record_of(s_first, c, a.max_faces);
        const int dst = a.commit[fj];
        if (dst < 0) continue;
        const unsigned char *from = a.scratch + fj * bytes;
        unsigned char *to = a.store_crops + (size_t)dst * bytes;
        if ((bytes & 15) == 0) {         // cudaMalloc'd bases, whole crops apart
            const uint4 *f16 = reinterpret_cast<const uint4 *>(from);
            uint4 *t16 = reinterpret_cast<uint4 *>(to);
            for (size_t w = threadIdx.x; w < bytes / 16; w += blockDim.x) t16[w] = f16[w];
        } else {
            for (size_t b = threadIdx.x; b < bytes; b += blockDim.x) to[b] = from[b];
        }
    }
}

int select_threads(int T) { return (T + 31) / 32 * 32; }

}  // namespace

// The four kernels of a detect chunk; k_best_select's instantiation from `l` (NULL: f11's).
static cudaError_t best_frames(const BestArgs &a, const BestTable &t, const BestLiveArgs *l, cudaStream_t s) {
    if (t.n <= 0) return cudaSuccess;
    const int T = a.max_tracks;
    bool oriented = false;
    for (int i = 0; i < t.n; i++) oriented |= t.img[i].orient != 0;
    if (oriented) k_best_measure<true><<<4 * a.num_sms, BEST_THREADS, 0, s>>>(a, t);
    else k_best_measure<false><<<4 * a.num_sms, BEST_THREADS, 0, s>>>(a, t);     // one wave: ~40 faces x 14 bands of a batch-8 call
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (l) k_best_select<true, true><<<t.nvideos, select_threads(T), sizeof(int) * 2 * T, s>>>(a, t, *l);
    else k_best_select<false, true><<<t.nvideos, select_threads(T), sizeof(int) * 2 * T, s>>>(a, t, BestLiveArgs{});
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    k_best_emit<<<dim3(T, t.n), EMIT_THREADS, 0, s>>>(a);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    k_best_commit<<<a.num_sms, BEST_THREADS, 0, s>>>(a, t.n);
    return cudaGetLastError();
}

cudaError_t launch_best_frames(const BestArgs &a, const BestTable &t, cudaStream_t s) { return best_frames(a, t, nullptr, s); }

cudaError_t launch_best_frames_live(const BestArgs &a, const BestTable &t, const BestLiveArgs &l, cudaStream_t s) { return best_frames(a, t, &l, s); }

cudaError_t launch_best_follow(const BestArgs &a, const BestTable &t, cudaStream_t s) {
    if (t.n <= 0) return cudaSuccess;
    const int T = a.max_tracks;
    k_best_select<false, false><<<t.nvideos, select_threads(T), sizeof(int) * 2 * T, s>>>(a, t, BestLiveArgs{});
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_best_emit<<<dim3(T, t.n), EMIT_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_best_finish(const BestArgs &a, int video, const TrackState *state, cudaStream_t s) {
    const int T = a.max_tracks;
    k_best_finish<<<1, select_threads(T), sizeof(int) * T, s>>>(a, video, state);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    k_best_emit<<<dim3(T, 1), EMIT_THREADS, 0, s>>>(a);
    return cudaGetLastError();
}

}  // namespace rf
