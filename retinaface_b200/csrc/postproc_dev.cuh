// postproc_dev.cuh -- device-side pieces of the post-process shared by postproc.cu (stand-alone kernels) and
// tile_chain.cuh (decode fused behind the SSH head GEMM, NMS run by the last CTA that finishes an image).
//
// Bit-exactness contract (see postproc.cu): every float operation spells its rounding (__fmul_rn / __fadd_rn: no FMA
// contraction whatever the translation unit's -fmad setting), the `0.5 * (x - 1.0)` sub-expressions run in double like the
// reference's C++ (retinaface/RetinaFace.cpp:378-398), ties in score are broken by emission order.
#pragma once
#include "postproc.cuh"

namespace rf {

constexpr int NMS_SMEM_CAP = 1024;  // candidates sorted / suppressed entirely in shared memory
constexpr int NMS_RANK_MAX = 256;   // up to here a one-pass rank sort replaces the bitonic ladder
constexpr int NMS_MASK_MAX = 64;    // up to here the whole IoU relation fits one 64-bit row per candidate: no barrier per kept face

__device__ __forceinline__ unsigned long long make_key(float score, int emit) {
    unsigned u = __float_as_uint(score);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // order-preserving float -> uint
    return ((unsigned long long)(~u) << 32) | (unsigned)emit;  // ascending key == score desc, emit asc
}

// Softmax over the (N,2,2h,w) view (prototxt:1448-1483): anchor a pairs channel a (bg) with a+2 (face).
__device__ __forceinline__ void softmax_pair(float s_bg, float s_face, float &p_bg, float &p_face) {
    const float m = fmaxf(s_bg, s_face);
    const float e0 = expf(__fsub_rn(s_bg, m)), e1 = expf(__fsub_rn(s_face, m));
    const float sum = __fadd_rn(e0, e1);
    p_bg = __fdiv_rn(e0, sum);
    p_face = __fdiv_rn(e1, sum);
}

// One anchor: RetinaFace.cpp:695-721 (+ :127-154 anchor, :378-398, :179-199, :418-432).
__device__ __forceinline__ void decode_one(float conf, const float reg[4], const float lmk[10],
                                           const LevelDesc &lv, int num, int ih, int iw, int net_w, int net_h,
                                           int emit, rf_det &d) {
    // anchors_plane: base + (iw*stride, ih*stride)   (int -> float conversions are exact here)
    const float sw = (float)(iw * lv.stride), sh = (float)(ih * lv.stride);
    const float ax1 = __fadd_rn(lv.base[4 * num + 0], sw), ay1 = __fadd_rn(lv.base[4 * num + 1], sh);
    const float ax2 = __fadd_rn(lv.base[4 * num + 2], sw), ay2 = __fadd_rn(lv.base[4 * num + 3], sh);
    const float width = __fadd_rn(__fsub_rn(ax2, ax1), 1.0f);
    const float height = __fadd_rn(__fsub_rn(ay2, ay1), 1.0f);
    const float ctr_x = (float)((double)ax1 + 0.5 * ((double)width - 1.0));
    const float ctr_y = (float)((double)ay1 + 0.5 * ((double)height - 1.0));
    const float pcx = __fadd_rn(__fmul_rn(reg[0], width), ctr_x);
    const float pcy = __fadd_rn(__fmul_rn(reg[1], height), ctr_y);
    const float pw = __fmul_rn((float)exp((double)reg[2]), width);
    const float ph = __fmul_rn((float)exp((double)reg[3]), height);
    float x1 = (float)((double)pcx - 0.5 * ((double)pw - 1.0));
    float y1 = (float)((double)pcy - 0.5 * ((double)ph - 1.0));
    float x2 = (float)((double)pcx + 0.5 * ((double)pw - 1.0));
    float y2 = (float)((double)pcy + 0.5 * ((double)ph - 1.0));
    // clip_boxes (single): x1,y1 only lower-clamped, x2,y2 only upper-clamped
    if (x1 < 0) x1 = 0;
    if (y1 < 0) y1 = 0;
    if (x2 > (float)(net_w - 1)) x2 = (float)(net_w - 1);
    if (y2 > (float)(net_h - 1)) y2 = (float)(net_h - 1);
    d.face.score = conf;
    d.face.x1 = x1; d.face.y1 = y1; d.face.x2 = x2; d.face.y2 = y2;
#pragma unroll
    for (int k = 0; k < 5; k++) {
        d.face.lx[k] = __fadd_rn(__fmul_rn(lmk[2 * k], width), ctr_x);
        d.face.ly[k] = __fadd_rn(__fmul_rn(lmk[2 * k + 1], height), ctr_y);
    }
    d.anchor_index = emit;
}

__device__ __forceinline__ void append_candidate(const PostBuffers &pb, int img, const rf_det &d) {
    const size_t base = (size_t)img * pb.anchors_per_image;
    pb.cand_recs[base + d.anchor_index] = d;
    int slot = atomicAdd(&pb.cand_count[img], 1);
    if (slot < pb.anchors_per_image) pb.cand_keys[base + slot] = make_key(d.face.score, d.anchor_index);
}

// IoU test of RetinaFace::nms (:470-487), operation by operation.
__device__ __forceinline__ bool suppresses(const float4 s, float area1, const float4 b, float thr) {
    float x = fmaxf(s.x, b.x), y = fmaxf(s.y, b.y);
    float w = __fadd_rn(__fsub_rn(fminf(s.z, b.z), x), 1.0f);
    float h = __fadd_rn(__fsub_rn(fminf(s.w, b.w), y), 1.0f);
    if (w <= 0 || h <= 0) return false;
    float area2 = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.0f), __fadd_rn(__fsub_rn(b.w, b.y), 1.0f));
    float inter = __fmul_rn(w, h);
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area1, area2), inter)) > thr;
}

// Shared-memory working set of one image's sort + greedy NMS.
struct NmsSmem {
    unsigned long long keys[NMS_SMEM_CAP];
    unsigned long long tmp[NMS_RANK_MAX];
    float4 box[NMS_SMEM_CAP];
    unsigned char flag[NMS_SMEM_CAP];
    int nkept;
};

// Sort + greedy NMS of image `img` by NT cooperating threads (tid in [0, NT)); `sync` is a barrier over exactly those
// threads (__syncthreads in k_nms, a named barrier over the epilogue warps in the tile kernel).  (1) sort the candidate keys
// (rank sort for <= 256 candidates -- one pass, no log^2 barrier ladder; bitonic above), (2) greedy suppression rounds: the
// next unsuppressed candidate is kept, then all threads test the remaining ones against it -- the same O(n * kept) work as
// the reference, parallel inside a round, (3) gather kept records.  Up to NMS_SMEM_CAP candidates live entirely in shared
// memory; beyond that (stress inputs) keys / flags use the global scratch of PostBuffers.
// `acquire`: the candidates were written by OTHER CTAs (last-block pattern): read them through L2 (__ldcg).
template <int NT, bool ACQUIRE, typename Sync>
__device__ __forceinline__ void nms_image(int img, int tid, float thr, const PostParams *params, const PostBuffers &pb, NmsSmem &S, int *s_kept, Sync sync) {
    const int A = pb.anchors_per_image;
    int n = ACQUIRE ? __ldcg(&pb.cand_count[img]) : pb.cand_count[img];
    if (n > A) n = A;
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    const bool small = np2 <= NMS_SMEM_CAP;
    unsigned long long *keys = small ? S.keys : pb.sort_scratch + (size_t)img * pb.anchors_pow2;
    unsigned char *flag = small ? S.flag : pb.flag_scratch + (size_t)img * pb.anchors_pow2;
    const unsigned long long *gkeys = pb.cand_keys + (size_t)img * A;
    const rf_det *recs = pb.cand_recs + (size_t)img * A;
    auto ldkey = [&](int i) { return ACQUIRE ? __ldcg(&gkeys[i]) : gkeys[i]; };
    auto ldbox = [&](unsigned e) {
        e = e < (unsigned)A ? e : (unsigned)A - 1u;     // a key is always an anchor index; never index past the records whatever was read
        const float *f = reinterpret_cast<const float *>(&recs[e].face);
        return ACQUIRE ? make_float4(__ldcg(f + 1), __ldcg(f + 2), __ldcg(f + 3), __ldcg(f + 4)) : make_float4(f[1], f[2], f[3], f[4]);
    };
    if (tid == 0) S.nkept = 0;

    if (n <= NMS_RANK_MAX) {
        // rank sort: keys are unique (the emission index is part of the key), so rank = #smaller keys
        for (int i = tid; i < n; i += NT) { S.tmp[i] = ldkey(i); S.flag[i] = 0; }
        sync();
        for (int i = tid; i < n; i += NT) {
            const unsigned long long k = S.tmp[i];
            int rank = 0;
            for (int j = 0; j < n; j++) rank += S.tmp[j] < k;
            S.keys[rank] = k;
        }
        sync();
    } else {
        for (int i = tid; i < np2; i += NT) {
            keys[i] = i < n ? ldkey(i) : ~0ull;
            flag[i] = 0;
        }
        sync();
        for (int k = 2; k <= np2; k <<= 1) {
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = tid; i < np2; i += NT) {
                    int ixj = i ^ j;
                    if (ixj > i) {
                        unsigned long long a = keys[i], b = keys[ixj];
                        bool up = (i & k) == 0;
                        if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
                    }
                }
                sync();
            }
        }
    }
    if (small) {
        for (int i = tid; i < n; i += NT) S.box[i] = ldbox((unsigned)(keys[i] & 0xffffffffu));
        sync();
    }
    auto box_at = [&](int i) -> float4 {
        if (small) return S.box[i];
        return ldbox((unsigned)(keys[i] & 0xffffffffu));
    };
    int nkept = 0;  // thread 0's running count (mirrored to S.nkept at the end)
    if (n <= NMS_MASK_MAX) {
        // few candidates (the usual case: tens per image): the whole suppression relation at once -- thread (i, half) tests box i
        // against 32 later boxes -> one 64-bit row per candidate; then ONE thread walks the rows.  Same greedy rule (a box is
        // suppressed only by a KEPT earlier box), no barrier per kept face.
        unsigned long long *rows = S.tmp;          // the rank sort is done with S.tmp
        for (int t = tid; t < 2 * n; t += NT) {
            const int i = t >> 1, j0 = (t & 1) * 32;
            const float4 s = S.box[i];
            const float area1 = __fmul_rn(__fadd_rn(__fsub_rn(s.z, s.x), 1.0f), __fadd_rn(__fsub_rn(s.w, s.y), 1.0f));
            unsigned bits = 0;
            for (int b = 0; b < 32; b++) {
                const int j = j0 + b;
                if (j > i && j < n && suppresses(s, area1, S.box[j], thr)) bits |= 1u << b;
            }
            reinterpret_cast<unsigned *>(rows + i)[t & 1] = bits;
        }
        sync();
        if (tid == 0) {
            unsigned long long removed = 0;
            for (int i = 0; i < n; i++) {
                if ((removed >> i) & 1ull) continue;
                if (nkept < pb.max_faces) s_kept[nkept] = i;
                nkept++;
                removed |= rows[i];
            }
        }
    } else
    for (int i = 0; i < n; i++) {
        if (flag[i]) continue;  // uniform: flags of position i are final once every earlier kept round has synchronised
        const float4 s = box_at(i);
        if (tid == 0) {
            if (nkept < pb.max_faces) s_kept[nkept] = i;
            nkept++;
        }
        const float area1 = __fmul_rn(__fadd_rn(__fsub_rn(s.z, s.x), 1.0f), __fadd_rn(__fsub_rn(s.w, s.y), 1.0f));
        for (int j = i + 1 + tid; j < n; j += NT) {
            if (!flag[j] && suppresses(s, area1, box_at(j), thr)) flag[j] = 1;
        }
        sync();
    }
    if (tid == 0) S.nkept = nkept;
    sync();
    const int total = S.nkept;
    const int kept = total < pb.max_faces ? total : pb.max_faces;
    // gather: 16 floats per record, one thread per float
    const float *src = reinterpret_cast<const float *>(recs);
    float *dst = reinterpret_cast<float *>(pb.out_dets + (size_t)img * pb.max_faces);
    const unsigned seq = pb.comm.world > 1 ? params->comm_seq : 0u;
    const size_t wslot = seq ? ((size_t)params->comm_slot * pb.comm.world + pb.comm.rank) * pb.max_batch + img : 0;
    for (int t = tid; t < kept * 16; t += NT) {
        int k = t >> 4, w = t & 15;
        unsigned e = (unsigned)(keys[s_kept[k]] & 0xffffffffu);
        const float v = ACQUIRE ? __ldcg(&src[(size_t)e * 16 + w]) : src[(size_t)e * 16 + w];
        dst[t] = v;
        if (seq)     // the same record into every rank's window (peer memory; this rank's own window included)
            for (int p = 0; p < pb.comm.world; p++) reinterpret_cast<float *>(pb.comm.dets[p] + wslot * pb.max_faces)[t] = v;
    }
    if (tid == 0) {
        pb.out_counts[img] = kept;
        pb.out_total_kept[img] = total;
        pb.cand_count[img] = 0;  // self-cleaning for the next launch
        if (seq) for (int p = 0; p < pb.comm.world; p++) pb.comm.counts[p][wslot] = kept;
    }
    if (seq) {
        __threadfence_system();  // records + count are visible system-wide before the flag
        sync();
        if (tid < pb.comm.world) *reinterpret_cast<volatile unsigned *>(&pb.comm.flags[tid][wslot]) = seq;
    }
    sync();                      // S may be reused by the caller
}

}  // namespace rf
