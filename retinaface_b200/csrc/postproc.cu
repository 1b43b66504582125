// postproc.cu -- GPU post-process of librf_b200: predictor 1x1 convs + softmax + threshold +
// anchor decode + clip (fused, all FPN levels in one launch) and sort + greedy NMS.
//
// Replaces the reference's HOST post-process, retinaface/RetinaFace.cpp:
//   :666-687  blob gather (second half of cls_prob = P(face))         -> k_head_decode / k_blob_decode
//   :689-723  threshold-first decode loop                              -> decode_one()
//   :378-398  bbox_pred, :179-199 clip_boxes, :418-432 landmark_pred   -> decode_one()
//   :127-154  anchors_plane (computed on the fly from (k, ih, iw))     -> decode_one()
//   :434-492  CompareBBox sort + greedy nms                            -> k_nms
// so that no head tensor (527 KB / image at 448x448) ever leaves the GPU.
//
// Bit-exactness contract: given identical head values, candidate selection, kept-face
// selection and order are identical to the reference's; scores and landmarks are bit-identical;
// box corners may differ by <= 1 ulp where the reference's expf (libm) is not correctly rounded
// (we round exp() computed in double).  Every float operation below therefore spells its
// rounding (__fmul_rn/__fadd_rn: no FMA contraction; the file is also built with -fmad=false),
// and the `0.5 * (x - 1.0)` sub-expressions run in double like the reference's C++ does.
// Ties in score (std::sort leaves them unspecified) are broken by emission order.
#include <algorithm>
#include <cmath>

#include "postproc_dev.cuh"
#include "preprocess.cuh"

namespace rf {

namespace {

constexpr int NMS_THREADS = 512;

struct HeadLaunch {
    const void *feat[3];
    HeadWeights hw[3];
    LevelDesc lv[3];
    int blk_base[4];   // first block of each level (level-aligned blocks)
    float *blobs[9];
};

// One thread per feature-map pixel; a block never straddles levels so its shared memory holds
// exactly one level's 32x64 predictor weights.
template <typename T, bool WRITE_BLOBS>
__global__ void __launch_bounds__(128) k_head_decode(HeadLaunch L, int net_w, int net_h,
                                                     const PostParams *__restrict__ params, PostBuffers pb, int fuse_nms) {
    __shared__ __align__(16) float sw[32 * 64];
    __shared__ float sb[32];
    __shared__ int s_last;
    const int blk = blockIdx.x;
    const int l = blk >= L.blk_base[2] ? 2 : (blk >= L.blk_base[1] ? 1 : 0);
    const LevelDesc lv = L.lv[l];
    pdl_trigger();
    for (int i = threadIdx.x; i < 32 * 64; i += blockDim.x) sw[i] = L.hw[l].w[i];   // weights: independent of the previous kernel
    if (threadIdx.x < 32) sb[threadIdx.x] = L.hw[l].b[threadIdx.x];
    __syncthreads();
    pdl_wait();
    const int hw = lv.h * lv.w;
    const int j = (blk - L.blk_base[l]) * blockDim.x + threadIdx.x;
    const int img = blockIdx.y;
    if (j < hw) {
    const float thr = params->score_thr;
    const T *f = reinterpret_cast<const T *>(L.feat[l]) + ((size_t)img * hw + j) * 64;
    float x[64];
#pragma unroll
    for (int g = 0; g < 8; g++) {
        Vec8<T> v;
        v.load(f + g * 8);
        v.to_float(&x[g * 8]);
    }
    if (sizeof(T) == 1) {                 // int8 features: dequantise with the concat tensor's scale
        const float sc = L.hw[l].in_scale;
#pragma unroll
        for (int c = 0; c < 64; c++) x[c] = __fmul_rn(x[c], sc);
    }
    auto dot = [&](int o) -> float {
        float acc = sb[o];
        const float4 *w4 = reinterpret_cast<const float4 *>(&sw[o * 64]);
#pragma unroll
        for (int c = 0; c < 16; c++) {
            float4 w = w4[c];
            acc = __fmaf_rn(x[4 * c + 0], w.x, acc);
            acc = __fmaf_rn(x[4 * c + 1], w.y, acc);
            acc = __fmaf_rn(x[4 * c + 2], w.z, acc);
            acc = __fmaf_rn(x[4 * c + 3], w.w, acc);
        }
        return acc;
    };
    float s[4];
#pragma unroll
    for (int o = 0; o < 4; o++) s[o] = dot(o);
    // Softmax over the (N,2,2h,w) view (prototxt:1448-1483): anchor a pairs channel a (bg) with a+2 (face).
    float pf[2], pbg[2];
#pragma unroll
    for (int a = 0; a < 2; a++) softmax_pair(s[a], s[a + 2], pbg[a], pf[a]);
    const int ih = j / lv.w, iw = j % lv.w;
    if (WRITE_BLOBS) {
        float *cls = L.blobs[3 * l] + (size_t)img * 4 * hw;
        cls[0 * hw + j] = pbg[0]; cls[1 * hw + j] = pbg[1]; cls[2 * hw + j] = pf[0]; cls[3 * hw + j] = pf[1];
    }
#pragma unroll
    for (int a = 0; a < 2; a++) {
        const bool pass = !(pf[a] <= thr);   // reference: `if (conf <= threshold) continue;`
        if (!pass && !WRITE_BLOBS) continue;
        float reg[4], lm[10];
#pragma unroll
        for (int c = 0; c < 4; c++) reg[c] = dot(4 + a * 4 + c);
#pragma unroll
        for (int c = 0; c < 10; c++) lm[c] = dot(12 + a * 10 + c);
        if (WRITE_BLOBS) {
            float *bb = L.blobs[3 * l + 1] + (size_t)img * 8 * hw;
            float *lb = L.blobs[3 * l + 2] + (size_t)img * 20 * hw;
#pragma unroll
            for (int c = 0; c < 4; c++) bb[(a * 4 + c) * hw + j] = reg[c];
#pragma unroll
            for (int c = 0; c < 10; c++) lb[(a * 10 + c) * hw + j] = lm[c];
        }
        if (pass) {
            rf_det d;
            decode_one(pf[a], reg, lm, lv, a, ih, iw, net_w, net_h, lv.anchor_base + a * hw + j, d);
            append_candidate(pb, img, d);
        }
    }
    }
    if (fuse_nms) {
        // decode -> NMS in ONE launch: the block that finishes an image's last pixels sorts and suppresses it (last-block pattern;
        // the counter cleans itself for the next forward)
        __shared__ NmsSmem S;
        extern __shared__ int s_kept[];
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) s_last = atomicAdd(&pb.tile_done[img], 1) == (int)gridDim.x - 1;
        __syncthreads();
        if (s_last) {
            __threadfence();
            nms_image<128, true>(img, threadIdx.x, params->nms_thr, params, pb, S, s_kept, [] { __syncthreads(); });
            if (threadIdx.x == 0) pb.tile_done[img] = 0;
        }
    }
}

struct BlobLaunch {
    const float *blobs[9];
    LevelDesc lv[3];
};

// rf_postprocess: one thread per anchor, reading caller-supplied NCHW head blobs.
__global__ void __launch_bounds__(256) k_blob_decode(BlobLaunch L, int net_w, int net_h,
                                                     const PostParams *__restrict__ params, PostBuffers pb) {
    pdl_trigger();
    pdl_wait();
    const int e = blockIdx.x * blockDim.x + threadIdx.x;  // emission index within the image
    if (e >= pb.anchors_per_image) return;
    const int img = blockIdx.y;
    const int l = e >= L.lv[2].anchor_base ? 2 : (e >= L.lv[1].anchor_base ? 1 : 0);
    const LevelDesc lv = L.lv[l];
    const int hw = lv.h * lv.w;
    const int r = e - lv.anchor_base;
    const int num = r / hw, j = r % hw;
    const float *cls = L.blobs[3 * l] + (size_t)img * 4 * hw;
    const float conf = cls[(2 + num) * hw + j];
    if (conf <= params->score_thr) return;
    const float *bb = L.blobs[3 * l + 1] + (size_t)img * 8 * hw;
    const float *lb = L.blobs[3 * l + 2] + (size_t)img * 20 * hw;
    float reg[4], lm[10];
#pragma unroll
    for (int c = 0; c < 4; c++) reg[c] = bb[(num * 4 + c) * hw + j];
#pragma unroll
    for (int c = 0; c < 10; c++) lm[c] = lb[(num * 10 + c) * hw + j];
    rf_det d;
    decode_one(conf, reg, lm, lv, num, j / lv.w, j % lv.w, net_w, net_h, e, d);
    append_candidate(pb, img, d);
}

// One CTA per image: sort + greedy NMS (postproc_dev.cuh nms_image).
__global__ void __launch_bounds__(NMS_THREADS) k_nms(const PostParams *__restrict__ params, PostBuffers pb) {
    extern __shared__ int s_kept[];                         // [max_faces]
    __shared__ NmsSmem S;
    pdl_trigger();
    pdl_wait();
    nms_image<NMS_THREADS, false>(blockIdx.x, threadIdx.x, params->nms_thr, params, pb, S, s_kept, [] { __syncthreads(); });
}


// ---- views and tiles -> candidate lists in image coordinates (postproc.cuh) ------------------------------------------------
// (x + origin) * map_back; the addition is skipped for origin 0 so that -0 stays -0 (views: the reference's map-back exactly)
__device__ __forceinline__ float map_back(float x, float origin, float mb) { return __fmul_rn(origin != 0.f ? __fadd_rn(x, origin) : x, mb); }

// One launch merges up to MERGE_MAX_SOURCES batch slots, first .. first + nsrc - 1; the descriptors travel as a __grid_constant__
// parameter, within the classic 4 KB parameter space together with the two PostBuffers.
constexpr int MERGE_MAX_SOURCES = 40;
struct MergeSet {
    int first, nsrc;
    MergeSource src[MERGE_MAX_SOURCES];
};
static_assert(sizeof(MergeSet) + 2 * sizeof(PostBuffers) + 8 <= 4096, "merge launch exceeds the classic 4 KB kernel parameter space");

template <bool ORIENTED>
__global__ void __launch_bounds__(256) k_merge(PostBuffers src, const __grid_constant__ MergeSet ms, int net_w, int net_h, PostBuffers dst) {
    const MergeSource &m = ms.src[blockIdx.x];
    const int b = ms.first + blockIdx.x;
    const int n = min(src.out_counts[b], src.max_faces);
    const float sc = m.map_back, wm1 = m.img_w_minus1;
    const bool flip = ORIENTED ? lb_mirrored(m.flip) : m.flip != 0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const rf_face f = src.out_dets[(size_t)b * src.max_faces + j].face;
        const float cx = __fmul_rn(__fadd_rn(f.x1, f.x2), 0.5f), cy = __fmul_rn(__fadd_rn(f.y1, f.y2), 0.5f);
        if (!(cx >= m.own_x0 && cx < m.own_x1 && cy >= m.own_y0 && cy < m.own_y1)) continue;     // another tile owns it
        if (((m.shared_sides & RF_TILE_SIDE_LEFT) && f.x1 <= 0.f) || ((m.shared_sides & RF_TILE_SIDE_TOP) && f.y1 <= 0.f) ||
            ((m.shared_sides & RF_TILE_SIDE_RIGHT) && f.x2 >= (float)(net_w - 1)) ||
            ((m.shared_sides & RF_TILE_SIDE_BOTTOM) && f.y2 >= (float)(net_h - 1)))
            continue;                                                                              // cut by a tile edge
        rf_det d;
        d.face.score = f.score;
        const float x1 = map_back(f.x1, m.x0, sc), x2 = map_back(f.x2, m.x0, sc);    // RetinaFace.cpp:733-734: rect.x1 * scale ...
        if (!ORIENTED) {
            d.face.y1 = map_back(f.y1, m.y0, sc);
            d.face.y2 = map_back(f.y2, m.y0, sc);
            d.face.x1 = flip ? __fsub_rn(wm1, x2) : x1;
            d.face.x2 = flip ? __fsub_rn(wm1, x1) : x2;
        } else {
            // displayed -> stored pixels: reflect (a reflection reverses the corners' order), then transpose
            const float hm1 = m.img_h_minus1, y1 = map_back(f.y1, m.y0, sc), y2 = map_back(f.y2, m.y0, sc);
            const bool fx = m.flip & LB_FLIP_X, fy = m.flip & LB_FLIP_Y, tr = m.flip & LB_TRANSPOSE;
            const float ax1 = fx ? __fsub_rn(wm1, x2) : x1, ax2 = fx ? __fsub_rn(wm1, x1) : x2;
            const float ay1 = fy ? __fsub_rn(hm1, y2) : y1, ay2 = fy ? __fsub_rn(hm1, y1) : y2;
            d.face.x1 = tr ? ay1 : ax1; d.face.x2 = tr ? ay2 : ax2;
            d.face.y1 = tr ? ax1 : ay1; d.face.y2 = tr ? ax2 : ay2;
        }
#pragma unroll
        for (int k = 0; k < 5; k++) {
            // mirrored source: the detector's "left eye" is the subject's right one -- swap 0<->1 and 3<->4 (2 = nose)
            const int ks = flip ? (k == 0 ? 1 : k == 1 ? 0 : k == 3 ? 4 : k == 4 ? 3 : 2) : k;
            const float x = map_back(f.lx[ks], m.x0, sc);                               // :739
            if (!ORIENTED) {
                d.face.lx[k] = flip ? __fsub_rn(wm1, x) : x;
                d.face.ly[k] = map_back(f.ly[ks], m.y0, sc);
            } else {
                const float y = map_back(f.ly[ks], m.y0, sc);
                const float ax = (m.flip & LB_FLIP_X) ? __fsub_rn(wm1, x) : x, ay = (m.flip & LB_FLIP_Y) ? __fsub_rn(m.img_h_minus1, y) : y;
                const bool tr = m.flip & LB_TRANSPOSE;
                d.face.lx[k] = tr ? ay : ax;
                d.face.ly[k] = tr ? ax : ay;
            }
        }
        d.anchor_index = m.id_base + j;
        append_candidate(dst, m.image, d);
    }
}

// f23: one launch merges up to RF_MAX_VIEWS_DEV warp views (postproc.cuh RotatedSource)
struct RotatedSet {
    RotatedSource src[RF_MAX_VIEWS_DEV];
};
static_assert(sizeof(RotatedSet) + 2 * sizeof(PostBuffers) <= 4096, "rotated merge launch exceeds the classic 4 KB kernel parameter space");

__device__ __forceinline__ double affine_row(double a, double b, double c, double x, double y) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a, x), __dmul_rn(b, y)), c);
}

__global__ void __launch_bounds__(256) k_merge_rotated(PostBuffers src, const __grid_constant__ RotatedSet rs, PostBuffers dst) {
    const RotatedSource &m = rs.src[blockIdx.x];
    const int b = m.slot;
    const int n = min(src.out_counts[b], src.max_faces);
    const double *im = m.im;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const rf_face f = src.out_dets[(size_t)b * src.max_faces + j].face;
        const double cx = __dmul_rn(__dadd_rn((double)f.x1, (double)f.x2), 0.5), cy = __dmul_rn(__dadd_rn((double)f.y1, (double)f.y2), 0.5);
        const double X = affine_row(im[0], im[1], im[2], cx, cy), Y = affine_row(im[3], im[4], im[5], cx, cy);
        const double hw = __dmul_rn(__dsub_rn((double)f.x2, (double)f.x1), m.half_inv), hh = __dmul_rn(__dsub_rn((double)f.y2, (double)f.y1), m.half_inv);
        rf_det d;
        d.face.score = f.score;
        d.face.x1 = (float)__dsub_rn(X, hw); d.face.x2 = (float)__dadd_rn(X, hw);
        d.face.y1 = (float)__dsub_rn(Y, hh); d.face.y2 = (float)__dadd_rn(Y, hh);
#pragma unroll
        for (int k = 0; k < 5; k++) {
            d.face.lx[k] = (float)affine_row(im[0], im[1], im[2], (double)f.lx[k], (double)f.ly[k]);
            d.face.ly[k] = (float)affine_row(im[3], im[4], im[5], (double)f.lx[k], (double)f.ly[k]);
        }
        d.anchor_index = m.id_base + j;
        append_candidate(dst, m.image, d);
    }
}

size_t nms_smem_bytes(int max_faces) { return sizeof(int) * (size_t)max_faces; }

}  // namespace

template <typename T>
cudaError_t launch_head_decode(const T *const feat[3], const HeadWeights hw[3], const LevelDesc lv[3], int n,
                        int net_w, int net_h, const PostParams *params, const PostBuffers &pb,
                        float *const blobs[9], cudaStream_t s, bool fuse_nms) {
    HeadLaunch L;
    int blk = 0;
    bool write = blobs && blobs[0];
    for (int l = 0; l < 3; l++) {
        L.feat[l] = feat[l];
        L.hw[l] = hw[l];
        L.lv[l] = lv[l];
        L.blk_base[l] = blk;
        blk += (lv[l].h * lv[l].w + 127) / 128;
    }
    L.blk_base[3] = blk;
    for (int i = 0; i < 9; i++) L.blobs[i] = write ? blobs[i] : nullptr;
    dim3 grid(blk, n);
    const size_t dyn = fuse_nms ? nms_smem_bytes(pb.max_faces) : 0;
    if (write) return launch_k(k_head_decode<T, true>, grid, dim3(128), dyn, s, L, net_w, net_h, params, pb, fuse_nms ? 1 : 0);
    return launch_k(k_head_decode<T, false>, grid, dim3(128), dyn, s, L, net_w, net_h, params, pb, fuse_nms ? 1 : 0);
}
template cudaError_t launch_head_decode<float>(const float *const[3], const HeadWeights[3], const LevelDesc[3], int, int, int,
                                        const PostParams *, const PostBuffers &, float *const[9], cudaStream_t, bool);
template cudaError_t launch_head_decode<__half>(const __half *const[3], const HeadWeights[3], const LevelDesc[3], int, int, int,
                                         const PostParams *, const PostBuffers &, float *const[9], cudaStream_t, bool);
template cudaError_t launch_head_decode<int8_t>(const int8_t *const[3], const HeadWeights[3], const LevelDesc[3], int, int, int,
                                         const PostParams *, const PostBuffers &, float *const[9], cudaStream_t, bool);

cudaError_t launch_blob_decode(const float *const blobs[9], const LevelDesc lv[3], int n, int net_w, int net_h,
                        const PostParams *params, const PostBuffers &pb, cudaStream_t s) {
    BlobLaunch L;
    for (int i = 0; i < 9; i++) L.blobs[i] = blobs[i];
    for (int l = 0; l < 3; l++) L.lv[l] = lv[l];
    dim3 grid((pb.anchors_per_image + 255) / 256, n);
    return launch_k(k_blob_decode, grid, dim3(256), 0, s, L, net_w, net_h, params, pb);
}

cudaError_t launch_nms(int n, const PostParams *params, const PostBuffers &pb, cudaStream_t s) {
    return launch_k(k_nms, dim3(n), dim3(NMS_THREADS), nms_smem_bytes(pb.max_faces), s, params, pb);
}

MergeSource view_source(int view, int max_faces, float scale, int flip, int img_w) {
    MergeSource m{};
    m.image = 0;
    m.id_base = view * max_faces;
    m.flip = flip;
    m.map_back = scale;
    m.img_w_minus1 = (float)(img_w - 1);
    m.own_x0 = m.own_y0 = -INFINITY;
    m.own_x1 = m.own_y1 = INFINITY;
    return m;
}

MergeSource oriented_view_source(int view, int max_faces, float scale, int bits, int disp_w, int disp_h) {
    MergeSource m = view_source(view, max_faces, scale, bits, disp_w);
    m.img_h_minus1 = (float)(disp_h - 1);
    return m;
}

MergeSource tile_source(int image, int tile, int max_faces, const rf_tile &t, int img_w) {
    MergeSource m{};
    m.image = image;
    m.id_base = tile * max_faces;
    m.flip = t.flip;
    m.shared_sides = t.shared_sides;
    m.x0 = (float)t.x0;
    m.y0 = (float)t.y0;
    m.map_back = t.map_back;
    m.img_w_minus1 = (float)(img_w - 1);
    m.own_x0 = (float)(t.own_x0 - t.x0); m.own_x1 = (float)(t.own_x1 - t.x0);
    m.own_y0 = (float)(t.own_y0 - t.y0); m.own_y1 = (float)(t.own_y1 - t.y0);
    // an axis held by one tile has no neighbour to hand a detection to: everything along it is owned, as rf_detect_batch keeps it
    if (!(t.shared_sides & (RF_TILE_SIDE_LEFT | RF_TILE_SIDE_RIGHT))) { m.own_x0 = -INFINITY; m.own_x1 = INFINITY; }
    if (!(t.shared_sides & (RF_TILE_SIDE_TOP | RF_TILE_SIDE_BOTTOM))) { m.own_y0 = -INFINITY; m.own_y1 = INFINITY; }
    return m;
}

cudaError_t launch_merge(const PostBuffers &src, const MergeSource *src_desc, int n, int net_w, int net_h, const PostBuffers &dst,
                         cudaStream_t s) {
    // dst.cand_count[] is zero before the first merge into it: cleared at allocation and by every k_nms on dst (self-cleaning)
    for (int b0 = 0; b0 < n; b0 += MERGE_MAX_SOURCES) {
        MergeSet ms{};
        ms.first = b0;
        ms.nsrc = std::min(MERGE_MAX_SOURCES, n - b0);
        bool oriented = false;
        for (int i = 0; i < ms.nsrc; i++) {
            ms.src[i] = src_desc[b0 + i];
            oriented |= (ms.src[i].flip & ~LB_FLIP_X) != 0;
        }
        if (oriented) k_merge<true><<<ms.nsrc, 256, 0, s>>>(src, ms, net_w, net_h, dst);
        else k_merge<false><<<ms.nsrc, 256, 0, s>>>(src, ms, net_w, net_h, dst);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_merge_rotated(const PostBuffers &src, const RotatedSource *src_desc, int n, const PostBuffers &dst, cudaStream_t s) {
    for (int i0 = 0; i0 < n; i0 += RF_MAX_VIEWS_DEV) {
        const int m = std::min(RF_MAX_VIEWS_DEV, n - i0);
        RotatedSet rs{};
        for (int i = 0; i < m; i++) rs.src[i] = src_desc[i0 + i];
        k_merge_rotated<<<m, 256, 0, s>>>(src, rs, dst);
        cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t postproc_init() {
    // static 27 KB + up to 32 KB dynamic (max_faces <= 8192) exceeds the 48 KB default: opt in once
    cudaError_t e;
    const int dyn = (int)nms_smem_bytes(8192);
#define RF_HD_ATTR(T_, W_) if ((e = cudaFuncSetAttribute(k_head_decode<T_, W_>, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn))) return e
    RF_HD_ATTR(float, true); RF_HD_ATTR(float, false); RF_HD_ATTR(__half, true); RF_HD_ATTR(__half, false); RF_HD_ATTR(int8_t, true); RF_HD_ATTR(int8_t, false);
#undef RF_HD_ATTR
    return cudaFuncSetAttribute(k_nms, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn);
}

}  // namespace rf
