// postproc.cuh -- launch wrappers of the GPU post-process (implemented in postproc.cu).
#pragma once
#include "common.cuh"

namespace rf {

// Multi-GPU exchange of the final detections (SURVEY.md 8e), fused into the NMS: the CTA that finishes an image stores its
// kept records straight into the gather window of EVERY rank (peer device memory over NVLink, mapped through CUDA IPC),
// then raises that image's flag there.  Window of one rank: [ring][world][max_batch] x {count, flag, max_faces records}.
constexpr int RF_COMM_MAX_WORLD = RF_COMM_MAX_WORLD_SIZE;
struct CommView {
    int world, rank, ring;
    rf_det *dets[RF_COMM_MAX_WORLD];       // rank p's window: [ring][world][max_batch][max_faces]
    int *counts[RF_COMM_MAX_WORLD];        //                  [ring][world][max_batch]
    unsigned *flags[RF_COMM_MAX_WORLD];    //                  [ring][world][max_batch]  == seq once the image's records have landed
};

struct PostBuffers {
    // per image i (capacity = anchors_per_image A):
    unsigned long long *cand_keys;  // [B][A]   sort keys of candidates in append order
    rf_det *cand_recs;              // [B][A]   decoded record, indexed by anchor emission index
    int *cand_count;                // [B]      number appended (reset by the head kernel's launch wrapper)
    unsigned long long *sort_scratch;  // [B][A_pow2] global scratch for sorts that do not fit in smem
    unsigned char *flag_scratch;    // [B][A_pow2]
    rf_det *out_dets;               // [B][max_faces]
    int *out_counts;                // [B]   kept (clamped to max_faces)
    int *out_total_kept;            // [B]   kept before clamping
    int *tile_done;                 // [B]   tiles of the image finished (tile_chain.cuh last-block NMS; self-cleaning)
    int anchors_per_image;
    int anchors_pow2;
    int max_faces;
    int max_batch;
    CommView comm;                  // world <= 1: single GPU, no exchange
};

struct HeadWeights {
    const float *w;     // [32][64]: rows 0-3 cls_score, 4-11 bbox_pred, 12-31 landmark_pred
    const float *b;     // [32]
    float in_scale;     // 1 for float/half features; the concat tensor's quantisation scale for int8 features
};

// fuse_nms: the block that completes an image also sorts + suppresses it (decode -> NMS in one launch; pb.tile_done counts).
// Fused per-level predictor + decode: 1x1 convs (cls 4, bbox 8, landmark 20), the 2-way softmax,
// threshold, anchor decode, clip -> candidate append.  One launch covers all three levels.
// feat[l]: NHWC [n][h][w][64] SSH output (post concat+ReLU) in T.  blobs (optional, may be all
// NULL): the 9 NCHW float32 head blobs in engine order, for rf_forward_heads.
template <typename T>
cudaError_t launch_head_decode(const T *const feat[3], const HeadWeights hw[3], const LevelDesc lv[3], int n,
                        int net_w, int net_h, const PostParams *params, const PostBuffers &pb,
                        float *const blobs[9], cudaStream_t s, bool fuse_nms = false);

// Decode from caller-provided head blobs (device, NCHW f32, engine order): rf_postprocess.
cudaError_t launch_blob_decode(const float *const blobs[9], const LevelDesc lv[3], int n, int net_w, int net_h,
                        const PostParams *params, const PostBuffers &pb, cudaStream_t s);

// Sort candidates by (score desc, emission index asc) and run greedy NMS; one CTA per image.
cudaError_t launch_nms(int n, const PostParams *params, const PostBuffers &pb, cudaStream_t s);

// Views (SURVEY.md 8f-2) and tiles (f7): gather the kept detections of the images of one batch (src.out_dets / out_counts, network
// coordinates; batch slot b = source b) into candidate lists in original-image coordinates, one list per destination image.  Per
// source, its descriptor decides which detections survive and how they map back:
//   - owned: the centre __fmul_rn(__fadd_rn(x1, x2), 0.5f) (likewise y) lies in [own_x0, own_x1) x [own_y0, own_y1) (tile pixels);
//   - not cut: dropped if it reaches a shared side (x1 <= 0 on a shared left side, x2 >= net_w - 1 on a shared right one, ...);
//   - mapped back: x -> (x + x0) * map_back, the addition skipped when the origin is 0 (views keep the reference's map-back,
//     RetinaFace.cpp:732-738, exactly); mirrored sources are un-mirrored (x -> img_w-1 - x, box corners and left/right landmarks
//     swapped);
//   - appended to image `image` with candidate id (rf_det::anchor_index) = id_base + rank in the source.
// launch_nms(n, ..., dst) then selects across the sources of each image.  Appends are atomic and the NMS orders by (score, id), so
// the result does not depend on which launch appended first.
// src_desc[b] describes batch slot b, b < n.
constexpr int RF_MAX_VIEWS_DEV = 16;
// f9 oriented views: `flip` holds LB_* bits (preprocess.cuh) and the source is the letter-box of the DISPLAYED image T_o(img), whose
// size is img_w x img_h (minus 1).  A kept face maps back to displayed pixels as above, then to STORED pixels: x -> img_w-1 - x under
// LB_FLIP_X, y -> img_h-1 - y under LB_FLIP_Y (box corners swapped), then x and y trade places under LB_TRANSPOSE; left and right
// landmarks swap when the bits mirror.  Sources with LB_FLIP_Y or LB_TRANSPOSE run in a separate instantiation of the kernel.
struct MergeSource {
    int image, id_base, flip, shared_sides;    // shared_sides: RF_TILE_SIDE_* bits
    float x0, y0, map_back, img_w_minus1;
    float own_x0, own_y0, own_x1, own_y1;      // tile pixels; +-infinity for a view (everything owned)
    float img_h_minus1;                        // displayed height - 1 (oriented views only)
};
MergeSource view_source(int view, int max_faces, float scale, int flip, int img_w);
// a view of the image in orientation `bits`, letter-boxed from its displayed disp_w x disp_h form
MergeSource oriented_view_source(int view, int max_faces, float scale, int bits, int disp_w, int disp_h);
MergeSource tile_source(int image, int tile, int max_faces, const rf_tile &t, int img_w);   // tile: its index in the image's layout
cudaError_t launch_merge(const PostBuffers &src, const MergeSource *src_desc, int n, int net_w, int net_h, const PostBuffers &dst,
                         cudaStream_t s);
// f23 warp views (rf_b200.h rf_rotated_view): batch slot `slot`'s kept faces mapped back through iM in FP64 -- the box centre through
// iM, half sizes (x2 - x1) * half_inv and (y2 - y1) * half_inv (half_inv = 1 / (2 f)), each corner and landmark rounded to float once
// -- and appended to image `image` of dst with candidate id id_base + rank.  A table of its own, so that MergeSource keeps its size.
// One launch per RF_MAX_VIEWS_DEV sources (none for n = 0).
struct RotatedSource {
    int slot, id_base, image;
    double im[6];
    double half_inv;
};
cudaError_t launch_merge_rotated(const PostBuffers &src, const RotatedSource *src_desc, int n, const PostBuffers &dst, cudaStream_t s);

// dynamic shared memory the NMS kernel wants (set once at init)
cudaError_t postproc_init();

}  // namespace rf
