// align.cuh -- f5 face alignment: the crops a face recogniser takes, cut from the original images on the GPU.
//
// For every kept face of a batch, k_align_faces fits the least-squares similarity transform from the face's five landmarks
// (in original image pixels) to a template of crop-pixel targets (the ArcFace 112x112 template by default), and warps the
// ORIGINAL image into the crop exactly the way cv2.warpAffine(img, M, (cw, ch), INTER_LINEAR, BORDER_CONSTANT, 0) does
// (OpenCV's fixed point: 1/1024-pixel coordinates, 1/32-pixel bilinear phases, integer weights).  The crop is stored as
// u8 BGR HWC, or as planar RGB float32 / float16 (u8 - mean) * (1 / std), the input of an ArcFace-style recogniser.
#pragma once
#include "common.cuh"
#include "postproc.cuh"
#include "preprocess.cuh"
#include "yuv.cuh"

namespace rf {

// One source image of the batch: u8 BGR HWC rows of row_bytes, and the factor that maps network-input coordinates to its
// pixels (the float letterbox_fill returns; 1 for network-sized images).  f9: `orient` (LB_* bits, preprocess.cuh) views the
// stored rows in another orientation; w x h is then the DISPLAYED size, which the warp's bounds test uses, and displayed tap (x, y)
// reads the stored pixel the letter-box would, so a crop is cv2.warpAffine(T_o(img), M).  0: the rows as they are.
struct AlignImage {
    const uint8_t *src;
    int w, h, row_bytes;
    float scale;
    int orient;
};

struct AlignArgs {
    const AlignImage *images;   // device [n]; NULL: image i is uniform_base + i * uniform_bytes, net-sized, packed, scale 1
    const uint8_t *uniform_base;
    size_t uniform_bytes;
    int uniform_w, uniform_h;
    int n, max_align;           // slots per image: crop j of image i is slot i * max_align + j, j < min(count_i, max_align)
    int crop_w, crop_h, format; // RF_CROP_*
    float mean, inv_std;
    double tmpl[10];            // template points (x0, y0 .. x4, y4), crop pixels
    size_t crop_bytes;          // align_crop_bytes(crop_w, crop_h, format)
    void *crops;                // [n][max_align][crop bytes]
    double *mats;               // optional [n][max_align][6]: M, image -> crop
};

// f6: one YUV 4:2:0 video frame of the batch (yuv.cuh), read in place; a.images / a.uniform_* are unused.  Each tap of the warp
// is converted to BGR first, so a crop is cv2.warpAffine(cv2.cvtColor(frame), M) byte for byte.
struct AlignYuvImage {
    YuvPlanes p;
    int w, h;           // displayed size
    float scale;
    int orient;         // LB_* bits, as AlignImage
};

constexpr int ALIGN_MIN_SIDE = 8, ALIGN_MAX_SIDE = 512, ALIGN_MAX_FRAMES = 32;

size_t align_crop_bytes(int crop_w, int crop_h, int format);
// One launch, the grid sized from the SM count: kept counts and landmarks are read from pb on the device, and only the crops
// that exist are cut.  n <= max_batch (<= 4096: the per-image scan lives in 4 n bytes of shared memory).
cudaError_t launch_align_faces(const AlignArgs &a, const PostBuffers &pb, int num_sms, cudaStream_t s);
// The same over a.n YUV frames [n]: the frame table travels as a kernel parameter (no host table a later call could rewrite
// before the copy ran), one launch per ALIGN_MAX_FRAMES frames.
// oriented (f9): the frames' `orient` bits apply (a separate instantiation; false reads the frames as stored).
cudaError_t launch_align_faces_yuv(const AlignArgs &a, const AlignYuvImage *frames, const PostBuffers &pb, int num_sms, cudaStream_t s,
                                   bool oriented = false);
// f8: the same over a.n BGR images [n] (a.images / a.uniform_* unused), the table a kernel parameter as the frames are above: an
// asynchronous call cannot have its table rewritten by a later one.  The tiled paths pass scale 1 (their records are already in
// image pixels; __fmul_rn(l, 1.f) is exact).
cudaError_t launch_align_faces(const AlignArgs &a, const AlignImage *images, const PostBuffers &pb, int num_sms, cudaStream_t s,
                               bool oriented = false);

}  // namespace rf
