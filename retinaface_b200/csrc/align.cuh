// align.cuh -- f5 face alignment: the crops a face recogniser takes, cut from the original images on the GPU.
//
// For every kept face of a batch, k_align_faces fits the least-squares similarity transform from the face's five landmarks
// (in original image pixels) to a template of crop-pixel targets (the ArcFace 112x112 template by default), and warps the
// ORIGINAL image into the crop exactly the way cv2.warpAffine(img, M, (cw, ch), INTER_LINEAR, BORDER_CONSTANT, 0) does
// (OpenCV's fixed point: 1/1024-pixel coordinates, 1/32-pixel bilinear phases, integer weights).  The crop is stored as
// u8 BGR HWC, or as planar RGB float32 / float16 (u8 - mean) * (1 / std), the input of an ArcFace-style recogniser.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "postproc.cuh"
#include "preprocess.cuh"
#include "yuv.cuh"

namespace rf {

// One source image of the batch, read in place: u8 BGR rows (BgrRows) or a YUV 4:2:0 frame (YuvPlanes; each tap of the warp is
// converted to BGR first, so a crop is cv2.warpAffine(cv2.cvtColor(frame), M) byte for byte), and the factor that maps
// network-input coordinates to its pixels (the float letterbox_fill returns; 1 for network-sized images and for records already in
// image pixels: __fmul_rn(l, 1.f) is exact).  f9: `orient` (LB_* bits, preprocess.cuh) views the stored pixels in another
// orientation; w x h is then the DISPLAYED size, which the warp's bounds test uses, and displayed tap (x, y) reads the stored pixel
// the letter-box would, so a crop is cv2.warpAffine(T_o(img), M).  0: the pixels as they are.
template <typename Src>
struct AlignImageT {
    Src src;
    int w, h;
    float scale;
    int orient;
};

struct AlignArgs {
    int n, max_align;           // slots per image: crop j of image i is slot i * max_align + j, j < min(count_i, max_align)
    int crop_w, crop_h, format; // RF_CROP_*
    float mean, inv_std;
    double tmpl[10];            // template points (x0, y0 .. x4, y4), crop pixels
    size_t crop_bytes;          // align_crop_bytes(crop_w, crop_h, format)
    void *crops;                // [n][max_align][crop bytes]
    double *mats;               // optional [n][max_align][6]: M, image -> crop
};

// Images per launch: the table travels as a kernel parameter within the classic 4 KB (static_assert in align.cu).
template <typename Src> constexpr int align_table_limit() { return std::is_same<Src, BgrRows>::value ? 64 : 32; }
constexpr int ALIGN_MIN_SIDE = 8, ALIGN_MAX_SIDE = 512;

size_t align_crop_bytes(int crop_w, int crop_h, int format);
// The crops of the a.n images of `table` [n], the grid sized from the SM count: kept counts and landmarks are read from pb on the
// device, and only the crops that exist are cut.  One launch per align_table_limit<Src>() images, each with its chunk of the table
// as a kernel parameter: no host table a later asynchronous call could rewrite before the copy ran.  oriented (f9): the images'
// `orient` bits apply (a separate instantiation; false reads the pixels as stored, with the code of the upright paths).
template <typename Src>
cudaError_t launch_align_faces(const AlignArgs &a, const AlignImageT<Src> *table, const PostBuffers &pb, int num_sms, cudaStream_t s,
                               bool oriented = false);

}  // namespace rf
