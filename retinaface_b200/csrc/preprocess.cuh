// preprocess.cuh -- the single preprocess kernel of librf_b200.
//
// Replaces, in one coalesced pass over the network-sized output, the reference's preprocess
// chain (retinaface/RetinaFace.cpp:593-647): cudaMemset of the resize buffer (:598), the
// resize (NPP imageROIResize8U3C, resizeconvertion.cu:279-316, or cv::resize :613-617) and
// copyMakeBorder (:614-623).  The remaining stages of that chain -- u8->f32, BGR->RGB
// (convertBGR2RGBfloat, resizeconvertion.cu:46-63) and HWC->CHW (imageSplit, :165-185) -- do
// not exist here at all: conv0 consumes the letter-boxed u8 BGR HWC image directly
// (kernels_simt.cuh k_conv0), so no float image is ever materialised.
//
// Resize definition: the reference's OpenCV branch, cv::resize(img, Size(), 1/scale, 1/scale)
// with INTER_LINEAR on 8UC3 -- OpenCV's fixed-point bilinear (coefficients rounded to 11 bits,
// horizontal pass in int, vertical pass ((b0*(S0>>4))>>16) + ((b1*(S1>>4))>>16) + 2 >> 2).
// Restated so results are BIT-IDENTICAL to cv2.resize (tests/test_preprocess.py).
// RF_FLAG_NPP_RESIZE selects the reference's OTHER branch instead (USE_NPP: imageROIResize8U3C -> nppiResizeSqrPixel_8u_C3R with
// NPPI_INTER_SUPER): coverage-weighted super-sampling with NPP's measured edge rule (preprocess.cu area_pixel; checked against
// NPP itself on a GPU box, oracle/npp_oracle.cu).
//
// The pixel source is a template parameter of the kernel: pitched u8 BGR rows (BgrRows: every BGR path), or a YUV 4:2:0 video frame
// (yuv.cuh), whose every tap -- identity, bilinear or super-sampling -- is converted to BGR before the unchanged resize
// arithmetic, so the network input is byte for byte the letter-box of cv2.cvtColor(frame).
#pragma once
#include <string>
#include <vector>

#include "common.cuh"
#include "yuv.cuh"

namespace rf {

// Host helper: output size + scale the way RetinaFace::detect + cv::resize compute them.
void letterbox_geometry(int w, int h, int net_w, int net_h, int *dw, int *dh, double *inv_scale);
// ... and the way imageROIResize8U3C + NPP do (resizeconvertion.cu:296-310): extent ceil(w f) x ceil(h f)
void letterbox_geometry_npp(int w, int h, int net_w, int net_h, int *dw, int *dh, double *inv_scale);

// The reference's own float `scale` of a letter-box into box_w x box_h (RetinaFace.cpp:587-591), the factor its map-back
// multiplies by (:732-738).
float letterbox_map_back(int w, int h, int box_w, int box_h);

// Batched letter-box: ONE launch for up to LB_MAX_IMAGES BGR images (LB_MAX_FRAMES YUV frames) per call chunk, each with its
// own source / destination buffer; 4 pixels (three 32-bit stores) per thread.  The items travel as __grid_constant__ kernel
// parameters: a chunk of either kind stays within the classic 4 KB parameter limit (static_assert in preprocess.cu).
// An item's output pixel (x, y) is pixel (x + x0, y + y0) of the whole resized image (dw x dh, zero beyond): origin 0 is the
// letter-box, another origin cuts one tile out of a resized pyramid level (tile_fill below).  scale < 1 up-scales.
constexpr int LB_MAX_IMAGES = 64, LB_MAX_FRAMES = 32;
// cv::resize(INTER_LINEAR) at exactly 2x down-scaling runs OpenCV's fast INTER_AREA code, whose border rule differs from the
// bilinear taps on a side of 3 mod 4.  Every item of OpenCV's definition at scale 2 uses it -- a letter-box or view whose binding
// side is exactly twice the box, and tile levels of scale 0.5 -- so that each is the cv::resize the header promises.
constexpr int LB_HALF_AREA = 2;
// f9 orientations.  An item's `flip` is a set of LB_* bits over the DISPLAYED image (sw x sh, the frame the taps are computed in):
// displayed pixel (x, y) reads stored pixel (x', y') with x' = FLIP_X ? sw-1-x : x, y' = FLIP_Y ? sh-1-y : y, swapped when
// TRANSPOSE.  0 / LB_FLIP_X are the plain and the mirrored view.  The EXIF orientation o (rf_b200.h) is lb_orientation_bits(o).
constexpr int LB_FLIP_X = 1, LB_FLIP_Y = 2, LB_TRANSPOSE = 4;
// EXIF orientation 1..8 -> LB_* bits (-1 outside 1..8)
inline int lb_orientation_bits(int o) {
    static const int bits[9] = {-1, 0, LB_FLIP_X, LB_FLIP_X | LB_FLIP_Y, LB_FLIP_Y, LB_TRANSPOSE, LB_TRANSPOSE | LB_FLIP_X,
                                LB_TRANSPOSE | LB_FLIP_X | LB_FLIP_Y, LB_TRANSPOSE | LB_FLIP_Y};
    return o >= 1 && o <= 8 ? bits[o] : -1;
}
// LB_* bits -> EXIF orientation 1..8, the inverse of lb_orientation_bits
inline int lb_exif(int bits) {
    static const int exif[8] = {1, 2, 4, 3, 5, 6, 8, 7};
    return exif[bits & 7];
}
// f25: the composition of two EXIF transforms, another EXIF transform: T_{exif_compose(inner, outer)}(S) = T_outer(T_inner(S)), so a
// view in orientation `outer` of a frame displayed in orientation `inner` reads the stored frame through one orientation.  Row
// inner - 1, column outer - 1 (tests/test_rotated_track_cpu.py checks all 64 pairs against oracle/orient.py).
constexpr int kExifCompose[8][8] = {
    {1, 2, 3, 4, 5, 6, 7, 8}, {2, 1, 4, 3, 8, 7, 6, 5}, {3, 4, 1, 2, 7, 8, 5, 6}, {4, 3, 2, 1, 6, 5, 8, 7},
    {5, 6, 7, 8, 1, 2, 3, 4}, {6, 5, 8, 7, 4, 3, 2, 1}, {7, 8, 5, 6, 3, 4, 1, 2}, {8, 7, 6, 5, 2, 1, 4, 3},
};
inline int exif_compose(int inner, int outer) { return kExifCompose[inner - 1][outer - 1]; }
// whether the orientation bits mirror the image (an odd number of reflections: left and right landmarks trade places)
__host__ __device__ inline bool lb_mirrored(int bits) { return ((bits & 1) ^ ((bits >> 1) & 1) ^ ((bits >> 2) & 1)) != 0; }
// u8 BGR rows `pitch` bytes apart, read in place: an upload into a raw buffer (pitch 3 w), a JPEG decode, or a caller's device
// image that may be a view of a larger allocation (f8)
struct BgrRows {
    const uint8_t *p;
    int pitch;
};
template <typename Src>
struct LbItemT {
    using Source = Src;
    Src src; uint8_t *dst;
    int sw, sh, dw, dh;   // sw x sh: the DISPLAYED source size (stored h x w when LB_TRANSPOSE)
    double scale;
    uint8_t identity, flip, area;   // flip: LB_* bits; area: 0 bilinear, 1 NPP super-sampling, LB_HALF_AREA OpenCV's 2x fast area path
    int16_t x0, y0;     // 16 bits keep 64 BGR items within 4 KB; origins are below the largest level side (16384)
};
using LbItem = LbItemT<BgrRows>;             // u8 BGR rows
using LbYuvItem = LbItemT<YuvPlanes>;        // a YUV 4:2:0 frame
// fills one item (geometry of either resize definition, origin 0); returns the reference's map-back factor
template <typename Src>
float letterbox_fill(LbItemT<Src> &it, typename LbItemT<Src>::Source src, int w, int h, uint8_t *dst, int box_w, int box_h, int flip, int area);
template <typename Src>
cudaError_t launch_letterbox_batch(const LbItemT<Src> *items, int n, int net_w, int net_h, cudaStream_t s);

// ---- f7 tiles (rf_b200.h rf_tile_layout) ------------------------------------------------------------------------------------------
// The one statement of the tile geometry: rf_tile_layout, the tiled detect paths and rf_preprocess_tile all call it.  Fills `out`
// with every tile of a w x h image (t may be NULL) and returns RF_OK, or a status with the reason in *err.
int tile_layout(int net_w, int net_h, int w, int h, const rf_tiling *t, std::vector<rf_tile> &out, std::string *err);
// tile_layout's refusals that hold whatever the image size -- nlevels, the overlap, then each given level's scale, with its messages
// (rf_tracker_set_tiling; levels NULL is not one of them: the tracker takes it as the default pyramid).
int tiling_check(int net_w, int net_h, const rf_tiling *t, std::string *err);
// The letter-box item of one tile: the image's level resized, mirrored when the tile's level is, and cut at the tile's origin.
// w x h is the DISPLAYED size and `bits` the image's own LB_* orientation bits (0: upright, f21); the tile's layout is that of w x h.
template <typename Src>
void tile_fill(LbItemT<Src> &it, typename LbItemT<Src>::Source src, int w, int h, int bits, uint8_t *dst, int net_w, int net_h,
               const rf_tile &tile);

// ---- f23 rotated views (rf_b200.h rf_rotated_view) -------------------------------------------------------------------------------
// The one statement of a view's geometry: the angle reduced, then either the EXIF orientation of a quarter turn (1, 8, 3, 6), or 0 and
// the warp view's fit f, M and iM = cv::invertAffineTransform(M).  Host, FP64, no FMA contraction (preprocess.cu is built so).
struct RotatedGeometry {
    int orientation;
    double f, M[6], iM[6];
};
RotatedGeometry rotated_geometry(float angle, int w, int h, int box_w, int box_h);
// One warp view: the image w x h (stored) read through iM into dst (net_h x net_w x 3), cv2.warpAffine's fixed point.
template <typename Src>
struct WarpItemT {
    Src src;
    int w, h;
    uint8_t *dst;
    double im[6];
};
using WarpItem = WarpItemT<BgrRows>;
using WarpYuvItem = WarpItemT<YuvPlanes>;     // f24: each tap converted as the letter-box converts it
constexpr int WARP_MAX_VIEWS = 16;     // items of one k_letterbox_warp launch
// k_letterbox_warp: one launch per WARP_MAX_VIEWS items (none for n = 0).  f25: bits (NULL: all 0) gives each item's LB_* orientation;
// an item with bits reads the DISPLAYED image D = T_o(src) -- its w x h the displayed size, iM of D -- through f9's map, as
// launch_align_faces(..., oriented) reads it.  A launch with some item oriented runs the oriented instantiation, else the upright one.
// Only YUV sources have one: BGR items with bits return cudaErrorNotSupported.
template <typename Src>
cudaError_t launch_letterbox_warp(const WarpItemT<Src> *items, int n, int net_w, int net_h, cudaStream_t s, const int *bits = nullptr);

}  // namespace rf
