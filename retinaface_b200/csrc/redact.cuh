// redact.cuh -- f12 redaction (rf_b200.h rf_redact_yuv_device): an in-place mosaic of every region of a frame -- its records and its
// LOST tracks -- on YUV 4:2:0 frames and u8 BGR images, exactly as the header defines it.  Per chunk of frames, three launches in
// order on one stream, so every read of `measure` precedes every write of `apply`:
//   k_redact_regions  one CTA per frame: the frame's region table (snapped rectangle, cell side, first work item of each kernel below)
//                     in region order, and the frame's totals
//   k_redact_measure  grid-stride over (frame, region, cell row): the u8 cell means of the original samples
//   k_redact_apply    grid-stride over (frame, region, band of rows): every pixel of the band no lower-index region covers takes its
//                     cell value; luma first, then chroma
// The counts are only known on the device: every CTA of measure / apply scans the frames' totals and strides over the work that
// exists, so unused max_faces capacity costs nothing.
// f20 oriented frames (YuvPlanesWO) run one more instantiation of each kernel: every position, cell, ellipse and blur tap is that of
// the displayed frame, and only the byte each sample is read from or written to moves.
// f14 styles (rf_redact_style) keep the regions kernel and the order.  MOSAIC with ELLIPSE runs measure unchanged and an apply that
// tests each region's ellipse.  BLUR replaces measure with
//   k_redact_blur     grid-stride over (frame, region, plane, strip of BLUR_W columns x band of BLUR_H rows): the triple-box blur of
//                     the ORIGINAL plane, written for every sample the region owns into the frame's scratch planes
// and its apply copies every owned sample from the scratch planes into the frame.
#pragma once
#include <type_traits>

#include "common.cuh"

namespace rf {

constexpr int REDACT_MAX_BLOCKS = 32, REDACT_THREADS = 256, REDACT_BAND = 16;
constexpr int REDACT_MOSAIC = 1, REDACT_BLUR = 2, REDACT_RECT = 1, REDACT_ELLIPSE = 2;
constexpr int BLUR_MAX_DETAIL = 64, BLUR_MAX_RADIUS = 127;

// Writable frame descriptors (the read-only YuvPlanes / BgrRows of the detect paths stay const).
struct YuvPlanesW {
    uint8_t *y, *u, *v;
    int y_pitch, uv_pitch, uv_step;
};
struct BgrRowsW {
    uint8_t *p;
    int pitch;
};
// f20: a YUV frame redacted as it is displayed.  y, u, v point at displayed sample (0, 0) of each plane (yuv.cuh plane_map's off
// applied), and displayed luma sample (x, y) is y[x * y_xs + y * y_ys], chroma u / v[x * c_xs + y * c_ys].  The kernels take it as
// their ORIENTED instantiation; RedactFrameT's w x h is then the displayed size.
struct YuvPlanesWO {
    uint8_t *y, *u, *v;
    int y_xs, y_ys, c_xs, c_ys;
};
template <typename Dst> constexpr bool kRedactYuv = !std::is_same<Dst, BgrRowsW>::value;

// One frame of a call: its pixels, size, and the factor its records map back by (1 for records already in frame pixels).
// blur: the frame's scratch planes (BLUR only; YUV: luma w x h, then U and V w/2 x h/2; BGR: 3 w x h), nullptr otherwise.
template <typename Dst>
struct RedactFrameT {
    Dst dst;
    int w, h;
    float scale;
    uint8_t *blur;
};
// Frames per launch: the table travels as a __grid_constant__ kernel parameter within the classic 4 KB (static_assert in redact.cu).
template <typename Dst> constexpr int redact_table_limit() { return std::is_same<Dst, BgrRowsW>::value ? 64 : 32; }

// One region: the snapped rectangle [x0, x1) x [y0, y1) (unclamped), cell side c, cells across nx, the first cell row inside the
// frame, and the region's first work item of measure (blur, for BLUR) / apply within its frame; rad: the blur radius a (0 for MOSAIC).
struct RedactRegion {
    int x0, y0, x1, y1, c, nx, cr0, m_first, a_first, rad;
};

struct RedactArgs {
    int n, blocks, max_faces, max_tracks, cap;   // cap: regions per frame, max_faces + max_tracks
    int kind, shape, detail;                     // rf_redact_style resolved (f12: MOSAIC, RECT, 0)
    double margin;
    const rf_det *dets;                          // [n][max_faces]
    const int *counts;                           // [n]
    const rf_track *tracks;                      // optional [n][max_tracks]
    const int *track_counts;                     // [n] with tracks
    RedactRegion *regions;                       // [n][cap]
    int *totals;                                 // [n][4]: regions, measure items, apply items, pad
    uint8_t *cells;                              // [n][cap][blocks^2][3]
};

// Scratch plane bytes of one w x h frame for BLUR.
inline size_t blur_plane_bytes(bool yuv, int w, int h) { return yuv ? (size_t)w * h + 2 * (size_t)(w / 2) * (h / 2) : 3 * (size_t)w * h; }
// Scratch bytes of a call of n frames with `cap` regions each (the layout redact_carve cuts).
size_t redact_scratch_bytes(int n, int cap, int blocks);
void redact_carve(RedactArgs &a, void *scratch);
// The three kernels of every chunk of redact_table_limit<Dst>() frames, in order on s.
template <typename Dst>
cudaError_t launch_redact(const RedactArgs &a, const RedactFrameT<Dst> *frames, int num_sms, cudaStream_t s);

}  // namespace rf
