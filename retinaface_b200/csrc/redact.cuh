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
#pragma once
#include <type_traits>

#include "common.cuh"

namespace rf {

constexpr int REDACT_MAX_BLOCKS = 32, REDACT_THREADS = 256, REDACT_BAND = 16;

// Writable frame descriptors (the read-only YuvPlanes / BgrRows of the detect paths stay const).
struct YuvPlanesW {
    uint8_t *y, *u, *v;
    int y_pitch, uv_pitch, uv_step;
};
struct BgrRowsW {
    uint8_t *p;
    int pitch;
};

// One frame of a call: its pixels, size, and the factor its records map back by (1 for records already in frame pixels).
template <typename Dst>
struct RedactFrameT {
    Dst dst;
    int w, h;
    float scale;
};
// Frames per launch: the table travels as a __grid_constant__ kernel parameter within the classic 4 KB (static_assert in redact.cu).
template <typename Dst> constexpr int redact_table_limit() { return std::is_same<Dst, BgrRowsW>::value ? 64 : 32; }

// One region: the snapped rectangle [x0, x1) x [y0, y1) (unclamped), cell side c, cells across nx, the first cell row inside the
// frame, and the region's first work item of measure / apply within its frame.
struct RedactRegion {
    int x0, y0, x1, y1, c, nx, cr0, m_first, a_first, pad;
};

struct RedactArgs {
    int n, blocks, max_faces, max_tracks, cap;   // cap: regions per frame, max_faces + max_tracks
    double margin;
    const rf_det *dets;                          // [n][max_faces]
    const int *counts;                           // [n]
    const rf_track *tracks;                      // optional [n][max_tracks]
    const int *track_counts;                     // [n] with tracks
    RedactRegion *regions;                       // [n][cap]
    int *totals;                                 // [n][4]: regions, measure items, apply items, pad
    uint8_t *cells;                              // [n][cap][blocks^2][3]
};

// Scratch bytes of a call of n frames with `cap` regions each (the layout redact_carve cuts).
size_t redact_scratch_bytes(int n, int cap, int blocks);
void redact_carve(RedactArgs &a, void *scratch);
// The three kernels of every chunk of redact_table_limit<Dst>() frames, in order on s.
template <typename Dst>
cudaError_t launch_redact(const RedactArgs &a, const RedactFrameT<Dst> *frames, int num_sms, cudaStream_t s);

}  // namespace rf
