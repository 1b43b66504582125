// lookback.cuh -- f15 look-back redaction (rf_b200.h rf_detect_yuv_redact_lookback_device): each video's last L frames kept on the
// device, every frame emitted L frames late and covered where the faces born in the following L frames already were.  Per call, on the
// forward's stream inside the tracker's event chain, after the track update:
//   k_lookback_log    one CTA per frame: the frame's (a) + (b) boxes, its births and its rf_motion into the video's log slot
//   k_lookback_swap   one launch over all frames: each thread moves one 16-byte chunk of a plane row -- the buffered frame out, the
//                     input in -- so an out frame equal to its input frame is safe
//   k_lookback_boxes  one CTA per emitted frame: its (a) + (b) + (c) boxes as rf_det records of scale 1, for f12 / f14's kernels
#pragma once
#include "common.cuh"

namespace rf {

constexpr int LOOKBACK_MAX_L = 64;
constexpr int LOOKBACK_TABLE = 32;        // frames per launch: the tables travel as __grid_constant__ parameters
constexpr int LOOKBACK_THREADS = 256;

// A log slot: this head, then float4 boxes[max_faces + max_tracks] ((a) then (b), frame pixels), then LookbackBirth[min(F, T)].
struct LookbackHead {
    int nab, nbirth, status, pad;         // status: the frame's rf_motion status (RF_MOTION_FIRST without motion)
    double m[6];
};
struct LookbackBirth {
    int id;
    float x1, y1, x2, y2;
};
size_t lookback_slot_bytes(int max_faces, int max_tracks);
// Records per emitted frame: (a) + (b) + L births of at most min(max_faces, max_tracks) each.
inline int lookback_records(int max_faces, int max_tracks, int L) { return max_faces + max_tracks + L * (max_faces < max_tracks ? max_faces : max_tracks); }

struct LookbackArgs {
    const rf_det *dets;           // [n][max_faces] the call's records
    const int *counts;            // [n]
    const rf_track *tracks;       // [n][max_tracks] the call's track lists
    const int *track_counts;      // [n]
    const rf_motion *motion;      // [n], NULL without motion
    int max_faces, max_tracks;
    size_t slot_bytes;            // lookback_slot_bytes
    int ring;                     // log slots per video: 2 L (a call holds frames num - L .. num + L - 1 of a video)
    double grow;
    rf_det *out;                  // [emitted][records]
    int *out_counts;              // [emitted]
    int records;
};

// k_lookback_log: frame i0 + k of the call into log slot `slot[k]`.
struct LookbackLogTable {
    int n, i0;
    float scale[LOOKBACK_TABLE];
    uint8_t *slot[LOOKBACK_TABLE];
};

// k_lookback_boxes: emitted frame k of the launch is frame e of the video whose log ring is `log[k]`, e in ring slot e_slot[k], with
// births taken from frames e + 1 .. e + span[k]; its records go to out[(j0 + k) * records].
struct LookbackBoxTable {
    int n, j0;
    const uint8_t *log[LOOKBACK_TABLE];
    int e_slot[LOOKBACK_TABLE], span[LOOKBACK_TABLE];
};

// k_lookback_swap: one frame, its planes as the caller lays them out and its buffer slot (packed: luma w x h, then the chroma as the
// frame lays it out -- one interleaved w x h/2 plane from its first byte, or U then V, w/2 x h/2 each).  out[0] NULL: the frame
// emits nothing (it only stores); in NULL: a drain (it only emits).
struct LookbackSwapFrame {
    const uint8_t *in[2];         // luma, chroma (semi-planar: its first byte; planar: U, with V at in_v)
    const uint8_t *in_v;
    uint8_t *out[2], *out_v;
    uint8_t *slot;
    int in_pitch[2], out_pitch[2];
    int w, h, planar;
};
struct LookbackSwapTable {
    int n;
    LookbackSwapFrame f[LOOKBACK_TABLE];
};

cudaError_t launch_lookback_log(const LookbackArgs &a, const LookbackLogTable &t, cudaStream_t s);
// max_rows: the most plane rows of a frame of the table (h + h / 2 semi-planar, 2 h planar).
cudaError_t launch_lookback_swap(const LookbackSwapTable &t, int max_rows, cudaStream_t s);
cudaError_t launch_lookback_boxes(const LookbackArgs &a, const LookbackBoxTable &t, cudaStream_t s);

}  // namespace rf
