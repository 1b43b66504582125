// lookback.cuh -- f15 look-back redaction (rf_b200.h rf_detect_yuv_redact_lookback_device): each video's last L frames kept on the
// device, every frame emitted L frames late and covered where the faces born in the following L frames already were.  Per call, on the
// forward's stream inside the tracker's event chain, after the track update:
//   k_lookback_log    one CTA per frame: the frame's (a) + (b) boxes, its births and its rf_motion into the video's log slot
//                     (f18: also a follow frame's, whose (a) are its OK-followed faces and which has no births)
//   k_lookback_swap   one launch over all frames: each thread moves one 16-byte chunk of a plane row -- the buffered frame out, the
//                     input in -- so an out frame equal to its input frame is safe
//   k_lookback_boxes  one CTA per emitted frame: its (a) + (b) + (c) boxes as rf_det records of scale 1, for f12 / f14's kernels
// f17 searching look-back (rf_tracker_set_lookback_search) adds, between the log and the swap (the swap overwrites the buffered frame a
// birth's last step reads):
//   k_lookback_search one CTA per (frame of the call, birth rank): the birth's template cut from the input frame into shared memory,
//                     then its chain of f16 searches back through the earlier frames of the call and the buffer (tsearch.cuh), the
//                     OK steps' boxes into the frame's log slot; k_lookback_boxes appends them as (d)
#pragma once
#include "follow.cuh"

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
// f17: a searching tracker's slot continues, from lookback_chain_offset, with float4 chain[min(F, T)][L] (each birth's OK steps'
// boxes, frame pixels) and int nok[min(F, T)] (how many of its first steps are OK).
__host__ __device__ inline size_t lookback_chain_offset(int max_faces, int max_tracks) {
    return (sizeof(LookbackHead) + 16 * (size_t)(max_faces + max_tracks) + sizeof(LookbackBirth) * (size_t)(max_faces < max_tracks ? max_faces : max_tracks) +
            15) & ~(size_t)15;
}
// search_L: L on a searching tracker, else 0.
size_t lookback_slot_bytes(int max_faces, int max_tracks, int search_L);
// Records per emitted frame: (a) + (b) + L births of at most min(max_faces, max_tracks) each, twice that on a searching tracker ((c)
// and (d)).
inline int lookback_records(int max_faces, int max_tracks, int L, bool search) {
    return max_faces + max_tracks + (search ? 2 : 1) * L * (max_faces < max_tracks ? max_faces : max_tracks);
}

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
    int search;                   // f17: R of a searching tracker, else 0 (k_lookback_boxes then appends no (d))
    int L;
    float max_mad;
    rf_follow *steps;             // k_lookback_search: [n][min(F, T)][L] the call's step records and [n][min(F, T)] chain lengths
    int *lengths;
};

// k_lookback_log: frame i0 + k of the call into log slot `slot[k]`.  per_frame: (a)'s records per frame of a.dets and their cap --
// max_faces on a detect call (the forward's records), max_tracks on an f18 follow call (the OK-followed faces).
struct LookbackLogTable {
    int n, i0, per_frame;
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

// k_lookback_search: the call's frames grouped by video, each video's frames of the launch consecutive and in number order.  Frame
// first + j of video v is number num0 + j; a step on frame e reads frame first + (e - num0) of the table when e >= num0, else the
// buffer slot e mod L (luma first, pitch w).
constexpr int LOOKBACK_SEARCH_FRAMES = 64;     // a video has at most L <= 64 frames in a call
constexpr int LOOKBACK_SEARCH_VIDEOS = 32;
struct LookbackSearchFrame {
    const uint8_t *y;             // the input frame's luma and pitch
    int pitch;
    int video;                    // its entry in v[]
    int i;                        // its index in the call (the row of the step records)
};
struct LookbackSearchVideo {
    const uint8_t *buf;           // the frame buffer (L slots of frame_bytes), then the log (2 L slots)
    const uint8_t *log;
    size_t frame_bytes;
    long long num0;               // the number of the video's first frame in the table
    int w, h, first;
    int bits;                     // f20: the video's orientation (LB_* bits; w x h the displayed size), read by the oriented launch
};
struct LookbackSearchTable {
    int n, nv;
    LookbackSearchFrame f[LOOKBACK_SEARCH_FRAMES];
    LookbackSearchVideo v[LOOKBACK_SEARCH_VIDEOS];
};

// The parts of a log slot (lookback_slot_bytes).
__device__ __forceinline__ const float4 *slot_boxes(const uint8_t *slot) { return reinterpret_cast<const float4 *>(slot + sizeof(LookbackHead)); }
__device__ __forceinline__ const LookbackBirth *slot_births(const uint8_t *slot, int max_faces, int max_tracks) {
    return reinterpret_cast<const LookbackBirth *>(slot_boxes(slot) + max_faces + max_tracks);
}
// f17: the chains of a searching tracker's slot (lookback.cuh)
__device__ __forceinline__ const float4 *slot_chain(const uint8_t *slot, int max_faces, int max_tracks) {
    return reinterpret_cast<const float4 *>(slot + lookback_chain_offset(max_faces, max_tracks));
}
__device__ __forceinline__ const int *slot_nok(const uint8_t *slot, int max_faces, int max_tracks, int L) {
    return reinterpret_cast<const int *>(slot_chain(slot, max_faces, max_tracks) + (size_t)min(max_faces, max_tracks) * L);
}

cudaError_t launch_lookback_log(const LookbackArgs &a, const LookbackLogTable &t, cudaStream_t s);
// max_rows: the most plane rows of a frame of the table (h + h / 2 semi-planar, 2 h planar).
cudaError_t launch_lookback_swap(const LookbackSwapTable &t, int max_rows, cudaStream_t s);
cudaError_t launch_lookback_boxes(const LookbackArgs &a, const LookbackBoxTable &t, cudaStream_t s);
// oriented (f20): some video's bits are not 0: the frames' luma is read as displayed (a separate instantiation).
cudaError_t launch_lookback_search(const LookbackArgs &a, const LookbackSearchTable &t, cudaStream_t s, bool oriented = false);
cudaError_t launch_lookback_search_oriented(const LookbackArgs &a, const LookbackSearchTable &t, cudaStream_t s);     // oriented_search.cu

}  // namespace rf
