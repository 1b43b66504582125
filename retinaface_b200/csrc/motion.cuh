// motion.cuh -- f13 camera-motion compensation (rf_b200.h rf_tracker_set_motion): per frame, a similarity from the previous frame of
// the same video to this one, estimated from luma thumbnails by block matching and a deterministic robust fit, every FP64 step one
// rounding in the order the header states.  k_track_update (track.cu) applies it to the tracks.
#pragma once
#include "common.cuh"
#include "postproc.cuh"
#include "track.cuh"

namespace rf {

constexpr int MOTION_THUMB = RF_MOTION_THUMB;
constexpr int MOTION_THUMB_BYTES = MOTION_THUMB * MOTION_THUMB;     // one thumbnail slot (packed rows of tw bytes)
constexpr int MOTION_BLOCK = RF_MOTION_BLOCK;
constexpr int MOTION_MAX_R = 32;
constexpr int MOTION_GRID = (MOTION_THUMB - 2) / MOTION_BLOCK;       // blocks per side at R = 1
constexpr int MOTION_MAX_BLOCKS = MOTION_GRID * MOTION_GRID;
constexpr int MOTION_REF_FIRST = -2;      // MotionFrame.ref: no reference
constexpr int MOTION_REF_STORE = -1;      //                  the video's stored thumbnail

// One frame of a call (host-decided): its luma plane, thumbnail geometry, video and reference.
// f20: xs != 1 or a negative pitch: the frame is read as displayed, luma sample (x, y) at y[x * xs + y * pitch] (yuv.cuh
// plane_map applied), and the thumbnail geometry is the displayed frame's.
struct MotionFrame {
    const uint8_t *y;
    int pitch, video, ref;        // ref: an earlier frame of the call (index), MOTION_REF_STORE or MOTION_REF_FIRST
    int D, tw, th, nbx, nby;
    float scale;                  // the records' map-back factor
    int xs;                       // 1 on a frame read as stored
};

// The frames of one launch (up to TRACK_MAX_FRAMES): frame i of the launch is call frame i0 + i.
struct MotionTable {
    int n, i0;
    MotionFrame f[TRACK_MAX_FRAMES];
};
static_assert(sizeof(MotionTable) <= 4096, "MotionTable travels as a kernel parameter");

// One block's point pair (kept) or nothing.
struct MotionBlock {
    double px, py, qx, qy;
    int kept, pad;
};

struct MotionArgs {
    uint8_t *thumbs;              // [max_batch][MOTION_THUMB_BYTES] this call's thumbnails
    uint8_t *store;               // [max_videos][MOTION_THUMB_BYTES] each video's reference
    MotionBlock *blocks;          // [max_batch][MOTION_MAX_BLOCKS]
    rf_motion *out;               // [n]
    const rf_det *dets;           // [n][max_faces] this call's records
    const int *counts;            // [n]
    int max_faces, search, min_inliers;
};

// Thumbnails, match and fit of the call's frames (tables: one per TRACK_MAX_FRAMES of them), in stream order on s.
cudaError_t launch_motion_estimate(const MotionArgs &a, const MotionTable *tables, int ntables, cudaStream_t s);
// Copies thumbnail frame[k] to the store slot of video[k], k < n (one per video of the call).
cudaError_t launch_motion_commit(const MotionArgs &a, const int *frames, const int *videos, const int *bytes, int n, cudaStream_t s);

}  // namespace rf
