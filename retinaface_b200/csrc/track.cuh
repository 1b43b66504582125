// track.cuh -- f10 face tracking across video frames (rf_b200.h rf_track_update): ByteTrack's association with SORT's
// constant-velocity Kalman filter, one CTA per video of a call, every step in FP64 in the order the header states.
#pragma once
#include "common.cuh"
#include "postproc.cuh"

namespace rf {

constexpr int TRACK_MAX_FRAMES = 32;     // frames per launch: the call's tables travel as a kernel parameter
constexpr int TRACK_MAX_TRACKS = 1024;
constexpr int TRACK_THREADS = 256;

// One track slot of one video (device).  id == 0: the slot is free.
struct TrackState {
    double m[4], u[4], p00[4], p01[4], p11[4];   // cx, cy, a = w / h, h
    rf_face face;                                // last matched record, frame pixels
    int id, state, hits, age, lost, det;
};

// Per video (device): ids issued (the last one), frames applied since create / reset, births skipped for want of a slot.  All zero
// after create / reset.
struct TrackVideo {
    int issued, frames, overflow, pad;
};

// A candidate pair of one stage: its IoU, the track's id and slot, the record.
struct TrackPair {
    double iou;
    int id;
    short slot, det;
};

struct TrackParams {
    int max_tracks, max_faces, max_lost;
    float high_thresh, new_thresh, iou_high, iou_low, iou_tentative;
};

// The call's host tables (one launch covers up to TRACK_MAX_FRAMES frames): frame i of the launch belongs to video[i] and maps by
// scale[i]; CTA b runs the frames of cta_video[b] in call order.
struct TrackTable {
    int n, nvideos;
    int video[TRACK_MAX_FRAMES];
    float scale[TRACK_MAX_FRAMES];
    int cta_video[TRACK_MAX_FRAMES];
};

// f11 (best.cuh): a track matched or born on a frame, at the index of its record (each such track holds a distinct record); slot -1:
// the record went to no track.
struct TrackSeen {
    int slot, id;
    rf_face face;                // the record in frame pixels, as the track keeps it
};

// f22: a track matched or born on a frame, after the frame, at the index of its record (where TrackSeen has it).
struct TrackLife {
    int hits, age, state, pad;
};

// f11: a track removed on a frame, at its slot; id 0: the slot lost no track.
struct TrackGone {
    int id, hits, age, confirmed;   // confirmed: the track was CONFIRMED at some point (its state at frame start was not TENTATIVE)
};

struct TrackArgs {
    TrackParams p;
    TrackVideo *videos;          // [max_videos]
    TrackState *state;           // [max_videos][max_tracks]
    TrackPair *pairs;            // [TRACK_MAX_FRAMES][max_tracks * max_faces]  per-CTA candidate pairs
    int *order;                  // [TRACK_MAX_FRAMES][max_tracks * max_faces]  their rank order
    const rf_det *dets;          // [n][max_faces] records of the launch's first frame
    const int *counts;           // [n]
    rf_track *tracks;            // [n][max_tracks]
    int *track_counts;           // [n]
    rf_det *due;                 // [n][max_faces] faces of the tracks confirmed on the frame, id order (crop_slot); NULL: no crops
    int *due_counts;             // [n]  min(due, max_align)
    int max_align;               // crop slots per frame (0 without crops)
    TrackSeen *seen;             // optional [n][max_faces]: every record's track on the frame (f11)
    TrackGone *gone;             // optional [n][max_tracks]: the tracks removed on the frame, by slot (f11)
    const rf_motion *motion;     // optional [n]: each frame's camera motion (f13), applied after predict when RF_MOTION_OK
    TrackLife *life;             // optional [n][max_faces]: with seen, each seen record's track after the frame (f22 live shots)
};

// n frames (videos[i], scales[i]; scales NULL: 1), one launch per TRACK_MAX_FRAMES of them, in stream order on s.
cudaError_t launch_track_update(const TrackArgs &a, const int *videos, const float *scales, int n, cudaStream_t s);

}  // namespace rf
