// follow.cuh -- f16 following tracked faces between detections (rf_b200.h rf_tracker_set_follow): luma templates cut on detect
// frames, a SAD search at three scales on follow frames, and the tracker step that replaces association on those frames.
#pragma once
#include "track.cuh"

namespace rf {

constexpr int FOLLOW_T = RF_FOLLOW_TEMPLATE;
constexpr int FOLLOW_BYTES = FOLLOW_T * FOLLOW_T;
constexpr int FOLLOW_MAX_R = RF_FOLLOW_MAX_SEARCH;
constexpr int FOLLOW_THREADS = 256;

// The template of one track slot: the id of the track it was cut for (0: none) and its FLAT test.
struct FollowEntry {
    int id, flat;
};

// The search's result for one (frame, slot): the record rf_tracker_follow returns and, when OK, the followed face.
struct FollowMeas {
    rf_follow rec;
    rf_face face;
};

// One frame of a launch: its luma plane, video and index in the call (the row of its lists, follow records and measurements).  f20:
// bits, the video's orientation (LB_* bits; w x h then the displayed size), read by the oriented launches only.
struct FollowFrame {
    const uint8_t *y;
    int pitch, w, h, video, frame, bits;
};

struct FollowTable {
    int n;
    FollowFrame f[TRACK_MAX_FRAMES];
};

struct FollowArgs {
    TrackParams p;
    TrackVideo *videos;          // [max_videos]
    TrackState *state;           // [max_videos][max_tracks]
    uint8_t *store;              // [max_videos][max_tracks][FOLLOW_BYTES]
    FollowEntry *entries;        // [max_videos][max_tracks]
    const rf_track *lists;       // cut: the call's track lists [n][max_tracks] and counts [n]
    const int *list_counts;
    FollowMeas *meas;            // follow: [n][max_tracks] by slot
    rf_follow *follow;           // follow: [n][max_tracks] in list order
    rf_track *tracks;            // follow: [n][max_tracks]
    int *track_counts;           // follow: [n]
    rf_det *regions;             // follow: [n][max_tracks] the OK-followed faces in id order (anchor_index: the id), f12's (a)
    int *region_counts;          // follow: [n]
    const rf_motion *motion;     // follow, optional: [n] each frame's camera motion (f13), applied after predict when RF_MOTION_OK
    rf_det *mask;                // follow with motion: [n][max_tracks] the faces the motion estimate skips, and their counts [n]
    int *mask_counts;
    int search;
    float max_mad;
    TrackGone *gone;             // follow, optional: [n][max_tracks] the tracks removed on each frame, by slot (f22, a following best-shot
                                 // tracker; age after the frame's increment)
};

// The templates of every track matched on the call's detect frames (after launch_track_update), one launch per TRACK_MAX_FRAMES.
// oriented (f20): some frame's bits are not 0, and the luma is read as displayed (a separate instantiation).
cudaError_t launch_follow_cut(const FollowArgs &a, const FollowFrame *frames, int n, cudaStream_t s, bool oriented = false);
// One round of a follow call: frames of distinct videos, searched, then stepped.
cudaError_t launch_follow_round(const FollowArgs &a, const FollowTable &t, cudaStream_t s, bool oriented = false);
// The motion estimate's face mask of a round's frames: every TENTATIVE or CONFIRMED track's face, before the frame.
cudaError_t launch_follow_mask(const FollowArgs &a, const FollowTable &t, cudaStream_t s);
// f20 (oriented_search.cu): k_follow_cut and k_follow_search on frames read as displayed, one table each.
cudaError_t launch_follow_cut_oriented(const FollowArgs &a, const FollowTable &t, cudaStream_t s);
cudaError_t launch_follow_search_oriented(const FollowArgs &a, const FollowTable &t, cudaStream_t s);

}  // namespace rf
