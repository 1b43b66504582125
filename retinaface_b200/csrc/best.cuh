// best.cuh -- f11 best shots (rf_b200.h rf_tracker_create_best): per-frame face quality of every tracked face's crop, a per-track
// store of the best crop on the device, and one emission per identity when its track ends.  Per call of up to TRACK_MAX_FRAMES
// frames, after k_track_update has written its seen / gone tables (track.cuh):
//   k_best_measure  a band of BEST_BAND crop rows of one seen record per work item: fits M, warps the band (and one halo row on each
//                   side) into shared grey and INSIDE tables, stores the band's u8 crop rows into the call's scratch, and adds its
//                   integer Laplacian sums to the record's accumulator; the last band computes coverage, sharpness and q
//   k_best_select   one CTA per video of the call, one thread per track slot: frames in call order, removals before seen tracks;
//                   each emission's record and source (the store, or the scratch crop of an earlier frame of the call), each slot's
//                   new best
//   k_best_emit     emissions: source -> the caller's buffer, with the format conversion
//   k_best_commit   the winning scratch crops -> the store (after the emissions read it: a slot freed and reused in one call is right)
// f22: a live tracker's k_best_select also emits LIVE shots of the matched CONFIRMED tracks (rf_tracker_set_best_live); the follow frames
// of a following best-shot tracker (rf_tracker_set_best_follow) run k_best_select on their removals and k_best_emit only.
#pragma once
#include "align.cuh"
#include "track.cuh"

namespace rf {

constexpr int BEST_THREADS = 256, BEST_BAND = 8;

// The quality of one scratch crop: q and its terms (rf_best_shot's), M and the record.
struct BestMeasure {
    double q;
    double M[6];
    float score, eye, frontal, sharpness, coverage;
    int pad;
    rf_face face;
};

// The stored best of one (video, slot): id 0, nothing stored.
struct BestEntry {
    BestMeasure m;
    int id, frame;
};

// Per video: frames applied since create / reset (the frame numbers of rf_best_shot).
struct BestVideo {
    int frames, pad;
};

// The integer sums of one scratch crop, added by each of its row bands (integer: the order does not matter); the band that brings
// `done` to the band count computes q and zeroes the entry for the next call.
struct BestAccum {
    unsigned long long n, s1, s2, inside;
    unsigned int done, pad;
};

struct BestArgs {
    AlignArgs u8;                 // geometry and template of the stored crops (u8 BGR; crop_bytes of u8)
    AlignArgs out;                // the emitted format; crops: the caller's [n][max_tracks], mats optional [n][max_tracks][6]
    int max_tracks, max_faces;
    double min_quality, sharp_half;
    BestEntry *store;             // [max_videos][max_tracks]
    unsigned char *store_crops;   // [max_videos][max_tracks][u8 crop bytes]
    BestVideo *videos;            // [max_videos]
    int num_sms;
    const int *counts;            // [n] the frames' kept record counts: records j < min(count, max_faces) may be seen
    BestAccum *acc;               // [n][max_faces], zero between calls
    const TrackSeen *seen;        // [n][max_faces]
    const TrackGone *gone;        // [n][max_tracks]
    BestMeasure *meas;            // [n][max_faces]
    unsigned char *scratch;       // [n][max_faces][u8 crop bytes]
    int *commit;                  // [n][max_faces] store index (video * max_tracks + slot) the scratch crop goes to, -1
    int *src;                     // [n][max_tracks] emission k's crop: >= 0 a store index, < 0 scratch index -1 - s
    rf_best_shot *best;           // [n][max_tracks]
    int *best_counts;             // [n]
};

// f22: the live state of one (video, slot): the track it belongs to (id 0 or another id: no live shot yet), its live shots so far, the
// frame number and q of the last one.  Kept apart from BestEntry so that the store's layout is f11's.
struct BestLive {
    int id, n, e, pad;
    double q;
};

// f22: the live policy's arguments, read by the live instantiation of k_best_select only.
struct BestLiveArgs {
    BestLive *live;               // [max_videos][max_tracks]
    const TrackLife *life;        // [n][max_faces]
    double first_quality;         // (double)first_quality
    double ratio;                 // 1.0 + (double)improve, one rounding
    int min_gap;
};

// The call's host tables: frame i belongs to video[i]; CTA b of k_best_select runs the frames of cta_video[b].
struct BestTable {
    int n, nvideos;
    int video[TRACK_MAX_FRAMES];
    int cta_video[TRACK_MAX_FRAMES];
    AlignImageT<YuvPlanes> img[TRACK_MAX_FRAMES];
};

// The four kernels of one call of t.n <= TRACK_MAX_FRAMES frames, in order on s.
cudaError_t launch_best_frames(const BestArgs &a, const BestTable &t, cudaStream_t s);
// f22: launch_best_frames with the live policy of `l`.
cudaError_t launch_best_frames_live(const BestArgs &a, const BestTable &t, const BestLiveArgs &l, cudaStream_t s);
// f22: the t.n follow frames of a call (a.gone their removals): select and emit only -- the EXIT shots, and each video's frame count.
cudaError_t launch_best_follow(const BestArgs &a, const BestTable &t, cudaStream_t s);
// rf_tracker_finish: the emissions of every live, ever-confirmed track of `video` (state: its [max_tracks] slots) into a.best[0],
// a.best_counts[0] and the caller's buffers.
cudaError_t launch_best_finish(const BestArgs &a, int video, const TrackState *state, cudaStream_t s);

}  // namespace rf
