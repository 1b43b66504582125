// tracker.cu -- the video tracker behind include/rf_b200.h: f10 tracking, f11 best shots, f13 camera motion, f16 following, f12 / f14
// redaction, f15 look-back, f17 searching look-back, f18 following look-back, f19 tiling, f20 oriented videos, f22 live and following
// best shots and f25 rotated views.  Detection itself is
// engine.cu's (yuv_device_impl).
// The entry points take their C linkage from rf_b200.h.
#include <array>
#include <cmath>

#include "engine_internal.cuh"
#include "best.cuh"
#include "redact.cuh"
#include "track.cuh"
#include "motion.cuh"
#include "lookback.cuh"
#include "follow.cuh"

// ---- f10 face tracking across video frames (track.cuh) ---------------------------------------------------------------------------
// The tracker owns every video's state and a ring of output slots.  Its kernels are ordered by an event chain: each update (and
// each reset) waits for `chain` on the stream it is issued on, which may belong to any context, and records it again, so the state
// of a video is only ever touched by one launch at a time while the forwards of the contexts still overlap.  A slot's `free` is
// recorded at the end of the call that took it (slot_begin), once its crops or redaction are issued; the next call on that slot
// waits for it.
//
// A tracker is of one kind: plain, best-shot (f11), follow (f16) or look-back (f15).  Camera motion (f13) is an option of any kind,
// the look-back search (f17) and following (f18) options of a look-back tracker, live shots and following (f22) options of a best-shot
// tracker.  admit() decides from them which calls it takes.
enum Kind { PLAIN, BEST, FOLLOW, LOOKBACK };

struct rf_tracker_s {
    rf_handle h = nullptr;
    rf_track_config cfg{};             // defaults applied
    TrackVideo *d_videos = nullptr;    // [max_videos]
    TrackState *d_state = nullptr;     // [max_videos][max_tracks]
    TrackPair *d_pairs = nullptr;      // [ctas][max_tracks * max_faces]
    int *d_order = nullptr;
    struct Slot {
        rf_track *tracks = nullptr;    // [max_batch][max_tracks]
        int *counts = nullptr;         // [max_batch]
        rf_det *due = nullptr;         // [max_batch][max_faces]
        int *due_counts = nullptr;     // [max_batch]
        rf_motion *motion = nullptr;   // [max_batch] f13, with motion on
        rf_det *lb_boxes = nullptr;    // [max(max_batch, L)][lookback_records] f15, the regions of the emitted frames
        int *lb_counts = nullptr;      // [max(max_batch, L)]
        rf_follow *lb_steps = nullptr; // [max_batch][min(max_faces, max_tracks)][L] f17, the step records of a look-back call
        int *lb_lengths = nullptr;     // [max_batch][min(max_faces, max_tracks)]
        rf_best_shot *best = nullptr;  // [max_batch][max_tracks] f11, the emitted shots
        int *best_counts = nullptr;    // [max_batch]
        rf_follow *follow = nullptr;   // [max_batch][max_tracks] f16, the follow records
        rf_det *fregions = nullptr;    // [max_batch][max_tracks] the OK-followed faces (redaction's records)
        int *fregion_counts = nullptr; // [max_batch]
        cudaEvent_t free = nullptr;
    };
    std::vector<Slot> slots;
    unsigned next_slot = 0;
    cudaEvent_t chain = nullptr;
    Kind kind = PLAIN;
    // f11 best shots (best.cuh); allocated on a BEST tracker.  The chain orders every best-shot kernel of every call, so one set of
    // per-call tables serves them all; only the emitted records live in the ring.
    BestArgs ba{};                     // store, per-video counters, per-call tables, formats (per-call pointers set per call)
    bool updated = false;              // a frame call was issued (rf_tracker_set_motion comes before)
    // f22 options of a BEST tracker: live shots (bl: the live state and the per-call track table, allocated with the option) and
    // following (f16's store below, and the follow frames' removals d_fgone [max_batch][max_tracks]).
    bool best_live = false, best_follow = false;
    BestLiveArgs bl{};
    TrackGone *d_fgone = nullptr;
    // f13 camera motion (motion.cuh); `motion` false: none of these allocated.  mref mirrors on the host what each video's
    // reference slot holds (the frame size it came from, 0 x 0: none): calls, resets and finishes are issued in host order, so the
    // reference of every frame is known when the call is issued.  The chain orders the per-call scratch as it orders f11's tables.
    bool motion = false;
    rf_motion_config mcfg{};
    uint8_t *d_mstore = nullptr;       // [max_videos][MOTION_THUMB_BYTES]
    uint8_t *d_mthumbs = nullptr;      // [max_batch][MOTION_THUMB_BYTES]
    MotionBlock *d_mblocks = nullptr;  // [max_batch][MOTION_MAX_BLOCKS]
    std::vector<std::array<int, 2>> mref;
    int motion_slot = -1;              // the ring slot of the latest frame call
    // f15 look-back (lookback.cuh); allocated on a LOOKBACK tracker.  lbv mirrors on the host each video's frame count and layout, so
    // that every frame's number, buffer slot and emission are known when a call is issued.  A video's device block is its frame buffer
    // (L packed frames of frame_bytes) followed by its log (2 L slots of lookback_slot_bytes).
    int lb_frames = 0;                 // L
    float lb_grow = 0.f;
    struct LookbackVideo {
        uint8_t *d = nullptr;
        size_t frame_bytes = 0;
        int w = 0, h = 0, step = 0;
        bool v_first = false;          // semi-planar with V before U (NV21)
        long long frames = 0;          // frames since create, reset or drain
    };
    std::vector<LookbackVideo> lbv;
    // f17 searching look-back: the step records live in the ring, the chains in the log slots.
    bool lb_search = false;
    rf_follow_config lscfg{};
    int lb_search_slot = -1;           // the ring slot of the latest look-back call
    // f18 following look-back: a LOOKBACK tracker that also takes follow frames, with f16's store and follow records below.
    bool lb_follow = false;
    // f16 following (follow.cuh); allocated on a FOLLOW tracker and on a following look-back tracker.  The chain orders the per-call
    // measurements as it orders f11's tables; the follow records live in the ring.
    rf_follow_config fcfg{};
    uint8_t *d_fstore = nullptr;         // [max_videos][max_tracks][FOLLOW_BYTES]
    FollowEntry *d_fentries = nullptr;   // [max_videos][max_tracks]
    FollowMeas *d_fmeas = nullptr;       // [max_batch][max_tracks]
    rf_det *d_fmask = nullptr;           // [max_batch][max_tracks] with motion: each follow frame's face mask
    int *d_fmask_counts = nullptr;       // [max_batch]
    int follow_slot = -1;                // the ring slot of the latest follow call
    // f19 tiling: every detect call detects through rf_detect_yuv_tiled_device's tiles of `tiling` (its levels in tile_levels).
    bool tiled = false;
    rf_tiling tiling{};
    std::vector<rf_tile_level> tile_levels;
    // f20 display orientations: each video's EXIF orientation (1: upright), kept across restarts, and whether the video has taken a
    // frame call since its last restart (create, reset, drain, finish), which fixes its orientation until the next one.
    std::vector<int> orient;
    std::vector<char> started;
    // f25 rotated views: every detect call detects through rf_detect_yuv_views_rotated_device's views (copied).  Empty: off.
    std::vector<rf_rotated_view> views;
};

// Whether some video of t is shown in an orientation other than 1.
static bool any_oriented(rf_tracker t) {
    return std::any_of(t->orient.begin(), t->orient.end(), [](int o) { return o != 1; });
}

// f20: video v's orientation as LB_* bits, and the displayed size of its stored w x h frames.
static int video_bits(rf_tracker t, int v) { return lb_orientation_bits(t->orient[v]); }
static std::array<int, 2> shown_size(rf_tracker t, int v, int w, int h) {
    return video_bits(t, v) & LB_TRANSPOSE ? std::array<int, 2>{h, w} : std::array<int, 2>{w, h};
}

template <typename... P>
static void free_null(P *&...p) {
    (cudaFree(p), ...);
    ((p = nullptr), ...);
}

// Each option's buffers, freed and nulled: by tracker_release, and by a setter whose allocation failed, so that the tracker is again
// exactly one that never saw the call.
static void free_motion(rf_tracker t) {
    free_null(t->d_mstore, t->d_mthumbs, t->d_mblocks);
    for (auto &s : t->slots) free_null(s.motion);
}

static void free_follow(rf_tracker t) {
    free_null(t->d_fstore, t->d_fentries, t->d_fmeas, t->d_fmask, t->d_fmask_counts, t->d_fgone);
    for (auto &s : t->slots) free_null(s.follow, s.fregions, s.fregion_counts);
}

static void free_lookback(rf_tracker t) {
    for (auto &s : t->slots) free_null(s.lb_boxes, s.lb_counts, s.lb_steps, s.lb_lengths);
    for (auto &v : t->lbv) free_null(v.d);
}

static void tracker_release(rf_tracker t) {
    if (t->chain) cudaEventSynchronize(t->chain);
    for (auto &s : t->slots) {
        if (s.free) { cudaEventSynchronize(s.free); cudaEventDestroy(s.free); }
        cudaFree(s.tracks); cudaFree(s.counts); cudaFree(s.due); cudaFree(s.due_counts); cudaFree(s.best); cudaFree(s.best_counts);
    }
    free_motion(t);
    free_follow(t);
    free_lookback(t);
    if (t->chain) cudaEventDestroy(t->chain);
    cudaFree(t->d_videos); cudaFree(t->d_state); cudaFree(t->d_pairs); cudaFree(t->d_order);
    const BestArgs &b = t->ba;
    cudaFree(b.store); cudaFree(b.store_crops); cudaFree(b.videos); cudaFree(b.acc); cudaFree((void *)b.seen); cudaFree((void *)b.gone); cudaFree(b.meas);
    cudaFree(b.scratch); cudaFree(b.commit); cudaFree(b.src);
    cudaFree(t->bl.live); cudaFree((void *)t->bl.life);
    delete t;
}

int rf_tracker_create(rf_handle h, const rf_track_config *cfg, rf_tracker *out) {
    static const char *who = "rf_tracker_create";
    if (!h) return RF_ERR_INVALID_ARG;
    if (!cfg || !out) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config or output", who));
    *out = nullptr;
    rf_track_config c = *cfg;
    if (c.max_videos < 1 || c.max_videos > 4096) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: max_videos %d, must be in [1, 4096]", who, c.max_videos));
    if (c.max_tracks == 0) c.max_tracks = 64;
    if (c.max_tracks < 1 || c.max_tracks > TRACK_MAX_TRACKS)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: max_tracks %d, must be in [1, %d]", who, c.max_tracks, TRACK_MAX_TRACKS));
    if (c.max_lost == 0) c.max_lost = 30;
    if (c.max_lost < 0) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: max_lost %d is negative", who, c.max_lost));
    float *th[5] = {&c.high_thresh, &c.new_thresh, &c.iou_high, &c.iou_low, &c.iou_tentative};
    const float dflt[5] = {0.6f, 0.7f, 0.2f, 0.5f, 0.3f};
    for (int k = 0; k < 5; k++) {
        if (*th[k] == 0.f) *th[k] = dflt[k];
        if (!(*th[k] > 0.f && *th[k] <= 1.f))
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: thresholds must be in (0, 1] (0: the default), got %g", who, (double)*th[k]));
    }
    std::unique_ptr<rf_tracker_s, void (*)(rf_tracker)> t(new rf_tracker_s, tracker_release);
    t->h = h;
    t->cfg = c;
    t->orient.assign(c.max_videos, 1);
    t->started.assign(c.max_videos, 0);
    try {
        CK(cudaSetDevice(h->device));
        const size_t T = c.max_tracks, F = h->cfg.max_faces, B = h->cfg.max_batch;
        const size_t ctas = std::min<size_t>({B, (size_t)TRACK_MAX_FRAMES, (size_t)c.max_videos});
        CK(cudaMalloc(&t->d_videos, sizeof(TrackVideo) * c.max_videos));
        CK(cudaMalloc(&t->d_state, sizeof(TrackState) * c.max_videos * T));
        CK(cudaMalloc(&t->d_pairs, sizeof(TrackPair) * ctas * T * F));
        CK(cudaMalloc(&t->d_order, sizeof(int) * ctas * T * F));
        CK(cudaMemset(t->d_videos, 0, sizeof(TrackVideo) * c.max_videos));
        CK(cudaMemset(t->d_state, 0, sizeof(TrackState) * c.max_videos * T));
        t->slots.resize(h->ctx.size());
        for (auto &s : t->slots) {
            CK(cudaMalloc(&s.tracks, sizeof(rf_track) * B * T));
            CK(cudaMalloc(&s.counts, sizeof(int) * B));
            CK(cudaMalloc(&s.due, sizeof(rf_det) * B * F));
            CK(cudaMalloc(&s.due_counts, sizeof(int) * B));
            CK(cudaEventCreateWithFlags(&s.free, cudaEventDisableTiming));
        }
        CK(cudaEventCreateWithFlags(&t->chain, cudaEventDisableTiming));
        CK(cudaDeviceSynchronize());      // the zeroed state is in place before any context's stream reads it
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    *out = t.release();
    return RF_OK;
}

void rf_tracker_destroy(rf_tracker t) {
    if (!t) return;
    cudaSetDevice(t->h->device);
    tracker_release(t);
}

// Restarts videos [v0, v0 + nv) on s, inside the chain: no tracks, and by the kind no stored shots and no live state (BEST, nothing is
// emitted), no templates (FOLLOW, a following LOOKBACK and a following BEST) and no buffered frames (LOOKBACK, nothing is emitted); with
// motion, no reference.
static void restart(rf_tracker t, size_t v0, size_t nv, cudaStream_t s) {
    const size_t T = t->cfg.max_tracks;
    CK(cudaMemsetAsync(t->d_videos + v0, 0, sizeof(TrackVideo) * nv, s));
    CK(cudaMemsetAsync(t->d_state + v0 * T, 0, sizeof(TrackState) * nv * T, s));
    if (t->kind == BEST) {
        CK(cudaMemsetAsync(t->ba.store + v0 * T, 0, sizeof(BestEntry) * nv * T, s));
        CK(cudaMemsetAsync(t->ba.videos + v0, 0, sizeof(BestVideo) * nv, s));
        if (t->best_live) CK(cudaMemsetAsync(t->bl.live + v0 * T, 0, sizeof(BestLive) * nv * T, s));
    }
    if (t->kind == FOLLOW || t->lb_follow || t->best_follow) CK(cudaMemsetAsync(t->d_fentries + v0 * T, 0, sizeof(FollowEntry) * nv * T, s));
    for (size_t v = v0; t->motion && v < v0 + nv; v++) t->mref[v] = {0, 0};
    for (size_t v = v0; t->kind == LOOKBACK && v < v0 + nv; v++) t->lbv[v].frames = 0;
    std::fill(t->started.begin() + v0, t->started.begin() + v0 + nv, 0);
}

int rf_tracker_reset(rf_tracker t, int video) {
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (video < -1 || video >= t->cfg.max_videos)
        return fail(h, RF_ERR_INVALID_ARG, fmt("rf_tracker_reset: video %d, must be -1 or in [0, %d)", video, t->cfg.max_videos));
    try {
        CK(cudaSetDevice(h->device));
        cudaStream_t s = h->ctx[0].stream;
        CK(cudaStreamWaitEvent(s, t->chain, 0));
        restart(t, video < 0 ? 0 : video, video < 0 ? t->cfg.max_videos : 1, s);
        CK(cudaEventRecord(t->chain, s));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// The calls admit() decides.  DETECT: rf_detect_yuv_track_device and rf_detect_yuv_redact_device(_style) with a tracker; FOLLOW:
// rf_track_follow_device and rf_track_follow_redact_device; LOOKBACK_FOLLOW: rf_track_follow_redact_lookback_device; BEST_FOLLOW:
// rf_track_follow_best_device; MOTION, FOLLOWS and LOOKBACK_SEARCH: the queries rf_tracker_motion, rf_tracker_follow and
// rf_tracker_lookback_search.
enum class Call {
    UPDATE, DETECT, BEST, FINISH, FOLLOW, LOOKBACK, DRAIN, LOOKBACK_FOLLOW, BEST_FOLLOW,
    SET_MOTION, SET_FOLLOW, SET_LOOKBACK, SET_LOOKBACK_SEARCH, SET_LOOKBACK_FOLLOW, SET_BEST_LIVE, SET_BEST_FOLLOW,
    SET_TILING, SET_VIEWS,                                                                             // the setters, SET_MOTION .. here
    MOTION, FOLLOWS, LOOKBACK_SEARCH
};

// Whether t takes `call`, from its kind, its options and whether a frame call was issued; checked before anything is launched.
static int admit(rf_tracker t, const char *who, Call call) {
    static const char *const name[] = {"plain", "best-shot", "follow", "look-back"};
    static const char *const made_by[] = {"rf_tracker_create", "rf_tracker_create_best", "rf_tracker_set_follow", "rf_tracker_set_lookback"};
    const Kind k = t->kind;
    std::string why;
    auto only = [&](Kind need) {
        if (k != need) why = fmt("not a %s tracker (%s)", name[need], made_by[need]);
    };
    auto only_through = [&]() {
        if (t->best_follow)
            return std::string("a best-shot tracker takes frames only through rf_detect_yuv_track_best_device and rf_track_follow_best_device");
        if (t->lb_follow)
            return std::string("a following look-back tracker takes frames only through rf_detect_yuv_redact_lookback_device and "
                               "rf_track_follow_redact_lookback_device");
        return fmt("a %s tracker takes frames only through %s", name[k],
                   k == BEST ? "rf_detect_yuv_track_best_device" : "rf_detect_yuv_redact_lookback_device");
    };
    switch (call) {
    case Call::UPDATE:
        if (k == BEST || t->lb_follow) why = only_through();
        else if (t->motion || k == FOLLOW) why = fmt("a %s tracker needs the frames (rf_detect_yuv_track_device)", t->motion ? "motion" : "follow");
        else if (k == LOOKBACK) why = only_through();
        break;
    case Call::DETECT: if (k == BEST || k == LOOKBACK) why = only_through(); break;
    case Call::BEST: case Call::FINISH: only(BEST); break;
    case Call::FOLLOW: if (t->lb_follow || t->best_follow) why = only_through(); else only(FOLLOW); break;
    case Call::FOLLOWS: if (!t->lb_follow && !t->best_follow) only(FOLLOW); break;
    case Call::LOOKBACK: case Call::DRAIN: only(LOOKBACK); break;
    case Call::LOOKBACK_FOLLOW: if (!t->lb_follow) why = "not a following look-back tracker (rf_tracker_set_lookback_follow)"; break;
    case Call::BEST_FOLLOW: if (!t->best_follow) why = "not a following best-shot tracker (rf_tracker_set_best_follow)"; break;
    case Call::SET_MOTION: if (t->motion) why = "motion is already on"; break;
    case Call::SET_FOLLOW: if (k != PLAIN) why = k == FOLLOW ? "following is already on" : fmt("a %s tracker cannot follow", name[k]); break;
    case Call::SET_LOOKBACK: if (k != PLAIN) why = k == LOOKBACK ? "look-back is already on" : fmt("a %s tracker cannot look back", name[k]); break;
    case Call::SET_LOOKBACK_SEARCH:
        only(LOOKBACK);
        if (why.empty() && t->lb_search) why = "the look-back search is already on";
        break;
    case Call::SET_LOOKBACK_FOLLOW:
        only(LOOKBACK);
        if (why.empty() && t->lb_follow) why = "look-back following is already on";
        break;
    case Call::SET_BEST_LIVE:
        only(BEST);
        if (why.empty() && t->best_live) why = "live shots are already on";
        break;
    case Call::SET_BEST_FOLLOW:
        only(BEST);
        if (why.empty() && t->best_follow) why = "best-shot following is already on";
        break;
    case Call::SET_TILING: if (t->tiled) why = "tiling is already on"; break;
    case Call::SET_VIEWS: if (!t->views.empty()) why = "rotated views are already on"; break;
    case Call::MOTION: if (!t->motion) why = "motion is off (rf_tracker_set_motion)"; break;
    case Call::LOOKBACK_SEARCH: if (!t->lb_search) why = "not a searching look-back tracker (rf_tracker_set_lookback_search)"; break;
    }
    if (why.empty() && call >= Call::SET_MOTION && call <= Call::SET_VIEWS && t->updated) why = "the tracker has already been updated";
    return why.empty() ? RF_OK : fail(t->h, RF_ERR_INVALID_ARG, fmt("%s: %s", who, why.c_str()));
}

// Everything a frame call refuses in its tracker, videos and scales, checked before anything is launched.
static int check_track_args(rf_tracker t, const char *who, Call call, const int *videos, int n, const float *scales) {
    rf_handle h = t->h;
    int rc = admit(t, who, call);
    if (rc || (rc = check_n(h, n))) return rc;
    if (n > 0 && !videos) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: videos is NULL", who));
    for (int i = 0; i < n; i++) {
        if (videos[i] < 0 || videos[i] >= t->cfg.max_videos)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: video %d, must be in [0, %d)", who, i, videos[i], t->cfg.max_videos));
        if (scales && !(std::isfinite(scales[i]) && scales[i] > 0.f))
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: scale %g, must be finite and positive", who, i, (double)scales[i]));
    }
    return RF_OK;
}

// Takes the next ring slot for a call issued on s: s waits for the slot's `free` and for the chain.  The call records the chain once
// its state is written and the slot's `free` at its end.
static unsigned slot_begin(rf_tracker t, cudaStream_t s) {
    const unsigned ring = t->next_slot++ % t->slots.size();
    CK(cudaStreamWaitEvent(s, t->slots[ring].free, 0));
    CK(cudaStreamWaitEvent(s, t->chain, 0));
    return ring;
}

static TrackParams track_params(rf_tracker t) {
    const rf_track_config &c = t->cfg;
    return TrackParams{c.max_tracks, t->h->cfg.max_faces, c.max_lost, c.high_thresh, c.new_thresh, c.iou_high, c.iou_low, c.iou_tentative};
}

// A redaction call's resolved style: f12's params are {MOSAIC, RECT, blocks, detail 0}.
struct RedactSpec {
    int kind = REDACT_MOSAIC, shape = REDACT_RECT, blocks = 8, detail = 0;
    double margin = 0.25;
};

// One tracker frame call: where its frames' records come from, what follows the update and where its outputs go.  Every exported
// frame call fills one and runs it through frame_call, which checks it (check_call) and issues it (issue_call).  `who` names the call
// in every message.
struct FrameCall {
    enum Source { RECORDS, DETECT, FOLLOW };           // the caller's records (rf_track_update), a forward, or the follow rounds
    enum Sink { NONE, CROPS, BEST, REDACT, LOOKBACK }; // after the update: nothing, the due faces' crops, best shots, redaction, look-back
    const char *who;
    Call call;
    Source source;
    Sink sink = NONE;
    rf_handle h = nullptr;             // DETECT: the caller's handle, which the tracker must belong to
    rf_tracker t;
    const rf_yuv_frame *frames = nullptr;
    const int *videos;
    int n;
    // the records the tracks move with, and the sink draws: RECORDS the caller's, DETECT the forward's, FOLLOW the OK-followed faces
    const rf_det *dets = nullptr;
    const int32_t *counts = nullptr;
    const float *scales = nullptr;     // their map-back factors (NULL: 1)
    int matrix = 0;                    // DETECT
    float thr = 0.f, nms = 0.f;
    const rf_align_params *align = nullptr;            // CROPS
    void *crops = nullptr;                             // CROPS, BEST
    double *mats = nullptr;
    const rf_redact_style *style = nullptr;            // REDACT, LOOKBACK
    const rf_yuv_frame *out_frames = nullptr;          // LOOKBACK
    int32_t *out_frame_numbers = nullptr;
    const rf_track **tracks = nullptr;                 // the outputs, each may be NULL
    const int32_t **track_counts = nullptr;
    const rf_det **out_dets = nullptr;
    const int32_t **out_counts = nullptr;
    float *out_scales = nullptr;
    const rf_best_shot **best = nullptr;
    const int32_t **best_counts = nullptr;
    // set by check_call
    AlignArgs a{};
    RedactSpec spec;
    std::vector<long long> num;                        // LOOKBACK: lb_numbers' frame numbers and videos
    std::vector<std::array<int, 3>> seen;
    std::vector<std::vector<rf_tile>> layouts;         // DETECT on a tiling tracker: each frame's tiles
    std::vector<int> orients;                          // f20: each frame's video's orientation, when `oriented`
    bool oriented = false;                             // some frame of the call is not at orientation 1
    // set by issue_call: a tiled or rotated detect's ring slot event, recorded again once the call has read the records
    cudaEvent_t detector_free = nullptr;
};

static int frame_call(FrameCall &c);


// The YUV source of a detect call: each frame in its video's orientation when some frame is oriented, else the upright source.
static YuvFrames detect_source(const FrameCall &c) { return YuvFrames{c.frames, c.matrix, c.oriented ? c.orients.data() : nullptr, c.oriented}; }

// ---- f13 camera motion (motion.cuh) ---------------------------------------------------------------------------------------------
// Each video's last frame of a call, whose thumbnail becomes the video's reference once the update has run.
struct MotionCommits {
    std::vector<int> frames, videos, bytes;
};

// The call's n frames in call order, `per` to a table, each with its reference: the previous frame of its video in the call, else the
// video's stored thumbnail, else none (FIRST); a frame size change is none.  Each video's last frame of the call goes into `commits`
// (videos in first-appearance order), and mref takes its size.
static std::vector<MotionTable> motion_tables(rf_tracker t, const rf_yuv_frame *frames, const int *videos, const float *scales, int n, int per,
                                              MotionCommits &commits) {
    const int R = t->mcfg.search;
    std::vector<MotionTable> tabs((n + per - 1) / per);
    std::vector<std::array<int, 2>> last;          // (video, its latest frame of the call)
    for (int i = 0; i < n; i++) {
        MotionTable &tb = tabs[i / per];
        tb.i0 = i - i % per;
        MotionFrame &f = tb.f[tb.n++];
        const rf_yuv_frame &fr = frames[i];
        const int v = videos[i];
        const std::array<int, 2> size = shown_size(t, v, fr.width, fr.height);      // f20: the displayed frame's thumbnail
        const PlaneMap m = plane_map(video_bits(t, v), size[0], size[1], fr.y_pitch, 1);
        f.y = fr.y + m.off;
        f.pitch = m.ys;
        f.xs = m.xs;
        f.video = v;
        f.scale = scales ? scales[i] : 1.f;
        f.D = (std::max(size[0], size[1]) + MOTION_THUMB - 1) / MOTION_THUMB;
        f.tw = size[0] / f.D;
        f.th = size[1] / f.D;
        f.nbx = f.tw - 2 * R >= MOTION_BLOCK ? (f.tw - 2 * R) / MOTION_BLOCK : 0;
        f.nby = f.th - 2 * R >= MOTION_BLOCK ? (f.th - 2 * R) / MOTION_BLOCK : 0;
        auto it = std::find_if(last.begin(), last.end(), [v](const std::array<int, 2> &e) { return e[0] == v; });
        if (it != last.end()) {
            const rf_yuv_frame &p = frames[(*it)[1]];
            f.ref = p.width == fr.width && p.height == fr.height ? (*it)[1] : MOTION_REF_FIRST;
            (*it)[1] = i;
        } else {
            f.ref = t->mref[v] == size ? MOTION_REF_STORE : MOTION_REF_FIRST;
            last.push_back({v, i});
        }
    }
    for (const auto &e : last) {
        t->mref[e[0]] = shown_size(t, e[0], frames[e[1]].width, frames[e[1]].height);
        commits.frames.push_back(e[1]);
        commits.videos.push_back(e[0]);
        const MotionFrame &f = tabs[e[1] / per].f[e[1] % per];
        commits.bytes.push_back(f.tw * f.th);
    }
    return tabs;
}

// The estimator's arguments into ring slot `ring`'s motions, masking the faces of `dets` (max_faces records per frame).
static MotionArgs motion_args(rf_tracker t, unsigned ring, const rf_det *dets, const int32_t *counts, int max_faces) {
    MotionArgs a{};
    a.thumbs = t->d_mthumbs;
    a.store = t->d_mstore;
    a.blocks = t->d_mblocks;
    a.out = t->slots[ring].motion;
    a.dets = dets;
    a.counts = counts;
    a.max_faces = max_faces;
    a.search = t->mcfg.search;
    a.min_inliers = t->mcfg.min_inliers;
    return a;
}

static void motion_commit(rf_tracker t, const MotionCommits &c, cudaStream_t s) {
    MotionArgs a{};
    a.thumbs = t->d_mthumbs;
    a.store = t->d_mstore;
    CK(launch_motion_commit(a, c.frames.data(), c.videos.data(), c.bytes.data(), (int)c.frames.size(), s));
}

// ---- f16 following (follow.cuh) -------------------------------------------------------------------------------------------------
static FollowArgs follow_args(rf_tracker t) {
    FollowArgs f{};
    f.p = track_params(t);
    f.videos = t->d_videos;
    f.state = t->d_state;
    f.store = t->d_fstore;
    f.entries = t->d_fentries;
    f.meas = t->d_fmeas;
    f.search = t->fcfg.search;
    f.max_mad = t->fcfg.max_mad;
    return f;
}

// f20: w x h the displayed size, and the video's orientation bits for the oriented launches.
static FollowFrame follow_frame(rf_tracker t, const rf_yuv_frame &fr, int video, int i) {
    const std::array<int, 2> size = shown_size(t, video, fr.width, fr.height);
    return FollowFrame{fr.y, fr.y_pitch, size[0], size[1], video, i, video_bits(t, video)};
}

// The templates of the tracks matched on a detect call's frames, from the call's lists in `slot`, on s inside the chain.
static void follow_cut(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_tracker_s::Slot &slot, cudaStream_t s) {
    FollowArgs f = follow_args(t);
    f.lists = slot.tracks;
    f.list_counts = slot.counts;
    std::vector<FollowFrame> tab(n);
    bool oriented = false;
    for (int i = 0; i < n; i++) {
        tab[i] = follow_frame(t, frames[i], videos[i], i);
        oriented |= tab[i].bits != 0;
    }
    CK(launch_follow_cut(f, tab.data(), n, s, oriented));
}

// The best-shot table of m frames of videos[]: each frame's video, and the videos in first-appearance order (one select CTA each).
static BestTable best_table(const int *videos, int m) {
    BestTable bt{};
    bt.n = m;
    for (int i = 0; i < m; i++) {
        const int v = videos[i];
        bt.video[i] = v;
        bool known = false;
        for (int j = 0; j < bt.nvideos; j++) known |= bt.cta_video[j] == v;
        if (!known) bt.cta_video[bt.nvideos++] = v;
    }
    return bt;
}

// The best-shot arguments of the chunk of call c from frame i0: the caller's crops and matrices, the slot's shot records.
static BestArgs best_args(rf_tracker t, const rf_tracker_s::Slot &slot, const FrameCall &c, int i0) {
    const int T = t->cfg.max_tracks;
    BestArgs b = t->ba;
    b.out.crops = static_cast<uint8_t *>(c.crops) + (size_t)i0 * T * b.out.crop_bytes;
    b.out.mats = c.mats ? c.mats + (size_t)i0 * T * 6 : nullptr;
    b.best = slot.best + (size_t)i0 * T;
    b.best_counts = slot.best_counts + i0;
    return b;
}

// The update of a records or detect call into ring slot `ring`'s lists, on s inside the chain: with motion, the estimate of its frames
// first (in tables of TRACK_MAX_FRAMES frames) and the commit after.  A best-shot call goes in chunks of TRACK_MAX_FRAMES frames, each
// tracked, then measured, selected, emitted and committed (the per-call tables hold one chunk); launch_track_update makes the same
// launches on a whole call.  With crops, the due faces go to the slot.
static void update_issue(rf_tracker t, unsigned ring, const FrameCall &c, cudaStream_t s) {
    rf_tracker_s::Slot &slot = t->slots[ring];
    const int T = t->cfg.max_tracks, F = t->h->cfg.max_faces;
    MotionCommits commits;
    if (t->motion) {
        const std::vector<MotionTable> tabs = motion_tables(t, c.frames, c.videos, c.scales, c.n, TRACK_MAX_FRAMES, commits);
        CK(launch_motion_estimate(motion_args(t, ring, c.dets, c.counts, F), tabs.data(), (int)tabs.size(), s));
        t->motion_slot = (int)ring;
    }
    TrackArgs ta{};
    ta.p = track_params(t);
    ta.videos = t->d_videos;
    ta.state = t->d_state;
    ta.pairs = t->d_pairs;
    ta.order = t->d_order;
    ta.tracks = slot.tracks;
    ta.track_counts = slot.counts;
    ta.motion = t->motion ? slot.motion : nullptr;
    if (c.sink == FrameCall::CROPS) {
        ta.due = slot.due;
        ta.due_counts = slot.due_counts;
        ta.max_align = c.a.max_align;
    }
    if (c.sink == FrameCall::BEST) {
        ta.seen = const_cast<TrackSeen *>(t->ba.seen);
        ta.gone = const_cast<TrackGone *>(t->ba.gone);
        if (t->best_live) ta.life = const_cast<TrackLife *>(t->bl.life);
    }
    const YuvFrames src = detect_source(c);
    const int chunk = c.sink == FrameCall::BEST ? TRACK_MAX_FRAMES : c.n;
    for (int i0 = 0; i0 < c.n; i0 += chunk) {
        const int m = std::min(chunk, c.n - i0);
        TrackArgs k = ta;
        k.dets = c.dets + (size_t)i0 * F;
        k.counts = c.counts + i0;
        k.tracks += (size_t)i0 * T;
        k.track_counts += i0;
        if (k.motion) k.motion += i0;
        CK(launch_track_update(k, c.videos + i0, c.scales ? c.scales + i0 : nullptr, m, s));
        if (c.sink != FrameCall::BEST) continue;
        BestTable bt = best_table(c.videos + i0, m);
        for (int i = 0; i < m; i++) {
            const int v = c.videos[i0 + i];
            const std::array<int, 2> size = shown_size(t, v, src.width(i0 + i), src.height(i0 + i));    // f20: as displayed
            bt.img[i] = AlignImageT<YuvPlanes>{src.in_place(i0 + i), size[0], size[1], 1.f, video_bits(t, v)};
        }
        BestArgs b = best_args(t, slot, c, i0);
        b.counts = c.counts + i0;
        CK(t->best_live ? launch_best_frames_live(b, bt, t->bl, s) : launch_best_frames(b, bt, s));
    }
    if (t->motion) motion_commit(t, commits, s);
}

int rf_track_update(rf_tracker t, const int *videos, int n, const rf_det *dev_dets, const int32_t *dev_counts, const float *scales,
                    const rf_track **dev_tracks, const int32_t **dev_track_counts) {
    FrameCall c{.who = "rf_track_update", .call = Call::UPDATE, .source = FrameCall::RECORDS, .t = t, .videos = videos, .n = n,
                .dets = dev_dets, .counts = dev_counts, .scales = scales, .tracks = dev_tracks, .track_counts = dev_track_counts};
    return frame_call(c);
}

int rf_detect_yuv_track_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix, float thr, float nms,
                               const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_track **dev_tracks,
                               const int32_t **dev_track_counts, const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    FrameCall c{.who = "rf_detect_yuv_track_device", .call = Call::DETECT, .source = FrameCall::DETECT,
                .sink = align ? FrameCall::CROPS : FrameCall::NONE, .h = h, .t = t, .frames = frames, .videos = videos, .n = n,
                .matrix = matrix, .thr = thr, .nms = nms, .align = align, .crops = dev_crops, .mats = dev_mats, .tracks = dev_tracks,
                .track_counts = dev_track_counts, .out_dets = dev_dets, .out_counts = dev_counts, .out_scales = out_scales};
    return frame_call(c);
}

// ---- f11 best shots (best.cuh) ---------------------------------------------------------------------------------------------------
int rf_tracker_create_best(rf_handle h, const rf_track_config *cfg, const rf_best_config *best, rf_tracker *out) {
    static const char *who = "rf_tracker_create_best";
    if (!h) return RF_ERR_INVALID_ARG;
    if (!cfg || !best || !out) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config or output", who));
    *out = nullptr;
    AlignArgs o;
    int rc = align_setup(h, who, &best->align, o);
    if (rc) return rc;
    if (best->align.max_faces != 0) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: align.max_faces %d, must be 0", who, best->align.max_faces));
    if (!(best->min_quality >= 0.f && best->min_quality <= 1.f))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: min_quality %g, must be in [0, 1]", who, (double)best->min_quality));
    const float half = best->sharp_half == 0.f ? 50.f : best->sharp_half;
    if (!(std::isfinite(half) && half > 0.f)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: sharp_half %g, must be finite and positive", who, (double)half));
    const size_t u8_bytes = align_crop_bytes(o.crop_w, o.crop_h, RF_CROP_BGR_U8);
    const int T = cfg->max_tracks == 0 ? 64 : cfg->max_tracks;
    if (cfg->max_videos >= 1 && cfg->max_videos <= 4096 && T >= 1 && T <= TRACK_MAX_TRACKS && (size_t)cfg->max_videos * T * u8_bytes > ((size_t)4 << 30))
        return fail(h, RF_ERR_CAPACITY, fmt("%s: a store of %d videos x %d tracks x %zu bytes exceeds 4 GiB", who, cfg->max_videos, T, u8_bytes));
    rf_tracker t = nullptr;
    if ((rc = rf_tracker_create(h, cfg, &t))) return rc;
    std::unique_ptr<rf_tracker_s, void (*)(rf_tracker)> g(t, tracker_release);
    t->kind = BEST;
    BestArgs &b = t->ba;
    b.out = o;
    b.u8 = o;
    b.u8.format = RF_CROP_BGR_U8;
    b.u8.crop_bytes = u8_bytes;
    b.max_tracks = t->cfg.max_tracks;
    b.max_faces = h->cfg.max_faces;
    b.min_quality = (double)best->min_quality;
    b.sharp_half = (double)half;
    b.num_sms = h->num_sms;
    try {
        const size_t V = t->cfg.max_videos, TT = t->cfg.max_tracks, F = h->cfg.max_faces, B = h->cfg.max_batch;
        const size_t M = std::min<size_t>(B, TRACK_MAX_FRAMES);
        CK(cudaMalloc(&b.store, sizeof(BestEntry) * V * TT));
        CK(cudaMalloc(&b.store_crops, u8_bytes * V * TT));
        CK(cudaMalloc(&b.videos, sizeof(BestVideo) * V));
        TrackSeen *seen = nullptr;
        TrackGone *gone = nullptr;
        CK(cudaMalloc(&seen, sizeof(TrackSeen) * M * F));
        b.seen = seen;
        CK(cudaMalloc(&gone, sizeof(TrackGone) * M * TT));
        b.gone = gone;
        CK(cudaMalloc(&b.meas, sizeof(BestMeasure) * M * F));
        CK(cudaMalloc(&b.acc, sizeof(BestAccum) * M * F));
        CK(cudaMemset(b.acc, 0, sizeof(BestAccum) * M * F));
        CK(cudaMalloc(&b.scratch, u8_bytes * M * F));
        CK(cudaMalloc(&b.commit, sizeof(int) * M * F));
        CK(cudaMalloc(&b.src, sizeof(int) * M * TT));
        for (auto &s : t->slots) {
            CK(cudaMalloc(&s.best, sizeof(rf_best_shot) * B * TT));
            CK(cudaMalloc(&s.best_counts, sizeof(int) * B));
        }
        CK(cudaMemset(b.store, 0, sizeof(BestEntry) * V * TT));
        CK(cudaMemset(b.videos, 0, sizeof(BestVideo) * V));
        CK(cudaDeviceSynchronize());
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    *out = g.release();
    return RF_OK;
}

int rf_detect_yuv_track_best_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix, float thr,
                                    float nms, void *dev_best_crops, double *dev_best_mats, const rf_best_shot **dev_best,
                                    const int32_t **dev_best_counts, const rf_track **dev_tracks, const int32_t **dev_track_counts,
                                    const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    FrameCall c{.who = "rf_detect_yuv_track_best_device", .call = Call::BEST, .source = FrameCall::DETECT, .sink = FrameCall::BEST, .h = h,
                .t = t, .frames = frames, .videos = videos, .n = n, .matrix = matrix, .thr = thr, .nms = nms, .crops = dev_best_crops,
                .mats = dev_best_mats, .tracks = dev_tracks, .track_counts = dev_track_counts, .out_dets = dev_dets, .out_counts = dev_counts,
                .out_scales = out_scales, .best = dev_best, .best_counts = dev_best_counts};
    return frame_call(c);
}

int rf_tracker_finish(rf_tracker t, int video, void *dev_best_crops, double *dev_best_mats, const rf_best_shot **dev_best,
                      const int32_t **dev_best_count) {
    static const char *who = "rf_tracker_finish";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    int rc = admit(t, who, Call::FINISH);
    if (rc) return rc;
    if (video < 0 || video >= t->cfg.max_videos) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: video %d, must be in [0, %d)", who, video, t->cfg.max_videos));
    if (!dev_best_crops) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: dev_best_crops is NULL", who));
    try {
        CK(cudaSetDevice(h->device));
        cudaStream_t s = h->ctx[0].stream;
        const rf_tracker_s::Slot &slot = t->slots[slot_begin(t, s)];
        BestArgs b = t->ba;
        b.out.crops = dev_best_crops;
        b.out.mats = dev_best_mats;
        b.best = slot.best;
        b.best_counts = slot.best_counts;
        CK(launch_best_finish(b, video, t->d_state + (size_t)video * t->cfg.max_tracks, s));
        restart(t, video, 1, s);     // then the video restarts as rf_tracker_reset restarts it
        CK(cudaEventRecord(t->chain, s));
        CK(cudaEventRecord(slot.free, s));
        if (dev_best) *dev_best = slot.best;
        if (dev_best_count) *dev_best_count = slot.best_counts;
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_tracker_set_motion(rf_tracker t, const rf_motion_config *cfg) {
    static const char *who = "rf_tracker_set_motion";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_MOTION);
    if (rc) return rc;
    const int R = cfg->search ? cfg->search : 12, mi = cfg->min_inliers ? cfg->min_inliers : 12;
    if (R < 1 || R > MOTION_MAX_R) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: search %d, must be 0 or in [1, %d]", who, cfg->search, MOTION_MAX_R));
    if (mi < 3 || mi > MOTION_MAX_BLOCKS)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: min_inliers %d, must be 0 or in [3, %d]", who, cfg->min_inliers, MOTION_MAX_BLOCKS));
    const size_t V = t->cfg.max_videos, B = h->cfg.max_batch;
    if (V * MOTION_THUMB_BYTES > ((size_t)4 << 30))
        return fail(h, RF_ERR_CAPACITY, fmt("%s: a store of %zu videos x %d bytes exceeds 4 GiB", who, V, MOTION_THUMB_BYTES));
    try {
        CK(cudaSetDevice(h->device));
        CK(cudaMalloc(&t->d_mstore, V * MOTION_THUMB_BYTES));
        CK(cudaMalloc(&t->d_mthumbs, B * MOTION_THUMB_BYTES));
        CK(cudaMalloc(&t->d_mblocks, sizeof(MotionBlock) * B * MOTION_MAX_BLOCKS));
        for (auto &s : t->slots) CK(cudaMalloc(&s.motion, sizeof(rf_motion) * B));
    } catch (const CudaFail &f) {
        free_motion(t);
        return fail_cuda(h, f);
    }
    t->motion = true;
    t->mcfg = rf_motion_config{R, mi};
    t->mref.assign(V, {0, 0});
    return RF_OK;
}

int rf_tracker_motion(rf_tracker t, const rf_motion **dev_motion) {
    if (!t) return RF_ERR_INVALID_ARG;
    if (!dev_motion) return fail(t->h, RF_ERR_INVALID_ARG, "rf_tracker_motion: dev_motion is NULL");
    int rc = admit(t, "rf_tracker_motion", Call::MOTION);
    if (rc) return rc;
    *dev_motion = t->motion_slot < 0 ? nullptr : t->slots[t->motion_slot].motion;
    return RF_OK;
}

// rf_follow_config with its defaults applied: search 8, max_mad 24.
static int follow_config(rf_handle h, const char *who, const rf_follow_config *cfg, rf_follow_config &out) {
    const int R = cfg->search ? cfg->search : 8;
    const float mad = cfg->max_mad != 0.f ? cfg->max_mad : 24.f;
    if (R < 1 || R > FOLLOW_MAX_R) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: search %d, must be 0 or in [1, %d]", who, cfg->search, FOLLOW_MAX_R));
    if (!(std::isfinite(mad) && mad > 0.f && mad <= 255.f))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: max_mad %g, must be 0 or finite in (0, 255]", who, (double)cfg->max_mad));
    out = rf_follow_config{R, mad};
    return RF_OK;
}

// f16's template store, measurements and face masks, and the ring's follow records and regions, for rf_tracker_set_follow and
// rf_tracker_set_lookback_follow (admitted, cfg checked).  On failure nothing stays allocated.
static int follow_alloc(rf_tracker t, const char *who, const rf_follow_config &fc) {
    rf_handle h = t->h;
    const size_t V = t->cfg.max_videos, T = t->cfg.max_tracks, B = h->cfg.max_batch;
    if (V * T * FOLLOW_BYTES > ((size_t)4 << 30))
        return fail(h, RF_ERR_CAPACITY, fmt("%s: a store of %zu videos x %zu tracks x %d bytes exceeds 4 GiB", who, V, T, FOLLOW_BYTES));
    try {
        CK(cudaSetDevice(h->device));
        CK(cudaMalloc(&t->d_fstore, V * T * FOLLOW_BYTES));
        CK(cudaMalloc(&t->d_fentries, sizeof(FollowEntry) * V * T));
        CK(cudaMalloc(&t->d_fmeas, sizeof(FollowMeas) * B * T));
        for (auto &s : t->slots) {
            CK(cudaMalloc(&s.follow, sizeof(rf_follow) * B * T));
            CK(cudaMalloc(&s.fregions, sizeof(rf_det) * B * T));
            CK(cudaMalloc(&s.fregion_counts, sizeof(int) * B));
        }
        CK(cudaMalloc(&t->d_fmask, sizeof(rf_det) * B * T));
        CK(cudaMalloc(&t->d_fmask_counts, sizeof(int) * B));
        CK(cudaMemset(t->d_fentries, 0, sizeof(FollowEntry) * V * T));
        CK(cudaDeviceSynchronize());
    } catch (const CudaFail &f) {
        free_follow(t);
        return fail_cuda(h, f);
    }
    t->fcfg = fc;
    return RF_OK;
}

int rf_tracker_set_follow(rf_tracker t, const rf_follow_config *cfg) {
    static const char *who = "rf_tracker_set_follow";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_FOLLOW);
    if (rc) return rc;
    rf_follow_config fc;
    if ((rc = follow_config(h, who, cfg, fc)) || (rc = follow_alloc(t, who, fc))) return rc;
    t->kind = FOLLOW;
    return RF_OK;
}

// The follow step of n frames into ring slot `ring`, on s inside the chain.  In rounds -- the r-th frame of every video of the call,
// then the next -- so that each frame is searched from the state its video's previous frame left; with motion, each round first
// masks the tracks' faces and estimates its frames' motion (the reference: the video's previous frame of the call, else its stored
// thumbnail), and each video's last thumbnail of the call becomes its reference afterwards.
static void follow_rounds(rf_tracker t, unsigned ring, const rf_yuv_frame *frames, const int *videos, int n, cudaStream_t s) {
    rf_tracker_s::Slot &slot = t->slots[ring];
    FollowArgs f = follow_args(t);
    f.follow = slot.follow;
    f.tracks = slot.tracks;
    f.track_counts = slot.counts;
    f.regions = slot.fregions;
    f.region_counts = slot.fregion_counts;
    f.gone = t->kind == BEST ? t->d_fgone : nullptr;      // f22: a following best-shot tracker's removals, by the frame's call index
    std::vector<int> round(n);
    int rounds = 0;
    for (int i = 0; i < n; i++) {
        int r = 0;
        for (int k = 0; k < i; k++) r += videos[k] == videos[i];
        round[i] = r;
        rounds = std::max(rounds, r + 1);
    }
    // f13: one single-frame table per frame, so that a frame's thumbnail, blocks and motion sit at its index in the call
    std::vector<MotionTable> mt;
    MotionCommits commits;
    MotionArgs ma{};
    if (t->motion) {
        mt = motion_tables(t, frames, videos, nullptr, n, 1, commits);
        ma = motion_args(t, ring, t->d_fmask, t->d_fmask_counts, t->cfg.max_tracks);
        f.motion = slot.motion;
        f.mask = t->d_fmask;
        f.mask_counts = t->d_fmask_counts;
        t->motion_slot = (int)ring;
    }
    for (int r = 0; r < rounds; r++) {
        FollowTable tab{};
        std::vector<MotionTable> rt;
        bool oriented = false;
        auto flush = [&]() {
            if (!tab.n) return;
            if (t->motion) {
                CK(launch_follow_mask(f, tab, s));
                CK(launch_motion_estimate(ma, rt.data(), (int)rt.size(), s));
            }
            CK(launch_follow_round(f, tab, s, oriented));
            tab.n = 0;
            oriented = false;
            rt.clear();
        };
        for (int i = 0; i < n; i++) {
            if (round[i] != r) continue;
            tab.f[tab.n] = follow_frame(t, frames[i], videos[i], i);
            oriented |= tab.f[tab.n++].bits != 0;
            if (t->motion) rt.push_back(mt[i]);
            if (tab.n == TRACK_MAX_FRAMES) flush();
        }
        flush();
    }
    if (t->motion) motion_commit(t, commits, s);
    t->follow_slot = (int)ring;
}

// f22: the best-shot half of a follow call of a following best-shot tracker, after follow_rounds on s: each chunk of TRACK_MAX_FRAMES
// frames selects its removals' EXIT shots (no records: nothing is measured or stored) and emits them.
static void best_follow_issue(rf_tracker t, const rf_tracker_s::Slot &slot, const FrameCall &c, cudaStream_t s) {
    const int T = t->cfg.max_tracks;
    for (int i0 = 0; i0 < c.n; i0 += TRACK_MAX_FRAMES) {
        const int m = std::min(TRACK_MAX_FRAMES, c.n - i0);
        BestArgs b = best_args(t, slot, c, i0);
        b.gone = t->d_fgone + (size_t)i0 * T;
        CK(launch_best_follow(b, best_table(c.videos + i0, m), s));
    }
}

int rf_track_follow_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_track **dev_tracks,
                           const int32_t **dev_track_counts) {
    FrameCall c{.who = "rf_track_follow_device", .call = Call::FOLLOW, .source = FrameCall::FOLLOW, .t = t, .frames = frames, .videos = videos,
                .n = n, .tracks = dev_tracks, .track_counts = dev_track_counts};
    return frame_call(c);
}

int rf_tracker_follow(rf_tracker t, const rf_follow **dev_follow) {
    if (!t) return RF_ERR_INVALID_ARG;
    if (!dev_follow) return fail(t->h, RF_ERR_INVALID_ARG, "rf_tracker_follow: dev_follow is NULL");
    int rc = admit(t, "rf_tracker_follow", Call::FOLLOWS);
    if (rc) return rc;
    *dev_follow = t->follow_slot < 0 ? nullptr : t->slots[t->follow_slot].follow;
    return RF_OK;
}

int rf_tracker_debug_state(rf_tracker t, int video, double *out, int cap) {
    static const char *who = "rf_tracker_debug_state";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (video < 0 || video >= t->cfg.max_videos) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: video %d, must be in [0, %d)", who, video, t->cfg.max_videos));
    if (cap > 0 && !out) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out is NULL", who));
    const int T = t->cfg.max_tracks;
    TrackVideo hv{};
    std::vector<TrackState> st(T);
    try {
        CK(cudaSetDevice(h->device));
        CK(cudaEventSynchronize(t->chain));
        CK(cudaMemcpy(&hv, t->d_videos + video, sizeof hv, cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(st.data(), t->d_state + (size_t)video * T, sizeof(TrackState) * T, cudaMemcpyDeviceToHost));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    std::vector<const TrackState *> live;
    for (const TrackState &k : st) if (k.id) live.push_back(&k);
    std::sort(live.begin(), live.end(), [](const TrackState *x, const TrackState *y) { return x->id < y->id; });
    std::vector<double> v = {(double)live.size(), (double)(hv.issued + 1), (double)hv.frames, (double)hv.overflow};
    for (const TrackState *k : live) {
        for (int x : {k->id, k->state, k->hits, k->age, k->lost}) v.push_back(x);
        for (const double *arr : {k->m, k->u, k->p00, k->p01, k->p11}) v.insert(v.end(), arr, arr + 4);
    }
    std::copy(v.begin(), v.begin() + std::min<size_t>(v.size(), (size_t)std::max(cap, 0)), out);
    return (int)live.size();
}

// ---- f22 live and following best shots ---------------------------------------------------------------------------------------
int rf_tracker_set_best_live(rf_tracker t, const rf_best_live_config *cfg) {
    static const char *who = "rf_tracker_set_best_live";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_BEST_LIVE);
    if (rc) return rc;
    const float fq = cfg->first_quality == 0.f ? 0.3f : cfg->first_quality, imp = cfg->improve == 0.f ? 0.2f : cfg->improve;
    const int gap = cfg->min_gap == 0 ? 30 : cfg->min_gap;
    if (!(fq > 0.f && fq <= 1.f)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: first_quality %g, must be 0 or in (0, 1]", who, (double)cfg->first_quality));
    if (!(std::isfinite(imp) && imp > 0.f)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: improve %g, must be 0 or finite and positive", who, (double)cfg->improve));
    if (gap < 1 || gap > (1 << 20)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: min_gap %d, must be 0 or in [1, %d]", who, cfg->min_gap, 1 << 20));
    BestLiveArgs l{};
    const size_t V = t->cfg.max_videos, T = t->cfg.max_tracks, F = h->cfg.max_faces, M = std::min<size_t>(h->cfg.max_batch, TRACK_MAX_FRAMES);
    try {
        CK(cudaSetDevice(h->device));
        CK(cudaMalloc(&l.live, sizeof(BestLive) * V * T));
        TrackLife *life = nullptr;
        CK(cudaMalloc(&life, sizeof(TrackLife) * M * F));
        l.life = life;
        CK(cudaMemset(l.live, 0, sizeof(BestLive) * V * T));
        CK(cudaDeviceSynchronize());
    } catch (const CudaFail &f) {
        cudaFree(l.live);
        cudaFree((void *)l.life);
        return fail_cuda(h, f);
    }
    l.first_quality = (double)fq;
    l.ratio = 1.0 + (double)imp;
    l.min_gap = gap;
    t->bl = l;
    t->best_live = true;
    return RF_OK;
}

int rf_tracker_set_best_follow(rf_tracker t, const rf_follow_config *cfg) {
    static const char *who = "rf_tracker_set_best_follow";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_BEST_FOLLOW);
    if (rc) return rc;
    rf_follow_config fc;
    if ((rc = follow_config(h, who, cfg, fc)) || (rc = follow_alloc(t, who, fc))) return rc;
    try {
        CK(cudaMalloc(&t->d_fgone, sizeof(TrackGone) * h->cfg.max_batch * t->cfg.max_tracks));
    } catch (const CudaFail &f) {
        free_follow(t);
        return fail_cuda(h, f);
    }
    t->best_follow = true;
    return RF_OK;
}

int rf_track_follow_best_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, void *dev_best_crops, double *dev_best_mats,
                                const rf_best_shot **dev_best, const int32_t **dev_best_counts, const rf_track **dev_tracks,
                                const int32_t **dev_track_counts) {
    FrameCall c{.who = "rf_track_follow_best_device", .call = Call::BEST_FOLLOW, .source = FrameCall::FOLLOW, .sink = FrameCall::BEST, .t = t,
                .frames = frames, .videos = videos, .n = n, .crops = dev_best_crops, .mats = dev_best_mats, .tracks = dev_tracks,
                .track_counts = dev_track_counts, .best = dev_best, .best_counts = dev_best_counts};
    return frame_call(c);
}

// ---- f12 redaction (redact.cuh) -------------------------------------------------------------------------------------------------
static int redact_margin(rf_handle h, const char *who, float margin, double &out) {
    const float m = margin != 0.f ? margin : 0.25f;
    if (!(std::isfinite(m) && m > 0.f && m <= 1.f))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: margin %g, must be 0 or finite in (0, 1]", who, (double)m));
    out = (double)m;
    return RF_OK;
}

// params (NULL: defaults) -> blocks and margin
static int redact_params(rf_handle h, const char *who, const rf_redact_params *p, RedactSpec &r) {
    r = RedactSpec{};
    r.blocks = p && p->blocks ? p->blocks : 8;
    if (r.blocks < 1 || r.blocks > REDACT_MAX_BLOCKS)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: blocks %d, must be 0 or in [1, %d]", who, r.blocks, REDACT_MAX_BLOCKS));
    return redact_margin(h, who, p ? p->margin : 0.f, r.margin);
}

// style (NULL: the zeroed struct) -> kind, shape, blocks, detail and margin
static int redact_style(rf_handle h, const char *who, const rf_redact_style *st, RedactSpec &r) {
    const rf_redact_style z{};
    if (!st) st = &z;
    r = RedactSpec{};
    r.kind = st->kind ? st->kind : REDACT_BLUR;
    r.shape = st->shape ? st->shape : REDACT_ELLIPSE;
    if (r.kind != REDACT_MOSAIC && r.kind != REDACT_BLUR)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: kind %d, must be 0, RF_REDACT_MOSAIC or RF_REDACT_BLUR", who, st->kind));
    if (r.shape != REDACT_RECT && r.shape != REDACT_ELLIPSE)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: shape %d, must be 0, RF_REDACT_RECT or RF_REDACT_ELLIPSE", who, st->shape));
    if (r.kind == REDACT_MOSAIC) {
        if (st->detail) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: detail %d, must be 0 for the mosaic", who, st->detail));
        r.blocks = st->blocks ? st->blocks : 8;
        if (r.blocks < 1 || r.blocks > REDACT_MAX_BLOCKS)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: blocks %d, must be 0 or in [1, %d]", who, r.blocks, REDACT_MAX_BLOCKS));
    } else {
        if (st->blocks) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: blocks %d, must be 0 for the blur", who, st->blocks));
        r.blocks = 1;         // the geometry's cell side, unused by the blur
        r.detail = st->detail ? st->detail : 4;
        if (r.detail < 1 || r.detail > BLUR_MAX_DETAIL)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: detail %d, must be 0 or in [1, %d]", who, r.detail, BLUR_MAX_DETAIL));
    }
    return redact_margin(h, who, st->margin, r.margin);
}

// The records, scales and tracks of a redaction call.
static int check_redact_inputs(rf_handle h, const char *who, int n, const rf_det *dets, const int32_t *counts, const float *scales, rf_tracker t,
                               const rf_track *tracks, const int32_t *track_counts) {
    if (n > 0 && (!dets || !counts)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL records or counts", who));
    const bool any = t || tracks || track_counts;
    if (any && !(t && tracks && track_counts))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: the tracker, its tracks and their counts go together (all three or none)", who));
    if (t && t->h != h) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: the tracker belongs to another handle", who));
    for (int i = 0; scales && i < n; i++)
        if (!(std::isfinite(scales[i]) && scales[i] > 0.f))
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: scale %g, must be finite and positive", who, i, (double)scales[i]));
    return RF_OK;
}

// Refuses two frames whose plane byte ranges overlap: a later chunk's measure would read pixels an earlier chunk has written, and
// within a chunk two regions' writes could land on one byte.  ranges: (first byte, one past the last, frame).  A sweep in address
// order that keeps the furthest end seen (and the furthest end of any other frame) finds every overlap of two frames.
static int check_disjoint(rf_handle h, const char *who, std::vector<std::array<uintptr_t, 3>> ranges) {
    std::sort(ranges.begin(), ranges.end());
    uintptr_t end1 = 0, end2 = 0;
    uintptr_t frame1 = ~(uintptr_t)0;        // end1: the furthest end, of frame1; end2: the furthest end of any other frame
    for (const auto &r : ranges) {
        const uintptr_t other = r[2] == frame1 ? end2 : end1;
        if (r[0] < other) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d overlaps the bytes of another frame of the call", who, (int)r[2]));
        if (r[1] > end1) {
            if (r[2] != frame1) { end2 = end1; frame1 = r[2]; }
            end1 = r[1];
        } else if (r[2] != frame1 && r[1] > end2) {
            end2 = r[1];
        }
    }
    return RF_OK;
}

static std::vector<std::array<uintptr_t, 3>> yuv_ranges(const rf_yuv_frame *frames, int n) {
    std::vector<std::array<uintptr_t, 3>> r;
    for (int i = 0; i < n; i++) {
        const rf_yuv_frame &f = frames[i];
        const uintptr_t y = (uintptr_t)f.y, u = (uintptr_t)f.u, v = (uintptr_t)f.v, ch = f.height / 2 - 1;
        r.push_back({y, y + (uintptr_t)(f.height - 1) * f.y_pitch + f.width, (uintptr_t)i});
        if (f.uv_step == 2) {
            const uintptr_t lo = std::min(u, v);
            r.push_back({lo, lo + ch * f.uv_pitch + f.width, (uintptr_t)i});
        } else {
            r.push_back({u, u + ch * f.uv_pitch + f.width / 2, (uintptr_t)i});
            r.push_back({v, v + ch * f.uv_pitch + f.width / 2, (uintptr_t)i});
        }
    }
    return r;
}

static Ctx &last_ctx(rf_handle h) {
    for (Ctx &c : h->ctx)
        if (c.stream == h->last_stream) return c;
    return h->ctx[0];
}

// Issues the redaction of `frames` on context c's stream, into c's scratch (sized for max_batch frames -- or more, for a drain -- of
// this call's region capacity and blocks, and for BLUR the frames' scratch planes; a larger need waits for the context before the
// scratch is replaced).  records: the records per frame of dets (0: max_faces; f15's look-back regions have more).
template <typename Dst>
static void redact_issue(rf_handle h, Ctx &c, std::vector<RedactFrameT<Dst>> frames, const rf_det *dets, const int32_t *counts, rf_tracker t,
                         const rf_track *tracks, const int32_t *track_counts, const RedactSpec &spec, int records = 0) {
    RedactArgs a{};
    a.n = (int)frames.size();
    a.blocks = spec.blocks;
    a.margin = spec.margin;
    a.kind = spec.kind;
    a.shape = spec.shape;
    a.detail = spec.detail;
    a.max_faces = records ? records : h->cfg.max_faces;
    a.max_tracks = t ? t->cfg.max_tracks : 0;
    a.cap = a.max_faces + a.max_tracks;
    a.dets = dets;
    a.counts = counts;
    a.tracks = tracks;
    a.track_counts = track_counts;
    const size_t tables = (redact_scratch_bytes(std::max(h->cfg.max_batch, a.n), a.cap, a.blocks) + 255) & ~(size_t)255;
    size_t need = tables;
    if (spec.kind == REDACT_BLUR)
        for (const auto &f : frames) need += (blur_plane_bytes(kRedactYuv<Dst>, f.w, f.h) + 255) & ~(size_t)255;
    if (need > c.redact_bytes) {
        CK(cudaStreamSynchronize(c.stream));
        CK(cudaFree(c.d_redact));
        c.d_redact = nullptr;
        c.redact_bytes = 0;
        CK(cudaMalloc(&c.d_redact, need));
        c.redact_bytes = need;
    }
    redact_carve(a, c.d_redact);
    if (spec.kind == REDACT_BLUR) {
        size_t off = tables;
        for (auto &f : frames) {
            f.blur = static_cast<uint8_t *>(c.d_redact) + off;
            off += (blur_plane_bytes(kRedactYuv<Dst>, f.w, f.h) + 255) & ~(size_t)255;
        }
    }
    CK(launch_redact(a, frames.data(), h->num_sms, c.stream));
}

static std::vector<RedactFrameT<YuvPlanesW>> yuv_redact_table(const rf_yuv_frame *frames, int n, const float *scales) {
    std::vector<RedactFrameT<YuvPlanesW>> v(n);
    for (int i = 0; i < n; i++) {
        const rf_yuv_frame &f = frames[i];
        v[i] = RedactFrameT<YuvPlanesW>{YuvPlanesW{const_cast<uint8_t *>(f.y), const_cast<uint8_t *>(f.u), const_cast<uint8_t *>(f.v), f.y_pitch,
                                                   f.uv_pitch, f.uv_step},
                                        f.width, f.height, scales ? scales[i] : 1.f, nullptr};
    }
    return v;
}

// f20: the frames shown in orientations orients[i] (EXIF), as the oriented redaction kernels address them: each plane's displayed
// sample (0, 0) and strides (yuv.cuh plane_map), and the displayed size.
static std::vector<RedactFrameT<YuvPlanesWO>> yuv_redact_table_oriented(const rf_yuv_frame *frames, const int *orients, int n, const float *scales) {
    std::vector<RedactFrameT<YuvPlanesWO>> v(n);
    for (int i = 0; i < n; i++) {
        const rf_yuv_frame &f = frames[i];
        const int bits = lb_orientation_bits(orients[i]);
        const bool tr = bits & LB_TRANSPOSE;
        const int dw = tr ? f.height : f.width, dh = tr ? f.width : f.height;
        const PlaneMap y = plane_map(bits, dw, dh, f.y_pitch, 1), c = plane_map(bits, dw / 2, dh / 2, f.uv_pitch, f.uv_step);
        v[i] = RedactFrameT<YuvPlanesWO>{YuvPlanesWO{const_cast<uint8_t *>(f.y) + y.off, const_cast<uint8_t *>(f.u) + c.off,
                                                     const_cast<uint8_t *>(f.v) + c.off, y.xs, y.ys, c.xs, c.ys},
                                         dw, dh, scales ? scales[i] : 1.f, nullptr};
    }
    return v;
}

// redact_issue on YUV frames, frame i shown in EXIF orientation orients[i] (NULL: every frame upright): the oriented kernels when some
// frame is not at orientation 1, else the upright ones.
static void redact_yuv_issue(rf_handle h, Ctx &c, const rf_yuv_frame *frames, const int *orients, int n, const float *scales, const rf_det *dets,
                             const int32_t *counts, rf_tracker t, const rf_track *tracks, const int32_t *track_counts, const RedactSpec &spec,
                             int records = 0) {
    if (orients && std::any_of(orients, orients + n, [](int o) { return o != 1; }))
        redact_issue(h, c, yuv_redact_table_oriented(frames, orients, n, scales), dets, counts, t, tracks, track_counts, spec, records);
    else
        redact_issue(h, c, yuv_redact_table(frames, n, scales), dets, counts, t, tracks, track_counts, spec, records);
}

// The f12 and f14 entry points share one implementation each: `resolve` checks the params or the style where f12 checks its params.
template <typename Resolve>
static int redact_yuv_impl(rf_handle h, const char *who, const rf_yuv_frame *frames, int n, const rf_det *dev_dets, const int32_t *dev_counts,
                           const float *scales, rf_tracker t, const rf_track *dev_tracks, const int32_t *dev_track_counts, Resolve resolve) {
    if (!h) return RF_ERR_INVALID_ARG;
    int rc = check_frames(h, who, frames, n, RF_YUV_BT601);      // the matrix plays no part: the mosaic is per plane
    if (rc) return rc;
    RedactSpec spec;
    if ((rc = resolve(spec))) return rc;
    if ((rc = check_redact_inputs(h, who, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts))) return rc;
    if ((rc = check_disjoint(h, who, yuv_ranges(frames, n)))) return rc;
    if (n == 0) return RF_OK;
    try {
        CK(cudaSetDevice(h->device));
        redact_issue(h, last_ctx(h), yuv_redact_table(frames, n, scales), dev_dets, dev_counts, t, dev_tracks, dev_track_counts, spec);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

template <typename Resolve>
static int redact_bgr_impl(rf_handle h, const char *who, uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides,
                           int n, const rf_det *dev_dets, const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                           const int32_t *dev_track_counts, Resolve resolve) {
    if (!h) return RF_ERR_INVALID_ARG;
    const BgrImages src{dev_bgr, widths, heights, row_strides, nullptr, false};
    int rc = src.check(h, who, n);
    if (rc) return rc;
    RedactSpec spec;
    if ((rc = resolve(spec))) return rc;
    if ((rc = check_redact_inputs(h, who, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts))) return rc;
    std::vector<std::array<uintptr_t, 3>> ranges;
    for (int i = 0; i < n; i++) {
        const uintptr_t p = (uintptr_t)dev_bgr[i];
        ranges.push_back({p, p + (uintptr_t)(heights[i] - 1) * src.stride(i) + 3 * (uintptr_t)widths[i], (uintptr_t)i});
    }
    if ((rc = check_disjoint(h, who, ranges))) return rc;
    if (n == 0) return RF_OK;
    try {
        CK(cudaSetDevice(h->device));
        std::vector<RedactFrameT<BgrRowsW>> v(n);
        for (int i = 0; i < n; i++) v[i] = RedactFrameT<BgrRowsW>{BgrRowsW{dev_bgr[i], src.stride(i)}, widths[i], heights[i], scales ? scales[i] : 1.f, nullptr};
        redact_issue(h, last_ctx(h), v, dev_dets, dev_counts, t, dev_tracks, dev_track_counts, spec);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

// With a tracker, the tracker's frame call; without, the detect and then the redaction of its records, on the forward's context.
static int detect_yuv_redact_impl(rf_handle h, const char *who, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix,
                                  float thr, float nms, const rf_redact_style *style, const rf_track **dev_tracks,
                                  const int32_t **dev_track_counts, const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    if (t) {
        FrameCall c{.who = who, .call = Call::DETECT, .source = FrameCall::DETECT, .sink = FrameCall::REDACT, .h = h, .t = t, .frames = frames,
                    .videos = videos, .n = n, .matrix = matrix, .thr = thr, .nms = nms, .style = style, .tracks = dev_tracks,
                    .track_counts = dev_track_counts, .out_dets = dev_dets, .out_counts = dev_counts, .out_scales = out_scales};
        return frame_call(c);
    }
    if (!h) return RF_ERR_INVALID_ARG;
    const YuvFrames src{frames, matrix, nullptr, false};
    int rc = src.check(h, who, n);
    if (rc) return rc;
    RedactSpec spec;
    if ((rc = redact_style(h, who, style, spec))) return rc;
    if ((rc = check_disjoint(h, who, yuv_ranges(frames, n)))) return rc;
    if (n == 0) return RF_OK;
    std::vector<float> scales(n);
    const rf_det *dets = nullptr;
    const int32_t *counts = nullptr;
    if ((rc = yuv_device_impl(h, who, src, n, thr, nms, nullptr, nullptr, nullptr, &dets, &counts, scales.data()))) return rc;
    if (dev_dets) *dev_dets = dets;
    if (dev_counts) *dev_counts = counts;
    if (out_scales) std::copy(scales.begin(), scales.end(), out_scales);
    if (dev_tracks) *dev_tracks = nullptr;
    if (dev_track_counts) *dev_track_counts = nullptr;
    try {
        redact_issue(h, last_ctx(h), yuv_redact_table(frames, n, scales.data()), dets, counts, nullptr, nullptr, nullptr, spec);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}


int rf_redact_yuv_device(rf_handle h, const rf_yuv_frame *frames, int n, const rf_det *dev_dets, const int32_t *dev_counts, const float *scales,
                         rf_tracker t, const rf_track *dev_tracks, const int32_t *dev_track_counts, const rf_redact_params *params) {
    static const char *who = "rf_redact_yuv_device";
    return redact_yuv_impl(h, who, frames, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts,
                           [&](RedactSpec &r) { return redact_params(h, who, params, r); });
}

int rf_redact_yuv_device_style(rf_handle h, const rf_yuv_frame *frames, int n, const rf_det *dev_dets, const int32_t *dev_counts, const float *scales,
                               rf_tracker t, const rf_track *dev_tracks, const int32_t *dev_track_counts, const rf_redact_style *style) {
    static const char *who = "rf_redact_yuv_device_style";
    return redact_yuv_impl(h, who, frames, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts,
                           [&](RedactSpec &r) { return redact_style(h, who, style, r); });
}

// f20: rf_redact_yuv_device_style on T_o(frame), mapped back.  A call whose frames are all at orientation 1 issues the upright kernels.
int rf_redact_yuv_oriented_device_style(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n, const rf_det *dev_dets,
                                        const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                                        const int32_t *dev_track_counts, const rf_redact_style *style) {
    static const char *who = "rf_redact_yuv_oriented_device_style";
    if (!h) return RF_ERR_INVALID_ARG;
    int rc = check_frames(h, who, frames, n, RF_YUV_BT601);
    if (rc || (rc = check_orientations(h, who, orientations, n))) return rc;
    RedactSpec spec;
    if ((rc = redact_style(h, who, style, spec))) return rc;
    if ((rc = check_redact_inputs(h, who, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts))) return rc;
    if ((rc = check_disjoint(h, who, yuv_ranges(frames, n)))) return rc;
    if (n == 0) return RF_OK;
    try {
        CK(cudaSetDevice(h->device));
        redact_yuv_issue(h, last_ctx(h), frames, orientations, n, scales, dev_dets, dev_counts, t, dev_tracks, dev_track_counts, spec);
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    return RF_OK;
}

int rf_redact_device(rf_handle h, uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides, int n,
                     const rf_det *dev_dets, const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                     const int32_t *dev_track_counts, const rf_redact_params *params) {
    static const char *who = "rf_redact_device";
    return redact_bgr_impl(h, who, dev_bgr, widths, heights, row_strides, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts,
                           [&](RedactSpec &r) { return redact_params(h, who, params, r); });
}

int rf_redact_device_style(rf_handle h, uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides, int n,
                           const rf_det *dev_dets, const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                           const int32_t *dev_track_counts, const rf_redact_style *style) {
    static const char *who = "rf_redact_device_style";
    return redact_bgr_impl(h, who, dev_bgr, widths, heights, row_strides, n, dev_dets, dev_counts, scales, t, dev_tracks, dev_track_counts,
                           [&](RedactSpec &r) { return redact_style(h, who, style, r); });
}

int rf_detect_yuv_redact_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix, float thr, float nms,
                                const rf_redact_params *params, const rf_track **dev_tracks, const int32_t **dev_track_counts,
                                const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    const rf_redact_style f12{REDACT_MOSAIC, REDACT_RECT, params ? params->blocks : 0, 0, params ? params->margin : 0.f};   // as RedactSpec
    return detect_yuv_redact_impl(h, "rf_detect_yuv_redact_device", t, frames, videos, n, matrix, thr, nms, &f12, dev_tracks, dev_track_counts,
                                  dev_dets, dev_counts, out_scales);
}

int rf_detect_yuv_redact_device_style(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix, float thr,
                                      float nms, const rf_redact_style *style, const rf_track **dev_tracks, const int32_t **dev_track_counts,
                                      const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales) {
    return detect_yuv_redact_impl(h, "rf_detect_yuv_redact_device_style", t, frames, videos, n, matrix, thr, nms, style, dev_tracks,
                                  dev_track_counts, dev_dets, dev_counts, out_scales);
}

int rf_track_follow_redact_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_redact_style *style,
                                  const rf_track **dev_tracks, const int32_t **dev_track_counts) {
    FrameCall c{.who = "rf_track_follow_redact_device", .call = Call::FOLLOW, .source = FrameCall::FOLLOW, .sink = FrameCall::REDACT, .t = t,
                .frames = frames, .videos = videos, .n = n, .style = style, .tracks = dev_tracks, .track_counts = dev_track_counts};
    return frame_call(c);
}

// ---- f15 look-back redaction (lookback.cuh) --------------------------------------------------------------------------------------
int rf_tracker_set_lookback(rf_tracker t, const rf_lookback_config *cfg) {
    static const char *who = "rf_tracker_set_lookback";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_LOOKBACK);
    if (rc) return rc;
    const int L = cfg->frames ? cfg->frames : 15;
    const float grow = cfg->grow != 0.f ? cfg->grow : 0.1f;
    if (L < 1 || L > LOOKBACK_MAX_L) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frames %d, must be 0 or in [1, %d]", who, cfg->frames, LOOKBACK_MAX_L));
    if (!(std::isfinite(grow) && grow > 0.f && grow <= 1.f))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: grow %g, must be 0 or finite in (0, 1]", who, (double)cfg->grow));
    const size_t rows = std::max(h->cfg.max_batch, L), recs = lookback_records(h->cfg.max_faces, t->cfg.max_tracks, L, false);
    try {
        CK(cudaSetDevice(h->device));
        for (auto &s : t->slots) {
            CK(cudaMalloc(&s.lb_boxes, sizeof(rf_det) * rows * recs));
            CK(cudaMalloc(&s.lb_counts, sizeof(int) * rows));
        }
    } catch (const CudaFail &f) {
        free_lookback(t);
        return fail_cuda(h, f);
    }
    t->kind = LOOKBACK;
    t->lb_frames = L;
    t->lb_grow = grow;
    t->lbv.assign(t->cfg.max_videos, {});
    return RF_OK;
}

int rf_tracker_set_lookback_search(rf_tracker t, const rf_follow_config *cfg) {
    static const char *who = "rf_tracker_set_lookback_search";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_LOOKBACK_SEARCH);
    if (rc) return rc;
    rf_follow_config fc;
    if ((rc = follow_config(h, who, cfg, fc))) return rc;
    const int L = t->lb_frames;
    const size_t B = h->cfg.max_batch, bcap = std::min(h->cfg.max_faces, t->cfg.max_tracks);
    const size_t rows = std::max(h->cfg.max_batch, L), recs = lookback_records(h->cfg.max_faces, t->cfg.max_tracks, L, true);
    std::vector<rf_tracker_s::Slot> grown(t->slots.size());
    try {
        CK(cudaSetDevice(h->device));
        for (auto &s : grown) {
            CK(cudaMalloc(&s.lb_boxes, sizeof(rf_det) * rows * recs));
            CK(cudaMalloc(&s.lb_steps, sizeof(rf_follow) * B * bcap * L));
            CK(cudaMalloc(&s.lb_lengths, sizeof(int) * B * bcap));
        }
    } catch (const CudaFail &f) {
        for (auto &s : grown) { cudaFree(s.lb_boxes); cudaFree(s.lb_steps); cudaFree(s.lb_lengths); }
        return fail_cuda(h, f);
    }
    for (size_t i = 0; i < t->slots.size(); i++) {     // no call has used the ring's region records yet
        cudaFree(t->slots[i].lb_boxes);
        t->slots[i].lb_boxes = grown[i].lb_boxes;
        t->slots[i].lb_steps = grown[i].lb_steps;
        t->slots[i].lb_lengths = grown[i].lb_lengths;
    }
    t->lb_search = true;
    t->lscfg = fc;
    return RF_OK;
}

int rf_tracker_lookback_search(rf_tracker t, const rf_follow **dev_steps, const int32_t **dev_lengths) {
    if (!t) return RF_ERR_INVALID_ARG;
    int rc = admit(t, "rf_tracker_lookback_search", Call::LOOKBACK_SEARCH);
    if (rc) return rc;
    const bool any = t->lb_search_slot >= 0;
    if (dev_steps) *dev_steps = any ? t->slots[t->lb_search_slot].lb_steps : nullptr;
    if (dev_lengths) *dev_lengths = any ? t->slots[t->lb_search_slot].lb_lengths : nullptr;
    return RF_OK;
}

// An out frame of a look-back call: a valid descriptor with the size and layout (uv_step, chroma order) of the frames it receives.
static int check_out_frame(rf_handle h, const char *who, const rf_yuv_frame &o, int i, int w, int ht, int step, bool v_first) {
    if (!o.y || !o.u || !o.v) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out frame %d has a NULL plane", who, i));
    if (o.width != w || o.height != ht || o.uv_step != step)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out frame %d is %dx%d with uv_step %d, its video's frames are %dx%d with uv_step %d", who, i,
                                               o.width, o.height, o.uv_step, w, ht, step));
    const uintptr_t u = (uintptr_t)o.u, v = (uintptr_t)o.v;
    if (step == 2 && ((v + 1 != u && u + 1 != v) || (v < u) != v_first))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out frame %d: semi-planar u and v must be adjacent, in the input's order", who, i));
    if (o.y_pitch < w || o.uv_pitch < w / 2 * step)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: out frame %d: pitches %d / %d below the row bytes %d / %d", who, i, o.y_pitch, o.uv_pitch, w, w / 2 * step));
    return RF_OK;
}

static bool same_frame(const rf_yuv_frame &a, const rf_yuv_frame &b) {
    return a.y == b.y && a.u == b.u && a.v == b.v && a.y_pitch == b.y_pitch && a.uv_pitch == b.uv_pitch && a.uv_step == b.uv_step &&
           a.width == b.width && a.height == b.height;
}

static uint8_t *lb_log(rf_tracker t, const rf_tracker_s::LookbackVideo &v) { return v.d + (size_t)t->lb_frames * v.frame_bytes; }
static size_t lb_slot_bytes(rf_tracker t) { return lookback_slot_bytes(t->h->cfg.max_faces, t->cfg.max_tracks, t->lb_search ? t->lb_frames : 0); }
static int lb_records(rf_tracker t) { return lookback_records(t->h->cfg.max_faces, t->cfg.max_tracks, t->lb_frames, t->lb_search); }

// The swap entry of one frame: its planes (in: NULL for a drain; out: NULL when it emits nothing) and its buffer slot.
static LookbackSwapFrame lb_swap_frame(const rf_yuv_frame *in, const rf_yuv_frame *out, uint8_t *slot) {
    const rf_yuv_frame &g = in ? *in : *out;
    LookbackSwapFrame f{};
    f.w = g.width;
    f.h = g.height;
    f.planar = g.uv_step == 1;
    f.slot = slot;
    if (in) {
        f.in[0] = in->y;
        f.in[1] = f.planar ? in->u : std::min(in->u, in->v);
        f.in_v = in->v;
        f.in_pitch[0] = in->y_pitch;
        f.in_pitch[1] = in->uv_pitch;
    }
    if (out) {
        f.out[0] = const_cast<uint8_t *>(out->y);
        f.out[1] = const_cast<uint8_t *>(f.planar ? out->u : std::min(out->u, out->v));
        f.out_v = const_cast<uint8_t *>(out->v);
        f.out_pitch[0] = out->y_pitch;
        f.out_pitch[1] = out->uv_pitch;
    }
    return f;
}

static void lb_swap(const std::vector<LookbackSwapFrame> &v, cudaStream_t s) {
    for (size_t i0 = 0; i0 < v.size(); i0 += LOOKBACK_TABLE) {
        LookbackSwapTable tb{};
        int rows = 0;
        for (size_t i = i0; i < std::min(v.size(), i0 + LOOKBACK_TABLE); i++) {
            tb.f[tb.n++] = v[i];
            rows = std::max(rows, v[i].h + (v[i].planar ? v[i].h : v[i].h / 2));
        }
        CK(launch_lookback_swap(tb, rows, s));
    }
}

// The (a) + (b) + (c) records of the emitted frames {video, e, span} into ring slot `slot`'s look-back boxes.
static void lb_boxes(rf_tracker t, rf_tracker_s::Slot &slot, const std::vector<std::array<long long, 3>> &em, cudaStream_t s) {
    LookbackArgs a{};
    a.max_faces = t->h->cfg.max_faces;
    a.max_tracks = t->cfg.max_tracks;
    a.slot_bytes = lb_slot_bytes(t);
    a.ring = 2 * t->lb_frames;
    a.grow = (double)t->lb_grow;
    a.out = slot.lb_boxes;
    a.out_counts = slot.lb_counts;
    a.records = lb_records(t);
    a.search = t->lb_search ? t->lscfg.search : 0;
    a.L = t->lb_frames;
    for (size_t j0 = 0; j0 < em.size(); j0 += LOOKBACK_TABLE) {
        LookbackBoxTable tb{};
        tb.j0 = (int)j0;
        for (size_t j = j0; j < std::min(em.size(), j0 + LOOKBACK_TABLE); j++, tb.n++) {
            tb.log[tb.n] = lb_log(t, t->lbv[em[j][0]]);
            tb.e_slot[tb.n] = (int)(em[j][1] % a.ring);
            tb.span[tb.n] = (int)em[j][2];
        }
        CK(launch_lookback_boxes(a, tb, s));
    }
}

// f17: the chains of the call's births (k_lookback_search), after the log and before the swap.  Tables take whole videos: each video's
// frames of the call, in number order, so that a step on an earlier frame of the call finds it in the same table.
static void lb_search(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const std::vector<long long> &num, const LookbackArgs &a,
                      cudaStream_t s) {
    std::vector<std::vector<int>> by;            // the call's frames of each video, in first-appearance order
    std::vector<int> vid;
    for (int i = 0; i < n; i++) {
        auto it = std::find(vid.begin(), vid.end(), videos[i]);
        if (it == vid.end()) {
            vid.push_back(videos[i]);
            by.emplace_back();
            it = vid.end() - 1;
        }
        by[it - vid.begin()].push_back(i);
    }
    LookbackSearchTable tb{};
    bool oriented = false;
    for (size_t q = 0; q <= by.size(); q++) {
        if (tb.n > 0 && (q == by.size() || tb.n + (int)by[q].size() > LOOKBACK_SEARCH_FRAMES || tb.nv == LOOKBACK_SEARCH_VIDEOS)) {
            CK(launch_lookback_search(a, tb, s, oriented));
            tb = LookbackSearchTable{};
            oriented = false;
        }
        if (q == by.size()) break;
        const rf_tracker_s::LookbackVideo &lv = t->lbv[vid[q]];
        LookbackSearchVideo &v = tb.v[tb.nv];
        v.buf = lv.d;
        v.log = lb_log(t, lv);
        v.frame_bytes = lv.frame_bytes;
        v.num0 = num[by[q][0]];
        const std::array<int, 2> size = shown_size(t, vid[q], lv.w, lv.h);      // f20: searched as displayed
        v.w = size[0];
        v.h = size[1];
        v.bits = video_bits(t, vid[q]);
        oriented |= v.bits != 0;
        v.first = tb.n;
        for (int i : by[q]) tb.f[tb.n++] = LookbackSearchFrame{frames[i].y, frames[i].y_pitch, tb.nv, i};
        tb.nv++;
    }
}

// Allocates (or, at a new frame size, replaces) the buffer of a video that has no buffered frames.  false: the allocation failed.
static bool lb_alloc(rf_tracker t, rf_tracker_s::LookbackVideo &v, const rf_yuv_frame &f) {
    const size_t fb = ((size_t)f.width * f.height * 3 / 2 + 255) & ~(size_t)255;
    const size_t bytes = (size_t)t->lb_frames * fb + 2 * (size_t)t->lb_frames * lb_slot_bytes(t);
    if (v.d && v.frame_bytes == fb) return true;
    if (v.d) {
        CK(cudaEventSynchronize(t->chain));      // the last drain's swap may still read it
        CK(cudaFree(v.d));
        v.d = nullptr;
    }
    if (cudaMalloc(&v.d, bytes) != cudaSuccess) {
        cudaGetLastError();
        v.d = nullptr;
        return false;
    }
    v.frame_bytes = fb;
    return true;
}

// The frame numbers of a look-back call's n frames (each video's count on), and every rule its frames and out frames must keep; checked
// before anything is launched.  A video's size and layout are those of its buffered frames, else of its first frame in the call.
// seen: (video, its first frame of the call, its frames in the call).
static int lb_numbers(rf_tracker t, const char *who, const rf_yuv_frame *frames, const int *videos, int n, const rf_yuv_frame *out_frames,
                      const int32_t *out_frame_numbers, std::vector<long long> &num, std::vector<std::array<int, 3>> &seen) {
    rf_handle h = t->h;
    if (n > 0 && (!out_frames || !out_frame_numbers)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL out frames or frame numbers", who));
    const int L = t->lb_frames;
    int rc;
    num.assign(n, 0);
    auto ranges = yuv_ranges(frames, n);
    for (int i = 0; i < n; i++) {
        const int v = videos[i];
        auto it = std::find_if(seen.begin(), seen.end(), [v](const std::array<int, 3> &e) { return e[0] == v; });
        if (it == seen.end()) it = seen.insert(seen.end(), std::array<int, 3>{v, i, 0});
        const rf_tracker_s::LookbackVideo &lv = t->lbv[v];
        const rf_yuv_frame &f = frames[i], &g = frames[(*it)[1]];
        const bool v_first = f.uv_step == 2 && f.v < f.u;
        const bool same = lv.frames > 0 ? f.width == lv.w && f.height == lv.h && f.uv_step == lv.step && v_first == lv.v_first
                                        : f.width == g.width && f.height == g.height && f.uv_step == g.uv_step && v_first == (g.uv_step == 2 && g.v < g.u);
        if (!same)
            return fail(h, RF_ERR_INVALID_ARG, fmt("%s: frame %d: video %d changes its frame size or layout; drain or reset it first", who, i, v));
        if (++(*it)[2] > L) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: video %d appears more than L = %d times in one call", who, v, L));
        num[i] = lv.frames + (*it)[2] - 1;
        if ((rc = check_out_frame(h, who, out_frames[i], i, f.width, f.height, f.uv_step, v_first))) return rc;
        if (!same_frame(out_frames[i], f))
            for (auto &r : yuv_ranges(out_frames + i, 1)) ranges.push_back({r[0], r[1], (uintptr_t)(n + i)});
    }
    return check_disjoint(h, who, ranges);
}

// The emission of a look-back call or a drain into `slot`, on c's stream inside the chain: the swap `sw`, the regions of the emitted
// frames `em`, then (a drain: `drained` >= 0) that video's restart, the chain, and the redaction of the emitted frames `outs`.
// f20: out frame j is redacted as its video `out_videos[j]` displays it.
static void lb_emit(rf_tracker t, Ctx &c, rf_tracker_s::Slot &slot, const std::vector<LookbackSwapFrame> &sw,
                    const std::vector<std::array<long long, 3>> &em, const std::vector<rf_yuv_frame> &outs, const std::vector<int> &out_videos,
                    const RedactSpec &spec, int drained = -1) {
    lb_swap(sw, c.stream);
    lb_boxes(t, slot, em, c.stream);
    if (drained >= 0) restart(t, drained, 1, c.stream);     // then the video restarts as rf_tracker_reset restarts it
    CK(cudaEventRecord(t->chain, c.stream));
    if (outs.empty()) return;
    std::vector<int> oo;
    for (int v : out_videos) oo.push_back(t->orient[v]);
    redact_yuv_issue(t->h, c, outs.data(), oo.data(), (int)outs.size(), nullptr, slot.lb_boxes, slot.lb_counts, nullptr, nullptr, nullptr, spec,
                     lb_records(t));
}

// The look-back half of call `fc`, whose tracking was issued on c's stream into ring slot `ring` (it recorded the chain; this follows
// it on the same stream and records it again).  (a): the call's records, per_frame of them to a frame.  Each frame's log, f17's chains
// on a detect call (a follow frame has no births), then the swap -- after every kernel that reads an input frame, since an out frame
// may be its own input -- the regions and the redaction of the emitted frames.
static void lb_issue(rf_tracker t, Ctx &c, unsigned ring, const FrameCall &fc, int per_frame) {
    rf_handle h = t->h;
    const rf_yuv_frame *frames = fc.frames, *out_frames = fc.out_frames;
    const int *videos = fc.videos, n = fc.n;
    const std::vector<long long> &num = fc.num;
    rf_tracker_s::Slot &slot = t->slots[ring];
    const int L = t->lb_frames;
    LookbackArgs a{};
    a.dets = fc.dets;
    a.counts = fc.counts;
    a.tracks = slot.tracks;
    a.track_counts = slot.counts;
    a.motion = t->motion ? slot.motion : nullptr;
    a.max_faces = h->cfg.max_faces;
    a.max_tracks = t->cfg.max_tracks;
    a.slot_bytes = lb_slot_bytes(t);
    a.ring = 2 * L;
    a.L = L;
    for (int i0 = 0; i0 < n; i0 += LOOKBACK_TABLE) {
        LookbackLogTable lt{};
        lt.i0 = i0;
        lt.per_frame = per_frame;
        for (int i = i0; i < std::min(n, i0 + LOOKBACK_TABLE); i++, lt.n++) {
            lt.scale[lt.n] = fc.scales ? fc.scales[i] : 1.f;
            lt.slot[lt.n] = lb_log(t, t->lbv[videos[i]]) + (size_t)(num[i] % a.ring) * a.slot_bytes;
        }
        CK(launch_lookback_log(a, lt, c.stream));
    }
    if (t->lb_search && fc.source == FrameCall::DETECT) {
        a.search = t->lscfg.search;
        a.max_mad = t->lscfg.max_mad;
        a.steps = slot.lb_steps;
        a.lengths = slot.lb_lengths;
        lb_search(t, frames, videos, n, num, a, c.stream);
        t->lb_search_slot = (int)ring;
    }
    std::vector<LookbackSwapFrame> sw;
    std::vector<std::array<long long, 3>> em;
    std::vector<rf_yuv_frame> outs;
    std::vector<int> out_videos;
    for (int i = 0; i < n; i++) {
        const rf_tracker_s::LookbackVideo &lv = t->lbv[videos[i]];
        const bool emits = num[i] >= L;
        sw.push_back(lb_swap_frame(frames + i, emits ? out_frames + i : nullptr, lv.d + (size_t)(num[i] % L) * lv.frame_bytes));
        if (emits) {
            em.push_back({videos[i], num[i] - L, L});
            outs.push_back(out_frames[i]);
            out_videos.push_back(videos[i]);
        }
    }
    lb_emit(t, c, slot, sw, em, outs, out_videos, fc.spec);
}

int rf_detect_yuv_redact_lookback_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix, float thr,
                                         float nms, const rf_redact_style *style, const rf_yuv_frame *out_frames, int32_t *out_frame_numbers,
                                         const rf_track **dev_tracks, const int32_t **dev_track_counts, const rf_det **dev_dets,
                                         const int32_t **dev_counts, float *out_scales) {
    FrameCall c{.who = "rf_detect_yuv_redact_lookback_device", .call = Call::LOOKBACK, .source = FrameCall::DETECT, .sink = FrameCall::LOOKBACK,
                .h = h, .t = t, .frames = frames, .videos = videos, .n = n, .matrix = matrix, .thr = thr, .nms = nms, .style = style,
                .out_frames = out_frames, .out_frame_numbers = out_frame_numbers, .tracks = dev_tracks, .track_counts = dev_track_counts,
                .out_dets = dev_dets, .out_counts = dev_counts, .out_scales = out_scales};
    return frame_call(c);
}

// ---- f18 following look-back ----------------------------------------------------------------------------------------------------
int rf_tracker_set_lookback_follow(rf_tracker t, const rf_follow_config *cfg) {
    static const char *who = "rf_tracker_set_lookback_follow";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    if (!cfg) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL config", who));
    int rc = admit(t, who, Call::SET_LOOKBACK_FOLLOW);
    if (rc) return rc;
    rf_follow_config fc;
    if ((rc = follow_config(h, who, cfg, fc)) || (rc = follow_alloc(t, who, fc))) return rc;
    t->lb_follow = true;
    return RF_OK;
}

int rf_track_follow_redact_lookback_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_redact_style *style,
                                           const rf_yuv_frame *out_frames, int32_t *out_frame_numbers, const rf_track **dev_tracks,
                                           const int32_t **dev_track_counts) {
    FrameCall c{.who = "rf_track_follow_redact_lookback_device", .call = Call::LOOKBACK_FOLLOW, .source = FrameCall::FOLLOW,
                .sink = FrameCall::LOOKBACK, .t = t, .frames = frames, .videos = videos, .n = n, .style = style, .out_frames = out_frames,
                .out_frame_numbers = out_frame_numbers, .tracks = dev_tracks, .track_counts = dev_track_counts};
    return frame_call(c);
}

int rf_tracker_drain(rf_tracker t, int video, const rf_redact_style *style, const rf_yuv_frame *out_frames, int cap, int *n_out,
                     int32_t *out_frame_numbers) {
    static const char *who = "rf_tracker_drain";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    int rc = admit(t, who, Call::DRAIN);
    if (rc) return rc;
    if (video < 0 || video >= t->cfg.max_videos) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: video %d, must be in [0, %d)", who, video, t->cfg.max_videos));
    RedactSpec spec;
    if ((rc = redact_style(h, who, style, spec))) return rc;
    if (!n_out) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: n_out is NULL", who));
    const rf_tracker_s::LookbackVideo &lv = t->lbv[video];
    const long long frames = lv.frames;        // the restart below clears the count
    const int L = t->lb_frames, k = (int)std::min<long long>(L, frames);
    if (cap < k) return fail(h, RF_ERR_CAPACITY, fmt("%s: video %d has %d buffered frames, cap is %d", who, video, k, cap));
    if (k > 0 && (!out_frames || !out_frame_numbers)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL out frames or frame numbers", who));
    for (int j = 0; j < k; j++)
        if ((rc = check_out_frame(h, who, out_frames[j], j, lv.w, lv.h, lv.step, lv.v_first))) return rc;
    if ((rc = check_disjoint(h, who, yuv_ranges(out_frames, k)))) return rc;
    try {
        CK(cudaSetDevice(h->device));
        Ctx &c = h->ctx[0];
        rf_tracker_s::Slot &slot = t->slots[slot_begin(t, c.stream)];
        std::vector<LookbackSwapFrame> sw;
        std::vector<std::array<long long, 3>> em;
        for (int j = 0; j < k; j++) {
            const long long e = frames - k + j;
            sw.push_back(lb_swap_frame(nullptr, out_frames + j, lv.d + (size_t)(e % L) * lv.frame_bytes));
            em.push_back({video, e, frames - 1 - e});
        }
        lb_emit(t, c, slot, sw, em, std::vector<rf_yuv_frame>(out_frames, out_frames + k), std::vector<int>(k, video), spec, video);
        CK(cudaEventRecord(slot.free, c.stream));
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    for (int j = 0; j < k; j++) out_frame_numbers[j] = (int32_t)(frames - k + j);
    *n_out = k;
    return RF_OK;
}

// ---- f19 tiled detection ------------------------------------------------------------------------------------------------------------
// An option of any kind: each detect call then takes its records from rf_detect_yuv_tiled_device's tiles (issue_call).  The tiling is
// copied; levels NULL or nlevels 0 is the default pyramid.  What depends on the frame size is refused by the frame calls.
int rf_tracker_set_tiling(rf_tracker t, const rf_tiling *tiling) {
    static const char *who = "rf_tracker_set_tiling";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    int rc = admit(t, who, Call::SET_TILING);
    if (rc || (rc = tiling_supported(h, who))) return rc;
    if (any_oriented(t))      // f20, in either order: tiled detection has no oriented path
        return fail(h, RF_ERR_UNSUPPORTED, fmt("%s: a video of this tracker is shown in an orientation other than 1 (rf_tracker_set_orientation), "
                                               "and tiled detection has no oriented path", who));
    std::string err;
    if (!t->views.empty())    // f25, in either order: a rotated view is not tiled
        return fail(h, RF_ERR_UNSUPPORTED, fmt("%s: this tracker detects through rotated views (rf_tracker_set_views), which are not tiled", who));
    if ((rc = tiling_check(h->cfg.net_w, h->cfg.net_h, tiling, &err))) return fail(h, rc, fmt("%s: %s", who, err.c_str()));
    const bool dflt = !tiling || !tiling->levels || tiling->nlevels == 0;
    t->tile_levels.assign(dflt ? nullptr : tiling->levels, dflt ? nullptr : tiling->levels + tiling->nlevels);
    t->tiling = rf_tiling{t->tile_levels.empty() ? nullptr : t->tile_levels.data(), (int)t->tile_levels.size(), tiling ? tiling->overlap : 0};
    t->tiled = true;
    return RF_OK;
}

// ---- f25 rotated views ----------------------------------------------------------------------------------------------------------------
// An option of any kind: each detect call then takes its records from rf_detect_yuv_views_rotated_device's views (issue_call).  The
// views are copied; an oriented video's views rotate its displayed frames.
int rf_tracker_set_views(rf_tracker t, const rf_rotated_view *views, int nviews) {
    static const char *who = "rf_tracker_set_views";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    int rc = admit(t, who, Call::SET_VIEWS);
    if (rc || (rc = rotated_views_check(h, who, views, nviews))) return rc;
    if (t->tiled)             // in either order: a rotated view is not tiled
        return fail(h, RF_ERR_UNSUPPORTED, fmt("%s: a tiling tracker (rf_tracker_set_tiling) cannot detect through rotated views", who));
    t->views.assign(views, views + nviews);
    return RF_OK;
}

// ---- f20 oriented videos -----------------------------------------------------------------------------------------------------------
// Each video's display orientation, fixed from its first frame call to its next restart: a call reads and writes every frame as it is
// displayed (issue_call, redact_issue), while descriptors, out frames and every size or layout check stay in stored geometry.
int rf_tracker_set_orientation(rf_tracker t, int video, int orientation) {
    static const char *who = "rf_tracker_set_orientation";
    if (!t) return RF_ERR_INVALID_ARG;
    rf_handle h = t->h;
    const int V = t->cfg.max_videos;
    if (video < -1 || video >= V) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: video %d, must be -1 or in [0, %d)", who, video, V));
    if (lb_orientation_bits(orientation) < 0)
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: orientation %d, must be in 1..8 (EXIF)", who, orientation));
    const int v0 = video < 0 ? 0 : video, v1 = video < 0 ? V : video + 1;
    for (int v = v0; v < v1; v++)
        if (t->started[v])
            return fail(h, RF_ERR_INVALID_ARG,
                        fmt("%s: video %d has taken a frame call since its last create, reset, drain or finish", who, v));
    if (orientation != 1 && t->tiled)      // f25: a views tracker rotates the displayed frames
        return fail(h, RF_ERR_UNSUPPORTED, fmt("%s: a tiling tracker has no oriented detection (rf_tracker_set_tiling)", who));
    std::fill(t->orient.begin() + v0, t->orient.begin() + v1, orientation);
    return RF_OK;
}

// ---- the frame call path --------------------------------------------------------------------------------------------------------
// Everything a frame call refuses, in the order it has always refused it, before anything is launched: the handle and the tracker,
// check_track_args, the source's frames (a detect call's YUV frames, a follow call's planes) or an update's records, then the sink's
// arguments (align params, best-shot crops, the redaction style) and the frames' disjointness or lb_numbers.
static int check_call(FrameCall &c) {
    rf_tracker t = c.t;
    const char *who = c.who;
    if (c.source == FrameCall::DETECT) {
        if (!c.h) return RF_ERR_INVALID_ARG;
        if (!t || t->h != c.h)
            return fail(c.h, RF_ERR_INVALID_ARG,
                        fmt("%s: the tracker %sbelongs to another handle", who, c.sink == FrameCall::REDACT ? "" : "is NULL or "));
    } else if (!t) {
        return RF_ERR_INVALID_ARG;
    }
    rf_handle h = t->h;
    const int n = c.n;
    int rc = check_track_args(t, who, c.call, c.videos, n, c.source == FrameCall::RECORDS ? c.scales : nullptr);
    if (rc) return rc;
    for (int i = 0; i < n; i++) c.oriented |= t->orient[c.videos[i]] != 1;
    for (int i = 0; c.oriented && i < n; i++) c.orients.push_back(t->orient[c.videos[i]]);
    if (c.source == FrameCall::RECORDS && n > 0 && (!c.dets || !c.counts))
        return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL records or counts", who));
    if (c.source == FrameCall::DETECT) {
        const YuvFrames src = detect_source(c);
        if (t->tiled) rc = yuv_tiled_check(h, who, src, n, &t->tiling, c.layouts);
        else if (!t->views.empty()) rc = yuv_rotated_check(h, who, src, n, t->views.data(), (int)t->views.size());
        else rc = src.check(h, who, n);
        if (rc) return rc;
    }
    if (c.source == FrameCall::FOLLOW && (rc = check_frames(h, who, c.frames, n, RF_YUV_BT601))) return rc;
    if (c.sink == FrameCall::CROPS && (rc = check_align(h, who, c.align, n, c.crops, 0, c.a))) return rc;
    if (c.sink == FrameCall::BEST && n > 0 && !c.crops) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: dev_best_crops is NULL", who));
    if ((c.sink == FrameCall::REDACT || c.sink == FrameCall::LOOKBACK) && (rc = redact_style(h, who, c.style, c.spec))) return rc;
    if (c.sink == FrameCall::REDACT && (rc = check_disjoint(h, who, yuv_ranges(c.frames, n)))) return rc;
    if (c.sink == FrameCall::LOOKBACK && (rc = lb_numbers(t, who, c.frames, c.videos, n, c.out_frames, c.out_frame_numbers, c.num, c.seen)))
        return rc;
    return RF_OK;
}

// Issues a checked frame call of n > 0 frames.  The buffers of the call's look-back videos that have none are allocated before the
// forward, so that a refusal launches nothing.  Then, on the forward's context (a records or follow call: rf_last_stream's; a tiled
// or rotated detect: that call's home) inside the chain and in the call's ring slot: the update or the follow rounds, the template cut,
// the chain, the sink -- a look-back call's swap after every kernel that reads an input frame -- and, last, the slot's `free` and a
// tiled or rotated detect's detector ring slot `free`, recorded again after the last read of its records.
static int issue_call(FrameCall &c) {
    rf_tracker t = c.t;
    rf_handle h = t->h;
    const int n = c.n;
    int rc;
    try {
        CK(cudaSetDevice(h->device));
        for (const auto &e : c.seen) {     // LOOKBACK: (video, its first frame of the call, its frames in the call)
            rf_tracker_s::LookbackVideo &lv = t->lbv[e[0]];
            if (lv.frames > 0) continue;
            const rf_yuv_frame &f = c.frames[e[1]];
            if (!lb_alloc(t, lv, f))
                return fail(h, RF_ERR_CAPACITY,
                            fmt("%s: video %d: no device memory for %d frames of %dx%d", c.who, e[0], t->lb_frames, f.width, f.height));
            lv.w = f.width;
            lv.h = f.height;
            lv.step = f.uv_step;
            lv.v_first = f.uv_step == 2 && f.v < f.u;
        }
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    const YuvFrames src = detect_source(c);
    std::vector<float> scales(n);
    if (c.source == FrameCall::DETECT) {
        if (t->tiled) {      // f19: the tiled ring's records, in frame pixels
            if ((rc = yuv_tiled_issue(h, src, n, c.layouts, c.thr, c.nms, &c.dets, &c.counts, &c.detector_free))) return rc;
            std::fill(scales.begin(), scales.end(), 1.f);
        } else if (!t->views.empty()) {      // f25: the rotated ring's records, in (displayed) frame pixels
            if ((rc = yuv_rotated_issue(h, src, n, t->views.data(), (int)t->views.size(), c.thr, c.nms, &c.dets, &c.counts, &c.detector_free)))
                return rc;
            std::fill(scales.begin(), scales.end(), 1.f);
        } else if ((rc = yuv_device_impl(h, c.who, src, n, c.thr, c.nms, nullptr, nullptr, nullptr, &c.dets, &c.counts, scales.data()))) {
            return rc;
        }
        c.scales = scales.data();
        if (c.out_dets) *c.out_dets = c.dets;
        if (c.out_counts) *c.out_counts = c.counts;
        if (c.out_scales) std::copy(scales.begin(), scales.end(), c.out_scales);
    }
    try {
        Ctx &ctx = last_ctx(h);
        cudaStream_t s = ctx.stream;
        const unsigned ring = slot_begin(t, s);
        rf_tracker_s::Slot &slot = t->slots[ring];
        t->updated = true;
        for (int i = 0; i < n; i++) t->started[c.videos[i]] = 1;
        if (c.source == FrameCall::FOLLOW) {
            follow_rounds(t, ring, c.frames, c.videos, n, s);
            c.dets = slot.fregions;      // in id order, max_tracks to a frame, at scale 1
            c.counts = slot.fregion_counts;
            if (c.sink == FrameCall::BEST) best_follow_issue(t, slot, c, s);
        } else {
            update_issue(t, ring, c, s);
        }
        // the template cut reads the input frames: before a look-back call's swap
        if (c.source == FrameCall::DETECT && (t->kind == FOLLOW || t->lb_follow || t->best_follow)) follow_cut(t, c.frames, c.videos, n, slot, s);
        CK(cudaEventRecord(t->chain, s));
        const int per_frame = c.source == FrameCall::FOLLOW ? t->cfg.max_tracks : h->cfg.max_faces;
        if (c.sink == FrameCall::CROPS) {
            // the due faces are already in frame pixels: scale 1, as the tiled paths crop their merged records.  f20: displayed pixels
            // of an oriented frame, whose crops f9's oriented warp cuts upright
            std::vector<AlignImageT<YuvPlanes>> table(n);
            for (int i = 0; i < n; i++) {
                const int bits = src.bits(i);
                const bool tr = bits & LB_TRANSPOSE;
                table[i] = AlignImageT<YuvPlanes>{src.in_place(i), tr ? src.height(i) : src.width(i), tr ? src.width(i) : src.height(i), 1.f, bits};
            }
            c.a.n = n;
            c.a.crops = c.crops;
            c.a.mats = c.mats;
            PostBuffers view{};
            view.out_dets = slot.due;
            view.out_counts = slot.due_counts;
            view.max_faces = h->cfg.max_faces;
            CK(launch_align_faces(c.a, table.data(), view, h->num_sms, s, c.oriented));
        } else if (c.sink == FrameCall::REDACT) {
            // (a) the records, (b) the LOST tracks of the lists: f12's geometry, f14's styles and ownership
            redact_yuv_issue(h, ctx, c.frames, c.oriented ? c.orients.data() : nullptr, n, c.scales, c.dets, c.counts, t, slot.tracks,
                             slot.counts, c.spec, per_frame);
        } else if (c.sink == FrameCall::LOOKBACK) {
            lb_issue(t, ctx, ring, c, per_frame);
        }
        CK(cudaEventRecord(slot.free, s));
        if (c.detector_free) CK(cudaEventRecord(c.detector_free, s));     // the detector's slot is free once the call has read its records
        if (c.tracks) *c.tracks = slot.tracks;
        if (c.track_counts) *c.track_counts = slot.counts;
        if (c.best) *c.best = slot.best;
        if (c.best_counts) *c.best_counts = slot.best_counts;
    } catch (const CudaFail &f) { return fail_cuda(h, f); }
    for (int i = 0; c.sink == FrameCall::LOOKBACK && i < n; i++) {     // each video's count, and each frame's emitted number (-1: none)
        t->lbv[c.videos[i]].frames = std::max(t->lbv[c.videos[i]].frames, c.num[i] + 1);
        c.out_frame_numbers[i] = c.num[i] >= t->lb_frames ? (int32_t)(c.num[i] - t->lb_frames) : -1;
    }
    return RF_OK;
}

static int frame_call(FrameCall &c) {
    int rc = check_call(c);
    return rc || c.n == 0 ? rc : issue_call(c);
}
