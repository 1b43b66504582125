// RetinaFace.h -- C++ host side of the GPU path: the reference's detector class surface
// (retinaface/RetinaFace.h:15-70) over the C ABI of librf_b200.so (include/rf_b200.h).
//
// Source-compatible with the reference's callers (retinaface/main.cpp:15,43-44):
//     RetinaFace *rf = new RetinaFace(path, "net3");
//     rf->detect(img, 0.9);
//     rf->detectBatchImages(imgs, 0.9);
// Same constructor arguments (model directory, network name, nms threshold), same record types.
// Differences, all additive: the reference's detect functions return void and DROP their result
// (RetinaFace.cpp:665,726,747); here the result is kept and readable through lastFaces() /
// lastBatchFaces(); the network input size, which the reference bakes into prototxt line 7, is a
// constructor option; errors throw std::runtime_error instead of abort()/exit().
#ifndef RF_B200_HOST_RETINAFACE_H
#define RF_B200_HOST_RETINAFACE_H

#include <map>
#include <string>
#include <utility>
#include <vector>

#include "cv_compat.hpp"
#include "rf_b200.h"

using namespace std;   // the reference header does this (RetinaFace.h:12); callers rely on it
using cv::Mat;

struct anchor_box { float x1, y1, x2, y2; };               // RetinaFace.h:23-29
struct FacePts { float x[5]; float y[5]; };                // RetinaFace.h:31-35
struct FaceDetectInfo { float score; anchor_box rect; FacePts pts; };   // RetinaFace.h:37-42
static_assert(sizeof(FaceDetectInfo) == sizeof(rf_face), "FaceDetectInfo must match rf_face");

struct RetinaFaceOptions {
    int net_w = 320, net_h = 320;        // the shipped mnet-deconv-0517.prototxt:7 says 320x320
    int max_batch = 8;                   // trtretinafacenet.cpp:21
    int max_faces = 256;
    int precision = RF_PREC_FP16;
    int device = 0;
    int max_image_w = 4096, max_image_h = 3072;   // RetinaFace.cpp:325
    string model_file = "mnet-deconv-0517.caffemodel";   // RetinaFace.cpp:276
    string int8_table_file = "mnet-deconv-0517.table.int8";   // used when precision == RF_PREC_INT8 (trtnetbase.cpp:13)
    string prototxt_file;                // e.g. "mnet-deconv-0517.prototxt" (RetinaFace.cpp:276): parsed, checked, drives the weight
                                         // folding; with net_w = net_h = 0 it also sets the network size.  Empty: built-in graph
    int track_videos = 16;               // sequences of the tracker trackYUV creates on its first call
    bool track_motion = false;           // f13: that tracker follows the camera's motion (rf_tracker_set_motion, default config)
    int detect_every = 1;                // f16: > 1 makes that tracker a follow tracker (rf_tracker_set_follow, default config);
                                         // trackYUV / redactYUV then detect a video's frames whose number is divisible by it and
                                         // follow the faces on the others (rf_track_follow_device / rf_track_follow_redact_device).
                                         // f18: with RedactOptions::lookback on the first tracked call, a following look-back
                                         // tracker instead (rf_tracker_set_lookback_follow; follow frames through
                                         // rf_track_follow_redact_lookback_device)
    bool track_tiling = false;           // f19: every detect call of that tracker (trackYUV, trackYUVBest, redactYUV with or without
                                         // lookback and detect_every) detects through tiles (rf_tracker_set_tiling), as detectTiled:
    vector<float> track_tile_scales;     //   the levels (0: the letter-box); empty: the default pyramid
    bool track_tile_flip = false;        //   each level also mirrored (needs track_tile_scales)
    int track_tile_overlap = 0;          //   pixels neighbouring tiles share (0: 64)
    float track_any_angle_step = 0.f;    // f25: > 0 makes every detect call of that tracker detect through detectAnyAngleYUV's sweep of
                                         // rotated views at this step (rf_tracker_set_views), for tilted cameras; 0: off.  Not with
                                         // track_tiling (rf_tracker_set_views refuses a tiling tracker)
    string cache_file;                   // folded-model cache (the reference's "retina.cache", trtnetbase.cpp:205-243, but with a
                                         // staleness check).  Empty: none
};

// f5 face alignment (rf_detect_align_batch): one u8 BGR crop per kept face, warped from the original image so that the five
// landmarks land on a template (cv::warpAffine INTER_LINEAR bit for bit, on the GPU)
struct AlignOptions {
    int crop_w = 112, crop_h = 112;
    float template_xy[10] = {0};         // crop-pixel targets (x0, y0 .. x4, y4); all 0: the ArcFace 112x112 template
    int max_faces = 0;                   // crops per image, best score first; 0: every kept face
};

// f12 / f14 redaction (rf_detect_yuv_redact_device_style): the mosaic or blur written over every face
// f22 best shots for live cameras, the opt-in trackYUVBest overload's options (the first call creates the tracker with them).
struct BestOptions {
    int detect_every = 1;                // > 1: a following best-shot tracker (rf_tracker_set_best_follow); each video's frames whose
                                         // number is divisible by it are detected, the others followed
    bool live = false;                   // live shots (rf_tracker_set_best_live) with live_config (zeros: its defaults)
    rf_best_live_config live_config{};
    float min_quality = 0.f;
};

struct RedactOptions {
    int blocks = 8;                      // mosaic: cells across a region's longer side, 1..32 (1: one flat patch); the blur ignores it
    float margin = 0.25f;                // each side of a box grows by margin x its side, (0, 1]
    int style = RF_REDACT_MOSAIC;        // RF_REDACT_MOSAIC or RF_REDACT_BLUR
    int shape = RF_REDACT_RECT;          // RF_REDACT_RECT or RF_REDACT_ELLIPSE (the ellipse inscribed in the region)
    int detail = 0;                      // blur: 0 (4) or 1..64, a larger detail a smaller radius; 0 for the mosaic
    int lookback = 0;                    // f15, with videos: L (1..64) frames of delay, so that faces are covered before their first
                                         // detection (rf_detect_yuv_redact_lookback_device); 0: redact in place, undelayed
    bool lookback_search = false;        // f17, with lookback: follow each new face back through the buffered frames by template
                                         // search (rf_tracker_set_lookback_search, default R and max_mad) and cover its path too;
                                         // the first tracked call decides, and a later call asking for it on a tracker made
                                         // without it throws
};

class RetinaFace {
   public:
    RetinaFace(string &model, string network = "net3", float nms = 0.4, const RetinaFaceOptions &opt = RetinaFaceOptions());
    ~RetinaFace();
    RetinaFace(const RetinaFace &) = delete;
    RetinaFace &operator=(const RetinaFace &) = delete;

    void detectBatchImages(vector<cv::Mat> imgs, float threshold = 0.5);
    void detect(const Mat &img, float threshold = 0.5, float scales = 1.0);
    // compressed input: what main.cpp:18-26 hands to cv::imread.  The JPEG bitstreams are decoded on the GPU
    // (rf_detect_jpeg_batch); results and lastScale() as for detectBatchImages
    void detectEncoded(const vector<vector<unsigned char>> &jpegs, float threshold = 0.5);

    // results of the last call, in network-input pixels (RetinaFace.cpp:707); multiply by
    // lastScale() to map back to the caller's image (RetinaFace.cpp:587-591, 732-738)
    const vector<FaceDetectInfo> &lastFaces() const { return last_.empty() ? empty_ : last_[0]; }
    const vector<vector<FaceDetectInfo>> &lastBatchFaces() const { return last_; }
    float lastScale(size_t i = 0) const { return i < scales_.size() ? scales_[i] : 1.f; }
    // SURVEY.md 8f-2 -- what the reference leaves commented out (RetinaFace.cpp:730-746) or unused (`scales`, RetinaFace.h:70):
    // faces of ONE image in ORIGINAL IMAGE pixels (x * scale), optionally with multi-scale / horizontal-flip test-time
    // augmentation: `scales` are fractions (0, 1] of the network input the image is fitted into; with `flip` each scale also
    // runs mirrored.  All views run as one batch and are merged by NMS on the GPU (rf_detect_views).
    vector<FaceDetectInfo> detectInImage(const Mat &img, float threshold = 0.5, const vector<float> &scales = vector<float>(1, 1.0f),
                                         bool flip = false);
    // detect + align: afterwards lastBatchFaces() holds the faces in ORIGINAL IMAGE pixels (lastScale() is 1) and lastCrops()[i]
    // the crops of image i's first min(faces, max_faces) faces, crop_h x crop_w 8UC3 Mats
    void detectAndAlign(vector<cv::Mat> imgs, float threshold, const AlignOptions &align = AlignOptions());
    const vector<vector<Mat>> &lastCrops() const { return crops_; }
    // f6 video frames (rf_detect_yuv_batch): 8-bit YUV 4:2:0 frames as OpenCV keeps them, CV_8UC1 Mats of (h * 3 / 2) x w in
    // `layout` (YUV_NV12 .. YUV_YV12; semi-planar frames may have a row step, planar ones must be continuous), BT.601 as
    // cv::cvtColor(COLOR_YUV2BGR_<layout>).  Afterwards lastBatchFaces() holds the faces in FRAME pixels (lastScale() is 1) and,
    // with `align`, lastCrops() the crops as detectAndAlign leaves them.
    enum YuvLayout { YUV_NV12 = 0, YUV_NV21 = 1, YUV_I420 = 2, YUV_YV12 = 3 };
    void detectYUV(const vector<Mat> &frames, int layout, float threshold, const AlignOptions *align = nullptr);
    // f7 small faces in large images (rf_detect_tiled): each image resized to a pyramid of levels, every level cut into overlapping
    // network-sized tiles, merged across tiles and levels on the GPU.  `scales`: the levels (may exceed 1; 0 is the letter-box of
    // detectBatchImages), each also mirrored with `flip`; empty: the default pyramid 1, 1/2, 1/4, ... down to the letter-box, which
    // has no mirrored levels (`flip` with empty `scales` throws std::invalid_argument).
    // `overlap`: pixels neighbouring tiles share (0: 64).  Afterwards lastBatchFaces() holds the faces in ORIGINAL IMAGE pixels
    // (lastScale() is 1) and, with `align` (rf_detect_tiled_align), lastCrops() the crops as detectAndAlign leaves them.
    void detectTiled(const vector<Mat> &imgs, float threshold = 0.5, const vector<float> &scales = vector<float>(), bool flip = false,
                     int overlap = 0, const AlignOptions *align = nullptr);
    // f21 small faces in rotated and mirrored images (rf_detect_tiled_oriented): detectTiled on imgs[i] shown in EXIF orientation
    // orientations[i] (1..8), tiled as the displayed image without a rotated copy.  Afterwards lastBatchFaces() holds the faces in
    // DISPLAYED image pixels and, with `align`, lastCrops() the crops of the displayed image.
    void detectTiled(const vector<Mat> &imgs, const vector<int> &orientations, float threshold = 0.5, const vector<float> &scales = vector<float>(),
                     bool flip = false, int overlap = 0, const AlignOptions *align = nullptr);
    // f9 rotated and mirrored images (rf_detect_oriented_batch): imgs[i] as stored, shown in EXIF orientation orientations[i] (1..8,
    // what cv::imread applies; rf_jpeg_exif_orientation reads it from JPEG bytes).  Afterwards lastBatchFaces() holds the faces in
    // DISPLAYED image pixels (lastScale() is 1) and, with `align`, lastCrops() the crops of the displayed image.  No rotated copy is made.
    void detectOriented(const vector<Mat> &imgs, const vector<int> &orientations, float threshold = 0.5, const AlignOptions *align = nullptr);
    // f9 unknown orientation (rf_detect_views_oriented): the image in its four rotations (EXIF 1, 6, 3, 8) as one batch, merged on
    // the GPU; faces in STORED image pixels, landmarks on the subject's sides (an aligned crop of a sideways face comes out upright).
    vector<FaceDetectInfo> detectAnyOrientation(const Mat &img, float threshold = 0.5);
    // f23 faces at any in-plane angle (rf_detect_views_rotated): the image rotated counter-clockwise by 0, step_deg, 2 step_deg ... below
    // 360 (at most RF_MAX_VIEWS views, else std::invalid_argument), merged on the GPU; faces in image pixels, landmarks carrying each
    // face's roll.  With `align`, lastCrops()[0] holds the upright crops of the first min(faces, max_faces) faces (lastBatchFaces() and
    // lastCrops() hold the one image).
    vector<FaceDetectInfo> detectAnyAngle(const Mat &img, float threshold = 0.5, float step_deg = 30, const AlignOptions *align = nullptr);
    // f24 faces at any in-plane angle in video (rf_detect_yuv_views_rotated_device, BT.601): detectAnyAngle's sweep on DEVICE 4:2:0
    // frames (descriptors of device planes, e.g. NVDEC surfaces; at most max_batch), all frames in one call.  Blocking: afterwards
    // lastBatchFaces()[i] holds frame i's faces in FRAME pixels (lastScale() is 1).
    void detectAnyAngleYUV(const vector<rf_yuv_frame> &device_frames, float threshold = 0.5, float step_deg = 30);
    // The views detectAnyAngle and detectAnyAngleYUV sweep: (0, 1), (step_deg, 1), (2 step_deg, 1) ... below 360 degrees; a step_deg
    // that is not positive, or that makes more than RF_MAX_VIEWS views, throws std::invalid_argument naming `who`.
    static vector<rf_rotated_view> angleSweep(const char *who, float step_deg);
    // f10 tracking (rf_detect_yuv_track_device): DEVICE 4:2:0 frames (descriptors of device planes, e.g. NVDEC surfaces; at most
    // max_batch per call), frame i of video videos[i] in [0, track_videos), detected and associated with the tracks of earlier frames
    // on the GPU.  Asynchronous on rf_last_stream(handle()).  Afterwards lastTracks() holds the device track lists; with `align`, the
    // crops of the tracks confirmed on each frame (new identities) land in dev_crops [n][A] u8 BGR at each such track's crop_slot.
    struct DeviceTracks {
        const rf_track *tracks = nullptr;   // device [n][max_tracks], each frame's live tracks sorted by id
        const int32_t *counts = nullptr;    // device [n]
        int n = 0, max_tracks = 0;
    };
    void trackYUV(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, float threshold = 0.5, const AlignOptions *align = nullptr,
                  void *dev_crops = nullptr);
    const DeviceTracks &lastTracks() const { return tracks_; }
    void resetTracks(int video = -1);
    // f20 oriented video (rf_tracker_set_orientation): video (-1: every video) is shown in EXIF orientation 1..8 -- portrait phone
    // video stored as landscape surfaces -- and trackYUV, trackYUVBest and redactYUV read and write its frames as displayed, with
    // tracks in displayed pixels.  Applied when this RetinaFace's tracker is created, or at once when it exists; before the video's
    // first tracked frame since creation or resetTracks.
    void setVideoOrientation(int video, int orientation);
    // f11 best shots (rf_detect_yuv_track_best_device): trackYUV on a best-shot tracker (created on the first call with min_quality;
    // one RetinaFace keeps one kind of tracker) that keeps the best 112x112 u8 crop of every track on the GPU.  Afterwards lastTracks()
    // holds the track lists and lastBestShots() the shots emitted on each frame -- one per ever-confirmed track that ended there, in
    // id order -- whose crops land in dev_best_crops [n][max_tracks] u8 BGR.  finishVideo emits the shots of a video's live tracks
    // into dev_best_crops [max_tracks] (lastBestShots() then has n = 1) and restarts the video.
    struct DeviceBestShots {
        const rf_best_shot *shots = nullptr;  // device [n][max_tracks]
        const int32_t *counts = nullptr;      // device [n]
        int n = 0, max_tracks = 0;
    };
    void trackYUVBest(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, void *dev_best_crops, float threshold = 0.5,
                      float min_quality = 0.f);
    // f22: the same with BestOptions: live shots (reason RF_BEST_LIVE) while tracks live, and a detection interval.  With
    // detect_every > 1 one call takes detect frames only or follow frames only (its videos' frame numbers agree modulo detect_every, as
    // when each call takes the next frame of every camera); a call mixing both is std::invalid_argument before anything is issued.
    // lastBestShots() and lastTracks() hold the call's records either way (a follow call's shots: the tracks removed on it), and
    // lastFollow() the follow records of the last follow call.
    void trackYUVBest(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, void *dev_best_crops, float threshold,
                      const BestOptions &opt);
    const DeviceBestShots &lastBestShots() const { return best_; }
    // f13 camera motion (options track_motion): the device rf_motion of each frame of the last trackYUV / trackYUVBest / tracked
    // redactYUV call -- the estimated similarity from the video's previous frame, applied to its tracks.
    struct DeviceMotion {
        const rf_motion *motion = nullptr;  // device [n]
        int n = 0;
    };
    const DeviceMotion &lastMotion() const { return motion_; }
    // f16 (options detect_every > 1): a call whose frames are of both kinds is issued as detect and follow calls, each video's frames
    // in order (the p-th run of one kind of every video after the (p - 1)-th, detect first); lastTracks() and lastMotion() then hold
    // the last of them.  lastFollow() holds the rf_follow records of the last follow call (nullptr before one).
    struct DeviceFollow {
        const rf_follow *follow = nullptr;  // device [n][max_tracks], each frame's in its list order
        int n = 0, max_tracks = 0;
    };
    const DeviceFollow &lastFollow() const { return follow_; }
    void finishVideo(int video, void *dev_best_crops);
    // f12 / f14 redaction (rf_detect_yuv_redact_device_style): detect on DEVICE 4:2:0 frames and mosaic (or blur) every detected face in place, on the
    // GPU; asynchronous on rf_last_stream(handle()).  With `videos` (one per frame, in [0, track_videos)) the frames are also tracked on
    // this RetinaFace's plain tracker (trackYUV's), lastTracks() holds the lists, and the predicted box of every LOST track -- a face the
    // detector missed on this frame -- is redacted too.
    // f15: with opt.lookback = L the tracker (created by the first tracked call) keeps each video's last L frames on the GPU, and
    // frame i writes frame num_i - L of its video, also covered where the faces first detected in the next L frames already were,
    // into out_frames[i] (nullptr: device_frames[i] itself); lastFrameNumbers()[i] is num_i - L, or -1 while the video fills.
    // drainVideo writes the video's remaining buffered frames into out_frames[0..) and restarts it (and its detect_every numbering);
    // it returns their numbers.  f18: lookback with options detect_every > 1 splits the call as f16 does and emits every frame, key
    // frame or not, L frames late; with L >= detect_every - 1 a face is also covered on the follow frames before its first detection.
    void redactYUV(const vector<rf_yuv_frame> &device_frames, const vector<int> *videos = nullptr, float threshold = 0.5,
                   const RedactOptions &opt = RedactOptions(), const vector<rf_yuv_frame> *out_frames = nullptr);
    const vector<int32_t> &lastFrameNumbers() const { return frame_numbers_; }
    vector<int32_t> drainVideo(int video, const vector<rf_yuv_frame> &out_frames, const RedactOptions &opt = RedactOptions());
    rf_handle handle() const { return h_; }
    // the reference's visualisation (RetinaFace.cpp:730-741): red box outline (thickness 2), green landmark dots, on a clone
    static Mat draw(const Mat &img, const vector<FaceDetectInfo> &faces);
    int netWidth() const { return opt_.net_w; }
    int netHeight() const { return opt_.net_h; }

   private:
    // faces (and, with crops, the u8 crops of the first min(count, per) faces) of images [start, start + n) of the last call
    void keepResults(size_t start, int n, const unsigned char *crops, int per, int cw, int ch);
    // both detectTiled overloads; orientations NULL: upright images (rf_detect_tiled / rf_detect_tiled_align)
    void tiled(const vector<Mat> &imgs, const vector<int> *orientations, float threshold, const vector<float> &scales, bool flip, int overlap,
               const AlignOptions *align);
    void trackerCreated(bool follow = true);   // motion (and, with follow, f16's following) on a new tracker, as the options say
    void noteMotion(int n);             // lastMotion() after a tracked call of n frames
    rf_tracker makeTracker(int lookback, bool lookback_search = false);   // trackYUV's / redactYUV's tracker, as the options say
    // f16: the call's frames as (detect?, frame indices) sub-calls in issue order; advances each video's frame number
    vector<std::pair<bool, vector<int>>> intervalCalls(const vector<int> &videos);
    // out_frames (f18): the following look-back call, its emitted numbers into frame_numbers
    void followCall(const vector<rf_yuv_frame> &frames, const vector<int> &videos, const rf_redact_style *style,
                    const vector<rf_yuv_frame> *out_frames = nullptr, int32_t *frame_numbers = nullptr);
    void lookbackCall(const vector<rf_yuv_frame> &frames, const vector<int> &videos, float threshold, const rf_redact_style &st,
                      const vector<rf_yuv_frame> &out_frames, int32_t *frame_numbers);
    void trackDetect(const vector<rf_yuv_frame> &frames, const vector<int> &videos, float threshold, const AlignOptions *align, void *dev_crops);
    rf_handle h_ = nullptr;
    rf_tracker tracker_ = nullptr;
    bool tracker_search_ = false;        // f17: tracker_ searches its look-back buffer
    bool tracker_lookback_follow_ = false;   // f18: tracker_ is a following look-back tracker
    bool best_tracker_ = false;
    bool best_follow_ = false;           // f22: tracker_ is a following best-shot tracker
    DeviceTracks tracks_;
    DeviceBestShots best_;
    DeviceMotion motion_;
    DeviceFollow follow_;
    std::map<int, long long> frame_no_;
    vector<std::pair<int, int>> orientations_;   // f20: setVideoOrientation's (video, orientation), replayed on a new tracker
    vector<int32_t> frame_numbers_;
    RetinaFaceOptions opt_;
    string network;
    float nms_threshold;
    vector<vector<FaceDetectInfo>> last_;
    vector<FaceDetectInfo> empty_;
    vector<float> scales_;
    vector<vector<Mat>> crops_;
    vector<rf_face> out_faces_;
    vector<int> out_counts_;
};

#endif
