// RetinaFace.cpp -- see RetinaFace.h.  Everything that computes lives behind the C ABI.
#include "RetinaFace.h"

#include <cmath>
#include <cstring>

#include <stdexcept>

RetinaFace::RetinaFace(string &model, string network_, float nms, const RetinaFaceOptions &opt)
    : opt_(opt), network(network_), nms_threshold(nms) {
    // RetinaFace.cpp:211-271: the network-name switch lives behind the C ABI (rf_network_config / rf_config.network); names the
    // reference itself has no anchor configuration for (fmc != 3) or whose models do not ship (net3a) are refused there
    int levels = 0, nratios = 0;
    if (rf_network_config(network.c_str(), &levels, nullptr, nullptr, nullptr, &nratios) != RF_OK)
        throw std::runtime_error("network setting error " + network + ": " + rf_last_error(nullptr));
    const string path = model + "/" + opt_.model_file;
    rf_config cfg{};
    const string table = model + "/" + opt_.int8_table_file;
    const string proto = opt_.prototxt_file.empty() ? string() : model + "/" + opt_.prototxt_file;
    cfg.network = network.c_str();
    cfg.prototxt_path = proto.empty() ? nullptr : proto.c_str();     // buildTrtContext(prototxt, caffemodel), RetinaFace.cpp:276
    cfg.cache_path = opt_.cache_file.empty() ? nullptr : opt_.cache_file.c_str();
    cfg.caffemodel_path = path.c_str();
    cfg.int8_table_path = opt_.precision == RF_PREC_INT8 ? table.c_str() : nullptr;
    cfg.precision = opt_.precision;
    cfg.net_w = opt_.net_w;
    cfg.net_h = opt_.net_h;
    cfg.max_batch = opt_.max_batch;
    cfg.max_faces = opt_.max_faces;
    cfg.device = opt_.device;
    cfg.max_image_w = opt_.max_image_w;
    cfg.max_image_h = opt_.max_image_h;
    int rc = rf_create(&cfg, &h_);
    if (rc != RF_OK) throw std::runtime_error(string("rf_create: ") + rf_status_string(rc) + ": " + rf_last_error(nullptr));
    rf_get_net_size(h_, &opt_.net_w, &opt_.net_h, nullptr, &opt_.max_faces);     // (0 x 0: the prototxt's input size)
    out_faces_.resize((size_t)opt_.max_batch * opt_.max_faces);
    out_counts_.resize(opt_.max_batch);
}

RetinaFace::~RetinaFace() {
    rf_tracker_destroy(tracker_);   // before its handle
    rf_destroy(h_);
}

void RetinaFace::detect(const Mat &img, float threshold, float /*scales*/) {
    if (img.empty()) {   // RetinaFace.cpp:578-580
        last_.clear();
        return;
    }
    vector<cv::Mat> one(1, img);
    detectBatchImages(one, threshold);
}

void RetinaFace::detectEncoded(const vector<vector<unsigned char>> &jpegs, float threshold) {
    last_.assign(jpegs.size(), vector<FaceDetectInfo>());
    scales_.assign(jpegs.size(), 1.f);
    const size_t mb = (size_t)opt_.max_batch;
    for (size_t start = 0; start < jpegs.size(); start += mb) {
        const int n = (int)std::min(mb, jpegs.size() - start);
        vector<const uint8_t *> ptrs(n);
        vector<size_t> lens(n);
        vector<int> ws(n), hs(n);
        for (int i = 0; i < n; i++) { ptrs[i] = jpegs[start + i].data(); lens[i] = jpegs[start + i].size(); }
        int rc = rf_detect_jpeg_batch(h_, ptrs.data(), lens.data(), n, threshold, nms_threshold, out_faces_.data(), out_counts_.data(), nullptr,
                                      ws.data(), hs.data());
        if (rc != RF_OK) throw std::runtime_error(string("rf_detect_jpeg_batch: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        for (int i = 0; i < n; i++) {
            float sw = 1.0f * ws[i] / opt_.net_w, sh = 1.0f * hs[i] / opt_.net_h;   // RetinaFace.cpp:587-591
            float sc = sw > sh ? sw : sh;
            scales_[start + i] = sc > 1.0f ? sc : 1.0f;
            const FaceDetectInfo *f = reinterpret_cast<const FaceDetectInfo *>(out_faces_.data() + (size_t)i * opt_.max_faces);
            last_[start + i].assign(f, f + out_counts_[i]);
        }
    }
}

void RetinaFace::detectBatchImages(vector<cv::Mat> imgs, float threshold) {
    last_.assign(imgs.size(), vector<FaceDetectInfo>());
    scales_.assign(imgs.size(), 1.f);
    const size_t mb = (size_t)opt_.max_batch;
    for (size_t start = 0; start < imgs.size(); start += mb) {   // the reference asserts n <= maxBatchSize; chunk instead
        const int n = (int)std::min(mb, imgs.size() - start);
        vector<const uint8_t *> ptrs(n);
        vector<int> ws(n), hs(n), strides(n);
        for (int i = 0; i < n; i++) {
            const cv::Mat &m = imgs[start + i];
            if (m.empty()) throw std::runtime_error("detectBatchImages: empty image");
            ptrs[i] = m.data; ws[i] = m.cols; hs[i] = m.rows; strides[i] = (int)m.step;
            float sw = 1.0f * m.cols / opt_.net_w, sh = 1.0f * m.rows / opt_.net_h;   // RetinaFace.cpp:587-591
            float sc = sw > sh ? sw : sh;
            scales_[start + i] = sc > 1.0f ? sc : 1.0f;
        }
        int rc = rf_detect_batch(h_, ptrs.data(), ws.data(), hs.data(), strides.data(), n, threshold, nms_threshold,
                                 out_faces_.data(), out_counts_.data(), nullptr);
        if (rc != RF_OK) throw std::runtime_error(string("rf_detect_batch: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        for (int i = 0; i < n; i++) {
            const FaceDetectInfo *f = reinterpret_cast<const FaceDetectInfo *>(out_faces_.data() + (size_t)i * opt_.max_faces);
            last_[start + i].assign(f, f + out_counts_[i]);
        }
    }
}

// rf_align_params of u8 BGR crops, and where they land: `per` crop slots per image of cw x ch
static rf_align_params crop_params(const AlignOptions &align, int max_faces, int *per, int *cw, int *ch) {
    rf_align_params p{};
    p.crop_w = align.crop_w;
    p.crop_h = align.crop_h;
    for (int k = 0; k < 10; k++) p.template_xy[k] = align.template_xy[k];
    p.max_faces = align.max_faces;
    p.format = RF_CROP_BGR_U8;
    *per = align.max_faces > 0 ? align.max_faces : max_faces;
    const bool dflt = align.crop_w == 0 && align.crop_h == 0;    // rf_align_params: 0 x 0 -> 112 x 112
    *cw = dflt ? 112 : align.crop_w;
    *ch = dflt ? 112 : align.crop_h;
    return p;
}

void RetinaFace::detectAndAlign(vector<cv::Mat> imgs, float threshold, const AlignOptions &align) {
    last_.assign(imgs.size(), vector<FaceDetectInfo>());
    scales_.assign(imgs.size(), 1.f);
    crops_.assign(imgs.size(), vector<Mat>());
    int per = 0, cw = 0, ch = 0;
    const rf_align_params p = crop_params(align, opt_.max_faces, &per, &cw, &ch);
    const size_t crop_bytes = (size_t)cw * ch * 3;
    const size_t mb = (size_t)opt_.max_batch;
    vector<unsigned char> crops(mb * per * crop_bytes);
    for (size_t start = 0; start < imgs.size(); start += mb) {
        const int n = (int)std::min(mb, imgs.size() - start);
        vector<const uint8_t *> ptrs(n);
        vector<int> ws(n), hs(n), strides(n);
        for (int i = 0; i < n; i++) {
            const cv::Mat &m = imgs[start + i];
            if (m.empty()) throw std::runtime_error("detectAndAlign: empty image");
            ptrs[i] = m.data; ws[i] = m.cols; hs[i] = m.rows; strides[i] = (int)m.step;
        }
        int rc = rf_detect_align_batch(h_, ptrs.data(), ws.data(), hs.data(), strides.data(), n, threshold, nms_threshold, &p,
                                       out_faces_.data(), out_counts_.data(), crops.data(), nullptr);
        if (rc != RF_OK) throw std::runtime_error(string("rf_detect_align_batch: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        keepResults(start, n, crops.data(), per, cw, ch);
    }
}

void RetinaFace::keepResults(size_t start, int n, const unsigned char *crops, int per, int cw, int ch) {
    const size_t crop_bytes = (size_t)cw * ch * 3;
    for (int i = 0; i < n; i++) {
        const FaceDetectInfo *f = reinterpret_cast<const FaceDetectInfo *>(out_faces_.data() + (size_t)i * opt_.max_faces);
        last_[start + i].assign(f, f + out_counts_[i]);
        for (int j = 0; crops && j < std::min(out_counts_[i], per); j++) {
            Mat c(ch, cw, CV_8UC3);
            const unsigned char *src = crops + ((size_t)i * per + j) * crop_bytes;
            for (int y = 0; y < ch; y++) std::memcpy(c.data + (size_t)y * c.step, src + (size_t)y * cw * 3, (size_t)cw * 3);
            crops_[start + i].push_back(c);
        }
    }
}

void RetinaFace::detectYUV(const vector<Mat> &frames, int layout, float threshold, const AlignOptions *align) {
    if (layout < YUV_NV12 || layout > YUV_YV12) throw std::runtime_error("detectYUV: unknown layout");
    last_.assign(frames.size(), vector<FaceDetectInfo>());
    scales_.assign(frames.size(), 1.f);
    crops_.assign(frames.size(), vector<Mat>());
    int per = 0, cw = 0, ch = 0;
    const rf_align_params p = align ? crop_params(*align, opt_.max_faces, &per, &cw, &ch) : rf_align_params{};
    const size_t mb = (size_t)opt_.max_batch;
    vector<unsigned char> crops(align ? mb * per * cw * ch * 3 : 0);
    for (size_t start = 0; start < frames.size(); start += mb) {
        const int n = (int)std::min(mb, frames.size() - start);
        vector<rf_yuv_frame> fr(n);
        for (int i = 0; i < n; i++) {
            // OpenCV's single buffer: the luma rows, then the chroma -- interleaved rows of the same step (NV12 / NV21), or the
            // U and V planes of w / 2 x h / 2 packed one after the other (I420: U first, YV12: V first)
            const cv::Mat &m = frames[start + i];
            if (m.empty() || m.rows % 3 || m.cols % 2) throw std::runtime_error("detectYUV: frames must be non-empty (h * 3 / 2) x w with even h and w");
            const int w = m.cols, hh = m.rows / 3 * 2;
            const unsigned char *c = m.data + m.step * hh;
            rf_yuv_frame &f = fr[i];
            f.y = m.data; f.y_pitch = (int)m.step; f.width = w; f.height = hh;
            if (layout == YUV_NV12 || layout == YUV_NV21) {
                f.uv_step = 2; f.uv_pitch = (int)m.step;
                f.u = c + (layout == YUV_NV21); f.v = c + (layout == YUV_NV12);
            } else {
                if (m.step != (size_t)w) throw std::runtime_error("detectYUV: planar (I420 / YV12) frames must be continuous");
                const unsigned char *q = c + (size_t)(w / 2) * (hh / 2);
                f.uv_step = 1; f.uv_pitch = w / 2;
                f.u = layout == YUV_I420 ? c : q; f.v = layout == YUV_I420 ? q : c;
            }
        }
        int rc = rf_detect_yuv_batch(h_, fr.data(), n, RF_YUV_BT601, threshold, nms_threshold, align ? &p : nullptr, out_faces_.data(), out_counts_.data(),
                                     nullptr, align ? crops.data() : nullptr, nullptr);
        if (rc != RF_OK) throw std::runtime_error(string("rf_detect_yuv_batch: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        keepResults(start, n, align ? crops.data() : nullptr, per, cw, ch);
    }
}

void RetinaFace::detectTiled(const vector<Mat> &imgs, float threshold, const vector<float> &scales, bool flip, int overlap,
                             const AlignOptions *align) {
    tiled(imgs, nullptr, threshold, scales, flip, overlap, align);
}

void RetinaFace::detectTiled(const vector<Mat> &imgs, const vector<int> &orientations, float threshold, const vector<float> &scales, bool flip,
                             int overlap, const AlignOptions *align) {
    if (orientations.size() != imgs.size()) throw std::invalid_argument("detectTiled: one orientation per image");
    tiled(imgs, &orientations, threshold, scales, flip, overlap, align);
}

void RetinaFace::tiled(const vector<Mat> &imgs, const vector<int> *orientations, float threshold, const vector<float> &scales, bool flip,
                       int overlap, const AlignOptions *align) {
    if (flip && scales.empty()) throw std::invalid_argument("detectTiled: flip mirrors the given scales; the default pyramid has none");
    last_.assign(imgs.size(), vector<FaceDetectInfo>());
    scales_.assign(imgs.size(), 1.f);
    crops_.assign(imgs.size(), vector<Mat>());
    vector<rf_tile_level> levels;
    for (float s : scales) {
        levels.push_back(rf_tile_level{s, 0});
        if (flip) levels.push_back(rf_tile_level{s, 1});
    }
    const rf_tiling t{levels.empty() ? nullptr : levels.data(), (int)levels.size(), overlap};
    int per = 0, cw = 0, ch = 0;
    const rf_align_params p = align ? crop_params(*align, opt_.max_faces, &per, &cw, &ch) : rf_align_params{};
    const size_t mb = (size_t)opt_.max_batch;
    vector<unsigned char> crops(align ? mb * per * cw * ch * 3 : 0);
    for (size_t start = 0; start < imgs.size(); start += mb) {
        const int n = (int)std::min(mb, imgs.size() - start);
        vector<const uint8_t *> ptrs(n);
        vector<int> ws(n), hs(n), strides(n);
        for (int i = 0; i < n; i++) {
            const cv::Mat &m = imgs[start + i];
            if (m.empty()) throw std::runtime_error("detectTiled: empty image");
            ptrs[i] = m.data; ws[i] = m.cols; hs[i] = m.rows; strides[i] = (int)m.step;
        }
        const char *who = orientations ? "rf_detect_tiled_oriented: " : align ? "rf_detect_tiled_align: " : "rf_detect_tiled: ";
        int rc = orientations ? rf_detect_tiled_oriented(h_, ptrs.data(), ws.data(), hs.data(), strides.data(), orientations->data() + start, n, &t,
                                                         threshold, nms_threshold, align ? &p : nullptr, out_faces_.data(), out_counts_.data(),
                                                         nullptr, align ? crops.data() : nullptr, nullptr)
               : align ? rf_detect_tiled_align(h_, ptrs.data(), ws.data(), hs.data(), strides.data(), n, &t, threshold, nms_threshold, &p,
                                               out_faces_.data(), out_counts_.data(), nullptr, crops.data(), nullptr)
                       : rf_detect_tiled(h_, ptrs.data(), ws.data(), hs.data(), strides.data(), n, &t, threshold, nms_threshold, out_faces_.data(),
                                         out_counts_.data(), nullptr);
        if (rc != RF_OK) throw std::runtime_error(string(who) + rf_status_string(rc) + ": " + rf_last_error(h_));
        keepResults(start, n, align ? crops.data() : nullptr, per, cw, ch);
    }
}

vector<FaceDetectInfo> RetinaFace::detectInImage(const Mat &img, float threshold, const vector<float> &scales, bool flip) {
    vector<FaceDetectInfo> out;
    if (img.empty()) return out;
    vector<rf_view> views;
    for (float s : scales) {
        views.push_back(rf_view{s, 0});
        if (flip) views.push_back(rf_view{s, 1});
    }
    int count = 0;
    int rc = rf_detect_views(h_, img.data, img.cols, img.rows, (int)img.step, views.data(), (int)views.size(), threshold, nms_threshold,
                             out_faces_.data(), &count, nullptr, nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_views: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    const FaceDetectInfo *f = reinterpret_cast<const FaceDetectInfo *>(out_faces_.data());
    out.assign(f, f + count);
    return out;
}

void RetinaFace::detectOriented(const vector<Mat> &imgs, const vector<int> &orientations, float threshold, const AlignOptions *align) {
    if (orientations.size() != imgs.size()) throw std::invalid_argument("detectOriented: one orientation per image");
    last_.assign(imgs.size(), vector<FaceDetectInfo>());
    scales_.assign(imgs.size(), 1.f);
    crops_.assign(imgs.size(), vector<Mat>());
    int per = 0, cw = 0, ch = 0;
    const rf_align_params p = align ? crop_params(*align, opt_.max_faces, &per, &cw, &ch) : rf_align_params{};
    const size_t mb = (size_t)opt_.max_batch;
    vector<unsigned char> crops(align ? mb * per * cw * ch * 3 : 0);
    for (size_t start = 0; start < imgs.size(); start += mb) {
        const int n = (int)std::min(mb, imgs.size() - start);
        vector<const uint8_t *> ptrs(n);
        vector<int> ws(n), hs(n), strides(n);
        for (int i = 0; i < n; i++) {
            const cv::Mat &m = imgs[start + i];
            if (m.empty()) throw std::runtime_error("detectOriented: empty image");
            ptrs[i] = m.data; ws[i] = m.cols; hs[i] = m.rows; strides[i] = (int)m.step;
        }
        int rc = rf_detect_oriented_batch(h_, ptrs.data(), ws.data(), hs.data(), strides.data(), orientations.data() + start, n, threshold,
                                          nms_threshold, align ? &p : nullptr, out_faces_.data(), out_counts_.data(), nullptr,
                                          align ? crops.data() : nullptr, nullptr);
        if (rc != RF_OK) throw std::runtime_error(string("rf_detect_oriented_batch: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        keepResults(start, n, align ? crops.data() : nullptr, per, cw, ch);
    }
}

vector<FaceDetectInfo> RetinaFace::detectAnyOrientation(const Mat &img, float threshold) {
    vector<FaceDetectInfo> out;
    if (img.empty()) return out;
    const rf_oriented_view views[4] = {{1.f, 1}, {1.f, 6}, {1.f, 3}, {1.f, 8}};
    int count = 0;
    int rc = rf_detect_views_oriented(h_, img.data, img.cols, img.rows, (int)img.step, views, 4, threshold, nms_threshold, out_faces_.data(),
                                      &count, nullptr, nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_views_oriented: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    const FaceDetectInfo *f = reinterpret_cast<const FaceDetectInfo *>(out_faces_.data());
    out.assign(f, f + count);
    return out;
}

vector<rf_rotated_view> RetinaFace::angleSweep(const char *who, float step_deg) {
    if (!(step_deg > 0.f)) throw std::invalid_argument(string(who) + ": step_deg must be positive");
    vector<rf_rotated_view> views;
    for (int k = 0; k * step_deg < 360.f; k++) {
        if (views.size() == RF_MAX_VIEWS) throw std::invalid_argument(string(who) + ": more than RF_MAX_VIEWS views");
        views.push_back(rf_rotated_view{k * step_deg, 1.f});
    }
    return views;
}

vector<FaceDetectInfo> RetinaFace::detectAnyAngle(const Mat &img, float threshold, float step_deg, const AlignOptions *align) {
    const vector<rf_rotated_view> views = angleSweep("detectAnyAngle", step_deg);
    last_.assign(1, vector<FaceDetectInfo>());
    scales_.assign(1, 1.f);
    crops_.assign(1, vector<Mat>());
    if (img.empty()) return last_[0];
    int per = 0, cw = 0, ch = 0;
    const rf_align_params p = align ? crop_params(*align, opt_.max_faces, &per, &cw, &ch) : rf_align_params{};
    vector<unsigned char> crops(align ? (size_t)per * cw * ch * 3 : 0);
    int count = 0;
    int rc = rf_detect_views_rotated(h_, img.data, img.cols, img.rows, (int)img.step, views.data(), (int)views.size(), threshold, nms_threshold,
                                     align ? &p : nullptr, out_faces_.data(), &count, nullptr, nullptr, nullptr, align ? crops.data() : nullptr,
                                     nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_views_rotated: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    out_counts_[0] = count;
    keepResults(0, 1, align ? crops.data() : nullptr, per, cw, ch);
    return last_[0];
}

void RetinaFace::detectAnyAngleYUV(const vector<rf_yuv_frame> &device_frames, float threshold, float step_deg) {
    const vector<rf_rotated_view> views = angleSweep("detectAnyAngleYUV", step_deg);
    const int n = (int)device_frames.size();
    if (n > opt_.max_batch) throw std::invalid_argument("detectAnyAngleYUV: at most max_batch frames per call");
    last_.assign(n, vector<FaceDetectInfo>());
    scales_.assign(n, 1.f);
    crops_.assign(n, vector<Mat>());
    if (n == 0) return;
    const rf_det *dets = nullptr;
    const int32_t *counts = nullptr;
    int rc = rf_detect_yuv_views_rotated_device(h_, device_frames.data(), n, RF_YUV_BT601, views.data(), (int)views.size(), threshold,
                                                nms_threshold, nullptr, nullptr, nullptr, &dets, &counts, nullptr, nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_yuv_views_rotated_device: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    rc = rf_fetch_dets(h_, dets, counts, n, out_faces_.data(), out_counts_.data(), nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_fetch_dets: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    keepResults(0, n, nullptr, 0, 0, 0);
}

void RetinaFace::trackYUV(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, float threshold, const AlignOptions *align,
                          void *dev_crops) {
    if (videos.size() != device_frames.size()) throw std::invalid_argument("trackYUV: one video index per frame");
    if (device_frames.size() > (size_t)opt_.max_batch) throw std::invalid_argument("trackYUV: at most max_batch frames per call");
    if (best_tracker_) throw std::logic_error("trackYUV: this RetinaFace tracks with best shots (trackYUVBest)");
    if (!tracker_) makeTracker(0);
    if (opt_.detect_every > 1) {
        for (const auto &call : intervalCalls(videos)) {
            vector<rf_yuv_frame> fr;
            vector<int> vi;
            for (int i : call.second) { fr.push_back(device_frames[i]); vi.push_back(videos[i]); }
            if (call.first) {
                // new-identity crops only when the call is one detect call: the crops' rows are the call's frames
                const bool whole = call.second.size() == device_frames.size();
                trackDetect(fr, vi, threshold, whole ? align : nullptr, whole ? dev_crops : nullptr);
            } else {
                followCall(fr, vi, nullptr);
            }
        }
        return;
    }
    trackDetect(device_frames, videos, threshold, align, dev_crops);
}

void RetinaFace::trackDetect(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, float threshold, const AlignOptions *align,
                             void *dev_crops) {
    int per = 0, cw = 0, ch = 0;
    const rf_align_params p = align ? crop_params(*align, opt_.max_faces, &per, &cw, &ch) : rf_align_params{};
    const int n = (int)device_frames.size();
    tracks_ = DeviceTracks{};
    int rc = rf_detect_yuv_track_device(h_, tracker_, device_frames.data(), videos.data(), n, RF_YUV_BT601, threshold, nms_threshold,
                                        align ? &p : nullptr, dev_crops, nullptr, &tracks_.tracks, &tracks_.counts, nullptr, nullptr, nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_yuv_track_device: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    tracks_.n = n;
    tracks_.max_tracks = 64;      // rf_track_config's default
    noteMotion(n);
}

rf_tracker RetinaFace::makeTracker(int lookback, bool lookback_search) {
    rf_track_config tc{};
    tc.max_videos = opt_.track_videos;
    int rc = rf_tracker_create(h_, &tc, &tracker_);
    if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_create: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    trackerCreated(!lookback);
    if (lookback) {
        const rf_lookback_config lc{lookback, 0.f};
        rc = rf_tracker_set_lookback(tracker_, &lc);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_lookback: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        if (lookback_search) {
            const rf_follow_config fc{0, 0.f};
            rc = rf_tracker_set_lookback_search(tracker_, &fc);
            if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_lookback_search: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
            tracker_search_ = true;
        }
        if (opt_.detect_every > 1) {      // f18: a following look-back tracker takes the follow frames
            const rf_follow_config fc{0, 0.f};
            rc = rf_tracker_set_lookback_follow(tracker_, &fc);
            if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_lookback_follow: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
            tracker_lookback_follow_ = true;
        }
    }
    return tracker_;
}

vector<std::pair<bool, vector<int>>> RetinaFace::intervalCalls(const vector<int> &videos) {
    std::map<std::pair<int, bool>, vector<int>> runs;     // (run p, follow?) -> frames: sorted, p first, then detect before follow
    std::map<int, std::pair<int, int>> seg;                // video -> (run, kind of that run: 1 detect, 0 follow)
    for (int i = 0; i < (int)videos.size(); i++) {
        const int v = videos[i];
        const bool det = frame_no_[v]++ % opt_.detect_every == 0;
        auto it = seg.find(v);
        int p = it == seg.end() ? 0 : it->second.first;
        if (it != seg.end() && it->second.second != (int)det) p++;
        seg[v] = {p, (int)det};
        runs[{p, !det}].push_back(i);
    }
    vector<std::pair<bool, vector<int>>> out;
    for (auto &r : runs) out.push_back({!r.first.second, r.second});
    return out;
}

void RetinaFace::followCall(const vector<rf_yuv_frame> &frames, const vector<int> &videos, const rf_redact_style *style,
                            const vector<rf_yuv_frame> *out_frames, int32_t *frame_numbers) {
    const int n = (int)frames.size();
    DeviceTracks t{};
    int rc = out_frames ? rf_track_follow_redact_lookback_device(tracker_, frames.data(), videos.data(), n, style, out_frames->data(), frame_numbers,
                                                                 &t.tracks, &t.counts)
             : style    ? rf_track_follow_redact_device(tracker_, frames.data(), videos.data(), n, style, &t.tracks, &t.counts)
                        : rf_track_follow_device(tracker_, frames.data(), videos.data(), n, &t.tracks, &t.counts);
    if (rc != RF_OK)
        throw std::runtime_error(string(out_frames ? "rf_track_follow_redact_lookback_device: "
                                        : style    ? "rf_track_follow_redact_device: "
                                                   : "rf_track_follow_device: ") +
                                 rf_status_string(rc) + ": " + rf_last_error(h_));
    tracks_ = t;
    tracks_.n = n;
    tracks_.max_tracks = 64;      // rf_track_config's default
    follow_ = DeviceFollow{};
    rc = rf_tracker_follow(tracker_, &follow_.follow);
    if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_follow: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    follow_.n = n;
    follow_.max_tracks = 64;
    noteMotion(n);
}

void RetinaFace::setVideoOrientation(int video, int orientation) {
    if (tracker_) {
        int rc = rf_tracker_set_orientation(tracker_, video, orientation);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_orientation: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    }
    orientations_.push_back({video, orientation});
}

void RetinaFace::trackerCreated(bool follow) {
    if (opt_.track_tiling) {
        if (opt_.track_tile_flip && opt_.track_tile_scales.empty())
            throw std::invalid_argument("track_tile_flip mirrors track_tile_scales; the default pyramid has none");
        vector<rf_tile_level> levels;
        for (float s : opt_.track_tile_scales) {
            levels.push_back(rf_tile_level{s, 0});
            if (opt_.track_tile_flip) levels.push_back(rf_tile_level{s, 1});
        }
        const rf_tiling t{levels.empty() ? nullptr : levels.data(), (int)levels.size(), opt_.track_tile_overlap};
        int rc = rf_tracker_set_tiling(tracker_, &t);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_tiling: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    }
    if (opt_.track_any_angle_step != 0.f) {
        const vector<rf_rotated_view> views = angleSweep("track_any_angle_step", opt_.track_any_angle_step);
        int rc = rf_tracker_set_views(tracker_, views.data(), (int)views.size());
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_views: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    }
    if (follow && opt_.detect_every > 1) {
        const rf_follow_config fc{};
        int rc = rf_tracker_set_follow(tracker_, &fc);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_follow: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    }
    if (opt_.track_motion) {
        const rf_motion_config mc{};
        int rc = rf_tracker_set_motion(tracker_, &mc);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_motion: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    }
    for (const auto &o : orientations_) {
        int rc = rf_tracker_set_orientation(tracker_, o.first, o.second);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_set_orientation: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    }
}

void RetinaFace::noteMotion(int n) {
    motion_ = DeviceMotion{};
    if (!opt_.track_motion) return;
    int rc = rf_tracker_motion(tracker_, &motion_.motion);
    if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_motion: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    motion_.n = n;
}

void RetinaFace::redactYUV(const vector<rf_yuv_frame> &device_frames, const vector<int> *videos, float threshold, const RedactOptions &opt,
                           const vector<rf_yuv_frame> *out_frames) {
    if (videos && videos->size() != device_frames.size()) throw std::invalid_argument("redactYUV: one video index per frame");
    if (opt.lookback && !videos) throw std::invalid_argument("redactYUV: lookback needs videos");
    if (out_frames && (!opt.lookback || out_frames->size() != device_frames.size()))
        throw std::invalid_argument("redactYUV: out_frames go with lookback, one per frame");
    if (device_frames.size() > (size_t)opt_.max_batch) throw std::invalid_argument("redactYUV: at most max_batch frames per call");
    if (videos && best_tracker_) throw std::logic_error("redactYUV: this RetinaFace tracks with best shots (trackYUVBest)");
    if (opt.lookback_search && !opt.lookback) throw std::invalid_argument("redactYUV: lookback_search needs lookback");
    if (videos && !tracker_) makeTracker(opt.lookback, opt.lookback_search);
    if (videos && opt.lookback_search && !tracker_search_)
        throw std::logic_error("redactYUV: lookback_search, but this RetinaFace's tracker was created without it (the first call decides)");
    if (videos && opt.lookback && opt_.detect_every > 1 && !tracker_lookback_follow_)
        throw std::logic_error("redactYUV: lookback with detect_every, but this RetinaFace's tracker was created without look-back (the first "
                               "call decides)");
    const rf_redact_style st{opt.style, opt.shape, opt.style == RF_REDACT_BLUR ? 0 : opt.blocks, opt.detail, opt.margin};
    const vector<rf_yuv_frame> &outs = out_frames ? *out_frames : device_frames;
    if (videos && opt_.detect_every > 1) {
        if (opt.lookback) frame_numbers_.assign(device_frames.size(), -1);
        for (const auto &call : intervalCalls(*videos)) {
            vector<rf_yuv_frame> fr, of;
            vector<int> vi;
            for (int i : call.second) { fr.push_back(device_frames[i]); vi.push_back((*videos)[i]); of.push_back(outs[i]); }
            vector<int32_t> nums(fr.size(), -1);
            if (opt.lookback) {       // f18: key frames through the look-back call, the others through its follow call
                if (call.first) lookbackCall(fr, vi, threshold, st, of, nums.data());
                else followCall(fr, vi, &st, &of, nums.data());
                for (size_t j = 0; j < call.second.size(); j++) frame_numbers_[call.second[j]] = nums[j];
            } else if (call.first) {
                DeviceTracks t{};
                int rc = rf_detect_yuv_redact_device_style(h_, tracker_, fr.data(), vi.data(), (int)fr.size(), RF_YUV_BT601, threshold,
                                                           nms_threshold, &st, &t.tracks, &t.counts, nullptr, nullptr, nullptr);
                if (rc != RF_OK)
                    throw std::runtime_error(string("rf_detect_yuv_redact_device_style: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
                tracks_ = t;
                tracks_.n = (int)fr.size();
                tracks_.max_tracks = 64;      // rf_track_config's default
                noteMotion((int)fr.size());
            } else {
                followCall(fr, vi, &st);
            }
        }
        return;
    }
    const int n = (int)device_frames.size();
    DeviceTracks t{};
    if (opt.lookback) {
        frame_numbers_.assign(n, -1);
        lookbackCall(device_frames, *videos, threshold, st, outs, frame_numbers_.data());
        return;
    }
    int rc = rf_detect_yuv_redact_device_style(h_, videos ? tracker_ : nullptr, device_frames.data(), videos ? videos->data() : nullptr, n,
                                               RF_YUV_BT601, threshold, nms_threshold, &st, &t.tracks, &t.counts, nullptr, nullptr, nullptr);
    if (rc != RF_OK)
        throw std::runtime_error(string("rf_detect_yuv_redact_device_style: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    if (videos) {
        tracks_ = t;
        tracks_.n = n;
        tracks_.max_tracks = 64;      // rf_track_config's default
        noteMotion(n);
    }
}

void RetinaFace::lookbackCall(const vector<rf_yuv_frame> &frames, const vector<int> &videos, float threshold, const rf_redact_style &st,
                              const vector<rf_yuv_frame> &out_frames, int32_t *frame_numbers) {
    const int n = (int)frames.size();
    DeviceTracks t{};
    int rc = rf_detect_yuv_redact_lookback_device(h_, tracker_, frames.data(), videos.data(), n, RF_YUV_BT601, threshold, nms_threshold, &st,
                                                  out_frames.data(), frame_numbers, &t.tracks, &t.counts, nullptr, nullptr, nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_yuv_redact_lookback_device: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    tracks_ = t;
    tracks_.n = n;
    tracks_.max_tracks = 64;      // rf_track_config's default
    noteMotion(n);
}

void RetinaFace::trackYUVBest(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, void *dev_best_crops, float threshold,
                              float min_quality) {
    if (videos.size() != device_frames.size()) throw std::invalid_argument("trackYUVBest: one video index per frame");
    if (device_frames.size() > (size_t)opt_.max_batch) throw std::invalid_argument("trackYUVBest: at most max_batch frames per call");
    if (tracker_ && !best_tracker_) throw std::logic_error("trackYUVBest: this RetinaFace already tracks without best shots (trackYUV)");
    if (!tracker_) {
        rf_track_config tc{};
        tc.max_videos = opt_.track_videos;
        rf_best_config bc{};
        bc.min_quality = min_quality;
        int rc = rf_tracker_create_best(h_, &tc, &bc, &tracker_);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_create_best: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        best_tracker_ = true;
        trackerCreated();
    }
    const int n = (int)device_frames.size();
    tracks_ = DeviceTracks{};
    best_ = DeviceBestShots{};
    int rc = rf_detect_yuv_track_best_device(h_, tracker_, device_frames.data(), videos.data(), n, RF_YUV_BT601, threshold, nms_threshold,
                                             dev_best_crops, nullptr, &best_.shots, &best_.counts, &tracks_.tracks, &tracks_.counts, nullptr,
                                             nullptr, nullptr);
    if (rc != RF_OK) throw std::runtime_error(string("rf_detect_yuv_track_best_device: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    tracks_.n = best_.n = n;
    tracks_.max_tracks = best_.max_tracks = 64;      // rf_track_config's default
    noteMotion(n);
}

void RetinaFace::trackYUVBest(const vector<rf_yuv_frame> &device_frames, const vector<int> &videos, void *dev_best_crops, float threshold,
                              const BestOptions &bo) {
    if (videos.size() != device_frames.size()) throw std::invalid_argument("trackYUVBest: one video index per frame");
    if (device_frames.size() > (size_t)opt_.max_batch) throw std::invalid_argument("trackYUVBest: at most max_batch frames per call");
    if (bo.detect_every < 1) throw std::invalid_argument("trackYUVBest: detect_every must be >= 1");
    if (tracker_ && !best_tracker_) throw std::logic_error("trackYUVBest: this RetinaFace already tracks without best shots (trackYUV)");
    if (tracker_ && bo.detect_every > 1 && !best_follow_)
        throw std::logic_error("trackYUVBest: detect_every > 1, but this RetinaFace's best-shot tracker was created without it (the first call decides)");
    bool detect = true;
    if (bo.detect_every > 1) {
        std::map<int, long long> nums = frame_no_;
        int kinds = 0;       // 1: a detect frame, 2: a follow frame
        for (int v : videos) kinds |= nums[v]++ % bo.detect_every == 0 ? 1 : 2;
        if (kinds == 3)
            throw std::invalid_argument("trackYUVBest: with detect_every > 1 a call takes detect frames only or follow frames only (its videos' frame "
                                        "numbers must agree modulo detect_every)");
        detect = kinds != 2;
        frame_no_ = nums;
    }
    if (!tracker_) {
        rf_track_config tc{};
        tc.max_videos = opt_.track_videos;
        rf_best_config bc{};
        bc.min_quality = bo.min_quality;
        int rc = rf_tracker_create_best(h_, &tc, &bc, &tracker_);
        if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_create_best: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        best_tracker_ = true;
        if (bo.live && (rc = rf_tracker_set_best_live(tracker_, &bo.live_config)) != RF_OK)
            throw std::runtime_error(string("rf_tracker_set_best_live: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        if (bo.detect_every > 1) {
            const rf_follow_config fc{};
            if ((rc = rf_tracker_set_best_follow(tracker_, &fc)) != RF_OK)
                throw std::runtime_error(string("rf_tracker_set_best_follow: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
            best_follow_ = true;
        }
        trackerCreated(false);
    }
    const int n = (int)device_frames.size();
    tracks_ = DeviceTracks{};
    best_ = DeviceBestShots{};
    int rc = detect ? rf_detect_yuv_track_best_device(h_, tracker_, device_frames.data(), videos.data(), n, RF_YUV_BT601, threshold, nms_threshold,
                                                      dev_best_crops, nullptr, &best_.shots, &best_.counts, &tracks_.tracks, &tracks_.counts,
                                                      nullptr, nullptr, nullptr)
                    : rf_track_follow_best_device(tracker_, device_frames.data(), videos.data(), n, dev_best_crops, nullptr, &best_.shots,
                                                  &best_.counts, &tracks_.tracks, &tracks_.counts);
    if (rc != RF_OK)
        throw std::runtime_error(string(detect ? "rf_detect_yuv_track_best_device: " : "rf_track_follow_best_device: ") + rf_status_string(rc) + ": " +
                                 rf_last_error(h_));
    tracks_.n = best_.n = n;
    tracks_.max_tracks = best_.max_tracks = 64;      // rf_track_config's default
    if (!detect) {
        const rf_follow *f = nullptr;
        if ((rc = rf_tracker_follow(tracker_, &f)) != RF_OK)
            throw std::runtime_error(string("rf_tracker_follow: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
        follow_ = DeviceFollow{f, n, 64};
    }
    noteMotion(n);
}

void RetinaFace::finishVideo(int video, void *dev_best_crops) {
    if (!tracker_ || !best_tracker_) throw std::logic_error("finishVideo: no best-shot tracker (trackYUVBest)");
    frame_no_.erase(video);      // the video restarts: with detect_every, its next frame is a detect frame
    best_ = DeviceBestShots{};
    int rc = rf_tracker_finish(tracker_, video, dev_best_crops, nullptr, &best_.shots, &best_.counts);
    if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_finish: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    best_.n = 1;
    best_.max_tracks = 64;
}

void RetinaFace::resetTracks(int video) {
    if (video < 0) frame_no_.clear();
    else frame_no_.erase(video);
    if (!tracker_) return;
    int rc = rf_tracker_reset(tracker_, video);
    if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_reset: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
}

Mat RetinaFace::draw(const Mat &img, const vector<FaceDetectInfo> &faces) {
    Mat out = img.clone();     // RetinaFace.cpp:744: drawing on the caller's image would accumulate boxes
    auto fill = [&out](int x0, int y0, int x1, int y1, unsigned char b, unsigned char g, unsigned char r) {
        x0 = std::max(x0, 0); y0 = std::max(y0, 0); x1 = std::min(x1, out.cols); y1 = std::min(y1, out.rows);
        for (int y = y0; y < y1; y++)
            for (int x = x0; x < x1; x++) {
                unsigned char *p = out.data + (size_t)y * out.step + (size_t)x * 3;
                p[0] = b; p[1] = g; p[2] = r;
            }
    };
    for (const FaceDetectInfo &f : faces) {
        const int x1 = (int)lroundf(f.rect.x1), y1 = (int)lroundf(f.rect.y1), x2 = (int)lroundf(f.rect.x2), y2 = (int)lroundf(f.rect.y2);
        fill(x1 - 1, y1 - 1, x2 + 1, y1 + 1, 0, 0, 255);      // Scalar(0, 0, 255), thickness 2 (:735)
        fill(x1 - 1, y2 - 1, x2 + 1, y2 + 1, 0, 0, 255);
        fill(x1 - 1, y1 - 1, x1 + 1, y2 + 1, 0, 0, 255);
        fill(x2 - 1, y1 - 1, x2 + 1, y2 + 1, 0, 0, 255);
        for (int k = 0; k < 5; k++) {                          // Scalar(0, 255, 0) dots (:739)
            const int cx = (int)lroundf(f.pts.x[k]), cy = (int)lroundf(f.pts.y[k]);
            fill(cx - 1, cy - 1, cx + 2, cy + 2, 0, 255, 0);
        }
    }
    return out;
}

vector<int32_t> RetinaFace::drainVideo(int video, const vector<rf_yuv_frame> &out_frames, const RedactOptions &opt) {
    if (!tracker_) throw std::logic_error("drainVideo: no look-back tracker (redactYUV with lookback first)");
    const rf_redact_style st{opt.style, opt.shape, opt.style == RF_REDACT_BLUR ? 0 : opt.blocks, opt.detail, opt.margin};
    vector<int32_t> nums(out_frames.size());
    int n = 0;
    int rc = rf_tracker_drain(tracker_, video, &st, out_frames.data(), (int)out_frames.size(), &n, nums.data());
    if (rc != RF_OK) throw std::runtime_error(string("rf_tracker_drain: ") + rf_status_string(rc) + ": " + rf_last_error(h_));
    frame_no_.erase(video);       // the drain restarts the video: its key frames count from 0 again, as the library's numbers do
    nums.resize(n);
    return nums;
}
