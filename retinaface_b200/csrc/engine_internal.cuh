// engine_internal.cuh -- what the translation units behind include/rf_b200.h share: the handle, the step / tensor records,
// the plan builder, and the functions each unit exports to the others.
//   plan_net.cu  the walk of the network every layer plan is built from, and the leaf helpers the plans share
//   plan_fp.cu   SIMT layer plans (FP32, FP16 without tensor cores), FP16 tensor-core per-layer operations and launch helpers
//   plan_tile.cu FP16 tensor-core layer plan: tile chains, and the per-layer operations where a chain is off or does not fit
//   plan_i8.cu   INT8 layer plan (build_plan_i8)
//   engine.cu    tensor placement, CUDA-graph executor, the detect C-ABI entry points
//   tracker.cu   the video tracker's C-ABI entry points (f10 - f17) and redaction
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "align.cuh"
#include "common.cuh"
#include "host_copy.h"
#include "model.h"
#include "postproc.cuh"
#include "preprocess.cuh"

using namespace rf;

#define RF_STR2(x) #x
#define RF_STR(x) RF_STR2(x)

namespace rf_eng {

// SMs assumed where no device is queried (rf_plan_describe): the H100 SXM.  rf_create takes the device's own count.
constexpr int RF_NUM_SMS = 132;

struct TileChain;                 // plan_tile.cu
std::string &create_error();      // thread-local text of the last failed rf_create (engine.cu)

struct CudaFail { cudaError_t e; const char *what; const char *file; int line; };
// a plan-time failure that is not a CUDA error: carries the rf_status and the full message to rf_create / the caller
struct PlanFail { int status; std::string msg; };
#define CK(call)                                                        \
    do {                                                                \
        cudaError_t _e = (call);                                        \
        if (_e != cudaSuccess) throw CudaFail{_e, #call, __FILE__, __LINE__}; \
    } while (0)

inline std::string fmt(const char *f, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, f);
    vsnprintf(buf, sizeof buf, f, ap);
    va_end(ap);
    return buf;
}

struct TensorInfo {
    std::string name;
    int h = 0, w = 0, c = 0;
    size_t bytes_per_img = 0;
    int first = -1, last = -1;
    size_t offset = 0;  // bytes into the arena (already scaled by max_batch)
};

// One execution context: everything a forward pass writes (activation arena, candidate / output buffers, run parameters)
// and everything it is issued on (stream, lane streams, events, captured graphs).  The asynchronous entry points rotate
// through the handle's contexts so that consecutive batches overlap on the GPU (most kernels of one batch-8 step fill well
// under one wave of the 132 SMs).
struct Ctx {
    static constexpr int kParamSlots = 1024;
    cudaStream_t stream = nullptr, lane_stream[3] = {nullptr, nullptr, nullptr};   // [0] unused (lane 0 runs on `stream`)
    std::vector<cudaEvent_t> step_event;
    unsigned char *arena = nullptr;
    PostBuffers pb{};
    PostParams *d_params = nullptr, *h_params = nullptr;   // h_params: pinned ring of kParamSlots (set_params)
    unsigned param_seq = 0;
    float cur_thr = 0.5f, cur_nms = 0.4f;
    std::map<int, cudaGraphExec_t> graphs;
    cudaEvent_t fence = nullptr;
    // rf_detect_yuv_batch_device (lazily allocated): this context's letter-boxed frames [max_batch][H][W][3].  One tensor per
    // context: the letter-box of a call on another context must not overwrite the input of a forward still running here.
    uint8_t *d_frames_in = nullptr;
    // f12 redaction scratch (redact.cuh; lazily allocated, grown when a call needs more): region tables and cell means of the calls
    // issued on this context's stream.  Per context: calls on two contexts' streams may run at once.
    void *d_redact = nullptr;
    size_t redact_bytes = 0;
};

// What one step launch writes into and where it is issued.
struct Run {
    const Ctx &ctx;                  // arena, pb, d_params
    int n;
    cudaStream_t stream;
    float *const *blobs = nullptr;   // rf_forward_heads: the head step also writes the nine raw head blobs here
    bool single = false;             // rf_profile_layers: a step launched on its own, out of its forward (no last-block NMS)
};

struct Step {
    std::string name;
    std::vector<int> in, out;
    std::function<void(const Run &)> launch;
    double flops_per_img = 0, bytes_per_img = 0;  // algorithmic
    int lane = 0;                 // 0 = main stream; 1, 2 = side branches of the forward graph
    std::vector<int> deps;        // producer steps in OTHER lanes this step must wait for (filled by link_steps)
    bool signals = false;         // some step in another lane waits for this one
    std::string geom;             // the tiles its launch arguments fix, "key=value ..." (rf_plan_describe; empty: none)
};

}  // namespace rf_eng
using namespace rf_eng;

namespace rf_eng {
// multi-GPU exchange state of a handle (comm.cu)
struct Comm {
    int rank = 0, world = 1, ring = 0;
    bool ready = false;
    unsigned char *window = nullptr;       // this rank's gather window (device)
    size_t bytes = 0;
    unsigned char *peer[RF_COMM_MAX_WORLD] = {nullptr};
    bool opened[RF_COMM_MAX_WORLD] = {false};
    unsigned seq = 0;                      // steps exchanged so far
    unsigned *d_err = nullptr, *h_err = nullptr;
    unsigned char blob[128] = {0};
    struct Slot { rf_det *h_dets = nullptr; int *h_counts = nullptr; } slots[RF_PIPELINE_DEPTH];   // pinned, [world][max_batch]...
};
}  // namespace rf_eng

struct rf_handle_s {
    rf_config cfg{};
    rf_eng::Comm comm;
    std::string caffemodel, table;
    std::string err;
    Model model;
    std::map<std::string, float> int8_scales;
    int device = 0;
    int num_sms = RF_NUM_SMS;   // plan heuristics ("does this layer fill one wave") and the persistent tile-chain grid
    bool on_device = false;     // the plan is built for launches (rf_create), not only described: occupancy may be queried
    int elem = 4;  // bytes per activation element
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;

    std::vector<TensorInfo> tensors;
    std::map<std::string, int> tensor_by_name;
    std::vector<Step> steps;
    std::vector<std::shared_ptr<TileChain>> chains;   // tile-chain launches of the FP16 plan (plan_tile.cu)
    int lane_last[3] = {-1, -1, -1};                  // last step of each side lane (joined at the end of the forward)
    int cache_status = 0;                             // model.h CACHE_*: how the folded model was obtained
    int tile_expected = 0;                            // tiles per image over the three SSH chains (last-block NMS)
    std::vector<float> tile_bias_tmp;                 // plan-time scratch
    unsigned *tile_dbg = nullptr, *tile_dbg_dev = nullptr;   // host-mapped word a timed-out hand-off of a tile chain reports into
    size_t arena_bytes = 0;                           // of each context's arena

    // weights
    std::vector<float> wstage;  // host staging of all fp32 weights
    float *d_weights = nullptr;
    std::vector<__half> wstage_h;  // FP16 tensor-core weight images (tc_conv.cuh B chunks)
    __half *d_weights_h = nullptr;
    std::vector<int8_t> wstage_q;  // INT8 tensor-core weight images (tc_conv_i8.cuh)
    int8_t *d_weights_q = nullptr;

    // io
    uint8_t *d_input = nullptr;       // [max_batch][H][W][3] u8 BGR
    uint8_t *h_input = nullptr;       // pinned mirror
    PostBuffers pb_merge{};           // rf_detect_views: candidates of all views of one image (lazily allocated)
    PostBuffers pb_tiles{};           // rf_detect_tiled: candidates of all tiles of each image (lazily grown to the largest layout)
    // rf_detect_tiled_device / rf_detect_yuv_tiled_device: a ring of `streams` output slots (created by the first such call).  A
    // slot holds one call's merged candidates and final records (grown lazily like pb_tiles); `free` is recorded once the call's
    // crops are cut, `start` once the call's home stream has waited for `free`.
    struct TiledSlot {
        PostBuffers pb{};
        cudaEvent_t free = nullptr, start = nullptr;
    };
    std::vector<TiledSlot> tiled_slots;
    unsigned next_tiled_slot = 0;
    // rf_detect_views_rotated_device / rf_detect_yuv_views_rotated_device (f24): a ring of their own, so that tiled records keep
    // their validity rule across rotated calls
    std::vector<TiledSlot> rotated_slots;
    unsigned next_rotated_slot = 0;
    uint8_t *d_raw = nullptr;         // one raw caller image (max_image) for the letterbox kernel
    uint8_t *h_raw = nullptr;         // pinned, TWO buffers of raw_bytes: staging of pageable caller images (upload_plane)
    size_t raw_bytes = 0;
    int raw_slots = 1;                // raw device buffers (one per batch element, capped)
    cudaEvent_t raw_ev[2] = {nullptr, nullptr};   // H2D out of staging buffer i has completed
    unsigned raw_seq = 0;
    std::unique_ptr<HostCopyPool> copy_pool;      // row-band parallel host copy into the staging buffers (lazily created)
    // the blocking align paths (lazily allocated): the crops (grown on demand) and the matrices [max_batch][max_faces][6]
    void *d_align_crops = nullptr;
    size_t align_crops_bytes = 0;
    double *d_align_mats = nullptr;
    LevelDesc lv[3];
    HeadWeights hw[3];
    int feat_tensor[3] = {-1, -1, -1};
    float *d_blobs[9] = {nullptr};    // rf_forward_heads / rf_postprocess staging (device)
    size_t blob_elems[9] = {0};       // per image
    rf_det *h_dets = nullptr;         // pinned [max_batch][max_faces]
    int *h_counts = nullptr;          // pinned [2*max_batch]: kept, candidates
    // pipelined end-to-end path (rf_submit_batch / rf_collect_batch)
    struct Slot {
        uint8_t *d_in = nullptr, *h_in = nullptr;     // device input, pinned staging for pageable sources
        rf_det *h_dets = nullptr;                      // pinned results
        int *h_counts = nullptr;
        cudaEvent_t ev_h2d = nullptr, ev_done = nullptr;
        int n = 0;
        bool busy = false, gather = false;
    } slots[RF_PIPELINE_DEPTH];
    cudaStream_t copy_stream = nullptr;
    unsigned submit_seq = 0, collect_seq = 0;
    // execution contexts (Ctx): the blocking entry points run on context 0, the asynchronous ones rotate through all
    std::vector<Ctx> ctx;
    unsigned next_dev_ctx = 0;
    cudaStream_t last_stream = nullptr;   // of the last device-resident call (rf_last_stream)
    void *jpeg = nullptr;             // nvJPEG decoder state (jpeg.cu), created by the first JPEG call
};

namespace rf_eng {
inline int fail(rf_handle h, int code, const std::string &msg) {
    if (h) h->err = msg; else create_error() = msg;
    return code;
}
inline int fail_cuda(rf_handle h, const CudaFail &f) {
    std::string extra;
    if (h && h->tile_dbg && h->tile_dbg[0])
        extra = fmt(" [tile chain: CTA %u timed out waiting at tile_chain.cuh:%u]", h->tile_dbg[0] >> 20, h->tile_dbg[0] & 0xfffffu);
    return fail(h, RF_ERR_CUDA, fmt("%s failed: %s (%s:%d)%s", f.what, cudaGetErrorString(f.e), f.file, f.line, extra.c_str()));
}

// ---------------------------------------------------------------------------------------------
// Plan builder
// ---------------------------------------------------------------------------------------------
struct Builder {
    rf_handle h;
    int H, W;
    size_t add_weights(const std::vector<float> &v) {
        size_t off = h->wstage.size();
        h->wstage.insert(h->wstage.end(), v.begin(), v.end());
        while (h->wstage.size() % 4) h->wstage.push_back(0.f);  // keep float4 alignment
        return off;
    }
    size_t add_weights_h(const std::vector<__half> &v) {
        size_t off = h->wstage_h.size();
        h->wstage_h.insert(h->wstage_h.end(), v.begin(), v.end());
        while (h->wstage_h.size() % 64) h->wstage_h.push_back(__float2half(0.f));  // 128-byte alignment for bulk copies
        return off;
    }
    size_t add_weights_q(const std::vector<int8_t> &v) {
        size_t off = h->wstage_q.size();
        h->wstage_q.insert(h->wstage_q.end(), v.begin(), v.end());
        while (h->wstage_q.size() % 128) h->wstage_q.push_back(0);
        return off;
    }
    int tensor(const std::string &name, int hh, int ww, int c) {
        TensorInfo t;
        t.name = name; t.h = hh; t.w = ww; t.c = c;
        t.bytes_per_img = (size_t)hh * ww * c * h->elem;
        h->tensors.push_back(t);
        h->tensor_by_name[name] = (int)h->tensors.size() - 1;
        return (int)h->tensors.size() - 1;
    }
    void step(Step s) { h->steps.push_back(std::move(s)); }
};

// ---- layer plans: one walk of the network (plan_net.cu) calls one set of operations per plan --------------------------------
// A destination of a convolution's output channels: n channels (the first destination; the second takes the rest) at channel
// `off` of rows of `ld` channels of tensor t (t < 0: none).
struct ConvOut { int t = -1, ld = 0, off = 0, n = 0, relu = 0; };
// One convolution step: convolutions sharing the input, concatenated along N.
struct ConvNode {
    std::string name;                       // step name without the plan's prefix
    std::vector<const FoldedConv *> cs;
    int in = -1, h = 0, w = 0;              // input tensor and its map size
    ConvOut out[2];                         // out[1].t < 0: one destination
    int lane = 0;
    int up = -1, up_which = 0;              // up >= 0: the FPN merge in + deconv(up, up_w[up_which]) fused into the staging ...
    std::string sum;                        // ... the name of that never materialised sum (its INT8 scale)
};
// Depthwise i + pointwise i+1 on an h x w input; the op creates the output tensor `out` (and, where it stores it, `mid`).
struct PairNode { int i; const FoldedConv *dw, *pw; std::string mid, out; int h, w; };
struct StemNode { const FoldedConv *conv0; std::string out0; PairNode pair; };   // conv0 -> out0, then pair 1 + 2
// Backbone segment: pairs, then optionally the lateral 1x1 conv `lat` on the last pair's output, into a new tensor `lat_out`
// (lat.in and lat.out[0].t are set by the op).
struct SegNode { std::vector<PairNode> pairs; ConvNode lat; std::string lat_out; };
struct SegOut { int out, lat; };
// FPN level `level` (1 = stride 16, 2 = stride 8): lat + upsample(up) -> the tensor `sum`, then aggr 3x3; `fused` is the
// aggr conv with the merge fused into it, `aggr` the one on the stand-alone sum (aggr.in set by the op).
struct MergeNode { std::string lv, sum; int level, lat, up, h, w; ConvNode fused, aggr; };
// SSH level `level` (0 = stride 32) on `in` into the concat tensor `cat`: conv1 + context conv1 (-> ctx1), context conv2 +
// conv3_1 (-> ctx31), context conv3_2; then the level's predictors (cls, bbox, landmark).
struct SshNode {
    std::string lv, ctx1, ctx31;
    int level, lane, in, h, w, cat;
    const FoldedConv *conv1, *ctx_conv1, *ctx_conv2, *ctx_conv3_1, *ctx_conv3_2;
    const FoldedConv *pred[3];
};
struct HeadsNode { const FoldedConv *pred[3][3]; };     // [level][cls, bbox, landmark]; inputs: h->feat_tensor

struct PlanOps {
    Builder B;
    explicit PlanOps(rf_handle h) : B{h, h->cfg.net_h, h->cfg.net_w} {}
    virtual ~PlanOps() = default;
    virtual int stem(const StemNode &n) = 0;                // returns the output of the stem's pair
    virtual int pair(const PairNode &p, int in) = 0;        // returns the pointwise output
    virtual void conv(const ConvNode &c) = 0;
    virtual int merge(const MergeNode &m) = 0;              // stand-alone FPN merge; returns the `sum` tensor
    virtual bool fuse_merge(const MergeNode &m) = 0;        // this plan's rule: merge fused into the aggr conv
    virtual void heads(const HeadsNode &n) = 0;             // predictors + decode + NMS of all levels
    // defaults built from the operations above (plan_net.cu)
    SegOut segment(const SegNode &s, int in);
    virtual void merge_aggr(const MergeNode &m);
    virtual void ssh(const SshNode &n);
};
void walk_network(PlanOps &ops);                            // plan_net.cu: the graph, in step order
// shared leaf helpers (plan_net.cu)
struct StemPack { std::vector<float> w0, wd, wp; };         // conv0 [27][8] (k = tap*3 + BGR channel), dw1 [9][8], pw2 [8][16]
StemPack pack_stem(const StemNode &n);
std::vector<float> pack_dw(const FoldedConv &dw, float scale = 1.f);   // depthwise 3x3 weights [9][C], times scale
struct DwGeom { int rows, nsplit, Rmax; };
DwGeom dw_geometry(int C, int N, int IH, int IW, int S, const std::function<bool(int rows, int N, int R)> &fits);
int dw2d_tile_w(rf_handle h, int C, int oh, int ow, int nsplit);     // 2-D tile width of a pair's kernel; 0: 1-D
bool aggr_fits_one_wave(rf_handle h, int fh, int fw);

// ---- exported by plan_fp.cu -----------------------------------------------------------------------------------------
constexpr int TC_SMEM_LIMIT = 200 * 1024;   // dynamic shared memory the tensor-core kernels may opt into (they also hold ~5 KB static)
template <typename T>
void build_plan(rf_handle h);               // the SIMT plans: T = float (RF_PREC_FP32) | __half (RF_PREC_FP16, RF_FLAG_NO_TENSORCORE)
cudaError_t tc_init();
template <typename OutT>
int plan_stem_fused(Builder &B, const StemNode &n, const char *suffix, float out_scale);   // conv0 + dw1 + pw2 in one kernel
int resident_ctas(rf_handle h, const void *kern, int threads, size_t smem);
// Persistent grid over `tiles` tiles: each CTA takes a run of consecutive tiles, the grid is what the device holds at once.
struct PersistentGrid { int run, grid; };
inline PersistentGrid persistent_grid(int tiles, int resident) {
    const int run = std::max(1, (tiles + resident - 1) / std::max(resident, 1));
    return {run, (tiles + run - 1) / run};
}
// the FP16 tensor-core operations (per layer)
int plan_pair_tc(Builder &B, const PairNode &p, int in);
void plan_conv_tc(Builder &B, const ConvNode &c);
int plan_fpn_merge_h2(Builder &B, const MergeNode &m);
template <typename T>
void plan_heads(Builder &B, const HeadsNode &n, const float scale[3], const char *prefix);
std::vector<__half> pack_tc_weights(const std::vector<const FoldedConv *> &cs, std::vector<float> &bias, int &Kpad, int nsplit = 1);
// ---- exported by plan_tile.cu ---------------------------------------------------------------------------------------
void build_plan_tiles(rf_handle h);         // RF_PREC_FP16 with tensor cores: per-layer kernels + (latency mode) tile chains (tile_chain.cuh)
cudaError_t tile_init();
std::string describe_chains(rf_handle h);
// ---- exported by comm.cu --------------------------------------------------------------------------------------------
void comm_release(rf_handle h);
void comm_wait_in_graph(rf_handle h, const Ctx &c, int n, cudaStream_t s);   // last node of the forward once a communicator exists
// ---- exported by jpeg.cu (f1 ingest: nvJPEG decode into device memory) ------------------------------------------------
int jpeg_info(rf_handle h, const uint8_t *data, size_t len, int *w, int *hgt);
int jpeg_decode(rf_handle h, const uint8_t *const *data, const size_t *len, int n, uint8_t *const *dst, const int *w, const int *hgt, cudaStream_t s);
void jpeg_release(rf_handle h);
const char *jpeg_backend(rf_handle h);
// ---- exported by plan_i8.cu -----------------------------------------------------------------------------------------
void build_plan_i8(rf_handle h);
cudaError_t tc_init_i8();

// ---- exported by engine.cu (the detect entry points) -----------------------------------------------------------------
int check_n(rf_handle h, int n);
int check_frames(rf_handle h, const char *who, const rf_yuv_frame *frames, int n, int matrix);
int check_orientations(rf_handle h, const char *who, const int *orientations, int n);
void upload_plane(rf_handle h, cudaStream_t s, uint8_t *d_dst, const uint8_t *src, size_t row_bytes, size_t pitch, int rows);
int align_setup(rf_handle h, const char *who, const rf_align_params *p, AlignArgs &a);
int check_align(rf_handle h, const char *who, const rf_align_params *p, int n, const void *crops, int resident, AlignArgs &a);

// ---- image sources ---------------------------------------------------------------------------------------------------------------
// Every detect entry point describes the caller's pixels with one of two sources.  A source checks the caller's description (every
// check runs before anything is copied or launched), reports image i's stored size and EXIF orientation, and hands the letter-box
// and crop kernels its pixels: upload(s, i, slot) copies host image i into raw buffer `slot` on s (the blocking paths),
// in_place(i) reads the caller's device memory (the asynchronous ones).  Src is what those kernels read.

// BGR images: u8 BGR HWC rows row_strides[i] bytes apart (NULL or 0: packed), shown in EXIF orientation orient[i] when `oriented`.
struct BgrImages {
    using Src = BgrRows;
    const uint8_t *const *imgs;
    const int *widths, *heights, *row_strides, *orient;
    bool oriented;
    int width(int i) const { return widths[i]; }
    int height(int i) const { return heights[i]; }
    int stride(int i) const { return row_strides && row_strides[i] ? row_strides[i] : widths[i] * 3; }
    int bits(int i) const { return oriented ? lb_orientation_bits(orient[i]) : 0; }
    // network-sized, packed and upright: copied straight into the input tensor, without a raw buffer or a letter-box
    bool direct(rf_handle h, int i) const {
        return widths[i] == h->cfg.net_w && heights[i] == h->cfg.net_h && stride(i) == h->cfg.net_w * 3 && bits(i) == 0;
    }
    int check(rf_handle h, const char *who, int n) const {
        int rc = check_n(h, n);
        if (rc) return rc;
        if (n > 0 && (!imgs || !widths || !heights)) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: NULL image arrays", who));
        for (int i = 0; i < n; i++) {
            if (!imgs[i] || widths[i] <= 0 || heights[i] <= 0) return fail(h, RF_ERR_INVALID_ARG, fmt("%s: image %d is empty", who, i));
            if (stride(i) < widths[i] * 3)
                return fail(h, RF_ERR_INVALID_ARG, fmt("%s: image %d: row stride %d below %d bytes", who, i, stride(i), widths[i] * 3));
            if (widths[i] > h->cfg.max_image_w || heights[i] > h->cfg.max_image_h)
                return fail(h, RF_ERR_CAPACITY, fmt("%s: image %d is %dx%d, larger than max_image %dx%d", who, i, widths[i], heights[i],
                                                    h->cfg.max_image_w, h->cfg.max_image_h));
        }
        return oriented ? check_orientations(h, who, orient, n) : RF_OK;
    }
    BgrRows upload(rf_handle h, cudaStream_t s, int i, int slot) const {
        uint8_t *d = h->d_raw + (size_t)slot * h->raw_bytes;
        upload_plane(h, s, d, imgs[i], (size_t)widths[i] * 3, (size_t)stride(i), heights[i]);
        return BgrRows{d, widths[i] * 3};
    }
    BgrRows in_place(int i) const { return BgrRows{imgs[i], stride(i)}; }
};

// YUV 4:2:0 frames (yuv.cuh) in `matrix`, shown in EXIF orientation orient[i] when `oriented`.
struct YuvFrames {
    using Src = YuvPlanes;
    const rf_yuv_frame *frames;
    int matrix;
    const int *orient;
    bool oriented;
    int width(int i) const { return frames[i].width; }
    int height(int i) const { return frames[i].height; }
    int bits(int i) const { return oriented ? lb_orientation_bits(orient[i]) : 0; }
    bool direct(rf_handle, int) const { return false; }
    int check(rf_handle h, const char *who, int n) const {
        int rc = check_frames(h, who, frames, n, matrix);
        if (rc || !oriented) return rc;
        return check_orientations(h, who, orient, n);
    }
    // 1.5 bytes per pixel: the luma packed, then the chroma as the frame lays it out (one interleaved w x h/2 plane, or two
    // w/2 x h/2 planes)
    YuvPlanes upload(rf_handle h, cudaStream_t s, int i, int slot) const {
        const rf_yuv_frame &f = frames[i];
        uint8_t *d = h->d_raw + (size_t)slot * h->raw_bytes, *dc = d + (size_t)f.width * f.height;
        const int cw = f.width / 2, ch = f.height / 2;
        upload_plane(h, s, d, f.y, f.width, f.y_pitch, f.height);
        YuvPlanes p{d, dc, dc, f.width, f.width, f.uv_step, matrix};
        if (f.uv_step == 2) {
            const uint8_t *first = std::min(f.u, f.v);
            upload_plane(h, s, dc, first, f.width, f.uv_pitch, ch);
            p.u = dc + (f.u - first);
            p.v = dc + (f.v - first);
        } else {
            upload_plane(h, s, dc, f.u, cw, f.uv_pitch, ch);
            upload_plane(h, s, dc + (size_t)cw * ch, f.v, cw, f.uv_pitch, ch);
            p.v = dc + (size_t)cw * ch;
            p.uv_pitch = cw;
        }
        return p;
    }
    YuvPlanes in_place(int i) const {
        const rf_yuv_frame &f = frames[i];
        return YuvPlanes{f.y, f.u, f.v, f.y_pitch, f.uv_pitch, f.uv_step, matrix};
    }
};

int yuv_device_impl(rf_handle h, const char *who, const YuvFrames &src, int n, float thr, float nms, const rf_align_params *align,
                    void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales);
// rf_detect_yuv_tiled_device without crops, split for the tracker (f19): the check (the frames, then each frame's layout, before
// anything is launched) and the issue into the tiled ring on its home context (rf_last_stream).  *free is the ring slot's event: a
// caller that reads the records later on home records it again there after its last read.  tiling_supported: the handle's
// refusal of any tiling (RF_FLAG_NPP_RESIZE), with the tiled paths' message.
int yuv_tiled_check(rf_handle h, const char *who, const YuvFrames &src, int n, const rf_tiling *t, std::vector<std::vector<rf_tile>> &layouts);
int yuv_tiled_issue(rf_handle h, const YuvFrames &src, int n, const std::vector<std::vector<rf_tile>> &layouts, float thr, float nms,
                    const rf_det **dev_dets, const int32_t **dev_counts, cudaEvent_t *free);
int tiling_supported(rf_handle h, const char *who);
// rf_detect_yuv_views_rotated_device without crops, split for the tracker as the tiled call is (f25): the views' own checks (NULL,
// 1..RF_MAX_VIEWS, each angle and shrink, with f23 / f24's statuses and messages), the check (the frames, then the views) and the issue
// into the rotated ring on its home context.  A frame of an oriented source (src.oriented) is rotated as it is displayed: its views are
// those of D = T_o(S), their records in displayed pixels.  *free is the ring slot's event, as yuv_tiled_issue's.
int rotated_views_check(rf_handle h, const char *who, const rf_rotated_view *views, int nviews);
int yuv_rotated_check(rf_handle h, const char *who, const YuvFrames &src, int n, const rf_rotated_view *views, int nviews);
int yuv_rotated_issue(rf_handle h, const YuvFrames &src, int n, const rf_rotated_view *views, int nviews, float thr, float nms,
                      const rf_det **dev_dets, const int32_t **dev_counts, cudaEvent_t *free);

}  // namespace rf_eng
