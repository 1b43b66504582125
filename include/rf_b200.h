/*
 * rf_b200.h -- C ABI of librf_b200.so: the H100-native (sm_90a) RetinaFace mnet25 detect path.
 *
 * This is the drop-in boundary.  The reference has no FFI layer of its own: its seam is the
 * C++ class `TrtRetinaFaceNet` plus three free CUDA launchers used by `RetinaFace`
 * (retinaface/RetinaFace.cpp:4-6,275-291,584-608,655,670-684).  Each entry point below names
 * the reference interface it replaces.  Plain pointers and sizes only; no C++/torch types.
 *
 * Conventions
 *   - every function returns RF_OK (0) or a negative rf_status; rf_last_error() gives text.
 *     Nothing aborts/exits (the reference abort()s/exit()s/throws: trtutility.h:9-16,
 *     trtnetbase.cpp:201-204, RetinaFace.cpp:327-335).
 *   - one handle = one device + one stream; calls on a handle are serialised by the caller
 *     (the reference is single-threaded and non re-entrant, SURVEY.md 8b).
 *   - there is NO CPU fallback: every compute entry point runs CUDA kernels on the handle's
 *     device and fails with RF_ERR_CUDA if that is impossible.
 *   - images are u8 BGR HWC like cv::Mat (RetinaFace.cpp:594), results are FaceDetectInfo
 *     records (RetinaFace.h:37-42) in network-input pixel coordinates (RetinaFace.cpp:707).
 */
#ifndef RF_B200_H
#define RF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RF_B200_ABI_VERSION 2     /* 2: rf_config gained prototxt_path / cache_path / network (appended) */

typedef enum rf_status {
    RF_OK = 0,
    RF_ERR_INVALID_ARG = -1,
    RF_ERR_IO = -2,          /* model file missing / unreadable */
    RF_ERR_MODEL = -3,       /* caffemodel does not hold the mnet25 topology */
    RF_ERR_CUDA = -4,        /* CUDA runtime / launch failure (text in rf_last_error) */
    RF_ERR_NO_DEVICE = -5,   /* no sm_90 device: the library has no CPU path */
    RF_ERR_CAPACITY = -6,    /* batch / image larger than the handle was created for */
    RF_ERR_UNSUPPORTED = -7
} rf_status;

/* Arithmetic of the network body.  Head 1x1 convs, softmax, decode and NMS are always FP32. */
typedef enum rf_precision {
    RF_PREC_FP32 = 0,   /* FP32 storage + FP32 SIMT math: the tight-parity mode */
    RF_PREC_FP16 = 1,   /* FP16 NHWC activations/weights, FP32 accumulate (wgmma where GEMM-shaped) */
    RF_PREC_INT8 = 2    /* INT8 activations with the TensorRT calibration-table scales */
} rf_precision;

/* == FaceDetectInfo (RetinaFace.h:37-42): score, rect(x1,y1,x2,y2), pts.x[5], pts.y[5]. */
typedef struct rf_face {
    float score;
    float x1, y1, x2, y2;
    float lx[5];
    float ly[5];
} rf_face;

/* Device/all-gather record: rf_face + the anchor's emission index (stride 32->16->8, anchor,
 * row-major position: the order of the reference's decode loop, RetinaFace.cpp:666-690).
 * 64 bytes. */
typedef struct rf_det {
    rf_face face;
    int32_t anchor_index;
} rf_det;

typedef struct rf_config {
    const char *caffemodel_path;   /* replaces buildTrtContext(prototxt, caffemodel), RetinaFace.cpp:276 */
    const char *int8_table_path;   /* TensorRT EntropyCalibration2 cache (trtnetbase.cpp:13) or NULL */
    int precision;                 /* rf_precision */
    int net_w, net_h;              /* network input size (prototxt line 7 in the reference); multiples of 32 */
    int max_batch;                 /* reference: maxBatchSize = 8 (trtretinafacenet.cpp:21) */
    int max_faces;                 /* per-image output capacity (faces kept after NMS); 0 -> 256 */
    int device;                    /* CUDA device ordinal */
    int max_image_w, max_image_h;  /* largest caller image (reference: 4096x3072, RetinaFace.cpp:325); 0 -> net size */
    unsigned flags;                /* RF_FLAG_* */
    int streams;                   /* execution contexts the asynchronous entry points rotate through so that
                                      consecutive batches overlap on the GPU; 0 -> RF_MAX_STREAMS (8).  The blocking
                                      rf_detect_batch always uses context 0.  1 selects the latency-oriented layer plan. */
    const char *prototxt_path;     /* optional: the Caffe prototxt of the model (buildTrtContext's first argument, RetinaFace.cpp:276).
                                      Parsed as protobuf text, checked to be the RetinaFace mnet25 graph, and its per-layer
                                      parameters (kernel, stride, group, bias_term, BatchNorm eps, ReLU) drive the weight folding;
                                      net_w / net_h == 0 take the input size from it (trtnetbase.cpp:163-187).  NULL: built-in graph. */
    const char *cache_path;        /* optional: file caching the folded model (the reference's engine cache, trtnetbase.cpp:205-243,
                                      which is never invalidated); reused only for the exact caffemodel (+ prototxt) bytes it was
                                      made from, rewritten otherwise.  NULL: no cache. */
    const char *network;           /* optional: the reference's network name (RetinaFace.cpp:205: "net3" default).  Names whose
                                      configuration the reference itself cannot run (net5, net6 ...: :266-268) or that need more
                                      anchors than the shipped models have (net3a) are refused with RF_ERR_UNSUPPORTED. */
} rf_config;

#define RF_FLAG_NO_GRAPH      0x1u  /* launch kernels directly instead of replaying a CUDA graph */
#define RF_FLAG_NO_TENSORCORE 0x2u  /* FP16: use the SIMT kernels for GEMM-shaped layers too (implies RF_FLAG_SIMT_STEM) */
#define RF_FLAG_SIMT_STEM     0x4u  /* FP16 / INT8: run all three layers of the stem on CUDA cores (FP32 conv0 weights) */
#define RF_FLAG_DW_1D         0x8u  /* FP16 / INT8: linear (1-D) tiles for every depthwise+pointwise layer, also on large maps */
#define RF_FLAG_NPP_RESIZE    0x20u /* letter-box with the reference's NPP branch semantics (USE_NPP: nppiResizeSqrPixel_8u_C3R,
                                       NPPI_INTER_SUPER, resizeconvertion.cu:279-316) -- coverage-weighted super-sampling, extent
                                       ceil(w f) x ceil(h f) -- instead of its OpenCV branch (cv::resize INTER_LINEAR, RetinaFace.cpp:613) */
#define RF_FLAG_LEGACY_TC     0x10u /* FP16: one tensor-core kernel per layer (pair) instead of the persistent tile chains
                                       (tile_chain.cuh) of a one-context handle; the cross-check of the chains */

typedef struct rf_handle_s *rf_handle;

/* Process-wide info, callable without a GPU. */
int rf_abi_version(void);
const char *rf_build_info(void);            /* arch flags etc. */
const char *rf_status_string(int status);

/* Replaces RetinaFace::RetinaFace's engine setup (RetinaFace.cpp:274-302): parses the
 * caffemodel, folds BatchNorm+Scale(+bias) in FP32, repacks weights, allocates device and
 * pinned memory, builds CUDA graphs lazily.  On failure *out = NULL and the message is
 * available from rf_last_error(NULL). */
int rf_create(const rf_config *cfg, rf_handle *out);
void rf_destroy(rf_handle h);
const char *rf_last_error(rf_handle h);     /* h may be NULL: last rf_create error */

/* Library-owned pinned staging for network-sized inputs: max_batch * net_h * net_w * 3 bytes.
 * Writing images here lets rf_detect_batch skip its host-side staging copy. */
uint8_t *rf_pinned_input(rf_handle h);
/* Library-owned DEVICE input buffer of the same shape: a caller that already has its images on
 * the GPU writes them here and passes this pointer to rf_detect_batch_device (no D2D copy). */
uint8_t *rf_device_input(rf_handle h);

/* Replaces RetinaFace::detect / detectBatchImages (RetinaFace.cpp:576-747, 749-940), end to
 * end: host u8 BGR HWC images (any size <= max_image; letter-boxed top-left into the network
 * size, never up-scaled) -> H2D -> network -> decode + threshold + NMS on the GPU -> D2H.
 * `row_strides` in bytes (NULL = packed).  Writes up to max_faces faces per image to
 * out_faces[i * max_faces ...] in descending score order and the count to out_counts[i].
 * out_anchor_index (optional, same layout) receives each face's anchor emission index.
 * Blocking: returns when the results are in the caller's arrays. */
int rf_detect_batch(rf_handle h, const uint8_t *const *bgr_images, const int *widths, const int *heights,
                    const int *row_strides, int n, float score_threshold, float nms_threshold,
                    rf_face *out_faces, int *out_counts, int32_t *out_anchor_index);

/* Pipelined end to end (throughput mode of the same path): rf_submit_batch queues H2D (on a copy
 * stream) + forward + D2H for one batch of NETWORK-SIZED images and returns at once with a ticket;
 * rf_collect_batch blocks until that batch's faces are in the caller's arrays.  Up to
 * RF_PIPELINE_DEPTH batches may be in flight, so the H2D copy of batch i+1 overlaps the kernels of
 * batch i (SURVEY.md 8f-1: host ingest).  Tickets must be collected in submission order.  Source
 * images may be pinned (copied in place) or pageable (staged through the library's pinned ring).
 * Every bgr_images[i] MUST point at net_h * net_w * 3 readable bytes (a packed network-sized image): there are no
 * width / height / stride arguments here -- other sizes go through rf_detect_batch. */
#define RF_MAX_STREAMS 8
#define RF_PIPELINE_DEPTH 6
int rf_submit_batch(rf_handle h, const uint8_t *const *bgr_images, int n, float score_threshold, float nms_threshold,
                    int *ticket);
int rf_collect_batch(rf_handle h, int ticket, rf_face *out_faces, int *out_counts, int32_t *out_anchor_index);

/* Device-resident variant: `dev_bgr` holds n network-sized u8 BGR HWC images (contiguous) in
 * device memory; results stay on the device: *dev_dets -> [max_batch][max_faces] rf_det,
 * *dev_counts -> [max_batch] int32 (kept count, clamped to max_faces).  Asynchronous on the
 * stream of the execution context the call landed on (rf_last_stream; rf_synchronize waits for all).
 * Consecutive calls rotate over the handle's execution contexts, each with its own output buffers: the
 * returned pointers stay valid until `streams` further calls.  This is the buffer a multi-GPU caller
 * all-gathers (SURVEY.md 8e). */
int rf_detect_batch_device(rf_handle h, const uint8_t *dev_bgr, int n, float score_threshold,
                           float nms_threshold, const rf_det **dev_dets, const int32_t **dev_counts);

/* f1 ingest, compressed: the reference decodes its test images on the host (cv::imread, main.cpp:18-26) and then copies
 * pixels; here the JPEG bitstreams are decoded ON the GPU (nvJPEG, opened at run time; hardware JPEG engines when the device
 * and the stream allow it, nvJPEG's hybrid back end otherwise) into the same device buffers the pixel path letter-boxes from,
 * so a camera-sized photo crosses PCIe as its compressed bytes.  jpegs[i] / jpeg_bytes[i]: host memory.  Images may have any
 * size up to max_image; out_widths / out_heights (optional) receive the decoded sizes (map-back: RetinaFace.cpp:732-738).
 * Results as rf_detect_batch.  RF_ERR_UNSUPPORTED when libnvjpeg is absent. */
int rf_detect_jpeg_batch(rf_handle h, const uint8_t *const *jpegs, const size_t *jpeg_bytes, int n, float score_threshold,
                         float nms_threshold, rf_face *out_faces, int *out_counts, int32_t *out_anchor_index, int *out_widths,
                         int *out_heights);
/* Decode only (parity / callers that want the pixels): BGR u8, packed rows, into out_bgr (host, out_capacity bytes);
 * out_bgr == NULL just reports the size.  rf_jpeg_backend: "hardware" | "default" | "none" (+ what the last call used). */
int rf_decode_jpeg(rf_handle h, const uint8_t *jpeg, size_t bytes, uint8_t *out_bgr, size_t out_capacity, int *width, int *height);
const char *rf_jpeg_backend(rf_handle h);

/* ---- Multi-GPU (SURVEY.md 8e; the reference is single-GPU: `ctx_id`, RetinaFace.h:89, is never used) --------------------
 * One process (handle) per GPU; the batch is sharded over the ranks, weights are replicated, and the ONLY exchange is an
 * all-gather of the per-image detection records -- fused into the NMS kernel: the CTA that finishes an image stores its kept
 * faces straight into the gather window of every rank (peer device memory over NVLink, mapped with CUDA IPC) and raises a
 * flag there.  Set-up: every rank calls rf_comm_export (allocates its window, fills an opaque 128-byte blob), the caller
 * all-gathers the blobs by any means (MPI, torch.distributed, a file ...), every rank calls rf_comm_init with all of them in
 * rank order.  rf_comm_init_nccl does the blob exchange itself through NCCL (libnccl.so.2 is opened at run time; the id
 * comes from rf_comm_nccl_unique_id on one rank and reaches the others by the caller's means).
 * All ranks must issue the same sequence of *_allgather calls with the same n. */
#define RF_COMM_BLOB_BYTES 128
#define RF_COMM_MAX_WORLD_SIZE 16
int rf_comm_export(rf_handle h, int rank, int world, void *blob);
int rf_comm_init(rf_handle h, const void *blobs /* world x RF_COMM_BLOB_BYTES, rank order */);
int rf_comm_nccl_unique_id(void *out128);
int rf_comm_init_nccl(rf_handle h, const void *nccl_unique_id /* 128 bytes */, int rank, int world);
int rf_comm_info(rf_handle h, int *rank, int *world);
/* rf_detect_batch_device + exchange: asynchronous; *all_dets -> [world][max_batch][max_faces] rf_det and *all_counts ->
 * [world][max_batch] int32 in this rank's gather window (rank r's image i at r * max_batch + i), complete -- every rank's
 * records have landed -- in stream order on rf_last_stream(); valid until 20 further exchanges. */
int rf_detect_batch_device_allgather(rf_handle h, const uint8_t *dev_bgr, int n, float score_threshold, float nms_threshold,
                                     const rf_det **all_dets, const int32_t **all_counts);
/* rf_submit_batch / rf_collect_batch + exchange: out_faces [world * max_batch][max_faces], out_counts [world * max_batch]
 * (host), rank r's image i at r * max_batch + i.  rf_detect_batch_allgather = submit + collect (blocking). */
int rf_submit_batch_allgather(rf_handle h, const uint8_t *const *bgr_images, int n, float score_threshold, float nms_threshold, int *ticket);
int rf_collect_batch_allgather(rf_handle h, int ticket, rf_face *out_faces, int *out_counts, int32_t *out_anchor_index);
int rf_detect_batch_allgather(rf_handle h, const uint8_t *const *bgr_images, int n, float score_threshold, float nms_threshold,
                              rf_face *out_faces, int *out_counts, int32_t *out_anchor_index);

/* Parity/debug: replaces TrtRetinaFaceNet::doInference + blob_by_name (trtretinafacenet.cpp:48-114).
 * Host network-sized images in, the 9 head blobs out in the reference's blob order
 * (trtretinafacenet.cpp:23-31), NCHW float32, each heads_out[k] sized n*C*h*w. */
int rf_forward_heads(rf_handle h, const uint8_t *bgr_net_sized, int n, float *const heads_out[9]);

/* Kernel-level parity: replaces the host decode loop + nms (RetinaFace.cpp:661-726, 439-492)
 * on caller-supplied head blobs (host, layout as rf_forward_heads).  Same outputs as
 * rf_detect_batch plus the pre-NMS candidate count per image (optional). */
int rf_postprocess(rf_handle h, const float *const heads[9], int n, float score_threshold,
                   float nms_threshold, rf_face *out_faces, int *out_counts, int32_t *out_anchor_index,
                   int *out_num_candidates);

/* Test-time augmentation + map-back (SURVEY.md 8f-2; the reference's `scales` parameter, RetinaFace.h:70, is unused and its
 * map-back is commented out, RetinaFace.cpp:730-746).  One image, `nviews` views of it (1..RF_MAX_VIEWS, <= max_batch): view v
 * is the image -- mirrored horizontally when views[v].flip -- letter-boxed into the top-left
 * floor(net_w*shrink) x floor(net_h*shrink) corner of the network input (shrink in (0, 1]; 1 = the plain detect view).
 * All views run as ONE batch; their detections are mapped back to ORIGINAL IMAGE pixels (x * scale_v, mirrored views
 * un-mirrored with left/right landmarks swapped) and merged by one more greedy NMS (same rule and threshold as per view)
 * across views, all on the GPU.  out_faces: [max_faces] in image coordinates; out_view_of (optional, [max_faces]): which view
 * each kept face came from; out_view_scales (optional, [nviews]): the map-back factor of each view.
 * views = {{1.0f, 0}} is detect + map-back. */
typedef struct rf_view {
    float shrink;
    int32_t flip;
} rf_view;
#define RF_MAX_VIEWS 16
int rf_detect_views(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_view *views, int nviews,
                    float score_threshold, float nms_threshold, rf_face *out_faces, int *out_count, int32_t *out_view_of,
                    float *out_view_scales);

/* f5 face alignment: detect, then cut one recognition-ready crop per kept face out of the ORIGINAL image, on the GPU.
 * For each face the least-squares similarity transform M (image -> crop; rotation, uniform scale, translation) from its five
 * landmarks to `template_xy` is fitted in FP64 (the minimiser of skimage's SimilarityTransform.estimate, which insightface's
 * norm_crop uses), and the image is warped into the crop bit for bit as
 * cv2.warpAffine(img, M, (crop_w, crop_h), INTER_LINEAR, BORDER_CONSTANT, 0) does.  Landmarks whose spread is zero give an
 * all-zero u8 crop and an all-zero M.  Crop layouts:
 *   RF_CROP_BGR_U8   crop_h x crop_w x 3 u8, HWC BGR (the warpAffine bytes)
 *   RF_CROP_RGB_F32  3 x crop_h x crop_w float32, planar RGB, (u8 - mean) * (1 / std)  (cv2.dnn.blobFromImages(crops, 1 / std,
 *                    size, (mean, mean, mean), swapRB = true): the input of an ArcFace recogniser)
 *   RF_CROP_RGB_F16  the same rounded to float16 */
#define RF_CROP_BGR_U8  0
#define RF_CROP_RGB_F32 1
#define RF_CROP_RGB_F16 2
typedef struct rf_align_params {
    int crop_w, crop_h;      /* 0, 0 -> 112 x 112; otherwise each in [8, 512] */
    float template_xy[10];   /* crop-pixel targets of the 5 landmarks (x0, y0 .. x4, y4); all 0 -> ArcFace 112x112 template */
    int max_faces;           /* crops per image, best score first; 0 -> every kept face (<= the handle's max_faces) */
    int format;              /* RF_CROP_BGR_U8 | RF_CROP_RGB_F32 | RF_CROP_RGB_F16 */
    float mean, std;         /* float formats; 0, 0 -> 127.5, 127.5 */
} rf_align_params;
/* Inputs as rf_detect_batch (any size up to max_image, row strides, pinned or pageable).  out_faces [n][max_faces] are in
 * ORIGINAL IMAGE pixels: every coordinate is rf_detect_batch's times the image's map-back scale, rounded to float.
 * With A = params->max_faces (or the handle's max_faces when 0): image i has crops j < min(out_counts[i], A) at
 * out_crops + (i * A + j) * crop bytes (host); later slots are not written.  out_mats (optional, host double [n][A][6]):
 * each crop's M, row-major 2 x 3.  Every image that is not network-sized needs its own raw device buffer while the crops
 * are cut: more of them in one call than the handle has (max_batch, capped at 2 GiB of max_image buffers) is
 * RF_ERR_CAPACITY.  Bad params: RF_ERR_INVALID_ARG.  Blocking. */
int rf_detect_align_batch(rf_handle h, const uint8_t *const *bgr_images, const int *widths, const int *heights,
                          const int *row_strides, int n, float score_threshold, float nms_threshold, const rf_align_params *params,
                          rf_face *out_faces, int *out_counts, void *out_crops, double *out_mats);
/* rf_detect_batch_device (network-sized device images, the same context rotation and outputs) followed by the crops of every
 * kept face, written into the caller's DEVICE buffer dev_crops [n][A][crop bytes] (e.g. a recogniser's input tensor) and,
 * optionally, dev_mats (device double [n][A][6]).  Asynchronous on rf_last_stream(). */
int rf_detect_align_batch_device(rf_handle h, const uint8_t *dev_bgr, int n, float score_threshold, float nms_threshold,
                                 const rf_align_params *params, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                                 const int32_t **dev_counts);

/* Preprocess parity: replaces imageROIResize8U3C + the OpenCV branch (RetinaFace.cpp:593-647):
 * letter-boxes one host image into a host net_h*net_w*3 u8 BGR buffer using the GPU kernel. */
int rf_preprocess(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, uint8_t *out_net_sized);

/* f6 video frames: detect (and align) on 8-bit YUV 4:2:0 frames -- NVDEC's NV12 surfaces, software decoders' I420, cameras' NV21
 * -- with the colour conversion fused into the letter-box kernel: each source tap is converted to BGR before the unchanged resize,
 * so the network input is byte for byte the letter-box of cv2.cvtColor(frame, COLOR_YUV2BGR_<layout>) (nearest chroma, OpenCV's
 * 20-bit fixed point), under either resize definition (RF_FLAG_NPP_RESIZE), and a crop is cv2.warpAffine(cvtColor(frame), M).
 * One descriptor covers all four layouts: NV12 = {y, u = uv, v = uv + 1, uv_step 2}, NV21 = {v = vu, u = vu + 1, uv_step 2},
 * I420 / YV12 = three planes, uv_step 1.  Chroma sample j of chroma row r is at u[r * uv_pitch + j * uv_step] (v likewise).
 * Invalid descriptors (size not positive and even, a NULL plane, uv_step not 1 or 2, semi-planar u and v not adjacent bytes,
 * y_pitch < width, uv_pitch < width / 2 * uv_step), an unknown matrix or bad align params: RF_ERR_INVALID_ARG; a frame larger
 * than max_image or n > max_batch: RF_ERR_CAPACITY; both before anything is launched. */
typedef struct rf_yuv_frame {
    const uint8_t *y, *u, *v;        /* plane origins */
    int y_pitch, uv_pitch, uv_step;  /* bytes; uv_step 2: semi-planar (NV12, NV21), 1: planar (I420, YV12) */
    int width, height;               /* even, <= max_image */
} rf_yuv_frame;
#define RF_YUV_BT601 0               /* == cv2.COLOR_YUV2BGR_{NV12,NV21,I420,YV12} */
#define RF_YUV_BT709 1               /* the same formula with round(c * 2^20) of the limited-range BT.709 matrix (NVDEC's HD output) */
/* Host frames (pinned or pageable): the planes are uploaded as they are, 1.5 bytes per pixel, into the raw buffers, letter-boxed
 * and detected on context 0; blocking.  out_faces [n][max_faces] / out_counts / out_anchor_index as rf_detect_batch, but in FRAME
 * pixels (rf_detect_align_batch's map-back).  align == NULL: no crops, frames are staged a chunk of raw buffers at a time.
 * Otherwise crops and matrices as rf_detect_align_batch (out_crops required, out_mats optional); every frame then needs its own
 * raw buffer while the crops are cut: more frames than the handle has is RF_ERR_CAPACITY. */
int rf_detect_yuv_batch(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, float score_threshold, float nms_threshold,
                        const rf_align_params *align, rf_face *out_faces, int *out_counts, int32_t *out_anchor_index, void *out_crops,
                        double *out_mats);
/* Device frames (frames: host array of descriptors of DEVICE planes), read in place and never written; the caller keeps them alive
 * until rf_last_stream() passes this call.  Asynchronous, rotating over the execution contexts like rf_detect_batch_device, each
 * context letter-boxing into an input tensor of its own; *dev_dets / *dev_counts as there (network-input pixels), out_scales
 * (host, [n]) receives each frame's map-back factor.  align != NULL: crops into dev_crops (required) and dev_mats (optional) as
 * rf_detect_align_batch_device. */
int rf_detect_yuv_batch_device(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, float score_threshold, float nms_threshold,
                               const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                               const int32_t **dev_counts, float *out_scales);
/* Preprocess parity of f6 (as rf_preprocess): one host frame letter-boxed into a host net_h*net_w*3 u8 BGR buffer. */
int rf_preprocess_yuv(rf_handle h, const rf_yuv_frame *frame, int matrix, uint8_t *out_net_sized);

/* f7 tiled detection: small faces in large images.  The letter-box of rf_detect_batch shrinks a 3840x2160 frame 8.6x on a 448x448
 * network, so a face narrower than ~137 pixels falls below the smallest anchor.  Here an image is resized to a pyramid of LEVELS,
 * each cv::resize(img, Size(), s, s, INTER_LINEAR) byte for byte (s may exceed 1; optionally of the mirrored image; at s = 0.5 that
 * is OpenCV's fast 2x INTER_AREA code, which cv::resize runs for INTER_LINEAR there), and every level is cut into
 * overlapping network-sized TILES that run as ordinary batches through the unchanged forward.  Detections are mapped back to image
 * pixels and merged across tiles and levels by one more greedy NMS (rf_detect_views' rule and threshold), all on the GPU.
 *
 * Geometry, per axis, with the level's size S = saturate_cast<int>(side * s) (round half to even), the tile size T (net_w or net_h)
 * and the overlap o:
 *   S <= T  one tile at origin 0, zeros beyond S, no shared sides;
 *   S >  T  k = ceil((S - o) / (T - o)) tiles at origins min(i (T - o), S - T): the last tile is flush with the far edge.
 * Each tile OWNS a half-open core: neighbours i, i + 1 split at floor((origin_i + origin_i+1 + T) / 2), the middle of the strip they
 * share; the first core starts at 0, the last ends at the far edge of the last tile (S on a tiled axis).  The cores partition the
 * level.  On an axis held by ONE tile nothing is filtered: that tile owns every detection along it, the zero padding beyond S
 * included (its core is reported as [0, T)), as rf_detect_batch keeps them.  Scale 0 is the FITTED level: exactly the
 * letter-box rf_detect_batch feeds the network (one tile, never up-scaled, the reference's float map-back factor).
 * Seams: a kept detection of a tile survives only if its centre (x1 + x2) * 0.5 (likewise y, in float) lies in the tile's core, and
 * it does not reach a SHARED side (x1 <= 0 on a shared left side, x2 >= net_w - 1 on a shared right one, likewise in y: the decode
 * clamps exactly there, so such a box was cut by the tile edge).  A face of side d < o at a level is therefore found whole by
 * exactly one tile; the default pyramid halves until the image fits, so every face is below o at some level until it is too small
 * to detect.  Survivors map back as image x = (x + origin) * map_back (mirrored levels then un-mirrored, landmarks swapped) and
 * join their image's candidate list with id tile * max_faces + rank, which is the tie order of the final NMS. */
typedef struct rf_tile_level {
    float scale;                   /* > 0: the level is the image resized by `scale`; 0: the fitted level */
    int32_t flip;                  /* non-zero: the level is of the horizontally mirrored image */
} rf_tile_level;
typedef struct rf_tiling {
    const rf_tile_level *levels;   /* NULL or nlevels == 0: the default pyramid -- levels 1, 1/2, 1/4, ... for as long as a level does
                                      not fit in one tile, then the fitted level (an image that fits gets the fitted level alone) */
    int nlevels;                   /* <= RF_MAX_TILE_LEVELS */
    int overlap;                   /* resized-image pixels neighbouring tiles share; 0 -> 64, else in [16, min(net_w, net_h) / 2] */
} rf_tiling;
typedef struct rf_tile {           /* one tile, in the order candidate ids are numbered: level by level, row-major within a level */
    int level, flip, scaled_w, scaled_h;          /* level index, mirrored, size of the resized level */
    int x0, y0;                                   /* tile origin in the level */
    int own_x0, own_y0, own_x1, own_y1;           /* ownership core in level pixels, half-open */
    int shared_sides;                             /* RF_TILE_SIDE_* bits */
    float scale, map_back;                        /* image pixel = (tile pixel + origin) * map_back, then un-mirrored */
} rf_tile;
#define RF_MAX_TILE_LEVELS 8
#define RF_MAX_TILES 256           /* per image, all levels */
#define RF_TILE_SIDE_LEFT   0x1
#define RF_TILE_SIDE_TOP    0x2
#define RF_TILE_SIDE_RIGHT  0x4
#define RF_TILE_SIDE_BOTTOM 0x8
/* Host-only (works without a GPU): the tiles of one width x height image on a net_w x net_h network (t may be NULL: the default
 * pyramid, overlap 64).  Returns the tile count and writes the first min(count, cap) tiles to out (out may be NULL when cap is 0),
 * or a status: RF_ERR_INVALID_ARG for a scale that is negative, NaN or infinite, whose resized side is 0 or exceeds 16384, an overlap
 * out of range, nlevels outside [0, RF_MAX_TILE_LEVELS] or bad sizes; RF_ERR_CAPACITY for more than RF_MAX_TILES tiles. */
int rf_tile_layout(int net_w, int net_h, int width, int height, const rf_tiling *t, rf_tile *out, int cap);
/* Host images as rf_detect_batch (any size up to max_image, pinned or pageable, row strides; at most max_batch per call); blocking.
 * out_faces [n][max_faces] in ORIGINAL IMAGE pixels, best first; out_counts [n]; out_tile_of (optional, [n][max_faces]): the tile
 * each kept face came from, an index into rf_tile_layout of its image.  Besides the statuses of rf_tile_layout: an image above
 * max_image is RF_ERR_CAPACITY, a handle created with RF_FLAG_NPP_RESIZE RF_ERR_UNSUPPORTED (NPPI_INTER_SUPER only down-samples;
 * levels are defined by cv::resize); all before anything is launched.
 * Execution contexts: the images are uploaded on context 0, a group of raw buffers at a time; their tiles are then letter-boxed,
 * detected and merged in chunks of up to max_batch tiles, each chunk on the next context of the rotation rf_detect_batch_device
 * uses (into that context's own input tensor), and the final NMS runs on context 0 once every context has finished.  Each chunk
 * counts as one call for the rule that rf_detect_batch_device's outputs stay valid for `streams` calls. */
int rf_detect_tiled(rf_handle h, const uint8_t *const *bgr_images, const int *widths, const int *heights, const int *row_strides,
                    int n, const rf_tiling *t, float score_threshold, float nms_threshold,
                    rf_face *out_faces, int *out_counts, int32_t *out_tile_of);
/* The same on host YUV 4:2:0 frames (rf_detect_yuv_batch's descriptors and checks): the tiles of cv2.cvtColor(frame). */
int rf_detect_yuv_tiled(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_tiling *t, float score_threshold,
                        float nms_threshold, rf_face *out_faces, int *out_counts, int32_t *out_tile_of);
/* Preprocess parity of rf_detect_yuv_tiled (as rf_preprocess_yuv): tile `tile` of one host frame's layout, converted and resized as
 * the network sees it, into a host net_h*net_w*3 u8 BGR buffer. */
int rf_preprocess_yuv_tile(rf_handle h, const rf_yuv_frame *frame, int matrix, const rf_tiling *t, int tile, uint8_t *out_net_sized);
/* Preprocess parity of f7 (as rf_preprocess): tile `tile` of one host image's layout, as the network sees it, into a host
 * net_h*net_w*3 u8 BGR buffer. */
int rf_preprocess_tile(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_tiling *t, int tile,
                       uint8_t *out_net_sized);

/* f8 small faces in device-resident frames, with crops: the tiled detection of f7 on images or NVDEC surfaces already on the GPU,
 * asynchronous, and the f5 crops of every kept face cut from the original image, so nothing leaves the GPU between the decoder and a
 * recogniser's input tensor.  Faces are those rf_detect_tiled / rf_detect_yuv_tiled return for the same pixels, bit for bit: in
 * ORIGINAL IMAGE (frame) pixels, best first.  Crops and matrices have the layout, formats, defaults and max_faces limit of
 * rf_detect_align_batch(_device); each M maps image to crop and is fitted on the returned landmarks (map-back factor 1), and a u8
 * crop is cv2.warpAffine(img, M, INTER_LINEAR, BORDER_CONSTANT) -- of cv2.cvtColor(frame) for YUV -- byte for byte.
 * Statuses as rf_detect_tiled / rf_detect_yuv_tiled (NULL arrays, empty images, a row stride below 3 w, bad frame descriptors,
 * rf_tile_layout's, an image above max_image, n > max_batch, RF_FLAG_NPP_RESIZE -> RF_ERR_UNSUPPORTED); bad align params, or align
 * without out_crops / dev_crops: RF_ERR_INVALID_ARG; all before anything is launched.
 *
 * Host, blocking: rf_detect_tiled / rf_detect_yuv_tiled plus the crops (align required; out_crops [n][A][crop bytes], out_mats
 * optional [n][A][6], host).  Every original stays resident in a raw buffer of its own until its crops are cut: more images than the
 * handle has raw buffers is RF_ERR_CAPACITY (rf_detect_yuv_batch's rule). */
int rf_detect_tiled_align(rf_handle h, const uint8_t *const *bgr_images, const int *widths, const int *heights, const int *row_strides,
                          int n, const rf_tiling *t, float score_threshold, float nms_threshold, const rf_align_params *align,
                          rf_face *out_faces, int *out_counts, int32_t *out_tile_of, void *out_crops, double *out_mats);
int rf_detect_yuv_tiled_align(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_tiling *t, float score_threshold,
                              float nms_threshold, const rf_align_params *align, rf_face *out_faces, int *out_counts,
                              int32_t *out_tile_of, void *out_crops, double *out_mats);
/* Device, asynchronous: dev_bgr[i] (u8 BGR rows row_strides[i] bytes apart; NULL or 0: packed) or the frames' planes are DEVICE
 * memory, read in place and never written; align may be NULL (no crops), else the crops go to dev_crops (required) and dev_mats
 * (optional), device memory.  *dev_dets -> [max_batch][max_faces] rf_det, *dev_counts -> [max_batch] int32 (kept count, clamped to
 * max_faces); anchor_index is the merge's candidate id, tile * max_faces + rank, so anchor_index / max_faces is the blocking paths'
 * out_tile_of.  Detections, counts, crops and matrices are complete in stream order on rf_last_stream(); the caller keeps the frames
 * alive and unmodified until that stream has passed the call.  The records live in a ring of `streams` output slots: the returned
 * pointers stay valid until `streams` further tiled device calls.  Tiles run in chunks over the rf_detect_batch_device rotation as
 * in rf_detect_tiled, each chunk counting as one call for that function's validity rule.  n = 0 launches nothing. */
int rf_detect_tiled_device(rf_handle h, const uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides,
                           int n, const rf_tiling *t, float score_threshold, float nms_threshold, const rf_align_params *align,
                           void *dev_crops, double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts);
int rf_detect_yuv_tiled_device(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_tiling *t, float score_threshold,
                               float nms_threshold, const rf_align_params *align, void *dev_crops, double *dev_mats,
                               const rf_det **dev_dets, const int32_t **dev_counts);

/* f9 rotated and mirrored images.  Orientation o in 1..8 is the EXIF tag: the DISPLAYED image is D = T_o(S), S the stored W x H
 * image and T_o the transform cv::imread applies (1 identity, 2 flip(1), 3 rotate 180, 4 flip(0), 5 transpose, 6 rotate 90
 * clockwise, 7 transpose + flip(-1), 8 rotate 90 counter-clockwise; 5..8 display H x W).  Displayed pixel (x, y) reads stored pixel
 *   1 (x, y)   2 (W-1-x, y)   3 (W-1-x, H-1-y)   4 (x, H-1-y)   5 (y, x)   6 (y, H-1-x)   7 (W-1-y, H-1-x)   8 (W-1-y, x)
 * and 2, 4, 5, 7 mirror.  The orientation moves integer tap addresses only -- tap positions, weights and rounding are those of the
 * displayed image -- so every letter-box (either resize definition) and crop byte is the one computed on T_o(S) (on
 * T_o(cvtColor(frame)) for YUV), and no rotated copy of the image is made.  Orientation 1 is the unoriented path.  An orientation
 * outside 1..8 is RF_ERR_INVALID_ARG, before anything is launched; every other argument is checked as by the unoriented twin.
 *
 * rf_detect_align_batch on T_o(img): host images (pinned or pageable), blocking; faces in DISPLAYED image pixels.  align == NULL: no
 * crops (out_crops / out_mats unused).  Otherwise crops and matrices as rf_detect_align_batch (M maps displayed image -> crop), with
 * its raw-buffer rule on the stored images: every image that is not a network-sized packed image in orientation 1 needs a raw
 * buffer of its own. */
int rf_detect_oriented_batch(rf_handle h, const uint8_t *const *bgr_images, const int *widths, const int *heights, const int *row_strides,
                             const int *orientations, int n, float score_threshold, float nms_threshold, const rf_align_params *align,
                             rf_face *out_faces, int *out_counts, int32_t *out_anchor_index, void *out_crops, double *out_mats);
/* rf_detect_yuv_batch_device on T_o(frame) (portrait NVDEC surfaces): the same context rotation, per-context input tensor and
 * validity rule; records in network-input pixels of the displayed frame, out_scales per displayed frame. */
int rf_detect_yuv_oriented_device(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n, int matrix, float score_threshold,
                                  float nms_threshold, const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                                  const int32_t **dev_counts, float *out_scales);
/* Preprocess parity (as rf_preprocess / rf_preprocess_yuv): the letter-box of T_o(img) / T_o(cvtColor(frame)). */
int rf_preprocess_oriented(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, int orientation, uint8_t *out_net_sized);
int rf_preprocess_yuv_oriented(rf_handle h, const rf_yuv_frame *frame, int matrix, int orientation, uint8_t *out_net_sized);
/* rf_detect_views with orientations: view v is T_{o_v}(img) letter-boxed into the shrunk box.  All views run as one batch, their
 * faces are mapped back to STORED image pixels (the table above, inverted; mirrored views swap left and right landmarks) and merged
 * by rf_detect_views' NMS.  {1, 6, 3, 8} at shrink 1 finds faces in any of the four rotations, and the landmarks, in stored pixels,
 * give f5 crops that come out upright.  Orientations 1 / 2 are rf_detect_views' flip 0 / 1, bit for bit. */
typedef struct rf_oriented_view {
    float shrink;
    int32_t orientation;
} rf_oriented_view;
int rf_detect_views_oriented(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_oriented_view *views, int nviews,
                             float score_threshold, float nms_threshold, rf_face *out_faces, int *out_count, int32_t *out_view_of,
                             float *out_view_scales);
/* Host-only (works without a GPU): the Exif orientation (tag 0x0112 of IFD0 in the first APP1 "Exif" segment, either TIFF byte order)
 * of a JPEG, 1..8; 1 when it is absent or malformed.  Never reads past `bytes`.  What cv::imread applies, for callers of
 * rf_decode_jpeg or their own decoder. */
int rf_jpeg_exif_orientation(const uint8_t *jpeg, size_t bytes);

/* f23 faces at any in-plane angle: rotated views.  View v shows the image (W x H, as stored) rotated counter-clockwise by
 * views[v].angle degrees -- the sign convention of cv2.getRotationMatrix2D -- fitted into the shrink box bw x bh of rf_detect_views
 * (bw = max(1, (int)(net_w * shrink)), likewise bh; shrink in (0, 1]).  In FP64, every operation rounded once (no FMA contraction):
 *   a = fmod(angle, 360), plus 360 when negative; a = 360 (a tiny negative angle) is 0.  A non-finite angle is RF_ERR_INVALID_ARG.
 *   a in {0, 90, 180, 270}: rf_detect_views_oriented's view (shrink, o) with o = 1, 8, 3, 6, bit for bit (letter-box, records and
 *   map-back).  Any other a is a WARP view:
 *     r = a * (M_PI / 180), c = cos(r), s = sin(r) (the C library's);  Wr = |c| * W + |s| * H,  Hr = |s| * W + |c| * H;
 *     f = min(1, bw / Wr, bh / Hr) (never up-scaled, like the letter-box);
 *     M = [[f * c, f * s, tx], [-(f * s), f * c, ty]] with
 *       tx = (f * Wr - 1) / 2 - (M00 * ((W - 1) / 2) + M01 * ((H - 1) / 2)),  ty = (f * Hr - 1) / 2 - (M10 * ((W - 1) / 2) + M11 * ((H - 1) / 2)),
 *     so the image centre lands on the centre of the rotated image's f Wr x f Hr bounding box, which sits at the input's top-left.
 *     The network input is cv2.warpAffine(img, M, (net_w, net_h), INTER_LINEAR, BORDER_CONSTANT, 0) byte for byte: zero outside the
 *     rotated image, like the letter-box padding.
 *     A kept face of a warp view maps back through iM = cv::invertAffineTransform(M): its box centre ((x1 + x2) / 2, (y1 + y2) / 2)
 *     goes through iM, the half sizes are (x2 - x1) * (1 / (2 f)) and (y2 - y1) * (1 / (2 f)), and the box is centre -/+ half size,
 *     each rounded to float once -- axis-aligned in image pixels, with the face's own size; the face's roll is the view's angle
 *     (out_view_of).  Each landmark is iM (lx, ly), rounded to float; a rotation does not mirror, so landmark sides are kept.
 * The faces of all views are merged by rf_detect_views' NMS, candidate id v * max_faces + rank.  Landmarks in image pixels carry the
 * face's roll, so f5 crops fitted on them come out upright. */
typedef struct rf_rotated_view {
    float angle;     /* degrees, counter-clockwise */
    float shrink;    /* (0, 1] */
} rf_rotated_view;
/* One host image (pinned or pageable, row_stride 0: packed), 1..RF_MAX_VIEWS views (else RF_ERR_CAPACITY); views beyond max_batch run
 * in consecutive batches on context 0.  Blocking.  out_faces [max_faces] in image pixels, *out_count; out_view_of (optional,
 * [max_faces]) the view of each face; out_view_scales (optional, [nviews]) the oriented views' map-back factor and (float)(1 / f) for
 * warp views; out_view_mats (optional, [nviews][6]) M of each warp view, all zero for the views that take the oriented path.
 * align != NULL: the crops of the merged faces, cut from the original image, in rf_detect_align_batch's layout for one image
 * (out_crops [A][crop bytes] required, out_mats [A][6] optional).  A non-finite angle, a shrink outside (0, 1], NULL views or bad align
 * params: RF_ERR_INVALID_ARG; the image is checked as by rf_detect_views; all before anything is launched or written. */
int rf_detect_views_rotated(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, const rf_rotated_view *views, int nviews,
                            float score_threshold, float nms_threshold, const rf_align_params *align, rf_face *out_faces, int *out_count,
                            int32_t *out_view_of, float *out_view_scales, double *out_view_mats, void *out_crops, double *out_mats);
/* Preprocess parity of f23 (as rf_preprocess): the network input of the view (angle, shrink) of one host image, either kind, into a
 * host net_h*net_w*3 u8 BGR buffer, and (out_mat optional, [6]) its M, all zero for a quarter turn. */
int rf_preprocess_rotated(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, float angle, float shrink,
                          uint8_t *out_net_sized, double *out_mat);

/* f24 faces at any in-plane angle in device frames and video: f23's rotated views of device BGR images or NVDEC surfaces, n frames a
 * call.  For each frame i the call returns exactly what rf_detect_views_rotated returns for that frame's pixels (for YUV,
 * cv2.cvtColor(frame)) with the same views, bit for bit: records, kept count, the view of each face (anchor_index / max_faces, the
 * candidate id v * max_faces + rank), crops and matrices.  A YUV warp view is cv2.warpAffine(cvtColor(frame), M) byte for byte (each
 * tap converted as f6's letter-box converts it) and a YUV crop is f6's crop.  RF_FLAG_NPP_RESIZE changes only the quarter turns'
 * letter-boxes, as in f23.
 * The call is rf_detect_tiled_device / rf_detect_yuv_tiled_device (f8) with views in place of tiles: the same views apply to all
 * n <= max_batch frames (more: RF_ERR_CAPACITY), frames are DEVICE memory read in place and never written, and the n * nviews network
 * inputs run in chunks of max_batch over the rf_detect_batch_device rotation, each chunk counting as one call for that function's
 * validity rule.  The final per-frame NMS and the crops run on the home stream, which rf_last_stream() returns.  *dev_dets ->
 * [max_batch][max_faces] rf_det in FRAME pixels, *dev_dets / *dev_counts complete in stream order there; with scales NULL they feed
 * rf_track_update, rf_redact_yuv_device_style and rf_redact_device_style.  The records live in a ring of `streams` output slots of
 * their own: the returned pointers stay valid for `streams` further rotated device calls, and tiled device calls keep their own ring.
 * out_view_scales (optional, host, [n][nviews]) and out_view_mats (optional, host, [n][nviews][6]) hold f23's values per frame -- a
 * quarter turn's map-back factor and zero M, a warp view's (float)(1 / f) and M -- filled before return.  align != NULL: crops into
 * dev_crops (required) and dev_mats (optional) as rf_detect_tiled_device's.  Checks, in this order and all before anything is launched
 * or written: the frames as by the f8 twin (n included), views NULL (RF_ERR_INVALID_ARG), 1..RF_MAX_VIEWS views (else
 * RF_ERR_CAPACITY), each view as by rf_detect_views_rotated, then the align params (align without dev_crops: RF_ERR_INVALID_ARG).
 * n = 0 launches nothing. */
int rf_detect_views_rotated_device(rf_handle h, const uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides,
                                   int n, const rf_rotated_view *views, int nviews, float score_threshold, float nms_threshold,
                                   const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                                   const int32_t **dev_counts, float *out_view_scales, double *out_view_mats);
int rf_detect_yuv_views_rotated_device(rf_handle h, const rf_yuv_frame *frames, int n, int matrix, const rf_rotated_view *views, int nviews,
                                       float score_threshold, float nms_threshold, const rf_align_params *align, void *dev_crops,
                                       double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts, float *out_view_scales,
                                       double *out_view_mats);
/* Preprocess parity of f24 (as rf_preprocess_rotated): the network input of the view (angle, shrink) of one HOST 4:2:0 frame, i.e.
 * of cv2.cvtColor(frame), into a host net_h*net_w*3 u8 BGR buffer, and (out_mat optional, [6]) its M, all zero for a quarter turn. */
int rf_preprocess_yuv_rotated(rf_handle h, const rf_yuv_frame *frame, int matrix, float angle, float shrink, uint8_t *out_net_sized,
                              double *out_mat);
/* The records of a device detect call (*dev_dets / *dev_counts of n <= max_batch images, while they are valid) on the host, for callers
 * without a CUDA runtime of their own such as the C++ shell.  Blocking: waits for every execution context, then copies them into
 * out_faces [n][max_faces] / out_counts [n] and, optional, their anchor_index into out_anchor_index [n][max_faces], rf_detect_batch's
 * layout.  n = 0 copies nothing. */
int rf_fetch_dets(rf_handle h, const rf_det *dev_dets, const int32_t *dev_counts, int n, rf_face *out_faces, int *out_counts,
                  int32_t *out_anchor_index);

/* f10 face tracking across video frames, on the GPU: per-video tracks with stable ids, so that a recogniser runs once per new
 * identity instead of once per face per frame, and counting / dwell time / "who entered" need no host round trip.  One tracker holds
 * max_videos independent sequences (cameras, files), each with up to max_tracks live tracks (tentative, confirmed and lost).
 *
 * Definition: ByteTrack's association (Zhang et al., 2022) with SORT's constant-velocity Kalman filter, in FP64, stated exactly so
 * that a scalar restatement reproduces every bit.  Per track and per coordinate c of (cx, cy, a = w / h, h): position m, velocity u and
 * a 2 x 2 covariance (P00, P01, P11) -- ByteTrack's 8 x 8 filter, which decouples into these four scalar filters.  With h the track's
 * current height m_h, sp = 1 / 20 and sv = 1 / 160:
 *   predict  (a LOST track first has u_h = 0) q_pos = sp * h (1e-2 for a), q_vel = sv * h (1e-5 for a);
 *            P00 = ((P00 + P01) + (P01 + P11)) + q_pos * q_pos, P01 = P01 + P11, P11 = P11 + q_vel * q_vel, m = m + u
 *   update   r = sp * h (1e-1 for a), S = P00 + r * r, K0 = P00 / S, K1 = P01 / S, y = z - m, m += K0 * y, u += K1 * y,
 *            P00 -= (K0 * S) * K0, P01 -= (K0 * S) * K1, P11 -= (K1 * S) * K1   (q and r use h before the step)
 *   birth    m = z, u = 0, P00 = ((2 * sp) * h)^2 (1e-2^2 for a), P11 = ((10 * sv) * h)^2 (1e-5^2 for a), P01 = 0
 *   z        from a record's float box in frame pixels, widened to double: w = x2 - x1, h = y2 - y1, cx = x1 + w / 2, cy = y1 + h / 2
 *            (records with w <= 0 or h <= 0 are ignored)
 *   box      of a mean: w = a * h, x1 = cx - w / 2, y1 = cy - h / 2, x2 = x1 + w, y2 = y1 + h
 * The match score is the IoU, in FP64, of a track's predicted box and a record's box with the reference NMS's +1 pixel convention.
 * Per frame of a video, after predicting every live track, with the frame's records (best score first; index = record index):
 *   1. records with score >= high_thresh are HIGH, the others LOW;
 *   2. CONFIRMED and LOST tracks against HIGH records, matched when IoU > iou_high;
 *   3. tracks CONFIRMED at frame start and still unmatched against LOW records, IoU > iou_low;
 *   4. TENTATIVE tracks against the remaining HIGH records, IoU > iou_tentative; an unmatched TENTATIVE track is removed;
 *   5. matched tracks: Kalman update, hits + 1, lost_frames = 0, the record's face kept; LOST and TENTATIVE ones become CONFIRMED
 *      (a LOST one keeps its id);
 *   6. unmatched CONFIRMED tracks become LOST (lost_frames = 1), unmatched LOST ones count lost_frames + 1; a LOST track is removed
 *      when lost_frames exceeds max_lost;
 *   7. each remaining HIGH record with score >= new_thresh, in record order, starts a track with the video's next id (ids start at 1
 *      and are not reused before a reset), TENTATIVE -- CONFIRMED on the video's first frame since create or reset.  Without a free
 *      slot the birth is skipped and the video's overflow counter (rf_tracker_debug_state) counts it.
 * Each stage is greedy by descending IoU: the highest-IoU pair whose track and record are both free is matched, and so on; ties go
 * to the lower track id, then the lower record index.  This equals ByteTrack's optimal assignment whenever no track has two
 * candidates above the threshold (the usual case for faces, which NMS keeps apart), and is deterministic.  ByteTrack's score fusion
 * and duplicate-track removal are not part of it.  age counts the frames since birth, the birth frame included. */
typedef struct rf_tracker_s *rf_tracker;
typedef struct rf_track_config {
    int max_videos;                 /* 1..4096 */
    int max_tracks;                 /* per video, LOST included; 0 -> 64, at most 1024 */
    float high_thresh, new_thresh;  /* 0 -> 0.6, 0.7; else in (0, 1] */
    float iou_high, iou_low, iou_tentative;   /* 0 -> 0.2, 0.5, 0.3; else in (0, 1] */
    int max_lost;                   /* frames; 0 -> 30 */
} rf_track_config;
#define RF_TRACK_TENTATIVE 0
#define RF_TRACK_CONFIRMED 1
#define RF_TRACK_LOST      2
typedef struct rf_track {
    int32_t id, state;              /* per-video id; RF_TRACK_* */
    int32_t det;                    /* index of the record matched on this frame, -1 */
    int32_t crop_slot;              /* this frame's crop j of the track, -1 */
    int32_t hits, age, lost_frames;
    int32_t followed;               /* f16: 1 when the track was moved by template search on this frame, else 0 */
    float kx1, ky1, kx2, ky2;       /* filtered box (mean after this frame), frame pixels */
    float vx, vy;                   /* centre velocity, pixels per frame */
    rf_face face;                   /* last matched detection, frame pixels */
} rf_track;
/* Creates a tracker on the handle's device (state of every video zeroed).  Bad config: RF_ERR_INVALID_ARG. */
int  rf_tracker_create(rf_handle h, const rf_track_config *cfg, rf_tracker *out);
void rf_tracker_destroy(rf_tracker t);                 /* before rf_destroy of its handle; waits for the tracker's work */
/* Restarts one video (ids from 1, first-frame rule) or all (-1).  Asynchronous, ordered after every update issued before it. */
int  rf_tracker_reset(rf_tracker t, int video);
/* Applies n frames of device records to the tracker: the records of any device detect call on the handle (rf_detect_batch_device,
 * rf_detect_yuv_batch_device, the oriented and tiled device calls, the all-gather call), laid out [n][max_faces] as they return them,
 * kept counts dev_counts [n].  Frame i belongs to video videos[i]; a video may appear more than once, its frames then apply in call
 * order.  Coordinates map to frame pixels as __fmul_rn(x, scales[i]) (f5's map-back); scales == NULL means 1 (tiled records, already
 * in image pixels).  Asynchronous, issued on rf_last_stream(), where the records complete; updates are ordered among themselves
 * whatever context they land on (an event chain), forwards still overlap.  *dev_tracks -> [n][max_tracks] rf_track: frame i's list
 * holds every live track after that frame, sorted by id, *dev_track_counts -> [n] int32 its length; crop_slot is -1.  The outputs live
 * in a ring of `streams` slots and stay valid for `streams` further tracker calls.  n = 0 launches nothing.  A video outside
 * [0, max_videos), n > max_batch (RF_ERR_CAPACITY), NULL arrays, a non-finite or non-positive scale: an error status before anything
 * is launched. */
int  rf_track_update(rf_tracker t, const int *videos, int n, const rf_det *dev_dets, const int32_t *dev_counts,
                     const float *scales, const rf_track **dev_tracks, const int32_t **dev_track_counts);
/* rf_detect_yuv_batch_device (same context rotation; *dev_dets, *dev_counts and out_scales as there), then rf_track_update of its
 * records on the same context.  align != NULL: crops only for the tracks that became CONFIRMED on this frame -- new identities, not
 * LOST tracks found again -- compacted per frame in id order into dev_crops [n][A][crop bytes] (A and formats as
 * rf_detect_align_batch_device; dev_mats optional [n][A][6]); each such track's crop_slot says where its crop is, and crops beyond A
 * are not cut (crop_slot -1).  A crop is the one rf_detect_yuv_batch_device cuts for the matched record, byte for byte.  Statuses of
 * both calls, before anything is launched. */
int  rf_detect_yuv_track_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix,
                                float score_threshold, float nms_threshold, const rf_align_params *align, void *dev_crops,
                                double *dev_mats, const rf_track **dev_tracks, const int32_t **dev_track_counts,
                                const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales);
/* Parity aid, blocking (waits for every issued update): video's FP64 state into out (cap doubles).  out[0..3] = live tracks, next id,
 * frames since reset, births skipped for want of a slot; then per live track in id order RF_TRACK_DEBUG_DOUBLES values: id, state,
 * hits, age, lost_frames, m[4], u[4], P00[4], P01[4], P11[4] (coordinates cx, cy, a, h).  Returns the live track count. */
#define RF_TRACK_DEBUG_DOUBLES 25
int  rf_tracker_debug_state(rf_tracker t, int video, double *out, int cap);

/* f13 camera-motion compensation: a tracker that has the frames estimates each frame's global motion from the previous frame of
 * the same video and moves every track with it before association, so that a pan, a shake or a zoom does not break the ids (BoT-SORT's
 * global motion compensation, here deterministic and on the GPU).  Per frame the estimate is a similarity in frame pixels from the
 * previous frame to this one, x' = a x - b y + tx, y' = b x + a y + ty, computed from luma alone (NV12, NV21, I420 and YV12 give the
 * same result), every FP64 step one rounding in the order written (oracle/motion.py restates it):
 *   1. thumbnail  D = ceil(max(W, H) / RF_MOTION_THUMB); tw = W / D, th = H / D (a partial last row / column of boxes is dropped);
 *                 thumb(x, y) = (sum of the D x D luma box at (D x, D y) + D*D / 2) / (D*D), integers.
 *   2. blocks     RF_MOTION_BLOCK-square blocks at (R + 16 i, R + 16 j) for every block that fits inside the thumbnail inset by the
 *                 search radius R, numbered row by row.  A block is skipped when 256 sum(p^2) - (sum p)^2 < RF_MOTION_MIN_VAR * 65536
 *                 (flat: walls, sky), or when it overlaps a record of this frame: the record's box (x1..y2 = __fmul_rn(coordinate,
 *                 scale), widened to double; w = x2 - x1, h = y2 - y1) grown by RF_MOTION_FACE_MARGIN * w (h) on each side, against
 *                 the block's frame rectangle [D x0, D (x0 + 16)) x [D y0, D (y0 + 16)): gx1 < X1 && gx2 > X0 && gy1 < Y1 && gy2 > Y0.
 *   3. match      SAD(dy, dx) = sum |cur(x0 + c, y0 + r) - ref(x0 + dx + c, y0 + dy + r)| over |dx|, |dy| <= R; the minimum under
 *                 the order (SAD, |dy| + |dx|, dy, dx).  The block is dropped when another offset has the same SAD or the minimum lies
 *                 on the search border.  Sub-pixel: f = (S(-1) - S(+1)) / (2 (S(-1) - 2 S(0) + S(+1))) per axis (integers, one
 *                 division).  The block gives the point pair p = (x0 + 7.5, y0 + 7.5) in this frame and q = ((px + dx) + fx,
 *                 (py + dy) + fy) in the previous one.
 *   4. fit        N kept blocks in block order (N < min_inliers: LOST).  Hypotheses h in [0, N + N / 2): h < N the translation
 *                 p_h - q_h of block h alone; h = N + k the exact similarity of blocks k and k + N / 2: dq = q2 - q1, dp = p2 - p1,
 *                 den = dqx dqx + dqy dqy (0: no inliers), a = (dpx dqx + dpy dqy) / den, b = (dpy dqx - dpx dqy) / den,
 *                 tx = px1 - (a qx1 - b qy1), ty = py1 - (b qx1 + a qy1).  Point k is an inlier of (a, b, tx, ty) when
 *                 ex = ((a qx - b qy) + tx) - px, ey = ((b qx + a qy) + ty) - py have ex ex + ey ey <= RF_MOTION_TOL^2.  The
 *                 hypothesis with the most inliers wins, ties to the lower h.  Its inliers (fewer than min_inliers: LOST) are refitted
 *                 by least squares, the centred closed form of the align fit: means m = S(v) / n, u = q - mq, v = p - mp,
 *                 den = S(ux ux + uy uy) (0: LOST), a = S(ux vx + uy vy) / den, b = S(ux vy - uy vx) / den, tx = (mpx - a mqx) + b mqy,
 *                 ty = (mpy - b mqx) - a mqy; then the inliers of that fit are selected once more (fewer than min_inliers: LOST) and
 *                 refitted once more.  S sums in 32 lanes -- lane l adds the terms l, l + 32, ... of the inlier list in order -- then
 *                 lane l += lane l + o for o = 16, 8, 4, 2, 1; the result is lane 0.
 *   5. frame      c = (D - 1) / 2: a and b stay, tx' = ((D tx) + c) - ((a c) - (b c)), ty' = ((D ty) + c) - ((b c) + (a c)).
 *   6. status     RF_MOTION_FIRST: no reference (the first frame since create / reset, or the frame size changed);
 *                 RF_MOTION_LOST: too few blocks or inliers, a degenerate fit, or s = sqrt(a a + b b) outside
 *                 [RF_MOTION_MIN_SCALE, RF_MOTION_MAX_SCALE] (scene cuts, flat frames); RF_MOTION_OK otherwise.  FIRST and LOST
 *                 report the identity and move nothing.
 * Compensation, after predict and before the first association stage, on every live track of an RF_MOTION_OK frame, with
 * s = sqrt(a a + b b) and ss = s * s:  cx = ((a cx) - (b cy)) + tx;  cy = ((b cx) + (a cy)) + ty  (old cx, cy on the right);
 * u_cx, u_cy likewise without t;  h = s h;  u_h = s u_h;  a and u_a stay;  P00, P01, P11 = ss * P for cx, cy and h.  This is
 * A8 P A8^T of ByteTrack's 8 x 8 filter exactly: the cx and cy filters are born with the same covariance and take the same steps,
 * so their covariances are equal bit for bit and a rotation keeps the four scalar filters decoupled.  After compensation rf_track.vx
 * and .vy are the face's motion relative to the scene, not to the frame. */
#define RF_MOTION_OK    0
#define RF_MOTION_FIRST 1
#define RF_MOTION_LOST  2
#define RF_MOTION_THUMB 320              /* the thumbnail's longer side is at most this */
#define RF_MOTION_BLOCK 16
#define RF_MOTION_MIN_VAR 16             /* texture floor: the block's luma variance, thumbnail levels squared */
#define RF_MOTION_FACE_MARGIN 0.5        /* records grow by this fraction of their size on each side */
#define RF_MOTION_TOL 1.0                /* inlier distance, thumbnail pixels */
#define RF_MOTION_MIN_SCALE 0.8
#define RF_MOTION_MAX_SCALE 1.25
typedef struct rf_motion_config {
    int search;                      /* R, thumbnail pixels: 0 -> 12 (about 72 frame pixels per frame at 1080p), else 1..32 */
    int min_inliers;                 /* 0 -> 12, else 3..361 */
} rf_motion_config;
typedef struct rf_motion {
    int32_t status;                  /* RF_MOTION_* */
    int32_t blocks, inliers, reserved;   /* blocks kept (step 4's N), inliers of the last selection */
    double m[6];                     /* {a, -b, tx, b, a, ty}, frame pixels, previous frame -> this one (the align matrices' layout) */
} rf_motion;
/* Turns motion compensation on for a plain or best-shot tracker, before its first update (afterwards, or a bad config:
 * RF_ERR_INVALID_ARG).  Allocates a reference store of max_videos thumbnails of RF_MOTION_THUMB^2 bytes (above 4 GiB:
 * RF_ERR_CAPACITY).  The frames are then estimated by rf_detect_yuv_track_device, rf_detect_yuv_track_best_device and
 * rf_detect_yuv_redact_device, on the forward's context inside the tracker's event chain: thumbnails, match, fit, the update, then
 * each video's last thumbnail of the call becomes its reference.  Frame k of a video is matched against that video's previous
 * frame of the same call, the first one against the reference.  rf_track_update, which has no pixels, refuses a motion tracker;
 * rf_tracker_reset and rf_tracker_finish drop the video's reference. */
int rf_tracker_set_motion(rf_tracker t, const rf_motion_config *cfg);
/* *dev_motion -> the [n] rf_motion of the tracker's latest frame call (NULL before the first), in the ring slot of its track lists:
 * valid for `streams` further tracker calls.  RF_ERR_INVALID_ARG on a tracker without motion. */
int rf_tracker_motion(rf_tracker t, const rf_motion **dev_motion);

/* f11 best shots: the best crop of every tracked face, kept on the GPU, and one crop per identity when its track ends -- the view a
 * recogniser should see, instead of the track's second detection (f10's new-identity crop), which is usually a face entering the
 * frame: at its edge, small, turned or blurred.
 *
 * A BEST-SHOT tracker is created by rf_tracker_create_best and fed only through rf_detect_yuv_track_best_device, which has the frame
 * pixels.  Tracking is f10's, unchanged: the same rf_track lists, bit for bit.  On every frame where a track is matched or born (its
 * rf_track.det >= 0 after the frame, TENTATIVE frames included), the call
 *   1. cuts the u8 BGR crop rf_detect_yuv_track_device would cut for the track's record: M fitted on rf_track.face (frame pixels,
 *      map-back 1) to the template, cv2.warpAffine(cv2.cvtColor(frame), M) byte for byte;
 *   2. computes the crop's quality q (below);
 *   3. keeps the crop, M, the quality terms, the record and the frame number if q is STRICTLY greater than the track's stored best;
 *      a track's first frame always stores, and on a tie the earlier frame stays.
 * A track that was ever CONFIRMED EMITS its best shot on the frame it is removed (a LOST track whose lost_frames exceeds max_lost);
 * a TENTATIVE track that is removed never emits; a shot whose stored q < min_quality is dropped.  A frame's emissions are compacted
 * in id order.  Within a video, a frame applies its removals (and their emissions) before its births, as f10 orders them, so a
 * slot freed and reused on one frame emits the old track's shot.  rf_tracker_finish(video) emits the best shot of every live,
 * ever-confirmed track of the video in id order, with the same filter, then resets the video as rf_tracker_reset does;
 * rf_tracker_reset on a best-shot tracker discards the stored shots and emits nothing.
 *
 * Quality.  Every step FP64, one rounding each, in the order written; landmarks l_k are the record's floats in frame pixels, widened:
 *   ex = lx1 - lx0, ey = ly1 - ly0, d2 = ex * ex + ey * ey   (d2 == 0 or M all zero: eye, frontal, sharpness, coverage and q are 0)
 *   eye       = sqrt(d2)
 *   t         = ((lx2 - (lx0 + lx1) / 2) * ex + (ly2 - (ly0 + ly1) / 2) * ey) / d2     (the nose's offset along the eye axis)
 *   frontal   = max(0, 1 - 2 * |t|)
 *   size      = min(1, eye / eye_ref)     eye_ref = the distance of template points 0 and 1 (35.24 px for the ArcFace 112 template)
 *   INSIDE    a crop pixel whose four cv::warpAffine taps (sx, sy) .. (sx + 1, sy + 1) (the fixed-point tap, after its saturate) all
 *             lie in the frame
 *   coverage  = #INSIDE / (crop_w * crop_h)
 *   g         = (3735 B + 19235 G + 9798 R + 16384) >> 15 per crop pixel   (cv2.cvtColor BGR2GRAY)
 *   L(x, y)   = g(x-1, y) + g(x+1, y) + g(x, y-1) + g(x, y+1) - 4 g(x, y)    (cv2.Laplacian(g, ksize = 1) in the interior), over
 *             1 <= x <= crop_w - 2, 1 <= y <= crop_h - 2 where (x, y) and its 4 neighbours are INSIDE: count N, S1 = sum L,
 *             S2 = sum L^2 in int64
 *   sharpness = N >= 2 ? (double)(N S2 - S1 S1) / ((double)N * (double)N) : 0      (the Laplacian's variance)
 *   sharp     = sharpness / (sharpness + sharp_half)
 *   q         = (((score * frontal) * size) * sharp) * coverage
 *
 * Outputs follow f10's rules: records and counts live in the tracker's ring of `streams` slots and stay valid for `streams` further
 * tracker calls.  *dev_best -> [n][max_tracks] rf_best_shot, frame i's emissions in id order, *dev_best_counts -> [n] int32; emission k
 * of frame i has its crop at dev_best_crops [i][k] ([n][max_tracks][crop bytes], the caller's device buffer) and, optionally, its M at
 * dev_best_mats [i][k] ([n][max_tracks][6]).  The bound is exact: the tracks removed on a frame were live.  For rf_tracker_finish
 * the buffers hold [max_tracks].  Float formats are the u8 crop converted as rf_detect_align_batch_device converts it, bit for bit.
 * Calls are asynchronous on rf_last_stream() (rf_tracker_finish: context 0's stream), ordered with every other call on the tracker
 * by its event chain. */
typedef struct rf_best_config {
    rf_align_params align;   /* geometry, template, format, mean / std of the EMITTED crops (max_faces must be 0); stored as u8 */
    float min_quality;       /* in [0, 1]; a shot is emitted only if q >= min_quality */
    float sharp_half;        /* 0 -> 50; else finite and > 0 */
} rf_best_config;
#define RF_BEST_EXIT   0     /* the track was removed */
#define RF_BEST_FINISH 1     /* rf_tracker_finish */
typedef struct rf_best_shot {
    int32_t id, video;
    int32_t frame;           /* the video's frame number (0: the first since create / reset) the crop was cut from */
    int32_t end_frame;       /* the frame number it was emitted on (rf_tracker_finish: the video's last frame) */
    int32_t hits, age, reason, reserved;   /* the track's hits / age when emitted; RF_BEST_* */
    float quality, score, eye, frontal, sharpness, coverage;   /* q and its terms at `frame`, rounded from double */
    rf_face face;            /* the track's record on `frame`, frame pixels */
} rf_best_shot;
/* A best-shot tracker.  Bad configs: RF_ERR_INVALID_ARG; a store (max_videos x max_tracks u8 crops) above 4 GiB: RF_ERR_CAPACITY. */
int rf_tracker_create_best(rf_handle h, const rf_track_config *cfg, const rf_best_config *best, rf_tracker *out);
/* rf_detect_yuv_track_device without new-identity crops, plus the best shots above (dev_best_crops required).  RF_ERR_INVALID_ARG
 * on a plain tracker; every status before anything is launched.  rf_detect_yuv_track_device and rf_track_update refuse a best-shot
 * tracker (RF_ERR_INVALID_ARG): frames the store never saw would break "the best of every frame". */
int rf_detect_yuv_track_best_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix,
                                    float score_threshold, float nms_threshold, void *dev_best_crops, double *dev_best_mats,
                                    const rf_best_shot **dev_best, const int32_t **dev_best_counts,
                                    const rf_track **dev_tracks, const int32_t **dev_track_counts,
                                    const rf_det **dev_dets, const int32_t **dev_counts, float *out_scales);
/* Ends `video` (see above).  *dev_best -> [max_tracks] rf_best_shot, *dev_best_count -> one int32. */
int rf_tracker_finish(rf_tracker t, int video, void *dev_best_crops, double *dev_best_mats,
                      const rf_best_shot **dev_best, const int32_t **dev_best_count);

/* f22 best shots for live cameras.  A live stream has no end, so f11's shot -- emitted when the track ends -- comes too late for
 * access control or a watch list; and f11 needs every frame detected.  Two options of a best-shot tracker, each set before its first
 * frame call, in either order and with rf_tracker_set_motion, rf_tracker_set_tiling and rf_tracker_set_orientation.
 *
 * LIVE shots (rf_tracker_set_best_live).  Per frame of a video, after f11's removals and store updates, every track that is CONFIRMED
 * after the frame and matched on it (rf_track.det >= 0; a track born CONFIRMED on a video's first frame included) is considered, with its
 * stored best (q, frame s) and its live state: n live shots so far, the last one's q_l and the frame number e_l it was emitted on.
 *   n == 0   the track emits when  q >= (double)first_quality && q >= (double)min_quality
 *   n > 0    the track emits when  frame - e_l >= min_gap && q > q_l * (1.0 + (double)improve)   (the sum and the product FP64, one
 *            rounding each)
 * An emission is the stored shot as an EXIT shot would carry it: frame = s, end_frame = this frame, the track's hits and age after this
 * frame, reason RF_BEST_LIVE; its crop and M go to the same buffers in the same format.  It then sets q_l = q, e_l = frame, n = n + 1.
 * A frame's EXIT shots (removed tracks) and LIVE shots (matched tracks) are compacted together in id order.  EXIT and FINISH are
 * unchanged: every ever-confirmed track still ends with exactly one EXIT or FINISH shot when its q clears min_quality, which may repeat
 * its last live crop (the same id and frame), so live shots are strictly additive.  LOST and TENTATIVE tracks never emit live; an
 * improvement held back by min_gap goes out on the track's next matched frame after the gap, or with its EXIT shot.  rf_tracker_reset
 * and rf_tracker_finish drop the live state with the store.
 * Bounds: at most one shot per slot per frame (removals come before births, and a birth is TENTATIVE except on a video's first frame,
 * where nothing can be removed), so the [n][max_tracks] buffers of f11 hold every frame; and, q being at most 1, at most
 * 1 + floor(ln(1 / first_quality) / ln(1 + improve)) live shots per track (7 with the defaults).
 *
 * Following (rf_tracker_set_best_follow).  f16's interval on a best-shot tracker: detect frames go through
 * rf_detect_yuv_track_best_device exactly as on a best-shot tracker (records, lists, quality, store and shots), and f16's Cut runs on
 * them; follow frames go through rf_track_follow_best_device: f16's follow step (lists and rf_follow records bit for bit a follow
 * tracker's), then f11's selection with no records -- the tracks removed on the frame emit their EXIT shots as on a detect frame, and
 * nothing is measured or stored.  Follow frames count in the frame numbers of rf_best_shot; live shots occur on detect frames only
 * (follow frames match no records).  rf_tracker_follow returns the latest follow call's records; motion, tiling and orientation work as
 * on the f16, f19 and f20 paths; reset and finish also drop the templates. */
#define RF_BEST_LIVE   2     /* f22: emitted while the track lives */
typedef struct rf_best_live_config {
    float first_quality;     /* 0 -> 0.3; else in (0, 1] */
    float improve;           /* 0 -> 0.2; else finite and > 0 */
    int   min_gap;           /* frames between two live shots of one track: 0 -> 30; else 1 .. 1 << 20 */
} rf_best_live_config;
/* Turns live shots on.  Not a best-shot tracker, a second call, a call after the first frame call, or bad values (NaN, out of
 * range): RF_ERR_INVALID_ARG, nothing changed. */
int rf_tracker_set_best_live(rf_tracker t, const rf_best_live_config *cfg);

/* f12 redaction: an in-place mosaic of every detected face -- and of every face the tracker still follows while the detector misses
 * it -- written into the caller's device frames, so that footage can be stored, published or annotated without its faces and no
 * frame leaves the GPU.  The calls WRITE the frames their descriptors point at (rf_yuv_frame's planes are declared const for the
 * detect calls, which only read them).  Records of the oriented entry points are in displayed pixels: redact with them through
 * rf_redact_yuv_oriented_device_style (f20).
 *
 * Regions.  Frame i's regions, in this order:
 *   (a) its records j < min(counts[i], max_faces), in rank order; box = each coordinate as __fmul_rn(x, scales[i]) (f5's map-back;
 *       scales == NULL means 1, as for tiled records);
 *   (b) with track lists: every track of frame i's list whose state is RF_TRACK_LOST, in list (id) order, box (kx1, ky1, kx2, ky2).
 *       Confirmed and tentative tracks with det >= 0 are already in (a); unmatched ones do not survive the frame.
 * A box with a non-finite coordinate, or with w <= 0 or h <= 0, is skipped.  A region's index is its position among the boxes that
 * were not skipped.
 * Geometry.  FP64, one rounding per step, in this order:
 *   w = x2 - x1, h = y2 - y1, mx = margin * w, my = margin * h
 *   X0 = floor(max(x1 - mx, -65536)), X1 = floor(min(x2 + mx, 65536)) + 1   (half-open; + 1 = the reference's inclusive x2); Y0, Y1 likewise
 *   snap outward to even: X0 = 2 floor(X0 / 2), X1 = 2 ceil(X1 / 2) (and Y)
 *   cell side C = 2 ceil(max(X1 - X0, Y1 - Y0) / (2 blocks))   (even, >= 2; a box wholly beyond +-65536 has an empty rectangle, C = 2)
 * Cells are C x C squares tiling the UNCLAMPED rectangle from (X0, Y0), the last cell of each axis possibly narrower: a face leaving
 * the frame keeps its cell size and phase.
 * Values.  Each cell's value is the mean of the ORIGINAL samples of the cell inside the frame, per plane, as (sum + cnt / 2) / cnt in integers: Y
 * over luma cells; U and V over chroma cells of side C / 2 anchored at (X0 / 2, Y0 / 2) (snapping makes that grid exact); BGR each
 * channel over the luma-coordinate cell.  "Original": before any region of the call was written, so overlapping regions never read
 * each other's output.
 * Output.  A luma (or BGR) pixel inside the frame and covered by at least one region's rectangle takes its cell value in the LOWEST-index region
 * covering it; a chroma sample likewise with the rectangles halved.  Every other byte is not written: pixels outside all regions,
 * pitch padding, and the bytes between NV12 chroma pairs that belong to other pixels. */
typedef struct rf_redact_params {
    int blocks;     /* cells across the longer side of a region; 0 -> 8; else 1..32 (1: one flat patch) */
    float margin;   /* each side grows by margin x the box's side; 0 -> 0.25; else finite, in (0, 1] */
} rf_redact_params;
/* Redacts n device frames in place from the records of any device detect call on h (dev_dets [n][max_faces], dev_counts [n], scales
 * as above) and, optionally, the track lists of a tracker of h (t, dev_tracks [n][max_tracks], dev_track_counts [n]: all three or
 * none), as rf_track_update and rf_detect_yuv_track_device return them.  params NULL: the defaults.  Asynchronous, issued on
 * rf_last_stream(), where those outputs complete; the caller keeps the frames alive until that stream has passed the call.
 * Statuses, all before anything is launched (the frames stay untouched): the frame checks of rf_detect_yuv_batch_device (or, for
 * rf_redact_device, of rf_detect_tiled_device's BGR images: dev_bgr[i], row stride NULL or 0 = packed); n > max_batch
 * RF_ERR_CAPACITY; bad params, a tracker of another handle, tracks given only partly, NULL records, a non-positive or non-finite
 * scale, or two frames whose plane byte ranges overlap: RF_ERR_INVALID_ARG.  n = 0 launches nothing.  Scratch is per execution
 * context, allocated on first use and grown with the call: max_batch x (max_faces + max_tracks) regions x blocks^2 cells x 3 bytes
 * at most. */
int rf_redact_yuv_device(rf_handle h, const rf_yuv_frame *frames, int n, const rf_det *dev_dets, const int32_t *dev_counts,
                         const float *scales, rf_tracker t, const rf_track *dev_tracks, const int32_t *dev_track_counts,
                         const rf_redact_params *params);
int rf_redact_device(rf_handle h, uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides, int n,
                     const rf_det *dev_dets, const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                     const int32_t *dev_track_counts, const rf_redact_params *params);
/* rf_detect_yuv_batch_device (t NULL) or rf_detect_yuv_track_device without crops (t a plain tracker of h; videos as there), then
 * rf_redact_yuv_device of the frames with those records, scales and tracks, all on the forward's execution context.  Detections,
 * tracks and the returned pointers are those of the two calls it replaces, bit for bit.  A best-shot tracker is RF_ERR_INVALID_ARG
 * (its store must see every frame through rf_detect_yuv_track_best_device).  dev_tracks / dev_track_counts may be NULL. */
int rf_detect_yuv_redact_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix,
                                float score_threshold, float nms_threshold, const rf_redact_params *params,
                                const rf_track **dev_tracks, const int32_t **dev_track_counts, const rf_det **dev_dets,
                                const int32_t **dev_counts, float *out_scales);

/* f14 redaction styles: a soft elliptical blur -- what broadcast, body-camera and street-level footage is published with -- or f12's
 * mosaic, over a rectangle or its inscribed ellipse, through the same regions.  Regions, their order, skipped boxes, the FP64
 * rectangle [X0, X1) x [Y0, Y1) snapped to even coordinates (unclamped) and "original" are f12's, above.  With W = X1 - X0 and
 * H = Y1 - Y0:
 * Shape.  RECT covers the rectangle, as f12.  ELLIPSE covers a sample whose centre lies in the ellipse inscribed in the rectangle:
 *   u = 2x + 1 - X0 - X1, v = 2y + 1 - Y0 - Y1, covered iff u^2 H^2 + v^2 W^2 <= W^2 H^2, in exact integers (W^2 H^2 reaches about
 *   3e20 under the +-65536 clamp: 128-bit on the device).  Chroma samples use the same test on the halved rectangle.  A rectangle
 *   empty on either axis (W <= 0 or H <= 0, only beyond the clamp) covers nothing, in either shape.  A sample takes its value from
 *   the LOWEST-index region whose shape covers it; no other byte is written.  With the default margin 0.25 the ellipse contains the
 *   whole detection box (a corner sits at 1 / (1 + 2 margin) <= 1 / sqrt(2) of each semi-axis); below margin ~0.207 the box's corners
 *   fall outside it.
 * MOSAIC.  f12's cells and cell values exactly; only the set of written samples follows the shape.
 * BLUR.  D = max(W, H); the luma / BGR radius a = clamp(ceil(D / (2 detail)), 1, 127), the chroma radius a_c = (a + 1) >> 1.  The
 *   filter is a box of width n = 2a + 1 applied three times per axis, as one integer kernel k = box * box * box (6a + 1 taps, sum n^3,
 *   sigma = sqrt(a (a + 1))).  The value of sample (x, y) of a plane is
 *     S = sum_{i,j} k[i] k[j] P[clampY(y + j)][clampX(x + i)]      (replicate borders, P the ORIGINAL plane)
 *     out = (S + (n^6 - 1) / 2) / n^6                               (integers; n^6 is odd, so no ties)
 *   over the plane of the frame: luma w x h, chroma w/2 x h/2, BGR per channel at w x h.  A one-axis sum is at most 255^4 < 2^32 and
 *   S at most 255^7 < 2^63 at a = 127.  No exp(): every implementation of this definition agrees bit for bit.
 * kind 0 is BLUR and shape 0 ELLIPSE, so a zeroed struct is a detail-4 elliptical blur at margin 0.25. */
#define RF_REDACT_MOSAIC 1
#define RF_REDACT_BLUR 2
#define RF_REDACT_RECT 1
#define RF_REDACT_ELLIPSE 2
typedef struct rf_redact_style {
    int kind;       /* RF_REDACT_MOSAIC or RF_REDACT_BLUR; 0 -> BLUR */
    int shape;      /* RF_REDACT_RECT or RF_REDACT_ELLIPSE; 0 -> ELLIPSE */
    int blocks;     /* mosaic only, as in rf_redact_params: 0 -> 8; else 1..32; must be 0 for BLUR */
    int detail;     /* blur only: 0 -> 4; else 1..64 (a larger detail, a smaller radius); must be 0 for MOSAIC */
    float margin;   /* as rf_redact_params: 0 -> 0.25; else finite, in (0, 1] */
} rf_redact_style;
/* The three f12 calls with a style (NULL: the zeroed struct's defaults).  Statuses, in the same order as the f12 call's, plus
 * RF_ERR_INVALID_ARG for a bad style where f12 checks its params; nothing is launched on any of them.  {MOSAIC, RECT} writes the bytes
 * the f12 call writes.  BLUR adds scratch planes per execution context, grown with the call: one frame's plane bytes per frame
 * (w h 3 / 2 for YUV, 3 w h for BGR) beside f12's region tables. */
int rf_redact_yuv_device_style(rf_handle h, const rf_yuv_frame *frames, int n, const rf_det *dev_dets, const int32_t *dev_counts,
                               const float *scales, rf_tracker t, const rf_track *dev_tracks, const int32_t *dev_track_counts,
                               const rf_redact_style *style);
int rf_redact_device_style(rf_handle h, uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides, int n,
                           const rf_det *dev_dets, const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                           const int32_t *dev_track_counts, const rf_redact_style *style);
int rf_detect_yuv_redact_device_style(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix,
                                      float score_threshold, float nms_threshold, const rf_redact_style *style,
                                      const rf_track **dev_tracks, const int32_t **dev_track_counts, const rf_det **dev_dets,
                                      const int32_t **dev_counts, float *out_scales);

/* f15 look-back redaction: a face is usually visible for a few frames before the detector first fires on it -- it walks in from the
 * edge, turns towards the camera, comes out from behind someone, or is too small or blurred at first.  f12 / f14 redact each frame as
 * it arrives, so those frames go out uncovered.  A LOOK-BACK tracker keeps the last L frames of each video on the GPU, emits every
 * frame L frames late, and by then knows every track born in the L frames that followed it: the emitted frame is also covered where
 * each of those faces already was.  oracle/lookback.py restates the definition; every FP64 step is one rounding in the order written.
 *
 * A look-back tracker is a plain tracker (with or without f13 motion) on which rf_tracker_set_lookback was called before its first
 * update.  It is fed only through rf_detect_yuv_redact_lookback_device.
 *   Frame numbers  each video counts its frames from 0 since create, reset or drain (the host knows every number when a call is issued).
 *   Births         the births of frame f are the tracks of f's list with age == 1, in list (id) order -- TENTATIVE births included: a
 *                  record at or above new_thresh is a confident face, and the rule errs towards covering it.
 *   Look-back box  of a birth on frame b with record box `face` (x1, y1, x2, y2, frame pixels, widened to double), on frame e = b - k,
 *                  1 <= k <= L, e at or after the first frame the video still buffers:
 *                    1. w = x2 - x1, h = y2 - y1, cx = x1 + w / 2, cy = y1 + h / 2 (f10's z);
 *                    2. with motion, for f = b, b - 1, ..., e + 1 with frame f's rf_motion {a, -B, tx, B, a, ty} of status RF_MOTION_OK
 *                       (FIRST and LOST move nothing), the motion undone: s2 = a a + B B, dx = cx - tx, dy = cy - ty,
 *                       cx = (a dx + B dy) / s2, cy = (a dy - B dx) / s2, s = sqrt(s2), w = w / s, h = h / s;
 *                    3. g = 0.5 + grow k, ex = g w, ey = g h; the box is (cx - ex, cy - ey, cx + ex, cy + ey), each rounded to float.
 *                  The face's own motion is not extrapolated (a birth's Kalman velocity is zero): the growth covers it.  At the
 *                  default, each side moves out by 10 % of the box per frame back -- 10 px per frame for a 100 px face.
 *   Regions        of an emitted frame e, in this order, each box through f12's geometry (margin, snap, skipped boxes):
 *                    (a) e's records in rank order, as __fmul_rn(x, scale);  (b) e's LOST tracks in id order, (kx1, ky1, kx2, ky2)
 *                    -- exactly what rf_redact_yuv_device_style draws on frame e --
 *                    (c) the look-back boxes of the births on frames e + 1 .. min(e + L, the video's last frame seen), frame by
 *                        frame, id order within a frame.
 *                  Shapes, styles and ownership are f14's: the lowest-index region whose shape covers a sample owns it.
 *   Output         frame e's ORIGINAL bytes (the input as it arrived) go to the caller's out frame, and the regions are redacted over
 *                  them with the call's rf_redact_style.  The out frame's pitch padding is not written.
 * Memory: a video's buffer is allocated on its first frame, L x w h 3 / 2 bytes packed in the frame's layout (47 MB per 1080p video
 * at L = 15), plus a log of 2 L frames' regions and births; it is kept until the tracker is destroyed and reallocated only when a
 * video restarts (reset, drain) at another frame size.  Each ring slot of the tracker gains max(max_batch, L) x (max_faces +
 * max_tracks + L min(max_faces, max_tracks)) records for the regions of the emitted frames. */
typedef struct rf_lookback_config {
    int frames;      /* L: 0 -> 15 (half a second at 30 fps); else 1..64 */
    float grow;      /* growth per frame back: 0 -> 0.1; else finite in (0, 1] */
} rf_lookback_config;
/* Makes t a look-back tracker.  Bad values, a call after the tracker's first update, a second call or a best-shot tracker:
 * RF_ERR_INVALID_ARG.  rf_detect_yuv_track_device, rf_track_update and rf_detect_yuv_redact_device(_style) refuse a look-back
 * tracker (RF_ERR_INVALID_ARG): the buffer must see every frame. */
int rf_tracker_set_lookback(rf_tracker t, const rf_lookback_config *cfg);
/* rf_detect_yuv_track_device without crops (records, scales, tracks and motion bit for bit the same), then: each frame is stored in
 * its video's buffer, and frame i, number num_i in its video, emits frame num_i - L of that video when num_i >= L: out_frames[i]
 * receives it, redacted as above with `style` (NULL: the zeroed struct's defaults), and out_frame_numbers[i] (host) = num_i - L;
 * otherwise out_frame_numbers[i] = -1 and out_frames[i] is not written.  An out frame must have its input frame's size and layout
 * (uv_step, and the chroma order for semi-planar frames; pitches are free) and be disjoint from every input and out frame of the call,
 * or be exactly frames[i]'s descriptor: delayed output into the caller's own surface.  The input frames are disjoint too.  A video may appear at most L times in one call
 * and its frame size and layout may not change before a drain or reset.  Statuses, all before anything is launched: those of
 * rf_detect_yuv_redact_device_style, a tracker that is not a look-back tracker, each rule above (RF_ERR_INVALID_ARG), a failed buffer
 * allocation (RF_ERR_CAPACITY).  Asynchronous on the forward's context; the tracker's event chain orders its state, and the caller
 * keeps the input and out frames alive until that stream has passed the call. */
int rf_detect_yuv_redact_lookback_device(rf_handle h, rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, int matrix,
                                         float score_threshold, float nms_threshold, const rf_redact_style *style,
                                         const rf_yuv_frame *out_frames, int32_t *out_frame_numbers, const rf_track **dev_tracks,
                                         const int32_t **dev_track_counts, const rf_det **dev_dets, const int32_t **dev_counts,
                                         float *out_scales);
/* Ends `video`: emits its min(L, frames seen) buffered frames in frame order into out_frames[0 ..) (windows end at the last frame
 * seen), *n_out of them with their numbers in out_frame_numbers, then restarts the video as rf_tracker_reset does.  cap below the
 * count: RF_ERR_CAPACITY; bad out frames (as above, against the video's frames): RF_ERR_INVALID_ARG; nothing launched on either.
 * Asynchronous on context 0's stream, inside the tracker's event chain.  rf_tracker_reset on a look-back tracker drops the buffered
 * frames and emits nothing. */
int rf_tracker_drain(rf_tracker t, int video, const rf_redact_style *style, const rf_yuv_frame *out_frames, int cap, int *n_out,
                     int32_t *out_frame_numbers);

/* f16 following between detections: run the detector on key frames only and move every known face on the frames in between by
 * searching for its own pixels, the way deployed detect + track pipelines run at a detection interval.  A FOLLOW tracker
 * (rf_tracker_set_follow) keeps, per track, a luma template cut on the track's last detection frame, and takes two kinds of frames:
 * detect frames through rf_detect_yuv_track_device / rf_detect_yuv_redact_device(_style) -- records, track lists and redacted
 * bytes exactly a plain tracker's, plus the cut below -- and follow frames through rf_track_follow_device, which runs no detector.
 * Every FP64 step is one rounding in the order written; pixels are integers (oracle/follow.py restates every bit).
 *   Grid        of a box (cx, cy, w, h) at scale c: gw = (w * G) * c, gh = (h * G) * c with G = 1 + 2 RF_FOLLOW_MARGIN;
 *               px = gw / T, py = gh / T (T = RF_FOLLOW_TEMPLATE); ox = ((cx - gw / 2) + px / 2) - 0.5, oy likewise: template pixel
 *               (i, j) is centred on frame point (ox + px i, oy + py j).
 *   Sampler     cv2.warpAffine(luma, [[px, 0, X], [0, py, Y]], INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT 0), byte for byte:
 *               Xf = (rint(X * 1024) + 16 + rint((px * i) * 1024)) >> 5, Yf = (rint((py * j + Y) * 1024) + 16) >> 5 (rint: half to
 *               even), then f5's 1/32-pixel integer bilinear; a pixel is INSIDE when its four taps lie in the frame.
 *   Cut         on every detect frame, for each track whose det >= 0 after the frame (births included; of several frames of one
 *               video in a call, the track's last such frame): the T x T template at (X, Y) = (ox, oy) of its face box (x1..y2 widened
 *               to double; w = x2 - x1, h = y2 - y1, cx = x1 + w / 2, cy = y1 + h / 2; c = 1).  The template is FLAT when
 *               T^2 sum(p^2) - (sum p)^2 < RF_FOLLOW_MIN_VAR T^4.  NV12, NV21, I420 and YV12 give the same templates.
 * On a follow frame every live track is predicted (f10) and, on a motion tracker, moved by the frame's camera motion (f13's
 * compensation, when RF_MOTION_OK); then each TENTATIVE or CONFIRMED track is searched from that state m (pcx = m_cx, pcy = m_cy,
 * pw = m_a * m_h, ph = m_h).  A state with ph or pw outside (0, 65536] or |pcx| or |pcy| above 65536 is not searched: MISMATCH.
 *   Windows     for scale k in {0, 1, 2}, c_k = {1 / RF_FOLLOW_SCALE, 1, RF_FOLLOW_SCALE} (1 / s one rounding): the grid of the
 *               predicted box at c_k, sampled as a (T + 2R) square at (X, Y) = (ox - R px, oy - R py) (R px one rounding).
 *   Match       SAD(k, dy, dx) = sum |template(i, j) - window_k(R + dx + i, R + dy + j)| over |dx|, |dy| <= R; the minimum under
 *               the order (SAD, |dx| + |dy|, k, dy, dx).  Sub-pixel per axis, when the minimum is inside the border: f =
 *               (S(-1) - S(+1)) / (2 (S(-1) - 2 S0 + S(+1))) (integers, one division; 0 when the denominator is 0), else 0.
 *   Box         ncx = pcx + ((double)dx + fx) * px_k, ncy likewise; nw = pw * c_k, nh = ph * c_k; x1 = ncx - nw / 2,
 *               y1 = ncy - nh / 2, x2 = ncx + nw / 2, y2 = ncy + nh / 2, each rounded to float.  Landmarks of the previous face f:
 *               ow = f.x2 - f.x1, ocx = f.x1 + ow / 2 (y likewise), l' = (float)(ncx + (l - ocx) * (nw / ow)); the score is kept.
 *   Status      (searched tracks) in this order: RF_FOLLOW_FLAT (the track's template is FLAT, or it has none), RF_FOLLOW_OUTSIDE (4 x the INSIDE
 *               pixels of the chosen candidate < 3 T^2), RF_FOLLOW_BORDER (|dx| or |dy| == R), RF_FOLLOW_MISMATCH (SAD > max_mad *
 *               T^2, in double, or the box is empty), else RF_FOLLOW_OK.
 *   Tracker     replaces f10's association on a follow frame: an OK track takes f10's Kalman update with z of the followed box,
 *               lost_frames = 0, face = the followed face, followed = 1, hits and state unchanged (hits count detector matches); a
 *               failed CONFIRMED track becomes LOST, a failed TENTATIVE track is removed; LOST tracks are predicted only and count
 *               lost_frames as in f10.  No births, no confirmations, det = -1 and crop_slot = -1 everywhere; age and the video's
 *               frame count advance.  Frames of one video in one call are applied in call order, each searched from the state
 *               the previous one left.
 *   Motion      f13 estimates a follow frame from luma as on a detect frame, except that its face mask (step 2) takes, in place of
 *               the frame's records, the face boxes of the video's TENTATIVE and CONFIRMED tracks before the frame (scale 1).
 *   Redaction   of a follow frame (rf_track_follow_redact_device): (a) every OK-followed track's face box, in id order, then (b) every
 *               LOST track of the frame's list, (kx1, ky1, kx2, ky2), in id order; f12's geometry, f14's styles and ownership.
 * Templates are cut on detect frames only, so a run of follow frames always compares against the detector-anchored appearance and
 * its error cannot build up. */
#define RF_FOLLOW_TEMPLATE 32
#define RF_FOLLOW_MARGIN 0.25            /* context around the face box, a fraction of its size on each side */
#define RF_FOLLOW_SCALE 1.05
#define RF_FOLLOW_MIN_VAR 16             /* texture floor of a template, luma levels squared */
#define RF_FOLLOW_MAX_SEARCH 16
#define RF_FOLLOW_OK       0
#define RF_FOLLOW_FLAT     1
#define RF_FOLLOW_BORDER   2
#define RF_FOLLOW_MISMATCH 3
#define RF_FOLLOW_OUTSIDE  4
#define RF_FOLLOW_LOST     5             /* a LOST track: predicted only, not searched */
typedef struct rf_follow_config {
    int search;          /* R, template pixels: 0 -> 8, else 1..RF_FOLLOW_MAX_SEARCH */
    float max_mad;       /* mean absolute difference bound, luma levels: 0 -> 24, else finite in (0, 255] */
} rf_follow_config;
typedef struct rf_follow {
    int32_t id, status;          /* track id; RF_FOLLOW_* */
    int32_t dx, dy, scale, sad;  /* the minimum: offset in template pixels, scale index k, its SAD (0 for LOST tracks) */
    float fx, fy;                /* sub-pixel fractions */
    float x1, y1, x2, y2;        /* the followed box, frame pixels (kept by the track only when status is OK) */
} rf_follow;
/* Makes a plain or motion tracker a follow tracker, before its first update.  Allocates a template store of max_videos x max_tracks x
 * RF_FOLLOW_TEMPLATE^2 bytes (above 4 GiB: RF_ERR_CAPACITY).  A best-shot or look-back tracker, a second call, a call after an
 * update, or bad values: RF_ERR_INVALID_ARG; rf_tracker_set_lookback refuses a follow tracker, rf_tracker_set_motion may come before
 * or after (both before the first update).
 * rf_track_update, which has no pixels, refuses a follow tracker; rf_tracker_reset drops the video's templates. */
int rf_tracker_set_follow(rf_tracker t, const rf_follow_config *cfg);
/* The follow step on n device frames (frame i of video videos[i]) of a follow tracker: windows sampled from each frame's luma,
 * then the tracker step above.  *dev_tracks / *dev_track_counts as rf_track_update's, in the same ring.  Statuses as rf_track_update
 * (frames checked as rf_detect_yuv_batch_device checks them), a tracker that is not a follow tracker: RF_ERR_INVALID_ARG; all
 * before anything is launched.  Asynchronous on rf_last_stream()'s stream, inside the tracker's event chain; the caller keeps the
 * frames alive until that stream has passed the call.  n = 0 launches nothing.  On a motion tracker rf_tracker_motion then returns
 * the call's [n] estimates. */
int rf_track_follow_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_track **dev_tracks,
                           const int32_t **dev_track_counts);
/* rf_track_follow_device (the same lists, bit for bit), then the frames redacted in place with `style` (NULL: the zeroed struct's
 * defaults) over the regions above.  Statuses of rf_track_follow_device, then a bad style or frames whose plane byte ranges overlap
 * (RF_ERR_INVALID_ARG), all before anything is launched; asynchronous on rf_last_stream()'s context. */
int rf_track_follow_redact_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_redact_style *style,
                                  const rf_track **dev_tracks, const int32_t **dev_track_counts);
/* *dev_follow -> [n][max_tracks] rf_follow of the tracker's latest follow call, each frame's records in its track-list order (NULL
 * before the first); valid for `streams` further tracker calls.  RF_ERR_INVALID_ARG on a tracker that is not a follow tracker or a
 * following look-back tracker (f18, below). */
int rf_tracker_follow(rf_tracker t, const rf_follow **dev_follow);

/* f17 searching look-back: f15's box only covers a face that moves less than grow x its size per frame back.  A SEARCHING look-back
 * tracker follows each birth back through the buffered frames with f16's template search (below), so the look-back regions take the
 * face's own path.  oracle/lookback_search.py restates the definition; every FP64 step is one rounding in the order written.
 *   Chain      of a birth (f15's births; record box `face`) on frame b:
 *                1. Template: f16's Cut of `face` on frame b's luma (the grid at c = 1, the Sampler, the FLAT test).
 *                2. Steps k = 1, 2, ..., K = min(L, b) (frame numbers since create, reset or drain: a chain never crosses a restart)
 *                   on frame e = b - k, from the box (x1, y1, x2, y2) of step k - 1 (`face` at k = 1), widened to double:
 *                   w = x2 - x1, h = y2 - y1, cx = x1 + w / 2, cy = y1 + h / 2;
 *                3. with motion, frame e + 1's rf_motion undone when RF_MOTION_OK, by f15's step-2 formulas;
 *                4. f16's search of the state z = (cx, cy, w / h, h) (pcx = cx, pcy = cy, pw = (w / h) h, ph = h): the bound
 *                   (MISMATCH, not searched), Windows, Match, Box and Status exactly as f16 states them, against the birth's template
 *                   (it is never re-cut, so error cannot build up along the chain);
 *                5. the chain stops at its first status other than RF_FOLLOW_OK (a FLAT template stops it at k = 1).
 *   Regions    of an emitted frame e: f15's (a), (b) and (c) unchanged and in the same order, then
 *                (d) for the births on frames e + 1 .. min(e + L, the video's last frame seen), frame by frame, id order within a
 *                    frame: the box of the birth's step b - e, when its chain reached that step with status OK.
 *              Geometry, shapes, styles and ownership are f12 / f14's.  Since (d) comes last, a searching tracker's out frame differs
 *              from a plain look-back tracker's only on samples (d) alone covers: a false match can add coverage, never remove it.
 * Memory: each log slot grows by min(max_faces, max_tracks) x L boxes and as many chain lengths; each ring slot by the step records
 * below; each emitted frame's region records from F + T + L min(F, T) to F + T + 2 L min(F, T). */
/* Makes a look-back tracker (with or without motion) a searching one, after rf_tracker_set_lookback and before the first update.
 * cfg: f16's rf_follow_config and bounds (search R 0 -> 8, max_mad 0 -> 24).  Not a look-back tracker, a second call, a call after
 * an update, or bad values: RF_ERR_INVALID_ARG, nothing changed.  A look-back tracker that never makes this call is unchanged. */
int rf_tracker_set_lookback_search(rf_tracker t, const rf_follow_config *cfg);
/* Of the tracker's latest rf_detect_yuv_redact_lookback_device call (NULL before the first): *dev_steps -> [n][min(max_faces,
 * max_tracks)][L] rf_follow, row (i, r) the r-th birth of frame i, step k - 1 its step on frame num_i - k; *dev_lengths -> [n][min(F,
 * T)] int32 the steps taken, the failing last one included (0 past the frame's births).  Valid for `streams` further tracker calls.
 * RF_ERR_INVALID_ARG on a tracker that is not searching. */
int rf_tracker_lookback_search(rf_tracker t, const rf_follow **dev_steps, const int32_t **dev_lengths);

/* f18 following look-back: f16 runs the detector every k-th frame only, so a face that first appears between two key frames goes out
 * uncovered until the next key frame; f15 covers a face on the L frames before its first detection, but detects every frame.  A
 * FOLLOWING look-back tracker does both: it is a look-back tracker (f15, with or without f13 motion and f17 search) on which
 * rf_tracker_set_lookback_follow was called before its first update, and it takes two kinds of frames.
 *   Detect frames  through rf_detect_yuv_redact_lookback_device, unchanged: records, scales, lists, motions, step records, out frames
 *                  and numbers are bit for bit a plain look-back tracker's in the same state; in addition f16's Cut runs on them.
 *   Follow frames  through rf_track_follow_redact_lookback_device: f16's follow step (lists and rf_follow records bit for bit a follow
 *                  tracker's for the same calls, f13 motion with f16's face mask included), then each frame is buffered and emitted L
 *                  frames late as a look-back frame is.
 *   Frame numbers  detect and follow frames share one count per video, restarted by reset and drain.
 *   Log            of a follow frame: (a) every OK-followed face's box in id order, at scale 1; (b) every LOST track in id order; no
 *                  births (no track there has age == 1); its motion, the frame's f13 estimate.
 *   Regions        of an emitted frame e: (a) and (b) of frame e -- f15's on a detect frame, the log above on a follow frame: what the
 *                  undelayed call draws on e -- then f15's (c) for the births on frames e + 1 .. min(e + L, last) (births happen on
 *                  detect frames only; the motion chain runs through every frame in between, follow frames included), then on a
 *                  searching tracker f17's (d), whose steps read follow frames from the buffer like any other.  Geometry, styles,
 *                  shapes and ownership are f12 / f14's, so an out frame differs from the undelayed redaction of e only on samples
 *                  that (c) or (d) alone cover.
 *   Coverage       with L >= k - 1, a face first detected on key frame b is covered on frames b - L .. b - 1 -- within f15's growth or
 *                  f17's search, detect and follow frames alike.  A face visible only between two key frames is never detected, so
 *                  it is never covered.
 * Drain and reset work as on a look-back tracker and, since both restart the video, also drop its templates. */
/* Makes a look-back tracker a following one, after rf_tracker_set_lookback and before the first update; before or after
 * rf_tracker_set_motion and rf_tracker_set_lookback_search.  cfg: f16's rf_follow_config and bounds; allocates f16's template store
 * (above 4 GiB: RF_ERR_CAPACITY).  Not a look-back tracker, a second call, a call after an update, or bad values: RF_ERR_INVALID_ARG,
 * nothing changed.  A following look-back tracker takes rf_detect_yuv_redact_lookback_device, rf_track_follow_redact_lookback_device,
 * rf_tracker_drain, rf_tracker_reset, rf_tracker_follow (the latest follow call's records) and the motion and search queries of its
 * options; it refuses rf_track_update, rf_detect_yuv_track_device, rf_detect_yuv_redact_device(_style), rf_track_follow_device and
 * rf_track_follow_redact_device (RF_ERR_INVALID_ARG): the buffer must see every frame. */
int rf_tracker_set_lookback_follow(rf_tracker t, const rf_follow_config *cfg);
/* The follow step of rf_track_follow_device on n device frames (frame i of video videos[i]), then the look-back half of
 * rf_detect_yuv_redact_lookback_device: each frame is stored, and frame i, number num_i, emits frame num_i - L of its video into
 * out_frames[i] with out_frame_numbers[i] = num_i - L, redacted with `style` (NULL: the zeroed struct's defaults) over the regions
 * above; otherwise out_frame_numbers[i] = -1 and out_frames[i] is not written.  Statuses, all before anything is launched: those of
 * rf_track_follow_device, a tracker that is not a following look-back tracker, a bad style, and the out-frame rules of
 * rf_detect_yuv_redact_lookback_device (same size and layout or exactly frames[i], disjoint frames, at most L frames of one video per
 * call, no size change before a drain or reset): RF_ERR_INVALID_ARG; a failed buffer allocation: RF_ERR_CAPACITY.  *dev_tracks /
 * *dev_track_counts as rf_track_follow_device's.  Asynchronous on rf_last_stream()'s context, inside the tracker's event chain; the
 * caller keeps the input and out frames alive until that stream has passed the call. */
int rf_track_follow_redact_lookback_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, const rf_redact_style *style,
                                           const rf_yuv_frame *out_frames, int32_t *out_frame_numbers, const rf_track **dev_tracks,
                                           const int32_t **dev_track_counts);

/* f22 following best-shot trackers (the f22 block above; here, after f16's rf_follow_config). */
/* Makes a best-shot tracker a following one: cfg, its bounds and its template store (above 4 GiB: RF_ERR_CAPACITY) are
 * rf_tracker_set_follow's.  Not a best-shot tracker, a second call, a call after the first frame call, or bad values:
 * RF_ERR_INVALID_ARG, nothing changed.  rf_tracker_set_follow keeps refusing a best-shot tracker.  A following best-shot tracker takes
 * rf_detect_yuv_track_best_device, rf_track_follow_best_device, rf_tracker_finish, rf_tracker_reset, rf_tracker_follow and its options'
 * queries; rf_track_update, rf_detect_yuv_track_device, rf_track_follow_device and rf_track_follow_redact_device refuse it
 * (RF_ERR_INVALID_ARG). */
int rf_tracker_set_best_follow(rf_tracker t, const rf_follow_config *cfg);
/* The follow step of rf_track_follow_device on n device frames (frame i of video videos[i]), then the frames' EXIT shots as above, in
 * rf_detect_yuv_track_best_device's outputs and buffers (dev_best_crops required when n > 0).  Statuses, all before anything is
 * launched: those of rf_track_follow_device, a tracker that is not a following best-shot tracker, a NULL dev_best_crops:
 * RF_ERR_INVALID_ARG.  Asynchronous on rf_last_stream()'s context, inside the tracker's event chain. */
int rf_track_follow_best_device(rf_tracker t, const rf_yuv_frame *frames, const int *videos, int n, void *dev_best_crops,
                                double *dev_best_mats, const rf_best_shot **dev_best, const int32_t **dev_best_counts,
                                const rf_track **dev_tracks, const int32_t **dev_track_counts);

/* f19 tiled detection in the tracker: on a 448x448 network the letter-box of a 3840x2160 frame hides every face narrower than ~137
 * pixels (f7), so a tracker fed by it leaks nearly every face of 4K street footage.  A TILING tracker detects through f7 / f8's tiles
 * instead.  Every call of it that runs the detector -- rf_detect_yuv_track_device, rf_detect_yuv_track_best_device,
 * rf_detect_yuv_redact_device(_style) and rf_detect_yuv_redact_lookback_device -- detects its frames exactly as
 *   rf_detect_yuv_tiled_device(h, frames, n, matrix, tiling, thr, nms, NULL, ...)
 * does: *dev_dets / *dev_counts are those records bit for bit (frame pixels; anchor_index = tile * max_faces + rank), they live in the
 * tiled ring (the call counts as one tiled device call for its validity rule, each of its chunks as one rf_detect_batch_device call),
 * and out_scales are all 1.  Everything after detection is what the same call does with those records at scale 1: the update,
 * motion, templates, crops, best shots, redaction and look-back.  The tracker's work runs on the tiled call's home context
 * (rf_last_stream()), and the tiled ring slot is released only after the tracker's last read of its records.
 * Statuses that depend on the frame size are the call's own, after the frame checks and before anything is launched or allocated:
 * a level side of 0 or above 16384 (RF_ERR_INVALID_ARG) and more than RF_MAX_TILES tiles (RF_ERR_CAPACITY), as rf_tile_layout
 * reports them.  rf_track_update, the follow calls, drain, finish and reset run no detector and are unchanged. */
/* Makes t a tiling tracker: an option of every kind (plain, best-shot, follow, look-back, with or without motion, search or
 * following), set before the first frame call, before or after the other setters.  tiling NULL, or levels NULL / nlevels 0: the
 * default pyramid; overlap 0: 64; the levels are copied.  A second call or a call after an update: RF_ERR_INVALID_ARG; a handle
 * created with RF_FLAG_NPP_RESIZE: RF_ERR_UNSUPPORTED; nlevels outside [0, RF_MAX_TILE_LEVELS], a negative, NaN or infinite scale or
 * an overlap out of range: RF_ERR_INVALID_ARG.  Nothing changes on a refusal. */
int rf_tracker_set_tiling(rf_tracker t, const rf_tiling *tiling);

/* f20 oriented videos in tracker calls: phones store portrait video as landscape frames with a rotation flag, and the detector only
 * finds upright faces, so a tracker fed the stored surfaces misses most faces of such a video and a redacting tracker leaves them
 * uncovered.  A tracker keeps a display orientation o (EXIF 1..8, f9's table) per video, 1 by default.  Any tracker call that reads or
 * writes the pixels of a frame of video v, on stored frames S, is exactly that call on the displayed frames D = T_o(S), each byte it
 * writes into D written into S at the stored address of that sample: luma by f9's A_o, chroma by A_o on the halved planes (even
 * sides: the 2x2 chroma blocks of D are chroma blocks of S).  As in f9 an orientation only moves integer addresses; tap positions,
 * weights, rounding, cells, blur kernels, ellipses and ownership are those of D.  So records, out_scales, track lists and state,
 * crops and matrices are bit for bit those of the same call on orient_planes(S, o) at orientation 1, and the written bytes are
 * that call's, mapped back.  Records, boxes, landmarks and tracks are in DISPLAYED frame pixels; crops come out upright.  Frame
 * descriptors, their size and layout checks, and pitch padding (never written) stay in stored geometry.  A call whose frames are
 * all at orientation 1 issues the kernels it issued before f20.  rf_track_update has no pixels and is unchanged: fed the records of
 * rf_detect_yuv_oriented_device it already tracks in displayed pixels.
 * Sets the orientation of `video`, or of every video when video is -1.  The videos must not have taken a frame call since create,
 * rf_tracker_reset, rf_tracker_drain or rf_tracker_finish (which keep the orientation: it belongs to the source, not to the run).
 * Every tracker kind and option takes it: plain, best-shot, follow and look-back, with motion, search or following.  A bad video, an
 * orientation outside 1..8, or a video already under way: RF_ERR_INVALID_ARG.  An orientation other than 1 on a tiling tracker, or
 * rf_tracker_set_tiling once some video is not at orientation 1: RF_ERR_UNSUPPORTED (a tiling tracker detects upright frames only;
 * f21's oriented tiled calls feed rf_track_update and rf_redact_yuv_oriented_device_style instead).
 * Nothing changes on a refusal.  Sizes that describe geometry -- motion thumbnails and references, follow and search frames,
 * redaction frames -- are the displayed ones; sizes that describe memory -- the look-back buffer, out frames, disjointness -- the
 * stored ones. */
int rf_tracker_set_orientation(rf_tracker t, int video, int orientation);
/* rf_redact_yuv_device_style over the records of rf_detect_yuv_oriented_device (with its out_scales) and, optionally, the lists of
 * rf_track_update fed those records: the redaction of T_o(frame) for o = orientations[i], mapped back.  rf_redact_yuv_device_style's
 * statuses, with f9's orientation check after the frame checks, all before anything is launched.  Orientation 1 writes
 * rf_redact_yuv_device_style's bytes. */
int rf_redact_yuv_oriented_device_style(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n, const rf_det *dev_dets,
                                        const int32_t *dev_counts, const float *scales, rf_tracker t, const rf_track *dev_tracks,
                                        const int32_t *dev_track_counts, const rf_redact_style *style);

/* f21 small faces in rotated and mirrored images and video: f7 / f8's tiled detection of the DISPLAYED image D = T_o(S) (f9's table;
 * D = T_o(cvtColor(frame)) for YUV), without a rotated copy.  An oriented tiled call is exactly the unoriented tiled call on D: the
 * layout is rf_tile_layout(net_w, net_h, Dw, Dh, t) of the displayed size (H x W for 5..8), a level is cv::resize(D) (of
 * cv::flip(D, 1) when mirrored), and faces, out_tile_of and anchor_index / max_faces are in DISPLAYED pixels and index the displayed
 * layout, as rf_detect_oriented_batch returns them (not mapped to stored pixels as rf_detect_views_oriented does).  Crops are cut
 * from D and M maps displayed image -> crop.  As in f9 the orientation moves integer addresses only, so every tile byte, record,
 * crop and matrix is that of the unoriented call on T_o(S), bit for bit; orientation 1 is the unoriented call.  Statuses are the
 * unoriented twin's, in its order: the source checks with f9's orientation check inside them (an orientation outside 1..8 or a NULL
 * orientations array with n > 0: RF_ERR_INVALID_ARG), then the layouts of the displayed sizes (level sides, RF_MAX_TILES,
 * the overlap), then the align checks, all before anything is launched; RF_FLAG_NPP_RESIZE: RF_ERR_UNSUPPORTED.
 *
 * Host BGR images, blocking: rf_detect_tiled with orientations; align == NULL: no crops (out_crops / out_mats unused), otherwise
 * rf_detect_tiled_align's crops and its raw-buffer rule (every original stays resident: more images than raw buffers is
 * RF_ERR_CAPACITY). */
int rf_detect_tiled_oriented(rf_handle h, const uint8_t *const *bgr_images, const int *widths, const int *heights, const int *row_strides,
                             const int *orientations, int n, const rf_tiling *t, float score_threshold, float nms_threshold,
                             const rf_align_params *align, rf_face *out_faces, int *out_counts, int32_t *out_tile_of, void *out_crops,
                             double *out_mats);
/* Device, asynchronous: rf_detect_tiled_device / rf_detect_yuv_tiled_device with orientations -- the same ring of output slots, home
 * context, rf_last_stream and validity rule.  A 4K portrait phone video (3840x2160 NV12 surfaces shown at 6) is tiled as 2160x3840. */
int rf_detect_tiled_oriented_device(rf_handle h, const uint8_t *const *dev_bgr, const int *widths, const int *heights, const int *row_strides,
                                    const int *orientations, int n, const rf_tiling *t, float score_threshold, float nms_threshold,
                                    const rf_align_params *align, void *dev_crops, double *dev_mats, const rf_det **dev_dets,
                                    const int32_t **dev_counts);
int rf_detect_yuv_tiled_oriented_device(rf_handle h, const rf_yuv_frame *frames, const int *orientations, int n, int matrix, const rf_tiling *t,
                                        float score_threshold, float nms_threshold, const rf_align_params *align, void *dev_crops,
                                        double *dev_mats, const rf_det **dev_dets, const int32_t **dev_counts);
/* Preprocess parity (as rf_preprocess_tile / rf_preprocess_yuv_tile): tile `tile` of the displayed image's layout. */
int rf_preprocess_tile_oriented(rf_handle h, const uint8_t *bgr, int width, int height, int row_stride, int orientation, const rf_tiling *t,
                                int tile, uint8_t *out_net_sized);
int rf_preprocess_yuv_tile_oriented(rf_handle h, const rf_yuv_frame *frame, int matrix, int orientation, const rf_tiling *t, int tile,
                                    uint8_t *out_net_sized);

/* f25 rotated views in the tracker: f23 / f24's views find the faces of a tilted camera (a body-worn camera, a camera over a bed, a
 * phone held at an angle), but a tracker fed by the upright letter-box leaks exactly those faces.  A VIEWS tracker detects through
 * rotated views instead.  Every call of it that runs the detector -- rf_detect_yuv_track_device, rf_detect_yuv_track_best_device,
 * rf_detect_yuv_redact_device(_style), rf_detect_yuv_redact_lookback_device, and so the key frames of follow, best-follow and
 * look-back-follow trackers -- detects its frames exactly as
 *   rf_detect_yuv_views_rotated_device(h, frames, n, matrix, views, nviews, thr, nms, NULL, NULL, NULL, dev_dets, dev_counts, NULL, NULL)
 * does: *dev_dets / *dev_counts are those records bit for bit (frame pixels; anchor_index / max_faces = the view), they live in the
 * rotated ring (the call counts as one rotated device call for its validity rule, each of its chunks as one rf_detect_batch_device
 * call), and out_scales are all 1.  Everything after detection is what the same call does with those records at scale 1: the update,
 * motion, templates, crops, best shots, redaction and look-back.  The tracker's work runs on the rotated call's home context
 * (rf_last_stream()), and the rotated ring slot is released only after the tracker's last read of its records.  rf_track_update, the
 * follow calls, drain, finish and reset run no detector and are unchanged.
 * Display orientations (f20) apply: the views of a video at orientation o rotate its displayed frames D = T_o(S), so records, tracks,
 * crops and shots are bit for bit those of the same views tracker on orient_planes(S, o) at orientation 1, and written bytes are that
 * tracker's, mapped back.  A quarter-turn view of D reads S through one composed EXIF orientation; a warp view reads D through f9's map.
 * Makes t a views tracker: an option of every kind (plain, best-shot with live shots or following, follow, look-back with search or
 * following, with or without motion), set before the first frame call, before or after the other setters.  The views are copied.
 * Statuses, in this order, nothing changed and nothing launched on a refusal: a second call or a call after a frame call
 * (RF_ERR_INVALID_ARG), views NULL (RF_ERR_INVALID_ARG), nviews outside 1..RF_MAX_VIEWS (RF_ERR_CAPACITY), a non-finite angle or a
 * shrink outside (0, 1] (RF_ERR_INVALID_ARG, f23's messages), a tiling tracker (RF_ERR_UNSUPPORTED; rf_tracker_set_tiling on a views
 * tracker is refused so too: tiling a rotated view is not supported). */
int rf_tracker_set_views(rf_tracker t, const rf_rotated_view *views, int nviews);

/* Introspection. */
int rf_get_net_size(rf_handle h, int *net_w, int *net_h, int *max_batch, int *max_faces);
int rf_num_anchors(rf_handle h);            /* per image: 8,232 @448x448, 47,040 @1280x896 */
void *rf_stream(rf_handle h);               /* cudaStream_t */
int rf_synchronize(rf_handle h);            /* all execution contexts */
/* rf_stream() is context 0's stream.  rf_fence() orders it after everything queued so far on every context
 * (for CUDA-event timing of a run of rf_detect_batch_device calls); rf_last_stream() is the stream the last
 * rf_detect_batch_device call was issued on (to order a collective on that call's device outputs). */
int rf_fence(rf_handle h);
void *rf_last_stream(rf_handle h);
/* Number of kernel launches (graph kernel nodes) one rf_detect_batch_device of batch n issues. */
int rf_launches_per_batch(rf_handle h, int n);
/* Names + device times (ms, CUDA events, direct launches) of each kernel of one forward of
 * batch n: fills up to cap entries, returns the count.  For bench.py's roofline line. */
int rf_profile_layers(rf_handle h, int n, int iters, char (*names)[64], float *ms, double *bytes, double *flops, int cap);

/* INT8 entropy calibration -- replaces the reference's offline INT8-Calibration-Tool (calibrationtable.cpp:399-583):
 * runs the n network-sized u8 BGR host images through an RF_PREC_FP32 handle twice (absmax, then 2048-bin histograms of
 * every activation tensor), searches the KL-optimal clipping threshold per tensor and writes a table in the reference's
 * own TensorRT cache format ("TRT-5102-EntropyCalibration2", one "<caffe top>: <hex float32 scale>" line per tensor) that
 * rf_create(RF_PREC_INT8) -- or the reference's Int8EntropyCalibrator2 reader (trtnetbase.cpp:31-44) -- consumes. */
int rf_calibrate_int8(rf_handle h, const uint8_t *bgr_net_sized, int n_images, const char *out_table_path);
/* Host-only: the threshold search of the calibrator on one histogram (returns the threshold in bins). */
double rf_kl_threshold_bins(const unsigned *hist, int bins, int levels);

/* Host-only (works without a GPU): the layer plan rf_create would build for `cfg`, one text line per kernel launch of a
 * forward plus the geometry / shared-memory budget of every persistent tile chain.  A launch's line is "step lane <lane>:
 * <name>", followed for a tiled launch by " | " and its tile geometry as space-separated key=value words.  Returns the launch
 * count. */
int rf_plan_describe(const rf_config *cfg, char *out, int cap);

/* Debug / parity aids (not part of the drop-in surface): fetch a materialised activation by its
 * Caffe top name (e.g. "mobilenet0_relu10_fwd", "_plus0", "rf_c1_det_concat_relu") as NCHW
 * float32 after a forward; rf_debug_keep_all disables activation-buffer reuse so every tensor
 * of the last forward survives. */
int rf_debug_get_tensor(rf_handle h, const char *name, int n, float *out_nchw, int *c, int *hh, int *ww);
int rf_debug_keep_all(rf_handle h);
/* Host-only (works without a GPU): the folded FP32 weights / bias of one convolution layer as the
 * engine holds them; dims = {cout, cin/groups, k, k}.  For CPU-side tests of the model front end. */
int rf_model_inspect(const char *caffemodel_path, const char *layer, float *w, int wcap, float *b, int bcap, int dims[4]);
/* Host-only model front end (SURVEY.md 8f-4).  rf_model_load: the complete load path of rf_create -- cache lookup, prototxt parse +
 * graph check, file-driven folding, cache write -- without a device; *cache_status: 0 no cache, 1 miss (written), 2 hit,
 * 3 stale (rewritten); input_dims: N, C, H, W of the prototxt (zeros without one); then rf_model_inspect semantics for `layer`
 * (may be NULL).  rf_network_config: the reference's network-name switch (RetinaFace.cpp:211-268): FPN strides, anchor scales per
 * level (2 each), ratios; RF_ERR_UNSUPPORTED where the reference prints "please reconfig anchor_cfg". */
int rf_model_load(const char *caffemodel_path, const char *prototxt_path, const char *cache_path, int *cache_status, int input_dims[4],
                  const char *layer, float *w, int wcap, float *b, int bcap, int dims[4]);
int rf_network_config(const char *network, int *num_levels, int strides[3], int scales[6], float ratios[2], int *num_ratios);
/* Cache state of a handle's model load (the enum above). */
int rf_cache_status(rf_handle h);

#ifdef __cplusplus
}
#endif
#endif /* RF_B200_H */
