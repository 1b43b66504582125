"""ctypes binding of include/rf_b200.h.  Fails loudly when librf_b200.so is missing: there is no
Python / CPU implementation of the path behind it."""
from __future__ import annotations

import ctypes as C
import os
import types
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

RF_PREC_FP32, RF_PREC_FP16, RF_PREC_INT8 = 0, 1, 2
RF_FLAG_NO_GRAPH, RF_FLAG_NO_TENSORCORE, RF_FLAG_SIMT_STEM, RF_FLAG_DW_1D, RF_FLAG_LEGACY_TC, RF_FLAG_NPP_RESIZE = 0x1, 0x2, 0x4, 0x8, 0x10, 0x20
FACE_FLOATS = 15
PIPELINE_DEPTH = 6   # RF_PIPELINE_DEPTH
COMM_BLOB_BYTES = 128


class _View(C.Structure):       # rf_view
    _fields_ = [("shrink", C.c_float), ("flip", C.c_int32)]


class _OrientedView(C.Structure):    # rf_oriented_view
    _fields_ = [("shrink", C.c_float), ("orientation", C.c_int32)]


class _RotatedView(C.Structure):     # rf_rotated_view
    _fields_ = [("angle", C.c_float), ("shrink", C.c_float)]


# EXIF orientations (rf_b200.h f9): 1 upright, 2 mirrored, 3 rotated 180, 4 upside-down mirror, 5 transposed, 6 rotated 90 clockwise,
# 7 transverse, 8 rotated 90 counter-clockwise; ANY_ORIENTATION are the four rotations rf_detect_views_oriented sweeps
ORIENTATIONS = tuple(range(1, 9))
ANY_ORIENTATION = (1, 6, 3, 8)


RF_CROP_BGR_U8, RF_CROP_RGB_F32, RF_CROP_RGB_F16 = 0, 1, 2
# crop format name -> (RF_CROP_*, element type, channels-last)
CROP_FORMATS = {"bgr_u8": (RF_CROP_BGR_U8, np.uint8, True), "rgb_f32": (RF_CROP_RGB_F32, np.float32, False),
                "rgb_f16": (RF_CROP_RGB_F16, np.float16, False)}


class AlignParams(C.Structure):  # rf_align_params
    _fields_ = [("crop_w", C.c_int), ("crop_h", C.c_int), ("template_xy", C.c_float * 10), ("max_faces", C.c_int),
                ("format", C.c_int), ("mean", C.c_float), ("std", C.c_float)]


def align_params(crop=(112, 112), template=None, fmt: str = "bgr_u8", max_faces: int = 0, mean: float = 0.0, std: float = 0.0) -> AlignParams:
    """rf_align_params.  crop = (width, height); template: 5 (x, y) crop-pixel targets, None -> the ArcFace 112x112 template;
    mean = std = 0 -> 127.5."""
    if fmt not in CROP_FORMATS:
        raise ValueError(f"crop format {fmt!r}: one of {sorted(CROP_FORMATS)}")
    t = np.zeros(10, np.float32) if template is None else np.asarray(template, np.float32).reshape(10)
    return AlignParams(int(crop[0]), int(crop[1]), (C.c_float * 10)(*t.tolist()), int(max_faces), CROP_FORMATS[fmt][0], float(mean), float(std))


def crop_shape(fmt: str, crop) -> Tuple[tuple, type]:
    """(shape, dtype) of one crop: (h, w, 3) u8 BGR or (3, h, w) planar RGB."""
    _, dt, hwc = CROP_FORMATS[fmt]
    w, h = int(crop[0]) or 112, int(crop[1]) or 112
    return ((h, w, 3) if hwc else (3, h, w)), dt


class YuvFrame(C.Structure):     # rf_yuv_frame
    _fields_ = [("y", C.c_void_p), ("u", C.c_void_p), ("v", C.c_void_p), ("y_pitch", C.c_int), ("uv_pitch", C.c_int), ("uv_step", C.c_int),
                ("width", C.c_int), ("height", C.c_int)]


RF_YUV_BT601, RF_YUV_BT709 = 0, 1
YUV_MATRICES = {"bt601": RF_YUV_BT601, "bt709": RF_YUV_BT709}
YUV_LAYOUTS = ("nv12", "nv21", "i420", "yv12")


def _plane(a):
    """(address, row pitch in bytes, rows, row bytes, on the GPU) of a 2-D u8 plane: a numpy array or a torch tensor whose rows are
    contiguous (pitch >= row bytes)."""
    if hasattr(a, "data_ptr"):          # torch
        if a.dtype.itemsize != 1 or a.dim() != 2 or a.stride(1) != 1:
            raise ValueError(f"2-D uint8 plane with contiguous rows expected, got {tuple(a.shape)} {a.dtype} strides {a.stride()}")
        return a.data_ptr(), a.stride(0), a.shape[0], a.shape[1], a.is_cuda
    a = np.asarray(a)
    if a.dtype != np.uint8 or a.ndim != 2 or a.strides[1] != 1:
        raise ValueError(f"2-D uint8 plane with contiguous rows expected, got {a.shape} {a.dtype} strides {a.strides}")
    return a.ctypes.data, a.strides[0], a.shape[0], a.shape[1], False


def yuv_frame(frame, layout: str = "nv12") -> Tuple[YuvFrame, bool]:
    """rf_yuv_frame of one 4:2:0 frame, and whether its planes are device memory.  `frame`: OpenCV's single buffer, a C-contiguous
    (h * 3 / 2, w) u8 array / tensor in `layout` (nv12 | nv21 | i420 | yv12); or planes with their own pitches, (y, uv) for nv12 /
    nv21 (uv: (h / 2, w) interleaved) or (y, u, v) in that order for i420 / yv12 (u, v: (h / 2, w / 2)).  The caller keeps the
    memory alive."""
    if layout not in YUV_LAYOUTS:
        raise ValueError(f"layout {layout!r}: one of {YUV_LAYOUTS}")
    semi = layout in ("nv12", "nv21")
    if isinstance(frame, (tuple, list)):
        planes = [_plane(p) for p in frame]
        if len(planes) != (2 if semi else 3):
            raise ValueError(f"{layout}: {'(y, uv)' if semi else '(y, u, v)'} planes expected, got {len(planes)}")
        (y, yp, h, w, dev), rest = planes[0], planes[1:]
        if any(p[4] != dev for p in rest):
            raise ValueError("planes must all be host or all be device memory")
        if semi:
            uv, uvp = rest[0][0], rest[0][1]
            u, v = (uv, uv + 1) if layout == "nv12" else (uv + 1, uv)
            return YuvFrame(y, u, v, yp, uvp, 2, w, h), dev
        if rest[0][1] != rest[1][1]:
            raise ValueError("u and v planes must share one pitch")
        return YuvFrame(y, rest[0][0], rest[1][0], yp, rest[0][1], 1, w, h), dev
    p, pitch, rows, w, dev = _plane(frame)
    contiguous = frame.is_contiguous() if hasattr(frame, "is_contiguous") else frame.flags.c_contiguous
    if not contiguous or rows % 3 or w % 2:
        raise ValueError(f"single-buffer 4:2:0 frame: C-contiguous (h * 3 / 2, w) with even h and w expected, got {rows}x{w}")
    h = rows * 2 // 3
    c = p + w * h
    if semi:
        u, v = (c, c + 1) if layout == "nv12" else (c + 1, c)
        return YuvFrame(p, u, v, w, w, 2, w, h), dev
    q = c + (w // 2) * (h // 2)
    u, v = (c, q) if layout == "i420" else (q, c)
    return YuvFrame(p, u, v, w, w // 2, 1, w, h), dev


def _matrix(matrix) -> int:
    if isinstance(matrix, str):
        if matrix not in YUV_MATRICES:
            raise ValueError(f"matrix {matrix!r}: one of {sorted(YUV_MATRICES)}")
        return YUV_MATRICES[matrix]
    return int(matrix)


class TileLevel(C.Structure):    # rf_tile_level
    _fields_ = [("scale", C.c_float), ("flip", C.c_int32)]


class Tiling(C.Structure):       # rf_tiling
    _fields_ = [("levels", C.POINTER(TileLevel)), ("nlevels", C.c_int), ("overlap", C.c_int)]


class Tile(C.Structure):         # rf_tile
    _fields_ = [(f, C.c_int) for f in ("level", "flip", "scaled_w", "scaled_h", "x0", "y0", "own_x0", "own_y0", "own_x1", "own_y1",
                                       "shared_sides")] + [("scale", C.c_float), ("map_back", C.c_float)]


MAX_TILE_LEVELS, MAX_TILES = 8, 256          # RF_MAX_TILE_LEVELS, RF_MAX_TILES
TILE_SIDE_LEFT, TILE_SIDE_TOP, TILE_SIDE_RIGHT, TILE_SIDE_BOTTOM = 0x1, 0x2, 0x4, 0x8


def tiling(levels=None, overlap: int = 0) -> Tiling:
    """rf_tiling.  levels: [(scale, flip), ...] (scale 0: the fitted level), None or [] -> the default pyramid; overlap 0 -> 64.
    The level array lives on the returned structure (keep it alive for the call)."""
    levels = list(levels or [])
    arr = (TileLevel * max(len(levels), 1))(*[TileLevel(float(s), int(bool(f))) for s, f in levels])
    t = Tiling(C.cast(arr, C.POINTER(TileLevel)) if levels else None, len(levels), int(overlap))
    t._keep = arr
    return t


def tile_dict(t: Tile) -> dict:
    return {f: getattr(t, f) for f, _ in Tile._fields_}


def tile_layout(net_w: int, net_h: int, width: int, height: int, levels=None, overlap: int = 0) -> List[dict]:
    """rf_tile_layout (host-only): the tiles of one width x height image, each as a dict of rf_tile's fields, in candidate-id order."""
    lib = load_library()
    t = tiling(levels, overlap)
    k = lib.rf_tile_layout(net_w, net_h, width, height, C.byref(t), None, 0)
    if k < 0:
        raise RfError(k, (lib.rf_last_error(None) or b"").decode())
    out = (Tile * max(k, 1))()
    k = lib.rf_tile_layout(net_w, net_h, width, height, C.byref(t), out, k)
    return [tile_dict(out[i]) for i in range(k)]


class TrackConfig(C.Structure):  # rf_track_config
    _fields_ = [("max_videos", C.c_int), ("max_tracks", C.c_int), ("high_thresh", C.c_float), ("new_thresh", C.c_float),
                ("iou_high", C.c_float), ("iou_low", C.c_float), ("iou_tentative", C.c_float), ("max_lost", C.c_int)]


class Face(C.Structure):         # rf_face
    _fields_ = [("score", C.c_float), ("x1", C.c_float), ("y1", C.c_float), ("x2", C.c_float), ("y2", C.c_float),
                ("lx", C.c_float * 5), ("ly", C.c_float * 5)]


def _record_dtype(struct) -> np.dtype:
    """The numpy record of a ctypes Structure: every field at its ctypes offset, a nested Face as FACE_FLOATS floats."""
    names = [f for f, _ in struct._fields_]
    return np.dtype(dict(names=names, formats=[("<f4", (FACE_FLOATS,)) if t is Face else np.dtype(t) for _, t in struct._fields_],
                         offsets=[getattr(struct, f).offset for f in names], itemsize=C.sizeof(struct)))


class TrackRecord(C.Structure):  # rf_track
    _fields_ = [(f, C.c_int32) for f in ("id", "state", "det", "crop_slot", "hits", "age", "lost_frames", "followed")] + \
               [(f, C.c_float) for f in ("kx1", "ky1", "kx2", "ky2", "vx", "vy")] + [("face", Face)]


TRACK_TENTATIVE, TRACK_CONFIRMED, TRACK_LOST = 0, 1, 2      # RF_TRACK_*
TRACK_DEBUG_DOUBLES = 25                                     # RF_TRACK_DEBUG_DOUBLES
TRACK_DTYPE = _record_dtype(TrackRecord)                     # one rf_track as a numpy record


class BestConfig(C.Structure):   # rf_best_config
    _fields_ = [("align", AlignParams), ("min_quality", C.c_float), ("sharp_half", C.c_float)]


def best_config(min_quality: float = 0.0, sharp_half: float = 0.0, **align) -> BestConfig:
    """rf_best_config: ``align_params`` keywords (crop, template, fmt, mean, std) for the emitted crops; sharp_half 0 -> 50."""
    return BestConfig(align_params(**align), float(min_quality), float(sharp_half))


class BestShot(C.Structure):     # rf_best_shot
    _fields_ = [(f, C.c_int32) for f in ("id", "video", "frame", "end_frame", "hits", "age", "reason", "reserved")] + \
               [(f, C.c_float) for f in ("quality", "score", "eye", "frontal", "sharpness", "coverage")] + [("face", Face)]


BEST_EXIT, BEST_FINISH, BEST_LIVE = 0, 1, 2                  # RF_BEST_*


class BestLiveConfig(C.Structure):   # rf_best_live_config (f22)
    _fields_ = [("first_quality", C.c_float), ("improve", C.c_float), ("min_gap", C.c_int)]
BEST_DTYPE = _record_dtype(BestShot)                         # one rf_best_shot as a numpy record


class MotionConfig(C.Structure):  # rf_motion_config
    _fields_ = [("search", C.c_int), ("min_inliers", C.c_int)]


def motion_config(search: int = 0, min_inliers: int = 0) -> MotionConfig:
    """rf_motion_config: search radius R in thumbnail pixels (0 -> 12), min_inliers (0 -> 12)."""
    return MotionConfig(int(search), int(min_inliers))


class Motion(C.Structure):       # rf_motion
    _fields_ = [(f, C.c_int32) for f in ("status", "blocks", "inliers", "reserved")] + [("m", C.c_double * 6)]


MOTION_OK, MOTION_FIRST, MOTION_LOST = 0, 1, 2               # RF_MOTION_*
MOTION_DTYPE = _record_dtype(Motion)                         # one rf_motion as a numpy record


class FollowConfig(C.Structure):  # rf_follow_config
    _fields_ = [("search", C.c_int), ("max_mad", C.c_float)]


class FollowRecord(C.Structure):  # rf_follow
    _fields_ = [(f, C.c_int32) for f in ("id", "status", "dx", "dy", "scale", "sad")] + \
               [(f, C.c_float) for f in ("fx", "fy", "x1", "y1", "x2", "y2")]


FOLLOW_OK, FOLLOW_FLAT, FOLLOW_BORDER, FOLLOW_MISMATCH, FOLLOW_OUTSIDE, FOLLOW_LOST = range(6)   # RF_FOLLOW_*
FOLLOW_DTYPE = _record_dtype(FollowRecord)                   # one rf_follow as a numpy record


class RedactParams(C.Structure):  # rf_redact_params
    _fields_ = [("blocks", C.c_int), ("margin", C.c_float)]


RF_REDACT_MOSAIC, RF_REDACT_BLUR = 1, 2
RF_REDACT_RECT, RF_REDACT_ELLIPSE = 1, 2


class RedactStyle(C.Structure):  # rf_redact_style
    _fields_ = [("kind", C.c_int), ("shape", C.c_int), ("blocks", C.c_int), ("detail", C.c_int), ("margin", C.c_float)]


def redact_style(style: str = "mosaic", shape: str = "rect", blocks: int = 0, detail: int = 0, margin: float = 0.0) -> Optional[RedactStyle]:
    """The rf_redact_style of the redaction keywords, or None for f12's mosaic over rectangles ({"mosaic", "rect"}, detail 0), which
    the f12 calls draw.  style: "mosaic" or "blur"; shape: "rect" or "ellipse"; detail: the blur's 0 (4) or 1..64."""
    kinds, shapes = {"mosaic": RF_REDACT_MOSAIC, "blur": RF_REDACT_BLUR}, {"rect": RF_REDACT_RECT, "ellipse": RF_REDACT_ELLIPSE}
    if style not in kinds or shape not in shapes:
        raise ValueError(f"style {style!r} / shape {shape!r}: style is one of {sorted(kinds)}, shape one of {sorted(shapes)}")
    if style == "mosaic" and shape == "rect" and not detail:
        return None
    return RedactStyle(kinds[style], shapes[shape], int(blocks), int(detail), float(margin))


class LookbackConfig(C.Structure):  # rf_lookback_config
    _fields_ = [("frames", C.c_int), ("grow", C.c_float)]


def _redaction(lib, name: str, style: str, shape: str, blocks: int, detail: int, margin: float):
    """(entry point, the rf_redact_params or rf_redact_style to pass it) of the redaction keywords for the call `name`.  An f12
    entry point draws f12's mosaic over rectangles from rf_redact_params and anything else through its `_style` variant; the
    calls that take only a style get one for every set of keywords, {MOSAIC, RECT} included."""
    st = redact_style(style, shape, blocks, detail, margin)
    if name + "_style" not in _SIGNATURES:
        return getattr(lib, name), st if st is not None else RedactStyle(RF_REDACT_MOSAIC, RF_REDACT_RECT, int(blocks), 0, float(margin))
    if st is None:
        return getattr(lib, name), RedactParams(int(blocks), float(margin))
    return getattr(lib, name + "_style"), st


class RfError(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"librf_b200 status {status}: {msg}")
        self.status = status


class _Config(C.Structure):
    _fields_ = [("caffemodel_path", C.c_char_p), ("int8_table_path", C.c_char_p), ("precision", C.c_int),
                ("net_w", C.c_int), ("net_h", C.c_int), ("max_batch", C.c_int), ("max_faces", C.c_int),
                ("device", C.c_int), ("max_image_w", C.c_int), ("max_image_h", C.c_int), ("flags", C.c_uint),
                ("streams", C.c_int), ("prototxt_path", C.c_char_p), ("cache_path", C.c_char_p), ("network", C.c_char_p)]


# The C signature of every function include/rf_b200.h declares: name -> (restype, argtypes), applied by load_library().
# rf_handle, rf_tracker and output arrays are plain addresses; _PP is the address of a pointer the call writes.
_P, _I, _F, _S = C.c_void_p, C.c_int, C.c_float, C.c_char_p
_PP, _PI = C.POINTER(C.c_void_p), C.POINTER(C.c_int)
_ALIGN, _FRAMES, _TILING, _STYLE = C.POINTER(AlignParams), C.POINTER(YuvFrame), C.POINTER(Tiling), C.POINTER(RedactStyle)
_DETECT_DEVICE = [_P, _P, _I, _F, _F, _PP, _PP]                 # rf_detect_batch_device and its allgather
_SUBMIT, _COLLECT = [_P, _PP, _I, _F, _F, _PI], [_P, _I, _P, _P, _P]
_REDACT_YUV = [_P, _FRAMES, _I, _P, _P, _P, _P, _P, _P]         # rf_redact_yuv_device(_style) before the params or style
_REDACT_BGR = [_P, _PP, _PI, _PI, _PI, _I, _P, _P, _P, _P, _P, _P]
_DETECT_YUV_TRACKED = [_P, _P, _FRAMES, _P, _I, _I, _F, _F]     # (h, t, frames, videos, n, matrix, thresholds) of the tracked calls
_TRACKED_OUT = [_PP, _PP, _PP, _PP, _P]                         # their (tracks, track counts, dets, counts, scales) outputs
_SIGNATURES = {
    "rf_abi_version": (_I, []), "rf_build_info": (_S, []), "rf_status_string": (_S, [_I]),
    "rf_create": (_I, [C.POINTER(_Config), _PP]), "rf_destroy": (None, [_P]), "rf_last_error": (_S, [_P]),
    "rf_pinned_input": (_P, [_P]), "rf_device_input": (_P, [_P]),
    "rf_detect_batch": (_I, [_P, _PP, _PI, _PI, _PI, _I, _F, _F, _P, _P, _P]),
    "rf_submit_batch": (_I, _SUBMIT), "rf_collect_batch": (_I, _COLLECT), "rf_detect_batch_device": (_I, _DETECT_DEVICE),
    "rf_forward_heads": (_I, [_P, _P, _I, _PP]),
    "rf_postprocess": (_I, [_P, _PP, _I, _F, _F, _P, _P, _P, _P]),
    "rf_preprocess": (_I, [_P, _P, _I, _I, _I, _P]),
    "rf_get_net_size": (_I, [_P, _PI, _PI, _PI, _PI]), "rf_num_anchors": (_I, [_P]), "rf_stream": (_P, [_P]),
    "rf_synchronize": (_I, [_P]), "rf_fence": (_I, [_P]), "rf_last_stream": (_P, [_P]), "rf_launches_per_batch": (_I, [_P, _I]),
    "rf_profile_layers": (_I, [_P, _I, _I, _P, _P, _P, _P, _I]),
    "rf_debug_get_tensor": (_I, [_P, _S, _I, _P, _PI, _PI, _PI]), "rf_debug_keep_all": (_I, [_P]),
    "rf_model_inspect": (_I, [_S, _S, _P, _I, _P, _I, _PI]),
    "rf_calibrate_int8": (_I, [_P, _P, _I, _S]), "rf_kl_threshold_bins": (C.c_double, [_P, _I, _I]),
    "rf_detect_views": (_I, [_P, _P, _I, _I, _I, C.POINTER(_View), _I, _F, _F, _P, _PI, _P, _P]),
    "rf_plan_describe": (_I, [C.POINTER(_Config), _S, _I]),
    "rf_comm_export": (_I, [_P, _I, _I, _P]), "rf_comm_init": (_I, [_P, _P]), "rf_comm_nccl_unique_id": (_I, [_P]),
    "rf_comm_init_nccl": (_I, [_P, _P, _I, _I]), "rf_comm_info": (_I, [_P, _PI, _PI]),
    "rf_detect_batch_device_allgather": (_I, _DETECT_DEVICE), "rf_submit_batch_allgather": (_I, _SUBMIT),
    "rf_collect_batch_allgather": (_I, _COLLECT), "rf_detect_batch_allgather": (_I, [_P, _PP, _I, _F, _F, _P, _P, _P]),
    "rf_model_load": (_I, [_S, _S, _S, _PI, _PI, _S, _P, _I, _P, _I, _PI]),
    "rf_network_config": (_I, [_S, _PI, _PI, _PI, C.POINTER(C.c_float), _PI]), "rf_cache_status": (_I, [_P]),
    "rf_detect_jpeg_batch": (_I, [_P, _P, _P, _I, _F, _F, _P, _P, _P, _P, _P]),
    "rf_decode_jpeg": (_I, [_P, _P, C.c_size_t, _P, C.c_size_t, _P, _P]), "rf_jpeg_backend": (_S, [_P]),
    "rf_detect_align_batch": (_I, [_P, _PP, _PI, _PI, _PI, _I, _F, _F, _ALIGN, _P, _P, _P, _P]),
    "rf_detect_align_batch_device": (_I, [_P, _P, _I, _F, _F, _ALIGN, _P, _P, _PP, _PP]),
    "rf_detect_yuv_batch": (_I, [_P, _FRAMES, _I, _I, _F, _F, _ALIGN, _P, _P, _P, _P, _P]),
    "rf_detect_yuv_batch_device": (_I, [_P, _FRAMES, _I, _I, _F, _F, _ALIGN, _P, _P, _PP, _PP, _P]),
    "rf_preprocess_yuv": (_I, [_P, _FRAMES, _I, _P]),
    "rf_tile_layout": (_I, [_I, _I, _I, _I, _TILING, C.POINTER(Tile), _I]),
    "rf_detect_tiled": (_I, [_P, _PP, _PI, _PI, _PI, _I, _TILING, _F, _F, _P, _P, _P]),
    "rf_detect_yuv_tiled": (_I, [_P, _FRAMES, _I, _I, _TILING, _F, _F, _P, _P, _P]),
    "rf_preprocess_tile": (_I, [_P, _P, _I, _I, _I, _TILING, _I, _P]),
    "rf_preprocess_yuv_tile": (_I, [_P, _FRAMES, _I, _TILING, _I, _P]),
    "rf_detect_tiled_align": (_I, [_P, _PP, _PI, _PI, _PI, _I, _TILING, _F, _F, _ALIGN, _P, _P, _P, _P, _P]),
    "rf_detect_yuv_tiled_align": (_I, [_P, _FRAMES, _I, _I, _TILING, _F, _F, _ALIGN, _P, _P, _P, _P, _P]),
    "rf_detect_tiled_device": (_I, [_P, _PP, _PI, _PI, _PI, _I, _TILING, _F, _F, _ALIGN, _P, _P, _PP, _PP]),
    "rf_detect_yuv_tiled_device": (_I, [_P, _FRAMES, _I, _I, _TILING, _F, _F, _ALIGN, _P, _P, _PP, _PP]),
    "rf_detect_oriented_batch": (_I, [_P, _PP, _PI, _PI, _PI, _PI, _I, _F, _F, _ALIGN, _P, _P, _P, _P, _P]),
    "rf_detect_yuv_oriented_device": (_I, [_P, _FRAMES, _PI, _I, _I, _F, _F, _ALIGN, _P, _P, _PP, _PP, _P]),
    "rf_preprocess_oriented": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "rf_preprocess_yuv_oriented": (_I, [_P, _FRAMES, _I, _I, _P]),
    "rf_detect_views_oriented": (_I, [_P, _P, _I, _I, _I, C.POINTER(_OrientedView), _I, _F, _F, _P, _PI, _P, _P]),
    "rf_jpeg_exif_orientation": (_I, [_P, C.c_size_t]),
    "rf_detect_views_rotated": (_I, [_P, _P, _I, _I, _I, C.POINTER(_RotatedView), _I, _F, _F, _ALIGN, _P, _PI, _P, _P, _P, _P, _P]),
    "rf_preprocess_rotated": (_I, [_P, _P, _I, _I, _I, _F, _F, _P, _P]),
    "rf_detect_views_rotated_device": (_I, [_P, _PP, _PI, _PI, _PI, _I, C.POINTER(_RotatedView), _I, _F, _F, _ALIGN, _P, _P, _PP, _PP, _P, _P]),
    "rf_detect_yuv_views_rotated_device": (_I, [_P, _FRAMES, _I, _I, C.POINTER(_RotatedView), _I, _F, _F, _ALIGN, _P, _P, _PP, _PP, _P, _P]),
    "rf_preprocess_yuv_rotated": (_I, [_P, _FRAMES, _I, _F, _F, _P, _P]),
    "rf_fetch_dets": (_I, [_P, _P, _P, _I, _P, _P, _P]),
    "rf_tracker_create": (_I, [_P, C.POINTER(TrackConfig), _PP]), "rf_tracker_destroy": (None, [_P]),
    "rf_tracker_reset": (_I, [_P, _I]),
    "rf_track_update": (_I, [_P, _P, _I, _P, _P, _P, _PP, _PP]),
    "rf_detect_yuv_track_device": (_I, _DETECT_YUV_TRACKED + [_ALIGN, _P, _P] + _TRACKED_OUT),
    "rf_tracker_debug_state": (_I, [_P, _I, _P, _I]),
    "rf_tracker_create_best": (_I, [_P, C.POINTER(TrackConfig), C.POINTER(BestConfig), _PP]),
    "rf_detect_yuv_track_best_device": (_I, _DETECT_YUV_TRACKED + [_P, _P, _PP, _PP] + _TRACKED_OUT),
    "rf_tracker_finish": (_I, [_P, _I, _P, _P, _PP, _PP]),
    "rf_tracker_set_motion": (_I, [_P, C.POINTER(MotionConfig)]), "rf_tracker_motion": (_I, [_P, _PP]),
    "rf_redact_yuv_device": (_I, _REDACT_YUV + [C.POINTER(RedactParams)]),
    "rf_redact_device": (_I, _REDACT_BGR + [C.POINTER(RedactParams)]),
    "rf_detect_yuv_redact_device": (_I, _DETECT_YUV_TRACKED + [C.POINTER(RedactParams)] + _TRACKED_OUT),
    "rf_redact_yuv_device_style": (_I, _REDACT_YUV + [_STYLE]), "rf_redact_device_style": (_I, _REDACT_BGR + [_STYLE]),
    "rf_detect_yuv_redact_device_style": (_I, _DETECT_YUV_TRACKED + [_STYLE] + _TRACKED_OUT),
    "rf_tracker_set_lookback": (_I, [_P, C.POINTER(LookbackConfig)]),
    "rf_detect_yuv_redact_lookback_device": (_I, _DETECT_YUV_TRACKED + [_STYLE, _FRAMES, _P] + _TRACKED_OUT),
    "rf_tracker_drain": (_I, [_P, _I, _STYLE, _FRAMES, _I, _PI, _P]),
    "rf_tracker_set_follow": (_I, [_P, C.POINTER(FollowConfig)]),
    "rf_track_follow_device": (_I, [_P, _FRAMES, _P, _I, _PP, _PP]), "rf_tracker_follow": (_I, [_P, _PP]),
    "rf_track_follow_redact_device": (_I, [_P, _FRAMES, _P, _I, _STYLE, _PP, _PP]),
    "rf_tracker_set_lookback_search": (_I, [_P, C.POINTER(FollowConfig)]), "rf_tracker_lookback_search": (_I, [_P, _PP, _PP]),
    "rf_tracker_set_lookback_follow": (_I, [_P, C.POINTER(FollowConfig)]),
    "rf_track_follow_redact_lookback_device": (_I, [_P, _FRAMES, _P, _I, _STYLE, _FRAMES, _P, _PP, _PP]),
    "rf_tracker_set_tiling": (_I, [_P, _TILING]),
    "rf_tracker_set_best_live": (_I, [_P, C.POINTER(BestLiveConfig)]),
    "rf_tracker_set_best_follow": (_I, [_P, C.POINTER(FollowConfig)]),
    "rf_track_follow_best_device": (_I, [_P, _FRAMES, _P, _I, _P, _P, _PP, _PP, _PP, _PP]),
    "rf_tracker_set_orientation": (_I, [_P, _I, _I]),
    "rf_redact_yuv_oriented_device_style": (_I, [_P, _FRAMES, _PI, _I, _P, _P, _P, _P, _P, _P, _STYLE]),
    "rf_detect_tiled_oriented": (_I, [_P, _PP, _PI, _PI, _PI, _PI, _I, _TILING, _F, _F, _ALIGN, _P, _P, _P, _P, _P]),
    "rf_detect_tiled_oriented_device": (_I, [_P, _PP, _PI, _PI, _PI, _PI, _I, _TILING, _F, _F, _ALIGN, _P, _P, _PP, _PP]),
    "rf_detect_yuv_tiled_oriented_device": (_I, [_P, _FRAMES, _PI, _I, _I, _TILING, _F, _F, _ALIGN, _P, _P, _PP, _PP]),
    "rf_tracker_set_views": (_I, [_P, C.POINTER(_RotatedView), _I]),
    "rf_preprocess_tile_oriented": (_I, [_P, _P, _I, _I, _I, _I, _TILING, _I, _P]),
    "rf_preprocess_yuv_tile_oriented": (_I, [_P, _FRAMES, _I, _I, _TILING, _I, _P]),
}
EXPORTS = list(_SIGNATURES)     # every symbol include/rf_b200.h declares (checked by tests/test_host_side.py)


def lib_path() -> str:
    return os.environ.get("RF_B200_LIB", os.path.join(_HERE, "librf_b200.so"))


_lib = None


def load_library() -> C.CDLL:
    """dlopen librf_b200.so (built in-tree by retinaface_b200/build.py or __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise ImportError(f"{p} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(retinaface_b200 has no CPU fallback)")
    lib = C.CDLL(p)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def model_inspect(caffemodel: str, layer: str):
    """(w, b) folded parameters of one convolution, from the library's host-side model front end."""
    lib = load_library()
    dims = (C.c_int * 4)()
    rc = lib.rf_model_inspect(caffemodel.encode(), layer.encode(), None, 0, None, 0, dims)
    if rc != 0:
        raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
    shape = tuple(dims)
    w = np.empty(shape, dtype=np.float32)
    b = np.empty(shape[0], dtype=np.float32)
    rc = lib.rf_model_inspect(caffemodel.encode(), layer.encode(), w.ctypes.data_as(C.c_void_p), w.size,
                              b.ctypes.data_as(C.c_void_p), b.size, dims)
    if rc != 0:
        raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
    return w, b


def plan_describe(caffemodel: str, net_h: int, net_w: int, precision: int = RF_PREC_FP16, max_batch: int = 8, flags: int = 0,
                  int8_table: Optional[str] = None, streams: int = 0, max_faces: int = 0, geometry: bool = False) -> str:
    """The layer plan rf_create would build (host-only entry point: no GPU needed).  `max_faces` as in Engine (0 -> 256): the tile
    chains reserve shared memory for the last-block NMS's kept list, so the plan depends on it.  Each launch is a line
    "step lane <lane>: <name>"; with `geometry`, a tiled launch's line goes on with " | " and its tile geometry (key=value
    words)."""
    lib = load_library()
    cfg = _Config(caffemodel.encode(), int8_table.encode() if int8_table else None, precision, net_w, net_h, max_batch, max_faces, 0, 0, 0,
                  flags, streams, None, None, None)
    buf = C.create_string_buffer(1 << 16)
    rc = lib.rf_plan_describe(C.byref(cfg), buf, len(buf))
    if rc < 0:
        raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
    text = buf.value.decode()
    if geometry:
        return text
    return "".join(ln.split(" | ", 1)[0] + "\n" if ln.startswith("step lane ") else ln + "\n" for ln in text.splitlines())


def model_load(caffemodel: str, prototxt: Optional[str] = None, cache: Optional[str] = None, layer: Optional[str] = None):
    """rf_model_load (host-only): the load path of rf_create.  Returns (cache_status, input_dims, (w, b) of `layer` or None)."""
    lib = load_library()
    cs = C.c_int(0)
    idims = (C.c_int * 4)()
    dims = (C.c_int * 4)()
    args = (caffemodel.encode(), prototxt.encode() if prototxt else None, cache.encode() if cache else None, C.byref(cs), idims, layer.encode() if layer else None)
    rc = lib.rf_model_load(*args, None, 0, None, 0, dims)
    if rc != 0:
        raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
    wb = None
    if layer:
        w = np.empty(tuple(dims), dtype=np.float32)
        b = np.empty(dims[0], dtype=np.float32)
        rc = lib.rf_model_load(*args, w.ctypes.data_as(C.c_void_p), w.size, b.ctypes.data_as(C.c_void_p), b.size, dims)
        if rc != 0:
            raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
        wb = (w, b)
    return cs.value, tuple(idims), wb


def network_config(network: str):
    """rf_network_config: (strides, scales per level, ratios) of the reference's network-name switch; RfError(-7) where unsupported."""
    lib = load_library()
    nl, nr = C.c_int(0), C.c_int(0)
    strides, scales, ratios = (C.c_int * 3)(), (C.c_int * 6)(), (C.c_float * 2)()
    rc = lib.rf_network_config(network.encode(), C.byref(nl), strides, scales, ratios, C.byref(nr))
    if rc != 0:
        raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
    return list(strides)[:nl.value], [list(scales)[2 * i:2 * i + 2] for i in range(nl.value)], list(ratios)[:nr.value]


def nccl_unique_id() -> bytes:
    """A fresh ncclUniqueId (rank 0 creates it, the caller ships it to the other ranks) for Engine.comm_init_nccl."""
    lib = load_library()
    buf = C.create_string_buffer(128)
    rc = lib.rf_comm_nccl_unique_id(buf)
    if rc != 0:
        raise RfError(rc, (lib.rf_last_error(None) or b"").decode())
    return buf.raw


def exif_orientation(jpeg: bytes) -> int:
    """rf_jpeg_exif_orientation (host-only): the EXIF orientation 1..8 cv::imread would apply to these JPEG bytes, 1 without one."""
    lib = load_library()
    buf = np.frombuffer(bytes(jpeg), dtype=np.uint8)
    return int(lib.rf_jpeg_exif_orientation(buf.ctypes.data if buf.size else None, buf.size))


def _orientations(orientations, n: int):
    """The int array of n EXIF orientations the oriented entry points take (their range is checked by the library)."""
    o = [int(v) for v in orientations]
    if len(o) != n:
        raise ValueError(f"{n} items but {len(o)} orientations")
    return (C.c_int * max(n, 1))(*o)


def kl_threshold_bins(hist: np.ndarray, levels: int = 128) -> float:
    """The calibrator's threshold search (host-only entry point of the library)."""
    lib = load_library()
    h = np.ascontiguousarray(hist, dtype=np.uint32)
    return float(lib.rf_kl_threshold_bins(h.ctypes.data_as(C.c_void_p), len(h), levels))


STRIDES = (32, 16, 8)


def head_shapes(net_h: int, net_w: int) -> List[Tuple[int, int, int]]:
    return [(c, net_h // s, net_w // s) for s in STRIDES for c in (4, 8, 20)]


def device_view(ptr: int, shape, typestr: str):
    """A torch CUDA tensor aliasing the `shape` array of numpy type `typestr` (e.g. "<f4") at device address ptr, without a copy."""
    import torch
    cai = dict(shape=tuple(shape), typestr=typestr, data=(int(ptr), False), version=3)
    return torch.as_tensor(types.SimpleNamespace(__cuda_array_interface__=cai), device="cuda")


def _addr(a: Optional[np.ndarray]):
    """The address of an optional host output array, as the C ABI takes it (NULL for None)."""
    return a.ctypes.data if a is not None else None


def _ref(s: Optional[C.Structure]):
    """An optional structure passed by reference (NULL for None)."""
    return C.byref(s) if s is not None else None


class Engine:
    """One rf_handle: one GPU, one stream."""

    def __init__(self, caffemodel: str, net_h: int, net_w: int, precision: int = RF_PREC_FP16, max_batch: int = 8,
                 max_faces: int = 256, device: int = 0, int8_table: Optional[str] = None,
                 max_image: Optional[Tuple[int, int]] = None, flags: int = 0, streams: int = 0, prototxt: Optional[str] = None,
                 cache: Optional[str] = None, network: Optional[str] = None):
        self.lib = load_library()
        cfg = _Config(caffemodel.encode(), int8_table.encode() if int8_table else None, precision, net_w, net_h,
                      max_batch, max_faces, device, max_image[1] if max_image else 0, max_image[0] if max_image else 0, flags, streams,
                      prototxt.encode() if prototxt else None, cache.encode() if cache else None, network.encode() if network else None)
        h = C.c_void_p()
        rc = self.lib.rf_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise RfError(rc, (self.lib.rf_last_error(None) or b"").decode())
        self.h = h
        if net_h == 0 and net_w == 0:          # taken from the prototxt
            nw, nh = C.c_int(), C.c_int()
            self.lib.rf_get_net_size(h, C.byref(nw), C.byref(nh), None, None)
            net_h, net_w = nh.value, nw.value
        self.net_h, self.net_w = net_h, net_w
        self.max_batch, self.precision, self.device = max_batch, precision, device
        mf = C.c_int()
        self.lib.rf_get_net_size(self.h, None, None, None, C.byref(mf))
        self.max_faces = mf.value
        self.num_anchors = self.lib.rf_num_anchors(self.h)

    def close(self):
        if getattr(self, "h", None):
            self.lib.rf_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc < 0:
            raise RfError(rc, (self.lib.rf_last_error(self.h) or b"").decode())
        return rc

    # -- buffers --------------------------------------------------------------------------
    def pinned_input(self) -> np.ndarray:
        """numpy view of the library's pinned staging: (max_batch, H, W, 3) u8."""
        p = self.lib.rf_pinned_input(self.h)
        n = self.max_batch * self.net_h * self.net_w * 3
        buf = (C.c_uint8 * n).from_address(p)
        return np.frombuffer(buf, dtype=np.uint8).reshape(self.max_batch, self.net_h, self.net_w, 3)

    def device_input_ptr(self) -> int:
        return int(self.lib.rf_device_input(self.h))

    def stream_ptr(self) -> int:
        return int(self.lib.rf_stream(self.h) or 0)

    def synchronize(self):
        self._check(self.lib.rf_synchronize(self.h))

    def fence(self):
        """Order stream_ptr() after everything queued so far on every execution context."""
        self._check(self.lib.rf_fence(self.h))

    def last_stream_ptr(self) -> int:
        return int(self.lib.rf_last_stream(self.h) or 0)

    def _fetch(self, ptr: int, dtype, *shape) -> np.ndarray:
        """A host copy of the `shape` array of `dtype` records at device address ptr, taken after rf_synchronize."""
        dtype = np.dtype(dtype)
        self._check(self.lib.rf_synchronize(self.h))
        return device_view(ptr, (int(np.prod(shape)) * dtype.itemsize,), "|u1").cpu().numpy().view(dtype).reshape(shape)

    def read_dets(self, dets_ptr: int, counts_ptr: int, n: int):
        """The rf_det records of n images of a device detect call, copied after rf_synchronize: (faces: one (k, 15) float32 array per
        image, anchor_index: one (k,) int32 array per image)."""
        rec = self._fetch(dets_ptr, np.float32, n, self.max_faces, FACE_FLOATS + 1)
        counts = self._fetch(counts_ptr, np.int32, n)
        return ([rec[i, :counts[i], :FACE_FLOATS].copy() for i in range(n)],
                [rec[i, :counts[i], FACE_FLOATS].view(np.int32).copy() for i in range(n)])

    # -- end to end ------------------------------------------------------------------------
    def detect_batch(self, images: Sequence[np.ndarray], thr: float, nms_thr: float, want_index: bool = False):
        """images: u8 BGR HWC arrays (any size <= max_image).  Returns list of (k,15) float32 arrays
        (FaceDetectInfo rows, score order) [+ list of anchor-index arrays]."""
        n = len(images)
        keep = [np.ascontiguousarray(im, dtype=np.uint8) if not (im.flags.c_contiguous and im.dtype == np.uint8) else im
                for im in images]
        for im in keep:
            if im.ndim != 3 or im.shape[2] != 3:
                raise ValueError(f"u8 BGR HWC images expected, got shape {im.shape}")
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in keep])
        ws = (C.c_int * n)(*[im.shape[1] for im in keep])
        hs = (C.c_int * n)(*[im.shape[0] for im in keep])
        faces = np.empty((n, self.max_faces, FACE_FLOATS), dtype=np.float32)
        counts = np.zeros(n, dtype=np.int32)
        idx = np.empty((n, self.max_faces), dtype=np.int32) if want_index else None
        self._check(self.lib.rf_detect_batch(self.h, ptrs, ws, hs, None, n, thr, nms_thr, faces.ctypes.data,
                                             counts.ctypes.data, idx.ctypes.data if want_index else None))
        out = [faces[i, :counts[i]].copy() for i in range(n)]
        if want_index:
            return out, [idx[i, :counts[i]].copy() for i in range(n)]
        return out

    # -- host arguments and results of the aligning, tiled and oriented calls ---------------------------------------------------
    @staticmethod
    def _bgr_strided(im):
        """The image as the C ABI takes it: u8 BGR HWC with contiguous pixels (rows may be strided)."""
        if im.ndim != 3 or im.shape[2] != 3:
            raise ValueError(f"u8 BGR HWC images expected, got shape {im.shape}")
        if not (im.dtype == np.uint8 and im.strides[1:] == (3, 1) and im.strides[0] >= 3 * im.shape[1]):
            im = np.ascontiguousarray(im, dtype=np.uint8)
        return im

    @staticmethod
    def _host_images(images):
        """(the arrays to keep alive, pointers, widths, heights, row strides) of host u8 BGR HWC images, each as _bgr_strided."""
        keep = [Engine._bgr_strided(im) for im in images]
        n = max(len(keep), 1)
        return (keep, (C.c_void_p * n)(*[im.ctypes.data for im in keep]), (C.c_int * n)(*[im.shape[1] for im in keep]),
                (C.c_int * n)(*[im.shape[0] for im in keep]), (C.c_int * n)(*[im.strides[0] for im in keep]))

    def _outputs(self, n: int, index: bool):
        """The host faces, counts and (with index) per-face int32 arrays a detect call on n images writes."""
        return (np.empty((n, self.max_faces, FACE_FLOATS), dtype=np.float32), np.zeros(n, dtype=np.int32),
                np.empty((n, self.max_faces), dtype=np.int32) if index else None)

    def _host_align(self, n: int, align: dict):
        """rf_align_params and the host crop / matrix arrays of detect_align's keywords: (params, A, crops, mats or None)."""
        kw = dict(align)
        want_mats = kw.pop("want_mats", False)
        p = align_params(**{"fmt": "bgr_u8", **kw})
        A = p.max_faces or self.max_faces
        shape, dt = crop_shape(kw.get("fmt", "bgr_u8"), (p.crop_w, p.crop_h))
        return p, A, np.empty((n, A) + shape, dtype=dt), (np.empty((n, A, 2, 3), dtype=np.float64) if want_mats else None)

    @staticmethod
    def _result(counts, faces, tile_of=None, A=0, crops=None, mats=None, idx=None):
        """A host call's per-image lists (faces[, tile_of][, crops[, mats]][, idx]), each array cut to its image's count (the crops
        and matrices to at most A); the faces alone when nothing else was asked for."""
        n = len(counts)
        out = [[a[i, :counts[i]].copy() for i in range(n)] for a in (faces, tile_of) if a is not None]
        out += [[a[i, :min(counts[i], A)].copy() for i in range(n)] for a in (crops, mats) if a is not None]
        if idx is not None:
            out.append([idx[i, :counts[i]].copy() for i in range(n)])
        return out[0] if len(out) == 1 else tuple(out)

    def detect_align(self, images: Sequence[np.ndarray], thr: float, nms_thr: float, crop=(112, 112), template=None, fmt: str = "bgr_u8",
                     max_faces: int = 0, want_mats: bool = False, mean: float = 0.0, std: float = 0.0):
        """rf_detect_align_batch: u8 BGR HWC images (any size <= max_image; rows may be strided, e.g. a slice of a larger array)
        -> (faces: list of (k, 15) float32 arrays in ORIGINAL IMAGE pixels, crops: list of (min(k, A), *crop_shape) arrays
        [, mats: list of (min(k, A), 2, 3) float64 image -> crop matrices]), A = max_faces or the engine's max_faces."""
        n = len(images)
        keep, ptrs, ws, hs, rs = self._host_images(images)
        p, A, crops, mats = self._host_align(n, dict(crop=crop, template=template, fmt=fmt, max_faces=max_faces, mean=mean, std=std,
                                                     want_mats=want_mats))
        faces, counts, _ = self._outputs(n, False)
        self._check(self.lib.rf_detect_align_batch(self.h, ptrs, ws, hs, rs, n, thr, nms_thr, C.byref(p), faces.ctypes.data, counts.ctypes.data,
                                                   crops.ctypes.data, _addr(mats)))
        return self._result(counts, faces, A=A, crops=crops, mats=mats)

    def detect_align_device(self, n: int, thr: float, nms_thr: float, dev_crops_ptr: int, crop=(112, 112), template=None, fmt: str = "bgr_u8",
                            max_faces: int = 0, mean: float = 0.0, std: float = 0.0, dev_mats_ptr: Optional[int] = None,
                            dev_ptr: Optional[int] = None):
        """rf_detect_align_batch_device: asynchronous; the crops of image i, face j land at dev_crops_ptr + (i * A + j) * crop bytes
        (device).  Returns the (dets_ptr, counts_ptr) device addresses of rf_detect_batch_device."""
        p = align_params(crop, template, fmt, max_faces, mean, std)
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_align_batch_device(self.h, dev_ptr if dev_ptr is not None else self.device_input_ptr(), n, thr, nms_thr,
                                                          C.byref(p), dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c)))
        return int(d.value), int(c.value)

    # -- f6 video frames (YUV 4:2:0) ----------------------------------------------------------------
    @staticmethod
    def _frames(frames, layout: str, device: bool):
        descs = [yuv_frame(f, layout) for f in frames]
        if any(dev != device for _, dev in descs):
            raise ValueError(f"{'device' if device else 'host'} frames expected")
        return (YuvFrame * max(len(descs), 1))(*[d for d, _ in descs])

    def detect_yuv(self, frames, thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601", align: Optional[dict] = None,
                   want_index: bool = False):
        """rf_detect_yuv_batch: host 4:2:0 frames (see yuv_frame for the forms) -> faces in FRAME pixels, one (k, 15) float32 array
        per frame.  align: detect_align's keywords (crop, template, fmt, max_faces, mean, std, want_mats) -> (faces, crops[, mats])
        as detect_align returns them.  want_index appends the anchor-index arrays."""
        n = len(frames)
        arr = self._frames(frames, layout, False)
        faces, counts, idx = self._outputs(n, want_index)
        p, A, crops, mats = self._host_align(n, align) if align is not None else (None, 0, None, None)
        self._check(self.lib.rf_detect_yuv_batch(self.h, arr, n, _matrix(matrix), thr, nms_thr, _ref(p), faces.ctypes.data, counts.ctypes.data,
                                                 _addr(idx), _addr(crops), _addr(mats)))
        return self._result(counts, faces, A=A, crops=crops, mats=mats, idx=idx)

    def detect_yuv_device(self, frames, thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601", align: Optional[dict] = None,
                          dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_yuv_batch_device: device 4:2:0 frames (torch CUDA tensors in yuv_frame's forms), asynchronous on
        last_stream_ptr().  Returns (dets_ptr, counts_ptr, map-back scale of each frame); detections in network-input pixels.
        align: detect_align's keywords; the crops land at dev_crops_ptr as in detect_align_device."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        p = align_params(**align) if align is not None else None
        scales = np.zeros(max(n, 1), dtype=np.float32)
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_yuv_batch_device(self.h, arr, n, _matrix(matrix), thr, nms_thr, _ref(p),
                                                        dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c), scales.ctypes.data))
        return int(d.value), int(c.value), scales[:n].copy()

    def preprocess_yuv(self, frame, layout: str = "nv12", matrix="bt601") -> np.ndarray:
        """rf_preprocess_yuv: one host frame letter-boxed into the (H, W, 3) u8 BGR network input."""
        arr = self._frames([frame], layout, False)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        self._check(self.lib.rf_preprocess_yuv(self.h, arr, _matrix(matrix), out.ctypes.data))
        return out

    # -- f7 tiled detection ----------------------------------------------------------------------------
    def detect_tiled(self, images: Sequence[np.ndarray], thr: float, nms_thr: float, levels=None, overlap: int = 0, align: Optional[dict] = None):
        """rf_detect_tiled: u8 BGR HWC images (any size <= max_image; rows may be strided) cut into tiles of a scale pyramid
        (levels: [(scale, flip), ...], scale 0 = the fitted level; None = the default pyramid).  Returns (faces: one (k, 15) float32
        array per image in ORIGINAL IMAGE pixels, tile_of: one (k,) array per image, indices into tile_layout).  align: detect_align's
        keywords (crop, template, fmt, max_faces, mean, std, want_mats) -> rf_detect_tiled_align, and the crops (and matrices) follow:
        (faces, tile_of, crops[, mats]) as detect_align returns them."""
        n = len(images)
        keep, ptrs, ws, hs, rs = self._host_images(images)
        t = tiling(levels, overlap)
        faces, counts, tile_of = self._outputs(n, True)
        if align is None:
            self._check(self.lib.rf_detect_tiled(self.h, ptrs, ws, hs, rs, n, C.byref(t), thr, nms_thr, faces.ctypes.data, counts.ctypes.data,
                                                 tile_of.ctypes.data))
            return self._result(counts, faces, tile_of)
        p, A, crops, mats = self._host_align(n, align)
        self._check(self.lib.rf_detect_tiled_align(self.h, ptrs, ws, hs, rs, n, C.byref(t), thr, nms_thr, C.byref(p), faces.ctypes.data,
                                                   counts.ctypes.data, tile_of.ctypes.data, crops.ctypes.data, _addr(mats)))
        return self._result(counts, faces, tile_of, A, crops, mats)

    def detect_yuv_tiled(self, frames, thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601", levels=None, overlap: int = 0,
                         align: Optional[dict] = None):
        """rf_detect_yuv_tiled: host 4:2:0 frames (yuv_frame's forms) -> (faces, tile_of) as detect_tiled, in FRAME pixels; with align,
        rf_detect_yuv_tiled_align and (faces, tile_of, crops[, mats]) as detect_tiled."""
        n = len(frames)
        arr = self._frames(frames, layout, False)
        t = tiling(levels, overlap)
        faces, counts, tile_of = self._outputs(n, True)
        if align is None:
            self._check(self.lib.rf_detect_yuv_tiled(self.h, arr, n, _matrix(matrix), C.byref(t), thr, nms_thr, faces.ctypes.data,
                                                     counts.ctypes.data, tile_of.ctypes.data))
            return self._result(counts, faces, tile_of)
        p, A, crops, mats = self._host_align(n, align)
        self._check(self.lib.rf_detect_yuv_tiled_align(self.h, arr, n, _matrix(matrix), C.byref(t), thr, nms_thr, C.byref(p), faces.ctypes.data,
                                                       counts.ctypes.data, tile_of.ctypes.data, crops.ctypes.data, _addr(mats)))
        return self._result(counts, faces, tile_of, A, crops, mats)

    @staticmethod
    def _device_images(images):
        """(pointers, widths, heights, row strides) of u8 BGR HWC torch CUDA tensors with contiguous pixels; the row stride is
        stride(0), so a slice of a larger tensor is read in place."""
        n = len(images)
        for im in images:
            if not (hasattr(im, "data_ptr") and getattr(im, "is_cuda", False)):
                raise ValueError(f"device images must be torch CUDA tensors, got {type(im).__name__}")
            if (str(im.dtype) != "torch.uint8" or im.dim() != 3 or im.shape[2] != 3 or im.stride(2) != 1 or im.stride(1) != 3
                    or im.stride(0) < 3 * im.shape[1]):
                raise ValueError(f"u8 BGR HWC tensor with contiguous pixels expected, got {tuple(im.shape)} {im.dtype} strides {im.stride()}")
        return ((C.c_void_p * max(n, 1))(*[im.data_ptr() for im in images]), (C.c_int * max(n, 1))(*[im.shape[1] for im in images]),
                (C.c_int * max(n, 1))(*[im.shape[0] for im in images]), (C.c_int * max(n, 1))(*[im.stride(0) for im in images]))

    def detect_tiled_device(self, images, thr: float, nms_thr: float, levels=None, overlap: int = 0, align: Optional[dict] = None,
                            dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_tiled_device: u8 BGR HWC torch CUDA tensors (rows may be strided), tiled as detect_tiled, asynchronous on
        last_stream_ptr().  Returns the (dets_ptr, counts_ptr) device addresses: [max_batch][max_faces] rf_det in ORIGINAL IMAGE pixels,
        anchor_index = tile * max_faces + rank, valid for `streams` further tiled device calls.  align: detect_align's keywords; the
        crops land at dev_crops_ptr as in detect_align_device.  Host arrays: ValueError."""
        n = len(images)
        ptrs, ws, hs, rs = self._device_images(images)
        t = tiling(levels, overlap)
        p = align_params(**align) if align is not None else None
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_tiled_device(self.h, ptrs, ws, hs, rs, n, C.byref(t), thr, nms_thr, _ref(p),
                                                    dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c)))
        return int(d.value or 0), int(c.value or 0)

    def detect_yuv_tiled_device(self, frames, thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601", levels=None, overlap: int = 0,
                                align: Optional[dict] = None, dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_yuv_tiled_device: device 4:2:0 frames (torch CUDA tensors in yuv_frame's forms), otherwise as detect_tiled_device
        (faces in FRAME pixels).  Host frames: ValueError."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        t = tiling(levels, overlap)
        p = align_params(**align) if align is not None else None
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_yuv_tiled_device(self.h, arr, n, _matrix(matrix), C.byref(t), thr, nms_thr,
                                                        _ref(p), dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c)))
        return int(d.value or 0), int(c.value or 0)

    def preprocess_tile(self, img: np.ndarray, tile: int, levels=None, overlap: int = 0) -> np.ndarray:
        """rf_preprocess_tile: tile `tile` of the image's layout as the network sees it, (H, W, 3) u8 BGR."""
        img = self._bgr_strided(img)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        t = tiling(levels, overlap)
        self._check(self.lib.rf_preprocess_tile(self.h, img.ctypes.data, img.shape[1], img.shape[0], img.strides[0], C.byref(t), int(tile),
                                                out.ctypes.data))
        return out

    def preprocess_yuv_tile(self, frame, tile: int, layout: str = "nv12", matrix="bt601", levels=None, overlap: int = 0) -> np.ndarray:
        """rf_preprocess_yuv_tile: tile `tile` of one host 4:2:0 frame's layout as the network sees it, (H, W, 3) u8 BGR."""
        arr = self._frames([frame], layout, False)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        t = tiling(levels, overlap)
        self._check(self.lib.rf_preprocess_yuv_tile(self.h, arr, _matrix(matrix), C.byref(t), int(tile), out.ctypes.data))
        return out

    def detect_jpeg(self, streams: Sequence[bytes], thr: float, nms_thr: float):
        """JPEG bitstreams (bytes) -> decoded on the GPU (nvJPEG), letter-boxed, detected.  Returns (list of (k,15) arrays in
        network-input pixels, list of (width, height) of the decoded images)."""
        n = len(streams)
        bufs = [np.frombuffer(b, dtype=np.uint8) for b in streams]
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        lens = (C.c_size_t * n)(*[b.size for b in bufs])
        faces = np.empty((n, self.max_faces, FACE_FLOATS), dtype=np.float32)
        counts = np.zeros(n, dtype=np.int32)
        ws, hs = (C.c_int * n)(), (C.c_int * n)()
        self._check(self.lib.rf_detect_jpeg_batch(self.h, ptrs, lens, n, thr, nms_thr, faces.ctypes.data, counts.ctypes.data, None, ws, hs))
        return [faces[i, :counts[i]].copy() for i in range(n)], [(ws[i], hs[i]) for i in range(n)]

    def decode_jpeg(self, stream: bytes) -> np.ndarray:
        """nvJPEG decode of one stream -> (h, w, 3) u8 BGR (what rf_detect_jpeg_batch letter-boxes)."""
        buf = np.frombuffer(stream, dtype=np.uint8)
        w, hh = C.c_int(), C.c_int()
        self._check(self.lib.rf_decode_jpeg(self.h, buf.ctypes.data, buf.size, None, 0, C.byref(w), C.byref(hh)))
        out = np.empty((hh.value, w.value, 3), dtype=np.uint8)
        self._check(self.lib.rf_decode_jpeg(self.h, buf.ctypes.data, buf.size, out.ctypes.data, out.nbytes, C.byref(w), C.byref(hh)))
        return out

    def jpeg_backend(self) -> str:
        return self.lib.rf_jpeg_backend(self.h).decode()

    def detect_pinned(self, n: int, thr: float, nms_thr: float, faces: np.ndarray, counts: np.ndarray):
        """Hot-loop variant for bench.py: the n images are already in pinned_input(); results go
        into caller-provided arrays.  Still the full H2D -> GPU -> D2H path."""
        base = self.lib.rf_pinned_input(self.h)
        sz = self.net_h * self.net_w * 3
        if not hasattr(self, "_pin_args") or self._pin_args[0] != n:
            self._pin_args = (n, (C.c_void_p * n)(*[base + i * sz for i in range(n)]),
                              (C.c_int * n)(*[self.net_w] * n), (C.c_int * n)(*[self.net_h] * n))
        _, ptrs, ws, hs = self._pin_args
        self._check(self.lib.rf_detect_batch(self.h, ptrs, ws, hs, None, n, thr, nms_thr, faces.ctypes.data,
                                             counts.ctypes.data, None))

    def _net_sized(self, images: Sequence[np.ndarray]):
        """rf_submit_batch reads net_h * net_w * 3 bytes from every pointer: refuse anything else."""
        for im in images:
            if im.shape != (self.net_h, self.net_w, 3) or im.dtype != np.uint8 or not im.flags.c_contiguous:
                raise ValueError(f"network-sized C-contiguous uint8 images of shape {(self.net_h, self.net_w, 3)} expected, got {im.shape} {im.dtype}")

    def submit(self, images: Sequence[np.ndarray], thr: float, nms_thr: float, allgather: bool = False) -> int:
        """Pipelined path: queue one batch of network-sized images (H2D on the copy stream + forward + D2H);
        returns a ticket for collect().  Up to PIPELINE_DEPTH batches in flight.  allgather: the multi-GPU exchange too."""
        n = len(images)
        self._net_sized(images)
        ptrs = (C.c_void_p * n)(*[im.ctypes.data for im in images])
        t = C.c_int()
        fn = self.lib.rf_submit_batch_allgather if allgather else self.lib.rf_submit_batch
        self._check(fn(self.h, ptrs, n, thr, nms_thr, C.byref(t)))
        self._inflight = getattr(self, "_inflight", {})
        self._inflight[t.value] = (n, images, allgather)      # keep the sources alive until collected
        return t.value

    def collect(self, ticket: int, faces: Optional[np.ndarray] = None, counts: Optional[np.ndarray] = None):
        n, _, allgather = self._inflight.pop(ticket)
        rows = self.comm_world * self.max_batch if allgather else n
        if faces is None:
            faces = np.empty((rows, self.max_faces, FACE_FLOATS), dtype=np.float32)
        if counts is None:
            counts = np.zeros(rows, dtype=np.int32)
        fn = self.lib.rf_collect_batch_allgather if allgather else self.lib.rf_collect_batch
        self._check(fn(self.h, ticket, faces.ctypes.data, counts.ctypes.data, None))
        return faces, counts

    # -- multi-GPU ---------------------------------------------------------------------------
    comm_world = 1

    def comm_export(self, rank: int, world: int) -> bytes:
        blob = C.create_string_buffer(COMM_BLOB_BYTES)
        self._check(self.lib.rf_comm_export(self.h, rank, world, blob))
        return blob.raw

    def comm_init(self, blobs: Sequence[bytes]):
        raw = b"".join(blobs)
        self._check(self.lib.rf_comm_init(self.h, raw))
        self.comm_world = len(blobs)

    def comm_init_nccl(self, unique_id: bytes, rank: int, world: int):
        self._check(self.lib.rf_comm_init_nccl(self.h, unique_id, rank, world))
        self.comm_world = world

    def detect_device_allgather(self, n: int, thr: float, nms_thr: float, dev_ptr: int):
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_batch_device_allgather(self.h, dev_ptr, n, thr, nms_thr, C.byref(d), C.byref(c)))
        return int(d.value), int(c.value)

    def detect_device(self, n: int, thr: float, nms_thr: float, dev_ptr: Optional[int] = None):
        """Asynchronous device-resident detect.  Returns (dets_ptr, counts_ptr) device addresses."""
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_batch_device(self.h, dev_ptr if dev_ptr is not None else self.device_input_ptr(),
                                                    n, thr, nms_thr, C.byref(d), C.byref(c)))
        return int(d.value), int(c.value)

    # -- parity entry points -----------------------------------------------------------------
    def forward_heads(self, images: np.ndarray) -> List[np.ndarray]:
        images = np.ascontiguousarray(images, dtype=np.uint8)
        n = images.shape[0]
        assert images.shape[1:] == (self.net_h, self.net_w, 3), images.shape
        outs = [np.empty((n,) + s, dtype=np.float32) for s in head_shapes(self.net_h, self.net_w)]
        ptrs = (C.c_void_p * 9)(*[o.ctypes.data for o in outs])
        self._check(self.lib.rf_forward_heads(self.h, images.ctypes.data, n, ptrs))
        return outs

    def postprocess(self, heads: Sequence[np.ndarray], thr: float, nms_thr: float):
        """heads: 9 arrays (n,C,h,w).  Returns (faces list, index list, candidate counts)."""
        keep = [np.ascontiguousarray(h, dtype=np.float32) for h in heads]
        n = keep[0].shape[0]
        ptrs = (C.c_void_p * 9)(*[k.ctypes.data for k in keep])
        faces = np.empty((n, self.max_faces, FACE_FLOATS), dtype=np.float32)
        idx = np.empty((n, self.max_faces), dtype=np.int32)
        counts = np.zeros(n, dtype=np.int32)
        ncand = np.zeros(n, dtype=np.int32)
        self._check(self.lib.rf_postprocess(self.h, ptrs, n, thr, nms_thr, faces.ctypes.data, counts.ctypes.data,
                                            idx.ctypes.data, ncand.ctypes.data))
        return ([faces[i, :counts[i]].copy() for i in range(n)], [idx[i, :counts[i]].copy() for i in range(n)], ncand)

    def preprocess(self, img: np.ndarray) -> np.ndarray:
        img = np.ascontiguousarray(img, dtype=np.uint8)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        self._check(self.lib.rf_preprocess(self.h, img.ctypes.data, img.shape[1], img.shape[0], 0, out.ctypes.data))
        return out

    def detect_views(self, img: np.ndarray, views, thr: float, nms: float):
        """rf_detect_views: one image, views = [(shrink, flip), ...] run as one batch, merged on the GPU.  Returns
        (faces [k, 15] in ORIGINAL IMAGE pixels, view index of each face [k], map-back scale of each view)."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        nv = len(views)
        varr = (_View * max(nv, 1))(*[_View(float(s), int(bool(f))) for s, f in views])
        faces = np.empty((self.max_faces, 15), dtype=np.float32)
        view_of = np.empty(self.max_faces, dtype=np.int32)
        scales = np.empty(max(nv, 1), dtype=np.float32)
        count = C.c_int(0)
        self._check(self.lib.rf_detect_views(self.h, C.c_void_p(img.ctypes.data), img.shape[1], img.shape[0], 0, varr, nv, C.c_float(thr),
                                             C.c_float(nms), C.c_void_p(faces.ctypes.data), C.byref(count),
                                             C.c_void_p(view_of.ctypes.data), C.c_void_p(scales.ctypes.data)))
        return faces[:count.value].copy(), view_of[:count.value].copy(), scales[:nv].copy()

    # -- f9 rotated and mirrored images (EXIF orientations 1..8) ---------------------------------------------------------------
    def detect_oriented(self, images: Sequence[np.ndarray], orientations: Sequence[int], thr: float, nms_thr: float, align: Optional[dict] = None,
                        want_index: bool = False):
        """rf_detect_oriented_batch: u8 BGR HWC images as STORED (any size <= max_image; rows may be strided), image i shown in EXIF
        orientation orientations[i].  Returns one (k, 15) float32 array per image in DISPLAYED image pixels -- detect_align's faces
        on T_o(img) -- without a rotated copy ever being made.  align: detect_align's keywords -> (faces, crops[, mats]), the crops
        cut from the displayed image.  want_index appends the anchor-index arrays."""
        n = len(images)
        keep, ptrs, ws, hs, rs = self._host_images(images)
        arr = _orientations(orientations, n)
        faces, counts, idx = self._outputs(n, want_index)
        p, A, crops, mats = self._host_align(n, align) if align is not None else (None, 0, None, None)
        self._check(self.lib.rf_detect_oriented_batch(self.h, ptrs, ws, hs, rs, arr, n, thr, nms_thr, _ref(p), faces.ctypes.data,
                                                      counts.ctypes.data, _addr(idx), _addr(crops), _addr(mats)))
        return self._result(counts, faces, A=A, crops=crops, mats=mats, idx=idx)

    def detect_yuv_oriented_device(self, frames, orientations: Sequence[int], thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601",
                                   align: Optional[dict] = None, dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_yuv_oriented_device: detect_yuv_device on frames shown in EXIF orientation orientations[i] (portrait NVDEC surfaces).
        Returns (dets_ptr, counts_ptr, map-back scale of each displayed frame); detections in network-input pixels of the displayed
        frame.  Host frames: ValueError."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        o = _orientations(orientations, n)
        p = align_params(**align) if align is not None else None
        scales = np.zeros(max(n, 1), dtype=np.float32)
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_yuv_oriented_device(self.h, arr, o, n, _matrix(matrix), thr, nms_thr, _ref(p),
                                                           dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c), scales.ctypes.data))
        return int(d.value or 0), int(c.value or 0), scales[:n].copy()

    def preprocess_oriented(self, img: np.ndarray, orientation: int) -> np.ndarray:
        """rf_preprocess_oriented: the (H, W, 3) u8 BGR letter-box of the image shown in EXIF orientation `orientation`."""
        img = self._bgr_strided(img)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        self._check(self.lib.rf_preprocess_oriented(self.h, img.ctypes.data, img.shape[1], img.shape[0], img.strides[0], int(orientation),
                                                    out.ctypes.data))
        return out

    def preprocess_yuv_oriented(self, frame, orientation: int, layout: str = "nv12", matrix="bt601") -> np.ndarray:
        """rf_preprocess_yuv_oriented: the letter-box of one host frame shown in EXIF orientation `orientation`."""
        arr = self._frames([frame], layout, False)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        self._check(self.lib.rf_preprocess_yuv_oriented(self.h, arr, _matrix(matrix), int(orientation), out.ctypes.data))
        return out

    def detect_views_oriented(self, img: np.ndarray, views, thr: float, nms: float):
        """rf_detect_views_oriented: one image, views = [(shrink, orientation), ...] run as one batch, mapped back into STORED image
        pixels and merged on the GPU.  Returns (faces [k, 15], view index of each face [k], map-back scale of each view)."""
        img = self._bgr_strided(img)
        nv = len(views)
        varr = (_OrientedView * max(nv, 1))(*[_OrientedView(float(s), int(o)) for s, o in views])
        faces = np.empty((self.max_faces, 15), dtype=np.float32)
        view_of = np.empty(self.max_faces, dtype=np.int32)
        scales = np.empty(max(nv, 1), dtype=np.float32)
        count = C.c_int(0)
        self._check(self.lib.rf_detect_views_oriented(self.h, C.c_void_p(img.ctypes.data), img.shape[1], img.shape[0], img.strides[0], varr, nv,
                                                      C.c_float(thr), C.c_float(nms), C.c_void_p(faces.ctypes.data), C.byref(count),
                                                      C.c_void_p(view_of.ctypes.data), C.c_void_p(scales.ctypes.data)))
        return faces[:count.value].copy(), view_of[:count.value].copy(), scales[:nv].copy()

    # -- f23 faces at any in-plane angle ---------------------------------------------------------------------------------------
    def detect_views_rotated(self, img: np.ndarray, views, thr: float, nms: float, align: Optional[dict] = None):
        """rf_detect_views_rotated: one image, views = [(angle, shrink), ...] (degrees counter-clockwise), run in batches of up to
        max_batch and merged on the GPU.  Returns (faces [k, 15] in image pixels, view index of each face [k], map-back scale of each
        view, M of each view [nviews, 2, 3], zeros for quarter turns); align: detect_align's keywords -> crops [min(k, A), ...]
        [and mats [min(k, A), 2, 3]] appended, cut from the image."""
        img = self._bgr_strided(img)
        nv = len(views)
        varr = (_RotatedView * max(nv, 1))(*[_RotatedView(float(a), float(s)) for a, s in views])
        faces = np.empty((self.max_faces, 15), dtype=np.float32)
        view_of = np.empty(self.max_faces, dtype=np.int32)
        scales = np.empty(max(nv, 1), dtype=np.float32)
        mats = np.empty((max(nv, 1), 2, 3), dtype=np.float64)
        p, A, crops, cmats = self._host_align(1, align) if align is not None else (None, 0, None, None)
        count = C.c_int(0)
        self._check(self.lib.rf_detect_views_rotated(self.h, img.ctypes.data, img.shape[1], img.shape[0], img.strides[0], varr, nv, C.c_float(thr),
                                                     C.c_float(nms), _ref(p), faces.ctypes.data, C.byref(count), view_of.ctypes.data,
                                                     scales.ctypes.data, mats.ctypes.data, _addr(crops), _addr(cmats)))
        k = count.value
        out = (faces[:k].copy(), view_of[:k].copy(), scales[:nv].copy(), mats[:nv].copy())
        if align is None:
            return out
        out += (crops[0, :min(k, A)].copy(),)
        return out + (cmats[0, :min(k, A)].copy(),) if cmats is not None else out

    def preprocess_rotated(self, img: np.ndarray, angle: float, shrink: float = 1.0):
        """rf_preprocess_rotated: (the (H, W, 3) u8 BGR network input of the view (angle, shrink), its M [2, 3], zeros for a quarter turn)."""
        img = self._bgr_strided(img)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        mat = np.empty((2, 3), dtype=np.float64)
        self._check(self.lib.rf_preprocess_rotated(self.h, img.ctypes.data, img.shape[1], img.shape[0], img.strides[0], C.c_float(angle),
                                                   C.c_float(shrink), out.ctypes.data, mat.ctypes.data))
        return out, mat

    # -- f24 faces at any in-plane angle in device frames ------------------------------------------------------------------------
    def _rotated_device(self, fn, sources, n: int, views, thr: float, nms: float, align: Optional[dict], dev_crops_ptr, dev_mats_ptr):
        """One rotated device call: fn(sources..., views, nviews, thr, nms, align, crops, mats, &dets, &counts, scales, mats) ->
        (dets_ptr, counts_ptr, view scales [n, nviews], view M [n, nviews, 2, 3])."""
        nv = len(views)
        varr = (_RotatedView * max(nv, 1))(*[_RotatedView(float(a), float(s)) for a, s in views])
        p = align_params(**align) if align is not None else None
        scales = np.zeros((max(n, 1), max(nv, 1)), dtype=np.float32)
        mats = np.zeros((max(n, 1), max(nv, 1), 2, 3), dtype=np.float64)
        d, c = C.c_void_p(), C.c_void_p()
        self._check(fn(self.h, *sources, varr, nv, C.c_float(thr), C.c_float(nms), _ref(p), dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c),
                       scales.ctypes.data, mats.ctypes.data))
        return int(d.value or 0), int(c.value or 0), scales[:n, :nv].copy(), mats[:n, :nv].copy()

    def detect_views_rotated_device(self, images, views, thr: float, nms: float, align: Optional[dict] = None,
                                    dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_views_rotated_device: u8 BGR HWC torch CUDA tensors (rows may be strided), each run through the views
        [(angle, shrink), ...] of detect_views_rotated, asynchronous on last_stream_ptr().  Returns (dets_ptr, counts_ptr, map-back
        scale of each view [n, nviews], M of each view [n, nviews, 2, 3], zeros for quarter turns): [max_batch][max_faces] rf_det in
        IMAGE pixels, anchor_index = view * max_faces + rank, valid for `streams` further rotated device calls.  align:
        detect_align's keywords; the crops land at dev_crops_ptr as in detect_align_device.  Host arrays: ValueError."""
        ptrs, ws, hs, rs = self._device_images(images)
        return self._rotated_device(self.lib.rf_detect_views_rotated_device, (ptrs, ws, hs, rs, len(images)), len(images), views, thr, nms,
                                    align, dev_crops_ptr, dev_mats_ptr)

    def detect_yuv_views_rotated_device(self, frames, views, thr: float, nms: float, layout: str = "nv12", matrix="bt601",
                                        align: Optional[dict] = None, dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_yuv_views_rotated_device: device 4:2:0 frames (torch CUDA tensors in yuv_frame's forms), otherwise as
        detect_views_rotated_device (faces in FRAME pixels).  Host frames: ValueError."""
        arr = self._frames(frames, layout, True)
        return self._rotated_device(self.lib.rf_detect_yuv_views_rotated_device, (arr, len(frames), _matrix(matrix)), len(frames), views, thr,
                                    nms, align, dev_crops_ptr, dev_mats_ptr)

    def preprocess_yuv_rotated(self, frame, angle: float, shrink: float = 1.0, layout: str = "nv12", matrix="bt601"):
        """rf_preprocess_yuv_rotated: (the (H, W, 3) u8 BGR network input of the view (angle, shrink) of one host frame, its M [2, 3],
        zeros for a quarter turn)."""
        arr = self._frames([frame], layout, False)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        mat = np.empty((2, 3), dtype=np.float64)
        self._check(self.lib.rf_preprocess_yuv_rotated(self.h, arr, _matrix(matrix), C.c_float(angle), C.c_float(shrink), out.ctypes.data,
                                                       mat.ctypes.data))
        return out, mat

    # -- f21 tiled detection of rotated and mirrored images ---------------------------------------------------------------------
    def detect_tiled_oriented(self, images: Sequence[np.ndarray], orientations: Sequence[int], thr: float, nms_thr: float, levels=None,
                              overlap: int = 0, align: Optional[dict] = None):
        """rf_detect_tiled_oriented: detect_tiled on the images shown in EXIF orientation orientations[i] -- the layout, tiles,
        faces, tile_of and crops of the DISPLAYED image, without a rotated copy.  Returns what detect_tiled returns."""
        n = len(images)
        keep, ptrs, ws, hs, rs = self._host_images(images)
        o = _orientations(orientations, n)
        t = tiling(levels, overlap)
        faces, counts, tile_of = self._outputs(n, True)
        p, A, crops, mats = self._host_align(n, align) if align is not None else (None, 0, None, None)
        self._check(self.lib.rf_detect_tiled_oriented(self.h, ptrs, ws, hs, rs, o, n, C.byref(t), thr, nms_thr, _ref(p), faces.ctypes.data,
                                                      counts.ctypes.data, tile_of.ctypes.data, _addr(crops), _addr(mats)))
        return self._result(counts, faces, tile_of, A, crops, mats)

    def detect_tiled_oriented_device(self, images, orientations: Sequence[int], thr: float, nms_thr: float, levels=None, overlap: int = 0,
                                     align: Optional[dict] = None, dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_tiled_oriented_device: detect_tiled_device on images shown in EXIF orientation orientations[i]; records in
        DISPLAYED image pixels.  Returns (dets_ptr, counts_ptr)."""
        n = len(images)
        ptrs, ws, hs, rs = self._device_images(images)
        o = _orientations(orientations, n)
        t = tiling(levels, overlap)
        p = align_params(**align) if align is not None else None
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_tiled_oriented_device(self.h, ptrs, ws, hs, rs, o, n, C.byref(t), thr, nms_thr, _ref(p),
                                                             dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c)))
        return int(d.value or 0), int(c.value or 0)

    def detect_yuv_tiled_oriented_device(self, frames, orientations: Sequence[int], thr: float, nms_thr: float, layout: str = "nv12",
                                         matrix="bt601", levels=None, overlap: int = 0, align: Optional[dict] = None,
                                         dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_yuv_tiled_oriented_device: detect_yuv_tiled_device on frames shown in EXIF orientation orientations[i] (portrait
        4K NVDEC surfaces); records in DISPLAYED frame pixels.  Returns (dets_ptr, counts_ptr)."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        o = _orientations(orientations, n)
        t = tiling(levels, overlap)
        p = align_params(**align) if align is not None else None
        d, c = C.c_void_p(), C.c_void_p()
        self._check(self.lib.rf_detect_yuv_tiled_oriented_device(self.h, arr, o, n, _matrix(matrix), C.byref(t), thr, nms_thr, _ref(p),
                                                                 dev_crops_ptr, dev_mats_ptr, C.byref(d), C.byref(c)))
        return int(d.value or 0), int(c.value or 0)

    def preprocess_tile_oriented(self, img: np.ndarray, orientation: int, tile: int, levels=None, overlap: int = 0) -> np.ndarray:
        """rf_preprocess_tile_oriented: tile `tile` of the displayed image's layout as the network sees it, (H, W, 3) u8 BGR."""
        img = self._bgr_strided(img)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        t = tiling(levels, overlap)
        self._check(self.lib.rf_preprocess_tile_oriented(self.h, img.ctypes.data, img.shape[1], img.shape[0], img.strides[0], int(orientation),
                                                         C.byref(t), int(tile), out.ctypes.data))
        return out

    def preprocess_yuv_tile_oriented(self, frame, orientation: int, tile: int, layout: str = "nv12", matrix="bt601", levels=None,
                                     overlap: int = 0) -> np.ndarray:
        """rf_preprocess_yuv_tile_oriented: tile `tile` of the displayed frame's layout as the network sees it, (H, W, 3) u8 BGR."""
        arr = self._frames([frame], layout, False)
        out = np.empty((self.net_h, self.net_w, 3), dtype=np.uint8)
        t = tiling(levels, overlap)
        self._check(self.lib.rf_preprocess_yuv_tile_oriented(self.h, arr, _matrix(matrix), int(orientation), C.byref(t), int(tile),
                                                             out.ctypes.data))
        return out

    # -- f10 face tracking across video frames ---------------------------------------------------------------------------------
    def tracker(self, max_videos: int = 1, max_tracks: int = 0, high_thresh: float = 0.0, new_thresh: float = 0.0, iou_high: float = 0.0,
                iou_low: float = 0.0, iou_tentative: float = 0.0, max_lost: int = 0, best: Optional[dict] = None,
                motion=None, lookback=None, follow=None, lookback_search=None, lookback_follow=None, tiling=None, best_live=None,
                best_follow=None, views=None) -> "Tracker":
        """rf_tracker_create: a tracker of max_videos independent sequences on this engine (0 -> the defaults of rf_track_config).
        best (``best_config`` keywords): a best-shot tracker (rf_tracker_create_best), fed through ``Tracker.detect_yuv_best_device``.
        motion (True or ``motion_config`` keywords): camera-motion compensation (rf_tracker_set_motion) from the frames of the
        detect_yuv_* calls; read each call's estimates with ``Tracker.motion``.  lookback (True, L, or ``set_lookback`` keywords): a
        look-back tracker (rf_tracker_set_lookback), fed through ``Tracker.detect_yuv_redact_lookback_device``.  follow (True or
        ``set_follow`` keywords): a follow tracker (rf_tracker_set_follow), whose frames between detections go through
        ``Tracker.follow_device``.  lookback_search (True or ``set_lookback_search`` keywords, with lookback): a searching look-back
        tracker (rf_tracker_set_lookback_search).  lookback_follow (True or ``set_lookback_follow`` keywords, with lookback): a
        following look-back tracker (rf_tracker_set_lookback_follow), whose frames between detections go through
        ``Tracker.follow_redact_lookback_device``.  tiling (True or ``set_tiling`` keywords): a tiling tracker
        (rf_tracker_set_tiling), whose detect calls detect through the tiles of ``detect_yuv_tiled_device``.  best_live (True or
        ``set_best_live`` keywords, with best): live shots while tracks live (rf_tracker_set_best_live).  best_follow (True or
        ``set_best_follow`` keywords, with best): a following best-shot tracker (rf_tracker_set_best_follow), whose frames between
        detections go through ``Tracker.follow_best_device``.  views ([(angle, shrink), ...]): a views tracker
        (rf_tracker_set_views), whose detect calls detect through the rotated views of ``detect_yuv_views_rotated_device``."""
        t = Tracker(self, TrackConfig(max_videos, max_tracks, high_thresh, new_thresh, iou_high, iou_low, iou_tentative, max_lost),
                    best_config(**best) if best is not None else None)
        try:
            if motion:
                t.set_motion(**(motion if isinstance(motion, dict) else {}))
            if lookback:
                t.set_lookback(**(lookback if isinstance(lookback, dict) else {} if lookback is True else {"frames": int(lookback)}))
            if follow:
                t.set_follow(**(follow if isinstance(follow, dict) else {}))
            if lookback_search:
                t.set_lookback_search(**(lookback_search if isinstance(lookback_search, dict) else {}))
            if lookback_follow:
                t.set_lookback_follow(**(lookback_follow if isinstance(lookback_follow, dict) else {}))
            if tiling:
                t.set_tiling(**(tiling if isinstance(tiling, dict) else {}))
            if best_live:
                t.set_best_live(**(best_live if isinstance(best_live, dict) else {}))
            if best_follow:
                t.set_best_follow(**(best_follow if isinstance(best_follow, dict) else {}))
            if views is not None:
                t.set_views(views)
        except Exception:
            t.close()
            raise
        return t

    # -- f12 redaction ---------------------------------------------------------------------------------------------------------
    @staticmethod
    def _scales(scales, n):
        if scales is None:
            return None
        sc = np.ascontiguousarray(scales, dtype=np.float32)
        if sc.size != n:
            raise ValueError(f"{n} frames but {sc.size} scales")
        return sc

    def redact_yuv_device(self, frames, dets_ptr: int, counts_ptr: int, scales=None, layout: str = "nv12", tracker: Optional["Tracker"] = None,
                          tracks_ptr: Optional[int] = None, track_counts_ptr: Optional[int] = None, blocks: int = 0, margin: float = 0.0,
                          style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_redact_yuv_device: mosaic, IN PLACE, every region of the device 4:2:0 frames (torch CUDA tensors in yuv_frame's forms):
        the records at dets_ptr / counts_ptr of a device detect call (scales: each frame's map-back factor; None for records already
        in frame pixels) and, with a tracker, the LOST tracks of its lists at tracks_ptr / track_counts_ptr.  Asynchronous on
        last_stream_ptr().  style / shape / detail other than the defaults: rf_redact_yuv_device_style (see redact_style)."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        sc = self._scales(scales, n)
        fn, p = _redaction(self.lib, "rf_redact_yuv_device", style, shape, blocks, detail, margin)
        self._check(fn(self.h, arr, n, dets_ptr, counts_ptr, _addr(sc), tracker.t if tracker is not None else None, tracks_ptr,
                       track_counts_ptr, C.byref(p)))

    def redact_yuv_oriented_device(self, frames, orientations: Sequence[int], dets_ptr: int, counts_ptr: int, scales=None, layout: str = "nv12",
                                   tracker: Optional["Tracker"] = None, tracks_ptr: Optional[int] = None, track_counts_ptr: Optional[int] = None,
                                   blocks: int = 0, margin: float = 0.0, style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_redact_yuv_oriented_device_style: redact_yuv_device of frames shown in EXIF orientation orientations[i], from the
        displayed-pixel records of ``detect_yuv_oriented_device`` (scales: its out_scales) and, with a tracker, the LOST tracks of
        lists fed those records.  The frames are redacted in place as displayed; every other byte stays as it was."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        o = _orientations(orientations, n)
        sc = self._scales(scales, n)
        st = redact_style(style, shape, blocks, detail, margin)
        if st is None:
            st = RedactStyle(RF_REDACT_MOSAIC, RF_REDACT_RECT, int(blocks), 0, float(margin))
        self._check(self.lib.rf_redact_yuv_oriented_device_style(self.h, arr, o, n, dets_ptr, counts_ptr, _addr(sc),
                                                                 tracker.t if tracker is not None else None, tracks_ptr, track_counts_ptr,
                                                                 C.byref(st)))

    def redact_device(self, images, dets_ptr: int, counts_ptr: int, scales=None, tracker: Optional["Tracker"] = None,
                      tracks_ptr: Optional[int] = None, track_counts_ptr: Optional[int] = None, blocks: int = 0, margin: float = 0.0,
                      style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_redact_device: redact_yuv_device on u8 BGR HWC torch CUDA tensors (rows may be strided), in place."""
        n = len(images)
        ptrs, ws, hs, rs = self._device_images(images)
        sc = self._scales(scales, n)
        fn, p = _redaction(self.lib, "rf_redact_device", style, shape, blocks, detail, margin)
        self._check(fn(self.h, ptrs, ws, hs, rs, n, dets_ptr, counts_ptr, _addr(sc), tracker.t if tracker is not None else None, tracks_ptr,
                       track_counts_ptr, C.byref(p)))

    def detect_yuv_redact_device(self, frames, thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601", blocks: int = 0,
                                 margin: float = 0.0, style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_detect_yuv_redact_device without a tracker: detect_yuv_device, then redact_yuv_device of its records on the same
        context.  Returns (dets_ptr, counts_ptr, scales) as detect_yuv_device; the frames are redacted in place."""
        n = len(frames)
        arr = self._frames(frames, layout, True)
        fn, p = _redaction(self.lib, "rf_detect_yuv_redact_device", style, shape, blocks, detail, margin)
        scales = np.zeros(max(n, 1), dtype=np.float32)
        d, c = C.c_void_p(), C.c_void_p()
        self._check(fn(self.h, None, arr, None, n, _matrix(matrix), thr, nms_thr, C.byref(p), None, None, C.byref(d), C.byref(c),
                       scales.ctypes.data))
        return int(d.value or 0), int(c.value or 0), scales[:n].copy()

    def calibrate_int8(self, images: np.ndarray, out_table: str):
        """INT8 entropy calibration on an RF_PREC_FP32 engine; writes a TensorRT-format table."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        assert images.shape[1:] == (self.net_h, self.net_w, 3)
        self._check(self.lib.rf_calibrate_int8(self.h, images.ctypes.data, images.shape[0], out_table.encode()))

    def debug_keep_all(self):
        self._check(self.lib.rf_debug_keep_all(self.h))

    def debug_tensor(self, name: str, n: int) -> np.ndarray:
        c, hh, ww = C.c_int(), C.c_int(), C.c_int()
        self._check(self.lib.rf_debug_get_tensor(self.h, name.encode(), n, None, C.byref(c), C.byref(hh), C.byref(ww)))
        out = np.empty((n, c.value, hh.value, ww.value), dtype=np.float32)
        self._check(self.lib.rf_debug_get_tensor(self.h, name.encode(), n, out.ctypes.data, C.byref(c), C.byref(hh), C.byref(ww)))
        return out

    def launches_per_batch(self, n: int) -> int:
        return self._check(self.lib.rf_launches_per_batch(self.h, n))

    def profile_layers(self, n: int, iters: int = 20):
        cap = 128
        names = C.create_string_buffer(64 * cap)
        ms = (C.c_float * cap)()
        by = (C.c_double * cap)()
        fl = (C.c_double * cap)()
        k = self._check(self.lib.rf_profile_layers(self.h, n, iters, names, ms, by, fl, cap))
        out = []
        for i in range(k):
            nm = names.raw[64 * i:64 * (i + 1)].split(b"\0", 1)[0].decode()
            out.append(dict(name=nm, ms=float(ms[i]), bytes=float(by[i]), flops=float(fl[i])))
        return out


class Tracker:
    """One rf_tracker of an Engine: per-video face tracks with stable ids, updated on the GPU.  Close it before its engine."""

    def __init__(self, engine: Engine, cfg: TrackConfig, best: Optional[BestConfig] = None):
        self.engine, self.lib = engine, engine.lib
        t = C.c_void_p()
        if best is None:
            engine._check(self.lib.rf_tracker_create(engine.h, C.byref(cfg), C.byref(t)))
        else:
            engine._check(self.lib.rf_tracker_create_best(engine.h, C.byref(cfg), C.byref(best), C.byref(t)))
        self.t = t
        self.best = best
        self.motion_on = False
        self.lookback = 0            # L of a look-back tracker
        self.follow_on = False
        self.lookback_search_on = False
        self.lookback_follow_on = False
        self.tiling_on = False
        self.views_on = False
        self.best_live_on = False
        self.best_follow_on = False
        self.max_videos = cfg.max_videos
        self.max_tracks = cfg.max_tracks or 64

    def close(self):
        if getattr(self, "t", None):
            self.lib.rf_tracker_destroy(self.t)
            self.t = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _ints(vals, n):
        v = [int(x) for x in vals]
        if len(v) != n:
            raise ValueError(f"{n} frames but {len(v)} video indices")
        return (C.c_int * max(n, 1))(*v)

    def update(self, videos: Sequence[int], dets_ptr: int, counts_ptr: int, scales=None):
        """rf_track_update on the device records of a detect call (frame i of video videos[i]; scales: the map-back factor of each
        frame, None for records already in image pixels).  Asynchronous.  Returns the (tracks_ptr, track_counts_ptr) device addresses."""
        n = len(videos)
        sc = self.engine._scales(scales, n)
        tp, cp = C.c_void_p(), C.c_void_p()
        self.engine._check(self.lib.rf_track_update(self.t, self._ints(videos, n), n, dets_ptr, counts_ptr, _addr(sc), C.byref(tp), C.byref(cp)))
        return int(tp.value or 0), int(cp.value or 0)

    def detect_yuv_device(self, frames, videos: Sequence[int], thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601",
                          align: Optional[dict] = None, dev_crops_ptr: Optional[int] = None, dev_mats_ptr: Optional[int] = None):
        """rf_detect_yuv_track_device: Engine.detect_yuv_device on device 4:2:0 frames, then the update; with align, the crops of the
        tracks confirmed on each frame at dev_crops_ptr [n][A].  Returns (tracks_ptr, track_counts_ptr, dets_ptr, counts_ptr, scales)."""
        n = len(frames)
        arr = self.engine._frames(frames, layout, True)
        p = align_params(**align) if align is not None else None
        scales = np.zeros(max(n, 1), dtype=np.float32)
        tp, tc, d, c = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        self.engine._check(self.lib.rf_detect_yuv_track_device(self.engine.h, self.t, arr, self._ints(videos, n), n, _matrix(matrix), thr, nms_thr,
                                                               _ref(p), dev_crops_ptr, dev_mats_ptr, C.byref(tp),
                                                               C.byref(tc), C.byref(d), C.byref(c), scales.ctypes.data))
        return int(tp.value or 0), int(tc.value or 0), int(d.value or 0), int(c.value or 0), scales[:n].copy()

    def detect_yuv_best_device(self, frames, videos: Sequence[int], thr: float, nms_thr: float, dev_best_crops_ptr: int,
                               dev_best_mats_ptr: Optional[int] = None, layout: str = "nv12", matrix="bt601"):
        """rf_detect_yuv_track_best_device on a best-shot tracker: detect, track, and keep every track's best crop; the shots emitted
        on frame i go to dev_best_crops_ptr [n][max_tracks] (and M to dev_best_mats_ptr [n][max_tracks][6]).  Returns (best_ptr,
        best_counts_ptr, tracks_ptr, track_counts_ptr, dets_ptr, counts_ptr, scales)."""
        n = len(frames)
        arr = self.engine._frames(frames, layout, True)
        scales = np.zeros(max(n, 1), dtype=np.float32)
        bp, bc, tp, tc, d, c = (C.c_void_p() for _ in range(6))
        self.engine._check(self.lib.rf_detect_yuv_track_best_device(self.engine.h, self.t, arr, self._ints(videos, n), n, _matrix(matrix), thr,
                                                                    nms_thr, dev_best_crops_ptr, dev_best_mats_ptr, C.byref(bp), C.byref(bc),
                                                                    C.byref(tp), C.byref(tc), C.byref(d), C.byref(c), scales.ctypes.data))
        return (int(bp.value or 0), int(bc.value or 0), int(tp.value or 0), int(tc.value or 0), int(d.value or 0), int(c.value or 0),
                scales[:n].copy())

    def detect_yuv_redact_device(self, frames, videos: Sequence[int], thr: float, nms_thr: float, layout: str = "nv12", matrix="bt601",
                                 blocks: int = 0, margin: float = 0.0, style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_detect_yuv_redact_device with this tracker: detect_yuv_device (no crops), the update, then the redaction of every record and
        every LOST track, in place.  Returns (tracks_ptr, track_counts_ptr, dets_ptr, counts_ptr, scales) as detect_yuv_device."""
        n = len(frames)
        arr = self.engine._frames(frames, layout, True)
        fn, p = _redaction(self.lib, "rf_detect_yuv_redact_device", style, shape, blocks, detail, margin)
        scales = np.zeros(max(n, 1), dtype=np.float32)
        tp, tc, d, c = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        self.engine._check(fn(self.engine.h, self.t, arr, self._ints(videos, n), n, _matrix(matrix), thr, nms_thr, C.byref(p), C.byref(tp),
                              C.byref(tc), C.byref(d), C.byref(c), scales.ctypes.data))
        return int(tp.value or 0), int(tc.value or 0), int(d.value or 0), int(c.value or 0), scales[:n].copy()

    def finish(self, video: int, dev_best_crops_ptr: int, dev_best_mats_ptr: Optional[int] = None):
        """rf_tracker_finish: emit the best shot of every live, ever-confirmed track of `video` (crops at dev_best_crops_ptr
        [max_tracks]), then restart the video.  Returns (best_ptr, count_ptr); read them with ``read_best(..., 1)``."""
        bp, bc = C.c_void_p(), C.c_void_p()
        self.engine._check(self.lib.rf_tracker_finish(self.t, int(video), dev_best_crops_ptr, dev_best_mats_ptr, C.byref(bp), C.byref(bc)))
        return int(bp.value or 0), int(bc.value or 0)

    def read_best(self, best_ptr: int, counts_ptr: int, n: int) -> List[np.ndarray]:
        """The emitted shots of n frames (BEST_DTYPE records, id order), copied to the host after the last stream."""
        raw = self.engine._fetch(best_ptr, BEST_DTYPE, n, self.max_tracks)
        counts = self.engine._fetch(counts_ptr, np.int32, n)
        return [raw[i, :counts[i]].copy() for i in range(n)]

    def set_best_live(self, first_quality: float = 0.0, improve: float = 0.0, min_gap: int = 0):
        """rf_tracker_set_best_live, on a best-shot tracker before the first frame call: emit a track's stored shot while it lives
        (RF_BEST_LIVE) once q >= first_quality (0 -> 0.3), then whenever q beats the last live shot's by the factor 1 + improve (0 ->
        0.2) at least min_gap (0 -> 30) frames later."""
        cfg = BestLiveConfig(float(first_quality), float(improve), int(min_gap))
        self.engine._check(self.lib.rf_tracker_set_best_live(self.t, C.byref(cfg)))
        self.best_live_on = True

    def set_best_follow(self, search: int = 0, max_mad: float = 0.0):
        """rf_tracker_set_best_follow, on a best-shot tracker before the first frame call: cut f16's templates on the detect frames so
        that the frames in between can go through ``follow_best_device`` (search: R in template pixels, 0 -> 8; max_mad: 0 -> 24)."""
        cfg = FollowConfig(int(search), float(max_mad))
        self.engine._check(self.lib.rf_tracker_set_best_follow(self.t, C.byref(cfg)))
        self.best_follow_on = True

    def follow_best_device(self, frames, videos: Sequence[int], dev_best_crops_ptr: int, dev_best_mats_ptr: Optional[int] = None,
                           layout: str = "nv12"):
        """rf_track_follow_best_device on a following best-shot tracker: follow the faces of the device 4:2:0 frames by template
        search, then emit the EXIT shots of the tracks removed on them into dev_best_crops_ptr [n][max_tracks] (as
        ``detect_yuv_best_device``).  Returns (best_ptr, best_counts_ptr, tracks_ptr, track_counts_ptr)."""
        n = len(frames)
        arr = self.engine._frames(frames, layout, True)
        bp, bc, tp, tc = (C.c_void_p() for _ in range(4))
        self.engine._check(self.lib.rf_track_follow_best_device(self.t, arr, self._ints(videos, n), n, dev_best_crops_ptr, dev_best_mats_ptr,
                                                                C.byref(bp), C.byref(bc), C.byref(tp), C.byref(tc)))
        return int(bp.value or 0), int(bc.value or 0), int(tp.value or 0), int(tc.value or 0)

    def set_motion(self, search: int = 0, min_inliers: int = 0):
        """rf_tracker_set_motion, before the first update."""
        cfg = motion_config(search, min_inliers)
        self.engine._check(self.lib.rf_tracker_set_motion(self.t, C.byref(cfg)))
        self.motion_on = True

    def motion(self, n: int) -> np.ndarray:
        """rf_tracker_motion: the n rf_motion records (MOTION_DTYPE) of the latest frame call, copied after the last stream."""
        p = C.c_void_p()
        self.engine._check(self.lib.rf_tracker_motion(self.t, C.byref(p)))
        if not p.value:
            raise RuntimeError("no frame call has been made on this tracker")
        return self.engine._fetch(p.value, MOTION_DTYPE, n)

    def set_lookback(self, frames: int = 0, grow: float = 0.0):
        """rf_tracker_set_lookback, before the first update: keep each video's last L frames (0 -> 15) on the GPU and emit every frame L
        frames late, covered where the faces born after it already were (grow: the box growth per frame back, 0 -> 0.1)."""
        cfg = LookbackConfig(int(frames), float(grow))
        self.engine._check(self.lib.rf_tracker_set_lookback(self.t, C.byref(cfg)))
        self.lookback = cfg.frames or 15

    def detect_yuv_redact_lookback_device(self, frames, videos: Sequence[int], out_frames, thr: float, nms_thr: float, layout: str = "nv12",
                                          matrix="bt601", blocks: int = 0, margin: float = 0.0, style: str = "mosaic", shape: str = "rect",
                                          detail: int = 0):
        """rf_detect_yuv_redact_lookback_device: detect and track the device 4:2:0 frames, store them, and write frame num - L of each
        frame's video, redacted, into out_frames[i] (the same forms as frames, in `layout`; out_frames[i] may be frames[i] itself).
        Returns (out frame numbers (-1: nothing emitted), tracks_ptr, track_counts_ptr, dets_ptr, counts_ptr, scales)."""
        n = len(frames)
        if len(out_frames) != n:
            raise ValueError(f"{n} frames but {len(out_frames)} out frames")
        arr = self.engine._frames(frames, layout, True)
        outs = self.engine._frames(out_frames, layout, True)
        fn, st = _redaction(self.lib, "rf_detect_yuv_redact_lookback_device", style, shape, blocks, detail, margin)
        nums = np.full(max(n, 1), -1, dtype=np.int32)
        scales = np.zeros(max(n, 1), dtype=np.float32)
        tp, tc, d, c = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        self.engine._check(fn(self.engine.h, self.t, arr, self._ints(videos, n), n, _matrix(matrix), thr, nms_thr, C.byref(st), outs,
                              nums.ctypes.data, C.byref(tp), C.byref(tc), C.byref(d), C.byref(c), scales.ctypes.data))
        return nums[:n].copy(), int(tp.value or 0), int(tc.value or 0), int(d.value or 0), int(c.value or 0), scales[:n].copy()

    def set_lookback_search(self, search: int = 0, max_mad: float = 0.0):
        """rf_tracker_set_lookback_search, after ``set_lookback`` and before the first update: follow every new face back through the
        buffered frames by f16's template search and cover its path too (search: R in template pixels, 0 -> 8; max_mad: 0 -> 24)."""
        cfg = FollowConfig(int(search), float(max_mad))
        self.engine._check(self.lib.rf_tracker_set_lookback_search(self.t, C.byref(cfg)))
        self.lookback_search_on = True

    def lookback_search(self, n: int):
        """rf_tracker_lookback_search: the latest look-back call's [n][min(max_faces, max_tracks)][L] step records (FOLLOW_DTYPE) and
        [n][min(max_faces, max_tracks)] chain lengths, copied after the last stream."""
        p, q = C.c_void_p(), C.c_void_p()
        self.engine._check(self.lib.rf_tracker_lookback_search(self.t, C.byref(p), C.byref(q)))
        if not p.value:
            raise RuntimeError("no look-back call has been made on this tracker")
        bcap = min(self.engine.max_faces, self.max_tracks)
        return self.engine._fetch(p.value, FOLLOW_DTYPE, n, bcap, self.lookback), self.engine._fetch(q.value, np.int32, n, bcap)

    def set_lookback_follow(self, search: int = 0, max_mad: float = 0.0):
        """rf_tracker_set_lookback_follow, after ``set_lookback`` and before the first update: cut f16's templates on the detect frames
        so that the frames in between can go through ``follow_redact_lookback_device`` (search: R in template pixels, 0 -> 8; max_mad:
        0 -> 24)."""
        cfg = FollowConfig(int(search), float(max_mad))
        self.engine._check(self.lib.rf_tracker_set_lookback_follow(self.t, C.byref(cfg)))
        self.lookback_follow_on = True

    def follow_redact_lookback_device(self, frames, videos: Sequence[int], out_frames, layout: str = "nv12", blocks: int = 0,
                                      margin: float = 0.0, style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_track_follow_redact_lookback_device on a following look-back tracker: follow the faces of the device 4:2:0 frames by
        template search, store the frames, and write frame num - L of each frame's video, redacted, into out_frames[i] (as
        ``detect_yuv_redact_lookback_device``).  Returns (out frame numbers (-1: nothing emitted), tracks_ptr, track_counts_ptr)."""
        n = len(frames)
        if len(out_frames) != n:
            raise ValueError(f"{n} frames but {len(out_frames)} out frames")
        arr = self.engine._frames(frames, layout, True)
        outs = self.engine._frames(out_frames, layout, True)
        fn, st = _redaction(self.lib, "rf_track_follow_redact_lookback_device", style, shape, blocks, detail, margin)
        nums = np.full(max(n, 1), -1, dtype=np.int32)
        tp, tc = C.c_void_p(), C.c_void_p()
        self.engine._check(fn(self.t, arr, self._ints(videos, n), n, C.byref(st), outs, nums.ctypes.data, C.byref(tp), C.byref(tc)))
        return nums[:n].copy(), int(tp.value or 0), int(tc.value or 0)

    def drain(self, video: int, out_frames, layout: str = "nv12", blocks: int = 0, margin: float = 0.0, style: str = "mosaic",
              shape: str = "rect", detail: int = 0) -> np.ndarray:
        """rf_tracker_drain: write the video's buffered frames (at most L, in frame order) into out_frames[0..), then restart the video.
        Returns the numbers of the frames written."""
        k = len(out_frames)
        outs = self.engine._frames(out_frames, layout, True) if k else None
        fn, st = _redaction(self.lib, "rf_tracker_drain", style, shape, blocks, detail, margin)
        nums = np.zeros(max(k, 1), dtype=np.int32)
        n_out = C.c_int(0)
        self.engine._check(fn(self.t, int(video), C.byref(st), outs, k, C.byref(n_out), nums.ctypes.data))
        return nums[:n_out.value].copy()

    def set_follow(self, search: int = 0, max_mad: float = 0.0):
        """rf_tracker_set_follow, before the first update: cut a luma template of every track on its detection frames, so that the
        frames in between can go through ``follow_device`` (search: R in template pixels, 0 -> 8; max_mad: 0 -> 24)."""
        cfg = FollowConfig(int(search), float(max_mad))
        self.engine._check(self.lib.rf_tracker_set_follow(self.t, C.byref(cfg)))
        self.follow_on = True

    def follow_device(self, frames, videos: Sequence[int], layout: str = "nv12"):
        """rf_track_follow_device: move every track of the device 4:2:0 frames' videos by template search, without the detector.
        Asynchronous.  Returns the (tracks_ptr, track_counts_ptr) device addresses; read them with ``read``."""
        n = len(frames)
        arr = self.engine._frames(frames, layout, True)
        tp, tc = C.c_void_p(), C.c_void_p()
        self.engine._check(self.lib.rf_track_follow_device(self.t, arr, self._ints(videos, n), n, C.byref(tp), C.byref(tc)))
        return int(tp.value or 0), int(tc.value or 0)

    def follow_redact_device(self, frames, videos: Sequence[int], layout: str = "nv12", blocks: int = 0, margin: float = 0.0,
                             style: str = "mosaic", shape: str = "rect", detail: int = 0):
        """rf_track_follow_redact_device: follow_device, then redact the frames IN PLACE over every OK-followed face and every LOST
        track (``redact_style``'s keywords).  Returns the (tracks_ptr, track_counts_ptr) device addresses."""
        n = len(frames)
        arr = self.engine._frames(frames, layout, True)
        fn, st = _redaction(self.lib, "rf_track_follow_redact_device", style, shape, blocks, detail, margin)
        tp, tc = C.c_void_p(), C.c_void_p()
        self.engine._check(fn(self.t, arr, self._ints(videos, n), n, C.byref(st), C.byref(tp), C.byref(tc)))
        return int(tp.value or 0), int(tc.value or 0)

    def follow(self, n: int) -> np.ndarray:
        """rf_tracker_follow: the [n][max_tracks] rf_follow records (FOLLOW_DTYPE) of the latest follow call (of a follow or a
        following look-back tracker), each frame's in its track-list order, copied after the last stream."""
        p = C.c_void_p()
        self.engine._check(self.lib.rf_tracker_follow(self.t, C.byref(p)))
        if not p.value:
            raise RuntimeError("no follow call has been made on this tracker")
        return self.engine._fetch(p.value, FOLLOW_DTYPE, n, self.max_tracks)

    def set_tiling(self, levels=None, overlap: int = 0):
        """rf_tracker_set_tiling, before the first update: every detect call of this tracker detects its frames through the tiles of
        ``Engine.detect_yuv_tiled_device`` (levels: [(scale, flip), ...], None -> the default pyramid; overlap 0 -> 64).  Its records
        are then in frame pixels, with scales all 1."""
        t = tiling(levels, overlap)
        self.engine._check(self.lib.rf_tracker_set_tiling(self.t, C.byref(t)))
        self.tiling_on = True

    def set_views(self, views):
        """rf_tracker_set_views, before the first update: every detect call of this tracker detects its frames through the rotated views
        [(angle, shrink), ...] of ``Engine.detect_yuv_views_rotated_device`` (the views are copied).  Its records are then in frame
        pixels (an oriented video's: displayed pixels), anchor_index // max_faces the view, with scales all 1."""
        views = list(views)
        varr = (_RotatedView * max(len(views), 1))(*[_RotatedView(float(a), float(s)) for a, s in views])
        self.engine._check(self.lib.rf_tracker_set_views(self.t, varr, len(views)))
        self.views_on = True

    def set_orientation(self, video: int, orientation: int):
        """rf_tracker_set_orientation: show video (-1: every video) in EXIF orientation 1..8 from its next frame call on, before its
        first frame call since create, reset, drain or finish.  Every frame call then reads and writes that video's frames as displayed
        (portrait phone video stored as landscape surfaces), with records and tracks in displayed pixels."""
        self.engine._check(self.lib.rf_tracker_set_orientation(self.t, int(video), int(orientation)))

    def reset(self, video: int = -1):
        """rf_tracker_reset: restart one video (ids from 1), or all with -1; ordered after every issued update."""
        self.engine._check(self.lib.rf_tracker_reset(self.t, int(video)))

    def debug_state(self, video: int):
        """rf_tracker_debug_state (blocking): (header [live, next id, frames, overflow], (live, 25) float64 per-track rows in id order)."""
        cap = 4 + TRACK_DEBUG_DOUBLES * self.max_tracks
        out = np.zeros(cap, dtype=np.float64)
        k = self.engine._check(self.lib.rf_tracker_debug_state(self.t, int(video), out.ctypes.data, cap))
        return out[:4].copy(), out[4:4 + k * TRACK_DEBUG_DOUBLES].reshape(k, TRACK_DEBUG_DOUBLES).copy()

    def read(self, tracks_ptr: int, counts_ptr: int, n: int) -> List[np.ndarray]:
        """The track lists of n frames of an update's outputs (TRACK_DTYPE records), copied to the host after the last stream."""
        raw = self.engine._fetch(tracks_ptr, TRACK_DTYPE, n, self.max_tracks)
        counts = self.engine._fetch(counts_ptr, np.int32, n)
        return [raw[i, :counts[i]].copy() for i in range(n)]
