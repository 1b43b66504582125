"""GPU (-m gpu): f21 oriented tiled detection.  Every case runs an oriented tiled call on stored images S against the unoriented tiled
twin on the materialised displayed copies orient(S, o) / orient_planes(S, o) (oracle/orient.py) and holds them equal bit
for bit: tile bytes, records, out_tile_of / anchor_index, crops and matrices.  Also: the small faces of a portrait 4K canvas that
neither the stored-frame tiles nor the oriented letter-box find, tracking and redaction of a portrait 4K video from these records,
calls in flight, every refusal with nothing changed, that nothing else changes, and the Python and C++ drivers."""
import ctypes as C
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.orient import INVERSE, orient, orient_planes, unorient_planes
from oracle.yuv import bgr_to_frame, frame_to_bgr
from tile_oracle import level_image, tile_bytes

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
F32 = np.float32
ALL = list(range(1, 9))
LEVELS = [(1.0, 0), (0.5, 1), (0.0, 0)]          # a mirrored level: on a non-square image at 5..8 it catches un-mirroring by stored width
INVALID, UNSUPPORTED = -1, -7
SEAMS = dict(levels=[(1.0, 0)], overlap=96)       # f7's seam protocol: every face below the overlap is whole in exactly one tile


def _engine(prec="fp16", **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (3840, 3840))       # landscape 4K and its materialised portrait twin
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), 448, 448, precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _cuda(a):
    """A device copy, complete before the library's streams (which do not wait for torch's) read it."""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    torch.cuda.synchronize()
    return t


def _layout(img, levels=None, overlap=0):
    from retinaface_b200 import capi
    return capi.tile_layout(448, 448, img.shape[1], img.shape[0], levels, overlap)


def _same(a, b, what):
    """Two (faces, tile_of[, crops[, mats]]) results, bit for bit."""
    for x, y in zip(a, b):
        assert len(x) == len(y), what
        for i, (p, q) in enumerate(zip(x, y)):
            assert p.shape == q.shape and (p.tobytes() == q.tobytes() if p.dtype == q.dtype else np.array_equal(p, q)), (what, i)


# ---- 1. tile bytes ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("o", ALL)
def test_tile_bytes_equal_the_rotated_copy(eng, golden_image, o):
    """Every tile of levels {0.37, 0.5, 1, 1.5, 2.75}, plain and mirrored, plus the fitted level: rf_preprocess_tile_oriented ==
    rf_preprocess_tile(orient(img, o)) == the slice of cv2.resize(cv2.flip(orient(img, o))) byte for byte, on the golden photo,
    517 x 333 and 519 x 335 (sides of 3 mod 4 at s = 0.5 in displayed geometry), and row-strided pageable and pinned copies."""
    import torch
    rng = np.random.default_rng(20 + o)
    odd, odd3 = rng.integers(0, 256, (333, 517, 3), np.uint8), rng.integers(0, 256, (335, 519, 3), np.uint8)
    big = np.full((886, 1301, 3), 0x5A, np.uint8)
    big[:, :1280] = golden_image
    pinned_t = torch.empty((886, 1300, 3), dtype=torch.uint8, pin_memory=True)
    pinned = pinned_t.numpy()
    pinned[:, :1280] = golden_image
    for name, img, src in (("golden", golden_image, golden_image), ("odd3", odd3, odd3), ("odd", odd, odd),
                           ("strided", golden_image, big[:, :1280]), ("pinned", golden_image, pinned[:, :1280])):
        shown = orient(img, o)
        for flip in (0, 1):
            levels = [(s, flip) for s in (0.37, 0.5, 1.0, 1.5, 2.75)] + [(0.0, flip)]
            cache = {}
            for k, t in enumerate(_layout(shown, levels, 64)):
                if t["scale"] and t["level"] not in cache:
                    cache[t["level"]] = level_image(shown, t["scale"], t["flip"])
                want = tile_bytes(shown, t, 448, 448, cache.get(t["level"]))
                got = eng.preprocess_tile_oriented(src, o, k, levels, 64)
                assert np.array_equal(got, want), (name, o, flip, k, t)
                assert np.array_equal(eng.preprocess_tile(shown, k, levels, 64), got), (name, o, flip, k)
            if name in ("strided", "pinned"):
                break              # their mirrored levels run the golden photo's kernel path


@pytest.mark.parametrize("layout,matrix", [("nv12", "bt601"), ("i420", "bt709")])
def test_yuv_tile_bytes_equal_the_rotated_frame(eng, golden_image, layout, matrix):
    """rf_preprocess_yuv_tile_oriented == rf_preprocess_yuv_tile(orient_planes(frame, o)) on a 1920 x 1080 frame and a random 1038 x 670
    one, all 8 orientations, levels {1.5, 1 mirrored, 0.5, 0.5 mirrored, fitted}; for 1, 6 also == the host tiles of the converted
    displayed frame."""
    rng = np.random.default_rng(8)
    frames = [bgr_to_frame(cv2.resize(golden_image, (1920, 1080)), layout), rng.integers(0, 256, (670 * 3 // 2, 1038), dtype=np.uint8)]
    levels = [(1.5, 0), (1.0, 1), (0.5, 0), (0.5, 1), (0.0, 0)]
    for fi, frame in enumerate(frames):
        for o in ALL:
            shown = orient_planes(frame, layout, o)
            bgr = frame_to_bgr(shown, layout, matrix) if o in (1, 6) else None
            cache = {}
            for k, t in enumerate(_layout(orient(frame_to_bgr(frame, layout, matrix), o), levels)):
                got = eng.preprocess_yuv_tile_oriented(frame, o, k, layout, matrix, levels)
                assert np.array_equal(got, eng.preprocess_yuv_tile(shown, k, layout, matrix, levels)), (layout, fi, o, k)
                if bgr is not None:
                    if t["scale"] and t["level"] not in cache:
                        cache[t["level"]] = level_image(bgr, t["scale"], t["flip"])
                    assert np.array_equal(got, tile_bytes(bgr, t, 448, 448, cache.get(t["level"]))), (layout, fi, o, k)


# ---- 2. records ---------------------------------------------------------------------------------------------------------------------
def _mixed(golden_image, n):
    """n images of mixed sizes (4K, the photo, 1279 x 887, noise, a crop) and mixed orientations (all 8 among n = 8)."""
    rng = np.random.default_rng(n)
    pool = [cv2.resize(golden_image, (3840, 2160)), golden_image, cv2.resize(golden_image, (1279, 887)), golden_image[100:700, 200:1100].copy(),
            rng.integers(0, 256, (500, 700, 3), np.uint8), cv2.resize(golden_image, (1920, 1080)), golden_image[:, ::-1].copy(), golden_image]
    if n == 1:
        return [golden_image], [6]
    return pool[:n], {3: [6, 5, 8], 8: [6, 3, 8, 5, 1, 7, 2, 4]}[n]


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
@pytest.mark.parametrize("n", [1, 3, 8])
def test_records_equal_the_rotated_copies(golden_image, prec, n):
    """rf_detect_tiled_oriented == rf_detect_tiled on orient(img, o): faces, counts and out_tile_of bit for bit, with the default
    pyramid and with levels {1, 0.5 mirrored, fitted}; at orientation 1 it equals rf_detect_tiled on the stored images."""
    imgs, os_ = _mixed(golden_image, n)
    e = _engine(prec)
    try:
        for levels in (None, LEVELS):
            got = e.detect_tiled_oriented(imgs, os_, THR, NMS, levels=levels)
            want = e.detect_tiled([orient(im, o) for im, o in zip(imgs, os_)], THR, NMS, levels=levels)
            _same(got, want, (prec, n, levels))
            assert sum(len(f) for f in got[0]) >= 3 * min(n, 3)
            _same(e.detect_tiled_oriented(imgs, [1] * n, THR, NMS, levels=levels), e.detect_tiled(imgs, THR, NMS, levels=levels),
                  (prec, n, levels, "o=1"))
    finally:
        e.close()


# ---- 3. crops -----------------------------------------------------------------------------------------------------------------------
def _warp(img, M, size=(112, 112)):
    return cv2.warpAffine(img, M, size, flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def test_crops_equal_the_rotated_copy(eng, golden_image):
    """u8 / F32 / F16 crops and M of rf_detect_tiled_oriented(align) equal rf_detect_tiled_align's on orient(img, o), faces and
    tile_of equal the call without crops, and each u8 crop == cv2.warpAffine(orient(img, o), M) byte for byte; all 8 orientations,
    two images per call."""
    imgs = [golden_image, cv2.resize(golden_image, (1279, 887))]
    for o in ALL:
        os_ = [o, 9 - o]
        shown = [orient(im, x) for im, x in zip(imgs, os_)]
        plain = eng.detect_tiled_oriented(imgs, os_, THR, NMS, levels=LEVELS)
        for fmt in ("bgr_u8", "rgb_f32", "rgb_f16"):
            got = eng.detect_tiled_oriented(imgs, os_, THR, NMS, levels=LEVELS, align=dict(fmt=fmt, want_mats=True))
            want = eng.detect_tiled(shown, THR, NMS, levels=LEVELS, align=dict(fmt=fmt, want_mats=True))
            _same(got, want, (o, fmt))
            _same(got[:2], plain, (o, fmt, "plain"))
            if fmt == "bgr_u8":
                for i in range(2):
                    assert len(got[2][i]) >= 3
                    for crop, M in zip(got[2][i], got[3][i]):
                        assert np.array_equal(crop, _warp(shown[i], M)), (o, i)


# ---- 4. device calls ----------------------------------------------------------------------------------------------------------------
def _nvdec_like(frame, pitch, coded_h):
    """NV12 on the device as NVDEC maps it: luma rows of `pitch` bytes, the chroma plane at pitch * coded height, padding 0xEE."""
    import torch
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]
    surf = torch.full((coded_h + coded_h // 2, pitch), 0xEE, dtype=torch.uint8, device="cuda")
    surf[:h, :w] = _cuda(frame[:h])
    surf[coded_h:coded_h + h // 2, :w] = _cuda(frame[h:])
    torch.cuda.synchronize()
    return (surf[:h, :w], surf[coded_h:coded_h + h // 2, :w]), surf


def _read_crops(buf, counts):
    return [buf[i, :k].cpu().numpy() for i, k in enumerate(counts)]


def test_device_bgr_equals_the_rotated_copies(eng, golden_image):
    """rf_detect_tiled_oriented_device on device images (one a row-strided view) == rf_detect_tiled_device on device copies of
    orient(img, o): records, crops and matrices bit for bit; == the blocking oriented call; the inputs are unchanged."""
    import torch
    imgs = [cv2.resize(golden_image, (3840, 2160)), golden_image, cv2.resize(golden_image, (1279, 887)), golden_image]
    os_ = [6, 8, 5, 7]
    big = torch.full((886, 1300, 3), 0x5A, dtype=torch.uint8, device="cuda")
    big[:, :1280] = _cuda(golden_image)
    dev = [_cuda(im) for im in imgs[:-1]] + [big[:, :1280]]
    twin = [_cuda(orient(im, o)) for im, o in zip(imgs, os_)]
    sums = [int(t.to(torch.int64).sum()) for t in dev] + [int(big.to(torch.int64).sum())]
    A, mf = eng.max_faces, eng.max_faces
    for levels in (LEVELS, None):
        out = []
        for oriented in (True, False):
            crops = torch.full((4, A, 112, 112, 3), 7, dtype=torch.uint8, device="cuda")
            mats = torch.zeros((4, A, 2, 3), dtype=torch.float64, device="cuda")
            kw = dict(levels=levels, align={}, dev_crops_ptr=crops.data_ptr(), dev_mats_ptr=mats.data_ptr())
            if oriented:
                d, c = eng.detect_tiled_oriented_device(dev, os_, THR, NMS, **kw)
            else:
                d, c = eng.detect_tiled_device(twin, THR, NMS, **kw)
            eng.synchronize()
            faces, ids = eng.read_dets(d, c, 4)
            counts = [len(f) for f in faces]
            out.append((faces, ids, _read_crops(crops, counts), _read_crops(mats, counts)))
        for a, b in zip(out[0], out[1]):
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b)), levels
        faces, tile_of = eng.detect_tiled_oriented(imgs, os_, THR, NMS, levels=levels)
        _same((out[0][0], [i // mf for i in out[0][1]]), (faces, tile_of), ("blocking", levels))
    torch.cuda.synchronize()
    assert [int(t.to(torch.int64).sum()) for t in dev] + [int(big.to(torch.int64).sum())] == sums


def test_device_yuv_equals_the_rotated_surfaces(eng, golden_image):
    """rf_detect_yuv_tiled_oriented_device (NV12 BT.601 and I420 BT.709, the 4K frame, the photo, 1038 x 670, and an NVDEC-like pitched
    4K NV12 surface) == rf_detect_yuv_tiled_device on device copies of orient_planes(frame, o): records and F16 crops bit for bit;
    the frames and the surface's 0xEE padding are untouched."""
    import torch
    bgr = [cv2.resize(golden_image, (3840, 2160)), golden_image, cv2.resize(golden_image, (1038, 670))]
    A = eng.max_faces
    for layout, matrix in (("nv12", "bt601"), ("i420", "bt709")):
        frames = [bgr_to_frame(b, layout) for b in bgr]
        os_ = [6, 3, 8]
        dev = [_cuda(f) for f in frames]
        surf = None
        if layout == "nv12":
            planes, surf = _nvdec_like(frames[0], 4096, 2176)
            dev.append(planes)
            frames.append(frames[0])
            os_.append(5)
            surf_before = surf.cpu().numpy()
        before = [d.cpu().numpy() if not isinstance(d, tuple) else None for d in dev]
        twin = [_cuda(orient_planes(f, layout, o)) for f, o in zip(frames, os_)]
        n = len(frames)
        out = []
        for oriented in (True, False):
            crops = torch.full((n, A, 3, 112, 112), 7.0, dtype=torch.float16, device="cuda")
            kw = dict(levels=None, align=dict(fmt="rgb_f16"), dev_crops_ptr=crops.data_ptr())
            if oriented:
                d, c = eng.detect_yuv_tiled_oriented_device(dev, os_, THR, NMS, layout, matrix, **kw)
            else:
                d, c = eng.detect_yuv_tiled_device(twin, THR, NMS, layout, matrix, **kw)
            eng.synchronize()
            faces, ids = eng.read_dets(d, c, n)
            out.append((faces, ids, _read_crops(crops, [len(f) for f in faces])))
        for a, b in zip(out[0], out[1]):
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b)), layout
        assert sum(len(f) for f in out[0][0]) >= 8
        for d, b in zip(dev, before):
            if b is not None:
                assert np.array_equal(d.cpu().numpy(), b)
        if surf is not None:
            assert np.array_equal(surf.cpu().numpy(), surf_before)


def _in_flight(e, golden_image, streams):
    """2 streams + 1 device tiled calls with no host synchronise between them, oriented and upright alternated (BGR and NV12), each
    with its own F16 crop buffer: every crop buffer and the records of the last `streams` calls equal one-at-a-time blocking calls.
    The oriented calls' images are stored so that they display upright, so every call has faces."""
    import torch
    calls = 2 * streams + 1
    A = e.max_faces
    host, dev, out, bufs = [], [], [], []
    for k in range(calls):
        imgs = [np.roll(cv2.resize(golden_image, (1920, 1080)), 16 * (2 * k + i) + 8, axis=1) for i in range(2)]
        os_ = [6, 8] if k % 2 == 0 else [1, 1]
        kind = "bgr" if k % 4 < 2 else "nv12"
        if kind == "bgr":
            srcs = [orient(im, INVERSE.get(o, o)) for im, o in zip(imgs, os_)]
        else:
            srcs = [unorient_planes(bgr_to_frame(im, "nv12"), "nv12", o) for im, o in zip(imgs, os_)]
        host.append((kind, srcs, os_))
        dev.append([_cuda(s) for s in srcs])
        bufs.append(torch.full((2, A, 3, 112, 112), 7.0, dtype=torch.float16, device="cuda"))
    torch.cuda.synchronize()
    for k in range(calls):
        kind, _, os_ = host[k]
        kw = dict(align=dict(fmt="rgb_f16"), dev_crops_ptr=bufs[k].data_ptr())
        if kind == "bgr":
            out.append(e.detect_tiled_oriented_device(dev[k], os_, THR, NMS, **kw) if k % 2 == 0 else e.detect_tiled_device(dev[k], THR, NMS, **kw))
        else:
            out.append(e.detect_yuv_tiled_oriented_device(dev[k], os_, THR, NMS, **kw) if k % 2 == 0 else
                       e.detect_yuv_tiled_device(dev[k], THR, NMS, **kw))
    e.synchronize()
    for k in range(calls):
        kind, srcs, os_ = host[k]
        if kind == "bgr":
            faces, tile_of, crops = e.detect_tiled_oriented(srcs, os_, THR, NMS, align=dict(fmt="rgb_f16"))
        else:
            faces, tile_of, crops = e.detect_yuv_tiled([orient_planes(f, "nv12", o) for f, o in zip(srcs, os_)], THR, NMS,
                                                       align=dict(fmt="rgb_f16"))
        for i in range(2):
            kk = len(crops[i])
            assert kk > 0 and np.array_equal(bufs[k][i, :kk].cpu().numpy(), crops[i]), (k, i)
            assert (bufs[k][i, kk:] == 7.0).all(), (k, i)
        if k >= calls - streams:
            df, ids = e.read_dets(out[k][0], out[k][1], 2)
            _same((df, [x // e.max_faces for x in ids]), (faces, tile_of), k)


@pytest.mark.parametrize("streams", [2, 8])
def test_calls_in_flight(golden_image, streams):
    e = _engine(max_batch=4, streams=streams, max_image=(1920, 1920))
    try:
        _in_flight(e, golden_image, streams)
    finally:
        e.close()


# ---- 5. behaviour: small faces in portrait 4K video ---------------------------------------------------------------------------------
def _iou(a, b):
    iw = min(a[3], b[3]) - max(a[1], b[1]) + 1
    ih = min(a[4], b[4]) - max(a[2], b[2]) + 1
    inter = max(iw, 0) * max(ih, 0)
    return inter / ((a[3] - a[1] + 1) * (a[4] - a[2] + 1) + (b[3] - b[1] + 1) * (b[4] - b[2] + 1) - inter)


def _portrait_canvas(golden_image, shift=0):
    """f7's seam canvas turned portrait: half-scale copies of the golden photo (faces about 50 x 70 px) upright on a black 2160 x 3840
    displayed frame; the copies and their expected offsets."""
    half = cv2.resize(golden_image, (640, 443), interpolation=cv2.INTER_AREA)
    xs, ys = (32, 704, 1376), (32, 512, 992, 1472, 1952, 2432, 2912, 3360)
    c = np.zeros((3840, 2160, 3), np.uint8)
    pos = [(x + shift, y) for y in ys for x in xs]
    for x, y in pos:
        c[y:y + 443, x:x + 640] = half
    return c, half, pos


def _expected(half, pos):
    """The expected faces: rf_detect_batch (score > 0.9) on one copy on a 672 x 448 handle, where it is not resized, shifted to each
    copy."""
    from retinaface_b200 import RF_PREC_FP16, Engine
    ref_eng = Engine(caffemodel("mnet25"), 448, 672, precision=RF_PREC_FP16, max_batch=1, max_image=(448, 672))   # net 672 wide, 448 high
    try:
        ref = ref_eng.detect_batch([half], 0.9, NMS)[0]
    finally:
        ref_eng.close()
    assert len(ref) >= 3
    out = []
    for x, y in pos:
        e = ref.copy()
        e[:, [1, 3]] += F32(x)
        e[:, [2, 4]] += F32(y)
        out.append(e)
    return np.concatenate(out)


def test_portrait_4k_small_faces_are_found_once(eng, golden_image):
    """The portrait seam canvas stored as 3840 x 2160 NV12 and shown at 6: rf_detect_yuv_tiled_oriented_device with the default
    pyramid, and at level 1 with overlap 96 (f7's seam protocol), finds every expected face exactly once (IoU >= 0.5) and no output
    matches two; the stored-frame tiles (rf_detect_yuv_tiled_device, faces turned 90 degrees) and the oriented letter-box
    (rf_detect_yuv_oriented_device, 8.6x shrink) each find fewer."""
    canvas, half, pos = _portrait_canvas(golden_image)
    expected = _expected(half, pos)
    shown = bgr_to_frame(canvas, "nv12")
    stored = _cuda(unorient_planes(shown, "nv12", 6))
    assert stored.shape == (3240, 3840)
    found = {}
    for name, kw in (("default pyramid", {}), ("level 1, overlap 96", SEAMS)):
        d, c = eng.detect_yuv_tiled_oriented_device([stored], [6], THR, NMS, **kw)
        eng.synchronize()
        faces = found[name] = eng.read_dets(d, c, 1)[0][0]
        used = np.zeros(len(faces), int)
        for e in expected:
            m = [j for j, f in enumerate(faces) if _iou(e, f) >= 0.5]
            assert len(m) == 1, (name, e[:5], [faces[j][:5] for j in m])
            used[m[0]] += 1
        assert (used <= 1).all(), name
    d, c = eng.detect_yuv_tiled_device([stored], THR, NMS)
    eng.synchronize()
    sideways = eng.read_dets(d, c, 1)[0][0]
    d, c, sc = eng.detect_yuv_oriented_device([stored], [6], THR, NMS)
    eng.synchronize()
    boxed = eng.read_dets(d, c, 1)[0][0]
    print(f"portrait 4K at 6: {len(expected)} expected faces; oriented tiles " + ", ".join(f"{len(f)} ({k})" for k, f in found.items()) +
          f"; stored-frame tiles {len(sideways)}, oriented letter-box {len(boxed)}")
    assert len(sideways) < len(expected) and len(boxed) < len(expected)


def test_portrait_4k_video_tracks_and_redacts(eng, golden_image):
    """A short portrait 4K video (3 frames, the canvas moving) stored at 6: records of rf_detect_yuv_tiled_oriented_device ->
    rf_track_update -> rf_redact_yuv_oriented_device_style.  orient_planes(S_out, 6) == the twin's output on the displayed frames
    (rf_detect_yuv_tiled_device -> rf_track_update -> rf_redact_yuv_device_style), and every expected face lies in a written region."""
    shown, expected = [], []
    for k in range(3):
        canvas, half, pos = _portrait_canvas(golden_image, shift=24 * k)
        shown.append(bgr_to_frame(canvas, "nv12"))
        expected.append(_expected(half, pos) if k == 0 else expected[0] + np.r_[0, 24 * k, 0, 24 * k, 0, [0] * 10].astype(F32))
    stored = [_cuda(unorient_planes(f, "nv12", 6)) for f in shown]
    twin = [_cuda(f) for f in shown]
    ta, tb = eng.tracker(max_videos=1), eng.tracker(max_videos=1)
    try:
        for k in range(3):
            d, c = eng.detect_yuv_tiled_oriented_device([stored[k]], [6], THR, NMS)
            tp, tc = ta.update([0], d, c)
            eng.redact_yuv_oriented_device([stored[k]], [6], d, c, tracker=ta, tracks_ptr=tp, track_counts_ptr=tc)
            eng.synchronize()
            d2, c2 = eng.detect_yuv_tiled_device([twin[k]], THR, NMS)
            tp2, tc2 = tb.update([0], d2, c2)
            eng.redact_yuv_device([twin[k]], d2, c2, tracker=tb, tracks_ptr=tp2, track_counts_ptr=tc2)
            eng.synchronize()
            out_s, out_d = stored[k].cpu().numpy(), twin[k].cpu().numpy()
            assert np.array_equal(orient_planes(out_s, "nv12", 6), out_d), k
            luma_before, luma_after = shown[k][:3840], out_d[:3840]
            for e in expected[k]:
                x1, y1, x2, y2 = (int(round(float(v))) for v in e[1:5])
                assert (luma_after[y1:y2, x1:x2] != luma_before[y1:y2, x1:x2]).mean() > 0.5, (k, e[:5])
    finally:
        ta.close()
        tb.close()


# ---- 6. refusals and 7. nothing else changes ----------------------------------------------------------------------------------------
def test_bad_orientations_launch_nothing_and_nothing_else_changes(golden_image):
    """Orientations 0, 9, -1 and a NULL array on every f21 entry point: RF_ERR_INVALID_ARG, the output canaries untouched; an NPP
    handle: RF_ERR_UNSUPPORTED.  rf_detect_tiled, rf_detect_yuv_tiled_device, rf_detect_batch and rf_launches_per_batch give the same
    results before and after oriented calls."""
    import torch
    from retinaface_b200 import RfError, capi
    imgs = [golden_image, cv2.resize(golden_image, (1920, 1080))]
    frame = bgr_to_frame(imgs[1], "nv12")
    e = _engine()
    try:
        d_frame = _cuda(frame)
        before = (e.detect_batch(imgs, THR, NMS, want_index=True), e.detect_tiled(imgs, THR, NMS, levels=LEVELS), e.launches_per_batch(8))
        d, c = e.detect_yuv_tiled_device([d_frame], THR, NMS)
        e.synchronize()
        yuv_before = e.read_dets(d, c, 1)

        lib, h = e.lib, e.h
        P, I = C.c_void_p, C.c_int
        d_img = _cuda(golden_image)
        canary = torch.full((4096,), 0xA5, dtype=torch.uint8, device="cuda")
        t, a = capi.tiling(), capi.align_params()
        faces = np.full((1, e.max_faces, 15), -3.0, np.float32)
        host_crops = np.full(e.max_faces * 112 * 112 * 3, 0xA5, np.uint8)
        counts = np.full(1, -3, np.int32)
        net = np.full((448, 448, 3), 0x33, np.uint8)
        hf, df = capi.yuv_frame(frame, "nv12")[0], capi.yuv_frame(d_frame, "nv12")[0]
        one = lambda ptr: ((P * 1)(ptr), (I * 1)(golden_image.shape[1]), (I * 1)(golden_image.shape[0]))
        for bad in (0, 9, -1, None):
            o = (I * 1)(bad) if bad is not None else None
            ov = bad if bad is not None else 0
            dd, cc = P(), P()
            rcs = [lib.rf_detect_tiled_oriented(h, *one(golden_image.ctypes.data), None, o, 1, C.byref(t), THR, NMS, C.byref(a),
                                                faces.ctypes.data, counts.ctypes.data, None, host_crops.ctypes.data, None),
                   lib.rf_detect_tiled_oriented_device(h, *one(d_img.data_ptr()), None, o, 1, C.byref(t), THR, NMS, C.byref(a),
                                                       canary.data_ptr(), None, C.byref(dd), C.byref(cc)),
                   lib.rf_detect_yuv_tiled_oriented_device(h, C.byref(df), o, 1, 0, C.byref(t), THR, NMS, None, None, None, C.byref(dd),
                                                           C.byref(cc))]
            if bad is not None:          # the parity hooks take the orientation by value
                rcs += [lib.rf_preprocess_tile_oriented(h, golden_image.ctypes.data, 1280, 886, 0, ov, C.byref(t), 0, net.ctypes.data),
                        lib.rf_preprocess_yuv_tile_oriented(h, C.byref(hf), 0, ov, C.byref(t), 0, net.ctypes.data)]
            assert rcs == [INVALID] * len(rcs), (bad, rcs)
            assert dd.value is None and cc.value is None
        torch.cuda.synchronize()
        assert (faces == -3.0).all() and (counts == -3).all() and (host_crops == 0xA5).all() and (net == 0x33).all()
        assert (canary == 0xA5).all()

        # oriented calls of every kind, then the unoriented results again
        e.detect_tiled_oriented(imgs, [6, 3], THR, NMS, align={})
        e.detect_tiled_oriented_device([d_img], [8], THR, NMS)
        e.detect_yuv_tiled_oriented_device([d_frame], [5], THR, NMS)
        e.preprocess_tile_oriented(golden_image, 7, 0)
        e.synchronize()
        after = (e.detect_batch(imgs, THR, NMS, want_index=True), e.detect_tiled(imgs, THR, NMS, levels=LEVELS), e.launches_per_batch(8))
        for x, y in zip(before[0], after[0]):
            assert all(np.array_equal(p, q) for p, q in zip(x, y))
        _same(before[1], after[1], "tiled")
        assert before[2] == after[2]
        d, c = e.detect_yuv_tiled_device([d_frame], THR, NMS)
        e.synchronize()
        _same(yuv_before, e.read_dets(d, c, 1), "yuv tiled device")
    finally:
        e.close()
    npp = _engine(flags=capi.RF_FLAG_NPP_RESIZE, max_image=(2160, 3840))
    try:
        for call in (lambda: npp.detect_tiled_oriented([golden_image], [6], THR, NMS),
                     lambda: npp.detect_tiled_oriented_device([_cuda(golden_image)], [6], THR, NMS),
                     lambda: npp.detect_yuv_tiled_oriented_device([_cuda(frame)], [6], THR, NMS),
                     lambda: npp.preprocess_tile_oriented(golden_image, 6, 0),
                     lambda: npp.preprocess_yuv_tile_oriented(frame, 6, 0)):
            with pytest.raises(RfError) as err:
                call()
            assert err.value.status == UNSUPPORTED
    finally:
        npp.close()


# ---- 8. drivers ---------------------------------------------------------------------------------------------------------------------
def test_python_driver_equals_the_c_call(golden_image):
    """RetinaFace.detectTiled(orientations=...) == Engine.detect_tiled_oriented's faces (and crops with align); orientations=None is
    the unoriented call."""
    from retinaface_b200 import RetinaFace
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(2160, 3840))
    imgs = [cv2.resize(golden_image, (3840, 2160)), golden_image]
    per = rf.detectTiled(imgs, 0.5, orientations=[6, 8])
    faces, _ = rf.engine.detect_tiled_oriented(imgs, [6, 8], 0.5, 0.4)
    assert [len(p) for p in per] == [len(f) for f in faces] and len(per[0]) >= 3
    for p, f in zip(per, faces):
        assert all(info.score == float(row[0]) and info.rect == tuple(map(float, row[1:5])) for info, row in zip(p, f))
    per = rf.detectTiled(imgs, 0.5, scales=[1.0, 0.0], flip=True, align={}, orientations=[5, 7])
    faces, _, crops = rf.engine.detect_tiled_oriented(imgs, [5, 7], 0.5, 0.4, levels=[(1.0, 0), (1.0, 1), (0.0, 0), (0.0, 1)], align={})
    for p, f, c in zip(per, faces, crops):
        assert len(p) == len(f)
        for (info, crop), row, want in zip(p, f, c):
            assert info.score == float(row[0]) and np.array_equal(crop, want)
    plain = rf.detectTiled(imgs, 0.5)
    want, _ = rf.engine.detect_tiled(imgs, 0.5, 0.4)
    assert [len(p) for p in plain] == [len(f) for f in want]


CPP_PROGRAM = r'''
#include "RetinaFace.h"
#include <cstdio>
#include <cstdlib>
#include <fstream>
// argv: model directory, images file (two 1280x886 BGR images), out file.  detectTiled with orientations {6, 3}, then the faces.
int main(int argc, char **argv) {
    string model = argv[1];
    std::vector<unsigned char> buf((size_t)1280 * 886 * 3 * 2);
    std::ifstream(argv[2], std::ios::binary).read((char *)buf.data(), buf.size());
    RetinaFaceOptions opt;
    opt.net_w = opt.net_h = 448;
    opt.model_file = "mnet25.caffemodel";
    RetinaFace rf(model, "net3", 0.4f, opt);
    vector<Mat> imgs;
    for (int i = 0; i < 2; i++) imgs.push_back(Mat(886, 1280, CV_8UC3, buf.data() + (size_t)i * 1280 * 886 * 3));
    rf.detectTiled(imgs, vector<int>{6, 3}, 0.5f, vector<float>{1.f, 0.f}, true);
    std::ofstream out(argv[3], std::ios::binary);
    for (const auto &per : rf.lastBatchFaces()) {
        int k = (int)per.size();
        out.write((const char *)&k, sizeof k);
        out.write((const char *)per.data(), sizeof(FaceDetectInfo) * per.size());
    }
    return 0;
}
'''


def test_host_shell_oriented_detect_tiled_equals_the_c_call(golden_image, tmp_path):
    """The C++ RetinaFace::detectTiled overload with orientations writes the faces of rf_detect_tiled_oriented, bit for bit."""
    import subprocess
    from conftest import ROOT
    from retinaface_b200.build import HERE, build_host
    from retinaface_b200 import Engine, RF_PREC_FP16
    build_host()
    imgs = [golden_image, np.ascontiguousarray(golden_image[::-1])]
    (tmp_path / "in.bin").write_bytes(b"".join(im.tobytes() for im in imgs))
    src = tmp_path / "user.cpp"
    src.write_text(CPP_PROGRAM)
    exe = tmp_path / "user"
    cuda = "/usr/local/cuda"
    hostdir = os.path.join(HERE, "host")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I", hostdir, "-I", os.path.join(ROOT, "include"), "-I", cuda + "/include", str(src),
                           os.path.join(hostdir, "RetinaFace.cpp"), "-o", str(exe), "-L", HERE, "-lrf_b200", "-L", cuda + "/lib64", "-lcudart",
                           "-Wl,-rpath," + HERE + ":" + cuda + "/lib64"])
    subprocess.check_call([str(exe), os.path.dirname(caffemodel("mnet25")), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")])
    raw = (tmp_path / "out.bin").read_bytes()
    e = Engine(caffemodel("mnet25"), 448, 448, precision=RF_PREC_FP16, max_batch=8, max_faces=256, max_image=(3072, 4096), network="net3")
    try:
        want, _ = e.detect_tiled_oriented(imgs, [6, 3], 0.5, 0.4, levels=[(1.0, 0), (1.0, 1), (0.0, 0), (0.0, 1)])
    finally:
        e.close()
    off = 0
    for w in want:
        k = int(np.frombuffer(raw[off:off + 4], np.int32)[0])
        off += 4
        assert k == len(w) >= 3
        got = np.frombuffer(raw[off:off + 60 * k], np.float32).reshape(k, 15)
        off += 60 * k
        assert got.tobytes() == w.tobytes()
    assert off == len(raw)
