"""GPU (-m gpu): f7 tiled detection -- rf_preprocess_tile against the host tile bytes (tests/tile_oracle.py), rf_detect_tiled
against every tile detected through rf_detect_batch and merged on the host, faces on tile seams, independence from the execution
contexts, the YUV twin, and that nothing else changes."""
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle.yuv import bgr_to_frame, frame_to_bgr
from tile_oracle import level_image, map_tile, tile_bytes

pytestmark = pytest.mark.gpu

F32 = np.float32


def _engine(prec="fp16", net=(448, 448), **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (2160, 3840))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), net[1], net[0], precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), net[1], net[0], precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


def _layout(eng, img, levels=None, overlap=0):
    from retinaface_b200 import capi
    return capi.tile_layout(eng.net_w, eng.net_h, img.shape[1], img.shape[0], levels, overlap)


def _canvas(golden_image, w=3840, h=2160, xs=(32, 704, 1376, 2048, 2720), ys=(32, 512, 992)):
    """Half-scale copies of the golden photo (640 x 443, faces about 50 x 70 px) on black, at 32-aligned positions."""
    half = cv2.resize(golden_image, (640, 443), interpolation=cv2.INTER_AREA)
    c = np.zeros((h, w, 3), np.uint8)
    for y in ys:
        for x in xs:
            c[y:y + 443, x:x + 640] = half
    return c, half, [(x, y) for y in ys for x in xs]


def test_tile_bytes_equal_the_host_tiles(golden_image):
    """Every tile of levels s in {0.37, 0.5, 1, 1.5, 2.75}, plain and mirrored, plus the fitted level, on the golden photo, a random
    517 x 333 image (sides of 1 mod 4), a random 519 x 335 image (3 mod 4: at s = 0.5 cv2.resize runs OpenCV's 2x area code, whose
    last column and row differ from the bilinear taps) and row-strided pinned and pageable copies: rf_preprocess_tile == slices of
    cv2.resize(cv2.flip(img)) padded with zeros (the fitted level: letterbox_bgr_u8), byte for byte."""
    import torch
    eng = _engine(max_batch=1)
    rng = np.random.default_rng(2)
    odd = rng.integers(0, 256, (333, 517, 3), dtype=np.uint8)
    odd3 = rng.integers(0, 256, (335, 519, 3), dtype=np.uint8)
    big = np.full((886, 1280 + 21, 3), 0x5A, np.uint8)
    big[:, :1280] = golden_image
    strided = big[:, :1280]
    pinned_t = torch.empty((886, 1300, 3), dtype=torch.uint8, pin_memory=True)
    pinned = pinned_t.numpy()
    pinned[:, :1280] = golden_image
    pinned_strided = pinned[:, :1280]
    try:
        for name, img, src in (("golden", golden_image, golden_image), ("odd3", odd3, odd3), ("odd", odd, odd), ("strided", golden_image, strided),
                               ("pinned", golden_image, pinned_strided)):
            for flip in (0, 1):
                levels = [(s, flip) for s in (0.37, 0.5, 1.0, 1.5, 2.75)] + [(0.0, flip)]
                tiles = _layout(eng, img, levels, 64)
                cache = {}
                for k, t in enumerate(tiles):
                    if t["scale"] and t["level"] not in cache:
                        cache[t["level"]] = level_image(img, t["scale"], t["flip"])
                    want = tile_bytes(img, t, 448, 448, cache.get(t["level"]))
                    got = eng.preprocess_tile(src, k, levels, 64)
                    assert np.array_equal(got, want), (name, flip, k, t)
                if name not in ("golden", "odd3"):
                    break               # the mirrored levels of the other sources: same kernel path as the golden one
    finally:
        eng.close()


@pytest.mark.parametrize("layout", ["nv12", "i420"])
def test_yuv_tile_bytes_equal_the_tiles_of_the_converted_frame(golden_image, layout):
    """rf_preprocess_yuv_tile (NV12 BT.601, I420 BT.709) == the host tiles of the oracle's conversion of the frame (== cv2.cvtColor
    for BT.601), byte for byte, on a 1920 x 1080 frame and a random 1038 x 670 one (sides of 3 mod 4 at s = 0.5: 519 x 335);
    rf_detect_yuv_tiled equals rf_detect_tiled on the converted frame."""
    matrix = "bt601" if layout == "nv12" else "bt709"
    rng = np.random.default_rng(8)
    frames = [bgr_to_frame(cv2.resize(golden_image, (1920, 1080)), layout), rng.integers(0, 256, (670 * 3 // 2, 1038), dtype=np.uint8)]
    eng = _engine(max_batch=8)
    try:
        levels = [(1.5, 0), (1.0, 1), (0.5, 0), (0.5, 1), (0.0, 0)]
        for fi, frame in enumerate(frames):
            bgr = frame_to_bgr(frame, layout, matrix)
            cache = {}
            for k, t in enumerate(_layout(eng, bgr, levels)):
                if t["scale"] and t["level"] not in cache:
                    cache[t["level"]] = level_image(bgr, t["scale"], t["flip"])
                want = tile_bytes(bgr, t, 448, 448, cache.get(t["level"]))
                assert np.array_equal(eng.preprocess_yuv_tile(frame, k, layout, matrix, levels), want), (layout, fi, k, t)
        f1, t1 = eng.detect_yuv_tiled([frames[0]], 0.5, 0.4, layout=layout, matrix=matrix, levels=levels)
        f2, t2 = eng.detect_tiled([frame_to_bgr(frames[0], layout, matrix)], 0.5, 0.4, levels=levels)
        assert np.array_equal(f1[0], f2[0]) and np.array_equal(t1[0], t2[0]) and len(f1[0]) >= 5
    finally:
        eng.close()


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_fitted_level_alone_equals_detect_batch(golden_image, prec):
    """levels = {{0, 0}}: the same faces in the same order as rf_detect_batch, coordinates == rf_detect_batch's * scale bit for bit,
    on mixed batches of 1, 3 and 8 images."""
    rng = np.random.default_rng(4)
    imgs = [golden_image, cv2.resize(golden_image, (1920, 1080)), letterbox_448(golden_image), golden_image[100:700, 200:1100],
            cv2.resize(golden_image, (3840, 2160)), golden_image[:, ::-1].copy(), cv2.resize(golden_image, (320, 222)),
            rng.integers(0, 256, (500, 700, 3), dtype=np.uint8)]
    eng = _engine(prec)
    try:
        for n in (1, 3, 8):
            batch = imgs[:n] if n < 8 else imgs
            plain = eng.detect_batch(batch, 0.5, 0.4)
            faces, tile_of = eng.detect_tiled(batch, 0.5, 0.4, levels=[(0.0, 0)])
            for i, im in enumerate(batch):
                sc = max(F32(im.shape[1] / 448), F32(im.shape[0] / 448), F32(1.0))
                want = plain[i].copy()
                want[:, 1:] = plain[i][:, 1:] * sc
                assert faces[i].shape == want.shape, (prec, n, i)
                assert np.array_equal(faces[i], want), (prec, n, i)
                assert (tile_of[i] == 0).all()
    finally:
        eng.close()


def letterbox_448(img):
    from oracle.inputs import letterbox_bgr_u8
    return letterbox_bgr_u8(img, 448, 448)


def _host_tiled(eng, img, levels, overlap, thr, nms, post_oracle):
    """The merge oracle: every tile built on the host, detected through rf_detect_batch in batches, mapped back and filtered in
    float32 numpy, merged by the oracle NMS.  Returns (faces, tile of each face, number of merged candidates)."""
    tiles = _layout(eng, img, levels, overlap)
    cache, ins = {}, []
    for t in tiles:
        if t["scale"] and t["level"] not in cache:
            cache[t["level"]] = level_image(img, t["scale"], t["flip"])
        ins.append(tile_bytes(img, t, eng.net_w, eng.net_h, cache.get(t["level"])))
    dets = []
    for k0 in range(0, len(ins), eng.max_batch):
        dets += eng.detect_batch(ins[k0:k0 + eng.max_batch], thr, nms)
    cands, tile_ids = [], []
    for k, (t, d) in enumerate(zip(tiles, dets)):
        m, _ = map_tile(d, t, img.shape[1], eng.net_w, eng.net_h)
        cands.append(m)
        tile_ids.append(np.full(len(m), k, np.int32))
    allc = np.concatenate(cands)
    ids = np.concatenate(tile_ids)
    want, pos = post_oracle.nms(allc, nms)
    want, pos = want[:eng.max_faces], pos[:eng.max_faces]        # the output capacity keeps the top-scoring prefix
    return want, ids[pos], len(allc)


def test_merge_equals_host_tiles_detected_one_by_one(golden_image):
    """Golden photo and a 3840 x 2160 canvas, levels {1.5 mirrored, 1.0, 0.5, fitted}: faces, order and out_tile_of identical bit for
    bit to the host merge of every tile detected through rf_detect_batch (FP32).  At thresholds 0.02 and 0.001 the canvas's 211 tiles
    send tens of thousands of candidates (ids tile * max_faces + rank) to the final k_nms, past its shared-memory working set; a
    handle with max_batch 48 runs 48 tiles per forward, which k_merge takes in two launches of at most 40 sources."""
    from oracle.postproc import PostprocOracle
    post_oracle = PostprocOracle()
    canvas, _, _ = _canvas(golden_image)
    levels = [(1.5, 1), (1.0, 0), (0.5, 0), (0.0, 0)]
    cases = [("fp32", dict(), "golden", golden_image, 0.5), ("fp32", dict(), "canvas", canvas, 0.5), ("fp32", dict(), "canvas", canvas, 0.02),
             ("fp32", dict(), "canvas", canvas, 0.001), ("fp32", dict(max_batch=48), "canvas", canvas, 0.5),
             ("fp32", dict(max_batch=48), "canvas", canvas, 0.02)]
    engines = {}
    try:
        for prec, kw, name, img, thr in cases:
            key = (prec, tuple(kw.items()))
            if key not in engines:
                engines[key] = _engine(prec, **kw)
            eng = engines[key]
            assert len(_layout(eng, img, levels)) > (40 if eng.max_batch > 40 else 0)
            want, want_tile, ncand = _host_tiled(eng, img, levels, 0, thr, 0.4, post_oracle)
            faces, tile_of = eng.detect_tiled([img], thr, 0.4, levels=levels)
            label = (name, thr, eng.max_batch)
            print(f"merge {label}: {ncand} candidates, {len(faces[0])} faces")
            assert len(want) >= 5, label
            if thr <= 0.001:
                assert ncand > 1024, label
            assert faces[0].shape == want.shape, (label, faces[0].shape, want.shape)
            assert np.array_equal(faces[0], want), label
            assert np.array_equal(tile_of[0], want_tile), label
    finally:
        for eng in engines.values():
            eng.close()


def _iou(a, b):
    iw = min(a[3], b[3]) - max(a[1], b[1]) + 1
    ih = min(a[4], b[4]) - max(a[2], b[2]) + 1
    inter = max(iw, 0) * max(ih, 0)
    return inter / ((a[3] - a[1] + 1) * (a[4] - a[2] + 1) + (b[3] - b[1] + 1) * (b[4] - b[2] + 1) - inter)


def test_faces_on_seams_are_found_once(golden_image):
    """A 3840 x 2160 canvas of 15 half-scale golden-photo copies (faces about 50 x 70 px).  Expected faces: rf_detect_batch (score
    > 0.9) on one 640 x 443 copy on a 672 x 448 handle, where the copy is not resized, shifted to each copy.  At least 10 of them
    have their centre within o of a shared tile edge.
    - levels {{1, 0}}, o = 96, threshold 0.5: every expected face is matched (IoU >= 0.5) by exactly one output and no output matches
      two faces; box corners within 2 px, scores within 0.05.
    - the default pyramid: every expected face is matched.
    - rf_detect_batch on the canvas finds strictly fewer faces."""
    canvas, half, pos = _canvas(golden_image)
    one = _engine("fp16", net=(672, 448), max_batch=1, max_image=(448, 672))
    try:
        ref = one.detect_batch([half], 0.9, 0.4)[0]
    finally:
        one.close()
    assert len(ref) >= 3
    expected = []
    for x, y in pos:
        e = ref.copy()
        e[:, [1, 3]] += F32(x)
        e[:, 5:10] += F32(x)
        e[:, [2, 4]] += F32(y)
        e[:, 10:15] += F32(y)
        expected.append(e)
    expected = np.concatenate(expected)
    eng = _engine("fp16")
    try:
        o = 96
        tiles = _layout(eng, canvas, [(1.0, 0)], o)
        edges_x = sorted({t["x0"] for t in tiles if t["shared_sides"] & 1} | {t["x0"] + 448 for t in tiles if t["shared_sides"] & 4})
        edges_y = sorted({t["y0"] for t in tiles if t["shared_sides"] & 2} | {t["y0"] + 448 for t in tiles if t["shared_sides"] & 8})
        cx, cy = (expected[:, 1] + expected[:, 3]) / 2, (expected[:, 2] + expected[:, 4]) / 2
        near = [min([abs(c - e) for e in edges_x] + [1e9]) < o or min([abs(d - e) for e in edges_y] + [1e9]) < o for c, d in zip(cx, cy)]
        assert sum(near) >= 10, sum(near)
        faces, _ = eng.detect_tiled([canvas], 0.5, 0.4, levels=[(1.0, 0)], overlap=o)
        out = faces[0]
        used = np.zeros(len(out), int)
        dcoord, dscore = 0.0, 0.0
        for e in expected:
            m = [j for j, f in enumerate(out) if _iou(e, f) >= 0.5]
            assert len(m) == 1, (e[:5], [out[j][:5] for j in m])
            used[m[0]] += 1
            dcoord = max(dcoord, float(np.abs(out[m[0]][1:5] - e[1:5]).max()))
            dscore = max(dscore, float(abs(out[m[0]][0] - e[0])))
        assert (used <= 1).all()
        print(f"seams: {len(expected)} expected faces, {sum(near)} near a seam, {len(out)} outputs; max |d corner| {dcoord:.3f} px, "
              f"max |d score| {dscore:.4f}")
        assert dcoord <= 2.0 and dscore <= 0.05
        pyr, _ = eng.detect_tiled([canvas], 0.5, 0.4)
        for e in expected:
            assert any(_iou(e, f) >= 0.5 for f in pyr[0]), e[:5]
        plain = eng.detect_batch([canvas], 0.5, 0.4)[0]
        print(f"seams: default pyramid {len(pyr[0])} faces, rf_detect_batch {len(plain)} faces")
        assert len(plain) < len(expected) <= len(pyr[0])
    finally:
        eng.close()


def test_contexts_and_raw_groups_do_not_change_the_result(golden_image):
    """The same tiled call on handles with streams = 2 and streams = 8 (one layer plan) gives bit-equal results; so does a handle
    whose raw buffers hold fewer images than the call has (two upload groups)."""
    canvas, _, _ = _canvas(golden_image)
    imgs = [canvas, golden_image, cv2.resize(golden_image, (1920, 1080)), golden_image[:, ::-1].copy(), canvas[:1500, :2500].copy(),
            cv2.resize(golden_image, (2560, 1772)), golden_image[50:800, 100:1200].copy(), cv2.resize(golden_image, (999, 691))]
    levels = [(1.0, 0), (0.5, 1), (0.0, 0)]
    results = []
    for kw in (dict(streams=2), dict(streams=8), dict(streams=8, max_image=(8192, 16384))):
        eng = _engine("fp16", **kw)
        try:
            from retinaface_b200 import capi  # noqa: F401
            results.append((eng.detect_tiled(imgs, 0.5, 0.4, levels=levels), eng.detect_tiled(imgs[:3], 0.5, 0.4)))
        finally:
            eng.close()
    for r in results[1:]:
        for (fa, ta), (fb, tb) in zip(results[0], r):
            assert all(np.array_equal(a, b) for a, b in zip(fa, fb)) and all(np.array_equal(a, b) for a, b in zip(ta, tb))
    assert sum(len(f) for f in results[0][0][0]) >= 20


def test_nothing_else_changes_and_bad_calls_launch_nothing(golden_image):
    from retinaface_b200 import RfError, capi
    imgs = [golden_image, cv2.resize(golden_image, (1920, 1080))]
    eng = _engine("fp16")
    try:
        before = eng.detect_batch(imgs, 0.5, 0.4, want_index=True)
        launches = eng.launches_per_batch(8)
        eng.detect_tiled(imgs, 0.5, 0.4)
        frame = bgr_to_frame(imgs[1], "nv12")
        eng.detect_yuv_tiled([frame], 0.5, 0.4)
        after = eng.detect_batch(imgs, 0.5, 0.4, want_index=True)
        for a, b in zip(before, after):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
        assert eng.launches_per_batch(8) == launches
        bad = [(dict(levels=[(-1.0, 0)]), -1), (dict(levels=[(float("nan"), 0)]), -1), (dict(levels=[(9.0, 0)]), -1),
               (dict(overlap=8), -1), (dict(overlap=300), -1), (dict(levels=[(1.0, 0)] * 9), -1),
               (dict(levels=[(2.0, 0), (1.0, 0)]), -6)]
        big = cv2.resize(golden_image, (3840, 2160))
        for kw, status in bad:
            with pytest.raises(RfError) as e:
                eng.detect_tiled([big], 0.5, 0.4, **kw)
            assert e.value.status == status, kw
            with pytest.raises(RfError) as e:
                eng.detect_yuv_tiled([bgr_to_frame(big, "nv12")], 0.5, 0.4, **kw)
            assert e.value.status == status, kw
        with pytest.raises(RfError) as e:
            eng.detect_tiled([np.zeros((2200, 3840, 3), np.uint8)], 0.5, 0.4)
        assert e.value.status == -6
        with pytest.raises(RfError) as e:
            eng.detect_tiled([golden_image] * 9, 0.5, 0.4)
        assert e.value.status == -6
        with pytest.raises(RfError) as e:
            eng.preprocess_tile(golden_image, 15, None, 0)         # the default layout of the photo has 15 tiles
        assert e.value.status == -1
        assert len(capi.tile_layout(448, 448, 1280, 886)) == 15
        again = eng.detect_batch(imgs, 0.5, 0.4, want_index=True)
        for a, b in zip(before, again):
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
    finally:
        eng.close()
    npp = _engine("fp16", flags=capi.RF_FLAG_NPP_RESIZE)
    try:
        with pytest.raises(RfError) as e:
            npp.detect_tiled([golden_image], 0.5, 0.4)
        assert e.value.status == -7
        with pytest.raises(RfError) as e:
            npp.preprocess_tile(golden_image, 0)
        assert e.value.status == -7
    finally:
        npp.close()


def test_detector_detect_tiled(golden_image):
    """RetinaFace.detectTiled: the Python surface over rf_detect_tiled (faces in image pixels)."""
    from retinaface_b200 import RetinaFace
    rf = RetinaFace(os.path.join(GOLDEN, "weights"), model_file="mnet25.caffemodel", max_image=(2160, 3840))
    canvas, _, _ = _canvas(golden_image)
    per = rf.detectTiled([canvas, golden_image], 0.5)
    want, _ = rf.engine.detect_tiled([canvas, golden_image], 0.5, 0.4)
    assert [len(p) for p in per] == [len(w) for w in want] and len(per[0]) > 20
    assert per[1][0].score == float(want[1][0][0])
    flipped = rf.detectTiled([golden_image], 0.5, scales=[1.0, 0.5], flip=True, overlap=96)
    assert len(flipped[0]) >= 5
    with pytest.raises(ValueError):
        rf.detectTiled([golden_image], 0.5, flip=True)       # the default pyramid has no mirrored levels
