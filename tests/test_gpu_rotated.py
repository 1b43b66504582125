"""GPU (-m gpu): f23 rotated views through the C ABI -- the warp view's bytes and M against oracle/rotate.py and cv2.warpAffine, quarter
turns against rf_detect_views_oriented, records rebuilt from the library's own parts (rf_preprocess_rotated -> rf_detect_batch -> the
oracle map-back -> the C NMS oracle), crops against oracle/align.py, tilted photos, refusals with nothing written, and that the other
detect calls do not change."""
import ctypes as C
import math
import os

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from oracle import rotate
from oracle.align import ARCFACE_112, blob, similarity_closed, warp_affine_fixed

pytestmark = pytest.mark.gpu

THR, NMS = 0.5, 0.4
ANGLES = (7.5, 30.0, 45.0, 135.0, -60.0, 359.9, 200.0)
QUARTERS = ((0.0, 1), (90.0, 8), (180.0, 3), (270.0, 6), (-90.0, 6), (450.0, 8))
SWEEP = [30.0 * k for k in range(12)]


def _engine(prec="fp16", net=(448, 448), **kw):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    kw.setdefault("max_batch", 8)
    kw.setdefault("max_image", (2160, 3840))
    if prec == "int8":
        return Engine(caffemodel("mnet-deconv-0517"), net[1], net[0], precision=RF_PREC_INT8,
                      int8_table=os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8"), **kw)
    return Engine(caffemodel("mnet25"), net[1], net[0], precision=RF_PREC_FP32 if prec == "fp32" else RF_PREC_FP16, **kw)


@pytest.fixture(scope="module")
def eng():
    e = _engine()
    yield e
    e.close()


def _tilted(img, angle):
    """img rotated counter-clockwise by `angle` onto a canvas that holds all of it, and the 2 x 3 matrix that put it there."""
    h, w = img.shape[:2]
    R = cv2.getRotationMatrix2D((w / 2, h / 2), angle, 1.0)
    c, s = abs(R[0, 0]), abs(R[0, 1])
    W, H = int(h * s + w * c), int(h * c + w * s)
    R[0, 2] += W / 2 - w / 2
    R[1, 2] += H / 2 - h / 2
    return cv2.warpAffine(img, R, (W, H)), R


@pytest.mark.parametrize("net", [(448, 448), (1280, 896)])
def test_preprocess_bytes_and_matrix(golden_image, net):
    g = golden_image
    padded_img = np.zeros((500, 420, 3), np.uint8)[:, :400]          # rows 1260 bytes apart
    padded_img[:] = cv2.resize(g, (400, 500))
    images = {"golden": g, "4k": cv2.resize(g, (3840, 2160)), "300x200": cv2.resize(g, (300, 200)), "padded": padded_img}
    e = _engine(net=net)
    try:
        for name, img in images.items():
            h, w = img.shape[:2]
            for angle in ANGLES:
                for shrink in (1.0, 0.6):
                    got, M = e.preprocess_rotated(img, angle, shrink)
                    o, f, want_M = rotate.geometry(angle, w, h, *rotate.shrink_box(net[0], net[1], shrink))
                    assert o == 0 and M.tobytes() == want_M.tobytes(), (name, angle, shrink)
                    if name == "300x200" and shrink == 1.0:
                        assert f == 1.0
                    assert np.array_equal(got, rotate.warp_view(np.ascontiguousarray(img), want_M, net[0], net[1])), (name, angle, shrink)
    finally:
        e.close()


def test_quarter_turns_take_the_oriented_path(eng, golden_image):
    img = cv2.resize(golden_image, (900, 620))
    for angle, o in QUARTERS:
        got, M = eng.preprocess_rotated(img, angle)
        assert np.array_equal(got, eng.preprocess_oriented(img, o)) and not M.any(), angle
        f, view_of, sc, mats = eng.detect_views_rotated(img, [(angle, 1.0), (angle, 0.6)], THR, NMS)
        rf, rview_of, rsc = eng.detect_views_oriented(img, [(1.0, o), (0.6, o)], THR, NMS)
        assert np.array_equal(f, rf) and np.array_equal(view_of, rview_of) and np.array_equal(sc, rsc) and not mats.any(), angle
    # the four quarter turns in one call: detectAnyOrientation's sweep
    a = eng.detect_views_rotated(img, [(0, 1.0), (270, 1.0), (180, 1.0), (90, 1.0)], THR, NMS)[:3]
    b = eng.detect_views_oriented(img, [(1.0, o) for o in (1, 6, 3, 8)], THR, NMS)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def _expected(e, img, views):
    """The merged faces and view_of rebuilt from the library's parts: each view's input (rf_preprocess_rotated) through rf_detect_batch,
    mapped back by the oracle (warp views) or by the one-view oriented call (quarter turns), then the C NMS oracle over ids
    v * max_faces + rank."""
    from oracle.postproc import PostprocOracle
    h, w = img.shape[:2]
    cands, ids = [], []
    for v, (angle, shrink) in enumerate(views):
        o, f, M = rotate.geometry(angle, w, h, *rotate.shrink_box(e.net_w, e.net_h, shrink))
        if o:
            mapped = e.detect_views_oriented(img, [(shrink, o)], THR, NMS)[0]
        else:
            inp, got_M = e.preprocess_rotated(img, angle, shrink)
            assert got_M.tobytes() == M.tobytes()
            mapped = rotate.map_back(e.detect_batch([inp], THR, NMS)[0], M, f)
        cands.append(mapped)
        ids += [v] * len(mapped)
    cands = np.concatenate(cands) if cands else np.zeros((0, 15), np.float32)
    out, pos = PostprocOracle().nms(cands, NMS)
    return out[:e.max_faces], np.asarray(ids, np.int32)[pos][:e.max_faces]


@pytest.mark.parametrize("prec", ["fp32", "fp16", "int8"])
def test_records_are_exact(golden_image, prec):
    e = _engine(prec)
    try:
        img = cv2.resize(golden_image, (1100, 760))
        tilted = _tilted(golden_image, 40.0)[0]
        for im, views in ((img, [(a, 1.0) for a in (0, 30, 45, 135, 270)]), (tilted, [(a, 1.0) for a in SWEEP]),
                          (tilted, [(a, 0.75) for a in SWEEP[:7]] + [(315.0, 1.0)])):
            f, view_of, sc, mats = e.detect_views_rotated(im, views, THR, NMS)
            want_f, want_v = _expected(e, im, views)
            assert np.array_equal(f, want_f) and np.array_equal(view_of, want_v), (prec, views, len(f), len(want_f))
            for v, (angle, shrink) in enumerate(views):
                o, fit, M = rotate.geometry(angle, im.shape[1], im.shape[0], *rotate.shrink_box(e.net_w, e.net_h, shrink))
                if not o:
                    assert sc[v] == np.float32(1.0 / fit) and mats[v].tobytes() == M.tobytes()
                else:
                    assert not mats[v].any()
    finally:
        e.close()


@pytest.mark.parametrize("fmt", ["bgr_u8", "rgb_f16"])
def test_crops_equal_the_align_oracle(eng, golden_image, fmt):
    img = _tilted(golden_image, 30.0)[0]
    views = [(a, 1.0) for a in SWEEP]
    plain = eng.detect_views_rotated(img, views, THR, NMS)
    f, view_of, sc, mats, crops, cmats = eng.detect_views_rotated(img, views, THR, NMS, align={"fmt": fmt, "want_mats": True})
    assert all(np.array_equal(x, y) for x, y in zip(plain, (f, view_of, sc, mats)))
    assert len(f) > 0 and len(crops) == len(f)
    for j, r in enumerate(f):
        M = similarity_closed(np.stack([r[5:10], r[10:15]], 1).astype(np.float64), ARCFACE_112.astype(np.float64))
        assert cmats[j].tobytes() == M.tobytes(), j
        u8 = warp_affine_fixed(img, M, (112, 112))
        want = u8 if fmt == "bgr_u8" else blob(u8[None])[0].astype(np.float16)
        assert np.array_equal(crops[j], want), j


def _angle(M):
    return math.degrees(math.atan2(M[1, 0], M[0, 0]))


@pytest.mark.parametrize("tilt", [30.0, 45.0, 60.0, 135.0])
def test_sweep_finds_the_faces_of_a_tilted_photo(eng, golden_image, tilt):
    """Every face the 30-degree sweep finds on the tilted photo is one of the upright photo's faces (mapped centre within a quarter of
    the box side), it finds at least four of the six where the plain letter-box finds fewer, and each crop fitted on its landmarks is
    the upright face's crop: its fitted angle is the upright one turned by the tilt, within 20 degrees.  The roll a crop takes is the
    detector's landmarks', and a face kept from a view up to 15 degrees off its tilt, shrunk to about 20 pixels, keeps part of that
    offset: 11.5, 18.1, 17.4 and 18.7 degrees at the worst face of the four tilts (FP16).  The rotated bounding box
    shrinks the faces (0.84x at 45 degrees for this 3:2 photo), so the smallest face can fall below the detector's reach."""
    from oracle.align import umeyama
    ref = eng.detect_views_rotated(golden_image, [(0.0, 1.0)], THR, NMS)[0]
    img, R = _tilted(golden_image, tilt)
    plain = eng.detect_batch([img], THR, NMS)[0]
    f, view_of, _, _, crops, cmats = eng.detect_views_rotated(img, [(a, 1.0) for a in SWEEP], THR, NMS, align={"want_mats": True})
    mapped = np.stack([R @ np.array([(r[1] + r[3]) / 2, (r[2] + r[4]) / 2, 1.0]) for r in ref])
    matched = set()
    for j, r in enumerate(f):
        d = np.hypot(*(mapped - [(r[1] + r[3]) / 2, (r[2] + r[4]) / 2]).T)
        i = int(np.argmin(d))
        assert d[i] < 0.25 * (ref[i, 3] - ref[i, 1]), (tilt, j, r[:5])
        matched.add(i)
        Mu = umeyama(np.stack([ref[i, 5:10], ref[i, 10:15]], 1).astype(np.float64), ARCFACE_112)[:2]
        dd = (_angle(cmats[j]) - tilt - _angle(Mu) + 180.0) % 360.0 - 180.0
        assert abs(dd) < 20.0, (tilt, j, dd)
    print(f"\ntilt {tilt}: rf_detect_batch finds {len(plain)} faces, the 30-degree sweep {len(f)} of the upright photo's {len(ref)}: "
          f"{sorted(matched)}")
    assert len(ref) == 6 and len(matched) >= 4 and len(matched) > len(plain)


def test_refusals_change_nothing(eng, golden_image):
    from retinaface_b200 import capi
    lib, h = eng.lib, eng.h
    img = np.ascontiguousarray(golden_image)
    mf = eng.max_faces
    faces = np.full((mf, 15), 7, np.float32)
    view_of = np.full(mf, 7, np.int32)
    scales = np.full(17, 7, np.float32)
    mats = np.full((17, 6), 7, np.float64)
    crops = np.full((mf, 112, 112, 3), 7, np.uint8)
    out = np.full((448, 448, 3), 7, np.uint8)
    m6 = np.full(6, 7, np.float64)
    good = capi.align_params()
    bad_align = capi.align_params(crop=(4, 4))

    def call(views, n, align=None):
        cnt = C.c_int(7)
        varr = None if views is None else (capi._RotatedView * max(len(views), 1))(*[capi._RotatedView(a, s) for a, s in views])
        rc = lib.rf_detect_views_rotated(h, img.ctypes.data, img.shape[1], img.shape[0], 0, varr, n, THR, NMS, None if align is None else C.byref(align),
                                         faces.ctypes.data, C.byref(cnt), view_of.ctypes.data, scales.ctypes.data, mats.ctypes.data,
                                         crops.ctypes.data, None)
        return rc, cnt.value

    cases = [([(math.nan, 1.0)], 1, None, -1), ([(math.inf, 1.0)], 1, None, -1), ([(-math.inf, 1.0)], 1, None, -1),
             ([(30.0, 0.0)], 1, None, -1), ([(30.0, 1.5)], 1, None, -1), ([(30.0, 1.0)] * 17, 17, None, None),
             ([(30.0, 1.0)], 0, None, None), ([(30.0, 1.0)], 1, bad_align, -1), (None, 1, None, -1),
             ([(30.0, 1.0), (0.0, math.nan)], 2, good, -1)]
    for views, n, align, status in cases:
        rc, cnt = call(views, n, align)
        assert rc != 0 and (status is None or rc == status) and cnt == 7, (views, n, rc)
        assert (faces == 7).all() and (view_of == 7).all() and (scales == 7).all() and (mats == 7).all() and (crops == 7).all()
    for angle, shrink in ((math.nan, 1.0), (math.inf, 1.0), (30.0, 0.0), (30.0, 1.5)):
        assert lib.rf_preprocess_rotated(h, img.ctypes.data, img.shape[1], img.shape[0], 0, angle, shrink, out.ctypes.data, m6.ctypes.data) == -1
        assert (out == 7).all() and (m6 == 7).all()
    assert eng.detect_views_rotated(img, [(30.0, 1.0)], THR, NMS)[0].shape[1] == 15     # the handle still works


def test_other_calls_do_not_change(golden_image):
    e = _engine()
    try:
        imgs = [golden_image, cv2.resize(golden_image, (640, 443))]

        def plain():
            out = [e.detect_batch(imgs, THR, NMS, want_index=True)]
            out.append(e.detect_align(imgs, THR, NMS, want_mats=True))
            out.append(e.detect_views(imgs[0], [(1.0, 0), (0.6, 1)], THR, NMS))
            out.append(e.detect_views_oriented(imgs[0], [(1.0, o) for o in (1, 6, 3, 8)], THR, NMS))
            return out
        launches = e.launches_per_batch(2)
        before = plain()
        e.detect_views_rotated(imgs[0], [(a, 1.0) for a in SWEEP], THR, NMS, align={})
        e.preprocess_rotated(imgs[1], 33.0, 0.5)
        after = plain()

        def flat(x):
            if isinstance(x, (list, tuple)):
                return [z for y in x for z in flat(y)]
            return [x]
        a, b = flat(before), flat(after)
        assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
        assert e.launches_per_batch(2) == launches
    finally:
        e.close()
