"""CPU: f9 orientations without a GPU -- the EXIF definition (orient() against cv2.imread of JPEGs carrying each tag in both TIFF byte
orders), rf_jpeg_exif_orientation on those and on malformed segments, the map-back into stored pixels as the inverse of the tap
address map A_o, the 4:2:0 plane orientation against cvtColor, and the C++ shell compiling the oriented calls (the entry points'
signatures are checked in test_signatures_cpu.py).
stored_points / stored_faces are the map-back oracle the GPU tests (test_gpu_oriented.py) use too; orient and orient_planes are
oracle/orient.py's."""
import os
import struct

import cv2
import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle.orient import orient, orient_planes
from oracle.yuv import bgr_to_frame, frame_to_bgr

MIRRORED = {2, 4, 5, 7}


def stored_of(o, x, y, w, h):
    """A_o: the stored pixel displayed pixel (x, y) reads (the table of rf_b200.h), for a stored w x h image."""
    return {1: (x, y), 2: (w - 1 - x, y), 3: (w - 1 - x, h - 1 - y), 4: (x, h - 1 - y), 5: (y, x), 6: (y, h - 1 - x),
            7: (w - 1 - y, h - 1 - x), 8: (w - 1 - y, x)}[o]


def stored_points(o, x, y, w, h):
    """The merge's map-back of displayed float32 points into stored pixels (postproc.cuh): reflect in the displayed frame, then
    transpose.  Returns float32 (x, y)."""
    bits = {1: 0, 2: 1, 3: 3, 4: 2, 5: 4, 6: 5, 7: 7, 8: 6}[o]
    f32 = np.float32
    dw, dh = (h, w) if bits & 4 else (w, h)
    x, y = np.asarray(x, f32), np.asarray(y, f32)
    ax = f32(dw - 1) - x if bits & 1 else x
    ay = f32(dh - 1) - y if bits & 2 else y
    return (ay, ax) if bits & 4 else (ax, ay)


def stored_faces(o, faces, w, h):
    """Faces (k, 15) in displayed pixels -> stored pixels, as k_merge maps an oriented view (corners re-ordered, landmarks swapped
    when o mirrors)."""
    out = faces.copy()
    x1, y1 = stored_points(o, faces[:, 1], faces[:, 2], w, h)
    x2, y2 = stored_points(o, faces[:, 3], faces[:, 4], w, h)
    out[:, 1], out[:, 3] = np.minimum(x1, x2), np.maximum(x1, x2)
    out[:, 2], out[:, 4] = np.minimum(y1, y2), np.maximum(y1, y2)
    perm = [1, 0, 2, 4, 3] if o in MIRRORED else [0, 1, 2, 3, 4]
    lx, ly = stored_points(o, faces[:, 5:10][:, perm], faces[:, 10:15][:, perm], w, h)
    out[:, 5:10], out[:, 10:15] = lx, ly
    return out


def with_exif(jpeg: bytes, o: int, little: bool = True) -> bytes:
    """The JPEG with an APP1 Exif segment whose IFD0 holds only Orientation = o, spliced in after SOI."""
    e = "<" if little else ">"
    tiff = (b"II" if little else b"MM") + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1)
    tiff += struct.pack(e + "HHIH", 0x0112, 3, 1, o) + b"\0\0" + struct.pack(e + "I", 0)
    body = b"Exif\0\0" + tiff
    return jpeg[:2] + b"\xff\xe1" + struct.pack(">H", len(body) + 2) + body + jpeg[2:]


def _golden_bytes():
    with open(os.path.join(GOLDEN, "data", "img.jpg"), "rb") as f:
        return f.read()


@pytest.mark.parametrize("little", [True, False])
@pytest.mark.parametrize("o", range(1, 9))
def test_orient_is_what_imread_applies(o, little):
    data = with_exif(_golden_bytes(), o, little)
    buf = np.frombuffer(data, np.uint8)
    stored = cv2.imdecode(buf, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
    shown = cv2.imdecode(buf, cv2.IMREAD_COLOR)
    assert np.array_equal(orient(stored, o), shown)


@pytest.mark.parametrize("little", [True, False])
@pytest.mark.parametrize("o", range(1, 9))
def test_exif_orientation_reads_the_spliced_tag(built_lib, o, little):
    from retinaface_b200 import capi
    assert capi.exif_orientation(with_exif(_golden_bytes(), o, little)) == o


def test_exif_orientation_defaults_to_upright(built_lib):
    from retinaface_b200 import capi
    j = _golden_bytes()
    assert capi.exif_orientation(j) == 1                       # no APP1
    assert capi.exif_orientation(b"") == 1
    assert capi.exif_orientation(b"not a jpeg") == 1
    for bad in (0, 9):
        assert capi.exif_orientation(with_exif(j, bad)) == 1
    full = with_exif(j, 6)
    seg_end = 4 + struct.unpack(">H", full[4:6])[0]
    for cut in range(2, seg_end):                              # every truncation inside the SOI + APP1 prefix
        assert capi.exif_orientation(full[:cut]) == 1, cut
    # a length field that overruns the buffer
    lying = bytearray(full[:seg_end])
    lying[4:6] = struct.pack(">H", 0xFFF0)
    assert capi.exif_orientation(bytes(lying)) == 1


@pytest.mark.parametrize("o", range(1, 9))
def test_map_back_inverts_the_tap_addresses(o):
    w, h = 7, 5
    stored = np.arange(w * h * 3, dtype=np.int32).reshape(h, w, 3)
    shown = orient(stored, o)
    dh, dw = shown.shape[:2]
    ys, xs = np.mgrid[0:dh, 0:dw]
    sx, sy = stored_of(o, xs, ys, w, h)
    assert np.array_equal(shown, stored[sy, sx])                     # T_o reads A_o
    mx, my = stored_points(o, xs.astype(np.float32), ys.astype(np.float32), w, h)
    assert np.array_equal(mx, sx.astype(np.float32)) and np.array_equal(my, sy.astype(np.float32))


@pytest.mark.parametrize("layout", ["nv12", "i420"])
@pytest.mark.parametrize("o", range(1, 9))
def test_plane_orientation_commutes_with_cvtcolor(layout, o):
    rng = np.random.default_rng(o)
    bgr = rng.integers(0, 256, (722, 1282, 3), dtype=np.uint8)
    frame = bgr_to_frame(bgr, layout)
    code = cv2.COLOR_YUV2BGR_NV12 if layout == "nv12" else cv2.COLOR_YUV2BGR_I420
    assert np.array_equal(orient(cv2.cvtColor(frame, code), o), cv2.cvtColor(orient_planes(frame, layout, o), code))
    assert np.array_equal(orient(frame_to_bgr(frame, layout), o), frame_to_bgr(orient_planes(frame, layout, o), layout))


def test_cpp_shell_compiles_oriented_calls(built_lib, tmp_path):
    import subprocess
    from retinaface_b200.build import build_host
    build_host()
    host = os.path.join(ROOT, "retinaface_b200", "host")
    src = tmp_path / "oriented_call.cpp"
    src.write_text('#include "RetinaFace.h"\n'
                   'int main(int argc, char **argv) {\n'
                   '    string dir = argv[1];\n'
                   '    RetinaFace rf(dir);\n'
                   '    vector<Mat> imgs(1, Mat(720, 1280, CV_8UC3));\n'
                   '    AlignOptions a;\n'
                   '    rf.detectOriented(imgs, vector<int>(1, 6), 0.5f, &a);\n'
                   '    return (int)rf.detectAnyOrientation(imgs[0], 0.5f).size();\n'
                   '}\n')
    subprocess.check_call(["g++", "-std=c++14", "-fsyntax-only", "-I", host, "-I", os.path.join(ROOT, "include"), str(src)])
