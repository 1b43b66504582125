"""CPU: the letter-box kernel's definition (oracle/letterbox.py, the numpy restatement of preprocess.cu) against cv2 wherever
cv::resize changes its code path: both sides of scale 1, 2, 3 and 4 with every side k * box + d (d = -3..3), every residue mod 4
at exactly 2x, sides whose resized size sits on a round-half-to-even tie, one-pixel sides and extreme aspect ratios, for four
network sizes and the view boxes of shrink 0.5 and 0.25 (mirrored, as rf_detect_views builds them), and every EXIF orientation.
No GPU: the kernels are held to the same definition byte for byte by tests/test_gpu_letterbox_edges.py."""
import cv2
import numpy as np
import pytest

from oracle import letterbox as lb
from oracle.inputs import letterbox_bgr_u8
from oracle.orient import orient

NETS = [(448, 448), (1280, 896), (416, 288), (160, 96)]      # (net_w, net_h)
SHRINKS = (0.5, 0.25)
F32 = np.float32


def view_box(net_w: int, net_h: int, shrink: float):
    """views_impl's box of a view: (int)(net * shrink) in float, at least 1."""
    return max(1, int(F32(net_w) * F32(shrink))), max(1, int(F32(net_h) * F32(shrink)))


def step_shapes(bw: int, bh: int, ks=(1, 2, 3, 4), ds=range(-3, 4)):
    """(h, w) with each side k * box + d: both sides of scale k, and at k = 2 every residue mod 4 of the side that is not binding."""
    return [(k * bh + dy, k * bw + dx) for k in ks for dy in ds for dx in ds]


def residue_shapes(bw: int, bh: int, ks=(1, 2, 3, 4)):
    """A binding side of exactly k * box and the other side of each residue mod 4, both ways round (503 x 896 into 448 x 448)."""
    out = []
    for k in ks:
        for r in range(4):
            other_h, other_w = (k * bh * 3 // 4) // 4 * 4 + r, (k * bw * 3 // 4) // 4 * 4 + r
            out += [(other_h, k * bw), (k * bh, other_w)]
    return out


def tie_shapes(bw: int, bh: int, per: int = 2):
    """Sides o whose resized size o * f is nearest a half-integer for a few binding sides: the round-half-to-even of dw / dh."""
    out = []
    for side in (bw + 1, 2 * bw + 3, 3 * bw - 1, 5 * bw // 2 + 1):
        _, _, scale = lb.geometry(side, 1, bw, bh)
        f = 1.0 / scale
        o = np.arange(2, 4 * bh + 1)
        frac = np.abs((o * f) % 1.0 - 0.5)
        for v in o[np.argsort(frac, kind="stable")[:per]]:
            if v * f < bh:
                out.append((int(v), side))
        hs = 2 * bh + 1 if side == 2 * bw + 3 else side * bh // bw       # the transposed case: height binding
        _, _, scale = lb.geometry(1, hs, bw, bh)
        f = 1.0 / scale
        o = np.arange(2, 4 * bw + 1)
        frac = np.abs((o * f) % 1.0 - 0.5)
        for v in o[np.argsort(frac, kind="stable")[:per]]:
            if v * f < bw:
                out.append((hs, int(v)))
    return out


def thin_shapes(bw: int, bh: int):
    """One-pixel sides and extreme aspect ratios: the side across the thin one rounds to 0 on the longest ones."""
    return [(1, 1), (1, bw + 1), (bh + 1, 1), (1, 2 * bw), (2 * bh, 1), (1, 5000), (5000, 1), (2, 5000), (5000, 2), (3, 4 * bw + 3)]


def _source(rng, h, w, cache):
    """A random image of h x w, sliced from one seeded buffer per sweep (contiguous, as cv2 wants it)."""
    big = cache.get("big")
    if big is None or big.shape[0] < h or big.shape[1] < w:
        big = cache["big"] = rng.integers(0, 256, (max(h, 5200), max(w, 5200), 3), dtype=np.uint8)
    return np.ascontiguousarray(big[:h, :w])


def _check(img, net_w, net_h, box, bits, flip_for_cv2, fails, label):
    """One item: the definition against cv2, or the degenerate rule where cv2 would refuse the size.  Returns 1 if compared."""
    bw, bh = box
    h, w = img.shape[:2]
    dw, dh, _ = lb.geometry(*((h, w) if bits & lb.LB_TRANSPOSE else (w, h)), bw, bh)
    mine = lb.letterbox(img, net_w, net_h, box=box, bits=bits)
    if dw == 0 or dh == 0:
        # cv2.resize asserts on an empty size; the engine's rule: the letter-box is all zero (no pixels, no faces, no fault)
        if mine.any():
            fails.append((label, "degenerate letter-box is not all zero"))
        return 0
    want = np.zeros((net_h, net_w, 3), np.uint8)
    want[:bh, :bw] = letterbox_bgr_u8(flip_for_cv2(img), bh, bw)
    if not np.array_equal(mine, want):
        d = np.argwhere(mine != want)
        fails.append((label, f"{len(d)} bytes differ, rows {np.unique(d[:, 0])[:4]}, cols {np.unique(d[:, 1])[:4]}"))
    return 1


@pytest.mark.parametrize("net", NETS, ids=[f"{w}x{h}" for w, h in NETS])
def test_definition_equals_cv2_where_resize_changes_path(net):
    net_w, net_h = net
    rng = np.random.default_rng(net_w * 7 + net_h)
    cache, fails, compared, degenerate = {}, [], 0, 0
    boxes = [((net_w, net_h), 0)] + [(view_box(net_w, net_h, s), lb.LB_FLIP_X if s == 0.5 else 0) for s in SHRINKS]
    for box, bits in boxes:
        bw, bh = box
        shapes = step_shapes(bw, bh) + residue_shapes(bw, bh) + tie_shapes(bw, bh) + thin_shapes(bw, bh)
        flip = (lambda a: cv2.flip(a, 1)) if bits & lb.LB_FLIP_X else (lambda a: a)
        for hw in dict.fromkeys(shapes):
            if min(hw) < 1:
                continue
            n = _check(_source(rng, *hw, cache), net_w, net_h, box, bits, flip, fails, (box, bits, hw))
            compared += n
            degenerate += 1 - n
    print(f"{net_w}x{net_h} and its view boxes: {compared} shapes compared with cv2, {degenerate} degenerate shapes all zero")
    assert not fails, fails[:20]
    assert compared >= 600 and degenerate >= 2


@pytest.mark.parametrize("o", range(1, 9))
def test_definition_of_every_orientation_equals_cv2_on_the_rotated_copy(o):
    """The reflections and the transposition: the item of orientation o is cv2's letter-box of T_o(img), on the exact-2x shapes of
    every residue (binding axis swapped by the transposition) and on both sides of scale 1 and 2."""
    rng = np.random.default_rng(o)
    cache, fails, compared = {}, [], 0
    for net_w, net_h in NETS[:3]:
        shapes = residue_shapes(net_w, net_h, ks=(2,)) + residue_shapes(net_h, net_w, ks=(2,)) + [
            (net_h + 1, net_w), (net_w, net_h + 1), (2 * net_w - 1, 2 * net_h + 1), (2 * net_h - 1, 2 * net_w - 3)]
        for hw in dict.fromkeys(shapes):
            compared += _check(_source(rng, *hw, cache), net_w, net_h, (net_w, net_h), lb.ORIENTATION_BITS[o], lambda a: orient(a, o),
                               fails, (net_w, net_h, hw, o))
    assert not fails, fails[:20]
    assert compared >= 40


@pytest.mark.parametrize("hw", [(503, 896), (896, 503)])
def test_bilinear_taps_at_exactly_2x_miss_opencvs_area_branch(hw):
    """Why the definition takes OpenCV's 2x branch: at exactly 2x with a side of 3 mod 4 (503 -> 252), the bilinear taps round the
    last row / column's one-pixel mean up where cv::resize rounds it half to even -- 1 LSB on a few hundred bytes, nowhere else."""
    img = np.random.default_rng(0).integers(0, 256, hw + (3,), dtype=np.uint8)
    want = letterbox_bgr_u8(img, 448, 448)
    assert np.array_equal(lb.letterbox(img, 448, 448), want)
    taps = lb.letterbox(img, 448, 448, half_area=False)
    d = np.argwhere(taps != want)
    assert len(d) > 100 and np.abs(taps.astype(int) - want).max() == 1
    edge = 0 if hw[0] == 503 else 1
    assert set(d[:, edge].tolist()) == {251}


def test_geometry_of_the_degenerate_and_npp_branches():
    """dw / dh of both branches where they round or clamp: the OpenCV branch rounds a thin side to 0 (an all-zero letter-box), the
    NPP branch takes the ceiling (never 0); neither exceeds the box, and a side at or below the box is kept."""
    assert lb.geometry(1, 5000, 448, 448)[:2] == (0, 448)
    assert lb.geometry(5000, 1, 448, 448)[:2] == (448, 0)
    assert lb.geometry_npp(1, 5000, 448, 448)[:2] == (1, 448)
    assert lb.geometry(1, 1, 448, 448) == (1, 1, 1.0) and lb.geometry_npp(1, 1, 448, 448) == (1, 1, 1.0)
    assert lb.geometry(896, 503, 448, 448) == (448, 252, 2.0)         # 251.5 rounds to even
    assert lb.geometry(896, 501, 448, 448) == (448, 250, 2.0)         # 250.5 rounds to even
    assert not lb.letterbox(np.full((1, 5000, 3), 200, np.uint8), 448, 448).any()
    for w, h in ((449, 3), (3, 449), (897, 1795), (5000, 7)):
        for g in (lb.geometry, lb.geometry_npp):
            dw, dh, _ = g(w, h, 448, 448)
            assert 0 <= dw <= 448 and 0 <= dh <= 448 and max(dw, dh) == 448


def test_half_rule_equals_cv2_on_tile_levels():
    """The same 2x rule at tile levels of scale 0.5 (tile_fill): resized() at scale 2 == cv2.resize(fx = fy = 0.5), plain and mirrored,
    for every pair of residues mod 4."""
    rng = np.random.default_rng(3)
    for h in range(61, 65):
        for w in range(97, 101):
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
            dw, dh = int(np.rint(w * 0.5)), int(np.rint(h * 0.5))
            for bits, src in ((0, img), (lb.LB_FLIP_X, cv2.flip(img, 1))):
                assert np.array_equal(lb.resized(img, dw, dh, 2.0, bits), cv2.resize(src, None, fx=0.5, fy=0.5)), (h, w, bits)
