"""ctypes loaders for the post-process oracle (C restatement) and ``oracle/_ref``.

Test infrastructure -- see ``oracle/__init__.py``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import List, Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
FACE_FLOATS = 15  # FaceDetectInfo: score, x1,y1,x2,y2, x[5], y[5]  (RetinaFace.h:37-42)
STRIDES = (32, 16, 8)  # _feat_stride_fpn, RetinaFace.cpp:246


def build(force: bool = False) -> None:
    """Compile the C restatement (always) and oracle/_ref (when /root/reference exists)."""
    so = os.path.join(_HERE, "liboracle_postproc.so")
    src = os.path.join(_HERE, "postproc.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle_postproc.so"], stdout=subprocess.DEVNULL)
    ref_so = os.path.join(_HERE, "_ref", "libref_postproc.so")
    if os.path.exists("/root/reference/retinaface/RetinaFace.cpp") and (force or not os.path.exists(ref_so)):
        subprocess.check_call([os.path.join(_HERE, "build_ref.sh")], stdout=subprocess.DEVNULL)


def head_shapes(net_h: int, net_w: int) -> List[Tuple[int, int, int]]:
    """(C,h,w) of the 9 head blobs in engine order (tensorrt/trtretinafacenet.cpp:23-31)."""
    out = []
    for s in STRIDES:
        for c in (4, 8, 20):
            out.append((c, net_h // s, net_w // s))
    return out


def _heads_ptrs(heads: Sequence[np.ndarray]):
    keep = [np.ascontiguousarray(h, dtype=np.float32) for h in heads]
    arr = (C.POINTER(C.c_float) * 9)(*[h.ctypes.data_as(C.POINTER(C.c_float)) for h in keep])
    return arr, keep


def compare_dets(mine, mine_idx, ref, label="", max_faces=None):
    """Detections against a PostprocOracle.postprocess result: selection (anchor emission indices, order) exact; scores and
    landmarks bit-exact; box corners within 4e-6 relative (the exp() rounding noted in postproc.cu).  With `max_faces`, the
    output capacity: the count is min(kept, max_faces) and the faces are the oracle's top-scoring prefix."""
    ridx, rfaces = ref["idx"], ref["faces"]
    if max_faces is not None and len(ridx) > max_faces:
        ridx, rfaces = ridx[:max_faces], rfaces[:max_faces]
    assert mine_idx.tolist() == ridx.tolist(), label
    a, b = mine, rfaces
    assert a.shape == b.shape, label
    if len(a) == 0:
        return
    assert np.array_equal(a[:, 0], b[:, 0]), label            # scores
    assert np.array_equal(a[:, 5:], b[:, 5:]), label          # landmarks
    assert np.allclose(a[:, 1:5], b[:, 1:5], rtol=4e-6, atol=1e-4), label


class PostprocOracle:
    """The plain-C restatement (oracle/postproc.c)."""

    def __init__(self):
        build()
        self.lib = C.CDLL(os.path.join(_HERE, "liboracle_postproc.so"))
        self.lib.rfo_postprocess.restype = C.c_int
        self.lib.rfo_nms.restype = C.c_int
        self.lib.rfo_base_anchors.restype = C.c_int

    def base_anchors(self, stride: int) -> np.ndarray:
        out = np.zeros(8, dtype=np.float32)
        n = self.lib.rfo_base_anchors(C.c_int(stride), out.ctypes.data_as(C.c_void_p))
        assert n == 2
        return out.reshape(2, 4)

    def postprocess(self, heads: Sequence[np.ndarray], net_h: int, net_w: int, thr: float, nms_thr: float):
        """heads: 9 arrays (C,h,w) for ONE image.  Returns dict(cand, cand_idx, faces, idx)."""
        cap = sum(2 * (net_h // s) * (net_w // s) for s in STRIDES)
        ptrs, keep = _heads_ptrs(heads)
        cand = np.zeros((cap, FACE_FLOATS), dtype=np.float32)
        cand_idx = np.zeros(cap, dtype=np.int32)
        out = np.zeros((cap, FACE_FLOATS), dtype=np.float32)
        out_idx = np.zeros(cap, dtype=np.int32)
        n_cand = C.c_int(0)
        kept = self.lib.rfo_postprocess(
            ptrs, C.c_int(net_h), C.c_int(net_w), C.c_float(thr), C.c_float(nms_thr),
            cand.ctypes.data_as(C.c_void_p), cand_idx.ctypes.data_as(C.c_void_p), C.c_int(cap), C.byref(n_cand),
            out.ctypes.data_as(C.c_void_p), out_idx.ctypes.data_as(C.c_void_p))
        n = n_cand.value
        return dict(cand=cand[:n].copy(), cand_idx=cand_idx[:n].copy(),
                    faces=out[:kept].copy(), idx=out_idx[:kept].copy())

    def check_engine(self, eng, batch, heads, thr: float, nms_thr: float, label: str = "", refs=None, dets=None) -> int:
        """An engine's detections of `batch` (rf_detect_batch, or `dets` = (faces, indices) it already returned) against this
        post-process of the engine's own `heads` (or `refs`, one postprocess() result per image), compared by compare_dets with
        the engine's max_faces.  Returns the number of faces compared."""
        h, w = batch.shape[1:3]
        faces, idx = dets if dets is not None else eng.detect_batch(list(batch), thr, nms_thr, want_index=True)
        for i in range(len(batch)):
            ref = refs[i] if refs is not None else self.postprocess([x[i] for x in heads], h, w, thr, nms_thr)
            compare_dets(faces[i], idx[i], ref, f"{label} image {i}", eng.max_faces)
        return sum(len(f) for f in faces)

    def nms(self, cands: np.ndarray, thr: float):
        cands = np.ascontiguousarray(cands, dtype=np.float32).reshape(-1, FACE_FLOATS)
        n = cands.shape[0]
        out = np.zeros((max(n, 1), FACE_FLOATS), dtype=np.float32)
        pos = np.zeros(max(n, 1), dtype=np.int32)
        k = self.lib.rfo_nms(cands.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_float(thr),
                             out.ctypes.data_as(C.c_void_p), pos.ctypes.data_as(C.c_void_p))
        return out[:k].copy(), pos[:k].copy()


class ReferencePostproc:
    """oracle/_ref: the reference's own compiled RetinaFace.cpp behind a fake engine."""

    @staticmethod
    def available() -> bool:
        return os.path.exists(os.path.join(_HERE, "_ref", "libref_postproc.so"))

    def __init__(self, net_h: int, net_w: int):
        self.lib = C.CDLL(os.path.join(_HERE, "_ref", "libref_postproc.so"))
        self.lib.ref_create.restype = C.c_void_p
        self.lib.ref_postprocess.restype = C.c_int
        self.lib.ref_nms.restype = C.c_int
        self.lib.ref_base_anchors.restype = C.c_int
        self.lib.ref_anchor_plane.restype = C.c_int
        self.net_h, self.net_w = net_h, net_w
        self.h = C.c_void_p(self.lib.ref_create(C.c_int(net_w), C.c_int(net_h)))

    def close(self):
        if self.h:
            self.lib.ref_destroy(self.h)
            self.h = None

    def base_anchors(self, stride: int) -> np.ndarray:
        out = np.zeros(8, dtype=np.float32)
        n = self.lib.ref_base_anchors(self.h, C.c_int(stride), out.ctypes.data_as(C.c_void_p))
        assert n == 2
        return out.reshape(2, 4)

    def anchor_plane(self, stride: int) -> np.ndarray:
        n = 2 * (self.net_h // stride) * (self.net_w // stride)
        out = np.zeros((n, 4), dtype=np.float32)
        m = self.lib.ref_anchor_plane(self.h, C.c_int(stride), out.ctypes.data_as(C.c_void_p), C.c_int(n))
        assert m == n, (m, n)
        return out

    def postprocess(self, heads: Sequence[np.ndarray], thr: float) -> np.ndarray:
        """Reference RetinaFace::postProcess (NMS 0.4 hard-coded, RetinaFace.cpp:571)."""
        cap = sum(2 * (self.net_h // s) * (self.net_w // s) for s in STRIDES)
        ptrs, keep = _heads_ptrs(heads)
        out = np.zeros((cap, FACE_FLOATS), dtype=np.float32)
        n = self.lib.ref_postprocess(self.h, ptrs, C.c_float(thr), out.ctypes.data_as(C.c_void_p), C.c_int(cap))
        return out[:n].copy()

    def nms(self, cands: np.ndarray, thr: float) -> np.ndarray:
        cands = np.ascontiguousarray(cands, dtype=np.float32).reshape(-1, FACE_FLOATS)
        out = np.zeros((max(len(cands), 1), FACE_FLOATS), dtype=np.float32)
        k = self.lib.ref_nms(self.h, cands.ctypes.data_as(C.c_void_p), C.c_int(len(cands)), C.c_float(thr),
                             out.ctypes.data_as(C.c_void_p))
        return out[:k].copy()


def synth_heads(net_h: int, net_w: int, n_cand: int, seed: int = 1, n_centres: int = 32,
                thr: float = 0.9) -> List[np.ndarray]:
    """S-nms synthetic head tensors (SURVEY.md section 8d): ~n_cand anchors above `thr`,
    clustered around `n_centres` centres so NMS suppresses most of them.  Scores are unique
    (no ties) so that the unstable std::sort of the reference is deterministic."""
    rng = np.random.default_rng(seed)
    shapes = head_shapes(net_h, net_w)
    heads = [np.zeros(s, dtype=np.float32) for s in shapes]
    total = sum(2 * (net_h // s) * (net_w // s) for s in STRIDES)
    centres = rng.uniform([0, 0], [net_w, net_h], size=(n_centres, 2))
    # choose anchors near centres with probability decaying with distance
    prob_list = []
    for li, s in enumerate(STRIDES):
        h, w = net_h // s, net_w // s
        ys, xs = np.mgrid[0:h, 0:w]
        cx = xs * s + 7.5
        cy = ys * s + 7.5
        d2 = ((cx[None] - centres[:, 0, None, None]) ** 2 + (cy[None] - centres[:, 1, None, None]) ** 2).min(0)
        p = np.exp(-d2 / (2 * (3.0 * s) ** 2))
        prob_list.append(np.stack([p, p]).reshape(-1))
    prob = np.concatenate(prob_list)
    prob = prob / prob.sum()
    n_cand = min(n_cand, total)
    chosen = rng.choice(total, size=n_cand, replace=False, p=prob)
    face = np.zeros(total, dtype=bool)
    face[chosen] = True
    # unique scores: candidates in (thr, 1), the rest in (0, thr)
    hi = thr + (1 - thr) * (rng.permutation(n_cand) + 0.5) / n_cand
    lo = thr * 0.98 * (rng.permutation(total) + 0.5) / total   # unique as float32 too
    score = lo.astype(np.float32)
    score[chosen] = hi.astype(np.float32)
    off = 0
    for li, s in enumerate(STRIDES):
        h, w = net_h // s, net_w // s
        n = 2 * h * w
        sc = score[off:off + n].reshape(2, h, w)
        heads[3 * li][2:4] = sc
        heads[3 * li][0:2] = 1.0 - sc
        heads[3 * li + 1][:] = rng.normal(0, 0.2, size=shapes[3 * li + 1]).astype(np.float32)
        heads[3 * li + 2][:] = rng.normal(0, 0.2, size=shapes[3 * li + 2]).astype(np.float32)
        off += n
    return heads
