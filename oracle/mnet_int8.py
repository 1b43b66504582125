"""Integer oracle of the INT8 path (RF_PREC_INT8).  Test infrastructure -- see ``oracle/__init__.py``.

What it restates.  The reference runs INT8 through TensorRT 5.1's closed-source kernels
(``retinaface/tensorrt/trtnetbase.cpp:295-311``); only their *inputs* are in the reference: the FP32
caffemodel and the per-tensor activation scales of ``model/mnet-deconv-0517.table.int8`` (symmetric,
dynamic range = 127 * scale; SURVEY.md Appendix C).  TensorRT's INT8 arithmetic itself cannot be reproduced
("parity unpinned" for INT8, DESIGN.md section 2), so the contract is the one north_star states: results
within the calibration's own tolerance of the FP32 path.  This module fixes the exact integer scheme the
CUDA engine implements, so that the engine can be checked to <= 1 LSB per tensor against it and the scheme
itself can be compared with the FP32 oracle:

* activations: q = clamp(rint(x * float32(1/s)), -127, 127), s = the table's scale of that Caffe top;
  quantised tensors are exactly the tensors that cross kernel boundaries in the engine (stem output
  relu2, every depthwise/pointwise output, laterals, FPN sums, aggr, SSH tensors); the stem interior and
  the predictor convs/softmax/decode stay FP32 (more accurate than quantising them, as TensorRT would).
* weights of GEMM-shaped convs: per output channel, s_w[o] = float32(max|w'[o]|)/127 on the BN-folded FP32
  weights, qw = rint(w'/s_w); depthwise weights stay FP32 (multiplied by the input scale).
* GEMM epilogue: v = float32(acc_int32) * m[o] + bq[o] (two float32 roundings), ReLU, requantise, with
  m[o] = float32(s_in * s_w[o] / s_out), bq[o] = float32(b'[o] / s_out)  (double arithmetic, then float32).
"""
from __future__ import annotations

import struct
from typing import Dict

import numpy as np

from .mnet_numpy import folded_params

F = np.float32


def read_table(path: str) -> Dict[str, float]:
    """TensorRT EntropyCalibration2 cache: '<tensor>: <8 hex digits>' = big-endian float32 scale."""
    out = {}
    lines = open(path).read().splitlines()
    assert lines[0].startswith("TRT-"), lines[0]
    for line in lines[1:]:
        if ": " not in line:
            continue
        k, v = line.rsplit(": ", 1)
        out[k] = struct.unpack(">f", bytes.fromhex(v.strip()))[0]
    return out


def quant(x, s):
    inv = F(1.0) / F(s)
    return np.clip(np.rint(x.astype(F) * inv), -127, 127).astype(np.int32)


def quant_weights(w):
    """w: (cout, K) float32 folded weights -> (qw int32, s_w float32[cout])."""
    mx = np.abs(w).max(axis=1).astype(F)
    sw = np.where(mx > 0, mx / F(127), F(1)).astype(F)
    qw = np.clip(np.rint(w.astype(np.float64) / sw.astype(np.float64)[:, None]), -127, 127).astype(np.int32)
    return qw, sw


def int_gemm(a, b):
    """Exact integer product a @ b of int32 matrices whose entries are within [-127, 127], as int64.  Multiplied in
    float64 so that numpy hands it to BLAS (it has no BLAS path for integers): every product and every partial sum is an
    integer far below 2**53, so each is exact in any summation order."""
    return (a.astype(np.float64) @ b.astype(np.float64)).astype(np.int64)


def _im2col(q, k, pad):
    """q: (n,c,h,w) int32 -> (n, h*w, k*k*c) with K ordered (tap, channel); stride 1."""
    n, c, h, w = q.shape
    qp = np.pad(q, ((0, 0), (0, 0), (pad, pad), (pad, pad))) if pad else q
    cols = np.empty((n, h, w, k * k, c), dtype=np.int32)
    for dy in range(k):
        for dx in range(k):
            cols[:, :, :, dy * k + dx, :] = qp[:, :, dy:dy + h, dx:dx + w].transpose(0, 2, 3, 1)
    return cols.reshape(n, h * w, k * k * c)


class Int8Oracle:
    def __init__(self, caffemodel: str, table: str):
        self.p = folded_params(caffemodel)
        self.t = read_table(table)

    # ---- building blocks ------------------------------------------------------------------------
    def gemm_conv(self, q_in, s_in, names, outs):
        """Conv (1x1 or 3x3, pad k//2, stride 1) of one or more convs sharing the input, concatenated along N.
        outs: list of (n_channels, s_out, relu) segments covering the concatenated N in order.
        Returns list of int32 tensors (n, c_seg, h, w), one per segment."""
        ws = [self.p[n]["w"] for n in names]
        bs = [self.p[n]["b"] for n in names]
        k = ws[0].shape[2]
        w = np.concatenate([x.transpose(0, 2, 3, 1).reshape(x.shape[0], -1) for x in ws])   # (N, taps*cin), (tap, cin) order
        b = np.concatenate(bs).astype(np.float64)
        qw, sw = quant_weights(w)
        n, c, h, wd = q_in.shape
        cols = _im2col(q_in, k, k // 2)
        acc = int_gemm(cols, qw.T)                                                        # exact integer GEMM
        assert np.abs(acc).max() < 2 ** 24
        res, o0 = [], 0
        for (cn, s_out, relu) in outs:
            m = (np.float64(s_in) * sw[o0:o0 + cn].astype(np.float64) / np.float64(s_out)).astype(F)
            bq = (b[o0:o0 + cn] / np.float64(s_out)).astype(F)
            v = (acc[:, :, o0:o0 + cn].astype(F) * m[None, None, :]).astype(F) + bq[None, None, :]
            if relu:
                v = np.maximum(v, F(0))
            q = np.clip(np.rint(v), -127, 127).astype(np.int32)
            res.append(q.reshape(n, h, wd, cn).transpose(0, 3, 1, 2))
            o0 += cn
        return res

    def dw_pw(self, q_in, s_in, i):
        """mobilenet0_conv{i} (depthwise, FP32 on dequantised input) + conv{i+1} (pointwise, integer GEMM)."""
        dw, pw = self.p[f"mobilenet0_conv{i}_fwd"], self.p[f"mobilenet0_conv{i + 1}_fwd"]
        s_mid, s_out = self.t[f"mobilenet0_relu{i}_fwd"], self.t[f"mobilenet0_relu{i + 1}_fwd"]
        c = q_in.shape[1]
        stride = 2 if i in (3, 7, 11, 23) else 1
        wf = (dw["w"].reshape(c, 9) * F(s_in)).astype(F)                     # input scale folded into the weights
        n, _, h, w = q_in.shape
        oh, ow = h // stride, w // stride
        xp = np.pad(q_in, ((0, 0), (0, 0), (1, 1), (1, 1))).astype(F)
        acc = np.broadcast_to(dw["b"].astype(F)[None, :, None, None], (n, c, oh, ow)).copy()
        for t in range(9):
            dy, dx = t // 3, t % 3
            acc = (acc + xp[:, :, dy:dy + stride * oh:stride, dx:dx + stride * ow:stride] * wf[None, :, t, None, None]).astype(F)
        q_mid = quant(np.maximum(acc, F(0)), s_mid)
        return self.gemm_conv(q_mid, s_mid, [f"mobilenet0_conv{i + 1}_fwd"], [(pw["w"].shape[0], s_out, True)])[0], s_out

    def stem(self, img_u8_nhwc):
        """conv0 + dw1 + pw2 in FP32 from the u8 image (exact inputs), output quantised with s(relu2)."""
        from .mnet_numpy import _conv2d, preprocess_bgr_u8
        x = np.concatenate([preprocess_bgr_u8(i) for i in img_u8_nhwc])
        for i, (s, g) in enumerate(((2, 1), (1, 8), (1, 1))):
            pr = self.p[f"mobilenet0_conv{i}_fwd"]
            x = np.maximum(_conv2d(x, pr["w"], pr["b"], s, 1 if pr["w"].shape[2] == 3 else 0, g), F(0))
        return quant(x, self.t["mobilenet0_relu2_fwd"]), self.t["mobilenet0_relu2_fwd"]

    def merge(self, q_lat, s_lat, q_up, s_up, which, s_out):
        """FPN merge: lateral + crop(deconv k4 s2 p1 depthwise(up)), requantised (prototxt:1553-1592)."""
        w = self.p["rf_c3_upsampling" if which == 0 else "rf_c2_upsampling"]["w"].reshape(-1, 4, 4)
        n, c, h, wd = q_lat.shape
        a_l = F(np.float64(s_lat) / np.float64(s_out))
        wq = (w.astype(np.float64) * np.float64(s_up) / np.float64(s_out)).astype(F)
        uh, uw = q_up.shape[2:]
        # same association as the kernels: the lateral term first, then the (up to) four taps in (ky, kx) order,
        # every product and every sum rounded to float32
        full = np.zeros((n, c, 2 * uh + 2, 2 * uw + 2), dtype=F)
        full[:, :, 1:1 + h, 1:1 + wd] = (q_lat.astype(F) * a_l).astype(F)
        for ky in range(4):
            for kx in range(4):
                full[:, :, ky:ky + 2 * uh:2, kx:kx + 2 * uw:2] += (q_up.astype(F) * wq[None, :, ky, kx, None, None]).astype(F)
        return np.clip(np.rint(full[:, :, 1:1 + h, 1:1 + wd]), -127, 127).astype(np.int32)

    def ssh(self, q_in, s_in, lv, tens=None):
        """The SSH context head of one level -> (concat, its scale); `tens`, when given, also receives the two quantised
        context tensors inside the head."""
        p = f"rf_{lv}_det"
        s_cat = self.t[p + "_concat_relu"]
        s_c1, s_c31 = self.t[p + "_context_conv1_relu"], self.t[p + "_context_conv3_1_relu"]
        det, ctx1 = self.gemm_conv(q_in, s_in, [p + "_conv1", p + "_context_conv1"], [(32, s_cat, True), (16, s_c1, True)])
        c2, c31 = self.gemm_conv(ctx1, s_c1, [p + "_context_conv2", p + "_context_conv3_1"], [(16, s_cat, True), (16, s_c31, True)])
        c32, = self.gemm_conv(c31, s_c31, [p + "_context_conv3_2"], [(16, s_cat, True)])
        if tens is not None:
            tens[p + "_context_conv1_relu"] = (ctx1, s_c1)
            tens[p + "_context_conv3_1_relu"] = (c31, s_c31)
        return np.concatenate([det, c2, c32], axis=1), s_cat

    def heads(self, q_cat, s_cat, stride):
        x = (q_cat.astype(F) * F(s_cat)).astype(F)
        out = {}
        for nm in ("cls_score", "bbox_pred", "landmark_pred"):
            pr = self.p[f"face_rpn_{nm}_stride{stride}"]
            out[nm] = (np.einsum("oc,nchw->nohw", pr["w"][:, :, 0, 0], x, optimize=True) + pr["b"][None, :, None, None]).astype(F)
        s = out["cls_score"]
        n, c, h, w = s.shape
        v = s.reshape(n, 2, 2 * h, w)
        v = v - v.max(axis=1, keepdims=True)
        e = np.exp(v)
        prob = (e / e.sum(axis=1, keepdims=True)).astype(F).reshape(n, c, h, w)
        return prob, out["bbox_pred"], out["landmark_pred"]

    # ---- whole network ---------------------------------------------------------------------------
    def forward(self, img_u8_nhwc, want_tensors=False, q_stem=None):
        """q_stem: optional int32 (n,16,h/2,w/2) stem output to continue from (lets a test separate the FP32 stem,
        whose summation order differs between implementations, from the bit-exact integer part)."""
        t = self.t
        if q_stem is None:
            q, s = self.stem(img_u8_nhwc)
        else:
            q, s = np.asarray(q_stem, dtype=np.int32), t["mobilenet0_relu2_fwd"]
        tens = {"mobilenet0_relu2_fwd": (q, s)}
        feats = {}
        for i in range(3, 27, 2):
            q, s = self.dw_pw(q, s, i)
            tens[f"mobilenet0_relu{i + 1}_fwd"] = (q, s)
            if i + 1 in (10, 22, 26):
                feats[i + 1] = (q, s)
        lat3, = self.gemm_conv(*feats[26], ["rf_c3_lateral"], [(64, t["rf_c3_lateral_relu"], True)])
        lat2, = self.gemm_conv(*feats[22], ["rf_c2_lateral"], [(64, t["rf_c2_lateral_relu"], True)])
        lat1, = self.gemm_conv(*feats[10], ["rf_c1_red_conv"], [(64, t["rf_c1_red_conv_relu"], True)])
        cat3, s3 = self.ssh(lat3, t["rf_c3_lateral_relu"], "c3", tens)
        plus0 = self.merge(lat2, t["rf_c2_lateral_relu"], lat3, t["rf_c3_lateral_relu"], 0, t["_plus0"])
        aggr2, = self.gemm_conv(plus0, t["_plus0"], ["rf_c2_aggr"], [(64, t["rf_c2_aggr_relu"], True)])
        cat2, s2 = self.ssh(aggr2, t["rf_c2_aggr_relu"], "c2", tens)
        plus1 = self.merge(lat1, t["rf_c1_red_conv_relu"], aggr2, t["rf_c2_aggr_relu"], 1, t["_plus1"])
        aggr1, = self.gemm_conv(plus1, t["_plus1"], ["rf_c1_aggr"], [(64, t["rf_c1_aggr_relu"], True)])
        cat1, s1 = self.ssh(aggr1, t["rf_c1_aggr_relu"], "c1", tens)
        tens.update({"rf_c3_lateral_relu": (lat3, t["rf_c3_lateral_relu"]), "rf_c2_lateral_relu": (lat2, t["rf_c2_lateral_relu"]),
                     "rf_c1_red_conv_relu": (lat1, t["rf_c1_red_conv_relu"]), "_plus0": (plus0, t["_plus0"]),
                     "rf_c2_aggr_relu": (aggr2, t["rf_c2_aggr_relu"]), "_plus1": (plus1, t["_plus1"]),
                     "rf_c1_aggr_relu": (aggr1, t["rf_c1_aggr_relu"]), "rf_c3_det_concat_relu": (cat3, s3),
                     "rf_c2_det_concat_relu": (cat2, s2), "rf_c1_det_concat_relu": (cat1, s1)})
        blobs = []
        for (cat, sc, stride) in ((cat3, s3, 32), (cat2, s2, 16), (cat1, s1, 8)):
            blobs += list(self.heads(cat, sc, stride))
        return (blobs, tens) if want_tensors else blobs
