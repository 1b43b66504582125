"""GPU (-m gpu): the post-process's sort + greedy NMS under load, in each of its three instantiations (the last block of
k_head_decode for float, half and int8 features; the last CTA of the SSH tile chains; stand-alone k_nms behind
rf_postprocess), on every branch of nms_image (tests/nms_load.py).  The score threshold of each call is derived from the
engine's own heads so that a target image has exactly a chosen number of candidates, on both sides of every branch boundary
and at every anchor; the NMS threshold is 0.4
(production), 1.0 (nothing suppressed: every candidate record is compared, and at every anchor each anchor is appended exactly
once) and 0.0 (any overlap suppresses); max_faces is the default 256, 4 and 8192.  Every image of every call must equal the C
oracle's post-process of the same heads (PostprocOracle.check_engine); so must rf_postprocess on those heads, and
rf_detect_batch_device's records must equal rf_detect_batch's bit for bit."""
import hashlib
import os
import time

import numpy as np
import pytest

from conftest import GOLDEN, caffemodel
from nms_load import ALL, MAX_FACES, PLANS, nms_constants, nms_variant, pface, pick_threshold, regime, regimes, targets
from oracle.inputs import mixed_batch
from oracle.postproc import PostprocOracle, compare_dets

pytestmark = pytest.mark.gpu

TABLE = os.path.join(GOLDEN, "weights", "mnet-deconv-0517.table.int8")
NMS = (0.4, 1.0, 0.0)
# nms 1.0 keeps every candidate, one suppression round each (and an O(n^2) oracle): beyond this many candidates in one image (the
# 1280 x 896 plans, 47,040 anchors) that case is skipped; 0.4 and 0.0 still run there at every anchor.
MAX_ROUNDS = 9000


def _engine(plan, max_faces):
    from retinaface_b200 import RF_PREC_FP16, RF_PREC_FP32, RF_PREC_INT8, Engine
    from retinaface_b200.capi import plan_describe
    prec = {"fp32": RF_PREC_FP32, "fp16": RF_PREC_FP16, "int8": RF_PREC_INT8}[plan.prec]
    kw = dict(precision=prec, max_batch=plan.max_batch, int8_table=TABLE if plan.prec == "int8" else None, streams=plan.streams)
    variant = nms_variant(plan_describe(caffemodel(plan.model), plan.hw[0], plan.hw[1], max_faces=max_faces, **kw))
    eng = Engine(caffemodel(plan.model), plan.hw[0], plan.hw[1], max_faces=max_faces, **kw)
    assert variant == plan.nms, (plan, max_faces, variant)
    assert eng.max_faces == max_faces and eng.num_anchors == plan.anchors
    return eng


def _batch(plan, photo):
    """A flat image (constant BGR: its interior anchors tie in score, so their order is the emission-index tie-break across every
    appending CTA) followed by mixed_batch's dissimilar neighbours (the photo, noise, all-255, all-0, shifted and mirrored
    copies)."""
    h, w = plan.hw
    flat = np.empty((h, w, 3), np.uint8)
    flat[:] = (90, 120, 160)
    return np.concatenate([flat[None], mixed_batch(photo, plan.max_batch - 1, h, w)])[:plan.max_batch]


class _Refs:
    """Oracle post-processes, cached by (image heads, thresholds): handles of one plan, and plans that differ only in how they
    schedule the same kernels, share heads."""
    cache = {}

    def __init__(self, plan):
        self.post, self.plan = PostprocOracle(), plan

    def keys(self, heads):
        return [hashlib.sha1(b"".join(np.ascontiguousarray(x[i]).tobytes() for x in heads)).hexdigest() for i in range(len(heads[0]))]

    def get(self, heads, keys, thr, nms):
        out = []
        for i, key in enumerate(keys):
            ck = (self.plan.hw, key, float(thr), nms)
            if ck not in self.cache:
                self.cache[ck] = self.post.postprocess([x[i] for x in heads], self.plan.hw[0], self.plan.hw[1], thr, nms)
            out.append(self.cache[ck])
        return out


def _threshold(ps, k, start):
    """(thr, count, target image) for target k: the first image from `start` on that has an untied count in k's regime."""
    lo, hi = (0, 1 << 31) if k is ALL else next((lo, hi) for _, lo, hi in regimes() if lo <= k <= hi)
    for d in range(len(ps)):
        t = (start + d) % len(ps)
        try:
            thr, kk = pick_threshold(ps[t], k, lo, hi)
            return thr, kk, t
        except ValueError:
            continue
    raise AssertionError(f"no image of the batch reaches {k} candidates in [{lo}, {hi}]")


def _device_records(eng, n, thr, nms, dev):
    d, c = eng.detect_device(n, float(thr), nms, dev.data_ptr())
    return list(zip(*eng.read_dets(d, c, n)))


@pytest.mark.parametrize("name", list(PLANS))
def test_nms_under_load_equals_the_oracle(name, golden_image):
    import torch
    plan = PLANS[name]
    refs = _Refs(plan)
    batch = _batch(plan, golden_image)
    n = len(batch)
    dev = torch.from_numpy(batch).cuda()
    smem_cap = nms_constants()["NMS_SMEM_CAP"]
    reached = set()
    t_plan = time.perf_counter()
    for mf in MAX_FACES:
        eng = _engine(plan, mf)
        try:
            label = f"{name} max_faces={mf} ({plan.nms} NMS)"
            heads = eng.forward_heads(batch)
            keys = refs.keys(heads)
            ps = [pface(heads, i) for i in range(n)]

            def run(thr, nms, sub=n):
                faces, idx = eng.detect_batch(list(batch[:sub]), float(thr), nms, want_index=True)
                rs = refs.get(heads, keys[:sub], thr, nms)
                refs.post.check_engine(eng, batch[:sub], None, thr, nms, f"{label} thr={thr} nms={nms}", refs=rs, dets=(faces, idx))
                return faces, idx, rs

            # a fresh handle's first call, at every anchor: the reference for the self-cleaning checks below
            thr_all = np.float32(-1.0)
            fresh = run(thr_all, 0.4)
            for i in range(n):
                assert len(fresh[2][i]["cand"]) == plan.anchors, (label, i)

            for ti, k in enumerate(targets()):
                thr, kk, t = _threshold(ps, k, ti)
                counts = [int((p > thr).sum()) for p in ps]
                assert counts[t] == kk and (k is ALL or regime(kk) == regime(k)), (label, k, kk)
                reached.add(regime(kk))
                for nms in NMS:
                    if nms == 1.0 and max(counts) > MAX_ROUNDS:
                        print(f"{label}: target {k} nms 1.0 skipped ({max(counts)} candidates in one image)")
                        continue
                    t0 = time.perf_counter()
                    faces, idx, rs = run(thr, nms)
                    dt = time.perf_counter() - t0
                    for i in range(n):
                        assert len(rs[i]["cand"]) == counts[i], (label, k, nms, i)
                        if nms == 1.0:      # nothing suppressed: every candidate kept, up to the output capacity
                            assert len(rs[i]["idx"]) == counts[i] and len(faces[i]) == min(counts[i], mf), (label, k, i)
                            if k is ALL:
                                assert sorted(rs[i]["idx"].tolist()) == list(range(plan.anchors))
                    # rf_postprocess (decode + k_nms) on the same heads: the same selection
                    pf, pidx, pc = eng.postprocess(heads, float(thr), nms)
                    assert pc.tolist() == counts, (label, k, nms)
                    for i in range(n):
                        compare_dets(pf[i], pidx[i], rs[i], f"{label} rf_postprocess k={k} nms={nms} image {i}", mf)
                    print(f"{label}: target {k} -> image {t} {kk} candidates ({regime(kk)}), nms {nms}: candidates "
                          f"{counts} (regimes {sorted({regime(c) for c in counts})}), kept {[len(f) for f in faces]}, "
                          f"detect {dt * 1e3:.1f} ms incl. oracle")

            # mixed loads in one call: the image with the lowest top score gets no candidate, its neighbours many
            tops = [float(p.max()) for p in ps]
            z = int(np.argmin(tops))
            thr = np.float32(tops[z])
            counts = [int((p > thr).sum()) for p in ps]
            faces, _, _ = run(thr, 0.4)
            assert counts[z] == 0 and len(faces[z]) == 0 and max(counts) > 0, (label, counts)
            print(f"{label}: mixed loads {counts}, {sum(c > smem_cap for c in counts)} image(s) past the shared-memory set")

            # self-cleaning state: light then heavy again, and a smaller batch after a full one, bit-equal to the fresh handle's
            thr64, _, _ = _threshold(ps, targets()[0], 0)
            run(thr64, 0.4)
            again = run(thr_all, 0.4)
            for i in range(n):
                assert np.array_equal(again[0][i], fresh[0][i]) and np.array_equal(again[1][i], fresh[1][i]), (label, i)
            sub = max(1, n // 2)
            part = run(thr_all, 0.4, sub)
            for i in range(sub):
                assert np.array_equal(part[0][i], fresh[0][i]) and np.array_equal(part[1][i], fresh[1][i]), (label, i)

            # the device entry point at the heavy loads: records bit-equal to rf_detect_batch's, over consecutive calls
            for k in (targets()[-2], ALL):
                thr = _threshold(ps, k, 1)[0]
                faces, idx = eng.detect_batch(list(batch), float(thr), 0.4, want_index=True)
                for _ in range(2):
                    recs = _device_records(eng, n, thr, 0.4, dev)
                    for i in range(n):
                        assert np.array_equal(recs[i][0], faces[i]) and np.array_equal(recs[i][1], idx[i]), (label, k, i)
        finally:
            eng.close()
    print(f"{name}: regimes reached {sorted(reached)}; {time.perf_counter() - t_plan:.1f} s")
    assert reached == {r for r, _, _ in regimes()}
