"""The load sweep of the post-process's sort + greedy NMS (tests/test_gpu_nms_load.py; its host-only guards are
tests/test_nms_load_cpu.py): the branch constants of `nms_image` (csrc/postproc_dev.cuh), candidate-count targets on both sides
of each, the score threshold that yields a chosen candidate count, and the plans whose NMS instantiations the sweep reaches."""
import os
import re
from dataclasses import dataclass

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POSTPROC_DEV = os.path.join(ROOT, "retinaface_b200", "csrc", "postproc_dev.cuh")
CONSTANTS = ("NMS_MASK_MAX", "NMS_RANK_MAX", "NMS_SMEM_CAP")
ALL = None            # the "every anchor" target: a threshold below every P(face)


def nms_constants() -> dict:
    """NMS_MASK_MAX (one 64-bit suppression row per candidate), NMS_RANK_MAX (rank sort) and NMS_SMEM_CAP (shared-memory working
    set), as compiled."""
    text = open(POSTPROC_DEV).read()
    out = {}
    for name in CONSTANTS:
        m = re.search(rf"constexpr int {name} = (\d+);", text)
        assert m, f"{name} not found in {POSTPROC_DEV}"
        out[name] = int(m.group(1))
    return out


def regimes() -> list:
    """(name, lo, hi): the candidate counts each branch of nms_image handles, in order."""
    c = nms_constants()
    m, r, s = c["NMS_MASK_MAX"], c["NMS_RANK_MAX"], c["NMS_SMEM_CAP"]
    return [("rows", 0, m), ("rank+rounds", m + 1, r), ("bitonic", r + 1, s), ("bitonic-global", s + 1, 1 << 31)]


def regime(n: int) -> str:
    return next(name for name, lo, hi in regimes() if lo <= n <= hi)


def targets() -> list:
    """Candidate counts on both sides of every branch boundary, then every anchor."""
    out = []
    for _, _, hi in regimes()[:-1]:
        out += [hi, hi + 1]
    return out + [ALL]


def pface(heads, i: int) -> np.ndarray:
    """P(face) of image i of 9 head blobs (n, C, h, w) in emission order: stride 32, 16, 8; anchor 0, 1; pixels row-major."""
    return np.concatenate([np.asarray(heads[3 * lv][i, 2:4], np.float32).reshape(-1) for lv in range(3)])


def pick_threshold(p: np.ndarray, k, lo: int = 0, hi: int = 1 << 31):
    """(thr, count): a score threshold that leaves exactly `count` of the scores `p` above it (decode and oracle skip
    `conf <= thr`), with count the k nearest to `k` in [lo, hi] whose k-th and (k+1)-th largest scores differ.  k = ALL: a threshold
    below every score."""
    p = np.asarray(p, np.float32)
    if k is ALL:
        return np.float32(-1.0), len(p)
    s = np.sort(p)[::-1]
    top = min(hi, len(p))
    for d in range(0, len(p) + 1):
        for kk in (k - d, k + d):
            if lo <= kk <= top and (kk == 0 or kk == len(p) or s[kk - 1] > s[kk]):
                thr = s[kk] if kk < len(p) else np.float32(-1.0)
                assert int((p > thr).sum()) == kk
                return thr, kk
    raise ValueError(f"no untied count in [{lo}, {top}] near {k}")


@dataclass(frozen=True)
class Plan:
    hw: tuple                # (H, W) of the network input
    prec: str                # fp32 | fp16 | int8
    max_batch: int
    streams: int = 0
    nms: str = "fused"       # which NMS instantiation the plan holds: fused (k_head_decode's last block) or chain (the SSH tile
                             # chains' last CTA)

    @property
    def model(self):
        return "mnet-deconv-0517" if self.prec == "int8" else "mnet25"

    @property
    def anchors(self):
        return sum(2 * (self.hw[0] // s) * (self.hw[1] // s) for s in (32, 16, 8))


PLANS = {
    "fp32_448": Plan((448, 448), "fp32", 4),
    "fp16_448_b8": Plan((448, 448), "fp16", 8),                                        # the benchmarked FP16 plan
    "fp16_448_latency_b8": Plan((448, 448), "fp16", 8, streams=1, nms="chain"),        # SSH + predictor + NMS chains
    "fp16_448_latency_b2": Plan((448, 448), "fp16", 2, streams=1, nms="chain"),        # + merge + aggr chains
    "int8_448_b32": Plan((448, 448), "int8", 32),                                      # the benchmarked INT8 plan
    "fp16_1280x896_b3": Plan((896, 1280), "fp16", 3),
    "fp16_1280x896_latency_b3": Plan((896, 1280), "fp16", 3, streams=1),             # the SSH chains do not fit this size
    "fp16_416x288_latency": Plan((416, 288), "fp16", 3, streams=1, nms="chain"),
}
MAX_FACES = (256, 4, 8192)


def nms_variant(plan_text: str) -> str:
    """Which NMS instantiation an rf_plan_describe text holds (see Plan.nms)."""
    steps = [ln.split(": ", 1)[1] for ln in plan_text.splitlines() if ln.startswith("step lane")]
    fused = [s for s in steps if s.endswith("heads_1x1+softmax+decode+nms_all_levels")]
    chain = [s for s in steps if re.fullmatch(r"tile_ssh_c\d\+heads\+decode", s)]
    if len(fused) == 1 and not chain:
        return "fused"
    if len(chain) == 3 and not fused:
        return "chain"
    return "unknown: " + ", ".join(steps[-4:])
