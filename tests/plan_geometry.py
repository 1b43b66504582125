"""The tile geometry of every plan the planner builds, reduced to classes (host-only: rf_plan_describe with geometry).

Every network size H, W in {32, 64, ..., 1280} -- both orientations -- is described for each precision, both models, and
the execution-context counts and max_batch values below.  Each size either plans or is refused (status and message).  Each
plan is reduced to geometry classes: how every tiled launch divides its map into tiles, at a forward of max_batch images.
The GPU sweep (tests/test_gpu_plan_geometry.py) runs CASES, and tests/test_plan_geometry_cpu.py checks that together they
reach every class the enumeration finds.

A class keeps what decides which code path of a kernel's tiling runs:
- 2-D depthwise+pointwise tiles (TH x TW): the layer (stride, C -> N), TW, and whether the last tile column (OW mod TW) and
  row (OH mod TH) are partial.  The kernel bounds a partial tile by one test per output position and one clamp of the
  staged input columns, the same code for every nonzero remainder, so the remainder's value is not part of the class (its
  eight values at dw11 alone would need 32 networks above 896 x 896).
- 1-D depthwise+pointwise tiles (rows positions of the flattened batch) and GEMM tiles (k_conv_gemm's 64, the staged
  tensor-core convolutions' 128 padded positions): the rows, nsplit, N tile (NT / bn), and how the tiles meet the image
  boundaries (tail_class).
- The stride-32 map's shape (1 x 1, 1 x k, k x 1, k x k) and the network's orientation, per precision.
- Tile chains: the chain, its weights resident or streamed, whether its last tile is partial, and its map's orientation.
"""
import os
import re
from typing import NamedTuple

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = os.path.join(ROOT, "tests", "golden", "weights")
TABLE = os.path.join(WEIGHTS, "mnet-deconv-0517.table.int8")   # names every quantised tensor of both models

FP32, FP16, INT8 = 0, 1, 2
PREC_NAMES = {FP32: "FP32", FP16: "FP16", INT8: "INT8"}
MODELS = ("mnet25", "mnet-deconv-0517")
SIDES = tuple(range(32, 1281, 32))
# (max_batch, streams) per precision: the planner reads max_batch for the FPN merge fusion, the tile chains and their tile
# height, and streams for the chains; the SIMT plan reads neither (its tails still depend on the batch)
CONFIGS = {FP32: ((1, 0), (3, 0)),
           FP16: ((1, 0), (3, 0), (8, 0), (1, 1), (2, 1), (3, 1), (8, 1)),
           INT8: ((1, 0), (3, 0), (8, 0))}


class Case(NamedTuple):
    prec: int
    hw: tuple               # network (H, W)
    max_batch: int
    n: int                  # images forwarded (1 or max_batch)
    streams: int = 0
    model: str = "mnet25"

    @property
    def key(self):
        return self.prec, self.model, self.hw[0], self.hw[1], self.max_batch, self.streams

    @property
    def cost(self):
        return self.hw[0] * self.hw[1] * self.n


# The GPU sweep: the 9:16 portrait network 640 x 352 of every precision, then the cases greedy_cases chose from the
# enumeration, cheapest first by H * W * n, less each one whose classes the others reach.  Every case reaches a class no
# other case of its precision reaches (tests/test_plan_geometry_cpu.py).  Together they forward 7.7 M pixels x images,
# a third of the FP16 step sweep's 24 M (tests/test_gpu_fp16_steps.py): the CPU oracles' time is what this budget bounds.
CASE_LIST = (
    Case(FP32, (640, 352), 1, 1, 0, 'mnet25'),
    Case(FP32, (32, 32), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP32, (64, 32), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP32, (32, 160), 3, 3, 0, 'mnet-deconv-0517'),
    Case(FP16, (640, 352), 1, 1, 0, 'mnet25'),
    Case(FP16, (32, 96), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP16, (64, 64), 1, 1, 1, 'mnet-deconv-0517'),
    Case(FP16, (128, 32), 1, 1, 1, 'mnet-deconv-0517'),
    Case(FP16, (64, 96), 2, 2, 1, 'mnet-deconv-0517'),
    Case(FP16, (32, 192), 3, 3, 0, 'mnet-deconv-0517'),
    Case(FP16, (32, 864), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP16, (32, 1024), 1, 1, 1, 'mnet-deconv-0517'),
    Case(FP16, (32, 864), 2, 2, 1, 'mnet-deconv-0517'),
    Case(FP16, (992, 64), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP16, (160, 416), 2, 2, 1, 'mnet-deconv-0517'),
    Case(FP16, (64, 1184), 2, 2, 1, 'mnet-deconv-0517'),
    Case(FP16, (256, 1280), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP16, (1056, 768), 1, 1, 0, 'mnet-deconv-0517'),
    Case(FP16, (800, 1216), 8, 1, 1, 'mnet-deconv-0517'),
    Case(FP16, (1152, 1152), 1, 1, 1, 'mnet-deconv-0517'),
    Case(FP16, (1184, 1152), 1, 1, 1, 'mnet-deconv-0517'),
    Case(INT8, (640, 352), 1, 1, 0, 'mnet-deconv-0517'),
    Case(INT8, (32, 32), 1, 1, 0, 'mnet-deconv-0517'),
    Case(INT8, (64, 32), 1, 1, 0, 'mnet-deconv-0517'),
    Case(INT8, (32, 448), 1, 1, 0, 'mnet-deconv-0517'),
    Case(INT8, (32, 416), 3, 3, 0, 'mnet-deconv-0517'),
    Case(INT8, (992, 64), 1, 1, 0, 'mnet-deconv-0517'),
    Case(INT8, (768, 1056), 1, 1, 0, 'mnet-deconv-0517'),
    Case(INT8, (1056, 768), 1, 1, 0, 'mnet-deconv-0517'),
)
CASES = {f"{PREC_NAMES[c.prec]}_{c.hw[0]}x{c.hw[1]}_mb{c.max_batch}_n{c.n}_s{c.streams}_{c.model}": c for c in CASE_LIST}
PORTRAIT = (640, 352)

# What the planner refuses over the grid, for every model, max_batch and stream count: the FP16 tensor-core plan, where a
# 1-D depthwise+pointwise layer's staged input range does not fit shared memory (conv23 / conv25 on maps 2 or 1 wide).
# FP32 and INT8 plan every size.
REFUSED = {FP32: set(), INT8: set(),
           FP16: {(32, 32), (32, 64), (64, 32), (96, 32), (32, 992)}}
REFUSAL = (-7, "does not fit shared memory")     # RF_ERR_UNSUPPORTED and the message's tail


def describe(prec, model, h, w, max_batch, streams):
    """rf_plan_describe with geometry; a refusal as ("refused", status, message)."""
    from retinaface_b200.capi import RfError, plan_describe
    try:
        return plan_describe(os.path.join(WEIGHTS, model + ".caffemodel"), h, w, precision=prec, max_batch=max_batch,
                             int8_table=TABLE if prec == INT8 else None, streams=streams, geometry=True)
    except RfError as e:
        return ("refused", e.status, str(e))


def parse(text):
    """[(name, {key: value})] of the step lines, and the chain lines."""
    steps = []
    for ln in text.splitlines():
        if not ln.startswith("step lane "):
            continue
        body = ln.split(": ", 1)[1]
        name, _, geom = body.partition(" | ")
        kv = {}
        for word in geom.split():
            k, v = word.split("=")
            kv[k] = int(v) if re.fullmatch(r"-?\d+", v) else v
        steps.append((name, kv))
    return steps


def tail_class(per_image, tile, n):
    """How tiles of `tile` positions over n images of `per_image` positions each (flattened) meet the image boundaries."""
    if per_image % tile == 0:
        return "aligned"
    if per_image < tile:
        return "several images per tile" if n > 1 else "one image, one partial tile"
    return "straddles images" if n > 1 else "ends mid-image"


def shape_class(h, w):
    return "1x1" if h == w == 1 else ("1xk" if h == 1 else ("kx1" if w == 1 else "kxk"))


def orientation(h, w):
    return "tall" if h > w else ("wide" if h < w else "square")


def classes(prec, h, w, n, steps):
    """The geometry classes of one plan forwarding n images."""
    out = {("net", orientation(h, w)), ("stride-32 map", shape_class(h // 32, w // 32))}
    for name, g in steps:
        if m := re.fullmatch(r"(tc2d|i8_2d)_dw\d+\+pw\d+_s(\d)_(\d+)to(\d+)", name):
            layer = ("2-D dw+pw", f"s{m[2]} {m[3]}->{m[4]}", f"TW={g['TW']}")
            out.add(layer + ("last column " + ("full" if g["OW"] % g["TW"] == 0 else "partial"),))
            out.add(layer + ("last row " + ("full" if g["OH"] % g["TH"] == 0 else "partial"),))
        elif m := re.fullmatch(r"(tc|i8)_dw\d+\+pw\d+_s(\d)_(\d+)to(\d+)", name):
            out.add(("1-D dw+pw", f"s{m[2]}", f"rows={g['rows']}", f"nsplit={g['nsplit']}",
                     tail_class(g["OH"] * g["OW"], g["rows"], n)))
        elif "NT" in g:
            taps = "3x3" if "_3x3_" in name else "1x1"
            out.add(("staged conv", taps, f"NT={g['NT']}", f"merge {g['merge']}", tail_class(g["Hp"] * g["Wp"], g["BM"], n)))
        elif "bn" in g:
            ks = "3x3" if "_3x3_" in name else "1x1"
            out.add(("SIMT GEMM", ks, f"bn={g['bn']}", tail_class(g["H"] * g["W"], g["BM"], n)))
        elif name.startswith("tile_"):
            chain = ("tile chain", re.sub(r"_c\d", "", name))
            out.add(chain + (f"{g['weights']} weights",))
            out.add(chain + ("last tile " + ("full" if g["H"] % g["TH"] == 0 else "partial"),))
            out.add(chain + (f"{orientation(g['H'], g['W'])} map",))
        elif "stem" in name:
            out.add(("stem", name, "last column " + ("full" if g["OW"] % g["TW"] == 0 else "partial"),
                     "last row " + ("full" if g["OH"] % g["TH"] == 0 else "partial")))
    return out


def _one(args):
    text = describe(*args)
    return args, text if isinstance(text, tuple) else parse(text)


def enumerate_plans(processes=None):
    """{(prec, model, h, w, max_batch, streams): parsed steps, or ("refused", status, message)} over the whole grid."""
    from multiprocessing import get_context
    jobs = [(prec, model, h, w, mb, s) for prec, cfgs in CONFIGS.items() for model in MODELS for mb, s in cfgs
            for h in SIDES for w in SIDES]
    # spawned workers: a fork of a process that already runs threads (torch, the engine's host copies) may deadlock
    with get_context("spawn").Pool(processes or min(8, os.cpu_count() or 1)) as pool:
        return dict(pool.map(_one, jobs, chunksize=64))


def candidates(plans, prec):
    """Every case of `prec` the grid plans: each plan forwarding one image and max_batch images, cheapest first."""
    out = []
    for (p, model, h, w, mb, s), steps in plans.items():
        if p == prec and not isinstance(steps, tuple):
            out += [Case(p, (h, w), mb, n, s, model) for n in sorted({1, mb})]
    return sorted(out, key=lambda c: (c.cost, c))


def case_classes(plans, case):
    steps = plans[case.key]
    assert not isinstance(steps, tuple), (case, steps)
    return classes(case.prec, case.hw[0], case.hw[1], case.n, steps)


def reachable(plans):
    """{prec: {class: cheapest Case reaching it}}"""
    out = {p: {} for p in CONFIGS}
    for prec in CONFIGS:
        for case in candidates(plans, prec):
            for c in case_classes(plans, case):
                if c not in out[prec]:
                    out[prec][c] = case
    return out


def greedy_cases(plans, prec, seed=()):
    """Cases that together reach every class of `prec`: the `seed` cases, then, cheapest first by H * W * n, each case
    that reaches a class none before it does."""
    need = set(reachable(plans)[prec])
    chosen = list(seed)
    for c in chosen:
        need -= case_classes(plans, c)
    for c in candidates(plans, prec):
        if not need:
            break
        new = case_classes(plans, c) & need
        if new:
            chosen.append(c)
            need -= new
    return chosen
