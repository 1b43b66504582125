"""Host-only guard of the GPU geometry sweep (tests/test_gpu_plan_geometry.py): rf_plan_describe over every network size
H, W in {32, ..., 1280} for each precision, both models, the max_batch values and execution-context counts of
tests/plan_geometry.py, reduced to tile-geometry classes.  The sweep's cases must reach every class the planner can
produce, each case must reach a class no other case does, and the sizes the planner refuses are stated."""
import pytest

import plan_geometry as pg


@pytest.fixture(scope="module")
def plans(built_lib):
    return pg.enumerate_plans()


@pytest.fixture(scope="module")
def reachable(plans):
    return pg.reachable(plans)


def test_refusals_are_the_stated_ones(plans):
    """Every size either plans or is refused with RF_ERR_UNSUPPORTED and a message naming what does not fit."""
    for prec in pg.CONFIGS:
        got = {}
        for (p, model, h, w, mb, s), steps in plans.items():
            if p == prec and isinstance(steps, tuple):
                assert steps[1] == pg.REFUSAL[0] and steps[2].endswith(pg.REFUSAL[1]), ((p, model, h, w, mb, s), steps)
                got.setdefault((h, w), set()).add((model, mb, s))
        every = {(m, mb, s) for m in pg.MODELS for mb, s in pg.CONFIGS[prec]}
        assert set(got) == pg.REFUSED[prec], (pg.PREC_NAMES[prec], sorted(got))
        assert all(v == every for v in got.values()), (pg.PREC_NAMES[prec], got)


def test_geometry_is_the_same_for_both_models(plans):
    for (p, model, h, w, mb, s), steps in plans.items():
        if model == pg.MODELS[0]:
            assert plans[(p, pg.MODELS[1], h, w, mb, s)] == steps, (pg.PREC_NAMES[p], h, w, mb, s)


def test_every_2d_tile_is_16_wide(reachable):
    """dw2d_tile_w (plan_net.cu) picks TW = 14 when (ow + 13) / 14 < (ow + 15) / 16, which no positive ow satisfies:
    ceil(ow / 14) >= ceil(ow / 16).  So every 2-D tile is 16 wide and the kernels have never run TW = 14.  A planner change
    that makes 14 reachable fails here until the sweep runs it."""
    tws = {c[2] for p in reachable for c in reachable[p] if c[0] == "2-D dw+pw"}
    assert tws == {"TW=16"}, tws


def test_gpu_cases_reach_every_class(plans, reachable):
    """Prints the class table with the case that reaches each class; fails naming every class no case reaches, with the
    cheapest size that reaches it."""
    missing = []
    for prec in pg.CONFIGS:
        cases = [(cid, c) for cid, c in pg.CASES.items() if c.prec == prec]
        covered = {}
        for cid, c in cases:
            for cl in pg.case_classes(plans, c):
                covered.setdefault(cl, cid)
        print(f"\n{pg.PREC_NAMES[prec]}: {len(reachable[prec])} classes, {len(cases)} cases, "
              f"{sum(c.cost for _, c in cases) / 1e6:.2f} M pixels x images")
        for cl in sorted(reachable[prec]):
            print(f"   {' / '.join(cl):<90} {covered.get(cl, 'NOT REACHED')}")
            if cl not in covered:
                best = reachable[prec][cl]
                missing.append(f"{pg.PREC_NAMES[prec]} class {cl}: not reached by any case; the cheapest that reaches it is "
                               f"{best.hw[0]}x{best.hw[1]} max_batch {best.max_batch} forwarding {best.n}, streams "
                               f"{best.streams}, {best.model}")
        assert set(covered) <= set(reachable[prec]), set(covered) - set(reachable[prec])
    assert not missing, "\n".join(missing)


def test_every_gpu_case_is_needed(plans):
    """Each case reaches a class no other case of its precision reaches, but for the 9:16 portrait network every precision
    runs, whose anchor order on a map taller than wide the end-to-end check also covers."""
    for prec in pg.CONFIGS:
        cases = {cid: c for cid, c in pg.CASES.items() if c.prec == prec}
        portrait = [cid for cid, c in cases.items() if c.hw == pg.PORTRAIT]
        assert len(portrait) == 1, (pg.PREC_NAMES[prec], portrait)
        for cid, c in cases.items():
            if cid in portrait:
                continue
            others = set().union(*(pg.case_classes(plans, o) for oid, o in cases.items() if oid != cid))
            assert pg.case_classes(plans, c) - others, f"{cid} reaches no class the other cases do not"


def test_sweep_reaches_tall_thin_and_straddling_geometry(plans):
    """The sweep's cases include a network whose stride-32 map is k x 1, and GEMM / 1-D tiles that straddle images and
    that end inside one, on every precision."""
    for prec in pg.CONFIGS:
        cl = set().union(*(pg.case_classes(plans, c) for c in pg.CASES.values() if c.prec == prec))
        assert ("stride-32 map", "kx1") in cl, pg.PREC_NAMES[prec]
        tails = {c[-1] for c in cl if c[0] in ("1-D dw+pw", "staged conv", "SIMT GEMM")}
        assert {"straddles images", "ends mid-image"} <= tails, (pg.PREC_NAMES[prec], tails)


def test_cpu_oracle_budget():
    """The sweep forwards no more pixels x images than the FP16 step sweep does."""
    from test_gpu_fp16_steps import CASES as FP16_STEPS
    budget = sum(c.hw[0] * c.hw[1] * sum(c.runs) for c in FP16_STEPS.values())
    total = sum(c.cost for c in pg.CASES.values())
    print(f"\ngeometry sweep: {total / 1e6:.2f} M pixels x images, FP16 step sweep: {budget / 1e6:.2f} M")
    assert total <= budget
