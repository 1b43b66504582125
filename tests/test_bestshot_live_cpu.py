"""CPU: the f22 live best-shot policy (rf_b200.h rf_tracker_set_best_live) as tests/bestshot_live_oracle.py restates it, on scripted
qualities: the first shot, the gap, the improvement ratio, a held-back improvement, LOST and TENTATIVE tracks, the count bound, EXIT and
FINISH unchanged, live=None equal to BestShotOracle, and a follow frame emitting only removals."""
import numpy as np
import pytest

import oracle.bestshot as bs
from bestshot_live_oracle import BEST_LIVE, LiveBestShotOracle, live_config, live_emits, max_live_shots
from oracle.bestshot import BEST_EXIT, BEST_FINISH, BestShotOracle
from oracle.track import CONFIRMED, LOST, TENTATIVE

CROP = np.zeros((4, 4, 3), np.int32)     # scripted: the first value carries the frame number
M = np.zeros(6)


@pytest.fixture
def scripted(monkeypatch):
    """quality() returns the q scripted for (frame, id) -- the crop's first byte carries the frame, the face's score the id."""
    script = {}

    def quality(crop, face, M, w, h, template=None, sharp_half=None):
        key = (int(crop[0, 0, 0]), int(round(float(np.asarray(face, np.float32)[0]))))
        q = script.get(key, 0.0)
        return dict(score=0.0, eye=0.0, frontal=0.0, sharpness=0.0, coverage=0.0, q=q)
    monkeypatch.setattr(bs, "quality", quality)
    return script


def _track(tid, state, det, hits, age):
    face = np.zeros(15, np.float32)
    face[0] = tid
    return dict(id=tid, state=state, det=det, hits=hits, age=age, face=face)


def _run(o, frames):
    """frames: per frame a list of (id, state, det, hits, age); every record's crop carries the frame number."""
    out = []
    for f, tracks in enumerate(frames):
        tr = [_track(*t) for t in tracks]
        crop = CROP.copy()
        crop[0, 0, 0] = f
        out.append(o.update(0, tr, [crop] * 8, [M] * 8, 100, 100))
    return out


def _confirmed_run(n, ids=(1,)):
    return [[(i, TENTATIVE if f == 0 else CONFIRMED, k, f + 1, f + 1) for k, i in enumerate(ids)] for f in range(n)]


def test_config_defaults_and_bounds():
    c = live_config()
    assert c["first_quality"] == float(np.float32(0.3)) and c["min_gap"] == 30 and c["ratio"] == 1.0 + float(np.float32(0.2))
    assert max_live_shots(c) == 7
    for bad in (dict(first_quality=1.5), dict(first_quality=-0.1), dict(first_quality=float("nan")), dict(improve=-1.0),
                dict(improve=float("inf")), dict(improve=float("nan")), dict(min_gap=-1), dict(min_gap=(1 << 20) + 1)):
        with pytest.raises(ValueError):
            live_config(**bad)


def test_policy_as_a_function():
    c = live_config(first_quality=0.5, improve=0.25, min_gap=3)
    assert not live_emits(0.49, 0, 0.0, 0, 5, c, 0.0) and live_emits(0.5, 0, 0.0, 0, 5, c, 0.0)
    assert not live_emits(0.6, 0, 0.0, 0, 5, c, 0.7)              # min_quality applies to the first shot too
    assert not live_emits(0.9, 1, 0.5, 4, 6, c, 0.0)              # the gap
    assert not live_emits(0.625, 1, 0.5, 4, 7, c, 0.0)            # exactly the ratio is not strictly better
    assert live_emits(0.6250001, 1, 0.5, 4, 7, c, 0.0)


def test_first_shot_gap_ratio_and_held_back(scripted):
    o = LiveBestShotOracle(live=dict(first_quality=0.4, improve=0.5, min_gap=3))
    qs = [0.1, 0.2, 0.45, 0.5, 0.9, 0.95, 0.95, 0.95, 0.95]
    for f, q in enumerate(qs):
        scripted[(f, 1)] = q
    out = _run(o, _confirmed_run(len(qs)))
    live = [(f, int(s["frame"]), float(s["quality"])) for f, per in enumerate(out) for s in per if s["reason"] == BEST_LIVE]
    # frame 2: the first q >= 0.4; frame 4 (0.9 > 0.45 * 1.5) is held back by the gap until frame 5, which emits its best so far
    assert [(f, fr) for f, fr, _ in live] == [(2, 2), (5, 5)]
    s = out[5][0]
    assert int(s["end_frame"]) == 5 and int(s["hits"]) == 6 and int(s["age"]) == 6 and s["reason"] == BEST_LIVE


def test_lost_and_tentative_never_emit(scripted):
    o = LiveBestShotOracle(live=dict(first_quality=0.1, min_gap=1))
    for f in range(6):
        scripted[(f, 1)] = 0.9
    frames = [[(1, TENTATIVE, 0, 1, 1)], [(1, TENTATIVE, 0, 1, 2)], [(1, LOST, -1, 1, 3)], [(1, LOST, -1, 1, 4)],
              [(1, CONFIRMED, 0, 2, 5)]]
    out = _run(o, frames)
    assert [len(p) for p in out] == [0, 0, 0, 0, 1] and out[4][0]["reason"] == BEST_LIVE
    # a born-CONFIRMED track on the video's first frame emits there
    o2 = LiveBestShotOracle(live=dict(first_quality=0.1))
    out = _run(o2, [[(1, CONFIRMED, 0, 1, 1)]])
    assert len(out[0]) == 1 and int(out[0][0]["frame"]) == 0


def test_count_bound_on_a_rising_ramp(scripted):
    o = LiveBestShotOracle(live=dict(min_gap=1))
    n = 400
    for f in range(n):
        scripted[(f, 1)] = min(1.0, 0.3 * 1.0005 ** (f * 10))
    out = _run(o, _confirmed_run(n))
    k = sum(s["reason"] == BEST_LIVE for p in out for s in p)
    assert k == max_live_shots(live_config()) == 7


def _exits_and_finish(o, frames):
    out = _run(o, frames)
    return out, o.finish(0)


def _strip(shots):
    return [{k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in s.items()} for s in shots]


def test_live_is_additive_and_none_is_the_f11_oracle(scripted):
    rng = np.random.default_rng(7)
    frames = []
    for f in range(40):
        tr = []
        if f < 25:
            tr.append((1, TENTATIVE if f == 0 else (LOST if 12 <= f < 15 else CONFIRMED), -1 if 12 <= f < 15 else 0, f + 1, f + 1))
        if 3 <= f < 30:
            tr.append((2, TENTATIVE if f == 3 else CONFIRMED, 1, f - 2, f - 2))
        if f >= 10:
            tr.append((3, TENTATIVE if f == 10 else CONFIRMED, 2, f - 9, f - 9))
        frames.append(tr)
        for i in (1, 2, 3):
            scripted[(f, i)] = float(rng.random())
    base_out, base_fin = _exits_and_finish(BestShotOracle(min_quality=0.1), frames)
    none_out, none_fin = _exits_and_finish(LiveBestShotOracle(min_quality=0.1), frames)
    assert [_strip(p) for p in none_out] == [_strip(p) for p in base_out] and _strip(none_fin) == _strip(base_fin)
    live_out, live_fin = _exits_and_finish(LiveBestShotOracle(min_quality=0.1, live=dict(first_quality=0.2, improve=0.1, min_gap=2)), frames)
    assert any(s["reason"] == BEST_LIVE for p in live_out for s in p)
    assert [_strip([s for s in p if s["reason"] != BEST_LIVE]) for p in live_out] == [_strip(p) for p in base_out]
    assert _strip(live_fin) == _strip(base_fin) and all(s["reason"] == BEST_FINISH for s in live_fin)
    for p in live_out:
        ids = [int(s["id"]) for s in p]
        assert ids == sorted(set(ids))          # one shot per track per frame, in id order
    assert any(s["reason"] == BEST_EXIT for p in live_out for s in p)


def test_a_follow_frame_emits_only_removals(scripted):
    o = LiveBestShotOracle(live=dict(first_quality=0.1, min_gap=1))
    for f in range(4):
        scripted[(f, 1)] = scripted[(f, 2)] = 0.5 + 0.1 * f
    # frames 0-1 detect; frame 2 a follow frame (det -1 everywhere): track 2 removed there, track 1 followed
    out = _run(o, [[(1, CONFIRMED, 0, 1, 1), (2, CONFIRMED, 1, 1, 1)], [(1, CONFIRMED, 0, 2, 2), (2, CONFIRMED, 1, 2, 2)],
                   [(1, CONFIRMED, -1, 2, 3)], [(1, CONFIRMED, 0, 3, 4)]])
    assert [s["reason"] for s in out[2]] == [BEST_EXIT] and int(out[2][0]["id"]) == 2 and int(out[2][0]["age"]) == 3
    assert [s["reason"] for s in out[3]] == [BEST_LIVE] and int(out[3][0]["frame"]) == 3
