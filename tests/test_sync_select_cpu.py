"""CPU: the host's candidate selection from a peak list (hostapi.stage_select = select_candidates_from_peaks, the selection `get`
runs on the local maxima awm_sync_peaks returns above a floor, lowering the floor until the selection is complete) against the
oracle chain select_local_maxima -> mask_avg_false_positives -> select_threshold_and_n_best (+ select_truncate_n in CLIP mode) on
the full score list.  Whenever stage_select reports the selection complete it must be the oracle's, at every floor of the cascade.
"""
import numpy as np
import pytest

import awm_oracle as O
from audiowmark_b200 import capi, hostapi as H

P = O.Params()
THRESHOLD = P.sync_threshold2 * 0.75
FLOORS = (THRESHOLD, THRESHOLD * 0.6, THRESHOLD * 0.35, THRESHOLD * 0.15, 0.0, -1.0)
STEP = P.sync_search_step


def background(m, seed, amp=0.05):
    rng = np.random.default_rng(seed)
    s = np.zeros(m, capi.SEARCH_SCORE)
    s["index"] = np.arange(m, dtype=np.uint64) * STEP
    s["raw_quality"] = (rng.random(m) - 0.5) * 2 * amp
    s["local_mean"] = (rng.random(m) - 0.5) * 0.002
    return s


def put(s, pos, q):
    """a score of |raw - mean| = |q| exactly, sign of q"""
    s["raw_quality"][pos] = q
    s["local_mean"][pos] = 0.0


def peaks_above(s, floor_q):
    """what awm_sync_peaks hands the host: |q| > floor, >= both neighbours (0 beyond the ends), sorted by index"""
    a = np.abs(s["raw_quality"] - s["local_mean"])
    prev = np.concatenate([[0.0], a[:-1]])
    nxt = np.concatenate([a[1:], [0.0]])
    return s[(a > floor_q) & (a >= prev) & (a >= nxt)]


def oracle_select(s, clip):
    sf = O.SyncFinder(P)
    sc = [O.SearchScore(int(r["index"]), float(r["raw_quality"]), float(r["local_mean"])) for r in s]
    sel = sf.select_threshold_and_n_best(sf.mask_avg_false_positives(sf.select_local_maxima(sc)), THRESHOLD)
    if clip:
        sel = sf.select_truncate_n(sel, max(P.get_n_best, 5))
    return sorted((w.index, w.raw_quality, w.local_mean) for w in sel)


def check(s, clip, expect_incomplete_above=None):
    """stage_select at every floor of the cascade; every complete answer equals the oracle's; floor -1 is always complete.
    Returns the floors that were complete."""
    want = oracle_select(s, clip)
    complete_at = []
    for floor_q in FLOORS:
        got, complete = H.stage_select(peaks_above(s, floor_q), floor_q, clip)
        if complete:
            got = sorted((int(g["index"]), float(g["raw_quality"]), float(g["local_mean"])) for g in got)
            assert got == want, (floor_q, clip, got, want)
            complete_at.append(floor_q)
    assert complete_at and complete_at[-1] == -1.0
    if expect_incomplete_above is not None:
        assert all(f < expect_incomplete_above for f in complete_at), complete_at
    return want, complete_at


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("n_above", [0, 3, P.get_n_best - 1, P.get_n_best, P.get_n_best + 1, 13])
def test_count_above_threshold(clip, n_above):
    """none, fewer, exactly get_n_best and more peaks above the threshold, plus weaker peaks that fill up to n-best by count"""
    rng = np.random.default_rng(n_above + 100 * clip)
    s = background(2000, seed=n_above)
    pos = 40 + 80 * np.arange(n_above + 6)
    q = np.concatenate([THRESHOLD + 0.01 + rng.random(n_above) * 0.5, THRESHOLD * (0.2 + 0.7 * rng.random(6))])
    for p, v, sg in zip(pos, q, rng.choice([-1, 1], len(pos))):
        put(s, p, sg * v)
    want, _ = check(s, clip)
    assert len(want) == (min(max(n_above, P.get_n_best), 8) if clip else max(n_above, P.get_n_best))


@pytest.mark.parametrize("clip", [False, True])
def test_tie_at_the_cut_by_count(clip):
    """5 peaks above the threshold, then equal peaks below it on both sides of position get_n_best: which of them the reference keeps
    is decided by std::sort over the full list of maxima, so no floor >= 0 may report the selection complete"""
    s = background(1500, seed=3)
    for k, v in enumerate([0.9, -0.8, 0.7, 0.6, -0.5, 0.2, -0.15]):
        put(s, 40 + 90 * k, v)
    for k in range(5):
        put(s, 700 + 90 * k, 0.1 if k % 2 else -0.1)      # positions 8 .. 12 of the sorted list: a tie across the cut
    want, _ = check(s, clip, expect_incomplete_above=0.0)
    assert len(want) == P.get_n_best


@pytest.mark.parametrize("clip", [False, True])
def test_tie_above_threshold(clip):
    """more than get_n_best peaks above the threshold with equal values: all are kept in BLOCK mode (a cut by value), and in CLIP
    mode the truncation to get_n_best cuts through the equal ones"""
    s = background(1500, seed=4)
    vals = [0.9, 0.8, 0.7, 0.6, 0.5, 0.4, 0.35, 0.3, 0.3, 0.3, 0.3]
    for k, v in enumerate(vals):
        put(s, 40 + 110 * k, v if k % 3 else -v)
    want, _ = check(s, clip)
    assert len(want) == (8 if clip else len(vals))


def test_adjacent_equal_maxima():
    """two directly adjacent scores of equal |q|: both are local maxima, the reference takes the first and skips the second"""
    s = background(600, seed=5)
    put(s, 100, 0.7)
    put(s, 101, 0.7)
    put(s, 300, -0.6)
    want, _ = check(s, False)
    idx = [w[0] for w in want]
    assert 100 * STEP in idx and 101 * STEP not in idx


@pytest.mark.parametrize("clip", [False, True])
def test_masking_distance(clip):
    """a peak is masked by an opposite-sign peak more than 3x stronger within 23 search steps: at 23 steps it is, at 24 it is not;
    a same-sign stronger peak never masks"""
    s = background(1500, seed=6)
    put(s, 100, 0.3)
    put(s, 123, -0.95)          # 23 steps: masks 100
    put(s, 400, 0.3)
    put(s, 424, -0.95)          # 24 steps: does not mask 400
    put(s, 700, -0.3)
    put(s, 710, -0.95)          # same sign: does not mask 700
    put(s, 1000, 0.3)
    put(s, 977, -0.95)          # 23 steps before: masks 1000
    want, _ = check(s, clip)
    idx = [w[0] for w in want]
    assert 100 * STEP not in idx and 1000 * STEP not in idx
    assert 400 * STEP in idx and 700 * STEP in idx


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("clip", [False, True])
def test_random_lists(seed, clip):
    """dense random spikes: maskers and masked peaks at every distance, values drawn from a short list so that ties are common"""
    rng = np.random.default_rng(1000 + seed)
    s = background(3000, seed=seed, amp=0.08)
    levels = np.array([0.1, 0.15, 0.2, 0.27, 0.3, 0.45, 0.9, 1.2])
    for p in rng.choice(3000, 60, replace=False):
        put(s, p, rng.choice([-1, 1]) * rng.choice(levels))
    check(s, clip)
