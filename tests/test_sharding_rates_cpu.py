"""CPU: the plan of the sharded get at sample rates other than 44.1 kHz.  The driver resamples the stream to the watermark rate
first, as the single GPU get does, and plans there; a rank holds only the input frames the resampler taps of its slices read.  The
C++ plan functions must equal their Python restatement (sharding.py), the taps of every output a rank searches must lie inside its
input range, and the range resampler's validator must refuse what the kernel cannot honour without a device."""
import math

import numpy as np
import pytest

from audiowmark_b200 import capi as C, hostapi as H, sharding as S

RATES = (22050, 32000, 48000, 96000)
WORLDS = (1, 2, 3, 4, 8)
MARK = 44100
GUARD = 1                      # frames balanced_input_range adds on each side of the exact taps


def _lengths(rate):
    """ragged stream lengths at `rate`: 0.3 h (one chunk), 1 h (three chunks), 1.37 h and 2 h plus an odd number of frames"""
    return [int(h * 3600 * rate) + extra for h, extra in ((0.3, 0), (1.0, 0), (1.37, 517), (2.0, 1023))]


def _resampler(rate):
    ratio = MARK / rate
    h = int(math.ceil(16 / min(ratio, 1.0)))
    return ratio, h, 1.0 / ratio


@pytest.mark.parametrize("rate", RATES)
def test_plan_is_the_plan_of_the_watermark_rate_stream(rate):
    """chunks and slices of balanced_plan at rate r are chunk_plan / rank_slices of the resampled stream's n_mark frames, and
    balanced_owner / balanced_input_range equal index_owners / rank_input_range, for every world size and ragged lengths"""
    H.set_params()
    mx, ov = H.chunk_geometry(MARK)
    rng = np.random.default_rng(rate)
    for n_total in _lengths(rate):
        ratio, _, _ = _resampler(rate)
        n_mark = H.resample_stream_frames(n_total, ratio)
        assert abs(n_mark - n_total * ratio) < 64
        plan = S.chunk_plan(n_mark, mx, ov)
        for world in WORLDS:
            for r in range(world):
                chunks, slices = H.balanced_plan(n_total, r, world, sample_rate=rate)
                assert [(a, b) for a, b, _ in chunks] == [(a, b) for a, b, _ in plan]
                assert np.allclose([t for _, _, t in chunks], [t for _, _, t in plan], rtol=0, atol=1e-9)
                mine = S.rank_slices(plan, r, world, n_mark)
                assert slices == [(sl.chunk, sl.sa, sl.sb, sl.a, sl.b, sl.lo, sl.hi) for sl in mine], (rate, n_total, world, r)
                assert H.balanced_input_range(n_total, r, world, rate) == S.rank_input_range(mine, n_total, rate), (rate, n_total, world, r)
            for c, (cs, cn, _) in enumerate(plan):
                idx = rng.integers(0, cn, 16)
                own = S.index_owners(plan, n_mark, world, c, idx)
                assert [H.balanced_owner(n_total, world, c, int(i), sample_rate=rate) for i in idx] == [int(o) for o in own]


@pytest.mark.parametrize("rate", RATES)
def test_input_range_holds_every_tap_of_the_rank(rate):
    """every tap of every watermark-rate frame in a rank's slices, c(n) - 2h + 2 .. c(n) + 1 with c(n) = floor((h - 1) + n step) in
    float64 over all outputs, lies in the rank's input range (clamped to the stream); the range is no wider than those taps plus
    one guard frame on each side"""
    H.set_params()
    ratio, h, step = _resampler(rate)
    for n_total in (int(0.3 * 3600 * rate), int(0.75 * 3600 * rate) + 517):          # one chunk; two chunks, ragged
        for world in (1, 3, 8):
            for r in range(world):
                _, slices = H.balanced_plan(n_total, r, world, sample_rate=rate)
                first, end = H.balanced_input_range(n_total, r, world, rate)
                if not slices:
                    assert (first, end) == (0, 0)
                    continue
                lo, hi = min(s[5] for s in slices), max(s[6] for s in slices)
                n = np.arange(lo, hi, dtype=np.float64)
                c = np.floor(np.float64(h - 1) + n * np.float64(step)).astype(np.int64)
                t0 = max(int(c.min()) - 2 * h + 2, 0)
                t1 = min(int(c.max()) + 2, n_total)
                assert np.all(np.diff(c) >= 0)
                for chunk, sa, sb, a, b, slo, shi in slices:              # each slice's taps, not only the union's
                    cs = c[slo - lo:shi - lo]
                    assert max(int(cs.min()) - 2 * h + 2, 0) >= first and min(int(cs.max()) + 2, n_total) <= end
                assert first <= t0 and end >= t1
                assert t0 - first <= GUARD and end - t1 <= GUARD, (rate, n_total, world, r, first, end, t0, t1)
                assert C.resample_taps(n_total, ratio, lo, hi - lo) == (t0, t1)


def test_input_range_at_44100_is_the_union_of_the_slices():
    H.set_params()
    for n_total in (int(0.3 * 3600 * MARK), 158760000, int(1.37 * 3600 * MARK) + 517):
        for world in WORLDS:
            for r in range(world):
                _, slices = H.balanced_plan(n_total, r, world)
                want = (min(s[5] for s in slices), max(s[6] for s in slices)) if slices else (0, 0)
                assert H.balanced_input_range(n_total, r, world, MARK) == want


def test_plan_refuses_rates_outside_the_resampler_range():
    H.set_params()
    n = 3600 * 48000
    for rate in (600, 689, 44100 * 64, 0, -48000):
        with pytest.raises(ValueError):
            H.balanced_plan(n, 0, 2, sample_rate=rate)
        with pytest.raises(ValueError):
            H.balanced_input_range(n, 0, 2, rate)
        with pytest.raises(ValueError):
            H.balanced_owner(n, 2, 0, 0, sample_rate=rate)
    assert H.balanced_plan(n, 0, 2, sample_rate=690)[0]          # 44100 / 690 < 64


def test_range_resampler_validator_refuses_bad_arguments():
    """awm_resample_range_validate needs no device; every refusal names its reason"""
    n, ratio = 480000, MARK / 48000
    n_out = H.resample_stream_frames(n, ratio)
    t0, t1 = C.resample_taps(n, ratio, 100000, 5000)
    assert 0 < t0 < t1 < n
    ok = dict(in_first=t0, in_frames=t1 - t0, n_in_total=n, channels=2, ratio=ratio, out_first=100000, out_frames=5000)
    assert C.resample_range_validate(**ok) == ""
    assert C.resample_range_validate(**dict(ok, in_first=t0 + 1, in_frames=t1 - t0 - 1))          # misses the first tap
    assert C.resample_range_validate(**dict(ok, in_frames=t1 - t0 - 1))                           # misses the last tap
    assert "ratio" in C.resample_range_validate(**dict(ok, ratio=64.0))
    assert "ratio" in C.resample_range_validate(**dict(ok, ratio=1.0 / 64))
    assert "ratio" in C.resample_range_validate(**dict(ok, hlen=7))
    assert "channels" in C.resample_range_validate(**dict(ok, channels=0))
    assert "channels" in C.resample_range_validate(**dict(ok, channels=-2))
    # outputs up to the resampled stream's end are fine (the last ones read zeros past the input), one more is refused
    end_taps = C.resample_taps(n, ratio, n_out - 10, 10)
    assert C.resample_range_validate(end_taps[0], end_taps[1] - end_taps[0], n, 2, ratio, n_out - 10, 10) == ""
    assert "past" in C.resample_range_validate(end_taps[0], n - end_taps[0], n, 2, ratio, n_out - 10, 11)
    # outputs at the start read taps below frame 0 as zero: a window from frame 0 suffices
    s0, s1 = C.resample_taps(n, ratio, 0, 50)
    assert s0 == 0 and C.resample_range_validate(0, s1, n, 1, ratio, 0, 50) == ""
    assert C.resample_range_validate(1, s1, n, 1, ratio, 0, 50)
    assert C.resample_range_validate(0, 0, n, 1, ratio, 0, 0) == ""                               # nothing asked, nothing read
    assert "2^48" in C.resample_range_validate(0, n, 1 << 49, 1, ratio, 0, 10)
