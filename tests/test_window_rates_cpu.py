"""CPU: the window planner of streaming and sharded `add` at other sample rates (awm_window_range_rates, hostapi.window_range) and
the refusals of the window entry points that need no device.  The planner's range must contain every input frame the owned
outputs depend on, as computed here from the resamplers' taps (capi.resample_taps), and exceed it by at most the one frame of
margin on each side."""
import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

N = 1024
MARK = 44100
FAR = capi.MAX_STREAM_FRAMES * 64
UNKNOWN = (1 << 64) - 1
RATES = [8000, 22050, 32000, 48000, 96000]


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def dependency_range(own_first, own_end, rate):
    """input frames the outputs [own_first, own_end) read: limiter blocks before / of / after them, the out-resampler's taps into the
    watermark, one 1024-frame of synthesis window on each side, the in-resampler's taps into the input"""
    L = rate                                          # 1000 ms limiter blocks
    b0, b1 = own_first // L, (own_end - 1) // L
    m0, m1 = max(b0 - 1, 0) * L, (b1 + 2) * L
    w0, w1 = capi.resample_taps(FAR, rate / MARK, m0, m1 - m0)
    x0, x1 = max(w0 // N - 1, 0) * N, ((w1 - 1) // N + 2) * N
    e0, e1 = capi.resample_taps(FAR, MARK / rate, x0, x1 - x0)
    return min(e0, m0), max(e1, m1)


def owned_ranges(rate, n_total):
    L = rate
    cuts = [(0, 1), (1, 2), (0, 1000), (1023, 1025), (1024, 2048), (1025, 5000), (L - 1, L), (L, L + 1), (L - 1, L + 1), (L + 1, 3 * L),
            (2 * L - 1, 2 * L + N), (5 * L + 333, 5 * L + 334), (3 * L + 17, 7 * L - 5)]
    cuts += [(n_total - 1, n_total), (n_total - 5 * N, n_total), (n_total - L - 1, n_total - L + 1)]
    return [(a, b) for a, b in cuts if 0 <= a < b <= n_total]


@pytest.mark.parametrize("rate", RATES)
@pytest.mark.parametrize("known", [True, False])
def test_planner_contains_the_dependency_range(rate, known):
    n_total = 10 * rate + 777
    for own in owned_ranges(rate, n_total):
        total = n_total if known else UNKNOWN
        e0, e1 = capi.window_range_rates(own[0], own[1], total, rate)
        lo, hi = dependency_range(own[0], own[1], rate)
        lo, hi = max(lo, 0), min(hi, total)
        assert e0 <= own[0] and own[1] <= e1, (own, e0, e1)
        assert 0 <= e0 and e1 <= total
        assert e0 <= lo and hi <= e1, (own, (e0, e1), (lo, hi))
        assert lo - e0 <= 1 and e1 - hi <= 1, (own, (e0, e1), (lo, hi))      # the smallest range, plus one frame of margin
        assert H.window_range(own[0], own[1], total, sample_rate=rate) == (e0, e1)


def test_planner_is_clamped_to_the_stream_and_known_ends_only_shorten_it():
    for rate in RATES:
        n_total = 3 * rate + 5
        assert capi.window_range_rates(0, n_total, n_total, rate) == (0, n_total)
        for own in owned_ranges(rate, n_total):
            k0, k1 = capi.window_range_rates(own[0], own[1], n_total, rate)
            u0, u1 = capi.window_range_rates(own[0], own[1], UNKNOWN, rate)
            assert k0 == u0 and k1 == min(u1, n_total)


def test_planner_refusals():
    with pytest.raises(ValueError):
        capi.window_range_rates(5, 5, 100, 48000)                 # empty
    with pytest.raises(ValueError):
        capi.window_range_rates(5, 101, 100, 48000)               # past the end
    with pytest.raises(ValueError):
        capi.window_range_rates(0, 10, 100, 689)                  # outside the resampler's range
    with pytest.raises(ValueError):
        capi.window_range_rates(0, 10, 100, 48000, limiter_ms=0)
    with pytest.raises(ValueError):
        capi.window_range_rates(0, 10, 100, 48000, hlen=4)
    with pytest.raises(ValueError):
        H.window_range(10, 5, 100, sample_rate=48000)


def test_window_range_at_the_watermark_rate_is_1024_aligned():
    for own in [(0, 1), (1, 2), (12345, 67890), (44100, 44101), (3 * 44100 - 1, 4 * 44100 + 1)]:
        e0, e1 = H.window_range(own[0], own[1], UNKNOWN)
        assert e0 % N == 0 and e0 <= own[0] and own[1] <= e1
        k0, k1 = H.window_range(own[0], own[1], 200000)
        assert (k0, k1) == (e0, min(e1, 200000))


def test_one_item_validator_refuses_what_the_window_call_refuses():
    v = capi.batch_rates_offsets_validate
    assert v([(0, 100, 2)], 200, [48000], [5], n_emit=[100]) == ""
    assert "n_emit 99 is less than n_frames 100" in v([(0, 100, 2)], 200, [48000], [5], n_emit=[99])
    assert "exceeds the stream length limit" in v([(0, 100, 2)], 200, [48000], [capi.MAX_STREAM_FRAMES], n_emit=[100])


def test_add_window_refuses_a_buffer_that_misses_the_window_before_gpu_work():
    rate = 48000
    x = np.zeros((4 * rate, 1), np.float32)
    e0, e1 = H.window_range(2 * rate, 2 * rate + 10, 10 * rate, sample_rate=rate)
    with pytest.raises(ValueError, match="does not cover"):
        H.add_window(x[e0 + 1 - e0:], T.PAYLOAD, e0 + 1, 10 * rate, 2 * rate, 2 * rate + 10, sample_rate=rate)
    with pytest.raises(ValueError, match="does not cover"):
        H.add_window(x[:e1 - e0 - 1], T.PAYLOAD, e0, 10 * rate, 2 * rate, 2 * rate + 10, sample_rate=rate)
    with pytest.raises(ValueError):
        H.add_window(x, T.PAYLOAD, 0, 10 * rate, 5, 5, sample_rate=rate)           # empty owned range
