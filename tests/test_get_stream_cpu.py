"""CPU: the chunk decisions of the streaming `get` (GetStream, host/awm_get.cc) against the reference's WavChunkLoader as the oracle
restates it (awm_oracle.chunk_ranges): the walker is driven without a device, piece by piece, with EOF at and near piece and chunk
boundaries, at 44.1 kHz and at rates it resamples; and the range resampler calls it makes are ones awm_resample_range accepts."""
import numpy as np
import pytest

import awm_oracle as O
from audiowmark_b200 import capi as C, hostapi as H

MARK = 44100


@pytest.fixture
def three_minute_chunks():
    H.set_params(chunk_size_min=3.0)
    P = O.Params()
    P.get_chunk_size = 3.0
    yield P
    H.set_params()


def _lengths(mx, ov, piece):
    """clip sized, around one chunk, around the first chunk plus k strides, and EOF at and next to piece boundaries"""
    step = mx - ov
    out = {0, 1, 2 * 44100, mx - 1, mx, mx + 1, mx + step - 1, mx + step, mx + step + 1, mx + 3 * step + 12345}
    for k in (1, 7, (mx + 2 * step) // piece):
        out |= {k * piece - 1, k * piece, k * piece + 1}
    return sorted(v for v in out if v >= 0)


@pytest.mark.parametrize("piece", [1, 4095, 1 << 20])
def test_chunks_follow_wavchunkloader_at_44k(three_minute_chunks, piece):
    P = three_minute_chunks
    mx, ov = H.chunk_geometry(MARK)
    lengths = _lengths(mx, ov, piece) if piece > 1 else [0, 1, 4095, mx - 1, mx, mx + 1]
    for n in lengths:
        got, mark = H.get_stream_plan(n, piece)
        want = O.chunk_ranges(n, P)
        assert mark == n
        assert [(a, b) for a, b, _ in got] == [(a, b) for a, b, _ in want], (n, piece)
        assert [t for *_, t in got] == [t for *_, t in want], (n, piece)      # the same sum of the same doubles
    # a stream that exactly fills a chunk gives one more, overlap-only chunk; an empty one none
    assert H.get_stream_plan(mx, 4095)[0][-1][:2] == (mx - ov, ov)
    assert H.get_stream_plan(0, 4095)[0] == []


@pytest.mark.parametrize("rate", [22050, 32000, 48000, 96000, 8000])
@pytest.mark.parametrize("piece", [4095, 1 << 20])
def test_chunks_at_other_rates_are_those_of_the_resampled_stream(three_minute_chunks, rate, piece):
    """at other rates the chunks are WavChunkLoader's over the resampled stream of resample_stream_frames (n) frames"""
    P = three_minute_chunks
    mx, ov = H.chunk_geometry(MARK)
    ratio = MARK / rate
    for m in (0, 1, 3 * 44100, mx - 1, mx, mx + 1, mx + 4 * (mx - ov) + 777):
        n = int(m / ratio)
        while H.resample_stream_frames(n, ratio) < m:
            n += 1
        for n_in in {n, n + 1, max(n - 1, 0), (n // piece) * piece}:
            got, mark = H.get_stream_plan(n_in, piece, rate)
            assert mark == H.resample_stream_frames(n_in, ratio)
            want = O.chunk_ranges(mark, P)
            assert [(a, b, t) for a, b, t in got] == [(a, b, t) for a, b, t in want], (rate, n_in, piece)


def test_refused_rates_and_channels():
    for rate in (0, -48000, 500, 44100 * 64):
        with pytest.raises(ValueError):
            H.get_stream_plan(1000, 100, rate)
        with pytest.raises(ValueError):
            H.GetStream(sample_rate=rate)
    with pytest.raises(ValueError):
        H.GetStream(channels=0)


@pytest.mark.parametrize("rate", [22050, 32000, 48000, 96000, 8000])
def test_outputs_below_the_available_count_need_only_the_fed_input(rate):
    """an output below resample_stream_available (fed) reads only frames below fed, so awm_resample_range accepts it with
    n_in_total = fed from a window that ends at fed -- the call the walker makes before the stream's end is known"""
    ratio = MARK / rate
    for fed in (1, 2, 40, 41, 4095, 100003, 1 << 20):
        avail = H.resample_stream_available(fed, ratio)
        if avail == 0:
            continue
        t0, t1 = C.resample_taps(fed, ratio, 0, avail)
        assert t1 <= fed
        for total in (fed, fed + 1, fed + 100000):
            assert C.resample_taps(total, ratio, avail - 1, 1)[1] <= fed
            assert C.resample_range_validate(t0, fed - t0, total, 2, ratio, 0, avail) == "", (rate, fed, total)
        # the next output reads frame fed - 1 or later: the window keeps at most 2h frames of input between launches
        h = int(np.ceil(16 / min(1.0, ratio)))
        assert C.resample_taps(fed, ratio, avail, 1)[0] >= fed - 2 * h
