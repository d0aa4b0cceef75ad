"""CPU: the batched embed at stream positions at any sample rate (hostapi.add_batch_rates(zero_frames=...) -> awmh_add_batch with
rate and offset lists -> awm_batch_rates_offsets_validate), and the add loop's frame counts (resampled_add_plan) that every item's
stream needs.  Malformed offset lists are rejected with ValueError (rc 2 from the host export) before any GPU work; the plan is
the old per-1024-frame loop's result, in time that does not grow with the stream."""
import os
import time

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

HAS_GPU = os.path.exists("/dev/nvidiactl")
X = [T.noise(0.1, 2, seed=1), T.noise(0.1, 1, seed=2)]
LIMIT = capi.MAX_STREAM_FRAMES
RATES = [8000, 22050, 32000, 48000, 96000, 192000]


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


@pytest.mark.parametrize("items, rates, zero_frames, why", [
    ([(0, 10, 2)], [48000], [], "1 items but 0 zero_frames"),
    ([(0, 10, 2), (20, 5, 1)], [48000, 32000], [0], "2 items but 1 zero_frames"),
    ([(0, 10, 2)], [48000], [LIMIT - 9], "item 0: zero_frames %d + n_frames 10 exceeds the stream length limit" % (LIMIT - 9)),
    ([(0, 10, 2), (20, 5, 1)], [48000, 44100], [0, 2 ** 64 - 1], "item 1: zero_frames 18446744073709551615 + n_frames 5 exceeds"),
    # at 8 kHz the stream at 44.1 kHz is 5.5 times longer: the first offset past its limit
    ([(0, 10, 2)], [8000], [LIMIT * 8000 // 44100 - 9], "at 8000 Hz exceeds the stream length limit of 2^48 frames at 44100 Hz"),
    ([(0, 10, 2)], [0], [0], "item 0: sample rate 0 must be > 0"),
    ([(0, 10, 2)], [689], [5], "outside the resampler's range"),
    ([(0, 10, 0)], [48000], [0], "channels must be >= 1"),
    ([(0, 60, 2)], [48000], [5], "extends past the end"),
])
def test_malformed_rate_offset_lists_are_rejected(items, rates, zero_frames, why):
    assert why in capi.batch_rates_offsets_validate(items, 100, rates, zero_frames)


def test_null_offset_list_is_rejected():
    it = np.array([(0, 10, 2)], capi.BATCH_ITEM)
    rates = np.array([48000], np.int32)
    err = H.ctypes.create_string_buffer(256)
    assert capi.load().awm_batch_rates_offsets_validate(capi._ptr(it), H.ctypes.c_size_t(1), H.ctypes.c_size_t(100), capi._ptr(rates), None, None,
                                                        H.ctypes.c_int(44100), err, H.ctypes.c_size_t(256)) != 0
    assert b"zero_frames list is NULL" in err.value


def test_well_formed_rate_offset_lists_pass():
    v = capi.batch_rates_offsets_validate
    assert v([], 0, [], []) == ""
    assert v([(0, 10, 2), (20, 80, 1)], 100, [48000, 44100], [0, 40 * 60 * 48000]) == ""
    assert v([(0, 10, 2)], 100, [48000], [LIMIT - 10 * 48000 // 44100 - 10]) == ""       # below the 44.1 kHz image limit
    assert v([(0, 10, 2)], 100, [44100], [LIMIT - 10]) == ""                             # exactly at the limit
    z8 = LIMIT * 8000 // 44100 - 10                                                       # (z + 10) * 44100 <= 2^48 * 8000: at the limit
    assert v([(0, 10, 2)], 100, [8000], [z8]) == ""
    assert "at 8000 Hz exceeds" in v([(0, 10, 2)], 100, [8000], [z8 + 1])
    # a 96 kHz stream is shorter at 44.1 kHz: only its own rate's limit applies
    assert v([(0, 10, 2)], 100, [96000], [LIMIT - 10]) == ""
    assert "exceeds" in v([(0, 10, 2)], 100, [96000], [LIMIT - 9])


def test_add_batch_rates_rejects_bad_offsets_before_gpu_work():
    with pytest.raises(ValueError, match="zero_frames"):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 32000], zero_frames=[0])          # list of the wrong length
    with pytest.raises(ValueError, match="zero_frames"):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 32000], zero_frames=[0, -1])      # negative
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 32000], zero_frames=[0, LIMIT])   # z + n past 2^48
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 8000], zero_frames=[0, LIMIT // 5])   # its 44.1 kHz image past 2^48
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, "not hex"], [48000, 32000], zero_frames=[0, 1024])
    x16 = [np.zeros((10, 2), np.int16), np.zeros((10, 1), np.int16)]
    with pytest.raises(ValueError):
        H.add_batch_rates(x16, [T.PAYLOAD, T.PAYLOAD], [48000, 32000], zero_frames=[0, LIMIT])


def test_host_export_returns_2_for_malformed_rate_offsets():
    lib = H.load()
    buf = np.zeros(100, np.float32)
    pay = (H.ctypes.c_char_p * 1)(T.PAYLOAD.encode())
    it = np.array([(0, 10, 2)], capi.BATCH_ITEM)
    for z, rate in (([LIMIT], 48000), ([2 ** 64 - 1], 44100), ([LIMIT // 5], 8000)):
        zf = np.array(z, np.uint64)
        rates = np.array([rate], np.int32)
        rc = lib.awmh_add_batch(H._key(None), 0, H._ptr(buf), H._ptr(np.zeros_like(buf)), 0, H.ctypes.c_size_t(buf.size), H._ptr(it),
                                H.ctypes.c_size_t(1), pay, 44100, H._ptr(rates), H._ptr(zf), H.ctypes.c_size_t(0), None, None)
        assert rc == 2, (z, rate)
        b16 = np.zeros(100, np.int16)
        rc = lib.awmh_add_batch(H._key(None), 0, H._ptr(b16), H._ptr(np.zeros_like(b16)), 1, H.ctypes.c_size_t(b16.size), H._ptr(it),
                                H.ctypes.c_size_t(1), pay, 44100, H._ptr(rates), H._ptr(zf), H.ctypes.c_size_t(0), None, None)
        assert rc == 2, (z, rate)


@pytest.mark.skipif(HAS_GPU, reason="box has a GPU")
def test_well_formed_rate_offsets_need_the_device():
    with pytest.raises(RuntimeError) as e:
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 32000], zero_frames=[0, 300 * 1024 + 517])
    assert e.type is RuntimeError


# ---- resampled_add_plan: the add loop's (n_emit, WatermarkGen::run calls) for a stream of n frames at another rate

class OldLoop:
    """the per-1024-frame loop resampled_add_plan used to run (src/wmadd.cc:520-589 with a WatermarkResampler), restated; the state
    after each iteration does not depend on n, so it is computed once per iteration number and shared by every n"""

    def __init__(self, rate, limiter):
        self.r_in, self.r_out = 44100 / rate, rate / 44100
        self.block = rate            # limiter block: 1000 ms
        self.limiter = limiter
        self.states = [None]

    def state(self, iteration):
        while len(self.states) <= iteration:
            k = len(self.states)
            runs = H.resample_stream_available(1024 * k, self.r_in) // 1024
            emit = H.resample_stream_available(runs * 1024, self.r_out) if runs else 0
            released = emit
            if self.limiter:
                released = (emit // self.block - 1) * self.block if emit // self.block >= 2 else 0
            self.states.append((emit, runs, released))
        return self.states[iteration]

    def plan(self, n):
        total_in = total_out = 0
        n_emit = runs = 0
        iteration = 1
        while True:
            real = min(1024, n - total_in)
            total_in += real
            if real < 1024 and total_in == total_out:
                return n_emit, runs
            n_emit, runs, released = self.state(iteration)
            total_out = min(released, total_in)
            iteration += 1


@pytest.mark.parametrize("limiter", [True, False], ids=["limiter", "no_limiter"])
@pytest.mark.parametrize("rate", RATES)
def test_plan_equals_the_old_loop(rate, limiter):
    H.set_params(test_no_limiter=not limiter)
    old = OldLoop(rate, limiter)
    ns = list(range(0, 300_000, 97)) + [300_000, 1_000_000, 3 * 1024 * 1024 + 1, 10 * 60 * rate + 333]
    for n in ns:
        assert H.resampled_add_plan(n, rate) == old.plan(n), (rate, limiter, n)


def test_plan_at_a_24_hour_offset_is_fast():
    z = 24 * 3600 * 48000
    t0 = time.perf_counter()
    plans = [H.resampled_add_plan(z + 12 * 48000 + i, 48000) for i in range(1024)]
    dt = time.perf_counter() - t0
    assert dt < 0.5, dt
    emit, runs = plans[0]
    n = z + 12 * 48000
    assert n <= emit < n + 3 * 48000 and runs * 1024 >= n * 44100 // 48000
