"""CPU: input checks of the batched embed at any sample rate (hostapi.add_batch_rates -> awmh_add_batch with a rate list ->
awm_batch_rates_validate).  Every malformed call is rejected with ValueError before any GPU work; well-formed input gets as far as
the device and fails there with RuntimeError when there is none."""
import os

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

HAS_GPU = os.path.exists("/dev/nvidiactl")
X = [T.noise(0.1, 2, seed=1), T.noise(0.1, 1, seed=2)]


@pytest.mark.parametrize("items, rates, n_emit, why", [
    ([(0, 10, 2)], [0], None, "item 0: sample rate 0 must be > 0"),
    ([(0, 10, 2), (20, 5, 1)], [48000, -1], None, "item 1: sample rate -1 must be > 0"),
    ([(0, 10, 2)], [689], None, "outside the resampler's range"),               # 44100 / 689 > 64
    ([(0, 10, 2)], [44100 * 64], None, "outside the resampler's range"),
    ([(0, 10, 2)], [48000], [9], "item 0: n_emit 9 is less than n_frames 10"),
    ([(0, 10, 0)], [48000], None, "channels must be >= 1"),
    ([(0, 60, 2)], [48000], None, "extends past the end"),
])
def test_malformed_rate_batches_are_rejected(items, rates, n_emit, why):
    assert why in capi.batch_rates_validate(items, 100, rates, n_emit)


def test_well_formed_rate_batches_pass():
    assert capi.batch_rates_validate([], 0, []) == ""
    assert capi.batch_rates_validate([(0, 10, 2), (20, 80, 1)], 100, [690, 44100 * 64 - 1]) == ""
    assert capi.batch_rates_validate([(0, 10, 2), (20, 80, 1)], 100, [44100, 48000], [0, 80]) == ""   # n_emit is ignored at 44.1 kHz
    assert "256 per call" in capi.batch_rates_validate([(0, 0, 1)] * 300, 0, list(range(8000, 8300)))


def test_add_batch_rates_rejects_bad_input_before_gpu_work():
    with pytest.raises(ValueError, match="sample rates"):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000])               # rate list of the wrong length
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 0])             # rate <= 0
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, -32000])
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 600])           # outside the resampler's ratio range
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 44100 * 64])
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD], [48000, 48000])                    # one payload for two items
    with pytest.raises(ValueError):
        H.add_batch_rates(X, [T.PAYLOAD, "not hex"], [48000, 32000])         # bad payload
    x16 = [np.zeros((10, 2), np.int16), np.zeros((10, 1), np.int16)]
    with pytest.raises(ValueError):
        H.add_batch_rates(x16, [T.PAYLOAD, T.PAYLOAD], [48000, 5])           # the 16 bit entry point checks the same way


def test_host_export_returns_2_for_malformed_rate_items():
    lib = H.load()
    buf = np.zeros(100, np.float32)
    out = np.zeros_like(buf)
    pay = (H.ctypes.c_char_p * 1)(T.PAYLOAD.encode())
    rates = np.array([48000], np.int32)
    for items in ([(0, 10, 0)], [(0, 60, 2)], [(101, 0, 1)]):
        it = np.array(items, capi.BATCH_ITEM)
        rc = lib.awmh_add_batch(H._key(None), 0, H._ptr(buf), H._ptr(out), 0, H.ctypes.c_size_t(buf.size), H._ptr(it), H.ctypes.c_size_t(1),
                                pay, 44100, H._ptr(rates), None, H.ctypes.c_size_t(0), None, None)
        assert rc == 2, items


@pytest.mark.skipif(HAS_GPU, reason="box has a GPU")
def test_well_formed_input_needs_the_device():
    with pytest.raises(RuntimeError) as e:
        H.add_batch_rates(X, [T.PAYLOAD, T.PAYLOAD], [48000, 44100])
    assert e.type is RuntimeError
