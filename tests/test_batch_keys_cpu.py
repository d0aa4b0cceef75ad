"""CPU: the batched embed with a key per item (hostapi.add_batch / add_batch_rates with keys= -> awmh_add_batch with per-item
keys -> awm_batch_keys_validate).  The validator accepts what the matching single-key validator accepts and, in addition, needs a
key index below the role set's key count for every item; malformed calls are rejected with ValueError before any GPU work."""
import ctypes

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

X = [T.noise(0.1, 2, seed=1), T.noise(0.1, 1, seed=2)]
PAY = ["0123456789abcdef0123456789abcdef", "fedcba9876543210fedcba9876543210"]
K = [bytes(range(16)), bytes(range(16, 32))]


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def _validate_raw(items, n_values, key_index, n_keys):
    it = np.array(items, capi.BATCH_ITEM)
    ki = None if key_index is None else np.array(key_index, np.uint32)
    err = ctypes.create_string_buffer(256)
    rc = capi.load().awm_batch_keys_validate(capi._ptr(it), ctypes.c_size_t(len(it)), ctypes.c_size_t(n_values), None, None, None, capi._ptr(ki),
                                             ctypes.c_size_t(n_keys), ctypes.c_int(44100), err, ctypes.c_size_t(256))
    return rc, err.value.decode()


def test_valid_calls_pass():
    items = [(0, 10, 2), (20, 5, 1)]
    assert capi.batch_keys_validate(items, 100, [1, 0], 2) == ""
    assert capi.batch_keys_validate(items, 100, [0, 0], 1, zero_frames=[0, 1 << 40]) == ""
    assert capi.batch_keys_validate(items, 100, [1, 1], 3, sample_rates=[48000, 44100], zero_frames=[5, 0]) == ""
    assert capi.batch_keys_validate(items, 100, [0, 2], 3, sample_rates=[32000, 96000]) == ""
    assert capi.batch_keys_validate([], 0, [], 0) == ""                    # no items need no keys


@pytest.mark.parametrize("key_index, n_keys, why", [
    ([0, 2], 2, "batch item 1: key index 2 is out of range (2 keys)"),
    ([7, 0], 3, "batch item 0: key index 7 is out of range (3 keys)"),
    ([0xFFFFFFFF, 0], 5, "batch item 0: key index 4294967295 is out of range (5 keys)"),
    ([0, 0], 0, "the role set has no keys"),
])
def test_key_index_out_of_range_is_rejected(key_index, n_keys, why):
    assert why in capi.batch_keys_validate([(0, 10, 2), (20, 5, 1)], 100, key_index, n_keys)


def test_null_key_index_list_is_rejected():
    rc, why = _validate_raw([(0, 10, 2)], 100, None, 1)
    assert rc != 0 and "key index list is NULL" in why
    assert _validate_raw([], 0, None, 0)[0] == 0                                 # nothing to index


@pytest.mark.parametrize("items, kw, why", [
    ([(0, 10, 0)], {}, "channels must be >= 1"),
    ([(0, 60, 2)], {}, "extends past the end"),
    ([(0, 10, 2)], {"zero_frames": [capi.MAX_STREAM_FRAMES - 9]}, "exceeds the stream length limit"),
    ([(0, 10, 2)], {"sample_rates": [0]}, "item 0: sample rate 0 must be > 0"),
    ([(0, 10, 2)], {"sample_rates": [689]}, "outside the resampler's range"),
    ([(0, 10, 2)], {"sample_rates": [8000], "zero_frames": [capi.MAX_STREAM_FRAMES * 8000 // 44100 - 9]},
     "at 8000 Hz exceeds the stream length limit of 2^48 frames at 44100 Hz"),
    ([(0, 10, 2)], {"sample_rates": [48000], "n_emit": [9]}, "n_emit 9 is less than n_frames 10"),
])
def test_what_the_single_key_validators_reject_is_rejected(items, kw, why):
    assert why in capi.batch_keys_validate(items, 100, [0] * len(items), 1, **kw)


def test_single_key_validators_agree_on_valid_and_invalid_lists():
    cases = [([(0, 10, 2), (20, 5, 1)], 100), ([(0, 10, 2), (20, 50, 1)], 60), ([(0, 10, 2), (10, 5, 3)], 25)]
    for items, n in cases:
        single = capi.batch_validate(items, n)
        assert capi.batch_keys_validate(items, n, [0] * len(items), 1) == single
        rates = [48000] * len(items)
        assert capi.batch_keys_validate(items, n, [0] * len(items), 1, sample_rates=rates) == capi.batch_rates_validate(items, n, rates)


def test_key_and_keys_together_raise():
    with pytest.raises(ValueError, match="either key= or keys="):
        H.add_batch(X, PAY, key=K[0], keys=K)
    with pytest.raises(ValueError, match="either key= or keys="):
        H.add_batch_rates(X, PAY, [48000, 44100], key=K[0], keys=K)


@pytest.mark.parametrize("keys, why", [
    ([K[0]], "2 items but 1 keys"),
    (K + [K[0]], "2 items but 3 keys"),
    ([K[0], b"short"], "every key must be 16 bytes"),
    ([K[0], bytes(17)], "every key must be 16 bytes"),
])
def test_wrong_keys_raise(keys, why):
    with pytest.raises(ValueError, match=why):
        H.add_batch(X, PAY, keys=keys)
    with pytest.raises(ValueError, match=why):
        H.add_batch_rates(X, PAY, [48000, 44100], keys=keys)
    with pytest.raises(ValueError, match=why):
        H.add_batch(X, PAY, keys=keys, zero_frames=[0, 5])


def test_malformed_calls_with_keys_are_rejected_before_gpu_work():
    with pytest.raises(ValueError):
        H.add_batch(X, ["xyz", PAY[1]], keys=K)                                  # payload does not parse
    with pytest.raises(ValueError):
        H.add_batch_rates(X, PAY, [48000, 689], keys=K)                          # rate outside the resampler's range
    with pytest.raises(ValueError):
        H.add_batch(X, PAY, keys=K, zero_frames=[0, capi.MAX_STREAM_FRAMES])     # stream too long
    with pytest.raises(ValueError):
        H.add_batch(X, PAY, keys=K, sample_rate=48000)                           # add_batch is 44.1 kHz only
