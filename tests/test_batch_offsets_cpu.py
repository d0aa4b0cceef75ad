"""CPU: input checks of the batched embed at stream offsets (hostapi.add_batch(zero_frames=...) -> awmh_add_batch with an offset
list -> awm_batch_offsets_validate).  Every malformed offset list is rejected with ValueError (rc 2 from the host export) before
any GPU work; well-formed input gets as far as the device and fails there with RuntimeError when there is none."""
import os

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

HAS_GPU = os.path.exists("/dev/nvidiactl")
X = [T.noise(0.1, 2, seed=1), T.noise(0.1, 1, seed=2)]
LIMIT = capi.MAX_STREAM_FRAMES


@pytest.mark.parametrize("items, zero_frames, rate, why", [
    ([(0, 10, 2)], [], 44100, "1 items but 0 zero_frames"),
    ([(0, 10, 2), (20, 5, 1)], [0], 44100, "2 items but 1 zero_frames"),
    ([(0, 10, 2)], [LIMIT - 9], 44100, "item 0: zero_frames %d + n_frames 10 exceeds the stream length limit" % (LIMIT - 9)),
    ([(0, 10, 2), (20, 5, 1)], [0, 2 ** 64 - 1], 44100, "item 1: zero_frames 18446744073709551615 + n_frames 5 exceeds"),
    ([(0, 0, 1)], [LIMIT + 1], 44100, "exceeds the stream length limit"),
    ([(0, 10, 2), (20, 5, 1)], [0, 1], 48000, "item 1: stream offsets are only supported at 44100 Hz"),
    ([(0, 10, 0)], [0], 44100, "channels must be >= 1"),
    ([(0, 60, 2)], [5], 44100, "extends past the end"),
])
def test_malformed_offset_lists_are_rejected(items, zero_frames, rate, why):
    assert why in capi.batch_offsets_validate(items, 100, zero_frames, rate)


def test_well_formed_offset_lists_pass():
    assert capi.batch_offsets_validate([], 0, []) == ""
    assert capi.batch_offsets_validate([(0, 10, 2), (20, 80, 1)], 100, [0, 40 * 60 * 44100]) == ""
    assert capi.batch_offsets_validate([(0, 10, 2)], 100, [LIMIT - 10]) == ""                 # exactly at the limit
    assert capi.batch_offsets_validate([(0, 10, 2), (20, 80, 1)], 100, [0, 0], 48000) == ""   # zero offsets at any rate


def test_add_batch_rejects_bad_offsets_before_gpu_work():
    with pytest.raises(ValueError, match="zero_frames"):
        H.add_batch(X, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0])                       # list of the wrong length
    with pytest.raises(ValueError, match="zero_frames"):
        H.add_batch(X, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0, -1])                   # negative
    with pytest.raises(ValueError):
        H.add_batch(X, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0, LIMIT])                # z + n past 2^48
    with pytest.raises(ValueError):
        H.add_batch(X, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0, 1024], sample_rate=48000)
    with pytest.raises(ValueError):
        H.add_batch(X, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0, 0], sample_rate=48000)  # batches are 44.1 kHz only anyway
    with pytest.raises(ValueError):
        H.add_batch(X, [T.PAYLOAD, "not hex"], zero_frames=[0, 1024])
    x16 = [np.zeros((10, 2), np.int16), np.zeros((10, 1), np.int16)]
    with pytest.raises(ValueError):
        H.add_batch(x16, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0, LIMIT])             # the 16 bit entry point checks the same way


def test_host_export_returns_2_for_malformed_offsets():
    lib = H.load()
    buf = np.zeros(100, np.float32)
    out = np.zeros_like(buf)
    pay = (H.ctypes.c_char_p * 1)(T.PAYLOAD.encode())
    it = np.array([(0, 10, 2)], capi.BATCH_ITEM)
    for z, rate in (([LIMIT], 44100), ([2 ** 64 - 1], 44100), ([1], 32000)):
        zf = np.array(z, np.uint64)
        rc = lib.awmh_add_batch(H._key(None), 0, H._ptr(buf), H._ptr(out), 0, H.ctypes.c_size_t(buf.size), H._ptr(it), H.ctypes.c_size_t(1),
                                pay, H.ctypes.c_int(rate), None, H._ptr(zf), H.ctypes.c_size_t(0), None, None)
        assert rc == 2, (z, rate)
        b16 = np.zeros(100, np.int16)
        rc = lib.awmh_add_batch(H._key(None), 0, H._ptr(b16), H._ptr(np.zeros_like(b16)), 1, H.ctypes.c_size_t(b16.size), H._ptr(it),
                                H.ctypes.c_size_t(1), pay, H.ctypes.c_int(rate), None, H._ptr(zf), H.ctypes.c_size_t(0), None, None)
        assert rc == 2, (z, rate)


@pytest.mark.skipif(HAS_GPU, reason="box has a GPU")
def test_well_formed_offsets_need_the_device():
    with pytest.raises(RuntimeError) as e:
        H.add_batch(X, [T.PAYLOAD, T.PAYLOAD], zero_frames=[0, 300 * 1024 + 517])
    assert e.type is RuntimeError
