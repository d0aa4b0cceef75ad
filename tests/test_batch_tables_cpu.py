"""CPU: the tables of the batched embed.  The FrameMod table of a (key, payload) is a key-only role table combined with the
payload's coded bits; rebuilt here from the role codes as include/awm_b200.h defines them, it must equal the single-payload
table byte for byte (and the oracle's) for every key, payload layout and mode.  Malformed batches are rejected before any
GPU work."""
import os

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

KEYS = [O.Key(), O.Key.test_key(1), O.Key(bytes(range(16)), "k")]
# (frames_per_bit, mix, short payload bits)
CONFIGS = [(2, True, 0), (3, True, 0), (2, False, 0), (3, False, 0), (2, True, 12), (2, True, 16), (2, True, 20)]
HAS_GPU = os.path.exists("/dev/nvidiactl")


def rebuild_frame_mod(roles, coded):
    """FrameMod [2][fpb][101] from role codes and coded bits [2][n_coded] (0 keep, 1 up, 2 down)"""
    mark = (roles & 1) != 0
    down = (roles & 2) != 0
    sync = (roles & 4) != 0
    index = (roles >> 3).astype(np.int64)
    out = np.zeros((2,) + roles.shape, np.uint8)
    for ab in (0, 1):
        data_bit = coded[ab][np.where(mark & ~sync, index, 0)].astype(bool)
        bit = np.where(sync, ((index + ab) & 1).astype(bool), data_bit)
        out[ab] = np.where(mark, np.where(bit ^ down, 1, 2), 0)
    return out


def random_payload(rng, bits):
    return "".join("%x" % v for v in rng.integers(0, 16, (bits or 128) // 4))


@pytest.fixture
def config(request):
    fpbit, mix, short = request.param
    H.set_params(frames_per_bit=fpbit, mix=mix)
    H.set_short_payload(short)
    yield fpbit, mix, short
    H.set_short_payload(0)
    H.set_params()


@pytest.mark.parametrize("config", CONFIGS, indirect=True, ids=lambda c: "fpbit%d_%s_short%d" % (c[0], "mix" if c[1] else "linear", c[2]))
@pytest.mark.parametrize("ki", range(len(KEYS)))
def test_roles_times_coded_bits_is_the_frame_mod_table(config, ki):
    fpbit, mix, short = config
    key = KEYS[ki]
    roles = H.embed_roles(key.aes_key)
    n_coded = H.n_coded_bits()
    assert roles.shape == (H.frames_per_block(), 101)
    # every data bit sits on frames_per_bit frames x 30 bands x (up + down), every sync bit on 85 frames x 60 bands
    mark = (roles & 1) != 0
    assert not mark[:, :20].any()
    idx, sync = roles >> 3, (roles & 4) != 0
    assert np.array_equal(np.bincount(idx[mark & ~sync], minlength=n_coded), np.full(n_coded, fpbit * 60))
    assert np.array_equal(np.bincount(idx[mark & sync], minlength=6), np.full(6, 85 * 60))
    rng = np.random.default_rng(100 + ki)
    payloads = [random_payload(rng, short) for _ in range(3)]
    if not short:
        payloads += ["0" * 32, "f" * 32]
    for payload in payloads:
        coded = H.coded_bits(key.aes_key, payload)
        assert coded.shape == (2, n_coded)
        got = rebuild_frame_mod(roles, coded)
        assert got.tobytes() == H.frame_mod(key.aes_key, payload).tobytes(), payload
    P = O.Params(frames_per_bit=fpbit, mix=mix, payload_size=short or 128, payload_short=bool(short))
    assert rebuild_frame_mod(roles, H.coded_bits(key.aes_key, payloads[0])).tobytes() == T.frame_mod_ab(key, payloads[0], P).tobytes()


def test_coded_bits_follow_the_payload():
    H.set_params()
    a = H.coded_bits(bytes(16), T.PAYLOAD)
    b = H.coded_bits(bytes(16), "1" + T.PAYLOAD[1:])
    assert a.shape == b.shape == (2, 858) and set(np.unique(a)) <= {0, 1}
    assert not np.array_equal(a, b)
    assert not np.array_equal(a, H.coded_bits(O.Key.test_key(1).aes_key, T.PAYLOAD))    # the bit order is keyed


@pytest.mark.parametrize("items, n_values, why", [
    ([(0, 10, 0)], 100, "channels must be >= 1"),
    ([(0, 10, -2)], 100, "channels must be >= 1"),
    ([(0, 10, 2), (90, 6, 2)], 100, "item 1: extends past the end"),
    ([(101, 0, 1)], 100, "extends past the end"),
    ([(0, 1 << 62, 4)], 100, "extends past the end"),             # n_frames * channels overflows 64 bits
    ([(1 << 63, 1, 1)], 100, "extends past the end"),
])
def test_malformed_item_lists_are_rejected(items, n_values, why):
    assert why in capi.batch_validate(items, n_values)


def test_well_formed_item_lists_pass():
    assert capi.batch_validate([], 0) == ""
    assert capi.batch_validate([(0, 0, 1), (100, 0, 3)], 100) == ""               # zero-length items, one at the very end
    assert capi.batch_validate([(0, 10, 2), (20, 80, 1), (100, 0, 2)], 100) == ""
    assert capi.batch_validate([(3, 4, 3), (0, 1, 3)], 15) == ""                  # any order, gaps allowed


def test_add_batch_rejects_bad_input_before_gpu_work():
    x = [T.noise(0.1, 2, seed=1), T.noise(0.1, 1, seed=2)]
    with pytest.raises(ValueError):
        H.add_batch(x, [T.PAYLOAD])                                # one payload for two items
    with pytest.raises(ValueError):
        H.add_batch(x, [T.PAYLOAD, "not hex"])
    with pytest.raises(ValueError):
        H.add_batch(x, [T.PAYLOAD, T.PAYLOAD], sample_rate=48000)   # the resampled path is not batched
    if not HAS_GPU:
        with pytest.raises(RuntimeError) as e:
            H.add_batch(x, [T.PAYLOAD, T.PAYLOAD])
        assert e.type is RuntimeError
