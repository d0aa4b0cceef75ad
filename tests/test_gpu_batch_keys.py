"""GPU: batched embedding with a key per item (hostapi.add_batch / add_batch_rates with keys= -> awm_set_embed_roles_keys ->
k_embed_roles_keys, then awm_embed_batch_keys -> k_embed_batch<true, true>).  The device-built role tables must equal the host's
gen_embed_roles byte for byte for every layout, and item i of a batch with mixed keys must come out bit identical to the single-key
call on it alone with its own key: float and 16 bit, host and device buffers, 1 to 3 channels, zero-length items, stream offsets and
other sample rates, with equal Data Blocks and SNR.  Marked items decode under their own key's name only."""
import math

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
RATE = 44100


def numbered_key(n):
    """Key::set_test_key: big-endian n in the first 8 bytes"""
    return int(n).to_bytes(8, "big") + bytes(8)


def random_keys(n, seed):
    rng = np.random.default_rng(seed)
    return [bytes(rng.integers(0, 256, 16, dtype=np.uint8)) for _ in range(n)]


def payloads(n, seed, nibbles=32):
    rng = np.random.default_rng(seed)
    return ["".join("%x" % v for v in rng.integers(0, 16, nibbles)) for _ in range(n)]


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    H.set_short_payload(0)
    yield
    H.set_params()
    H.set_short_payload(0)


def assert_tables_equal(keys):
    dev = H.embed_roles_device(keys)
    assert dev.shape == (len(keys), H.frames_per_block(), 101)
    for k, key in enumerate(keys):
        host = H.embed_roles(key)
        assert np.array_equal(dev[k], host), (k, key.hex(), int(np.sum(dev[k] != host)))


def test_tables_equal_the_host_for_many_keys():
    assert_tables_equal(random_keys(64, seed=1) + [bytes(16), numbered_key(42), numbered_key(1)])


@pytest.mark.parametrize("layout", ["frames_per_bit_3", "frames_per_bit_1", "short_12", "short_16", "short_20", "linear", "linear_short_16"])
def test_tables_equal_the_host_for_every_layout(layout):
    if layout.startswith("frames_per_bit"):
        H.set_params(frames_per_bit=int(layout[-1]))          # 3: 77220 mix entries, the index array lives in global memory
    if layout.startswith("linear"):
        H.set_params(mix=False)
    if "short" in layout:
        H.set_short_payload(int(layout[-2:]))
    assert_tables_equal(random_keys(6, seed=2) + [bytes(16), numbered_key(7)])


# ---- batches with mixed keys

KEYS = random_keys(5, seed=3)
ITEM_KEYS = [0, 1, 0, 2, 3, 0, 1, 4, 2, 0, 3, 1]                 # keys 0 and 1 repeated, 4 used once
LENGTHS = [3.0, 0, 2.5, 1025, 4.0, 1, 6.0, 1023, 3.5, 5.0, 0, 2.0]   # float: seconds, int: frames


def make_items(seed):
    pcms = []
    for i, n in enumerate(LENGTHS):
        ch = 1 + i % 3
        pcms.append(T.noise(n if isinstance(n, float) else (n + 1) / RATE, ch, seed=seed + i)[: None if isinstance(n, float) else n])
    return pcms


PCMS = make_items(100)
PAYLOADS = payloads(len(PCMS), seed=4)
ITEM_KEY_BYTES = [KEYS[k] for k in ITEM_KEYS]


def same_snr(a, b):
    """--snr sums are accumulated with atomics: equal to 1e-12 relative, as the single-key batch tests hold them"""
    return (math.isinf(a) and math.isinf(b)) or abs(a - b) <= 1e-12 * abs(b)


def to_s16(x):
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


def test_mixed_keys_equal_single_adds_float_and_s16():
    outs, blocks, snr = H.add_batch(PCMS, PAYLOADS, keys=ITEM_KEY_BYTES, want_stats=True)
    for i, x in enumerate(PCMS):
        ref, b, s = H.add(x, PAYLOADS[i], key=ITEM_KEY_BYTES[i], want_stats=True)
        assert np.array_equal(outs[i], ref), i
        if x.shape[0]:
            assert blocks[i] == b and same_snr(snr[i], s), (i, blocks[i], b, snr[i], s)
    x16 = [to_s16(x) for x in PCMS]
    outs16, blocks16, snr16 = H.add_batch(x16, PAYLOADS, keys=ITEM_KEY_BYTES, want_stats=True)
    for i, x in enumerate(x16):
        ref, b, s = H.add_s16(x, PAYLOADS[i], key=ITEM_KEY_BYTES[i], want_stats=True)
        assert np.array_equal(outs16[i], ref), i
        if x.shape[0]:
            assert blocks16[i] == b and same_snr(snr16[i], s), i


def test_mixed_keys_on_device_buffers():
    import torch
    host_outs = H.add_batch(PCMS, PAYLOADS, keys=ITEM_KEY_BYTES)
    flat = np.concatenate([x.reshape(-1) for x in PCMS])
    items, off = [], 0
    for x in PCMS:
        items.append((off, x.shape[0], x.shape[1]))
        off += x.size
    dev = torch.from_numpy(flat).cuda()
    outs = H.add_batch(dev, PAYLOADS, keys=ITEM_KEY_BYTES, items=items)
    for i in range(len(PCMS)):
        assert np.array_equal(outs[i].cpu().numpy(), host_outs[i]), i
    dev16 = torch.from_numpy(to_s16(flat)).cuda()
    outs16 = H.add_batch(dev16, PAYLOADS, keys=ITEM_KEY_BYTES, items=items)
    for i, x in enumerate(PCMS):
        assert np.array_equal(outs16[i].cpu().numpy(), H.add_s16(to_s16(x), PAYLOADS[i], key=ITEM_KEY_BYTES[i])), i


def test_mixed_keys_at_stream_offsets_equal_add_windowed():
    zs = [0, 1023, 1024 + 517, 2 * RATE + 1, 300 * 1024 + 517, 57 * RATE, 5, 1 << 20, 3 * RATE - 1, 40 * 60 * RATE + 333, 17, 2048]
    outs, blocks, snr = H.add_batch(PCMS, PAYLOADS, keys=ITEM_KEY_BYTES, zero_frames=zs, want_stats=True)
    for i, x in enumerate(PCMS):
        if not x.shape[0]:
            assert outs[i].shape == x.shape
            continue
        ref, b, s = H.add_windowed(x, PAYLOADS[i], key=ITEM_KEY_BYTES[i], zero_frames=zs[i])
        assert np.array_equal(outs[i], ref), (i, zs[i])
        assert blocks[i] == b and same_snr(snr[i], s), (i, blocks[i], b, snr[i], s)


def test_mixed_keys_at_other_sample_rates_equal_single_adds():
    rates = [32000, 44100, 48000] * 4
    pcms = [x[: int(x.shape[0] * r / RATE)] for x, r in zip(PCMS, rates)]
    outs, blocks, snr = H.add_batch_rates(pcms, PAYLOADS, rates, keys=ITEM_KEY_BYTES, want_stats=True)
    for i, x in enumerate(pcms):
        ref, b, s = H.add(x, PAYLOADS[i], key=ITEM_KEY_BYTES[i], sample_rate=rates[i], want_stats=True)
        assert np.array_equal(outs[i], ref), (i, rates[i])
        if x.shape[0]:
            assert blocks[i] == b and same_snr(snr[i], s), (i, rates[i])
    # and with stream offsets: the single-key call with the same offsets
    zs = [0, 1023, 48000 * 5 + 517, 1 << 16, 3, 0, 32000 * 57, 2048, 1, 44100 * 2, 0, 77]
    outs = H.add_batch_rates(pcms, PAYLOADS, rates, keys=ITEM_KEY_BYTES, zero_frames=zs)
    for i, x in enumerate(pcms):
        ref = H.add_batch_rates([x], [PAYLOADS[i]], [rates[i]], key=ITEM_KEY_BYTES[i], zero_frames=[zs[i]])[0]
        assert np.array_equal(outs[i], ref), (i, rates[i], zs[i])


def test_one_key_for_all_items_equals_add_batch():
    key = KEYS[2]
    outs, blocks, snr = H.add_batch(PCMS, PAYLOADS, keys=[key] * len(PCMS), want_stats=True)
    ref, rblocks, rsnr = H.add_batch(PCMS, PAYLOADS, key=key, want_stats=True)
    assert all(np.array_equal(a, b) for a, b in zip(outs, ref))
    assert blocks == rblocks and all(same_snr(a, b) for a, b in zip(snr, rsnr))
    assert H.add_batch([], [], keys=[]) == []


def test_round_trip_decodes_under_own_key_name_only():
    names = ["customer-%d" % k for k in range(8)]
    keys = random_keys(8, seed=5)
    pcms = [T.noise(30.0, 1 + k % 2, seed=300 + k) for k in range(8)]      # long enough for a clip to decode its whole payload
    pays = payloads(8, seed=6)
    outs = H.add_batch(pcms, pays, keys=keys)
    for k, y in enumerate(outs):
        doc = H.get(y, keys=keys, names=names)
        hits = [m for m in doc["matches"] if m["bits"] == pays[k] and m["quality"] > 0.35]
        assert hits and {m["key"] for m in hits} == {names[k]}, (k, doc["matches"][:4])
        # a clip also yields weak spurious decodes (quality below 0.4 here); no other key finds the payload or anything strong
        assert not [m for m in doc["matches"] if m["key"] != names[k] and (m["bits"] == pays[k] or m["quality"] > 0.5)], (k, doc["matches"][:4])
