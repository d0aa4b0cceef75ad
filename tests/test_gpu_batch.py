"""GPU: batched embed (hostapi.add_batch -> awm_embed_batch -> k_embed_batch / k_limiter_batch).  Item i of a batch must come out
bit identical to a separate `add` of that item with payload i: float and 16 bit PCM, host and device buffers, limiter on / off /
engaged, any channel count and length (zero, shorter than a frame, frame edges, seconds to minutes)."""
import math

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
RATE = 44100
LENGTHS = [0, 1, 1023, 1024, 1025, 3 * RATE, 10 * RATE, 61 * RATE, 180 * RATE]


def make_items():
    """~30 items: every length with 1, 2 and 3 channels, the same audio twice with two payloads, two loud (limiter) items"""
    rng = np.random.default_rng(11)
    pcms = []
    for i, n in enumerate(LENGTHS):
        for ch in (1, 2, 3):
            pcms.append(T.noise(n / RATE, ch, seed=100 + 3 * i + ch) if n else np.zeros((0, ch), np.float32))
    pcms.append(pcms[19].copy())                          # 10 s stereo once more, other payload
    pcms.append(T.noise(12.0, 2, seed=7, amp=1.0))         # full-scale noise: the watermark pushes it over the ceiling
    pcms.append(T.noise(4.0, 1, seed=8, amp=1.0))
    payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in pcms]
    return pcms, payloads


PCMS, PAYLOADS = make_items()


def single(x, payload, s16=False, stats=False):
    if s16:
        return H.add_s16(x, payload, want_stats=stats)
    return H.add(x, payload, want_stats=stats)


def to_s16(x):
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def test_batch_float_host_equals_single_items():
    assert len(PCMS) >= 30 and PAYLOADS[19] != PAYLOADS[27]
    outs, blocks, snr = H.add_batch(PCMS, PAYLOADS, want_stats=True)
    assert len(outs) == len(PCMS)
    for i, (x, p, y) in enumerate(zip(PCMS, PAYLOADS, outs)):
        want, want_blocks, want_snr = single(x, p, stats=True)
        assert y.shape == x.shape and np.array_equal(y, want), i
        assert blocks[i] == want_blocks, i
        assert (math.isinf(snr[i]) and math.isinf(want_snr)) or abs(snr[i] - want_snr) <= 1e-12 * abs(want_snr), (i, snr[i], want_snr)
    assert not np.array_equal(outs[19], outs[27])          # same audio, two payloads
    loud = outs[-2]
    assert np.abs(PCMS[-2]).max() > 0.99 and np.abs(loud).max() <= 0.99 + 1e-6   # the limiter is engaged


def test_batch_without_limiter_equals_single_items():
    H.set_params(test_no_limiter=True)
    outs = H.add_batch(PCMS, PAYLOADS)
    for i, (x, p, y) in enumerate(zip(PCMS, PAYLOADS, outs)):
        assert np.array_equal(y, single(x, p)), i
    assert np.abs(outs[-2]).max() > 0.99                   # without the limiter the loud item clips past the ceiling


def test_batch_s16_host_equals_single_items():
    x16 = [to_s16(x) for x in PCMS]
    outs = H.add_batch(x16, PAYLOADS)
    for i, (x, p, y) in enumerate(zip(x16, PAYLOADS, outs)):
        assert y.dtype == np.int16 and np.array_equal(y, single(x, p, s16=True)), i


@pytest.mark.parametrize("s16", [False, True], ids=["f32", "s16"])
def test_batch_device_buffers_equal_single_items(s16):
    """one packed device tensor with gaps between the items: items as host `add`, the gaps pass through unchanged"""
    torch = pytest.importorskip("torch")
    xs = [to_s16(x) for x in PCMS] if s16 else PCMS
    dt = np.int16 if s16 else np.float32
    parts, items, off = [], [], 0
    rng = np.random.default_rng(5)
    for x in xs:
        gap = int(rng.integers(0, 5))
        parts.append((rng.random(gap) * 100).astype(dt))
        off += gap
        items.append((off, x.shape[0], x.shape[1]))
        parts.append(x.reshape(-1))
        off += x.size
    packed = np.concatenate(parts)
    xd = torch.from_numpy(packed).cuda()
    yd = torch.full_like(xd, 7)
    outs = H.add_batch(xd, PAYLOADS, items=items, out=yd)
    got = yd.cpu().numpy()
    covered = np.zeros(packed.size, bool)
    for i, ((o, n, c), x, p) in enumerate(zip(items, xs, PAYLOADS)):
        assert np.array_equal(got[o:o + n * c].reshape(n, c), single(x, p, s16=s16)), i
        assert np.array_equal(outs[i].cpu().numpy(), got[o:o + n * c].reshape(n, c))
        covered[o:o + n * c] = True
    assert np.array_equal(got[~covered], packed[~covered])


def test_empty_batch_and_zero_length_items():
    assert H.add_batch([], []) == []
    outs = H.add_batch([np.zeros((0, 2), np.float32), np.zeros((0, 1), np.float32)], [T.PAYLOAD, T.PAYLOAD])
    assert [o.shape for o in outs] == [(0, 2), (0, 1)]


def test_batch_round_trip_finds_each_items_payload():
    sel = [i for i, x in enumerate(PCMS) if x.shape[0] >= 10 * RATE]
    assert len(sel) >= 10
    outs = H.add_batch([PCMS[i] for i in sel], [PAYLOADS[i] for i in sel])
    for i, y in zip(sel, outs):
        doc = H.get(y)
        found = {m["bits"] for m in doc["matches"] if m["quality"] > 0.35}     # (short clips also list n-best decodes of noise)
        others = set(PAYLOADS) - {PAYLOADS[i]}
        assert PAYLOADS[i] in found and not found & others, (i, PAYLOADS[i], doc["matches"][:3])
