"""GPU: batched embed at any sample rate (hostapi.add_batch_rates -> awm_embed_batch_rates -> k_resample_batch, k_embed_batch,
k_resample_mix_batch, k_limiter_rates).  Item i of a batch must come out bit identical to a separate `add` of that item at its own
rate with payload i: float and 16 bit PCM, host and device buffers, limiter on / off / engaged, 1 to 3 channels, lengths from zero
frames to three minutes, five rates in one batch, any split into waves."""
import ctypes
import math

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

pytestmark = pytest.mark.gpu
RATES = [32000, 44100, 48000, 96000, 22050]
LENGTHS = [0, 1, 1023, 1025, 3.0, 11.3, 61.0, 180.0]      # int: frames, float: seconds at the item's rate


def noise(n_frames, channels, seed, amp=0.5):
    rng = np.random.default_rng(seed)
    return ((rng.random((n_frames, channels), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


def make_items():
    """28 items: every length with 1, 2 and 3 channels at rotating rates, two loud (limiter) items, two more 10 s items"""
    rng = np.random.default_rng(12)
    pcms, rates = [], []
    for i, n in enumerate(LENGTHS):
        for ch in (1, 2, 3):
            r = RATES[(3 * i + ch) % len(RATES)]
            pcms.append(noise(n if isinstance(n, int) else int(n * r), ch, seed=200 + 3 * i + ch))
            rates.append(r)
    pcms.append(noise(12 * 48000, 2, seed=7, amp=1.0))     # full-scale noise: the watermark pushes it over the ceiling
    rates.append(48000)
    pcms.append(noise(4 * 32000, 1, seed=8, amp=1.0))
    rates.append(32000)
    pcms.append(noise(10 * 22050, 2, seed=9))
    rates.append(22050)
    pcms.append(noise(10 * 96000, 1, seed=10))
    rates.append(96000)
    payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in pcms]
    return pcms, rates, payloads


PCMS, RATES_OF, PAYLOADS = make_items()
LOUD = len(PCMS) - 4
_SINGLE = {}


def single(i, no_limiter=False):
    """H.add of item i alone at its rate -> (output, data blocks, snr dB), cached per limiter setting"""
    k = (i, no_limiter)
    if k not in _SINGLE:
        H.set_params(test_no_limiter=no_limiter)
        try:
            _SINGLE[k] = H.add(PCMS[i], PAYLOADS[i], sample_rate=RATES_OF[i], want_stats=True)
        finally:
            H.set_params()
    return _SINGLE[k]


def to_s16(x):
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def test_items_cover_the_issue_grid():
    assert len(PCMS) >= 28 and set(RATES_OF) == set(RATES)
    assert {x.shape[1] for x in PCMS} == {1, 2, 3} and min(x.shape[0] for x in PCMS) == 0 and max(x.shape[0] for x in PCMS) >= 180 * 22050


def test_float_items_equal_single_add():
    outs, blocks, snr = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF, want_stats=True)
    assert len(outs) == len(PCMS)
    for i, y in enumerate(outs):
        want, want_blocks, want_snr = single(i)
        assert y.shape == PCMS[i].shape and np.array_equal(y, want), (i, RATES_OF[i], PCMS[i].shape)
        assert blocks[i] == want_blocks, i
        assert (math.isinf(snr[i]) and math.isinf(want_snr)) or abs(snr[i] - want_snr) <= 1e-12 * abs(want_snr), (i, snr[i], want_snr)
    assert np.abs(PCMS[LOUD]).max() > 0.99 and np.abs(outs[LOUD]).max() <= 0.99 + 1e-6      # the limiter is engaged


def test_float_items_equal_single_add_without_limiter():
    H.set_params(test_no_limiter=True)
    outs, blocks, snr = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF, want_stats=True)
    for i, y in enumerate(outs):
        want, want_blocks, want_snr = single(i, no_limiter=True)
        assert np.array_equal(y, want), (i, RATES_OF[i], PCMS[i].shape)
        assert blocks[i] == want_blocks, i
        assert (math.isinf(snr[i]) and math.isinf(want_snr)) or abs(snr[i] - want_snr) <= 1e-12 * abs(want_snr), (i, snr[i], want_snr)
    assert np.abs(outs[LOUD]).max() > 0.99                  # without the limiter the loud item clips past the ceiling


def test_s16_items_equal_float_add_between_conversions():
    x16 = [to_s16(x) for x in PCMS]
    outs = H.add_batch_rates(x16, PAYLOADS, RATES_OF)
    for i, (x, p, r, y) in enumerate(zip(x16, PAYLOADS, RATES_OF, outs)):
        want = O.quantize_sndfile16(H.add(O.int16_to_float(x), p, sample_rate=r)) if x.size else x
        assert y.dtype == np.int16 and np.array_equal(y, want.reshape(x.shape)), (i, r, x.shape)


@pytest.mark.parametrize("s16", [False, True], ids=["f32", "s16"])
def test_device_buffers_with_gaps(s16):
    """one packed device tensor with gaps between the items: the items as host `add_batch_rates`, the gaps pass through unchanged"""
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
    want = H.add_batch_rates(xs, PAYLOADS, RATES_OF)
    xd = torch.from_numpy(packed).cuda()
    yd = torch.full_like(xd, 7)
    outs = H.add_batch_rates(xd, PAYLOADS, RATES_OF, items=items, out=yd)
    got = yd.cpu().numpy()
    covered = np.zeros(packed.size, bool)
    for i, (o, n, c) in enumerate(items):
        assert np.array_equal(got[o:o + n * c].reshape(n, c), want[i]), i
        assert np.array_equal(outs[i].cpu().numpy(), want[i])
        covered[o:o + n * c] = True
    assert np.array_equal(got[~covered], packed[~covered])          # as add_batch: the gaps keep the input's values


def test_waves_give_the_same_bytes():
    """a scratch cap far below the batch: several waves, the 3 min 96 kHz stereo item alone above the cap"""
    scratch = [x.shape[0] * 44100 / r * x.shape[1] * 8 if r != 44100 else 0 for x, r in zip(PCMS, RATES_OF)]   # ~2 x n44 x C floats
    cap = 64 << 20
    assert max(scratch) > cap and sum(scratch) > 3 * cap
    n0 = H.gpu_launches()
    want = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF)
    n1 = H.gpu_launches()
    got = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF, scratch_bytes=cap)
    n2 = H.gpu_launches()
    assert (n2 - n1) - (n1 - n0) >= 2 * 4            # every wave after the first adds resample, embed, mix and limiter launches
    for i, (a, b) in enumerate(zip(want, got)):
        assert a.tobytes() == b.tobytes(), i


@pytest.mark.parametrize("name", ["rate32000_add", "rate48000_add_nolimiter"])
def test_reference_inputs_inside_a_batch(name):
    """the golden inputs that test_add_other_sample_rates_vs_reference pins single `add` to, as items of a larger batch"""
    import json
    import os
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden.json")))[name]
    x = O.int16_to_float(O.quantize_sndfile16(O.gen_noise(g["seconds"], g["rate"])))
    no_lim = "--test-no-limiter" in g["add_args"]
    H.set_params(test_no_limiter=no_lim)
    msg = "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"
    want, want_blocks, want_snr = H.add(x, msg, want_stats=True, sample_rate=g["rate"])
    sel = [0, 5, 13, 20]
    pcms = [PCMS[sel[0]], PCMS[sel[1]], x, PCMS[sel[2]], PCMS[sel[3]]]
    outs, blocks, snr = H.add_batch_rates(pcms, [PAYLOADS[sel[0]], PAYLOADS[sel[1]], msg, PAYLOADS[sel[2]], PAYLOADS[sel[3]]],
                                          [RATES_OF[sel[0]], RATES_OF[sel[1]], g["rate"], RATES_OF[sel[2]], RATES_OF[sel[3]]], want_stats=True)
    assert np.array_equal(outs[2], want)
    assert blocks[2] == want_blocks and ("Data Blocks:  %d\n" % blocks[2]) in g["add_stderr"]
    assert abs(snr[2] - want_snr) <= 1e-12 * abs(want_snr)
    for k, i in enumerate(sel):
        assert np.array_equal(outs[k if k < 2 else k + 1], single(i, no_limiter=no_lim)[0]), i


def test_44k_items_equal_add_batch():
    sel = [i for i, r in enumerate(RATES_OF) if r == 44100]
    assert len(sel) >= 4
    want = H.add_batch([PCMS[i] for i in sel], [PAYLOADS[i] for i in sel])
    got = H.add_batch_rates([PCMS[i] for i in sel], [PAYLOADS[i] for i in sel], [44100] * len(sel))
    for a, b in zip(want, got):
        assert np.array_equal(a, b)


def test_bound_pcm_survives():
    """a binding made before the call (here one pushed through the resampler, which lives in a context buffer) is still there after it"""
    lib = capi.load()
    lib.awm_pcm_device.restype = ctypes.c_void_p
    h = ctypes.c_void_p(H.engine_ctx())
    x = T.noise(5.0, 2, seed=3)
    n_out = int(x.shape[0] * 48000 / 44100)
    assert lib.awm_pcm_bind(h, H._ptr(x), ctypes.c_size_t(x.shape[0]), ctypes.c_int(2), ctypes.c_size_t(0), ctypes.c_size_t(0)) == 0
    assert lib.awm_pcm_push_resampled(h, ctypes.c_double(48000 / 44100), ctypes.c_int(16), ctypes.c_size_t(n_out)) == 0

    def bound():
        n, ch = ctypes.c_size_t(), ctypes.c_int()
        p = lib.awm_pcm_device(h, ctypes.byref(n), ctypes.byref(ch))
        assert p
        buf = np.empty((n.value, ch.value), np.float32)
        assert lib.awm_copy_to_host(h, H._ptr(buf), ctypes.c_void_p(p), ctypes.c_size_t(buf.nbytes)) == 0
        return p, buf

    p0, before = bound()
    H.add_batch_rates(PCMS[:12], PAYLOADS[:12], RATES_OF[:12])
    p1, after = bound()
    assert p0 == p1 and np.array_equal(before, after)
    assert lib.awm_pcm_pop(h) == 0
    _, orig = bound()
    assert np.array_equal(orig, x)


def test_round_trip_finds_each_items_payload():
    sel = [i for i, x in enumerate(PCMS) if x.shape[0] >= 10 * RATES_OF[i]]
    assert len(sel) >= 10 and len({RATES_OF[i] for i in sel}) == len(RATES)
    outs = H.add_batch_rates([PCMS[i] for i in sel], [PAYLOADS[i] for i in sel], [RATES_OF[i] for i in sel])
    for i, y in zip(sel, outs):
        doc = H.get(y, sample_rate=RATES_OF[i])
        found = {m["bits"] for m in doc["matches"] if m["quality"] > 0.35}
        others = set(PAYLOADS) - {PAYLOADS[i]}
        assert PAYLOADS[i] in found and not found & others, (i, RATES_OF[i], PAYLOADS[i], doc["matches"][:3])


def test_empty_batch_and_zero_length_items():
    assert H.add_batch_rates([], [], []) == []
    outs = H.add_batch_rates([np.zeros((0, 2), np.float32), np.zeros((0, 1), np.float32)], [T.PAYLOAD, T.PAYLOAD], [48000, 44100])
    assert [o.shape for o in outs] == [(0, 2), (0, 1)]
