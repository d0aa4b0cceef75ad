"""GPU: batched embed at stream positions at any sample rate (hostapi.add_batch_rates(zero_frames=...) ->
awm_embed_batch_rates_offsets -> k_resample_batch<true>, k_embed_batch<true>, k_resample_mix_batch<true>, k_limiter_rates<true>).
Item i continues a stream at its own rate that began zero_frames[i] frames earlier with silence, as an HLS segment of a 48 kHz master
does, and must come out bit identical to add_batch_rates([zeros (z) ++ item])[z:]: float and 16 bit PCM, host and device buffers,
1 to 3 channels, lengths from zero frames to a minute, offsets around frame and limiter block edges and far into the stream.  Data
Blocks are those of the whole stream; --snr counts the item's own positions.  The HLS recipe (segments with 3 s of context on each
side) must reproduce `add` of the whole 48 kHz stream, for one payload and for many viewers' payloads in one call."""

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
import test_oracle_segments_rates as S
from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
RATES = [8000, 32000, 48000, 96000, 44100]
LENGTHS = [0, 1, 1023, 1025, 3.0, 61.0]                 # int: frames, float: seconds at the item's rate
FAR = 40 * 60                                           # seconds: 40 min into the stream


def offsets(r):
    """offsets (frames at rate r) around 0, 1024, 2048, the limiter block edges (r frames), 57 s and 40 min + 333"""
    return [0, 1, 1023, 1024, 1025, 2047, 2048, r - 1, r, r + 1, 2 * r + 1, 57 * r, FAR * r + 333]


def noise(n_frames, channels, seed, amp=0.5):
    rng = np.random.default_rng(seed)
    return ((rng.random((n_frames, channels), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


def make_items():
    """every length at every rate, channels and offsets rotating, a 2 s mono item 40 min + 333 frames into the stream at every
    resampled rate, and two loud items that engage the limiter"""
    rng = np.random.default_rng(31)
    pcms, rates, zs = [], [], []
    k = 0
    for i, n in enumerate(LENGTHS):
        for j, r in enumerate(RATES):
            ch = 1 + (i + j) % 3
            pcms.append(noise(n if isinstance(n, int) else int(n * r), ch, seed=400 + k))
            rates.append(r)
            zo = offsets(r)
            z = zo[k % len(zo)]
            if z > 60 * r and (n == 61.0 or ch > 1 or r == 96000):
                z = zo[(k + 1) % len(zo)]       # keep the materialised whole streams of this file affordable
            zs.append(z)
            k += 1
    for r in RATES[:4]:                         # 40 min + 333 into the stream at every resampled rate: short mono items
        pcms.append(noise(2 * r, 1, seed=r))
        rates.append(r)
        zs.append(FAR * r + 333)
    pcms.append(noise(8 * 48000, 2, seed=7, amp=1.0))
    rates.append(48000)
    zs.append(48000 * 5 + 517)
    pcms.append(noise(4 * 32000, 1, seed=8, amp=1.0))
    rates.append(32000)
    zs.append(1024 + 3)
    payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in pcms]
    return pcms, rates, zs, payloads


PCMS, RATES_OF, ZS, PAYLOADS = make_items()


def zero_extended(x, z):
    return np.concatenate([np.zeros((z, x.shape[1]), x.dtype), x])


def whole(x, z, payload, rate, want_stats=False):
    """the whole stream zeros (z) ++ x through add_batch_rates, trimmed to x's positions"""
    r = H.add_batch_rates([zero_extended(x, z)], [payload], [rate], want_stats=want_stats)
    if want_stats:
        return r[0][0][z:], r[1][0], r[2][0]
    return r[0][z:]


def to_s16(x):
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def test_items_equal_their_whole_streams():
    assert {r for r in RATES_OF} == set(RATES) and len(PCMS) >= 30
    outs, blocks, snr = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF, zero_frames=ZS, want_stats=True)
    for i, (x, r, z, p, y) in enumerate(zip(PCMS, RATES_OF, ZS, PAYLOADS, outs)):
        assert y.shape == x.shape, i
        if not x.shape[0]:
            continue
        want, want_blocks, want_snr = whole(x, z, p, r, want_stats=True)
        assert np.array_equal(y, want), (i, r, z, x.shape)
        assert blocks[i] == want_blocks, (i, r, z, blocks[i], want_blocks)
        # --snr sums the item's own positions: the watermark before z (on silence) is left out, which only matters for short items
        assert snr[i] >= want_snr - 1e-9, (i, r, z, snr[i], want_snr)
        if x.shape[0] >= 3 * r:
            assert snr[i] - want_snr < 0.05, (i, r, z, snr[i], want_snr)
    assert np.abs(PCMS[-2]).max() > 0.99 and np.abs(outs[-2]).max() <= 0.99 + 1e-6      # the limiter is engaged


def test_no_limiter_items_equal_their_whole_streams():
    H.set_params(test_no_limiter=True)
    sel = [i for i in range(len(PCMS)) if PCMS[i].shape[0] and PCMS[i].shape[0] <= 3 * RATES_OF[i]]
    outs = H.add_batch_rates([PCMS[i] for i in sel], [PAYLOADS[i] for i in sel], [RATES_OF[i] for i in sel], zero_frames=[ZS[i] for i in sel])
    for i, y in zip(sel, outs):
        assert np.array_equal(y, whole(PCMS[i], ZS[i], PAYLOADS[i], RATES_OF[i])), (i, RATES_OF[i], ZS[i])


def test_s16_and_device_buffers_equal_their_whole_streams():
    torch = pytest.importorskip("torch")
    sel = [i for i in range(len(PCMS)) if PCMS[i].shape[0] and ZS[i] < 60 * RATES_OF[i]][:12]
    x16 = [to_s16(PCMS[i]) for i in sel]
    wants = [whole(x, ZS[i], PAYLOADS[i], RATES_OF[i]) for i, x in zip(sel, x16)]
    outs = H.add_batch_rates(x16, [PAYLOADS[i] for i in sel], [RATES_OF[i] for i in sel], zero_frames=[ZS[i] for i in sel])
    for i, y, want in zip(sel, outs, wants):
        assert y.dtype == np.int16 and np.array_equal(y, want), (i, RATES_OF[i], ZS[i])
    for s16 in (False, True):
        xs = x16 if s16 else [PCMS[i] for i in sel]
        parts, items, off = [], [], 0
        for x in xs:                                    # one value of gap: odd offsets for every other item
            parts += [np.full(1, 3, x.dtype), x.reshape(-1)]
            items.append((off + 1, x.shape[0], x.shape[1]))
            off += 1 + x.size
        packed = np.concatenate(parts)
        xd = torch.from_numpy(packed).cuda()
        yd = torch.full_like(xd, 7)
        H.add_batch_rates(xd, [PAYLOADS[i] for i in sel], [RATES_OF[i] for i in sel], items=items, out=yd, zero_frames=[ZS[i] for i in sel])
        got = yd.cpu().numpy()
        for i, (o, n, c), x, w16 in zip(sel, items, xs, wants):
            want = w16 if s16 else whole(x, ZS[i], PAYLOADS[i], RATES_OF[i])
            assert np.array_equal(got[o:o + n * c].reshape(n, c), want), (s16, i, RATES_OF[i], ZS[i])
            assert got[o - 1] == packed[o - 1]


def test_zero_offsets_and_mark_rate_items_are_the_existing_calls():
    a = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF, zero_frames=[0] * len(PCMS), want_stats=True)
    b = H.add_batch_rates(PCMS, PAYLOADS, RATES_OF, want_stats=True)
    assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1]
    assert all(snr_equal(x, y) for x, y in zip(a[2], b[2]))
    sel = [i for i in range(len(PCMS)) if RATES_OF[i] == 44100]
    xs, ps, zs = [PCMS[i] for i in sel], [PAYLOADS[i] for i in sel], [ZS[i] for i in sel]
    a = H.add_batch_rates(xs, ps, [44100] * len(sel), zero_frames=zs, want_stats=True)
    b = H.add_batch(xs, ps, zero_frames=zs, want_stats=True)
    assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1]
    assert all(snr_equal(x, y) for x, y in zip(a[2], b[2]))


def snr_equal(got, want):
    """--snr sums are added atomically in no fixed order: equal to 1e-12 relative"""
    return (np.isinf(got) and np.isinf(want)) or abs(got - want) <= 1e-12 * abs(want)


def test_far_item_with_a_small_scratch():
    """an item 24 h into a 48 kHz stream with a 32 MiB scratch: its scratch window is sized by its own length, not by its offset"""
    x = noise(12 * 48000, 2, seed=77)
    y = H.add_batch_rates([x], [T.PAYLOAD], [48000], zero_frames=[24 * 3600 * 48000 + 333], scratch_bytes=32 << 20)[0]
    assert np.isfinite(y).all() and 0 < T.rms(y - x) < 0.01


# ---- the HLS recipe (src/hls.cc:529-613) on a 48 kHz master: 6 s segments, 3 s of context, zero_frames = start_pos - prev_size

RATE = 48000
SEG, CTX = 6 * RATE, 3 * RATE


def hls_items(x):
    out = []
    for start in range(0, x.shape[0], SEG):
        size = min(SEG, x.shape[0] - start)
        prev = min(start, CTX)
        nxt = min(x.shape[0] - start - size, CTX)
        out.append((start, size, prev, x[start - prev:start + size + nxt]))
    return out


def trim(segs, ys):
    return np.concatenate([y[prev:prev + size] for (start, size, prev, _), y in zip(segs, ys)])


def test_vod_segments_concatenate_to_the_whole_stream():
    x = noise(180 * RATE, 2, seed=33, amp=0.25)
    segs = hls_items(x)
    assert len(segs) == 30
    ys = H.add_batch_rates([s[3] for s in segs], [T.PAYLOAD] * len(segs), [RATE] * len(segs), zero_frames=[s[0] - s[2] for s in segs])
    y = trim(segs, ys)
    assert np.array_equal(y, H.add(x, T.PAYLOAD, sample_rate=RATE))
    found = {m["bits"] for m in H.get(y, sample_rate=RATE)["matches"] if m["quality"] > 0.35}
    assert T.PAYLOAD in found, found


def test_live_fan_out_far_into_the_stream():
    """256 viewers, one segment (with context) 40 min into the stream, each with its own payload"""
    start = FAR * RATE
    seg = noise(SEG + 2 * CTX, 2, seed=44, amp=0.25)
    viewers = ["%032x" % (0x9e3779b97f4a7c15 * (v + 1) % (1 << 128)) for v in range(256)]
    ys = H.add_batch_rates([seg] * len(viewers), viewers, [RATE] * len(viewers), zero_frames=[start - CTX] * len(viewers))
    for v in (0, 101, 255):
        assert np.array_equal(ys[v], whole(seg, start - CTX, viewers[v], RATE)), v
    assert not np.array_equal(ys[0], ys[1])


# ---- against the reference: the cases of tests/golden/golden_segments_rates.json through the batch, 16 bit in and out

def test_golden_cases_equal_the_reference():
    """The oracle reproduces the reference's whole-stream output of every case bit for bit (test_oracle_segments_rates.py, checked
    again here).  The batch's 16 bit output is within 1 LSB of it on fewer than 1e-3 of the values: the same bound as single `add`
    at other rates against the reference (test_gpu_speed.py::test_add_other_sample_rates_vs_reference), whose float sums the batch
    reproduces bit for bit (the tests above).  Data Blocks equal the reference's; --snr, which counts only the item's own positions,
    is at least the reference's whole-stream SNR line and within 0.05 dB of it."""
    cases = [S.G["cases"][k] for k in sorted(S.G["cases"])]
    assert any(g["zero_frames"] == 57 * g["rate"] for g in cases)
    key = O.Key().aes_key
    for no_limiter in (False, True):
        sel = [g for g in cases if ("--test-no-limiter" in g["add_args"]) == no_limiter]
        H.set_params(test_no_limiter=no_limiter)
        xs = [S.case_input(g) for g in sel]
        ys, blocks, snr = H.add_batch_rates(xs, [S.G["payload"]] * len(sel), [g["rate"] for g in sel], key=key,
                                            zero_frames=[g["zero_frames"] for g in sel], want_stats=True)
        for g, x, y, b, s in zip(sel, xs, ys, blocks, snr):
            what = (g["rate"], g["zero_frames"], g["channels"], g["amp"])
            assert S.sha16(x) == g["input_sha256"] and y.dtype == np.int16 and y.shape == x.shape
            ref16 = O.quantize_sndfile16(S.oracle_whole(g, x)[1])
            assert S.sha16(ref16) == g["output_sha256"], what
            d = np.abs(y.astype(np.int32) - ref16.astype(np.int32))
            assert d.max() <= 1 and np.count_nonzero(d) < 1e-3 * d.size, (what, int(d.max()), int(np.count_nonzero(d)))
            assert b == g["data_blocks"], (what, b, g["data_blocks"])
            assert g["snr_db"] - 1e-3 <= s < g["snr_db"] + 0.05, (what, s, g["snr_db"])
