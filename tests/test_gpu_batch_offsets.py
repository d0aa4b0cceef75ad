"""GPU: batched embed at stream offsets (hostapi.add_batch(zero_frames=...) -> awm_embed_batch_offsets -> k_embed_batch /
k_limiter_batch).  Item i continues a stream that began zero_frames[i] frames earlier with silence, as an HLS segment does, and
must come out bit identical to add_windowed(item, zero_frames=z) = add(zeros (z) ++ item)[z:] (16 bit: add_s16 of the same), with
that call's data blocks and SNR: float and 16 bit PCM, host and device buffers, limiter on / off / engaged.  The HLS recipe of
hls-prepare / hls-add (segments with 3 s of context on each side, zero_frames = start_pos - prev_size) must reproduce `add` of the
whole stream, for one payload and for several viewers' payloads in one call."""
import math

import numpy as np
import pytest

import awm_testlib as T
import test_oracle_segments as S
from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
RATE = 44100
FAR = 40 * 60 * RATE + 333            # about 40 minutes into a stream: checked against add_windowed only
LENGTHS = [0, 1, 1023, 1024, 1025, 3 * RATE, 10 * RATE, 61 * RATE, 180 * RATE]
OFFSETS = [0, 100, 1023, 1024, 1025, 2048, 300 * 1024, 300 * 1024 + 517, 2 * RATE, 3 * RATE - 1, 4 * RATE + 1, 57 * RATE]


def make_items():
    """~30 items: every length with 1, 2 and 3 channels, each at its own offset (< 1024, whole frames, frame + remainder, limiter
    block edges, an HLS start_pos - prev_size), two loud items that engage the limiter, one item about 40 minutes in"""
    rng = np.random.default_rng(21)
    pcms, zs = [], []
    k = 0
    for i, n in enumerate(LENGTHS):
        for ch in (1, 2, 3):
            pcms.append(T.noise(n / RATE, ch, seed=200 + 3 * i + ch) if n else np.zeros((0, ch), np.float32))
            zs.append(OFFSETS[k % len(OFFSETS)])
            k += 1
    pcms.append(T.noise(12.0, 2, seed=17, amp=1.0))        # full-scale noise: the watermark pushes it over the ceiling
    zs.append(300 * 1024 + 517)
    pcms.append(T.noise(4.0, 1, seed=18, amp=1.0))
    zs.append(2 * RATE - 5)
    pcms.append(T.noise(12.0, 2, seed=19))
    zs.append(FAR)
    payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in pcms]
    return pcms, zs, payloads


PCMS, ZS, PAYLOADS = make_items()


def to_s16(x):
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


def zero_extended(x, z):
    return np.concatenate([np.zeros((z, x.shape[1]), x.dtype), x])


def single(x, z, payload, s16=False):
    """the single-item result the batch must reproduce, from a materialised silent prefix"""
    if s16:
        return H.add_s16(zero_extended(x, z), payload)[z:]
    return H.add(zero_extended(x, z), payload)[z:]


def assert_snr_equal(got, want, what):
    assert (math.isinf(got) and math.isinf(want)) or abs(got - want) <= 1e-12 * abs(want), (what, got, want)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


@pytest.mark.parametrize("limiter", [True, False], ids=["limiter", "no_limiter"])
def test_batch_float_host_equals_single_items(limiter):
    H.set_params(test_no_limiter=not limiter)
    assert len(PCMS) >= 30
    outs, blocks, snr = H.add_batch(PCMS, PAYLOADS, zero_frames=ZS, want_stats=True)
    for i, (x, z, p, y) in enumerate(zip(PCMS, ZS, PAYLOADS, outs)):
        assert y.shape == x.shape, i
        if x.shape[0]:
            want, want_blocks, want_snr = H.add_windowed(x, p, zero_frames=z)
            assert np.array_equal(y, want), (i, z)
            assert blocks[i] == want_blocks, (i, z, blocks[i], want_blocks)
            assert_snr_equal(snr[i], want_snr, (i, z))
        if z < FAR:
            assert np.array_equal(y, single(x, z, p)), (i, z)
    loud = outs[-3]
    if limiter:
        assert np.abs(PCMS[-3]).max() > 0.99 and np.abs(loud).max() <= 0.99 + 1e-6      # the limiter is engaged
    else:
        assert np.abs(loud).max() > 0.99


def test_zero_offsets_are_the_plain_batch():
    assert all(np.array_equal(a, b) for a, b in zip(H.add_batch(PCMS, PAYLOADS, zero_frames=[0] * len(PCMS)), H.add_batch(PCMS, PAYLOADS)))


def test_batch_s16_host_equals_single_items():
    sel = [i for i, z in enumerate(ZS) if z < FAR]
    x16 = [to_s16(PCMS[i]) for i in sel]
    outs = H.add_batch(x16, [PAYLOADS[i] for i in sel], zero_frames=[ZS[i] for i in sel])
    for i, x, y in zip(sel, x16, outs):
        assert y.dtype == np.int16 and np.array_equal(y, single(x, ZS[i], PAYLOADS[i], s16=True)), (i, ZS[i])


@pytest.mark.parametrize("s16", [False, True], ids=["f32", "s16"])
def test_batch_device_buffers_equal_single_items(s16):
    """one packed device tensor with gaps between the items: items as on the host, the gaps pass through unchanged"""
    torch = pytest.importorskip("torch")
    sel = [i for i, z in enumerate(ZS) if z < FAR] if s16 else list(range(len(PCMS)))
    xs = [to_s16(PCMS[i]) if s16 else PCMS[i] for i in sel]
    dt = np.int16 if s16 else np.float32
    parts, items, off = [], [], 0
    rng = np.random.default_rng(6)
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
    outs = H.add_batch(xd, [PAYLOADS[i] for i in sel], items=items, out=yd, zero_frames=[ZS[i] for i in sel])
    got = yd.cpu().numpy()
    covered = np.zeros(packed.size, bool)
    for k, (i, (o, n, c), x) in enumerate(zip(sel, items, xs)):
        if ZS[i] < FAR:
            want = single(x, ZS[i], PAYLOADS[i], s16=s16)
        else:
            want = H.add_windowed(x, PAYLOADS[i], zero_frames=ZS[i])[0]
        assert np.array_equal(got[o:o + n * c].reshape(n, c), want), (i, ZS[i])
        assert np.array_equal(outs[k].cpu().numpy(), got[o:o + n * c].reshape(n, c))
        covered[o:o + n * c] = True
    assert np.array_equal(got[~covered], packed[~covered])


# ---- the HLS recipe (src/hls.cc:529-613): 6 s segments, up to 3 s of context before and after, zero_frames = start_pos - prev_size

SEG, CTX = 6 * RATE, 3 * RATE
STREAM = T.noise(180.0, 2, seed=33)


def hls_items(x):
    """-> [(start_pos, size, prev_size, the item with its context)] as hls-prepare cuts and hls-add embeds them"""
    out = []
    for start in range(0, x.shape[0], SEG):
        size = min(SEG, x.shape[0] - start)
        prev = min(start, CTX)
        nxt = min(x.shape[0] - start - size, CTX)
        out.append((start, size, prev, x[start - prev:start + size + nxt]))
    return out


def trim(segs, ys):
    return np.concatenate([y[prev:prev + size] for (start, size, prev, _), y in zip(segs, ys)])


@pytest.mark.parametrize("s16", [False, True], ids=["f32", "s16"])
def test_hls_segments_concatenate_to_the_whole_stream(s16):
    x = to_s16(STREAM) if s16 else STREAM
    segs = hls_items(x)
    assert len(segs) == 30
    ys = H.add_batch([s[3] for s in segs], [T.PAYLOAD] * len(segs), zero_frames=[start - prev for start, size, prev, _ in segs])
    want = H.add_s16(x, T.PAYLOAD) if s16 else H.add(x, T.PAYLOAD)
    assert np.array_equal(trim(segs, ys), want)


def test_hls_viewers_fan_out_in_one_call():
    viewers = ["%032x" % (0x1234567 * (v + 1)) for v in range(4)]
    segs = hls_items(STREAM)
    items = [s[3] for s in segs] * len(viewers)
    payloads = [p for p in viewers for _ in segs]
    zs = [start - prev for start, size, prev, _ in segs] * len(viewers)
    ys = H.add_batch(items, payloads, zero_frames=zs)
    for v, p in enumerate(viewers):
        y = trim(segs, ys[v * len(segs):(v + 1) * len(segs)])
        assert np.array_equal(y, H.add(STREAM, p)), v
        found = {m["bits"] for m in H.get(y)["matches"] if m["quality"] > 0.35}
        assert p in found and not found & (set(viewers) - {p}), (v, found)


# ---- against the reference: the golden cases of tests/golden/golden_segments.json through the batch

def test_batch_items_equal_oracle_on_golden_cases():
    cases = [S.G["cases"][k] for k in sorted(S.G["cases"])]
    for no_limiter in (False, True):
        sel = [g for g in cases if ("--test-no-limiter" in g["add_args"]) == no_limiter]
        H.set_params(test_no_limiter=no_limiter)
        xs = [S.case_input(g) for g in sel]
        ys = H.add_batch(xs, [S.G["payload"]] * len(sel), zero_frames=[g["zero_frames"] for g in sel])
        for g, x, y in zip(sel, xs, ys):
            ref = S.oracle_at(x, g["zero_frames"], no_limiter)
            r = T.rms(y - ref)
            assert r < 1e-5, (g["zero_frames"], g["channels"], r)
