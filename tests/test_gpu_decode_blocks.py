"""Block decode (awm_decode_blocks: k_decode_fft + k_mix_decode) against a float64 reference of fft_range + mix_decode + the decode
bit order, written here in plain numpy: per frame and channel np.fft.rfft of the windowed samples, band dB (-96 for a power of
exactly zero), then for coded bit o and every mix entry of its frames_per_bit frames and every channel
    umag += D[i][up] - (D[prev][up] + D[next][up]) / 2,   i = frame * C + ch, next / prev = i +- C, reflected at the block's ends
(dmag the same with the down band), raw[bit_order[o]] = umag - dmag.  test_reference_matches_oracle pins it to
O.raw_bits_for_block.

Error bound of a raw bit: the kernels accumulate in double, so only the fp32 dB values carry error.  Every term carries
m = |dB| + (20 / ln 10) log2(1024) ||x w|| / |X_k| (its condition with respect to the fp32 FFT of the frame), in units of
u = 2^-24, weighted 1 for the frame itself and 1/2 for each neighbour; the bound is LAMBDA u sum(weight m) with LAMBDA = 4 (the dB
rounding, the FFT and the fp32 sum of the two neighbours).
"""
import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi

U = 2.0 ** -24
LAMBDA = 4.0
N = 1024
KEY = O.Key.test_key(3)
RATIO = [0.0]


def block_db(x, index, fpb):
    """D [fpb * C][81] float64 and the per-term magnitudes m [fpb * C][81] (units of u) of the block at sample frame `index`"""
    C = x.shape[1]
    win = O.analysis_window(N).astype(np.float64)
    idx = index + np.arange(fpb)[:, None] * N + np.arange(N)[None, :]
    D = np.zeros((fpb, C, 81))
    M = np.zeros((fpb, C, 81))
    for ch in range(C):
        xw = x[idx, ch].astype(np.float64) * win
        X = np.fft.rfft(xw, axis=1)[:, 20:101]
        pw = X.real ** 2 + X.imag ** 2
        pos = pw > 0
        D[:, ch] = np.where(pos, 10 * np.log10(np.where(pos, pw, 1.0)), -96.0)
        nx = np.sqrt((xw * xw).sum(axis=1))[:, None]
        M[:, ch] = np.abs(D[:, ch]) + np.where(pos, (20 / np.log(10)) * 10 * nx / np.sqrt(np.where(pos, pw, 1.0)), 0.0)
    return D.reshape(fpb * C, 81), M.reshape(fpb * C, 81)


def decode_ref(x, index, mix, order, frames_per_bit, fpb):
    """(raw bits in decode order, their bounds) of one block"""
    C = x.shape[1]
    D, M = block_db(x, index, fpb)
    n_spect = fpb * C
    n_coded = len(order)
    fr = mix["frame"].astype(np.int64).reshape(n_coded, frames_per_bit * 30)
    up = mix["up"].astype(np.int64).reshape(n_coded, -1) - 20
    dn = mix["down"].astype(np.int64).reshape(n_coded, -1) - 20
    um = np.zeros(n_coded)
    bd = np.zeros(n_coded)
    for ch in range(C):
        i = fr * C + ch
        nxt = np.where(i + C < n_spect, i + C, i - C)
        prv = np.where(i - C >= 0, i - C, i + C)
        for b, sign in ((up, 1.0), (dn, -1.0)):
            um += sign * (D[i, b] - (D[prv, b] + D[nxt, b]) * 0.5).sum(axis=1)
            bd += (M[i, b] + 0.5 * (M[prv, b] + M[nxt, b])).sum(axis=1)
    raw = np.zeros(n_coded)
    bound = np.zeros(n_coded)
    raw[order] = um
    bound[order] = LAMBDA * U * bd
    return raw, bound


def real_mix(key, P, linear=False):
    """the mix tables the host passes for P: the shuffled entries, or with --linear the same triples unshuffled"""
    if not linear:
        rows = O.gen_mix_entries(key, P)
    else:
        udg, bpg = O.UpDownGen(key, O.STREAM_DATA_UP_DOWN, P), O.BitPosGen(key, P)
        rows = []
        for f in range(O.mark_data_frame_count(P)):
            u, d = udg.get(f)
            rows += [(bpg.data_frame(f), a, b) for a, b in zip(u, d)]
    ent = np.zeros(len(rows), capi.MIX_ENTRY)
    ent["frame"], ent["up"], ent["down"] = zip(*rows)
    n_coded = O.code_size(O.A, P)
    order = np.array(O.randomize_bit_order(key, list(range(n_coded)), True), np.uint16)
    return ent, order


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def check_blocks(ctx, x, indices, mix, order, frames_per_bit, fpb, slot=3, name=""):
    ctx.set_mix_tables(slot, mix, order, frames_per_bit, fpb)
    ctx.pcm_bind(x)
    raw, valid = ctx.decode_blocks(indices, len(order), key_slot=slot)
    for k, i in enumerate(indices):
        ok = i + fpb * N <= x.shape[0]
        assert valid[k] == ok, (name, k, i)
        if not ok:
            continue
        want, bound = decode_ref(x, i, mix, order, frames_per_bit, fpb)
        err = np.abs(raw[k] - want)
        RATIO[0] = max(RATIO[0], (err / bound).max())
        bad = np.nonzero(err > bound)[0]
        assert len(bad) == 0, (name, k, i, bad[:5], err[bad[:5]], bound[bad[:5]])
    print("%-36s max err/bound so far %.3g" % (name, RATIO[0]))
    return raw, valid


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3, 4])
@pytest.mark.parametrize("params", ["fpbit1", "fpbit2", "fpbit3", "short12", "short20", "linear"])
def test_real_tables(ctx, C, params):
    """real mix tables for frames_per_bit 1, 2, 3, the --short payload lengths and --linear; blocks at index 0, at odd indices, one
    ending exactly at the last sample frame and one a sample frame later (valid = 0)"""
    P = {"fpbit1": O.Params(frames_per_bit=1), "fpbit2": O.Params(), "fpbit3": O.Params(frames_per_bit=3),
         "short12": O.Params(payload_size=12, payload_short=True), "short20": O.Params(payload_size=20, payload_short=True, frames_per_bit=3),
         "linear": O.Params(mix=False)}[params]
    fpb = O.frames_per_block(P)
    mix, order = real_mix(KEY, P, linear=not P.mix)
    n = fpb * N + 4097
    x = T.noise(n / 44100.0 + 1, C, seed=C * 10 + len(params))[:n]
    check_blocks(ctx, x, [0, 1, 4097, 2047, n - fpb * N + 1], mix, order, P.frames_per_bit, fpb, name="%s C=%d" % (params, C))


def synthetic_mix(fpb, n_coded, frames_per_bit, seed):
    """mix entries whose frames include 0 and fpb - 1, where the neighbour of a frame is reflected at the block's ends"""
    rng = np.random.default_rng(seed)
    n = n_coded * frames_per_bit * 30
    mix = np.zeros(n, capi.MIX_ENTRY)
    mix["frame"] = rng.integers(0, fpb, n)
    mix["frame"][::7] = 0
    mix["frame"][3::7] = fpb - 1
    mix["up"] = rng.integers(20, 101, n)
    mix["down"] = rng.integers(20, 101, n)
    order = rng.permutation(n_coded).astype(np.uint16)
    return mix, order


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3, 4])
def test_synthetic_block_edges(ctx, C):
    fpb, n_coded, fpbit = 9, 40, 2
    mix, order = synthetic_mix(fpb, n_coded, fpbit, seed=C)
    n = 40 * N + 333
    x = T.noise(1.0, C, seed=50 + C)[:n]
    check_blocks(ctx, x, [0, 3, 1025, 777, n - fpb * N, n - fpb * N + 1], mix, order, fpbit, fpb, name="synthetic C=%d" % C)


@pytest.mark.gpu
def test_more_blocks_than_a_batch(ctx):
    """mono, more blocks than one batch holds (2^30 bytes of band dB): a sample of the blocks on both sides of the batch boundary is
    bit-identical to the same blocks decoded one per call, and within the bound of the reference"""
    P = O.Params()
    fpb = O.frames_per_block(P)
    batch = (1 << 30) // (fpb * 1 * 81 * 4)
    mix, order = real_mix(KEY, P)
    n = fpb * N + 4000
    x = T.noise(n / 44100.0 + 1, 1, seed=99)[:n]
    idx = np.arange(batch + 40) * 97 % 4000
    raw, valid = check_blocks(ctx, x, [], mix, order, P.frames_per_bit, fpb, name="batch")
    ctx.pcm_bind(x)
    raw, valid = ctx.decode_blocks(idx, len(order), key_slot=3)
    assert valid.all()
    for k in (0, 1, batch - 2, batch - 1, batch, batch + 1, len(idx) - 1):
        one, v1 = ctx.decode_blocks(idx[k:k + 1], len(order), key_slot=3)
        assert one[0].tobytes() == raw[k].tobytes(), k
    for k in (batch - 1, batch):
        want, bound = decode_ref(x, int(idx[k]), mix, order, P.frames_per_bit, fpb)
        assert (np.abs(raw[k] - want) <= bound).all(), k


def test_reference_matches_oracle():
    """decode_ref against O.raw_bits_for_block (mix and linear): pins the reference, no GPU involved"""
    for P in (O.Params(payload_size=12, payload_short=True), O.Params(payload_size=12, payload_short=True, mix=False)):
        fpb = O.frames_per_block(P)
        x = T.noise((fpb * N + 3000) / 44100.0 + 1, 2, seed=5)
        mix, order = real_mix(KEY, P, linear=not P.mix)
        for i in (0, 1001):
            want = O.raw_bits_for_block(KEY, x, i, P)
            got, bound = decode_ref(x, i, mix, order, P.frames_per_bit, fpb)
            assert np.abs(got - want).max() < 1e-3 * np.abs(want).mean()
            assert (np.abs(got - want) <= bound).all()
