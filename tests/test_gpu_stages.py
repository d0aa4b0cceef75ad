"""GPU parity, stage by stage: every C-ABI entry point against the CPU oracle on the same
seeded input.  Tables come from the oracle so that only the kernels are under test here.

Tolerances (floating point; integer results are compared exactly):
  FFT           1e-6 relative to the spectrum maximum
  embed         RMS(out_gpu - out_oracle) < 1e-5         (north star)
  sync quality  |dq| < 2e-4 (quality is ~1 for a real sync, ~0.05 noise floor)
  refine index  within 8 samples (one sync_search_fine step; SURVEY H1), quality 1e-3
  soft bits     1e-3 relative to mean |soft bit|
  Viterbi       decoded bits identical, error metric 1e-5
"""
import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi

pytestmark = pytest.mark.gpu

P = O.Params()
KEY = O.Key()


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    T.setup_ctx(c, KEY, P, T.PAYLOAD)
    yield c
    c.close()


@pytest.fixture(scope="module")
def marked():
    """115 s stereo noise watermarked by the ORACLE (limiter on): contains one full A block."""
    x = T.noise(115.0)
    return x, O.embed(x, KEY, T.PAYLOAD, P).samples


def test_fft_roundtrip_and_numpy(ctx):
    rng = np.random.default_rng(0)
    for count in (1, 2, 7, 64):
        x = rng.standard_normal((count, 1024)).astype(np.float32)
        X = ctx.fft_r2c(x)
        ref = np.fft.rfft(x.astype(np.float64), axis=1)
        assert np.abs(X - ref).max() < 1e-6 * np.abs(ref).max() * 4
        back = ctx.fft_c2r(X)
        assert np.abs(back / 1024 - x).max() < 2e-6 * np.abs(x).max() * 4
        # unnormalised c2r of an arbitrary Hermitian spectrum (FFTW semantics)
        S = (rng.standard_normal((count, 513)) + 1j * rng.standard_normal((count, 513))).astype(np.complex64)
        S[:, 0] = S[:, 0].real
        S[:, 512] = S[:, 512].real
        y = ctx.fft_c2r(S)
        yr = np.fft.irfft(S.astype(np.complex128), n=1024, axis=1) * 1024
        assert np.abs(y - yr).max() < 1e-6 * np.abs(yr).max() * 4


@pytest.mark.parametrize("limiter", [True, False])
@pytest.mark.parametrize("seconds,channels", [(12.0, 2), (3.3, 1), (2.0, 3), (0.01, 2)])
def test_embed_vs_oracle(ctx, limiter, seconds, channels):
    x = T.noise(seconds, channels, seed=7, amp=1.0 if limiter else 0.5)
    Pl = O.Params(test_no_limiter=not limiter)
    ref = O.embed(x, KEY, T.PAYLOAD, Pl, keep_wm=True)
    out, (dpow, spow) = ctx.embed(x, limiter_block=44100 if limiter else 0, want_snr=True)
    assert out.shape == x.shape
    d = T.rms(out - ref.samples)
    assert d < 1e-5, d
    assert np.abs(out - ref.samples).max() < 1e-4
    if ref.wm is not None and seconds > 1:
        assert T.rms(ref.wm) > 1e-4          # a watermark was actually added
        snr = 10 * np.log10(spow / dpow)
        assert abs(snr - ref.snr_db) < 1e-3


@pytest.mark.parametrize("seconds,limiter", [(20.0, True), (3.3, False), (0.01, True)])
def test_embed_strip_kernel_equals_tile_kernel(ctx, seconds, limiter):
    """k_embed_strip (streaming, TMA-fed, neighbours' window tails carried in registers) and k_embed (CTA tiles with a halo frame on
    each side) run the same arithmetic in the same order: identical bits, identical limiter peaks, for whole and ragged lengths.
    The same stereo samples on the device take k_embed_strip from a 16-byte aligned start and k_embed from one stereo frame further."""
    torch = pytest.importorskip("torch")
    x = T.noise(seconds, 2, seed=21, amp=1.0 if limiter else 0.5)
    aligned = torch.from_numpy(x).cuda()
    shifted = torch.empty((x.shape[0] + 1, 2), dtype=torch.float32, device="cuda")[1:]
    shifted.copy_(aligned)
    assert aligned.data_ptr() % 16 == 0 and shifted.data_ptr() % 16 == 8
    out = [torch.empty_like(aligned) for _ in range(2)]
    torch.cuda.synchronize()
    _, strip_snr = ctx.embed(aligned.data_ptr(), out[0].data_ptr(), n_frames=x.shape[0], channels=2,
                             limiter_block=44100 if limiter else 0, want_snr=True)
    _, tile_snr = ctx.embed(shifted.data_ptr(), out[1].data_ptr(), n_frames=x.shape[0], channels=2,
                            limiter_block=44100 if limiter else 0, want_snr=True)
    ctx.synchronize()
    strip, tile = (o.cpu().numpy() for o in out)
    bad = np.nonzero((tile != strip).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:8], float(np.abs(tile - strip).max()), tile[bad[:3]], strip[bad[:3]])
    assert np.allclose(tile_snr, strip_snr, rtol=1e-12)


def test_embed_device_pointers_match_host_path(ctx):
    torch = pytest.importorskip("torch")
    x = T.noise(5.0, 2, seed=3)
    host = ctx.embed(x)
    xin = torch.from_numpy(x).cuda()
    xout = torch.empty_like(xin)
    torch.cuda.synchronize()
    ctx.embed(xin.data_ptr(), xout.data_ptr(), n_frames=x.shape[0], channels=2)
    ctx.synchronize()
    assert np.array_equal(xout.cpu().numpy(), host)


def test_sync_approx_vs_oracle(ctx, marked):
    _, y = marked
    ctx.pcm_bind(y)
    got = ctx.sync_approx(0, capi.MODE_BLOCK)
    sf = O.SyncFinder(P)
    sf.first, sf.last = 0, y.size
    want = sf.search_approx(O.get_sync_bits(KEY, O.BLOCK, P), y, O.BLOCK)
    assert len(got) == len(want) > 0
    assert np.array_equal(got["index"], np.array([s.index for s in want], np.uint64))
    dq = np.abs(got["raw_quality"] - np.array([s.raw_quality for s in want]))
    dm = np.abs(got["local_mean"] - np.array([s.local_mean for s in want]))
    assert dq.max() < 2e-4 and dm.max() < 2e-4, (dq.max(), dm.max())
    # the embedded block is found where the reference puts it: first A block at sample 256000
    best = got[np.argmax(np.abs(got["raw_quality"] - got["local_mean"]))]
    assert best["index"] == 256000 and best["raw_quality"] > 1.0


def test_tensor_core_entry_sums_match_fp32_pipes(ctx, marked, monkeypatch):
    """k_stft_mags_tc (wgmma on fp16 hi/lo terms of the dB values, fp32 accumulation, masks by TMA) against k_stft_mags
    (the same sums on the fp32 pipes): the two differ only by the rounding of the additions -- far below the 2e-4 bar against the
    oracle that test_sync_approx_vs_oracle holds the default path to.  Both ways the FFT warps read PCM are run: a device buffer
    bound in place one stereo frame past a 16-byte boundary (global loads), then PCM bound from the host (TMA bulk copies)."""
    torch = pytest.importorskip("torch")
    _, y = marked
    y = np.ascontiguousarray(y, np.float32)
    shifted = torch.empty((y.shape[0] + 1, 2), dtype=torch.float32, device="cuda")[1:]
    shifted.copy_(torch.from_numpy(y))
    assert shifted.data_ptr() % 16 == 8
    torch.cuda.synchronize()
    for path, bind in (("ldg", lambda: ctx.pcm_bind(shifted.data_ptr(), n_frames=y.shape[0], channels=2)),
                       ("tma", lambda: ctx.pcm_bind(y))):
        bind()
        monkeypatch.setenv("AWM_APPROX", "simt")
        simt = ctx.sync_approx(0, capi.MODE_BLOCK)
        monkeypatch.delenv("AWM_APPROX")
        tc = ctx.sync_approx(0, capi.MODE_BLOCK)
        assert len(tc) == len(simt) > 0
        assert np.array_equal(tc["index"], simt["index"])
        d = np.abs(tc["raw_quality"] - simt["raw_quality"]).max()
        assert d < 2e-5, (path, d)
        assert np.abs(tc["local_mean"] - simt["local_mean"]).max() < 2e-5, path


def test_sync_refine_vs_oracle(ctx, marked):
    """stereo, mono and three channels (stereo plus their mean): stereo and mono take the sliding pass, three channels score every
    offset exactly"""
    _, y2 = marked
    for y in (y2, y2[:, :1], np.stack([y2[:, 0], y2[:, 1], 0.5 * (y2[:, 0] + y2[:, 1])], axis=1)):
        refine_vs_oracle(ctx, np.ascontiguousarray(y, np.float32))


def refine_vs_oracle(ctx, y):
    channels = y.shape[1]
    ctx.pcm_bind(y)
    sf = O.SyncFinder(P)
    sf.first, sf.last = 0, y.size
    sb = O.get_sync_bits(KEY, O.BLOCK, P)
    approx = sf.search_approx(sb, y, O.BLOCK)
    sel = sf.select_threshold_and_n_best(sf.mask_avg_false_positives(sf.select_local_maxima(approx)), P.sync_threshold2 * 0.75)
    # include a candidate near the start (index < 256) and one whose window runs past the end
    sel = sel + [O.SearchScore(128, 0.01, 0.0), O.SearchScore(approx[-1].index, approx[-1].raw_quality, approx[-1].local_mean)]
    want = sf.search_refine(y, O.BLOCK, sel, sb, KEY)
    inp = np.zeros(len(sel), capi.SEARCH_SCORE)
    inp["index"] = [s.index for s in sel]
    inp["raw_quality"] = [s.raw_quality for s in sel]
    inp["local_mean"] = [s.local_mean for s in sel]
    got = np.sort(ctx.sync_refine(inp, 0, capi.MODE_BLOCK), order="index")
    assert len(got) == len(want), channels
    for g, w in zip(got, want):
        assert int(g["index"]) == w.index, (channels, g, w)     # sync positions are exact, not "within one fine step"
        assert abs(g["raw_quality"] - w.raw_quality) < 2e-4, (channels, g, w)
        assert g["local_mean"] == w.local_mean
    # error bound behind the exactness claim (awm_capi.cu: kVerifyMargin = 1e-3): the sliding-DFT ranking S and the exact scores E
    # of all 65 offsets differ by less than half the margin, so the exact arg-max is always among the re-scored offsets
    S, vs = ctx.sync_refine_offsets(inp, exact=False)
    E, ve = ctx.sync_refine_offsets(inp, exact=True)
    assert np.array_equal(vs, ve) and vs.sum() > 60 * (len(sel) - 2), channels
    assert np.abs(S - E)[vs].max() < 5e-4 * 0.5, (channels, np.abs(S - E)[vs].max())
    # the result is the exact kernel's: the reference rule (start from the approx index, replace on strictly larger |q - mean|,
    # offsets ascending) applied to E alone gives the indices awm_sync_refine returns
    unsorted = ctx.sync_refine(inp, 0, capi.MODE_BLOCK)
    for k, (i, m) in enumerate(zip(inp["index"], inp["local_mean"])):
        start = max(int(i) - 256, 0)
        o_self = (int(i) - start) // 8
        if not ve[k][o_self]:
            continue
        best_o, best_v = o_self, abs(E[k][o_self] - m)
        for o in range(65):
            if ve[k][o] and abs(E[k][o] - m) > best_v:
                best_o, best_v = o, abs(E[k][o] - m)
        assert int(unsorted[k]["index"]) == start + 8 * best_o, (channels, k, int(unsorted[k]["index"]), start + 8 * best_o)
        assert abs(abs(unsorted[k]["raw_quality"] - m) - best_v) < 1e-12, (channels, k)
    # the exact per-offset qualities are the reference's sync_decode (sync_fft (fine)) on every offset of the best candidates and of
    # the one whose window runs past the end
    d = []
    for k in (0, 1, 2, len(sel) - 1):
        for o, (fine, q) in enumerate(sf.refine_qualities(y, O.BLOCK, sel[k].index, sb, KEY)):
            assert ve[k][o] == (q is not None), (channels, k, o)
            if q is not None:
                d.append(abs(E[k][o] - q))
    assert len(d) > 3 * 65 and max(d) < 2e-4, (channels, max(d))
    print("channels %d: max |E - oracle| over %d offsets = %.3g" % (channels, len(d), max(d)))


def test_decode_blocks_vs_oracle(ctx, marked):
    _, y = marked
    ctx.pcm_bind(y)
    n_coded = O.conv_code_size(O.A, P.payload_size)
    idx = [256000, 256008, 100, y.shape[0] - 100]
    raw, valid = ctx.decode_blocks(idx, n_coded)
    assert list(valid) == [1, 1, 1, 0]
    for i in range(3):
        want = O.raw_bits_for_block(KEY, y, idx[i], P)
        scale = np.abs(want).mean()
        assert np.abs(raw[i] - want).max() < 1e-3 * scale, i
    # and the payload comes out
    bits, err = ctx.viterbi(raw[:1], [capi.BLOCK_A])
    assert O.bit_vec_to_str(list(bits[0])) == T.PAYLOAD


def test_viterbi_vs_oracle(ctx):
    """k_viterbi (one CTA per code word) against the oracle: identical bits, error within 1e-5"""
    rng = np.random.default_rng(5)
    msg = [int(b) for b in rng.integers(0, 2, 128)]
    for bt, cbt in ((O.A, capi.BLOCK_A), (O.B, capi.BLOCK_B), (O.AB, capi.BLOCK_AB)):
        coded = np.array(O.conv_encode(bt, msg), np.float32)
        jobs = []
        for noise in (0.0, 0.6, 1.5, 4.0):
            jobs.append(((coded * 2 - 1) + noise * rng.standard_normal(len(coded))).astype(np.float32))
        bits, err = ctx.viterbi(jobs, [cbt] * len(jobs))
        hbits, herr = ctx.viterbi(jobs, [cbt] * len(jobs), hard=True)
        for j in range(len(jobs)):
            wb, we = O.conv_decode_soft(bt, O.normalize_soft_bits(jobs[j], P))
            assert list(bits[j]) == wb, (bt, j)
            assert abs(err[j] - we) < 1e-5 * max(1.0, we)
            Ph = O.Params(hard=True)
            wb, we = O.conv_decode_soft(bt, O.normalize_soft_bits(jobs[j], Ph))
            assert list(hbits[j]) == wb
        assert list(bits[0]) == msg


def test_clip_mode_approx_with_silence(ctx):
    """CLIP tables + zero padding: frames in digital silence are skipped (have = 0) like sync_fft :583-588."""
    x = T.noise(20.0, 2, seed=11)
    y = O.embed(x, KEY, T.PAYLOAD, P).samples
    fpb = O.frames_per_block(P)
    npad = (fpb + 5) * 1024
    pad_start = npad + (npad - y.shape[0])
    ctx.pcm_bind(y, pad_start=pad_start, pad_end=npad)
    ext = np.concatenate([np.zeros((pad_start, 2), np.float32), y, np.zeros((npad, 2), np.float32)])
    flat = ext.reshape(-1)
    nz = np.nonzero(flat)[0]
    first, last = int(nz[0]), int(nz[-1]) + 1
    got = ctx.sync_approx(0, capi.MODE_CLIP, first, last)
    sf = O.SyncFinder(P)
    sf.first, sf.last = first, last
    want = sf.search_approx(O.get_sync_bits(KEY, O.CLIP, P), ext, O.CLIP)
    assert len(got) == len(want) > 0
    dq = np.abs(got["raw_quality"] - np.array([s.raw_quality for s in want]))
    assert dq.max() < 2e-4, dq.max()
