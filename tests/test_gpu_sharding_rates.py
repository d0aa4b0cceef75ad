"""GPU: the sharded get at sample rates other than 44.1 kHz.  Every rank holds only its input range (balanced_input_range),
resamples what its slices need on its own device with awm_resample_range, and the document rank 0 returns equals the single GPU
get at that rate.  Several ranks run in one process on one GPU, the exchanges are simulated in lock step (as in
test_gpu_sharding.py); the range resampler is compared byte for byte with awm_resample of the whole stream."""
import json

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi as C, hostapi as H

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MARK = 44100


def _noise(seconds, rate, channels=2, seed=1):
    rng = np.random.default_rng(seed)
    return ((rng.random((int(seconds * rate), channels), dtype=np.float32) - 0.5)).astype(np.float32)


# ---- the range resampler ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ctx():
    c = C.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("channels", [1, 2, 3])
@pytest.mark.parametrize("ratio", [MARK / 48000, MARK / 32000, MARK / 96000, 2.0])
def test_range_resampler_equals_whole_stream_resampler(ctx, channels, ratio):
    """outputs at the stream start (taps below frame 0), in the middle and over the end (outputs zeroed past the post-roll), read
    from exact windows and from windows that start earlier at odd frames, host and device, 8-byte aligned and at a 4-byte offset"""
    n = 150001
    x = _noise(n / 48000, 48000, channels, seed=channels)[:n]
    n = x.shape[0]
    n_out = H.resample_stream_frames(n, ratio)
    whole = ctx.resample(x, ratio, n_out=n_out)
    assert np.any(whole[n_out // 2])
    flat = torch.zeros(n * channels + 1, dtype=torch.float32, device="cuda")
    flat[1:] = torch.from_numpy(x.reshape(-1)).cuda()              # the stream at a 4-byte offset
    aligned = torch.from_numpy(x).cuda()
    out = torch.empty((n_out + 1) * channels, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ranges = [(0, 300), (0, 1), (n_out // 3, 4097), (n_out // 2 + 1, 1), (n_out - 300, 300), (n_out - 1, 1), (0, n_out)]
    for o0, no in ranges:
        t0, t1 = C.resample_taps(n, ratio, o0, no)
        for w0 in sorted({t0, max(t0 - 1, 0), max(t0 - 7, 0)}):        # exact, and starting at frames of the other parity
            w1 = min(t1 + 3, n)
            want = whole[o0:o0 + no].tobytes()
            ctx.resample_range(np.ascontiguousarray(x[w0:w1]), w0, n, ratio, out.data_ptr(), o0, no)
            ctx.synchronize()
            assert out[:no * channels].cpu().numpy().tobytes() == want, ("host", o0, no, w0)
            for base, off in ((aligned.data_ptr(), 0), (flat.data_ptr(), 4)):
                for o_off in (0, 4):                                    # output 8-byte aligned and at a 4-byte offset
                    ptr = base + off + w0 * channels * 4
                    ctx.resample_range(ptr, w0, n, ratio, out.data_ptr() + o_off, o0, no, in_frames=w1 - w0, channels=channels)
                    ctx.synchronize()
                    got = out.cpu().numpy().tobytes()[o_off:o_off + no * channels * 4]
                    assert got == want, ("device", o0, no, w0, off, o_off)


def test_range_resampler_refuses_before_any_work(ctx):
    n, ratio = 96000, MARK / 48000
    x = _noise(2.0, 48000, 2)
    out = torch.empty(4096 * 2, dtype=torch.float32, device="cuda")
    t0, t1 = C.resample_taps(n, ratio, 1000, 4096)
    before = ctx.launches
    for args in ((x[t0 + 1:t1], t0 + 1, ratio, 1000, 4096), (x[t0:t1 - 1], t0, ratio, 1000, 4096), (x[t0:t1], t0, 100.0, 1000, 4096),
                 (x, 0, ratio, H.resample_stream_frames(n, ratio) - 10, 11)):
        win, w0, r, o0, no = args
        with pytest.raises(C.AwmError):
            ctx.resample_range(np.ascontiguousarray(win), w0, n, r, out.data_ptr(), o0, no)
    with pytest.raises(C.AwmError):                                      # a host output buffer
        ctx.resample_range(np.ascontiguousarray(x[t0:t1]), t0, n, ratio, np.zeros((4096, 2), np.float32), 1000, 4096)
    assert ctx.launches == before


# ---- simulated ranks ------------------------------------------------------------------------------------------------------

def _ranks_doc(y, rate, world):
    """the sharded driver stage by stage, every rank with its own device copy of only its input range -> every rank's document"""
    n = y.shape[0]
    ranks, keep = [], []
    try:
        for r in range(world):
            lo, hi = H.balanced_input_range(n, r, world, rate)
            assert hi > lo and (world == 1 or hi - lo < n)
            part = torch.from_numpy(np.ascontiguousarray(y[lo:hi])).cuda()
            keep.append(part)
            torch.cuda.synchronize()
            ranks.append(H.BalancedStages(r, world, n, part.data_ptr(), hi - lo, y.shape[1], lo, sample_rate=rate))
        pay = [rk.stage(0) for rk in ranks]                          # peaks
        retry = [rk.stage(1, pay) for rk in ranks]                   # select
        assert all(rt == retry[0] for rt in retry)
        if retry[0]:
            pay = [rk.stage(2, [retry[0]]) for rk in ranks]
            assert all(rk.stage(1, pay) == b"" for rk in ranks)
        pay = [rk.stage(3) for rk in ranks]                          # refine + soft bits
        pay = [rk.stage(4, pay) for rk in ranks]                     # viterbi
        return [json.loads(rk.stage(5, pay).decode()) for rk in ranks]
    finally:
        for rk in ranks:
            rk.close()


@pytest.fixture(scope="module")
def marked48():
    """700 s of stereo noise at 48 kHz, watermarked at 48 kHz with 4 minute chunks (four chunks at the watermark rate)"""
    H.set_params(chunk_size_min=4.0)
    y = H.add(_noise(700.0, 48000, 2, seed=41), T.PAYLOAD, sample_rate=48000)
    doc = H.get(y, sample_rate=48000)
    H.set_params()
    assert sum(m["bits"] == T.PAYLOAD for m in doc["matches"]) >= 3
    return y, doc


@pytest.mark.parametrize("world", [1, 2, 3])
def test_sharded_get_at_48k_equals_single_gpu(marked48, world):
    y, doc = marked48
    H.set_params(chunk_size_min=4.0)
    try:
        assert len(H.balanced_plan(y.shape[0], 0, 1, sample_rate=48000)[0]) >= 3
        assert all(d == doc for d in _ranks_doc(y, 48000, world))
    finally:
        H.set_params()


@pytest.mark.parametrize("rate", [32000, 96000])
def test_sharded_get_at_other_rates_equals_single_gpu(rate):
    H.set_params(chunk_size_min=4.0)
    try:
        y = H.add(_noise(700.0, rate, 2, seed=rate), T.PAYLOAD, sample_rate=rate)
        doc = H.get(y, sample_rate=rate)
        assert sum(m["bits"] == T.PAYLOAD for m in doc["matches"]) >= 3
        assert all(d == doc for d in _ranks_doc(y, rate, 3))
    finally:
        H.set_params()


def test_sharded_get_at_48k_with_short_payload():
    H.set_params(chunk_size_min=4.0)
    H.set_short_payload(16)
    try:
        y = H.add(_noise(500.0, 48000, 2, seed=43), "beef", sample_rate=48000)
        doc = H.get(y, sample_rate=48000)
        assert sum(m["bits"] == "beef" for m in doc["matches"]) >= 3
        assert all(d == doc for d in _ranks_doc(y, 48000, 3))
    finally:
        H.set_short_payload(0)
        H.set_params()


# ---- the single-rank entry point --------------------------------------------------------------------------------------------

def test_balanced_get_at_48k_single_rank(marked48):
    """balanced_get without a communicator is a world of one: float host, float device and 16 bit host input at 48 kHz give the
    single GPU get's document"""
    y, doc = marked48
    H.set_params(chunk_size_min=4.0)
    try:
        n = y.shape[0]
        assert H.balanced_get(y, 0, n, sample_rate=48000) == doc
        yd = torch.from_numpy(y).cuda()
        torch.cuda.synchronize()
        assert H.balanced_get(yd.data_ptr(), 0, n, n_frames=n, channels=2, sample_rate=48000) == doc
        y16 = O.quantize_sndfile16(y)
        want16 = H.get_s16(y16, sample_rate=48000)
        assert sum(m["bits"] == T.PAYLOAD for m in want16["matches"]) >= 3
        assert H.balanced_get(y16, 0, n, sample_rate=48000) == want16
    finally:
        H.set_params()


# ---- refusals ---------------------------------------------------------------------------------------------------------------

def test_sharded_get_refusals(marked48):
    """a rank buffer one frame short of its input range, clip-sized 48 kHz input and a rate outside the resampler's range are
    refused before any kernel runs"""
    y, _ = marked48
    n = y.shape[0]
    H.set_params(chunk_size_min=4.0)
    ctx = C.Context.from_handle(H.engine_ctx())
    try:
        lo, hi = H.balanced_input_range(n, 1, 3, 48000)
        part = torch.from_numpy(np.ascontiguousarray(y[lo:hi])).cuda()
        torch.cuda.synchronize()
        before = ctx.launches
        with pytest.raises(RuntimeError):
            H.BalancedStages(1, 3, n, part.data_ptr() + 2 * 4, hi - lo - 1, 2, lo + 1, sample_rate=48000)   # first frame missing
        with pytest.raises(RuntimeError):
            H.BalancedStages(1, 3, n, part.data_ptr(), hi - lo - 1, 2, lo, sample_rate=48000)               # last frame missing
        clip = np.ascontiguousarray(y[:100 * 48000])
        with pytest.raises(RuntimeError):
            H.balanced_get(clip, 0, clip.shape[0], sample_rate=48000)
        with pytest.raises(RuntimeError):
            H.balanced_get(y, 0, n, sample_rate=600)                                                       # 44100 / 600 > 64
        assert ctx.launches == before
        rk = H.BalancedStages(1, 3, n, part.data_ptr(), hi - lo, 2, lo, sample_rate=48000)                 # the exact range is enough
        rk.close()
    finally:
        H.set_params()
