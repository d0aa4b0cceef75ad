"""The sliding pass of the sync refine (k_refine_slide) only ranks the 65 fine offsets of a candidate; the offsets within 1e-3 of the
best sliding score are scored again exactly.  So its sums must stay within a quarter of that margin of the exact per-offset sums,
on every offset, and the offsets it hands to the exact re-score must contain the exact arg-max.  Stereo and mono input, candidates
whose last offsets run past the end of the buffer (fewer than 65 valid offsets), and candidates whose sync frames border digital
silence (frames wholly inside the silence are not counted, so the counts change from one offset to the next)."""
import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi

pytestmark = pytest.mark.gpu

P = O.Params()
KEY = O.Key()
MARGIN = 1e-3
SILENT = 5 * 44100                      # frames of digital silence at the start of the silence input


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    T.setup_ctx(c, KEY, P, T.PAYLOAD)
    yield c
    c.close()


@pytest.fixture(scope="module")
def marked():
    """60 s stereo noise watermarked by the oracle"""
    return O.embed(T.noise(60.0, seed=77), KEY, T.PAYLOAD, P).samples.astype(np.float32)


def candidates(ctx, y, extra=()):
    """the approx search's best scores, every 40th score, a candidate near the start and the last ones (window past the end)"""
    sc = ctx.sync_approx(0, capi.MODE_BLOCK)
    q = np.abs(sc["raw_quality"] - sc["local_mean"])
    pick = sorted(set(np.argsort(q)[-24:]) | set(range(0, len(sc), 40)) | set(range(len(sc) - 3, len(sc))))
    out = np.zeros(len(pick) + 1 + len(extra), capi.SEARCH_SCORE)
    out[:len(pick)] = sc[pick]
    out[len(pick)] = (128, 0.01, 0.0)
    for i, idx in enumerate(extra):
        out[len(pick) + 1 + i] = (idx, 0.01, 0.0)
    return out


def check(ctx, inp, **kw):
    S, vs = ctx.sync_refine_offsets(inp, exact=False, **kw)
    E, ve = ctx.sync_refine_offsets(inp, exact=True, **kw)
    assert np.array_equal(vs, ve)
    d = np.abs(S - E)[vs].max()
    assert d < MARGIN / 4, d
    kept = ctx.sync_refine_rescored(inp, **kw)
    for k, (i, m) in enumerate(zip(inp["index"], inp["local_mean"])):
        if not ve[k].any():
            continue
        o_best = max(np.nonzero(ve[k])[0], key=lambda o: abs(E[k][o] - m))
        assert kept[k][o_best], (k, o_best)
    return vs


def test_sliding_sums_stereo(ctx, marked):
    ctx.pcm_bind(marked)
    vs = check(ctx, candidates(ctx, marked))
    n_valid = vs.sum(axis=1)
    assert (n_valid == 65).sum() > 30 and ((n_valid > 0) & (n_valid < 65)).any()


def test_sliding_sums_mono(ctx, marked):
    y = np.ascontiguousarray(marked[:, :1])
    ctx.pcm_bind(y)
    check(ctx, candidates(ctx, y))


def test_sliding_sums_border_digital_silence(ctx, marked):
    """sync frames that start inside the silence and end after it: counted from the offset on which they reach the first sample"""
    y = marked.copy()
    y[:SILENT] = 0
    nz = np.nonzero(y.reshape(-1))[0]
    kw = dict(wav_first=int(nz[0]), wav_last=int(nz[-1]))
    ctx.pcm_bind(y)
    extra = [SILENT - 1024 * k - 100 for k in range(40)]         # frame k of the block crosses the border
    inp = candidates(ctx, y, extra)
    check(ctx, inp, **kw)
    # the counts really change across the offsets of the border candidates: their sliding qualities differ from the ones with
    # every frame counted by far more than the margin on some offsets
    S, vs = ctx.sync_refine_offsets(inp[-len(extra):], exact=False, **kw)
    A, va = ctx.sync_refine_offsets(inp[-len(extra):], exact=False)
    assert np.array_equal(vs, va) and (np.abs(S - A)[vs] > MARGIN).any()
