"""The offsets awm_sync_refine scores again exactly are picked on the device (k_refine_rank).  They must be the ones the host rule
picks from the same sliding qualities: every valid offset whose -|q - local_mean| lies within 1e-3 of the smallest, plus the
offset of the approx index if it is valid.  Candidates: the golden selection of test_gpu_stages.py::test_sync_refine_vs_oracle (with
a candidate near the start and one past the end) and every local maximum of the approx scores."""
import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi

pytestmark = pytest.mark.gpu

P = O.Params()
KEY = O.Key()
MARGIN = 1e-3


def host_rule(scores, S, valid):
    keep = np.zeros(valid.shape, bool)
    for k, (i, m) in enumerate(zip(scores["index"], scores["local_mean"])):
        start = max(int(i) - 256, 0)
        keys = {o: -abs(S[k][o] - m) for o in range(65) if valid[k][o]}
        if keys:
            best = min(keys.values())
            for o, v in keys.items():
                keep[k][o] = v <= best + MARGIN
        o_self = (int(i) - start) // 8
        if valid[k][o_self]:
            keep[k][o_self] = True
    return keep


def test_device_ranking_equals_host_rule():
    c = capi.Context(0)
    try:
        T.setup_ctx(c, KEY, P, T.PAYLOAD)
        y = O.embed(T.noise(115.0), KEY, T.PAYLOAD, P).samples
        c.pcm_bind(y)
        sf = O.SyncFinder(P)
        sf.first, sf.last = 0, y.size
        approx = sf.search_approx(O.get_sync_bits(KEY, O.BLOCK, P), y, O.BLOCK)
        maxima = sf.select_local_maxima(approx)
        sel = sf.select_threshold_and_n_best(sf.mask_avg_false_positives(maxima), P.sync_threshold2 * 0.75)
        sel = sel + [O.SearchScore(128, 0.01, 0.0), O.SearchScore(approx[-1].index, approx[-1].raw_quality, approx[-1].local_mean)] + list(maxima)
        inp = np.zeros(len(sel), capi.SEARCH_SCORE)
        inp["index"] = [s.index for s in sel]
        inp["raw_quality"] = [s.raw_quality for s in sel]
        inp["local_mean"] = [s.local_mean for s in sel]
        S, valid = c.sync_refine_offsets(inp, exact=False)
        want = host_rule(inp, S, valid)
        got = c.sync_refine_rescored(inp)
        bad = np.nonzero((got != want).any(axis=1))[0]
        assert len(bad) == 0, (len(bad), bad[:5])
        assert want.sum() >= len(sel) - 1 and len(sel) > 100
    finally:
        c.close()
