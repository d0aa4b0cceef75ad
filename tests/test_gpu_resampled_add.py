"""GPU: single `add` at sample rates other than 44.1 kHz (hostapi.add -> add_watermark_buffer -> the batched resampled embed) against
tests/golden/resampled_add.json (tests/golden/make_resampled_add.py): for every case, with and without the limiter, from host and from
device buffers, the output bytes and the Data Blocks count exactly and snr_db to 1e-12 relative (its sums use double atomics).
Six rates from 8 to 192 kHz, 1 to 3 channels, lengths from zero frames to 10 minutes, full-scale input that engages the limiter."""
import hashlib
import json
import math
import os

import numpy as np
import pytest

from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resampled_add.json")))["cases"]


def noise(frames, channels, seed, amp):
    """make_resampled_add.py's input"""
    rng = np.random.default_rng(seed)
    return ((rng.random((frames, channels), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def test_cases_cover_the_grid():
    assert {c["rate"] for c in G.values()} == {8000, 22050, 32000, 48000, 96000, 192000}
    assert {c["channels"] for c in G.values()} == {1, 2, 3}
    assert {0, 1, 1023, 1025} <= {c["frames"] for c in G.values()} and max(c["frames"] for c in G.values()) >= 600 * 48000
    assert any(c["amp"] == 1.0 for c in G.values())


@pytest.mark.parametrize("name", sorted(G))
def test_single_add_matches_golden(name):
    torch = pytest.importorskip("torch")
    c = G[name]
    x = noise(c["frames"], c["channels"], c["seed"], c["amp"])
    for run, want in sorted(c["runs"].items()):
        H.set_params(test_no_limiter=run.startswith("nolimiter"))
        if run.endswith("device"):
            xd = torch.from_numpy(x).cuda()
            yd = torch.empty_like(xd)
            _, blocks, snr = H.add(xd.data_ptr(), c["payload"], pcm_out=yd.data_ptr(), n_frames=x.shape[0], channels=x.shape[1],
                                   sample_rate=c["rate"], want_stats=True)
            y = yd.cpu().numpy()
        else:
            y, blocks, snr = H.add(x, c["payload"], sample_rate=c["rate"], want_stats=True)
        assert hashlib.sha256(y.tobytes()).hexdigest() == want["output_sha256"], (name, run)
        assert blocks == want["data_blocks"], (name, run, blocks)
        if want["snr_db"] is None:
            assert math.isinf(snr), (name, run, snr)
        else:
            assert abs(snr - want["snr_db"]) <= 1e-12 * abs(want["snr_db"]), (name, run, snr, want["snr_db"])
        if c["amp"] == 1.0:         # full scale: the limiter holds the ceiling, without it the watermark clips past it
            assert (np.abs(y).max() <= 0.99 + 1e-6) != run.startswith("nolimiter"), (name, run)
