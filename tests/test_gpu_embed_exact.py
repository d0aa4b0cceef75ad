"""GPU: single `add` at 44.1 kHz (hostapi.add / add_s16 / add_windowed -> awm_embed, awm_embed_s16, awm_embed_window) against
tests/golden/embed_exact.json (tests/golden/make_embed_exact.py, whose run_case this test shares): for every case, with and without
the limiter, the output bytes and the Data Blocks count exactly and snr_db to 1e-12 relative (its sums use double atomics).
Stereo, mono and 3 channels, lengths from zero frames to 5 minutes (the pipelined host path), float and 16 bit host buffers,
device buffers on both embed kernels, shards, windows at stream offsets, full-scale input that engages the limiter, and payloads
that alternate within one process."""
import importlib.util
import json
import math
import os

import pytest

from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
G = json.load(open(os.path.join(GOLDEN, "embed_exact.json")))["cases"]
_spec = importlib.util.spec_from_file_location("make_embed_exact", os.path.join(GOLDEN, "make_embed_exact.py"))
M = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(M)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def test_cases_cover_the_grid():
    assert G.keys() == M.cases().keys()
    assert {c["kind"] for c in G.values()} == {"add", "add_s16", "add_device", "add_windowed"}
    assert {c["channels"] for c in G.values()} == {1, 2, 3}
    assert {0, 1, 1023, 1025} <= {c["frames"] for c in G.values()}
    assert any(c["kind"] == "add" and c["frames"] > 2 * 6144 * 1024 for c in G.values())
    assert {c.get("shift") for c in G.values() if c["kind"] == "add_device"} == {0, 1}
    assert any(c.get("first_frame_number") for c in G.values()) and any(c.get("zero_frames") for c in G.values())
    loud = [c for c in G.values() if c["amp"] == 1.0]
    assert loud and all(c["runs"]["limiter"][0]["output_sha256"] != c["runs"]["nolimiter"][0]["output_sha256"] for c in loud)
    assert any(len(c["payloads"]) == 3 and c["payloads"][0] != c["payloads"][1] for c in G.values())


@pytest.mark.parametrize("name", sorted(G))
def test_single_add_matches_golden(name):
    if G[name]["kind"] == "add_device":
        pytest.importorskip("torch")
    c = G[name]
    for run in ("limiter", "nolimiter"):
        H.set_params(test_no_limiter=run == "nolimiter")
        for bits, want in zip(c["payloads"], c["runs"][run]):
            h, blocks, snr = M.run_case(c, bits)
            assert h == want["output_sha256"], (name, run, bits)
            assert blocks == want["data_blocks"], (name, run, bits, blocks)
            if want["snr_db"] is None:
                assert snr is None, (name, run, bits, snr)
            else:
                assert abs(snr - want["snr_db"]) <= 1e-12 * abs(want["snr_db"]), (name, run, bits, snr, want["snr_db"])
