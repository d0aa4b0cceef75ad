"""GPU: the sync refine on 1, 2, 3 and 6 channels against tests/golden/refine_exact.json (tests/golden/make_refine_exact.py), bit for
bit: per-offset exact and sliding qualities and valid flags, refined indices and qualities, the offsets picked for the exact re-score,
and the `get` document and sync positions of 150 s on 3 and 6 channels and of a 30 s 3 channel clip (clip decoder).
BLOCK cases start with digital silence, CLIP cases are zero padded; their candidates include windows past the end and sync frames
that border the silence."""
import json
import os
import sys

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLDEN)
import make_refine_exact as M  # noqa: E402

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(GOLDEN, "refine_exact.json")))


@pytest.fixture(scope="module")
def ctx():
    c = M.setup()
    yield c
    c.close()


def test_cases_cover_the_channel_counts():
    assert {c["channels"] for c in G["refine"].values()} == {1, 2, 3, 6}
    assert {c["mode"] for c in G["refine"].values()} == {"BLOCK", "CLIP"}
    assert {c["channels"] for c in G["get"].values()} == {3, 6}


@pytest.mark.parametrize("name", sorted(G["refine"]))
def test_refine_matches_golden(ctx, name):
    want = G["refine"][name]
    got = M.refine_case(ctx, want["channels"], want["mode"], want["seconds"], want["seed"])
    assert got["input_sha256"] == want["input_sha256"], name
    for k, v in got.items():
        assert v == want[k], (name, k)
    assert set(got) == set(want) - {"channels", "mode", "seconds", "seed"}


def test_rescored_on_three_channels_flags_every_valid_offset(ctx):
    """more than two channels have no sliding pass: every valid offset is scored exactly, and the caller's scores stay as they were"""
    want = G["refine"]["c3_block"]
    y, m, first, last, cand = M.refine_input(ctx, 3, "BLOCK", want["seconds"], want["seed"])
    kw = dict(mode=m, wav_first=first, wav_last=last)
    before = cand.copy()
    rescored = ctx.sync_refine_rescored(cand, **kw)
    assert np.array_equal(cand, before)
    _, valid = ctx.sync_refine_offsets(cand, exact=True, **kw)
    assert valid.any() and np.array_equal(rescored, valid)


@pytest.mark.parametrize("name", sorted(G["get"]))
def test_get_matches_golden(name):
    want = G["get"][name]
    got = M.get_case(want["channels"], want["seconds"], want["seed"], want["clip_start"])
    assert got["input_sha256"] == want["input_sha256"], name
    assert got["json"] == want["json"], name
    assert got["sync"] == want["sync"], name
