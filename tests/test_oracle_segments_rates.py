"""CPU: pins the meaning of a stream offset at other sample rates to the reference.  tests/golden/golden_segments_rates.json holds
what the unmodified reference's `audiowmark add` writes for the whole stream zeros (z) ++ x at 32 and 48 kHz, cut to x's positions
(tests/golden/make_golden_segments_rates.py).  The oracle's embed of that stream must give the same 16 bit output, Data Blocks and
SNR line: that is the contract of add_batch_rates(zero_frames = [...]), which tests/test_gpu_batch_rates_offsets.py holds against this
oracle computation."""
import hashlib
import json
import os

import numpy as np
import pytest

import awm_oracle as O

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_segments_rates.json")))


def case_input(g):
    """the case's input as 16 bit PCM, as make_golden_segments_rates.py wrote it"""
    rng = np.random.default_rng(g["seed"])
    x = ((rng.random((int(g["seconds"] * g["rate"]), g["channels"]), dtype=np.float32) - 0.5) * (2 * g["amp"])).astype(np.float32)
    return O.quantize_sndfile16(x)


def oracle_whole(g, x):
    """oracle `add` of the whole stream zeros (z) ++ x at the case's rate -> (result, the part at x's positions)"""
    z = g["zero_frames"]
    P = O.Params(test_no_limiter="--test-no-limiter" in g["add_args"])
    ext = np.concatenate([np.zeros((z, x.shape[1]), np.float32), O.int16_to_float(x)])
    r = O.embed(ext, O.Key(), G["payload"], P, g["rate"])
    return r, r.samples[z:]


def sha16(x16):
    return hashlib.sha256(np.ascontiguousarray(x16).tobytes()).hexdigest()


@pytest.mark.parametrize("name", sorted(G["cases"]))
def test_whole_stream_embed_equals_reference(name):
    g = G["cases"][name]
    x = case_input(g)
    assert sha16(x) == g["input_sha256"]
    r, y = oracle_whole(g, x)
    assert sha16(O.quantize_sndfile16(y)) == g["output_sha256"], name
    assert r.data_blocks == g["data_blocks"]
    # the printed SNR line; without the limiter the oracle's --snr sums end 5e-5 dB off the reference loop's
    assert abs(r.snr_db - g["snr_db"]) < 1e-4, (name, r.snr_db, g["snr_db"])


def test_golden_covers_the_cases_that_matter():
    cases = list(G["cases"].values())
    for rate in (32000, 48000):
        zs = {g["zero_frames"] for g in cases if g["rate"] == rate}
        assert {0, 1023, 1024 + 517, 50 * 1024 + 517, 57 * rate} <= zs      # 57 s: HLS segment 10's start_pos - prev_size
        assert {g["channels"] for g in cases if g["rate"] == rate} == {1, 2}
        assert any(g["amp"] >= 1.0 for g in cases if g["rate"] == rate)    # limiter engaged
        assert any("--test-no-limiter" in g["add_args"] and g["zero_frames"] < 1024 + 2 * rate for g in cases if g["rate"] == rate)
