"""CPU: pins the meaning of a stream offset to the reference.  tests/golden/golden_segments.json holds what the unmodified
reference's add_stream_watermark (src/wmadd.cc:448-618) writes for an input that continues a stream begun zero_frames earlier with
silence, as hls-add calls it (oracle/_ref/add_at, tests/golden/make_golden_segments.py).  The oracle's embed of zeros (z) ++ x
with the first z frames dropped must give the same 16 bit output: that is the contract of add_windowed (zero_frames = z) and of
add_batch (zero_frames = [...]), which the GPU tests hold against this oracle computation."""
import hashlib
import json
import os

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T

G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_segments.json")))


def sha16(x16):
    return hashlib.sha256(np.ascontiguousarray(x16).tobytes()).hexdigest()


def case_input(g):
    """the case's input on the 16 bit grid, as make_golden_segments.py wrote it"""
    return O.int16_to_float(O.quantize_sndfile16(T.noise(g["seconds"], g["channels"], seed=g["seed"], amp=g["amp"])))


def oracle_at(x, z, no_limiter=False):
    """oracle embed of x continuing a stream that began z frames earlier with silence"""
    P = O.Params(test_no_limiter=no_limiter)
    ext = np.concatenate([np.zeros((z, x.shape[1]), np.float32), x])
    return O.embed(ext, O.Key(), G["payload"], P).samples[z:]


@pytest.mark.parametrize("name", sorted(G["cases"]))
def test_offset_embed_equals_reference(name):
    g = G["cases"][name]
    x = case_input(g)
    assert sha16(O.quantize_sndfile16(x)) == g["input_sha256"]
    y = oracle_at(x, g["zero_frames"], "--test-no-limiter" in g["add_args"])
    assert y.shape == x.shape
    assert sha16(O.quantize_sndfile16(y)) == g["output_sha256"], (name, g["zero_frames"])


def test_golden_covers_the_offsets_that_matter():
    cases = G["cases"].values()
    zs = {g["zero_frames"] for g in cases}
    assert {0, 100, 300 * 1024, 300 * 1024 + 517} <= zs and any(z % 44100 == 0 and z > 0 for z in zs)    # an HLS start_pos - prev_size
    assert {g["channels"] for g in cases} == {1, 2}
    assert {"--test-no-limiter" in g["add_args"] for g in cases} == {False, True}
    assert any(g["amp"] >= 1.0 for g in cases)                                                          # limiter engaged
