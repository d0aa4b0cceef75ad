"""GPU end to end: the host-side drivers (`add`, `get`; C++ over the C ABI, same code the CLI runs)
against the reference's golden outputs (tests/golden/golden.json) and the oracle.

Bars: decoded payload bits, block types, positions and pattern order identical to the reference for
every real detection (quality > sync threshold); qualities within 1e-3, decode errors within 2e-3;
embedded samples RMS < 1e-5 and at most 1 LSB apart after 16 bit quantisation."""
import json
import os
import subprocess

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden.json")))
P = O.Params()


def q16(x):
    return O.int16_to_float(O.quantize_sndfile16(x))


CASES = {
    "clip10_mono": lambda: (q16(T.noise(10.0, 1, seed=1234)), O.Key()),
    "block115": lambda: (q16(T.noise(115.0, 2, seed=1234)), O.Key()),
    "block115_nolimiter": lambda: (q16(T.noise(115.0, 2, seed=1234)), O.Key()),
    "block115_testkey3": lambda: (q16(T.noise(115.0, 2, seed=1234)), O.Key.test_key(3)),
    "limiter30": lambda: (q16(T.noise(30.7, 2, seed=99, amp=1.0)), O.Key()),
}


def check_matches(got, want, thr=0.35):
    """got/want: --json documents.  Real detections must agree exactly; fillers (n-best entries below the
    sync threshold, i.e. decoded noise) must agree in number."""
    assert got["length"] == want["length"]
    gm, wm = got["matches"], want["matches"]
    assert len(gm) == len(wm)
    real_w = [m for m in wm if m["quality"] > thr]
    real_g = [m for m in gm if m["quality"] > thr]
    assert len(real_g) == len(real_w)
    for g, w in zip(real_g, real_w):
        assert (g["key"], g["pos"], g["bits"], g["type"]) == (w["key"], w["pos"], w["bits"], w["type"]), (g, w)
        assert abs(g["quality"] - w["quality"]) < 1e-3 and abs(g["error"] - w["error"]) < 2e-3 and abs(g["rating"] - w["rating"]) < 1e-2
    return len(real_w)


@pytest.mark.parametrize("name", sorted(CASES))
def test_add_vs_reference(name):
    g = G[name]
    x, key = CASES[name]()
    no_lim = "--test-no-limiter" in g["add_args"]
    H.set_params(test_no_limiter=no_lim)
    out, blocks, snr = H.add(x, g["payload"], key.aes_key, want_stats=True)
    ref = O.embed(x, key, g["payload"], O.Params(test_no_limiter=no_lim))
    assert T.rms(out - ref.samples) < 1e-5
    assert ("Data Blocks:  %d\n" % blocks) in g["add_stderr"]
    assert abs(snr - ref.snr_db) < 1e-3
    d = O.quantize_sndfile16(out).astype(np.int32) - O.quantize_sndfile16(ref.samples).astype(np.int32)
    assert np.abs(d).max() <= 1 and np.count_nonzero(d) < 1e-3 * d.size


@pytest.mark.parametrize("name", sorted(CASES))
def test_get_vs_reference(name):
    g = G[name]
    x, key = CASES[name]()
    no_lim = "--test-no-limiter" in g["add_args"]
    y = q16(O.embed(x, key, g["payload"], O.Params(test_no_limiter=no_lim)).samples)     # == the reference's output file
    H.set_params()
    doc = H.get(y, [key.aes_key], [key.name])
    n_real = check_matches(doc, g["json"])
    want_bits = g["payload"] if len(g["payload"]) == 32 else None
    if name != "clip10_mono" and want_bits:
        assert n_real >= 1 and all(m["bits"] == want_bits for m in doc["matches"][:n_real])


def test_round_trip_gpu_add_then_get():
    x, key = CASES["block115"]()
    H.set_params()
    y = H.add(x, T.PAYLOAD, key.aes_key)
    doc = H.get(q16(y))
    check_matches(doc, G["block115"]["json"])


def test_sync_after_cut():
    g = G["noise200"]
    x = q16(O.gen_noise(200))
    H.set_params()
    y = q16(H.add(x, "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"))
    doc = H.get(y)
    bits = [m["bits"] for m in doc["matches"] if m["quality"] > 0.35]
    assert bits == ["f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"] * 5           # tests/block-decoder-test.sh: A, B, AB, A, all
    doc = H.get(y[882300:])
    assert check_matches(doc, g["cut_json"]) == 3                      # tests/sync-test.sh


def test_wrong_key_finds_nothing():
    x, _ = CASES["block115"]()
    H.set_params()
    y = q16(H.add(x, T.PAYLOAD, O.Key.test_key(1).aes_key))
    right = H.get(y, [O.Key.test_key(1).aes_key], ["test-key-1"])
    wrong = H.get(y, [O.Key.test_key(2).aes_key], ["test-key-2"])
    both = H.get(y, [O.Key.test_key(2).aes_key, O.Key.test_key(1).aes_key], ["test-key-2", "test-key-1"])
    assert any(m["bits"] == T.PAYLOAD and m["quality"] > 1 for m in right["matches"])
    assert not any(m["bits"] == T.PAYLOAD for m in wrong["matches"])
    assert [m["key"] for m in both["matches"] if m["bits"] == T.PAYLOAD][0] == "test-key-1"


def test_cli_round_trip(tmp_path):
    """The reference's shell tests in miniature (tests/block-decoder-test.sh, clip-decoder-test.sh, key-test.sh)."""
    cli = H.CLI_PATH
    src, wm, cut = (str(tmp_path / n) for n in ("n.wav", "wm.wav", "cut.wav"))
    msg = "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"
    subprocess.check_call([cli, "test-gen-noise", src, "200", "44100"])
    p = subprocess.run([cli, "add", src, wm, msg], capture_output=True, text=True)
    assert p.returncode == 0 and "Data Blocks:  3" in p.stderr, p.stderr
    assert subprocess.check_output([cli, "test-info", wm, "frames"], text=True) == subprocess.check_output([cli, "test-info", src, "frames"], text=True)
    p = subprocess.run([cli, "cmp", wm, msg, "--expect-matches", "5"], capture_output=True, text=True)
    assert p.returncode == 0 and "match_count 5 10" in p.stdout and "sync_match 3 8" in p.stdout, p.stdout
    assert subprocess.run([cli, "cmp", wm, msg, "--test-key", "1", "--expect-matches", "0"], capture_output=True).returncode == 0
    # 16 bit file output of `add` against the reference's file: hash differs only through +-1 LSB samples
    got = O.quantize_sndfile16(O.read_wav(wm)[0]).astype(np.int32)
    ref = O.quantize_sndfile16(O.embed(q16(O.gen_noise(200)), O.Key(), msg, P).samples).astype(np.int32)
    assert np.abs(got - ref).max() <= 1 and np.count_nonzero(got - ref) < 1e-3 * got.size
    subprocess.check_call([cli, "cut-start", wm, cut, "882300"])
    p = subprocess.run([cli, "cmp", cut, msg, "--expect-matches", "3", "--test-cut", "882300"], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout
    # no-limiter SNR bound of tests/block-decoder-test.sh
    subprocess.check_call([cli, "add", "--test-no-limiter", src, wm, msg], stderr=subprocess.DEVNULL)
    assert float(subprocess.check_output([cli, "test-snr", src, wm], text=True)) >= 32.4
    # json on stdout
    p = subprocess.run([cli, "get", "--json", "-", wm], capture_output=True, text=True)
    assert json.loads(p.stdout)["matches"][0]["bits"] == msg


@pytest.mark.parametrize("name", ["short12", "short16", "short20", "linear120"])
def test_short_payload_and_linear_vs_reference(name):
    """--short 12/16/20 (tests/short-payload-test.sh) and --linear: GPU add within 1e-5 RMS of the oracle (== reference PCM,
    CPU test), GPU get reproduces the reference's pattern list"""
    g = G[name]
    opts = g["opts"]
    Pc = O.Params()
    short = int(opts[opts.index("--short") + 1]) if "--short" in opts else 0
    if short:
        Pc.payload_short, Pc.payload_size = True, short
    if "--linear" in opts:
        Pc.mix = False
    x = q16(O.gen_noise(120))
    H.set_params(mix="--linear" not in opts)
    H.set_short_payload(short)
    try:
        out = H.add(x, g["payload"])
        ref = O.embed(x, O.Key(), g["payload"], Pc)
        assert T.rms(out - ref.samples) < 1e-5
        y = q16(ref.samples)
        doc = H.get(y)
    finally:
        H.set_short_payload(0)
        H.set_params()
    n_real = check_matches(doc, g["json"])
    assert n_real >= 3 and all(m["bits"] == g["payload"] for m in doc["matches"][:n_real])


def test_s16_entry_points_equal_host_side_conversion():
    """16 bit PCM buffers converted on the device (awm_embed_s16 / awm_pcm_stage): bit identical to converting on the host
    with the reference's rules (src/sfinputstream.cc:189-210, src/rawconverter.hh:34-50 + src/sfoutputstream.cc:148-155) around
    the float entry points, for add (incl. clipping at full scale), get (block and clip decoder) and get --detect-speed"""
    H.set_params()
    for seconds, ch, seed, amp in ((130.0, 2, 5, 0.5), (30.7, 2, 99, 1.0), (12.0, 1, 3, 0.5)):
        x16 = O.quantize_sndfile16(T.noise(seconds, ch, seed=seed, amp=amp))
        xf = O.int16_to_float(x16)
        want = O.quantize_sndfile16(H.add(xf, T.PAYLOAD))
        got, blocks, snr = H.add_s16(x16, T.PAYLOAD, want_stats=True)
        assert got.dtype == np.int16 and np.array_equal(got, want)
        doc_f = H.get(O.int16_to_float(got))
        doc_s = H.get_s16(got)
        assert doc_s == doc_f and len(doc_s["matches"]) >= 1
    # pipelined path (> 2 * 12288 frames of 1024): 10 minutes
    x16 = O.quantize_sndfile16(T.noise(600.0, 2, seed=8))
    want = O.quantize_sndfile16(H.add(O.int16_to_float(x16), T.PAYLOAD))
    got = H.add_s16(x16, T.PAYLOAD)
    assert np.array_equal(got, want)
    assert H.get_s16(got) == H.get(O.int16_to_float(got))
    H.set_speed_params(detect_speed=True)
    try:
        y16 = O.quantize_sndfile16(T.speed_changed(30, 1.01))
        assert H.get_s16(y16) == H.get(O.int16_to_float(y16))
    finally:
        H.set_speed_params()
