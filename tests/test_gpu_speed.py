"""GPU: resampler and speed detection (SURVEY.md section 8a rows wmspeed / resample) against the oracle and the
reference goldens (tests/detect-speed-test.sh, tests/sample-rate-test.sh).

Bars: the resampler is bit exact against the oracle (same filter table, same float operation order); the MagMatrix /
compare scores of a scan agree with the oracle to 2e-5 relative (the 512-point spectra come out of a different FFT
factorisation); the detected speed agrees with the reference's printed value to 2e-6, its quality to 1e-4; the decoded
patterns (bits, type incl. -SPEED, position) are identical for every real detection."""
import json
import os

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi
from audiowmark_b200 import hostapi as H
from test_gpu_e2e import check_matches

pytestmark = pytest.mark.gpu
G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden.json")))
P = O.Params()


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("channels,ratio,n", [(2, 44100 / 48000.0, 200000), (2, 48000 / 44100.0, 150001), (1, 1 / 1.01, 99999),
                                              (2, 0.9764 / 2, 300000), (3, 1.25 / 2, 70000), (2, 1.0371, 1000), (1, 0.5, 40), (2, 2.0, 5)])
def test_resample_bit_exact_vs_oracle(ctx, channels, ratio, n):
    rng = np.random.default_rng(7)
    x = (rng.random((n, channels), dtype=np.float32) - 0.5).astype(np.float32)
    want = O.resample_ratio(x, ratio)
    got = ctx.resample(x, ratio)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # streaming frame count (WavChunkLoader semantics) and a longer output than the taps allow: trailing zeros like the oracle
    n_stream = O.stream_out_count(n, ratio)
    assert H.resample_stream_frames(n, ratio) == n_stream
    got2 = ctx.resample(x, ratio, n_out=n_stream + 3)
    want2 = O.resample_ratio(x, ratio, n_out=n_stream + 3)
    assert np.array_equal(got2.view(np.uint32), want2.view(np.uint32))
    assert not got2[n_stream:].any()


def test_resample_linearity_and_identity_at_large_size(ctx):
    """size independent properties at a chunk-sized input: integer positions reproduce the input exactly, and the
    operator is linear"""
    rng = np.random.default_rng(11)
    n = 3_000_000
    x = (rng.random((n, 2), dtype=np.float32) - 0.5).astype(np.float32)
    up = ctx.resample(x, 2.0)
    assert np.array_equal(up[0::2], x)                    # t = n / 2: every second output sits on an input sample
    y = (rng.random((n, 2), dtype=np.float32) - 0.5).astype(np.float32)
    r = 44100 / 48000.0
    a, b, ab = ctx.resample(x, r), ctx.resample(y, r), ctx.resample(x + y, r)
    assert T.rms(ab - (a + b)) < 2e-7


def test_speed_scan_vs_oracle(ctx):
    key = O.Key()
    T.setup_ctx(ctx, key, P)
    y = T.speed_changed(30, 1.01)
    clip = O.get_speed_clip(0.3, y, 44100, 25 * 1.3)
    entries = O.speed_sync_entries(key, P)
    centers = [1.0 * 1.0007 ** (11 * c) for c in (-28, -3, 1, 14, 28)]
    rel = [[1.0007 ** p * c / c for p in range(-5, 6)] for c in centers]
    got = ctx.speed_scan(clip, 25.0, centers, rel)
    for ci, c in enumerate(centers):
        mags = O.speed_prepare_mags(clip, 44100, c, 25.0, entries)
        want = O.speed_compare(mags, entries, rel[ci], P)
        assert np.allclose(got[ci], want, rtol=2e-5, atol=1e-7), (c, got[ci], want)
    assert got.max() > 0.5          # centre 1.0007^11 ~ 1.0077 with relative steps reaches the true speed 1.01


@pytest.mark.parametrize("idx", [0, 1, 2, 3])
def test_detect_speed_vs_reference(idx):
    """tests/detect-speed-test.sh: speed 0.9764 / 1.0 / 1.01 --detect-speed, 1.01 --detect-speed-patient"""
    c = G["speed30"]["cases"][idx]
    y = T.speed_changed(30, c["speed"])
    H.set_params()
    H.set_speed_params(detect_speed=not c["opt"].endswith("patient"), detect_speed_patient=c["opt"].endswith("patient"))
    try:
        speed, quality, accepted = H.detect_speed(y)
    finally:
        H.set_speed_params()
    line = c["cmp_stdout"].split("\n")[0].split()
    assert line[0] == "detect_speed"
    assert abs(speed - float(line[1])) < 2e-6 and abs(quality - float(line[2])) < 1e-4
    assert accepted == ("\nspeed " in c["cmp_stdout"])
    assert 100 * abs(speed - T.cli_float(c["speed"])) / c["speed"] < 0.01


@pytest.mark.parametrize("idx", [0, 2])
def test_get_detect_speed_vs_reference(idx):
    c = G["speed30"]["cases"][idx]
    y = T.speed_changed(30, c["speed"])
    H.set_params()
    H.set_speed_params(detect_speed=True, test_speed=T.cli_float(c["speed"]))
    try:
        doc = H.get(y)
    finally:
        H.set_speed_params()
    n_real = check_matches(doc, c["json"])
    assert n_real >= 1
    m = doc["matches"][0]
    assert m["bits"] == "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0" and m["type"].endswith("-SPEED")
    assert abs(m["speed"] - c["json"]["matches"][0]["speed"]) < 2e-6


def test_get_try_speed_vs_reference():
    g = G["speed30"]["try_speed_1.01"]
    y = T.speed_changed(30, 1.01)
    H.set_params()
    H.set_speed_params(try_speed=T.cli_float(1.01))
    try:
        doc = H.get(y)
    finally:
        H.set_speed_params()
    assert check_matches(doc, g["json"]) >= 1


def test_get_48000_vs_reference():
    """tests/sample-rate-test.sh, second half: a 48 kHz file decodes after resampling to the watermark rate"""
    g = G["rate48000"]
    z = O.int16_to_float(O.quantize_sndfile16(O.resample(T.watermarked_noise(200), 44100, 48000)))
    H.set_params()
    doc = H.get(z, sample_rate=48000)
    assert check_matches(doc, g["json"]) == 5


def test_speed_long_input_detect_and_decode():
    """size independent property at a larger size: 200 s at speed 1.01 -> five SPEED matches, like the reference binary"""
    y = O.int16_to_float(O.quantize_sndfile16(O.resample_ratio(T.watermarked_noise(200), 1 / T.cli_float(1.01))))
    H.set_params()
    H.set_speed_params(detect_speed=True)
    try:
        doc = H.get(y)
    finally:
        H.set_speed_params()
    hits = [m for m in doc["matches"] if m["bits"] == "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"]
    assert len(hits) == 5 and all(m["type"].endswith("SPEED") for m in hits)
    assert abs(hits[0]["speed"] - 1.010014) < 3e-6


@pytest.mark.parametrize("name", ["rate32000_add", "rate48000_add_nolimiter"])
def test_add_other_sample_rates_vs_reference(name):
    """`add` through the WatermarkResampler path: GPU output against the oracle (== reference PCM, see the CPU test)"""
    g = G[name]
    x = O.int16_to_float(O.quantize_sndfile16(O.gen_noise(g["seconds"], g["rate"])))
    no_lim = "--test-no-limiter" in g["add_args"]
    H.set_params(test_no_limiter=no_lim)
    try:
        out, blocks, snr = H.add(x, "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0", want_stats=True, sample_rate=g["rate"])
    finally:
        H.set_params()
    ref = O.embed(x, O.Key(), "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0", O.Params(test_no_limiter=no_lim), g["rate"])
    assert T.rms(out - ref.samples) < 1e-5
    d = O.quantize_sndfile16(out).astype(np.int32) - O.quantize_sndfile16(ref.samples).astype(np.int32)
    assert np.abs(d).max() <= 1 and np.count_nonzero(d) < 1e-3 * d.size
    assert ("Data Blocks:  %d\n" % blocks) in g["add_stderr"]
    assert abs(snr - ref.snr_db) < 1e-3
    if name == "rate32000_add":
        doc = H.get(O.int16_to_float(O.quantize_sndfile16(out)), sample_rate=g["rate"])
        assert check_matches(doc, g["json"]) == 5


def test_cli_reference_shell_tests(tmp_path):
    """the reference's tests/detect-speed-test.sh, sample-rate-test.sh and short-payload-test.sh run against bin/audiowmark
    (same argv grammar, same pass criteria: `cmp` exits 0 iff the message was found; --expect-matches where the scripts use it)"""
    import subprocess
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "audiowmark_b200", "bin", "audiowmark")
    msg = "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"
    a, b, c = (str(tmp_path / n) for n in ("in.wav", "out.wav", "spd.wav"))
    # detect-speed-test.sh
    subprocess.check_call([cli, "test-gen-noise", a, "30", "44100"])
    subprocess.check_call([cli, "add", "-q", a, b, msg])
    for speed in ("0.9764", "1.01"):
        subprocess.check_call([cli, "test-change-speed", b, c, speed])
        for opt in ("--detect-speed", "--detect-speed-patient"):
            p = subprocess.run([cli, "cmp", c, msg, opt, "--test-speed", speed], capture_output=True, text=True)
            assert p.returncode == 0, p.stdout + p.stderr
            line = p.stdout.split("\n")[0].split()
            assert line[0] == "detect_speed" and float(line[3]) < 0.01          # relative error in percent
            assert "\nspeed " in p.stdout and "-SPEED" in p.stdout
        # without speed detection the message is not found at this speed
        assert subprocess.run([cli, "cmp", c, msg], capture_output=True).returncode == 1
    # sample-rate-test.sh
    subprocess.check_call([cli, "test-gen-noise", a, "200", "32000"])
    subprocess.check_call([cli, "add", "-q", a, b, msg])
    assert subprocess.run([cli, "cmp", "--expect-matches", "5", b, msg], capture_output=True).returncode == 0
    subprocess.check_call([cli, "test-resample", b, c, "48000"])
    assert subprocess.run([cli, "cmp", "--expect-matches", "5", c, msg], capture_output=True).returncode == 0
    # short-payload-test.sh
    subprocess.check_call([cli, "test-gen-noise", a, "200", "44100"])
    for bits, m in (("12", "abc"), ("16", "abcd"), ("20", "abcde")):
        subprocess.check_call([cli, "add", "-q", "--short", bits, a, b, m])
        assert subprocess.run([cli, "cmp", "--short", bits, b, m], capture_output=True).returncode == 0
    # --linear round trip
    subprocess.check_call([cli, "add", "-q", "--linear", a, b, msg])
    assert subprocess.run([cli, "cmp", "--linear", b, msg], capture_output=True).returncode == 0


def test_cli_reference_order_kernels_give_the_same_answer(tmp_path):
    """AWM_APPROX=ring selects the approx search kernel that keeps the reference's exact float summation order (one thread per
    start frame); the default one (entry sums + gather) must print the same patterns, positions and three-digit qualities.
    The refine always ends in the reference's order: test_gpu_stages.py::test_sync_refine_vs_oracle holds it to the oracle."""
    import subprocess
    cli = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "audiowmark_b200", "bin", "audiowmark")
    a, b = str(tmp_path / "in.wav"), str(tmp_path / "out.wav")
    subprocess.check_call([cli, "test-gen-noise", a, "200", "44100"])
    subprocess.check_call([cli, "add", "-q", a, b, "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0"])
    fast = subprocess.run([cli, "get", b], capture_output=True, text=True, check=True).stdout
    env = dict(os.environ, AWM_APPROX="ring")
    exact = subprocess.run([cli, "get", b], capture_output=True, text=True, check=True, env=env).stdout
    real = lambda out: [l for l in out.split("\n") if "f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0f0" in l]
    assert len(real(fast)) == 5 and real(fast) == real(exact)
    assert "\n".join(real(fast)) + "\n" == "\n".join(G["noise200"]["cmp_stdout"].split("\n")[:5]) + "\n"      # and they are the reference's lines
