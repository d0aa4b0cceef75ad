"""GPU: streaming and sharded `add` at sample rates other than 44.1 kHz, window by window (add_watermark_window ->
awm_embed_window_rates).  Every window's owned frames must equal the whole-stream `add` at that rate bit for bit: the bounded-memory
loop (hostapi.add_windowed, the CLI) for window sizes down to 3 1024-frames (shorter than a limiter block and than the halo), with
stream offsets far into a stream, and sharded ranks that each mark their own span (hostapi.window_range + hostapi.add_window) from
host and from device buffers.  Data Blocks must be equal and the SNR within 1e-9 dB (its sums are added in another order)."""
import hashlib
import json
import math
import os
import subprocess
import threading
import wave

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import capi, hostapi as H

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "resampled_add.json")))["cases"]


def noise(frames, channels, seed, amp=1.0):
    rng = np.random.default_rng(seed)
    return ((rng.random((frames, channels), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


@pytest.fixture(autouse=True)
def default_params():
    H.set_params()
    yield
    H.set_params()


def check_windowed(x, rate, window, zero_frames=0):
    y, blocks, snr = H.add_windowed(x, T.PAYLOAD, zero_frames=zero_frames, window_frames=window, sample_rate=rate)
    return y, blocks, snr


def same_snr(a, b):
    return (math.isinf(a) and math.isinf(b)) or abs(a - b) <= 1e-9


# ---- 1. the bounded-memory loop equals the whole-stream add: 130 s of full-scale noise, so the limiter is engaged

CASES = [(r, c, lim, w) for r in (8000, 32000, 48000, 96000) for c in (1, 2, 3) for lim in (True, False) for w in (0, 37)]
CASES += [(r, 2, True, 1000) for r in (8000, 32000, 48000, 96000)] + [(48000, 1, False, 1000)]
CASES += [(48000, 2, True, 3), (8000, 1, False, 3), (96000, 3, True, 3)]


@pytest.mark.parametrize("rate, channels, limiter, window", CASES)
def test_windowed_add_equals_the_whole_stream_add(rate, channels, limiter, window):
    H.set_params(test_no_limiter=not limiter)
    x = noise(130 * rate + 321, channels, seed=rate + channels)
    want, want_blocks, want_snr = H.add(x, T.PAYLOAD, sample_rate=rate, want_stats=True)
    y, blocks, snr = check_windowed(x, rate, window)
    assert np.array_equal(y, want), (rate, channels, limiter, window, np.flatnonzero((y != want).any(axis=1))[:5])
    assert blocks == want_blocks and same_snr(snr, want_snr), (blocks, want_blocks, snr, want_snr)
    if limiter:
        assert np.abs(y).max() <= 1.0 and np.abs(x).max() > 0.99        # the limiter holds the ceiling on full-scale input


# ---- 2. stream offsets: the input continues a stream that began z frames earlier with silence

@pytest.mark.parametrize("rate", [48000, 32000])
def test_windowed_add_at_stream_offsets(rate):
    x = noise(20 * rate + 77, 2, seed=5, amp=0.9)
    for z in (0, 1, 1023, 1024, 1025, rate - 1, rate, rate + 1):
        y, blocks, snr = check_windowed(x, rate, 37, zero_frames=z)
        (b,), bb, bs = H.add_batch_rates([x], [T.PAYLOAD], [rate], zero_frames=[z], want_stats=True)
        assert np.array_equal(y, b), (rate, z)
        assert blocks == bb[0] and same_snr(snr, bs[0]), (z, blocks, bb, snr, bs)
        whole = H.add(np.concatenate([np.zeros((z, 2), np.float32), x]), T.PAYLOAD, sample_rate=rate)
        assert np.array_equal(y, whole[z:]), (rate, z)


def test_windowed_add_a_day_into_the_stream():
    rate = 48000
    z = 24 * 3600 * rate + 333
    x = noise(12 * rate, 2, seed=9, amp=0.9)
    y, blocks, snr = check_windowed(x, rate, 0, zero_frames=z)
    (b,), bb, bs = H.add_batch_rates([x], [T.PAYLOAD], [rate], zero_frames=[z], want_stats=True)
    assert np.array_equal(y, b)
    assert blocks == bb[0] and same_snr(snr, bs[0])
    y37, _, _ = check_windowed(x, rate, 37, zero_frames=z)
    assert np.array_equal(y37, b)


# ---- 3. sharded: each rank marks its own span from the window window_range names

def cuts_of(n, rate, world, kind):
    if kind == "arbitrary":
        inner = sorted(np.random.default_rng(world).integers(1, n - 1, world - 1).tolist())
    elif kind == "frame_edges":
        inner = [(n // world * k) // 1024 * 1024 for k in range(1, world)]
    elif kind == "block_edges":
        inner = [k * rate * 7 for k in range(1, world)]
    else:                                                                   # one rank owns a single frame
        inner = [n // 2, n // 2 + 1] + [n // 2 + 1 + k * rate for k in range(1, world - 2)]
    return [0] + inner + [n]


@pytest.mark.parametrize("rate", [48000, 32000, 96000])
@pytest.mark.parametrize("world, kind", [(2, "arbitrary"), (3, "arbitrary"), (2, "frame_edges"), (3, "block_edges"), (3, "one_frame")])
def test_sharded_ranks_concatenate_to_the_whole_stream(rate, world, kind):
    torch = pytest.importorskip("torch")
    x = noise(40 * rate + 555, 2, seed=rate // 1000 + world)
    n = x.shape[0]
    want, _, want_snr = H.add(x, T.PAYLOAD, sample_rate=rate, want_stats=True)
    cuts = cuts_of(n, rate, world, kind)
    xd = torch.from_numpy(x).cuda()
    parts, parts_d, sums = [], [], np.zeros(2)
    for a, b in zip(cuts[:-1], cuts[1:]):
        e0, e1 = H.window_range(a, b, n, sample_rate=rate)
        assert e0 <= a < b <= e1 <= n
        y, sd, ss = H.add_window(x[e0:e1], T.PAYLOAD, e0, n, a, b, sample_rate=rate, want_stats=True)
        parts.append(y[a - e0:b - e0])
        sums += (sd, ss)
        win = xd[e0:e1]                                      # a view into the whole stream's device buffer
        out = torch.zeros_like(win)
        H.add_window(win.data_ptr(), T.PAYLOAD, e0, n, a, b, pcm_out=out.data_ptr(), n_frames=e1 - e0, channels=2, sample_rate=rate)
        torch.cuda.synchronize()
        parts_d.append(out[a - e0:b - e0].cpu().numpy())
    assert np.array_equal(np.concatenate(parts), want), (rate, world, kind, cuts)
    assert np.array_equal(np.concatenate(parts_d), want), (rate, world, kind, cuts)
    assert same_snr(10 * math.log10(sums[1] / sums[0]), want_snr)


def test_sharded_window_with_a_larger_buffer_and_at_the_watermark_rate():
    for rate in (44100, 48000):
        xs = noise(30 * rate + 9, 1, seed=rate)
        n = xs.shape[0]
        want = H.add(xs, T.PAYLOAD, sample_rate=rate)
        a, b = 11 * rate + 5, 19 * rate - 7
        e0, e1 = H.window_range(a, b, n, sample_rate=rate)
        if rate == 44100:
            assert e0 % 1024 == 0
        s0 = max(e0 - 1000, 0)
        y = H.add_window(xs[s0:], T.PAYLOAD, s0, n, a, b, sample_rate=rate)
        assert np.array_equal(y[a - s0:b - s0], want[a:b])
        assert np.array_equal(y[:e0 - s0], xs[s0:e0])                # outside the window the buffer is not touched


# ---- 4. the golden single-add cases through the windowed loop

@pytest.mark.parametrize("name", sorted(GOLDEN))
def test_golden_cases_through_the_windowed_loop(name):
    c = GOLDEN[name]
    rng = np.random.default_rng(c["seed"])
    x = ((rng.random((c["frames"], c["channels"]), dtype=np.float32) - 0.5) * (2 * c["amp"])).astype(np.float32)
    for run in ("limiter_host", "nolimiter_host"):
        want = c["runs"][run]
        H.set_params(test_no_limiter=run.startswith("nolimiter"))
        y, blocks, snr = H.add_windowed(x, c["payload"], window_frames=64 if c["frames"] < 4_000_000 else 1000, sample_rate=c["rate"])
        assert hashlib.sha256(y.tobytes()).hexdigest() == want["output_sha256"], (name, run)
        assert blocks == want["data_blocks"], (name, run)
        if want["snr_db"] is None:
            assert math.isinf(snr)
        else:
            assert abs(snr - want["snr_db"]) <= 1e-9, (name, run, snr, want["snr_db"])


# ---- 5. the CLI: 48 kHz WAV files and raw pipes stream through the windowed loop

def wav_out_rule(y):
    """16 bit WAV output: float_to_int_clip<32> (f) >> 16"""
    v = np.clip(y.astype(np.float64) * 2147483648.0, -2147483648.0, 2147483647.0)
    return (np.trunc(v).astype(np.int64) >> 16).astype(np.int16)


def raw_out_rule(y):
    """16 bit raw output: float_to_int_clip<16> (f)"""
    v = np.clip(y.astype(np.float64) * 32768.0, -32768.0, 32767.0)
    return np.trunc(v).astype(np.int16)


def stat_lines(stderr):
    lines = {l.split(":")[0].strip(): l.split(":", 1)[1].strip() for l in stderr.splitlines() if ":" in l}
    return int(lines["Data Blocks"]), float(lines["SNR"].split()[0])


def test_cli_at_48khz_equals_the_whole_stream_add(tmp_path):
    rate = 48000
    x16 = (noise(70 * rate + 13, 2, seed=21, amp=0.5) * 32767).astype(np.int16)
    xf = x16.astype(np.float32) * np.float32(2 ** -15)
    want, want_blocks, want_snr = H.add(xf, T.PAYLOAD, sample_rate=rate, want_stats=True)
    src, dst = str(tmp_path / "in.wav"), str(tmp_path / "out.wav")
    with wave.open(src, "wb") as w:
        w.setnchannels(2)
        w.setsampwidth(2)
        w.setframerate(rate)
        w.writeframes(x16.tobytes())
    p = subprocess.run([H.CLI_PATH, "add", "--snr", src, dst, T.PAYLOAD], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    with wave.open(dst, "rb") as w:
        y = np.frombuffer(w.readframes(w.getnframes()), np.int16).reshape(-1, 2)
    assert np.array_equal(y, wav_out_rule(want))
    blocks, snr = stat_lines(p.stderr)
    assert blocks == want_blocks and abs(snr - want_snr) <= 1e-6
    p = subprocess.run([H.CLI_PATH, "add", "--snr", "--input-format", "raw", "--raw-rate", str(rate), "--output-format", "raw", "-", "-",
                        T.PAYLOAD], input=x16.tobytes(), capture_output=True)
    assert p.returncode == 0, p.stderr
    assert np.array_equal(np.frombuffer(p.stdout, np.int16).reshape(-1, 2), raw_out_rule(want))
    blocks, snr = stat_lines(p.stderr.decode())
    assert blocks == want_blocks and abs(snr - want_snr) <= 1e-6


def test_cli_pipe_gets_output_before_its_input_ends():
    rate, window = 48000, 4096 * 1024
    x16 = (noise(3 * window, 2, seed=22, amp=0.5) * 32767).astype(np.int16)
    p = subprocess.Popen([H.CLI_PATH, "add", "--input-format", "raw", "--raw-rate", str(rate), "--output-format", "raw", "-", "-", T.PAYLOAD],
                         stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    fed, got, out = threading.Event(), threading.Event(), []

    def writer():
        p.stdin.write(x16.tobytes())
        p.stdin.flush()
        fed.set()

    def reader():
        n = 0
        while True:
            b = p.stdout.read1(1 << 20)
            if not b:
                return
            out.append(b)
            n += len(b)
            if n >= window * 4:
                got.set()

    tw, tr = threading.Thread(target=writer), threading.Thread(target=reader)
    tw.start()
    tr.start()
    try:
        assert got.wait(120), "no window of output arrived while stdin was still open"
        assert not p.stdin.closed
    finally:
        tw.join(120)
        p.stdin.close()
        tr.join(300)
        p.wait(300)
    assert fed.is_set() and p.returncode == 0
    y = np.frombuffer(b"".join(out), np.int16).reshape(-1, 2)
    want = H.add(x16.astype(np.float32) * np.float32(2 ** -15), T.PAYLOAD, sample_rate=rate)
    assert np.array_equal(y, raw_out_rule(want))


# ---- 6. refusals

def test_window_call_refusals():
    ctx = capi.Context.from_handle(H.load().awmh_ctx())
    lib = capi.load()
    x = np.zeros((4096, 2), np.float32)
    y = np.zeros_like(x)
    coded = H.coded_bits(None, T.PAYLOAD)
    H.add(x[:10], T.PAYLOAD, sample_rate=48000)             # the role table of the zero key is on the device

    def call(rate, n_emit, snr_first=0, snr_last=2 ** 64 - 1):
        rc = lib.awm_embed_window_rates(ctx.h, capi._ptr(x), capi._ptr(y), H.ctypes.c_size_t(4096), H.ctypes.c_int(2), capi._ptr(coded),
                                        H.ctypes.c_int(rate), H.ctypes.c_int(44100), H.ctypes.c_uint64(0), H.ctypes.c_uint64(n_emit),
                                        H.ctypes.c_int(250), H.ctypes.c_double(0.01), H.ctypes.c_int(1000), H.ctypes.c_float(0.999),
                                        H.ctypes.c_uint64(snr_first), H.ctypes.c_uint64(snr_last), None)
        return rc, lib.awm_last_error(ctx.h).decode()

    launches = ctx.launches
    rc, msg = call(44100, 4096)
    assert rc and "awm_embed_window" in msg and "watermark rate" in msg
    rc, msg = call(48000, 4096, 10, 9)
    assert rc and "--snr range" in msg
    rc, msg = call(48000, 4095)
    assert rc and "n_emit 4095 is less than n_frames 4096" in msg
    assert ctx.launches == launches                          # refused before any work
    rc, msg = call(48000, 4096)
    assert rc == 0, msg


def test_add_window_raises_when_the_buffer_misses_its_range():
    rate = 48000
    x = noise(10 * rate, 2, seed=1)
    n = x.shape[0]
    e0, e1 = H.window_range(4 * rate, 5 * rate, n, sample_rate=rate)
    with pytest.raises(ValueError):
        H.add_window(x[e0 + 1:e1], T.PAYLOAD, e0 + 1, n, 4 * rate, 5 * rate, sample_rate=rate)
    with pytest.raises(ValueError):
        H.add_window(x[e0:e1 - 1], T.PAYLOAD, e0, n, 4 * rate, 5 * rate, sample_rate=rate)
