"""GPU: the streaming `get` (GetStream, host/awm_get.cc).  A stream fed piece by piece returns the document get() returns for the
whole buffer, byte for byte, at 44.1 kHz and at the rates it resamples on the device; at those rates the document also equals get()
at 44.1 kHz of the whole stream resampled by awm_resample, what get() computed before it streamed.  Device memory does not grow
with the stream, host memory of `audiowmark get -` does not either, and the CLI prints the same for a file and a pipe."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import awm_testlib as T
from audiowmark_b200 import hostapi as H

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

MARK = 44100
RATES = [22050, 32000, 44100, 48000, 96000]
CHUNK_MIN = 3.0


def _noise(n, channels, seed):
    rng = np.random.default_rng(seed)
    return (rng.random((n, channels), dtype=np.float32) - 0.5).astype(np.float32)


def _input_frames(mark_frames, rate):
    """the smallest input length at `rate` whose resampled stream has at least mark_frames frames"""
    if rate == MARK:
        return mark_frames
    ratio = MARK / rate
    n = max(int(mark_frames / ratio) - 64, 0)
    while H.resample_stream_frames(n, ratio) < mark_frames:
        n += 1
    return n


_MARKED = {}


def _marked(rate, channels, seconds=290.0):
    """noise marked with add() at `rate` (several 3-minute chunks at the watermark rate); only one rate is kept at a time"""
    k = (rate, channels)
    for old in [o for o in _MARKED if o[0] != rate]:
        del _MARKED[old]
    if k not in _MARKED:
        H.set_params(chunk_size_min=CHUNK_MIN)
        _MARKED[k] = H.add(_noise(int(seconds * rate), channels, seed=rate + channels), T.PAYLOAD, sample_rate=rate)
    return _MARKED[k]


def _stream_doc(y, rate, piece, keys=None, names=None, device=False):
    s = H.GetStream(keys=keys, names=names, channels=y.shape[1], sample_rate=rate)
    try:
        if device:
            yd = torch.from_numpy(np.ascontiguousarray(y)).cuda()
            torch.cuda.synchronize()
            for i in range(0, y.shape[0], piece):
                k = min(piece, y.shape[0] - i)
                s.feed(yd[i:].data_ptr(), n_frames=k)
        else:
            for i in range(0, y.shape[0], piece):
                s.feed(y[i:i + piece])
        return s.finish(parse=False)
    finally:
        s.close()


def _anchor(y, rate, keys=None, names=None):
    """what get() at another rate computed before it streamed: awm_resample of the whole stream, then get() at 44.1 kHz"""
    ratio = MARK / rate
    r = H.resample(y, ratio, n_out=H.resample_stream_frames(y.shape[0], ratio))
    return H.get(r, keys=keys, names=names, parse=False)


@pytest.fixture(autouse=True)
def _three_minute_chunks():
    H.set_params(chunk_size_min=CHUNK_MIN)
    yield
    H.set_params()
    H.set_speed_params()
    H.set_short_payload(0)


LENGTHS = ["clip", "max-1", "max", "max+1", "several"]


@pytest.mark.parametrize("length", LENGTHS)
@pytest.mark.parametrize("rate", RATES)
def test_stream_equals_buffer(rate, length):
    ch = [1, 2, 3][(RATES.index(rate) + LENGTHS.index(length)) % 3]
    y = _marked(rate, ch)
    mx, ov = H.chunk_geometry(MARK)
    m = {"clip": 100 * MARK, "max-1": mx - 1, "max": mx, "max+1": mx + 1, "several": mx + 2 * (mx - ov) + MARK * 7}[length]
    n = _input_frames(m, rate)
    assert n <= y.shape[0]
    y = np.ascontiguousarray(y[:n])
    want = H.get(y, sample_rate=rate, parse=False)
    assert '"bits"' in want or length == "clip"
    if rate != MARK:
        assert want == _anchor(y, rate)
    for piece in (4095, 1 << 20):
        assert _stream_doc(y, rate, piece) == want, (rate, length, piece)
    assert _stream_doc(y, rate, n, device=True) == want
    if length == "several":
        assert _stream_doc(y, rate, 4095, device=True) == want
    if length == "max":      # the document of a stream that exactly fills a chunk includes the overlap-only chunk
        assert len(H.get_stream_plan(n, 4095, rate)[0]) == 2


@pytest.mark.parametrize("rate", RATES)
def test_stream_of_single_frames_and_empty_stream(rate):
    y = _marked(rate, 2)
    n = int(0.5 * rate)
    short = np.ascontiguousarray(y[:n])
    want = H.get(short, sample_rate=rate, parse=False)
    assert _stream_doc(short, rate, 1) == want
    if rate != MARK:
        assert want == _anchor(short, rate)
    empty = np.zeros((0, 2), np.float32)
    assert _stream_doc(empty, rate, 4095) == H.get(empty, sample_rate=rate, parse=False)


def test_device_and_16_bit_buffers_at_other_rates():
    y = np.ascontiguousarray(_marked(48000, 2)[:int(200 * 48000)])
    want = H.get(y, sample_rate=48000, parse=False)
    yd = torch.from_numpy(y).cuda()
    torch.cuda.synchronize()
    assert H.get(yd.data_ptr(), n_frames=y.shape[0], channels=2, sample_rate=48000, parse=False) == want
    y16 = np.clip(np.floor(y * 32768), -32768, 32767).astype(np.int16)
    assert H.get_s16(y16, sample_rate=48000, parse=False) == _anchor(y16.astype(np.float32) / 32768, 48000)


def _option_case(rate, seconds, payload, keys=None, names=None, piece=4095):
    y = H.add(_noise(int(seconds * rate), 2, seed=7), payload, key=keys[0] if keys else None, sample_rate=rate)
    want = H.get(y, keys=keys, names=names, sample_rate=rate, parse=False)
    assert _stream_doc(y, rate, piece, keys=keys, names=names) == want
    if rate != MARK:
        assert want == _anchor(y, rate, keys=keys, names=names)
    return want


@pytest.mark.parametrize("rate", [44100, 48000])
def test_options(rate):
    k1, k2 = bytes(range(16)), bytes(range(16, 32))
    doc = _option_case(rate, 250.0, T.PAYLOAD, keys=[k1, k2], names=["alpha", "beta"])
    assert '"alpha"' in doc
    H.set_short_payload(16)
    H.set_params(chunk_size_min=CHUNK_MIN, frames_per_bit=3)
    assert '"bits"' in _option_case(rate, 250.0, "beef")
    H.set_short_payload(0)
    H.set_params(chunk_size_min=CHUNK_MIN, mix=False, hard=True)
    _option_case(rate, 250.0, T.PAYLOAD, piece=1 << 20)
    H.set_params(chunk_size_min=CHUNK_MIN)
    H.set_speed_params(try_speed=T.cli_float(1.01))
    _option_case(rate, 250.0, T.PAYLOAD)


def test_detect_speed_over_two_chunks():
    rate = 48000
    y = H.add(_noise(int(250 * rate), 2, seed=11), T.PAYLOAD, sample_rate=rate)
    y = np.ascontiguousarray(H.resample(y, 1 / T.cli_float(1.01)))
    H.set_speed_params(detect_speed=True)
    assert len(H.get_stream_plan(y.shape[0], 4095, rate)[0]) >= 2
    want = H.get(y, sample_rate=rate, parse=False)
    assert _stream_doc(y, rate, 4095) == want
    assert want == _anchor(y, rate)


@pytest.mark.parametrize("rate", [8000, 22050, 32000, 48000, 96000])
def test_resampler_windows_before_the_end_is_known(rate):
    """outputs below resample_stream_available (fed), computed with n_in_total = fed, equal awm_resample of the whole stream"""
    from audiowmark_b200 import capi as C
    ctx = C.Context(0)
    try:
        ratio = MARK / rate
        n = 300007
        x = _noise(n, 2, seed=rate)
        whole = ctx.resample(x, ratio, n_out=H.resample_stream_frames(n, ratio))
        out = torch.empty(whole.size + 2, dtype=torch.float32, device="cuda")
        for fed in (37, 4095, 65536, 200001, n):
            avail = H.resample_stream_available(fed, ratio)
            if not avail:
                continue
            t0, _ = C.resample_taps(fed, ratio, 0, avail)
            ctx.resample_range(np.ascontiguousarray(x[t0:fed]), t0, fed, ratio, out.data_ptr(), 0, avail)
            ctx.synchronize()
            assert out[:avail * 2].cpu().numpy().tobytes() == whole[:avail].tobytes(), (rate, fed)
    finally:
        ctx.close()


def test_device_memory_does_not_grow_with_the_stream():
    rate, ch = 48000, 2
    piece = _noise(10 * 60 * rate, ch, seed=3)
    pd = torch.from_numpy(piece).cuda()
    torch.cuda.synchronize()
    peaks = []
    for minutes in (10, 40):
        s = H.GetStream(channels=ch, sample_rate=rate)
        for _ in range(minutes // 10):
            s.feed(pd.data_ptr(), n_frames=piece.shape[0])
        s.finish()
        peaks.append(s.peak_bytes())
        s.close()
    mx, _ = H.chunk_geometry(MARK)
    h = int(np.ceil(16 / min(1.0, MARK / rate)))
    assert peaks[0] == peaks[1] <= (mx + (1 << 20) + 2 * h + 2) * ch * 4, peaks


def _wav_header(rate, ch, n_frames=None):
    data = 0xFFFFFFFF if n_frames is None else n_frames * ch * 2
    riff = 0xFFFFFFFF if n_frames is None else 36 + data
    return b"RIFF" + struct.pack("<I", riff) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, 1, ch, rate, rate * ch * 2, ch * 2, 16) \
        + b"data" + struct.pack("<I", data)


# the CLI's peak RSS is read by a small launcher process: Linux carries the high-water mark of a forked copy of this process (which
# holds the test audio) across exec, so a child forked from here would report at least this process's size
_LAUNCHER = r"""
import os, sys
pid = os.fork()
if pid == 0:
    os.execv(sys.argv[1], sys.argv[1:])
_, status, usage = os.wait4(pid, 0)
print(os.waitstatus_to_exitcode(status), usage.ru_maxrss * 1024)
"""


def _pipe_get_maxrss(minutes, rate=48000, ch=2):
    p = subprocess.Popen([sys.executable, "-c", _LAUNCHER, H.CLI_PATH, "-q", "get", "--chunk-size", "10", "-"], stdin=subprocess.PIPE,
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    rng = np.random.default_rng(minutes)
    p.stdin.write(_wav_header(rate, ch))
    for _ in range(minutes * 6):
        p.stdin.write(rng.integers(-3000, 3000, (10 * rate, ch), dtype=np.int16).tobytes())
    p.stdin.close()
    out = p.stdout.read().decode().split("\n")
    p.wait()
    rc, maxrss = (int(v) for v in [ln for ln in out if ln.strip()][-1].split())
    assert rc == 0
    return maxrss


def test_cli_pipe_host_memory_does_not_grow_with_the_stream():
    short, long = _pipe_get_maxrss(20), _pipe_get_maxrss(60)
    assert long - short < 128 << 20, (short, long)


def _cli(args, stdin=None):
    p = subprocess.run([H.CLI_PATH] + args, input=stdin, capture_output=True)
    return p.returncode, p.stdout


@pytest.mark.parametrize("rate", [44100, 48000])
def test_cli_file_and_pipe(tmp_path, rate):
    H.set_params()
    y = H.add(_noise(int(200 * rate), 2, seed=5), T.PAYLOAD, sample_rate=rate)
    pcm = np.clip(np.floor(y * 32768), -32768, 32767).astype(np.int16)
    data = _wav_header(rate, 2, pcm.shape[0]) + pcm.tobytes()
    wav = tmp_path / "in.wav"
    wav.write_bytes(data)
    want = H.get(pcm.astype(np.float32) / 32768, sample_rate=rate)
    results = []
    for src, stdin in ((str(wav), None), ("-", data)):
        js = tmp_path / ("%s.json" % len(results))
        rc, out = _cli(["get", "--json", str(js), src], stdin)
        assert rc == 0 and out
        import json
        assert json.loads(js.read_text()) == want
        results.append((rc, out, js.read_text(), _cli(["cmp", src, T.PAYLOAD], stdin), _cli(["cmp", src, "f" * 32], stdin)))
        rc, out = _cli(["get", "--test-truncate", "90", "--json", str(js), src], stdin)
        assert rc == 0 and json.loads(js.read_text()) == H.get(pcm[:90 * rate].astype(np.float32) / 32768, sample_rate=rate)
    assert results[0] == results[1]
    assert results[0][3][0] == 0 and results[0][4][0] == 1


def test_refusals_do_no_gpu_work():
    H.engine_ctx()
    before = H.gpu_launches()
    with pytest.raises(ValueError):
        H.GetStream(sample_rate=500)
    s = H.GetStream(channels=2, sample_rate=48000)
    with pytest.raises(ValueError):
        s.feed(np.zeros((100, 3), np.float32))
    s.finish()
    with pytest.raises(ValueError):
        s.feed(np.zeros((100, 2), np.float32))
    with pytest.raises(ValueError):
        s.finish()
    s.close()
    assert H.gpu_launches() == before
