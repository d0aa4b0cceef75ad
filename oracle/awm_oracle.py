"""awm_oracle -- CPU restatement of the reference's spectral watermark path.

TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline leg may import this module, and only as the checker.  The product
(audiowmark_b200/) never imports it and has no CPU fallback.

What it restates (citations are /root/reference/src/<file>:<lines>):
  * keyed PRNG                     random.cc:97-161, random.hh:53-113
  * key-derived tables             wmcommon.hh:91-123,165-185, wmcommon.cc:143-202,
                                   syncfinder.cc:30-77, wmadd.cc:49-162
  * convolutional code             convcode.cc:42-125 (encoder), :128-213 (Viterbi, in oracle_c.cc)
  * embed (add)                    wmcommon.cc:68-121, wmadd.cc:61-84,169-351,520-589, limiter.cc:33-124
  * sync search                    syncfinder.cc:80-658
  * block / clip decode, results   wmget.cc:40-161,163-474,492-939, wavchunkloader.cc:54-163

Parity pin: the float32 inner loops live in oracle_c.cc and use the same in-repo FFT
that backs the reference build oracle/_ref/audiowmark (the reference's own FFT is
FFTW, a third-party library that is not installed and not vendored), so this oracle
reproduces that binary's output exactly; tests/test_oracle_vs_reference.py and the
fixtures in tests/golden/ (made by tests/golden/make_golden.py with oracle/_ref)
check that.  Against a reference built on real FFTW the pin is behavioural only
(SURVEY.md section 8c): payload bits, block types and match counts.
"""
from __future__ import annotations

import ctypes
import math
import os
import struct
from dataclasses import dataclass, field

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "_build", "liboracle.so")
        if not os.path.exists(path):
            import importlib.util
            spec = importlib.util.spec_from_file_location("build_oracle", os.path.join(_HERE, "build_oracle.py"))
            mod = importlib.util.module_from_spec(spec)
            spec.loader.exec_module(mod)
            mod.build_liboracle()
        _LIB = ctypes.CDLL(path)
        _LIB.orc_viterbi.restype = ctypes.c_float
    return _LIB


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# --------------------------------------------------------------------------- params

@dataclass
class Params:
    """wmcommon.hh:33-89 / wmcommon.cc:27-58 (defaults)."""
    frame_size: int = 1024
    frames_per_bit: int = 2
    bands_per_frame: int = 30
    max_band: int = 100
    min_band: int = 20
    water_delta: float = 0.01
    mix: bool = True
    hard: bool = False
    payload_size: int = 128
    payload_short: bool = False
    sync_bits: int = 6
    sync_frames_per_bit: int = 85
    sync_search_step: int = 256
    sync_search_fine: int = 8
    sync_threshold2: float = 0.35
    get_n_best: int = 8
    frames_pad_start: int = 250
    mark_sample_rate: int = 44100
    limiter_block_size_ms: int = 1000
    limiter_ceiling: float = 0.99
    get_chunk_size: float = 30.0
    test_no_limiter: bool = False

    @property
    def n_bands(self):
        return self.max_band - self.min_band + 1


A, B, AB = 0, 1, 2          # ConvBlockType (convcode.hh:24)
BLOCK, CLIP = 0, 1          # SyncFinder::Mode
STREAM_DATA_UP_DOWN, STREAM_SYNC_UP_DOWN, STREAM_SPEED_CLIP, STREAM_MIX, STREAM_BIT_ORDER, STREAM_FRAME_POSITION = 1, 2, 3, 4, 5, 6


# --------------------------------------------------------------------------- keyed PRNG

class Key:
    """random.hh:27-47; default key = 16 zero bytes, name ''."""

    def __init__(self, aes_key: bytes = bytes(16), name: str = ""):
        assert len(aes_key) == 16
        self.aes_key = bytes(aes_key)
        self.name = name

    @staticmethod
    def test_key(n: int) -> "Key":           # random.cc:202-207
        return Key(struct.pack(">Q", n) + bytes(8), "test-key-%d" % n)

    def __eq__(self, o):
        return self.aes_key == o.aes_key and self.name == o.name

    def __hash__(self):
        return hash((self.aes_key, self.name))


class Random:
    """AES-128 CTR keystream as big-endian u64 words (random.cc:97-161)."""

    def __init__(self, key: Key, seed: int, stream: int):
        from cryptography.hazmat.primitives.ciphers import Cipher, algorithms, modes
        self._Cipher, self._alg, self._modes = Cipher, algorithms.AES(key.aes_key), modes
        self._ecb = Cipher(self._alg, modes.ECB()).encryptor()
        self.seed(seed, stream)

    def seed(self, seed: int, stream: int):          # random.cc:116-136
        plain = struct.pack(">Q", seed & 0xFFFFFFFFFFFFFFFF) + bytes([stream]) + bytes(7)
        iv = self._ecb.update(plain)
        self._ctr = self._Cipher(self._alg, self._modes.CTR(iv)).encryptor()
        self._buf = ()
        self._pos = 0

    def __call__(self) -> int:                       # random.hh:73-80, random.cc:144-161
        if self._pos == len(self._buf):
            self._buf = struct.unpack(">32Q", self._ctr.update(bytes(256)))
            self._pos = 0
        v = self._buf[self._pos]
        self._pos += 1
        return v

    def bulk_u64(self, n: int) -> np.ndarray:
        """n consecutive outputs (only valid on a freshly seeded generator)."""
        assert self._pos == len(self._buf)
        nbytes = ((n + 31) // 32) * 256
        return np.frombuffer(self._ctr.update(bytes(nbytes)), dtype=">u8")[:n].astype(np.uint64)

    def shuffle(self, seq: list):                    # random.hh:102-113
        n = len(seq)
        for i in range(n):
            j = i + self() % (n - i)
            seq[i], seq[j] = seq[j], seq[i]

    def random_double(self) -> float:                # random.hh:93-98 (libstdc++ generate_canonical, one draw)
        r = float(self()) / 18446744073709551616.0
        return math.nextafter(1.0, 0.0) if r >= 1.0 else r


def u64_to_unit_double(u: np.ndarray) -> np.ndarray:
    r = u.astype(np.float64) / 18446744073709551616.0
    return np.where(r >= 1.0, np.nextafter(1.0, 0.0), r)


def gen_noise(seconds: float, rate: int = 44100, key: Key | None = None) -> np.ndarray:
    """test_gen_noise (audiowmark.cc:399-417): stereo, Random(key, 0, data_up_down), 2u-1 -> float."""
    key = key or Key()
    n = int(rate * seconds) * 2
    rng = Random(key, 0, STREAM_DATA_UP_DOWN)
    d = u64_to_unit_double(rng.bulk_u64(n)) * 2 - 1
    return d.astype(np.float32).reshape(-1, 2)


# --------------------------------------------------------------------------- sample format helpers

def float_to_int_clip(f: np.ndarray, bits: int) -> np.ndarray:
    """rawconverter.hh:34-50."""
    inorm = 1 << (bits - 1)
    snorm = f.astype(np.float32) * np.float32(inorm)
    out = np.trunc(np.clip(snorm, -float(inorm), float(inorm))).astype(np.int64)
    out = np.where(snorm >= np.float32(inorm - 1), inorm - 1, out)
    out = np.where(snorm <= np.float32(-inorm), -inorm, out)
    return out


def quantize_sndfile16(samples: np.ndarray) -> np.ndarray:
    """16-bit file write as the reference does through libsndfile's int API
    (sfoutputstream.cc:148-155: float_to_int_clip<32>, file keeps the top 16 bits)."""
    return (float_to_int_clip(samples, 32) >> 16).astype(np.int16)


def int16_to_float(pcm: np.ndarray) -> np.ndarray:
    """sfinputstream.cc:189-210 / rawconverter.cc:257-263: left-justified int32 * 2^-31."""
    return (pcm.astype(np.int32).astype(np.float32) * np.float32(65536.0)) * np.float32(1.0 / 0x80000000)


def write_wav16(path: str, samples: np.ndarray, rate: int = 44100):
    pcm = quantize_sndfile16(samples)
    nch = pcm.shape[1]
    data = pcm.astype("<i2").tobytes()
    hdr = b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, 1, nch, rate, rate * nch * 2, nch * 2, 16)
    hdr += b"data" + struct.pack("<I", len(data))
    with open(path, "wb") as f:
        f.write(hdr + data)


def read_wav(path: str):
    """Minimal RIFF reader (PCM16/24/32, float32) -> (float32 [n, ch], rate, bits)."""
    raw = open(path, "rb").read()
    assert raw[:4] in (b"RIFF", b"RF64") and raw[8:12] == b"WAVE"
    pos, fmt, data = 12, None, None
    while pos + 8 <= len(raw):
        cid, sz = raw[pos:pos + 4], struct.unpack("<I", raw[pos + 4:pos + 8])[0]
        if cid == b"fmt ":
            fmt = struct.unpack("<HHIIHH", raw[pos + 8:pos + 24])
        elif cid == b"data":
            data = raw[pos + 8:] if sz == 0xFFFFFFFF else raw[pos + 8:pos + 8 + sz]
            break
        pos += 8 + sz + (sz & 1)
    tag, nch, rate, _, _, bits = fmt
    if tag == 3:
        x = np.frombuffer(data[:len(data) // 4 * 4], "<f4").astype(np.float32)
    elif bits == 16:
        x = int16_to_float(np.frombuffer(data[:len(data) // 2 * 2], "<i2"))
    elif bits == 32:
        x = np.frombuffer(data[:len(data) // 4 * 4], "<i4").astype(np.float32) * np.float32(1.0 / 0x80000000)
    elif bits == 24:
        b = np.frombuffer(data[:len(data) // 3 * 3], np.uint8).reshape(-1, 3).astype(np.int32)
        v = (b[:, 0] << 8) | (b[:, 1] << 16) | (b[:, 2] << 24)
        x = v.astype(np.int32).astype(np.float32) * np.float32(1.0 / 0x80000000)
    else:
        raise ValueError("unsupported wav")
    n = len(x) // nch
    return x[:n * nch].reshape(n, nch), rate, bits


# --------------------------------------------------------------------------- bits / payload

def bit_str_to_vec(s: str) -> list:                  # utils.cc:95-111
    out = []
    for ch in s:
        try:
            c = int(ch, 16)
        except ValueError:
            return []
        out += [(c >> 3) & 1, (c >> 2) & 1, (c >> 1) & 1, c & 1]
    return out


def bit_vec_to_str(v) -> str:                        # utils.cc:113-133
    s = ""
    for pos in range(0, len(v) - 3, 4):
        nib = 0
        for j in range(4):
            if v[pos + j]:
                nib |= 1 << (3 - j)
        s += "0123456789abcdef"[nib]
    return s


def parse_payload(bits: str, P: Params) -> list:     # wmcommon.cc:210-238
    v = bit_str_to_vec(bits)
    if P.payload_short and len(v) != P.payload_size:
        return []
    if not v or len(v) > P.payload_size:
        return []
    if len(v) < P.payload_size:
        v = [v[i % len(v)] for i in range(P.payload_size)]
    return v


# --------------------------------------------------------------------------- convolutional code

AB_GENERATORS = [0o66561, 0o75211, 0o71545, 0o54435, 0o63635, 0o52475,
                 0o63543, 0o75307, 0o52547, 0o45627, 0o67657, 0o51757]   # convcode.cc:42-46
ORDER = 15


def block_generators(block_type: int) -> list:       # convcode.cc:77-98
    if block_type == A:
        return AB_GENERATORS[0::2]
    if block_type == B:
        return AB_GENERATORS[1::2]
    return list(AB_GENERATORS)


def conv_code_size(block_type: int, msg_size: int) -> int:   # convcode.cc:65-75
    return (msg_size + ORDER) * 12 // 2 if block_type in (A, B) else (msg_size + ORDER) * 12


def conv_encode(block_type: int, in_bits: list) -> list:     # convcode.cc:100-125
    gens = block_generators(block_type)
    out, reg = [], 0
    for b in list(in_bits) + [0] * ORDER:
        reg = ((reg << 1) | b) & 0xFFFFFFFF
        for poly in gens:
            out.append(bin(reg & poly).count("1") & 1)
    return out


def conv_decode_soft(block_type: int, coded: np.ndarray):    # convcode.cc:128-213
    gens = np.array(block_generators(block_type), dtype=np.uint32)
    coded = np.ascontiguousarray(coded, dtype=np.float32)
    steps = len(coded) // len(gens)
    dec = np.zeros(steps, dtype=np.int32)
    err = lib().orc_viterbi(_p(gens), ctypes.c_int(len(gens)), ctypes.c_int(ORDER), _p(coded), ctypes.c_int64(len(coded)), _p(dec))
    return [int(b) for b in dec[:steps - ORDER]], float(err)


# --------------------------------------------------------------------------- key-derived tables

SHORT_CODES = {      # shortcode.cc:26-83: best known linear codes [n, k] over GF(2); row i as a bit mask, bit j = column j
    12: (56, [0xfeb8b646cb1001, 0x05d0daf7f1b002, 0x68aec1274e8804, 0x73c692698c2808, 0xda51f4b6048810, 0x57617a230f1020, 0xb9eda54a308040, 0x3f9dfcd0163080, 0xd4b8e8ef2d2900, 0x6b339794612200, 0x8acc5794991c00, 0x9ff7fc1fffc000]),
    16: (61, [0x0498284fd74f0001, 0x0930509fae9e0002, 0x1260a13f5d3c0004, 0x139f97d14b610008, 0x1061fa0d67db0010, 0x179d21b53eaf0020, 0x186496c58c470040, 0x0797f824e9970080, 0x0f2ff049d32e0100, 0x1e5fe093a65c0200, 0x0be11488bda10400, 0x17c229117b420800, 0x18da878d079d1000, 0x06ebdab5fe232000, 0x0dd7b56bfc464000, 0x1baf6ad7f88c8000]),
    20: (65, [0x1dcfaff02fec40001, 0x1fb826f058a840002, 0x1b5734f0b62040004, 0x128910f16b3040008, 0x013558f2d11040010, 0x1ab9a385b11e00020, 0x1448828b599e00040, 0x09aac096889e00080, 0x0e9a2fdd3ed040100, 0x05e74dda6e9e00200, 0x16013544f2d040400, 0x08251299e2d440800, 0x08993753d69601000, 0x0cfdc15782c442000, 0x012891cf16b204000, 0x1f9e8d6e028848000, 0x1b1a62cc026450000, 0x1213bc8803b860000, 0x18d31360133a80000, 0x109de2401dd300000]),
}


def short_encode_blk(in_bits, k):                    # shortcode.cc:136-157
    n, rows = SHORT_CODES[k]
    w = 0
    for bit in range(k):
        if in_bits[bit]:
            w ^= rows[bit]
    return [(w >> j) & 1 for j in range(n)]


def short_decode_blk(coded_bits, k):                 # shortcode.cc:171-213 (first message whose code word matches; [] if none)
    n, rows = SHORT_CODES[k]
    r = 0
    for j, b in enumerate(coded_bits):
        r |= (int(b) & 1) << j
    table = _short_codebook(k)
    c = table.get(r)
    return [] if c is None else [(c >> bit) & 1 for bit in range(k)]


_SHORT_BOOK = {}


def _short_codebook(k):
    if k not in _SHORT_BOOK:
        n, rows = SHORT_CODES[k]
        book = {0: 0}
        words = [0]
        for bit in range(k):                          # gray-free doubling: words of messages < 2^(bit+1)
            words = words + [w ^ rows[bit] for w in words]
        for c, w in enumerate(words):
            book.setdefault(w, c)                    # ascending message order: first match wins
        _SHORT_BOOK[k] = book
    return _SHORT_BOOK[k]


def code_message_bits(P: Params) -> int:
    return SHORT_CODES[P.payload_size][0] if P.payload_short else P.payload_size


def code_size(block_type: int, P: Params) -> int:    # shortcode.cc:123-127
    return conv_code_size(block_type, code_message_bits(P))


def code_encode(block_type: int, in_bits: list, P: Params) -> list:      # shortcode.cc:117-121
    return conv_encode(block_type, short_encode_blk(in_bits, P.payload_size) if P.payload_short else in_bits)


def code_decode_soft(block_type: int, coded, P: Params):                 # shortcode.cc:129-133
    bits, err = conv_decode_soft(block_type, coded)
    if P.payload_short:
        bits = short_decode_blk(bits, P.payload_size)
    return bits, err


def mark_data_frame_count(P: Params) -> int:         # wmcommon.cc:167-171
    return code_size(A, P) * P.frames_per_bit


def mark_sync_frame_count(P: Params) -> int:         # wmcommon.cc:173-177
    return P.sync_bits * P.sync_frames_per_bit


def frames_per_block(P: Params) -> int:
    return mark_data_frame_count(P) + mark_sync_frame_count(P)


class UpDownGen:                                     # wmcommon.hh:91-123
    def __init__(self, key: Key, stream: int, P: Params):
        self.stream, self.P = stream, P
        self.random = Random(key, 0, stream)

    def get(self, f: int):
        P = self.P
        bands = list(range(P.min_band, P.max_band + 1))
        self.random.seed(f, self.stream)
        self.random.shuffle(bands)
        return bands[:P.bands_per_frame], bands[P.bands_per_frame:2 * P.bands_per_frame]


class BitPosGen:                                     # wmcommon.cc:143-165
    def __init__(self, key: Key, P: Params):
        self.P = P
        self.pos = list(range(frames_per_block(P)))
        Random(key, 0, STREAM_FRAME_POSITION).shuffle(self.pos)

    def sync_frame(self, f):
        return self.pos[f]

    def data_frame(self, f):
        return self.pos[f + mark_sync_frame_count(self.P)]


def gen_mix_entries(key: Key, P: Params) -> list:    # wmcommon.cc:179-202
    udg, bpg = UpDownGen(key, STREAM_DATA_UP_DOWN, P), BitPosGen(key, P)
    entries = []
    for f in range(mark_data_frame_count(P)):
        idx = bpg.data_frame(f)
        up, down = udg.get(f)
        entries += [(idx, u, d) for u, d in zip(up, down)]
    Random(key, 0, STREAM_MIX).shuffle(entries)
    return entries


def randomize_bit_order(key: Key, vec, encode: bool):  # wmcommon.hh:165-185
    order = list(range(len(vec)))
    Random(key, 0, STREAM_BIT_ORDER).shuffle(order)
    out = [0] * len(vec)
    for i in range(len(vec)):
        if encode:
            out[i] = vec[order[i]]
        else:
            out[order[i]] = vec[i]
    return out


KEEP, UP, DOWN = 0, 1, 2


def init_frame_mod(key: Key, ab: int, bitvec: list, P: Params) -> np.ndarray:
    """wmadd.cc:49-59,86-162 -> uint8 [frames_per_block][max_band+1]."""
    fm = np.zeros((frames_per_block(P), P.max_band + 1), dtype=np.uint8)
    fec = randomize_bit_order(key, code_encode(B if ab else A, bitvec, P), True)
    # mark_sync (wmadd.cc:129-146)
    udg, bpg = UpDownGen(key, STREAM_SYNC_UP_DOWN, P), BitPosGen(key, P)
    for f in range(mark_sync_frame_count(P)):
        idx = bpg.sync_frame(f)
        bit = (f // P.sync_frames_per_bit + ab) & 1
        up, down = udg.get(f)
        fm[idx, up] = UP if bit else DOWN
        fm[idx, down] = DOWN if bit else UP
    # mark_data (wmadd.cc:86-127)
    if P.mix:
        mix = gen_mix_entries(key, P)
        for f in range(mark_data_frame_count(P)):
            bit = fec[f // P.frames_per_bit]
            for fb in range(P.bands_per_frame):
                idx, u, d = mix[f * P.bands_per_frame + fb]
                fm[idx, u] = UP if bit else DOWN
                fm[idx, d] = DOWN if bit else UP
    else:
        udg = UpDownGen(key, STREAM_DATA_UP_DOWN, P)
        for f in range(mark_data_frame_count(P)):
            idx = bpg.data_frame(f)
            bit = fec[f // P.frames_per_bit]
            up, down = udg.get(f)
            fm[idx, up] = UP if bit else DOWN
            fm[idx, down] = DOWN if bit else UP
    return fm


@dataclass
class SyncBits:
    """syncfinder.cc:30-77 flattened: bit b owns entries off[b]..off[b+1]."""
    off: np.ndarray
    frame: np.ndarray
    up: np.ndarray
    down: np.ndarray


def get_sync_bits(key: Key, mode: int, P: Params) -> SyncBits:
    first_block_end = frames_per_block(P)
    block_count = 2 if mode == CLIP else 1
    udg, bpg = UpDownGen(key, STREAM_SYNC_UP_DOWN, P), BitPosGen(key, P)
    off, frames, ups, downs = [0], [], [], []
    for bit in range(P.sync_bits):
        fbs = []
        for f in range(P.sync_frames_per_bit):
            fu, fd = udg.get(f + bit * P.sync_frames_per_bit)
            for block in range(block_count):
                fr = bpg.sync_frame(f + bit * P.sync_frames_per_bit) + block * first_block_end
                u = [x - P.min_band for x in (fu if block == 0 else fd)]
                d = [x - P.min_band for x in (fd if block == 0 else fu)]
                fbs.append((fr, sorted(u), sorted(d)))
        fbs.sort(key=lambda t: t[0])
        for fr, u, d in fbs:
            frames.append(fr); ups.append(u); downs.append(d)
        off.append(len(frames))
    return SyncBits(np.array(off, np.int32), np.array(frames, np.int32),
                    np.array(ups, np.int32).reshape(-1), np.array(downs, np.int32).reshape(-1))


# --------------------------------------------------------------------------- FFT analysis

def window_cos(x):                                   # wmcommon.hh:187-193
    return np.where(np.abs(x) > 1, 0.0, 0.5 * np.cos(x * np.pi) + 0.5)


def gen_normalized_window(n: int) -> np.ndarray:     # wmcommon.cc:68-89
    i = np.arange(n, dtype=np.float64)
    win = window_cos((i - n / 2.0) / (n / 2.0)).astype(np.float32)   # window[i] = win (float store)
    weight = 0.0
    for w in window_cos((i - n / 2.0) / (n / 2.0)):                  # double running sum
        weight += w
    return (win.astype(np.float64) * (2.0 / weight)).astype(np.float32)  # window[i] *= 2.0 / weight


_WINDOWS = {}


def analysis_window(n: int) -> np.ndarray:
    if n not in _WINDOWS:
        _WINDOWS[n] = gen_normalized_window(n)
    return _WINDOWS[n]


def analyze_frames(samples: np.ndarray, starts, n: int = 1024) -> np.ndarray:
    """FFTAnalyzer::run_fft for many start positions -> complex64 [jobs][ch][n/2+1]."""
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    nch = samples.shape[1]
    starts = np.ascontiguousarray(starts, dtype=np.int64)
    assert len(starts) == 0 or (starts.min() >= 0 and starts.max() + n <= samples.shape[0])
    out = np.zeros((len(starts), nch, n + 2), dtype=np.float32)
    win = analysis_window(n)
    lib().orc_analyze_frames(_p(samples), ctypes.c_int(nch), _p(starts), ctypes.c_int64(len(starts)), _p(win), ctypes.c_int(n), _p(out))
    return out


def db_bands(spect: np.ndarray, P: Params) -> np.ndarray:
    jobs, nch, n2 = spect.shape
    out = np.zeros((jobs, P.n_bands), dtype=np.float32)
    lib().orc_db_bands(_p(np.ascontiguousarray(spect)), ctypes.c_int64(jobs), ctypes.c_int(nch), ctypes.c_int(n2 - 2),
                       ctypes.c_int(P.min_band), ctypes.c_int(P.max_band), _p(out))
    return out


# --------------------------------------------------------------------------- embed

def synth_window(P: Params) -> np.ndarray:           # wmadd.cc:177-206
    n = P.frame_size
    i = np.arange(3 * n, dtype=np.float64)
    norm_pos = (i - n) / n
    norm_pos = np.where(norm_pos > 0.5, 1 - norm_pos, norm_pos)
    overlap = 0.1
    tri = np.where(norm_pos < -overlap, 0.0, np.where(norm_pos < overlap, 0.5 + norm_pos / (2 * overlap), 1.0))
    return ((np.cos(tri * np.pi + np.pi) + 1) * 0.5).astype(np.float32)


def limiter(x: np.ndarray, rate: int, P: Params) -> np.ndarray:
    """limiter.cc:33-124 on a zero-extended signal x [n, ch] (see add_stream_watermark :539-546)."""
    n, nch = x.shape
    bs = rate * P.limiter_block_size_ms // 1000
    ceiling = np.float32(P.limiter_ceiling)
    nblocks = (n + bs - 1) // bs
    bm = np.full(nblocks + 2, ceiling, dtype=np.float32)          # bm[b+1] = block b, bm[0] = "last" before start
    for b in range(nblocks):
        seg = x[b * bs:(b + 1) * bs]
        if seg.size:
            bm[b + 1] = max(ceiling, np.float32(np.abs(seg).max()))
    out = np.empty_like(x)
    i_f = np.arange(bs, dtype=np.float32)
    for b in range(nblocks):
        last, cur, nxt = bm[b], bm[b + 1], bm[b + 2]
        scale_start = ceiling / max(last, cur)
        scale_end = ceiling / max(cur, nxt)
        scale_step = np.float32(scale_end - scale_start) / np.float32(bs)
        scale = scale_start + i_f * scale_step
        seg = x[b * bs:(b + 1) * bs]
        out[b * bs:(b + 1) * bs] = seg * scale[:len(seg), None]
    return out


@dataclass
class EmbedResult:
    samples: np.ndarray
    data_blocks: int
    snr_db: float
    wm: np.ndarray = None


def embed(samples: np.ndarray, key: Key, bits: str, P: Params | None = None, rate: int = 44100, keep_wm: bool = False) -> EmbedResult:
    """add_stream_watermark (wmadd.cc:448-618), zero_frames = 0; other rates than 44.1 kHz go through embed_resampled."""
    P = P or Params()
    if rate != P.mark_sample_rate:
        return embed_resampled(samples, key, bits, P, rate, keep_wm)
    bitvec = parse_payload(bits, P)
    assert bitvec, "bad payload"
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    n, nch = samples.shape
    N = P.frame_size
    F = (n + N - 1) // N
    fpb = frames_per_block(P)
    ext = np.zeros(((F + 1) * N, nch), dtype=np.float32)
    ext[:n] = samples

    fm_tab = [init_frame_mod(key, 0, bitvec, P), init_frame_mod(key, 1, bitvec, P)]
    spect = analyze_frames(ext, np.arange(F, dtype=np.int64) * N, N)          # [F][ch][N+2]
    delta = np.zeros_like(spect)
    L = lib()
    for f in range(F):
        r = (2 * fpb - P.frames_pad_start + f) % (2 * fpb)                  # wmadd.cc:295,326-344
        fm = fm_tab[1][r - fpb] if r >= fpb else fm_tab[0][r]
        for ch in range(nch):
            L.orc_apply_frame_mod(_p(fm), ctypes.c_int(len(fm)), _p(spect[f, ch]), _p(delta[f, ch]), ctypes.c_double(P.water_delta))
    wmf = np.zeros((F + 2, nch, N), dtype=np.float32)                        # wmf[f+1] = ifft of frame f; wmf[0], wmf[F+1] = 0
    tmp = np.zeros((F * nch, N), dtype=np.float32)
    L.orc_irfft(_p(delta), _p(tmp), ctypes.c_int(N), ctypes.c_int64(F * nch))
    wmf[1:F + 1] = tmp.reshape(F, nch, N)

    w = synth_window(P)
    w0, w1, w2 = w[:N], w[N:2 * N], w[2 * N:]
    # output frame m = ((0 + wm[m-1]*w2) + wm[m]*w1) + wm[m+1]*w0      (wmadd.cc:215-250, one frame of delay)
    a = wmf[0:F + 1] * w2
    b = wmf[1:F + 2] * w1
    wm = (a + b)
    wm[:F] = wm[:F] + wmf[2:F + 2] * w0
    wm = np.ascontiguousarray(wm.transpose(0, 2, 1)).reshape((F + 1) * N, nch)
    mixed = wm + ext                                                          # wmadd.cc:564-565
    bs = rate * P.limiter_block_size_ms // 1000
    runs = embed_gen_runs(n, N, not P.test_no_limiter, bs)
    # --snr sums every frame the loop emits (runs - 1 of them, wmadd.cc:553-563): the zero-padded tail of the last
    # frame always, the spill frame F only when the limiter keeps the loop running
    d = wm[:min(runs - 1, F + 1) * N].astype(np.float64)
    o = samples.astype(np.float64)
    snr = 10 * math.log10((o * o).sum() / max((d * d).sum(), 1e-300))
    out = mixed if P.test_no_limiter else limiter(mixed, rate, P)
    # data block counter (wmadd.cc:311-313,345-350): number of WatermarkGen::run calls made by the loop
    f0 = 2 * fpb - P.frames_pad_start
    m_data_blocks = (f0 + runs) // fpb - f0 // fpb
    return EmbedResult(out[:n].copy(), max(m_data_blocks - 1, 0), snr, wm[:n].copy() if keep_wm else None)


def embed_resampled(samples: np.ndarray, key: Key, bits: str, P: Params, rate: int, keep_wm: bool = False) -> EmbedResult:
    """add_stream_watermark with WatermarkResampler (wmadd.cc:353-430, 520-589): the input is resampled to the watermark
    rate, WatermarkGen produces the watermark signal there, it is resampled back and added to the untouched input; the
    limiter runs at the input rate.  Whole-buffer restatement of the streaming loop: zero frames keep being fed after
    EOF, so both resamplers see zero-extended signals."""
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    n, nch = samples.shape
    N = P.frame_size
    n_emit, runs = resampled_add_plan(n, rate, P)
    r_in, r_out = float(P.mark_sample_rate) / rate, float(rate) / P.mark_sample_rate
    h_out = int(math.ceil(16 / min(1.0, r_out)))
    top = int(math.floor((n_emit - 1) * (1.0 / r_out))) + h_out            # highest watermark-rate frame any emitted output touches
    n44 = (top // N + 1) * N
    xz = np.zeros((n + 4 * 64, nch), np.float32)                           # post-roll >> filter length: true zero extension
    xz[:n] = samples
    x44 = resample_ratio(xz, r_in, n_out=n44)
    Pn = Params(**{**{k: getattr(P, k) for k in Params.__annotations__}, "test_no_limiter": True})
    wm44 = embed(x44, key, bits, Pn, P.mark_sample_rate, keep_wm=True).wm  # WatermarkGen::run output of every frame
    wm = resample_ratio(wm44, r_out, n_out=n_emit)
    ext = np.zeros((n_emit, nch), np.float32)
    ext[:n] = samples
    mixed = wm + ext                                                        # wmadd.cc:564-565
    d = wm.astype(np.float64)
    o = samples.astype(np.float64)
    snr = 10 * math.log10((o * o).sum() / max((d * d).sum(), 1e-300))       # wmadd.cc:553-563 over everything emitted
    out = mixed if P.test_no_limiter else limiter(mixed, rate, P)
    fpb = frames_per_block(P)
    f0 = 2 * fpb - P.frames_pad_start
    m_data_blocks = (f0 + runs) // fpb - f0 // fpb
    return EmbedResult(out[:n].copy(), max(m_data_blocks - 1, 0), snr, wm[:n].copy() if keep_wm else None)


def embed_gen_runs(n: int, N: int, limiter_on: bool, bs: int) -> int:
    """How often the loop wmadd.cc:520-589 calls WatermarkGen::run: zero frames keep being fed
    after EOF until total_output == total_input; the synth delays by one frame (wmadd.cc:240-249)
    and the limiter holds back until two complete blocks are buffered (limiter.cc:53-58)."""
    if n == 0:
        return 0
    if not limiter_on:
        return 1 + (n + N - 1) // N
    need = ((n + bs - 1) // bs + 1) * bs
    return 1 + (need + N - 1) // N


# --------------------------------------------------------------------------- sync finder

@dataclass
class SearchScore:
    index: int
    raw_quality: float
    local_mean: float = 0.0

    def abs_quality(self):
        return abs(self.raw_quality - self.local_mean)


@dataclass
class Score:
    index: int
    quality: float
    block_type: int


class SyncFinder:
    local_mean_distance = 20

    def __init__(self, P: Params):
        self.P = P
        self.first = 0
        self.last = 0

    # -- sync_fft (syncfinder.cc:560-605)
    def sync_fft(self, samples, index, frame_count, want):
        P, N = self.P, self.P.frame_size
        n, nch = samples.shape
        if n * nch < (index + frame_count * N) * nch:
            return None, None
        f = np.arange(frame_count, dtype=np.int64)
        f_first = (index + f * N) * nch
        f_last = (index + (f + 1) * N) * nch
        ok = ~((f_last < self.first) | (f_first > self.last))
        if want is not None:
            ok &= want.astype(bool)
        db = np.zeros((frame_count, P.n_bands), dtype=np.float32)
        sel = np.nonzero(ok)[0]
        if len(sel):
            for c0 in range(0, len(sel), 8192):
                s = sel[c0:c0 + 8192]
                db[s] = db_bands(analyze_frames(samples, index + s * N, N), P)
        return db, ok.astype(np.int8)

    def sync_decode(self, sb: SyncBits, start_frames, db, have):
        start_frames = np.ascontiguousarray(start_frames, dtype=np.int64)
        q = np.zeros(len(start_frames), dtype=np.float64)
        P = self.P
        lib().orc_sync_decode(_p(db), _p(have), ctypes.c_int(P.n_bands), ctypes.c_int(P.sync_bits), _p(sb.off), _p(sb.frame),
                              _p(sb.up), _p(sb.down), ctypes.c_int(P.bands_per_frame), _p(start_frames),
                              ctypes.c_int64(len(start_frames)), ctypes.c_double(P.water_delta), _p(q))
        return q

    # -- search_approx (syncfinder.cc:171-256)
    def search_approx(self, sb: SyncBits, samples, mode):
        P, N = self.P, self.P.frame_size
        n, nch = samples.shape
        fc = (n * nch) // nch // N
        total = frames_per_block(P) * (2 if mode == CLIP else 1)
        idx_all, q_all = [], []
        for shift in range(0, N, P.sync_search_step):
            nfr = max(fc - 1, 0)
            if nfr == 0:
                continue
            db, have = self.sync_fft(samples, shift, nfr, None)
            starts = np.arange(max(fc, 0), dtype=np.int64)
            starts = starts[(starts + total) * P.n_bands < nfr * P.n_bands]
            if len(starts) == 0:
                continue
            q = self.sync_decode(sb, starts, db, have)
            idx_all.append(starts * N + shift)
            q_all.append(q)
        if not idx_all:
            return []
        idx = np.concatenate(idx_all)
        q = np.concatenate(q_all)
        order = np.argsort(idx, kind="stable")
        idx, q = idx[order], q[order]
        # local mean (:234-254): sequential double sum over j = -20..20, |j| >= 4
        m = len(q)
        lm = np.zeros(m)
        cnt = np.zeros(m, dtype=np.int64)
        for j in range(-self.local_mean_distance, self.local_mean_distance + 1):
            if abs(j) >= 4:
                lo, hi = max(0, -j), min(m, m - j)
                if hi > lo:
                    lm[lo:hi] += q[lo + j:hi + j]
                    cnt[lo:hi] += 1
        lm = np.where(cnt > 0, lm / np.maximum(cnt, 1), lm)
        return [SearchScore(int(i), float(r), float(l)) for i, r, l in zip(idx, q, lm)]

    # -- selectors (syncfinder.cc:258-391)
    @staticmethod
    def select_local_maxima(scores):
        out, i, m = [], 0, len(scores)
        while i < m:
            qv = scores[i].abs_quality()
            ql = scores[i - 1].abs_quality() if i > 0 else 0
            qn = scores[i + 1].abs_quality() if i + 1 < m else 0
            if qv >= ql and qv >= qn:
                out.append(scores[i])
                i += 1
            i += 1
        return out

    def mask_avg_false_positives(self, scores):
        mask_distance, mask_factor = self.local_mean_distance + 3, 3
        m = len(scores)
        if m == 0:
            return scores
        idx = np.array([s.index for s in scores], dtype=np.int64)
        d = np.array([s.raw_quality - s.local_mean for s in scores])
        aq = np.abs(d)
        sign = np.where(d < 0, -1, 1)
        masked = np.zeros(m, dtype=bool)
        for dd in range(-mask_distance, mask_distance + 1):
            if dd == 0:
                continue
            lo, hi = max(0, -dd), min(m, m - dd)
            if hi <= lo:
                continue
            i = np.arange(lo, hi)
            j = i + dd
            dist = np.abs(idx[i] - idx[j]) // self.P.sync_search_step
            cond = (dist <= mask_distance) & (aq[j] > aq[i] * mask_factor) & (sign[j] != sign[i])
            masked[i] |= cond
        return [s for s, mk in zip(scores, masked) if not mk]

    @staticmethod
    def std_sort_desc(scores):
        """std::sort by descending abs_quality, unstable like the reference's (ties: see orc_std_sort_desc)"""
        keys = np.array([s.abs_quality() for s in scores], dtype=np.float64)
        perm = np.zeros(len(scores), dtype=np.int64)
        if len(scores):
            lib().orc_std_sort_desc(_p(keys), ctypes.c_int64(len(scores)), _p(perm))
        return [scores[i] for i in perm]

    def select_threshold_and_n_best(self, scores, threshold):
        scores = self.std_sort_desc(scores)
        i = 0
        while i < len(scores) and scores[i].abs_quality() > threshold:
            i += 1
        if i >= self.P.get_n_best:
            return scores[:i]
        if len(scores) > self.P.get_n_best:
            return scores[:self.P.get_n_best]
        return scores

    def select_truncate_n(self, scores, n):
        return self.std_sort_desc(scores)[:n]

    # -- search_refine (syncfinder.cc:393-458)
    def refine_qualities(self, samples, mode, index, sb: SyncBits, key: Key):
        """the fine offsets search_refine scores around one approx index -> [(fine, quality or None if past the end)]"""
        P = self.P
        total = frames_per_block(P)
        first_block_end = total
        if mode == CLIP:
            total *= 2
        bpg = BitPosGen(key, P)
        want = np.zeros(total, dtype=np.int8)
        for f in range(mark_sync_frame_count(P)):
            want[bpg.sync_frame(f)] = 1
            if mode == CLIP:
                want[first_block_end + bpg.sync_frame(f)] = 1
        out = []
        start = max(int(index) - P.sync_search_step, 0)
        for fine in range(start, int(index) + P.sync_search_step + 1, P.sync_search_fine):
            db, have = self.sync_fft(samples, fine, total, want)
            out.append((fine, None if db is None else float(self.sync_decode(sb, [0], db, have)[0])))
        return out

    def search_refine(self, samples, mode, scores, sb: SyncBits, key: Key):
        out = []
        for sc in scores:
            best_q, best_i = sc.raw_quality, sc.index
            for fine, q in self.refine_qualities(samples, mode, sc.index, sb, key):
                if q is not None and abs(q - sc.local_mean) > abs(best_q - sc.local_mean):
                    best_q, best_i = q, fine
            out.append(SearchScore(best_i, best_q, sc.local_mean))
        out.sort(key=lambda s: s.index)
        return out

    # -- search (syncfinder.cc:487-558)
    def search(self, key: Key, samples, mode, stages: dict | None = None):
        P = self.P
        samples = np.ascontiguousarray(samples, dtype=np.float32)
        flat = samples.reshape(-1)
        if mode == CLIP:                             # scan_silence :155-169
            nz = np.nonzero(flat)[0]
            if len(nz):
                self.first, self.last = int(nz[0]), int(nz[-1]) + 1
            else:
                self.first, self.last = len(flat), len(flat)
        else:
            self.first, self.last = 0, len(flat)
        sb = get_sync_bits(key, mode, P)
        scores = self.search_approx(sb, samples, mode)
        if stages is not None:
            stages["approx"] = scores
        scores = self.select_local_maxima(scores)
        scores = self.mask_avg_false_positives(scores)
        scores = self.select_threshold_and_n_best(scores, P.sync_threshold2 * 0.75)
        if mode == CLIP:
            scores = self.select_truncate_n(scores, max(P.get_n_best, 5))
        if stages is not None:
            stages["selected"] = list(scores)
        scores = self.search_refine(samples, mode, scores, sb, key)
        if stages is not None:
            stages["refined"] = list(scores)
        scores = self.select_threshold_and_n_best(scores, P.sync_threshold2)
        scores.sort(key=lambda s: s.index)
        out = []
        for s in scores:
            q = s.raw_quality - s.local_mean
            out.append(Score(s.index, abs(q), A if q > 0 else B))
        return out


# --------------------------------------------------------------------------- decode

def fft_range(samples, index, count, P: Params):     # wmcommon.cc:123-141
    n, nch = samples.shape
    if n * nch < (index + count * P.frame_size) * nch:
        return None
    sp = analyze_frames(samples, index + np.arange(count, dtype=np.int64) * P.frame_size, P.frame_size)
    return sp.reshape(count * nch, P.frame_size + 2)


_MIX_CACHE = {}


def _mix_arrays(key: Key, P: Params):
    k = (key.aes_key, P.payload_size, P.frames_per_bit, P.payload_short)
    if k not in _MIX_CACHE:
        m = gen_mix_entries(key, P)
        _MIX_CACHE[k] = tuple(np.array([e[i] for e in m], dtype=np.int32) for i in range(3))
    return _MIX_CACHE[k]


def mix_decode(key: Key, spect, nch, P: Params) -> np.ndarray:      # wmget.cc:67-108
    fc = mark_data_frame_count(P)
    mf, mu, md = _mix_arrays(key, P)
    out = np.zeros(fc // P.frames_per_bit, dtype=np.float32)
    lib().orc_mix_decode(_p(spect), ctypes.c_int64(spect.shape[0]), ctypes.c_int(P.frame_size), ctypes.c_int(nch),
                         _p(mf), _p(mu), _p(md), ctypes.c_int(fc), ctypes.c_int(P.bands_per_frame), ctypes.c_int(P.frames_per_bit), _p(out))
    return out


def linear_decode(key: Key, spect, nch, P: Params) -> np.ndarray:   # wmget.cc:110-152
    fc = mark_data_frame_count(P)
    k = ("linear", key.aes_key, P.payload_size, P.frames_per_bit, P.payload_short)
    if k not in _MIX_CACHE:                              # key tables are the same for every block: build them once
        udg, bpg = UpDownGen(key, STREAM_DATA_UP_DOWN, P), BitPosGen(key, P)
        df, up, down = [], [], []
        for f in range(fc):
            df.append(bpg.data_frame(f))
            u, d = udg.get(f)
            up += u; down += d
        _MIX_CACHE[k] = tuple(np.array(x, dtype=np.int32) for x in (df, up, down))
    df, up, down = _MIX_CACHE[k]
    out = np.zeros(fc // P.frames_per_bit, dtype=np.float32)
    lib().orc_linear_decode(_p(spect), ctypes.c_int64(spect.shape[0]), ctypes.c_int(P.frame_size), ctypes.c_int(nch),
                            _p(df), _p(up), _p(down), ctypes.c_int(fc), ctypes.c_int(P.bands_per_frame), ctypes.c_int(P.frames_per_bit), _p(out))
    return out


def raw_bits_for_block(key: Key, samples, index, P: Params):
    sp = fft_range(samples, index, frames_per_block(P), P)
    if sp is None:
        return None
    raw = mix_decode(key, sp, samples.shape[1], P) if P.mix else linear_decode(key, sp, samples.shape[1], P)
    return np.array(randomize_bit_order(key, list(raw), False), dtype=np.float32)


def normalize_soft_bits(soft, P: Params) -> np.ndarray:             # wmget.cc:40-65
    soft = np.asarray(soft, dtype=np.float32)
    if P.hard:
        return (soft > 0).astype(np.float32)
    mean = float(np.cumsum(np.abs(soft).astype(np.float64))[-1]) / len(soft)
    return (0.5 * (soft.astype(np.float64) / mean + 1)).astype(np.float32)


TYPE_BLOCK, TYPE_CLIP, TYPE_ALL = 0, 1, 2


@dataclass
class Pattern:
    key: Key
    time: float
    bit_vec: list
    decode_error: float
    sync_score: Score
    type: int
    speed: float = 1.0
    rating: float = 0.0

    def approx_match(self, p):                       # wmget.cc:178-190
        time_delta = 1024 / 44100.0
        return (self.key == p.key and (abs(self.time - p.time) < time_delta or self.type == TYPE_ALL)
                and self.bit_vec == p.bit_vec and self.sync_score.block_type == p.sync_score.block_type
                and self.type == p.type and abs(self.speed - p.speed) < 0.01)

    def block_str(self):
        s = {A: "A", B: "B", AB: "AB"}[self.sync_score.block_type]
        if self.type == TYPE_CLIP:
            s = "CLIP-" + s
        if self.speed != 1:
            s += "-SPEED"
        return s


class ResultSet:                                     # wmget.cc:163-474
    def __init__(self):
        self.patterns = []
        self.debug_sync = ""

    def add_pattern(self, key, time, sync_score, bit_vec, decode_error, ptype, speed=1.0):
        if not len(bit_vec):                         # short payload: no code word matched (wmget.cc:549,594,698,814)
            return
        self.patterns.append(Pattern(key, time, list(bit_vec), np.float32(decode_error), sync_score, ptype, speed))

    def apply_time_offset(self, off):
        for p in self.patterns:
            p.time += off

    def merge(self, other):
        for p in sorted(other.patterns, key=lambda p: p.time):
            if not any(mp.approx_match(p) for mp in self.patterns):
                self.patterns.append(p)
        if not self.debug_sync:
            self.debug_sync = other.debug_sync

    def sort(self, key_list):
        for key in key_list:
            rating = {}
            for p in self.patterns:
                if p.key == key:
                    bits = bit_vec_to_str(p.bit_vec)
                    # map<string,float> accumulation (wmget.cc:184-200)
                    rating[bits] = np.float32(float(rating.get(bits, 0.0)) + p.sync_score.quality * (2.0 if p.type == TYPE_ALL else 1.0))
            for p in self.patterns:
                if p.key == key:
                    p.rating = float(rating[bit_vec_to_str(p.bit_vec)])
        self.patterns.sort(key=lambda p: (p.key.name, -p.rating, 1 if p.type == TYPE_ALL else 0, p.time,
                                          p.sync_score.block_type, bit_vec_to_str(p.bit_vec)))

    def lines(self):                                 # print() wmget.cc:384-441
        out, last_key, print_speed = [], "", True
        for p in self.patterns:
            if p.key.name != last_key:
                out.append("key %s" % p.key.name)
                last_key = p.key.name
                print_speed = True                   # one speed per key (wmget.cc:391-406)
            if print_speed:
                for q in self.patterns:
                    if q.key == p.key and q.speed != 1:
                        out.append("speed %.6f" % q.speed)
                        break
                print_speed = False
            if p.type == TYPE_ALL:
                out.append("pattern   all %s %.3f %.3f%s" % (bit_vec_to_str(p.bit_vec), p.sync_score.quality, p.decode_error, " SPEED" if p.speed != 1 else ""))
            else:
                sec = int(p.time)
                out.append("pattern %2d:%02d %s %.3f %.3f %s" % (sec // 60, sec % 60, bit_vec_to_str(p.bit_vec), p.sync_score.quality, p.decode_error, p.block_str()))
        return out

    def json_doc(self, time_length: int) -> dict:
        """print_json (wmget.cc:339-382): numbers are kept as the strings the reference prints."""
        m = []
        for p in self.patterns:
            btype = {A: "A", B: "B", AB: "AB"}[p.sync_score.block_type]
            if p.type == TYPE_ALL:
                btype = "ALL"
            if p.type == TYPE_CLIP:
                btype = "CLIP-" + btype
            if p.speed != 1:
                btype += "-SPEED"
            sec = int(p.time)
            m.append({"key": p.key.name, "pos": "%d:%02d" % (sec // 60, sec % 60), "bits": bit_vec_to_str(p.bit_vec),
                      "quality": "%.5f" % p.sync_score.quality, "error": "%.6f" % p.decode_error, "rating": "%.5f" % p.rating,
                      "type": btype, "speed": "%.6f" % p.speed})
        return {"length": "%d:%02d" % (time_length // 60, time_length % 60), "matches": m}

    def match_count(self, orig_bits):
        return sum(1 for p in self.patterns if p.bit_vec == orig_bits)


@dataclass
class RawBits:
    index: int
    quality: float
    raw: np.ndarray
    block_type: int


def block_decoder_run(key: Key, samples, result_set: ResultSet, P: Params, rate=44100, trace: dict | None = None, speed=1.0):
    """BlockDecoder::run (wmget.cc:502-706) for one key."""
    sf = SyncFinder(P)
    stages = {} if trace is not None else None
    sync_scores = sf.search(key, samples, BLOCK, stages)
    if trace is not None:
        trace["sync_scores"] = sync_scores
        trace["stages"] = stages
    count = frames_per_block(P)
    prv = []
    for sc in sync_scores:
        raw = raw_bits_for_block(key, samples, sc.index, P)
        if raw is None:
            continue
        prv.append(RawBits(sc.index, sc.quality, raw, sc.block_type))
        bits, err = code_decode_soft(sc.block_type, normalize_soft_bits(raw, P), P)
        result_set.add_pattern(key, sc.index / rate, sc, bits, err, TYPE_BLOCK, speed)
    if trace is not None:
        trace["raw_bits"] = prv
    # AB (:554-604)
    for i in range(len(prv)):
        if prv[i].block_type == B:
            best_j, best_abs = -1, P.frame_size // 2
            for j in range(i):
                if prv[j].block_type == A:
                    ad = abs(int(prv[i].index - prv[j].index) - count * P.frame_size)
                    if ad < best_abs:
                        best_j, best_abs = j, ad
            if best_j >= 0:
                a, b = prv[best_j], prv[i]
                ab = np.empty(len(a.raw) * 2, dtype=np.float32)
                ab[0::2], ab[1::2] = a.raw, b.raw
                bits, err = code_decode_soft(AB, normalize_soft_bits(ab, P), P)
                result_set.add_pattern(key, b.index / rate, Score(b.index, (a.quality + b.quality) / 2, AB), bits, err, TYPE_BLOCK, speed)
    # all (:606-701)
    best_all = []

    def sync_sum(blocks):
        s = np.float32(0)
        for bi in blocks:
            s = np.float32(float(s) + prv[bi].quality)
        return s
    for i in range(len(prv)):
        max_block_idx = int(round_half_even(prv[-1].index / float(count * P.frame_size) + 0.5))
        all_blocks = [i]
        block_idx = 1
        while block_idx <= max_block_idx:
            expect_start = prv[all_blocks[-1]].index + block_idx * (count * P.frame_size)
            best_j, best_abs = -1, block_idx * P.frame_size // 2
            ebt = prv[all_blocks[-1]].block_type
            if block_idx & 1:
                ebt = B if ebt == A else A
            for j in range(all_blocks[-1], len(prv)):
                ad = abs(int(expect_start) - int(prv[j].index))
                if ad < best_abs and prv[j].block_type == ebt:
                    best_j, best_abs = j, ad
            if best_j >= 0:
                all_blocks.append(best_j)
                block_idx = 1
            else:
                block_idx += 1
        if sync_sum(all_blocks) > sync_sum(best_all):
            best_all = all_blocks
    if len(best_all) > 1:
        raw_all = np.zeros(code_size(AB, P), dtype=np.float32)
        norm = [0, 0]
        q = 0.0
        for bi in best_all:
            p = prv[bi]
            q += p.quality
            ab = 1 if p.block_type == B else 0
            raw_all[ab::2] = raw_all[ab::2] + p.raw
            norm[ab] += 1
        raw_all[0::2] = raw_all[0::2] / np.float32(max(norm[0], 1))
        raw_all[1::2] = raw_all[1::2] / np.float32(max(norm[1], 1))
        q /= norm[0] + norm[1]
        bits, err = code_decode_soft(AB, normalize_soft_bits(raw_all, P), P)
        result_set.add_pattern(key, 0.0, Score(0, q, A), bits, err, TYPE_ALL, speed)
    return sync_scores


def round_half_even(x):
    return np.rint(x)     # lrint with the default rounding mode


def clip_decoder_run(key: Key, samples, result_set: ResultSet, P: Params, rate=44100, speed=1.0):
    """ClipDecoder::run (wmget.cc:764-884) for one key."""
    fpb = frames_per_block(P)
    n, nch = samples.shape
    wav_frames = (n * nch) // (P.frame_size * nch)
    if not wav_frames < fpb * 3.1:
        return
    nvals = n * nch
    flat = samples.reshape(-1)
    npad = (fpb + 5) * P.frame_size * nch
    for pos in ("START", "END"):
        pad_start = pad_end = npad
        if pos == "START":
            first, last = 0, min(npad, nvals)
            if last < npad:
                pad_start += npad - last
        else:
            if nvals <= npad:
                continue
            first, last = nvals - npad, nvals
        time_offset = float(first) / rate / nch
        ext = np.concatenate([np.zeros(pad_start, np.float32), flat[first:last], np.zeros(pad_end, np.float32)]).reshape(-1, nch)
        sf = SyncFinder(P)
        for sc in sf.search(key, ext, CLIP):
            r1 = raw_bits_for_block(key, ext, sc.index, P)
            r2 = raw_bits_for_block(key, ext, sc.index + fpb * P.frame_size, P)
            if r1 is None or r2 is None:
                continue
            raw = np.empty(len(r1) * 2, dtype=np.float32)
            if sc.block_type == A:
                raw[0::2], raw[1::2] = r1, r2
            else:
                raw[0::2], raw[1::2] = r2, r1
            bits, err = code_decode_soft(AB, normalize_soft_bits(raw, P), P)
            result_set.add_pattern(key, time_offset, Score(int(time_offset * rate), sc.quality, sc.block_type), bits, err, TYPE_CLIP, speed)


def chunk_ranges(n_frames: int, P: Params, rate=44100):
    """WavChunkLoader (wavchunkloader.cc:54-163) for a file of known length at 44.1 kHz:
    yields (first_frame, n_frames_in_chunk, time_offset)."""
    max_frames = int(np.rint(P.get_chunk_size * 60 * rate))
    overlap = int(np.rint(2 * (frames_per_block(P) * P.frame_size / float(P.mark_sample_rate)) * 1.3 * rate))
    out, start, time_offset = [], 0, 0.0
    have = min(max_frames, n_frames)
    if have == 0:
        return out
    out.append((0, have, 0.0))
    end = have
    # the loader reaches EOF only when a refill returns nothing: a file that exactly fills the
    # chunk produces one more (overlap-only) chunk, like the reference.
    eof = have < max_frames
    while not eof:
        time_offset += (end - start - overlap) / float(rate)
        start = end - overlap
        new_end = min(start + max_frames, n_frames)
        eof = (new_end - start) < max_frames
        end = new_end
        out.append((start, end - start, time_offset))
    return out


# --------------------------------------------------------------------------- resampler

def resample_ratio(samples: np.ndarray, ratio: float, n_out: int | None = None, hlen: int = 16) -> np.ndarray:
    """resample_ratio / resample (resample.cc:52-131): out has lrint(n * ratio) frames (or n_out)."""
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    n, nch = samples.shape
    if n_out is None:
        n_out = int(np.rint(n * ratio))
    out = np.zeros((n_out, nch), np.float32)
    rc = lib().orc_resample(_p(samples), ctypes.c_int64(n), ctypes.c_int(nch), ctypes.c_double(ratio), ctypes.c_int(hlen),
                            _p(out), ctypes.c_int64(n_out))
    assert rc == 0, "resampler setup failed for ratio %r" % ratio
    return out


def resample(samples: np.ndarray, old_rate: int, new_rate: int) -> np.ndarray:      # resample.cc:52-95
    return resample_ratio(samples, float(new_rate) / old_rate)


def stream_avail(fed: int, ratio: float, hlen: int = 16) -> int:
    """outputs a streaming resampler (BufferedResamplerImpl::write_frames, resample.cc:168-196) has delivered once `fed`
    frames (after the k/2 - 1 frames of pre-roll) have been written: every output whose 2h taps are buffered."""
    fc = min(1.0, ratio)
    h = int(math.ceil(hlen / fc))
    step = 1.0 / ratio
    if fed - 2 < h - 1:
        return 0
    n = max(int((fed - 1 - h) * ratio) - 2, 0)
    while n > 0 and math.floor((h - 1) + float(n - 1) * step) > fed - 2:
        n -= 1
    while math.floor((h - 1) + float(n) * step) <= fed - 2:
        n += 1
    return n


def stream_out_count(n_in: int, ratio: float, hlen: int = 16) -> int:
    """... plus write_trailing_frames (k/2 zero frames, resample.cc:198-204): what WavChunkLoader gets for n_in input frames"""
    h = int(math.ceil(hlen / min(1.0, ratio)))
    return stream_avail(n_in + h, ratio, hlen)


def resampled_add_plan(n: int, rate: int, P: Params):
    """Frame counts of the add loop (wmadd.cc:520-589) when a WatermarkResampler is active: returns
    (frames pushed through mixer / --snr sums / limiter, number of WatermarkGen::run calls)."""
    N = P.frame_size
    r_in, r_out = float(P.mark_sample_rate) / rate, float(rate) / P.mark_sample_rate
    bs = rate * P.limiter_block_size_ms // 1000
    total_in = total_out = 0
    emitted = runs = 0
    j = 0
    while True:
        real = min(N, n - total_in)
        total_in += real
        if real < N and total_in == total_out:
            break
        x44 = stream_avail(N * (j + 1), r_in)
        runs = x44 // N
        emitted = stream_avail(runs * N, r_out) if runs else 0
        lim = emitted if P.test_no_limiter else max(emitted // bs - 1, 0) * bs
        total_out = min(lim, total_in)
        j += 1
    return emitted, runs


def resample_stream(samples: np.ndarray, old_rate: int, new_rate: int) -> np.ndarray:
    """what WavChunkLoader (wavchunkloader.cc:66-73,196-221) hands on for an input that is not at the watermark rate"""
    ratio = float(new_rate) / old_rate
    return resample_ratio(samples, ratio, stream_out_count(samples.shape[0], ratio))


def resample_ratio_truncate(samples, rate, ratio, max_in_seconds):                   # resample.cc:97-125
    n = samples.shape[0]
    if max_in_seconds > 0:
        n = min(n, int(np.rint(rate * max_in_seconds)))
    return resample_ratio(samples[:n], ratio)


# --------------------------------------------------------------------------- speed detection (wmspeed.cc)

@dataclass
class SpeedScanParams:                               # wmspeed.cc:54-60
    seconds: float
    step: float
    n_steps: int
    n_center_steps: int = 0


def get_speed_clip(location, samples, rate, clip_seconds):          # wmspeed.cc:33-52
    n = samples.shape[0]
    end_sec = float(n) / rate
    start_sec = location * (end_sec - clip_seconds)
    if start_sec < 0:
        start_sec = 0
    start_point = int(start_sec * rate)
    end_point = min(int(start_point + clip_seconds * rate), n)
    return samples[start_point:end_point]


def get_clip_locations(key: Key, samples, n):                        # wmspeed.cc:533-552
    rng = Random(key, 0, STREAM_SPEED_CLIP)
    flat = samples.reshape(-1)
    idx, pos, size = [], 0, flat.shape[0]
    while pos < size:
        idx.append(pos)
        pos += rng() % 1000
    xs = np.ascontiguousarray(flat[np.array(idx, np.int64)], dtype=np.float32)
    import hashlib
    seed = struct.unpack(">Q", hashlib.sha1(xs.tobytes()).digest()[:8])[0]     # Random::seed_from_hash, random.cc:184-190
    rng.seed(seed, STREAM_SPEED_CLIP)
    return [rng.random_double() for _ in range(n)]


def get_best_clip_location(key: Key, samples, rate, seconds, candidates):       # wmspeed.cc:554-575
    clip_location, best_energy = 0.0, 0.0
    for location in get_clip_locations(key, samples, candidates):
        wd = get_speed_clip(location, samples, rate, seconds).reshape(-1)
        sq = (wd * wd).astype(np.float64)            # float product, double running sum
        energy = float(np.cumsum(sq)[-1]) if sq.size else 0.0
        if energy > best_energy:
            best_energy, clip_location = energy, location
    return clip_location


def speed_sync_entries(key: Key, P: Params):
    """SpeedSync constructor (wmspeed.cc:144-161): BLOCK sync entries of all bits, sorted by frame."""
    sb = get_sync_bits(key, BLOCK, P)
    n = len(sb.frame)
    bit = np.zeros(n, np.int32)
    for b in range(P.sync_bits):
        bit[sb.off[b]:sb.off[b + 1]] = b
    order = np.argsort(sb.frame, kind="stable")
    up = sb.up.reshape(n, -1)[order]
    down = sb.down.reshape(n, -1)[order]
    return (np.ascontiguousarray(sb.frame[order], np.int32), np.ascontiguousarray(bit[order], np.int32),
            np.ascontiguousarray(up, np.int32), np.ascontiguousarray(down, np.int32))


def speed_prepare_mags(clip, rate, center, seconds, entries):                   # SpeedSync::prepare_mags, wmspeed.cc:203-268
    frame, bit, up, down = entries
    sub = resample_ratio_truncate(clip, rate, center / 2, seconds / center)
    L = lib()
    L.orc_speed_rows.restype = ctypes.c_int64
    rows = int(L.orc_speed_rows(ctypes.c_int64(sub.shape[0])))
    mags = np.zeros((len(frame), rows, 2), np.float32)
    window = gen_normalized_window(512)
    L.orc_speed_mags(_p(sub), ctypes.c_int64(sub.shape[0]), ctypes.c_int(sub.shape[1]), _p(window), ctypes.c_int(len(frame)),
                     ctypes.c_int(up.shape[1]), _p(up), _p(down), _p(mags))
    return mags


def speed_compare(mags, entries, relative_speeds, P: Params):                   # SpeedSync::compare, wmspeed.cc:328-375
    frame, bit, up, down = entries
    rel = np.ascontiguousarray(relative_speeds, np.float64)
    out = np.zeros(len(rel), np.float64)
    lib().orc_speed_compare(_p(mags), ctypes.c_int64(mags.shape[1]), ctypes.c_int(len(frame)), _p(frame), _p(bit), ctypes.c_int(P.sync_bits),
                            ctypes.c_int(frames_per_block(P)), _p(rel), ctypes.c_int(len(rel)), ctypes.c_double(P.water_delta), _p(out))
    return out


def speed_search(key: Key, samples, rate, clip_location, scan: SpeedScanParams, speeds, P: Params, trace=None):
    """SpeedSearch::get_jobs + the job execution of run_search (wmspeed.cc:459-484, 688-722): list of (speed, quality)."""
    clip = get_speed_clip(clip_location, samples, rate, scan.seconds * 1.3)
    entries = speed_sync_entries(key, P)
    scores = []
    for speed in speeds:
        for c in range(-scan.n_center_steps, scan.n_center_steps + 1):
            center = speed * math.pow(scan.step, c * (scan.n_steps * 2 + 1))
            mags = speed_prepare_mags(clip, rate, center, scan.seconds, entries)
            rel = [math.pow(scan.step, p) * center / center for p in range(-scan.n_steps, scan.n_steps + 1)]
            q = speed_compare(mags, entries, rel, P)
            scores += [(r * center, float(qq)) for r, qq in zip(rel, q)]
            if trace is not None:
                trace.append((center, rel, [float(x) for x in q]))
    return scores


def select_n_best_scores(scores, n):                                            # wmspeed.cc:487-530
    scores = sorted(scores, key=lambda s: s[0])

    def get_quality(pos):
        return scores[pos][1] if 0 <= pos < len(scores) else 0.0
    lmax, x = [], 0
    while x < len(scores):
        q1, q2, q3 = get_quality(x - 1), get_quality(x), get_quality(x + 1)
        if q1 <= q2 and q2 >= q3:
            lmax.append(scores[x])
            x += 1
        x += 1
    lmax.sort(key=lambda s: -s[1])
    return lmax[:n]


def score_smooth_find_best(scores, step, distance):                             # wmspeed.cc:385-419
    scores = sorted(scores, key=lambda s: s[0])
    sp = np.array([s[0] for s in scores], np.float64)
    qu = np.array([s[1] for s in scores], np.float64)
    L = lib()
    L.orc_score_smooth_find_best.restype = ctypes.c_double
    return float(L.orc_score_smooth_find_best(_p(sp), _p(qu), ctypes.c_int(len(sp)), ctypes.c_double(step), ctypes.c_double(distance)))


@dataclass
class DetectSpeedInfo:
    speed: float = 0.0
    quality: float = 0.0
    accepted: bool = False
    line: str = ""
    clip_location: float = 0.0
    stages: dict = field(default_factory=dict)


def detect_speed(key: Key, samples, P: Params, rate=44100, patient=False, test_speed=-1.0) -> DetectSpeedInfo | None:
    """detect_speed (wmspeed.cc:622-781) for one key; None for inputs shorter than 0.25 s."""
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    if float(samples.shape[0]) / rate < 0.25:
        return None
    scan1 = SpeedScanParams(50, 1.00035, 11, 28) if patient else SpeedScanParams(25, 1.0007, 5, 28)
    scan2 = SpeedScanParams(50, 1.000175, 1) if patient else SpeedScanParams(50, 1.00035, 1)
    scan3 = SpeedScanParams(50, 1.00005, 40)
    n_best = 15 if patient else 5
    info = DetectSpeedInfo()
    info.clip_location = get_best_clip_location(key, samples, rate, scan1.seconds, 5)
    s1 = speed_search(key, samples, rate, info.clip_location, scan1, [1.0], P)
    best = select_n_best_scores(s1, n_best)
    s2 = speed_search(key, samples, rate, info.clip_location, scan2, [b[0] for b in best], P)
    best1 = select_n_best_scores(s2, 1)
    s3 = speed_search(key, samples, rate, info.clip_location, scan3, [best1[0][0]], P)
    info.stages = {"scan1": s1, "scan2": s2, "scan3": s3}
    info.speed = score_smooth_find_best(s3, 1 - scan3.step, 20)
    info.quality = max([0.0] + [q for _, q in s3])
    delta = -1.0
    if test_speed > 0:
        delta = 100 * abs(info.speed - test_speed) / test_speed
    info.line = "detect_speed %f %f %.4f" % (info.speed, info.quality, delta)
    info.accepted = info.quality > 0.4 and (info.speed < 0.9999 or info.speed > 1.0001)
    return info


def get_watermark(samples, key_list, P: Params | None = None, rate=44100, detect=False, patient=False, try_speed=-1.0,
                  test_speed=-1.0, speed_lines: list | None = None) -> ResultSet:
    """get_watermark / decode (wmget.cc:886-939,971-1013); detect / patient / try_speed = --detect-speed,
    --detect-speed-patient, --try-speed."""
    P = P or Params()
    samples = np.ascontiguousarray(samples, dtype=np.float32)
    if rate != P.mark_sample_rate:
        samples = resample_stream(samples, rate, P.mark_sample_rate)
        rate = P.mark_sample_rate
    rs = ResultSet()
    first = True
    for start, cnt, toff in chunk_ranges(samples.shape[0], P, rate):
        chunk = samples[start:start + cnt]
        crs = ResultSet()
        if detect or patient or try_speed > 0:
            speed_results = []
            if detect or patient:
                for key in key_list:
                    info = detect_speed(key, chunk, P, rate, patient, test_speed)
                    if info is not None:
                        if speed_lines is not None:
                            speed_lines.append(info.line)
                        if info.accepted:
                            speed_results.append((key, info.speed))
            else:
                speed_results = [(key, try_speed) for key in key_list]
            for key, speed in speed_results:
                stretched = resample_ratio(chunk, speed)
                srate = int(P.mark_sample_rate * speed)
                block_decoder_run(key, stretched, crs, P, srate, speed=speed)
                if first:
                    clip_decoder_run(key, stretched, crs, P, srate, speed=speed)
        for key in key_list:
            block_decoder_run(key, chunk, crs, P, rate)
        if first:
            for key in key_list:
                clip_decoder_run(key, chunk, crs, P, rate)
        crs.apply_time_offset(toff)
        rs.merge(crs)
        first = False
    rs.sort(key_list)
    return rs
