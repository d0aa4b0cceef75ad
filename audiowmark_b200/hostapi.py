"""ctypes binding of lib/libawm_host.so: the host-side C++ (key tables, `add`, `get`) behind plain C
entry points (audiowmark_b200/host/awm_hostapi.cc).  This is the reference-facing call path the CLI
uses; bench.py's e2e number and the end-to-end parity tests go through it."""
from __future__ import annotations

import ctypes
import json
import os

import numpy as np

from . import capi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libawm_host.so")
CLI_PATH = os.path.join(_HERE, "bin", "audiowmark")

EXPORTS = ["awmh_set_params", "awmh_frames_per_block", "awmh_n_coded_bits", "awmh_random_u64", "awmh_gen_noise", "awmh_sync_table",
           "awmh_mix_table", "awmh_frame_mod", "awmh_conv_encode", "awmh_add", "awmh_get", "awmh_merge_chunks", "awmh_chunk_geometry", "awmh_ctx", "awmh_key_slot", "awmh_stage_select", "awmh_gpu_launches", "awmh_gpu_stream", "awmh_synchronize", "awmh_profile_enable", "awmh_profile_report", "awmh_shutdown", "awmh_set_speed_params", "awmh_detect_speed", "awmh_resample", "awmh_resample_stream_frames", "awmh_resample_stream_available", "awmh_resampled_add_plan", "awmh_set_short_payload", "awmh_add_s16", "awmh_get_s16", "awmh_short_encode", "awmh_short_decode", "awmh_sync_trace", "awmh_sync_trace_fetch", "awmh_dist_unique_id", "awmh_dist_init", "awmh_balanced_get", "awmh_bg_create", "awmh_bg_destroy", "awmh_bg_stage", "awmh_bg_plan", "awmh_bg_owner", "awmh_bg_input_range", "awmh_add_windowed",
           "awmh_embed_roles", "awmh_coded_bits", "awmh_add_batch", "awmh_role_layout", "awmh_embed_roles_device",
           "awmh_window_range", "awmh_add_window", "awmh_gs_create", "awmh_gs_feed", "awmh_gs_finish", "awmh_gs_destroy", "awmh_gs_peak_bytes",
           "awmh_gs_plan"]

_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("%s is missing: run __graft_entry__.build()" % LIB_PATH)
        capi.load()        # libawm_b200.so first (rpath $ORIGIN also finds it)
        lib = ctypes.CDLL(LIB_PATH)
        lib.awmh_gpu_launches.restype = ctypes.c_uint64
        lib.awmh_gpu_stream.restype = ctypes.c_void_p
        lib.awmh_ctx.restype = ctypes.c_void_p
        lib.awmh_gs_create.restype = ctypes.c_void_p
        lib.awmh_gs_peak_bytes.restype = ctypes.c_uint64
        _lib = lib
    return _lib


_BUFS = {}


def _outbuf(tag: str, cap: int):
    """persistent ctypes output buffer (create_string_buffer zero-fills: megabytes per call add up in the per-step path)"""
    b = _BUFS.get(tag)
    if b is None or len(b) < cap:
        b = ctypes.create_string_buffer(cap)
        _BUFS[tag] = b
    return b


def _ptr(x):
    if x is None:
        return ctypes.c_void_p(0)
    if isinstance(x, (int, np.integer)):
        return ctypes.c_void_p(int(x))
    assert x.flags["C_CONTIGUOUS"]
    return x.ctypes.data_as(ctypes.c_void_p)


def _key(key) -> bytes:
    k = bytes(key) if key is not None else bytes(16)
    assert len(k) == 16
    return k


_PARAMS = {"sync_threshold2": 0.35, "n_best": 8, "water_delta": 0.01}


def get_param(name):
    return _PARAMS[name]


def set_params(water_delta=0.01, frames_per_bit=2, mix=True, hard=False, sync_threshold2=0.35, n_best=8, chunk_size_min=30.0,
               test_no_limiter=False, test_no_sync=False, gpu_device=0, quiet=True):
    _PARAMS.update(sync_threshold2=sync_threshold2, n_best=n_best, water_delta=water_delta)
    load().awmh_set_params(ctypes.c_double(water_delta), ctypes.c_int(frames_per_bit), ctypes.c_int(mix), ctypes.c_int(hard),
                           ctypes.c_double(sync_threshold2), ctypes.c_int(n_best), ctypes.c_double(chunk_size_min),
                           ctypes.c_int(test_no_limiter), ctypes.c_int(test_no_sync), ctypes.c_int(gpu_device), ctypes.c_int(quiet))


def frames_per_block() -> int:
    return load().awmh_frames_per_block()


def n_coded_bits() -> int:
    return load().awmh_n_coded_bits()


def random_u64(key, seed: int, stream: int, n: int) -> np.ndarray:
    out = np.zeros(n, np.uint64)
    load().awmh_random_u64(_key(key), ctypes.c_uint64(seed), ctypes.c_int(stream), _ptr(out), ctypes.c_int(n))
    return out


def gen_noise(key, n_values: int) -> np.ndarray:
    out = np.zeros(n_values, np.float32)
    load().awmh_gen_noise(_key(key), _ptr(out), ctypes.c_size_t(n_values))
    return out


def sync_table(key, mode: int):
    ent = np.zeros(4096, capi.SYNC_ENTRY)
    off = np.zeros(7, np.int32)
    n = load().awmh_sync_table(_key(key), ctypes.c_int(mode), _ptr(ent), ctypes.c_int(len(ent)), _ptr(off))
    assert n > 0
    return ent[:n].copy(), off


def mix_table(key):
    ent = np.zeros(200000, capi.MIX_ENTRY)
    order = np.zeros(8192, np.uint16)
    n = load().awmh_mix_table(_key(key), _ptr(ent), ctypes.c_int(len(ent)), _ptr(order), ctypes.c_int(len(order)))
    assert n > 0
    return ent[:n].copy(), order[:n_coded_bits()].copy()


def frame_mod(key, payload_hex: str) -> np.ndarray:
    fpb = frames_per_block()
    out = np.zeros((2, fpb, 101), np.uint8)
    n = load().awmh_frame_mod(_key(key), payload_hex.encode(), _ptr(out), ctypes.c_size_t(out.size))
    assert n == out.size
    return out


def embed_roles(key) -> np.ndarray:
    """key-only role codes uint16 [frames_per_block, 101] of the FrameMod table (codes: include/awm_b200.h)"""
    out = np.zeros((frames_per_block(), 101), np.uint16)
    n = load().awmh_embed_roles(_key(key), _ptr(out), ctypes.c_size_t(out.size))
    assert n == out.size
    return out


def role_layout() -> np.ndarray:
    """awm_role_layout of the current parameters as int32 [6]: sync frames, sync frames per bit, data frames, frames per bit, mix,
    coded bits"""
    out = np.zeros(6, np.int32)
    load().awmh_role_layout(_ptr(out))
    return out


def embed_roles_device(keys) -> np.ndarray:
    """the role tables of many keys, built on the device in one launch: uint16 [len(keys), frames_per_block, 101], each equal to
    embed_roles(key)"""
    kb = _keys(keys, "embed_roles_device")
    out = np.zeros((len(kb) // 16, frames_per_block(), 101), np.uint16)
    if not out.size:
        return out
    rc = load().awmh_embed_roles_device(kb, ctypes.c_size_t(len(kb) // 16), _ptr(out), ctypes.c_size_t(out.size))
    if rc:
        raise RuntimeError("awmh_embed_roles_device failed (rc=%d); see stderr" % rc)
    return out


def _keys(keys, name, n=None) -> bytes:
    """a list of 16-byte keys -> their concatenation (ValueError for a wrong key length or, with n, a wrong count)"""
    keys = list(keys)
    if n is not None and len(keys) != n:
        raise ValueError("%s: %d items but %d keys" % (name, n, len(keys)))
    kb = [bytes(k) for k in keys]
    if any(len(k) != 16 for k in kb):
        raise ValueError("%s: every key must be 16 bytes" % name)
    return b"".join(kb)


def coded_bits(key, payload_hex: str) -> np.ndarray:
    """one payload's coded data bits uint8 [2 (A, B), n_coded]: randomize_bit_order (code_encode (A | B, payload))"""
    out = np.zeros((2, n_coded_bits()), np.uint8)
    n = load().awmh_coded_bits(_key(key), payload_hex.encode(), _ptr(out), ctypes.c_size_t(out.size))
    if n != out.size:
        raise ValueError("cannot encode payload %r" % payload_hex)
    return out


def conv_encode(block_type: int, bits) -> np.ndarray:
    b = np.ascontiguousarray(bits, np.uint8)
    out = np.zeros((len(b) + 15) * 12, np.uint8)
    n = load().awmh_conv_encode(ctypes.c_int(block_type), _ptr(b), ctypes.c_int(len(b)), _ptr(out), ctypes.c_int(len(out)))
    return out[:n].copy()


def short_encode(bits) -> np.ndarray:
    """block code of the current --short mode: k message bits -> n code bits"""
    b = np.ascontiguousarray(bits, np.uint8)
    out = np.zeros(128, np.uint8)
    n = load().awmh_short_encode(_ptr(b), ctypes.c_int(len(b)), _ptr(out), ctypes.c_int(len(out)))
    if n < 0:
        raise ValueError("short payload mode is off or the message length does not match")
    return out[:n].copy()


def short_decode(coded) -> np.ndarray:
    """n code bits -> k message bits; empty if no code word matches"""
    c = np.ascontiguousarray(coded, np.uint8)
    out = np.zeros(32, np.uint8)
    n = load().awmh_short_decode(_ptr(c), ctypes.c_int(len(c)), _ptr(out), ctypes.c_int(len(out)))
    if n < 0:
        raise ValueError("short payload mode is off or the code length does not match")
    return out[:n].copy()


def add(pcm_in, payload_hex: str, key=None, pcm_out=None, n_frames=None, channels=None, sample_rate=44100, want_stats=False, first_frame_number=0):
    """add_stream_watermark on a buffer: numpy arrays (host) or device pointers (ints)."""
    if isinstance(pcm_in, np.ndarray):
        pcm_in = np.ascontiguousarray(pcm_in, np.float32)
        n_frames, channels = pcm_in.shape
        if pcm_out is None:
            pcm_out = np.empty_like(pcm_in)
    blocks, snr = ctypes.c_int(), ctypes.c_double()
    rc = load().awmh_add(_key(key), _ptr(pcm_in), _ptr(pcm_out), ctypes.c_size_t(n_frames), ctypes.c_int(channels), ctypes.c_int(sample_rate),
                         payload_hex.encode(), ctypes.byref(blocks) if want_stats else None, ctypes.byref(snr) if want_stats else None,
                         ctypes.c_uint64(first_frame_number))
    if rc:
        raise RuntimeError("awmh_add failed (rc=%d); see stderr" % rc)
    return (pcm_out, blocks.value, snr.value) if want_stats else pcm_out


def _pack_batch(name, pcms, payloads, items, out):
    """the packed buffers of a batch call -> (s16, item array, n_values, in pointer, out pointer, split (offset, frames, channels) ->
    output view, buffers to keep alive); see add_batch for the two input forms"""
    if items is None:
        arrays = [np.asarray(p) for p in pcms]
        s16 = bool(arrays) and all(a.dtype == np.int16 for a in arrays)
        dt = np.int16 if s16 else np.float32
        arrays = [a.reshape(-1, 1) if a.ndim == 1 else a for a in arrays]
        items = []
        off = 0
        for a in arrays:
            items.append((off, a.shape[0], a.shape[1]))
            off += a.size
        packed = np.concatenate([np.ascontiguousarray(a, dt).reshape(-1) for a in arrays]) if arrays else np.zeros(0, dt)
        res = np.empty_like(packed)
        n_values, p_in, p_out = packed.size, _ptr(packed), _ptr(res)
        split = lambda o, n, c: res[o:o + n * c].reshape(n, c)
    else:
        import torch
        if not (pcms.is_cuda and pcms.is_contiguous() and pcms.dtype in (torch.float32, torch.int16)):
            raise ValueError("%s: pcms must be a contiguous float32 or int16 CUDA tensor" % name)
        s16 = pcms.dtype == torch.int16
        res = torch.empty_like(pcms) if out is None else out
        if res.dtype != pcms.dtype or res.numel() != pcms.numel() or not res.is_contiguous():
            raise ValueError("%s: out must be a contiguous tensor like pcms" % name)
        flat = res.view(-1)
        torch.cuda.current_stream(pcms.device).synchronize()      # the context works on its own stream
        n_values, p_in, p_out = pcms.numel(), ctypes.c_void_p(pcms.data_ptr()), ctypes.c_void_p(res.data_ptr())
        split = lambda o, n, c: flat[o:o + n * c].view(n, c)
        packed = pcms
    if len(payloads) != len(items):
        raise ValueError("%s: %d items but %d payloads" % (name, len(items), len(payloads)))
    it = np.array([tuple(int(v) for v in t) for t in items], capi.BATCH_ITEM)
    return s16, it, n_values, p_in, p_out, split, (packed, res)


def _zero_frames(name, zero_frames, n_items):
    """a stream offset list -> uint64 array of n_items (ValueError for a wrong length or a value outside 0 .. 2^64-1)"""
    z = list(zero_frames)
    if len(z) != n_items:
        raise ValueError("%s: %d items but %d zero_frames" % (name, n_items, len(z)))
    if any(int(v) < 0 or int(v) >= 1 << 64 for v in z):
        raise ValueError("%s: zero_frames must be in 0 .. 2^64-1" % name)
    return np.array([int(v) for v in z], np.uint64)


def _add_batch(name, pcms, payloads, key, keys, items, out, want_stats, zero_frames, sample_rate=44100, sample_rates=None, scratch_bytes=0):
    """add_batch, or add_batch_rates when sample_rates is given, through awmh_add_batch"""
    payloads = list(payloads)
    rates = None if sample_rates is None else np.array([int(r) for r in sample_rates], np.int64)
    s16, it, n_values, p_in, p_out, split, _keep = _pack_batch(name, pcms, payloads, items, out)
    if rates is not None:
        if len(rates) != len(it):
            raise ValueError("%s: %d items but %d sample rates" % (name, len(it), len(rates)))
        if np.any(rates <= 0) or np.any(rates > np.iinfo(np.int32).max):
            raise ValueError("%s: sample rates must be positive 32 bit integers" % name)
        rates = np.ascontiguousarray(rates, np.int32)
    z = None if zero_frames is None else _zero_frames(name, zero_frames, len(it))
    if keys is None:
        kb = _key(key)
    else:
        if rates is None and sample_rate != 44100:
            raise ValueError("%s: only 44.1 kHz input is accepted (use add_batch_rates)" % name)
        if key is not None:
            raise ValueError("%s: pass either key= or keys=, not both" % name)
        kb = _keys(keys, name, len(it))
    pay = (ctypes.c_char_p * max(len(payloads), 1))(*[p.encode() for p in payloads])
    blocks = np.zeros(max(len(it), 1), np.int32)
    snr = np.zeros(max(len(it), 1), np.float64)
    rc = load().awmh_add_batch(kb or None, ctypes.c_int(keys is not None), p_in, p_out, ctypes.c_int(s16), ctypes.c_size_t(n_values), _ptr(it),
                               ctypes.c_size_t(len(it)), pay, ctypes.c_int(sample_rate), _ptr(rates), _ptr(z), ctypes.c_size_t(scratch_bytes),
                               _ptr(blocks) if want_stats else None, _ptr(snr) if want_stats else None)
    if rc == 2:
        raise ValueError("%s: malformed item list, %soffset list or payload; see stderr" % (name, "" if rates is None else "sample rate, "))
    if rc:
        raise RuntimeError("awmh_add_batch failed (rc=%d); see stderr" % rc)
    synchronize()
    outs = [split(int(t["value_offset"]), int(t["n_frames"]), int(t["channels"])) for t in it]
    return (outs, blocks[:len(it)].tolist(), snr[:len(it)].tolist()) if want_stats else outs


def add_batch(pcms, payloads, key=None, sample_rate=44100, items=None, out=None, want_stats=False, zero_frames=None, keys=None):
    """`add` for many items with one key and one payload each, in one pass over the GPU; item i comes out bit identical to
    add / add_s16 of that item alone with payloads[i].
      pcms: a list of numpy arrays [n, channels] (all float32 or all int16; channels may differ), or one packed device tensor
            (float32 or int16, contiguous) with items = [(value_offset, n_frames, channels), ...] in values of that tensor;
            out: a device tensor like pcms for the result (default: a new one).
      zero_frames: None, or one stream offset per item (sample-frames): item i continues a stream that began zero_frames[i]
            frames earlier with silence, as an HLS segment does (`audiowmark hls-add`).  It comes out bit identical to
            add_windowed(item, payloads[i], zero_frames=zero_frames[i]) = add(zeros(z) ++ item)[z:] (16 bit: add_s16 of the same),
            with that call's data blocks and SNR.  zero_frames + n_frames is limited to 2^48 per item.
      keys: None, or one 16-byte key per item (instead of key=): item i comes out bit identical to this call with key=keys[i].  The
            role tables of the distinct keys are built on the device in one launch.
    Returns the list of outputs (numpy arrays, or views of the output tensor), with want_stats also the lists of data blocks
    and SNR dB per item.  Only 44.1 kHz input is accepted.  Raises ValueError for a malformed item list, offset list or payload."""
    return _add_batch("add_batch", pcms, payloads, key, keys, items, out, want_stats, zero_frames, sample_rate=sample_rate)


def add_batch_rates(pcms, payloads, sample_rates, key=None, items=None, out=None, want_stats=False, scratch_bytes=0, zero_frames=None, keys=None):
    """add_batch for items that each have their own sample rate: item i comes out bit identical to add(item, payloads[i],
    sample_rate=sample_rates[i]) of that item alone (16 bit items: to that `add` between int16_to_float and 16 bit quantisation, what
    `audiowmark add` computes on a 16 bit file).  pcms / items / out / want_stats as in add_batch.  scratch_bytes: device scratch
    per wave of resampled items (0: the library's default of 4 GiB; a smaller value runs more, smaller waves with the same result).
    zero_frames: None, or one stream offset per item in frames at that item's rate: item i continues a stream that began
    zero_frames[i] frames earlier with silence (an HLS segment of a 48 kHz master).  It comes out bit identical to
    add_batch_rates([zeros(z) ++ item], ...)[z:], with the data blocks of that whole stream and the SNR of the item's own positions;
    the silent prefix is never allocated.  zero_frames + n_frames is limited to 2^48 per item, at the item's rate and at 44.1 kHz.
    keys: None, or one 16-byte key per item (instead of key=), as in add_batch.
    Raises ValueError for a malformed item list, rate list, offset list or payload."""
    return _add_batch("add_batch_rates", pcms, payloads, key, keys, items, out, want_stats, zero_frames, sample_rates=sample_rates,
                      scratch_bytes=scratch_bytes)


def add_windowed(pcm_in: np.ndarray, payload_hex: str, key=None, zero_frames=0, window_frames=0, sample_rate=44100):
    """the bounded-memory loop of `audiowmark add` (add_watermark_windowed) on a host buffer -> (output, data blocks, snr dB), at any
    sample rate: the output equals add(zeros(zero_frames) ++ pcm_in, sample_rate=sample_rate)[zero_frames:] bit for bit.  window_frames
    (in 1024-frames; 0: the default of 4096) sets how much is marked per window."""
    pcm_in = np.ascontiguousarray(pcm_in, np.float32)
    out = np.empty_like(pcm_in)
    blocks, snr = ctypes.c_int(), ctypes.c_double()
    rc = load().awmh_add_windowed(_key(key), _ptr(pcm_in), _ptr(out), ctypes.c_size_t(pcm_in.shape[0]), ctypes.c_int(pcm_in.shape[1]), ctypes.c_int(sample_rate),
                                  payload_hex.encode(), ctypes.c_size_t(zero_frames), ctypes.c_size_t(window_frames), ctypes.byref(blocks), ctypes.byref(snr))
    if rc:
        raise RuntimeError("awmh_add_windowed failed (rc=%d); see stderr" % rc)
    return out, blocks.value, snr.value


UNKNOWN = (1 << 64) - 1        # n_total of a stream whose end is not known yet


def window_range(own_first: int, own_end: int, n_total: int, sample_rate=44100) -> tuple[int, int]:
    """the input frames [ext_first, ext_end) that add_window needs so that its owned frames [own_first, own_end) come out as in add()
    of the whole stream of n_total frames (UNKNOWN: the end is not known yet).  At 44.1 kHz ext_first is a multiple of 1024; at other
    rates it is the smallest such range (awm_window_range_rates).  ValueError for an empty range, one past n_total or a bad rate."""
    first, end = ctypes.c_uint64(), ctypes.c_uint64()
    rc = load().awmh_window_range(ctypes.c_uint64(own_first), ctypes.c_uint64(own_end), ctypes.c_uint64(n_total), ctypes.c_int(sample_rate),
                                  ctypes.byref(first), ctypes.byref(end))
    if rc:
        raise ValueError("window_range: owned range [%d, %d) of %d frames at %d Hz is refused; see stderr" % (own_first, own_end, n_total, sample_rate))
    return first.value, end.value


def add_window(pcm, payload_hex: str, stream_first: int, n_total: int, own_first: int, own_end: int, key=None, pcm_out=None, n_frames=None,
               channels=None, sample_rate=44100, want_stats=False):
    """`add` of one window of a stream at any rate: how a rank marks its own span of a master.  pcm holds stream frames
    [stream_first, stream_first + n_frames) (a numpy array [n, channels], or a device pointer with n_frames / channels and pcm_out)
    and must cover window_range(own_first, own_end, n_total, sample_rate); n_total may be UNKNOWN for a window that does not end the
    stream.  The window's frames of pcm_out are written (a numpy result starts as a copy of pcm), and its owned frames [own_first,
    own_end) equal those of add() of the whole stream bit for bit.  want_stats: also the --snr sums (watermark power, signal power) of
    the owned frames (the window that ends the stream includes the frames emitted after it); summed over all windows,
    10 log10 (signal / watermark) is the stream's SNR.  ValueError when the buffer misses part of the window or the range is bad."""
    if isinstance(pcm, np.ndarray):
        pcm = np.ascontiguousarray(pcm, np.float32)
        n_frames, channels = pcm.shape
        if pcm_out is None:
            pcm_out = pcm.copy()
    snr = np.zeros(2, np.float64)
    rc = load().awmh_add_window(_key(key), _ptr(pcm), _ptr(pcm_out), ctypes.c_uint64(stream_first), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                                ctypes.c_int(sample_rate), payload_hex.encode(), ctypes.c_uint64(n_total), ctypes.c_uint64(own_first),
                                ctypes.c_uint64(own_end), _ptr(snr) if want_stats else None)
    if rc == 2:
        raise ValueError("add_window: buffer [%d, +%d) at %d Hz does not cover the window of [%d, %d), or the range is bad; see stderr"
                         % (stream_first, n_frames, sample_rate, own_first, own_end))
    if rc:
        raise RuntimeError("awmh_add_window failed (rc=%d); see stderr" % rc)
    return (pcm_out, float(snr[0]), float(snr[1])) if want_stats else pcm_out


def get(pcm, keys=None, names=None, n_frames=None, channels=None, sample_rate=44100, parse=True):
    """get_watermark on a buffer -> the --json document (dict) of the run."""
    keys = keys or [bytes(16)]
    names = names or [""] * len(keys)
    if isinstance(pcm, np.ndarray):
        pcm = np.ascontiguousarray(pcm, np.float32)
        n_frames, channels = pcm.shape
    kb = b"".join(_key(k) for k in keys)
    name_arr = (ctypes.c_char_p * len(keys))(*[n.encode() for n in names])
    cap = 1 << 22
    buf = _outbuf("get", cap)
    n_pat = ctypes.c_int()
    rc = load().awmh_get(kb, name_arr, ctypes.c_int(len(keys)), _ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                         ctypes.c_int(sample_rate), buf, ctypes.c_size_t(cap), ctypes.byref(n_pat))
    if rc:
        raise RuntimeError("awmh_get failed (rc=%d); see stderr" % rc)
    text = buf.value.decode()
    return json.loads(text) if parse else text


class GetStream:
    """`get` over a stream that arrives piece by piece (a pipe, a long recording), in bounded memory: the pieces go into one device
    chunk buffer (at other rates through a small device input window and the resampler), each chunk is decoded once it is full, and
    finish() returns the --json document (parse=False: its text) of get() on the whole stream, byte for byte.  feed(pcm) takes a
    numpy array [n, channels] (float32) or a float32 device pointer with n_frames.  ValueError for a sample rate outside the resampler's
    range, a channel count that does not match and a feed or finish after finish."""

    def __init__(self, keys=None, names=None, channels=2, sample_rate=44100):
        keys = keys or [bytes(16)]
        names = names or [""] * len(keys)
        self.channels, self.sample_rate, self._finished = int(channels), int(sample_rate), False
        kb = b"".join(_key(k) for k in keys)
        name_arr = (ctypes.c_char_p * len(keys))(*[n.encode() for n in names])
        self.h = load().awmh_gs_create(kb, name_arr, ctypes.c_int(len(keys)), ctypes.c_int(self.channels), ctypes.c_int(self.sample_rate), ctypes.c_int(0))
        if not self.h:
            raise ValueError("GetStream: %d channels at %d Hz are not supported; see stderr" % (self.channels, self.sample_rate))

    def _check(self, what):
        if self.h is None:
            raise ValueError("GetStream.%s: the stream is closed" % what)
        if self._finished:
            raise ValueError("GetStream.%s: the stream is finished" % what)

    def feed(self, pcm, n_frames=None):
        self._check("feed")
        if isinstance(pcm, np.ndarray):
            if pcm.ndim != 2 or pcm.shape[1] != self.channels:
                raise ValueError("GetStream.feed: expected [n, %d] frames, got shape %s" % (self.channels, pcm.shape))
            pcm = np.ascontiguousarray(pcm, np.float32)
            n_frames = pcm.shape[0]
        elif n_frames is None:
            raise ValueError("GetStream.feed: a device pointer needs n_frames")
        rc = load().awmh_gs_feed(ctypes.c_void_p(self.h), _ptr(pcm), ctypes.c_size_t(int(n_frames)))
        if rc:
            raise RuntimeError("awmh_gs_feed failed (rc=%d); see stderr" % rc)

    def finish(self, parse=True):
        self._check("finish")
        self._finished = True
        cap = 1 << 22
        buf = _outbuf("get", cap)
        n_pat = ctypes.c_int()
        rc = load().awmh_gs_finish(ctypes.c_void_p(self.h), buf, ctypes.c_size_t(cap), ctypes.byref(n_pat))
        if rc:
            raise RuntimeError("awmh_gs_finish failed (rc=%d); see stderr" % rc)
        text = buf.value.decode()
        return json.loads(text) if parse else text

    def peak_bytes(self) -> int:
        """device bytes the stream holds at most: its chunk buffer plus, at other rates, its input window"""
        if self.h is None:
            raise ValueError("GetStream.peak_bytes: the stream is closed")
        return int(load().awmh_gs_peak_bytes(ctypes.c_void_p(self.h)))

    def close(self):
        if self.h:
            load().awmh_gs_destroy(ctypes.c_void_p(self.h))
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            self.close()


def get_stream_plan(n_total: int, piece_frames: int, sample_rate=44100):
    """test aid (CPU): the chunks GetStream decodes for a stream of n_total frames fed in pieces of piece_frames, without a device ->
    ([(first, n_frames, time_offset)], watermark-rate length), frames at the watermark rate"""
    cap = 4096
    chunks = np.zeros((cap, 3), np.float64)
    n, m = ctypes.c_int(), ctypes.c_uint64()
    if load().awmh_gs_plan(ctypes.c_uint64(n_total), ctypes.c_uint64(piece_frames), ctypes.c_int(sample_rate), _ptr(chunks), ctypes.c_int(cap),
                           ctypes.byref(n), ctypes.byref(m)):
        raise ValueError("get_stream_plan: sample rate %d Hz or piece size %d refused" % (sample_rate, piece_frames))
    if n.value > cap:
        raise ValueError("get_stream_plan: more than %d chunks" % cap)
    return [(int(a), int(b), float(t)) for a, b, t in chunks[:n.value]], m.value


def sync_trace(on=True):
    """test aid: record what every SyncFinder::search call returns from now on (see sync_trace_fetch)"""
    load().awmh_sync_trace(ctypes.c_int(1 if on else 0))


def sync_trace_fetch():
    """-> list of searches in call order: {"mode": "BLOCK"|"CLIP", "n_frames": int, "scores": [[index, quality, "A"|"B"], ...]}
    (the format of oracle/ref_shims/sync_dump.cc's print-out as tests/golden/make_golden_large.py stores it)"""
    cap = 1 << 16
    rows = np.zeros((cap, 5), np.float64)
    n = ctypes.c_size_t()
    if load().awmh_sync_trace_fetch(_ptr(rows), ctypes.c_size_t(cap), ctypes.byref(n)):
        raise RuntimeError("sync trace longer than %d rows" % cap)
    out = []
    for r in rows[:n.value]:
        if r[3] < 0:
            out.append({"mode": "CLIP" if r[1] else "BLOCK", "n_frames": int(r[2]), "scores": []})
        else:
            out[-1]["scores"].append([int(r[1]), float(r[2]), "B" if r[3] else "A"])
    return out


def set_short_payload(bits=0):
    """--short <bits> (12, 16, 20); 0 = normal 128 bit payload"""
    if load().awmh_set_short_payload(ctypes.c_int(bits)) < 0:
        raise ValueError("unsupported short payload size %d" % bits)


def set_speed_params(detect_speed=False, detect_speed_patient=False, try_speed=-1.0, test_speed=-1.0):
    """--detect-speed / --detect-speed-patient / --try-speed / --test-speed of `audiowmark get`"""
    load().awmh_set_speed_params(ctypes.c_int(int(detect_speed)), ctypes.c_int(int(detect_speed_patient)), ctypes.c_double(try_speed),
                                 ctypes.c_double(test_speed))


def detect_speed(pcm, key=None, n_frames=None, channels=None, sample_rate=44100):
    """detect_speed for one key on one chunk -> (speed, quality, accepted)"""
    if isinstance(pcm, np.ndarray):
        pcm = np.ascontiguousarray(pcm, np.float32)
        n_frames, channels = pcm.shape
    sp, q, acc = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
    rc = load().awmh_detect_speed(_key(key or bytes(16)), _ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels), ctypes.c_int(sample_rate),
                                  ctypes.byref(sp), ctypes.byref(q), ctypes.byref(acc))
    if rc:
        raise RuntimeError("awmh_detect_speed failed (rc=%d); see stderr" % rc)
    return sp.value, q.value, bool(acc.value)


def resample(pcm, ratio, n_out=None, out=None, n_frames=None, channels=None):
    """resample_ratio: numpy in -> numpy out, or device pointers with n_frames / channels / n_out given"""
    if isinstance(pcm, np.ndarray):
        pcm = np.ascontiguousarray(pcm, np.float32)
        n_frames, channels = pcm.shape
    if n_out is None:
        n_out = int(np.rint(n_frames * ratio))
    res = out
    if out is None:
        res = np.zeros((n_out, channels), np.float32)
    rc = load().awmh_resample(_ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels), ctypes.c_double(ratio), _ptr(res), ctypes.c_size_t(n_out))
    if rc:
        raise RuntimeError("awmh_resample failed (rc=%d); see stderr" % rc)
    return res


def resample_stream_frames(n_in, ratio):
    L = load()
    L.awmh_resample_stream_frames.restype = ctypes.c_uint64
    return int(L.awmh_resample_stream_frames(ctypes.c_uint64(n_in), ctypes.c_double(ratio)))


def resample_stream_available(fed, ratio):
    L = load()
    L.awmh_resample_stream_available.restype = ctypes.c_uint64
    return int(L.awmh_resample_stream_available(ctypes.c_uint64(fed), ctypes.c_double(ratio)))


def resampled_add_plan(n_frames, sample_rate):
    """(frames through the mixer, WatermarkGen::run calls) of `add` at a sample rate other than 44.1 kHz"""
    e, r = ctypes.c_uint64(), ctypes.c_uint64()
    load().awmh_resampled_add_plan(ctypes.c_uint64(n_frames), ctypes.c_int(sample_rate), ctypes.byref(e), ctypes.byref(r))
    return e.value, r.value


def add_s16(pcm_in, payload_hex: str, key=None, pcm_out=None, sample_rate=44100, want_stats=False, first_frame_number=0):
    """`add` between 16 bit PCM host buffers (int16 numpy [n, ch]): the int <-> float conversions run on the device"""
    pcm_in = np.ascontiguousarray(pcm_in, np.int16)
    n_frames, channels = pcm_in.shape
    if pcm_out is None:
        pcm_out = np.empty_like(pcm_in)
    blocks, snr = ctypes.c_int(), ctypes.c_double()
    rc = load().awmh_add_s16(_key(key), _ptr(pcm_in), _ptr(pcm_out), ctypes.c_size_t(n_frames), ctypes.c_int(channels), ctypes.c_int(sample_rate),
                             payload_hex.encode(), ctypes.byref(blocks) if want_stats else None, ctypes.byref(snr) if want_stats else None,
                             ctypes.c_uint64(first_frame_number))
    if rc:
        raise RuntimeError("awmh_add_s16 failed (rc=%d); see stderr" % rc)
    return (pcm_out, blocks.value, snr.value) if want_stats else pcm_out


def get_s16(pcm, keys=None, names=None, sample_rate=44100, parse=True):
    """`get` on a 16 bit PCM host buffer (int16 numpy [n, ch]) -> the --json document"""
    keys = keys or [bytes(16)]
    names = names or [""] * len(keys)
    pcm = np.ascontiguousarray(pcm, np.int16)
    n_frames, channels = pcm.shape
    kb = b"".join(_key(k) for k in keys)
    name_arr = (ctypes.c_char_p * len(keys))(*[n.encode() for n in names])
    cap = 1 << 22
    buf = _outbuf("get", cap)
    n_pat = ctypes.c_int()
    rc = load().awmh_get_s16(kb, name_arr, ctypes.c_int(len(keys)), _ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                             ctypes.c_int(sample_rate), buf, ctypes.c_size_t(cap), ctypes.byref(n_pat))
    if rc:
        raise RuntimeError("awmh_get_s16 failed (rc=%d); see stderr" % rc)
    text = buf.value.decode()
    return json.loads(text) if parse else text


def chunk_geometry(sample_rate=44100):
    """(max_frames, overlap_frames) of the reference's WavChunkLoader for the current --chunk-size."""
    m, o = ctypes.c_uint64(), ctypes.c_uint64()
    load().awmh_chunk_geometry(ctypes.c_int(sample_rate), ctypes.byref(m), ctypes.byref(o))
    return m.value, o.value


def merge_chunks(blobs, time_offsets, total_seconds: float, keys=None, names=None) -> dict:
    """test aid (CPU): ResultSet::merge in chunk order + sort -> the --json document, from per-chunk pattern records (bytes in the
    record format of host/awm_hostapi.cc) that a test writes, so that the C++ ResultSet can be checked against the oracle's."""
    keys = keys or [bytes(16)]
    names = names or [""] * len(keys)
    kb = b"".join(_key(k) for k in keys)
    name_arr = (ctypes.c_char_p * len(keys))(*[n.encode() for n in names])
    n = len(blobs)
    bufs = [(ctypes.c_ubyte * max(len(b), 1)).from_buffer_copy(b if b else b"\0") for b in blobs]
    ptrs = (ctypes.POINTER(ctypes.c_ubyte) * n)(*[ctypes.cast(b, ctypes.POINTER(ctypes.c_ubyte)) for b in bufs])
    lens = (ctypes.c_size_t * n)(*[len(b) for b in blobs])
    offs = (ctypes.c_double * n)(*time_offsets)
    cap = 1 << 22
    out = _outbuf("merge", cap)
    rc = load().awmh_merge_chunks(kb, name_arr, ctypes.c_int(len(keys)), ptrs, lens, offs, ctypes.c_int(n), ctypes.c_double(total_seconds),
                                  out, ctypes.c_size_t(cap))
    if rc:
        raise RuntimeError("awmh_merge_chunks failed (rc=%d)" % rc)
    return json.loads(out.value.decode())


# ---- sharded get: one long stream over several GPUs, one process per GPU (host/awm_balanced.hh) -----------------------------

def dist_unique_id() -> bytes:
    """NCCL unique id of a new job (rank 0 creates it, the launcher hands it to every rank)"""
    buf = ctypes.create_string_buffer(128)
    if load().awmh_dist_unique_id(buf):
        raise RuntimeError("NCCL is not available")
    return buf.raw


def dist_init(rank: int, world: int, unique_id: bytes):
    """join the job's NCCL communicator (exchanges of the sharded get run on the context stream)"""
    if load().awmh_dist_init(ctypes.c_int(rank), ctypes.c_int(world), ctypes.c_char_p(unique_id)):
        raise RuntimeError("awmh_dist_init failed; see stderr")


def dist_init_from_torch():
    """the usual launcher: torch.distributed is up (torchrun); rank 0's id is broadcast through it"""
    import torch
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", torch.cuda.current_device())
    t = torch.zeros(128, dtype=torch.uint8, device=dev)
    if rank == 0:
        t.copy_(torch.frombuffer(bytearray(dist_unique_id()), dtype=torch.uint8))
    dist.broadcast(t, 0)
    dist_init(rank, world, bytes(t.cpu().numpy().tobytes()))


def balanced_get(pcm, pcm_start: int, n_total: int, key=None, n_frames=None, channels=None, sample_rate=44100, parse=True):
    """this rank's part of the stream (numpy float32 / int16 [n, ch], or a float32 device pointer) -> the --json document on rank 0
    (parse=False: its text, as `audiowmark get --json` writes it), None on the other ranks.  The part starts at stream frame
    pcm_start and must cover balanced_input_range(n_total, rank, world, sample_rate); at a rate other than 44.1 kHz every rank
    resamples only that part, on its device"""
    is_s16 = 0
    if isinstance(pcm, np.ndarray):
        if pcm.dtype == np.int16:
            pcm, is_s16 = np.ascontiguousarray(pcm), 1
        else:
            pcm = np.ascontiguousarray(pcm, np.float32)
        n_frames, channels = pcm.shape
    cap = 1 << 22
    buf = _outbuf("get", cap)
    n_pat = ctypes.c_int()
    rc = load().awmh_balanced_get(_key(key), _ptr(pcm), ctypes.c_int(is_s16), ctypes.c_uint64(pcm_start), ctypes.c_uint64(n_frames), ctypes.c_uint64(n_total),
                                  ctypes.c_int(channels), ctypes.c_int(sample_rate), buf, ctypes.c_size_t(cap), ctypes.byref(n_pat))
    if rc:
        raise RuntimeError("awmh_balanced_get failed (rc=%d); see stderr" % rc)
    if n_pat.value < 0:
        return None
    text = buf.value.decode()
    return json.loads(text) if parse else text


class BalancedStages:
    """one rank of the sharded get with the stages callable one by one (tests run several ranks in one process on one GPU)"""

    def __init__(self, rank, world, n_total, pcm_device_ptr: int, pcm_frames: int, channels: int, pcm_start, key=None, sample_rate=44100):
        """pcm_device_ptr: float32 [pcm_frames, channels] in device memory that stays valid while the object lives (several ranks in
        one process share the context, so each needs its own device copy -- a host buffer would land in the context's single
        upload buffer); stream frames [pcm_start, pcm_start + pcm_frames) at sample_rate, covering balanced_input_range"""
        self.n_total = n_total
        L = load()
        L.awmh_bg_create.restype = ctypes.c_void_p
        self.h = L.awmh_bg_create(_key(key), ctypes.c_int(rank), ctypes.c_int(world), ctypes.c_void_p(pcm_device_ptr), ctypes.c_uint64(pcm_start),
                                  ctypes.c_uint64(pcm_frames), ctypes.c_uint64(n_total), ctypes.c_int(channels), ctypes.c_int(sample_rate))
        if not self.h:
            raise RuntimeError("awmh_bg_create failed; see stderr")

    def stage(self, number: int, payloads=()) -> bytes:
        n = len(payloads)
        arr = (ctypes.c_char_p * max(n, 1))(*[bytes(p) for p in payloads]) if n else None
        lens = (ctypes.c_size_t * max(n, 1))(*[len(p) for p in payloads])
        cap = 1 << 24
        out = _outbuf("bg", cap)
        out_len = ctypes.c_size_t()
        rc = load().awmh_bg_stage(ctypes.c_void_p(self.h), ctypes.c_int(number), arr, lens, ctypes.c_int(n), ctypes.c_uint64(self.n_total), out, ctypes.c_size_t(cap),
                                  ctypes.byref(out_len))
        if rc:
            raise RuntimeError("awmh_bg_stage %d failed (rc=%d)" % (number, rc))
        return out.raw[:out_len.value]

    def close(self):
        if self.h:
            load().awmh_bg_destroy(ctypes.c_void_p(self.h))
            self.h = None


def balanced_plan(n_total: int, rank: int, world: int, sample_rate=44100):
    """-> (chunks [(first, count, time offset)], slices [(chunk, sa, sb, a, b, lo, hi)]) as the C++ driver computes them.  A stream of
    n_total frames at sample_rate is planned as the driver runs it: in 44.1 kHz frames of the stream resampled to the watermark rate"""
    chunks = np.zeros((64, 3), np.float64)
    slices = np.zeros((64, 7), np.int64)
    nc, ns = ctypes.c_int(), ctypes.c_int()
    if load().awmh_bg_plan(ctypes.c_uint64(n_total), ctypes.c_int(sample_rate), ctypes.c_int(rank), ctypes.c_int(world), _ptr(chunks), ctypes.c_int(64),
                           ctypes.byref(nc), _ptr(slices), ctypes.c_int(64), ctypes.byref(ns)):
        raise ValueError("sharded get: sample rate %d Hz is outside the resampler's range" % sample_rate)
    return [(int(a), int(b), float(t)) for a, b, t in chunks[:nc.value]], [tuple(int(v) for v in row) for row in slices[:ns.value]]


def balanced_owner(n_total: int, world: int, chunk: int, index: int, sample_rate=44100) -> int:
    r = load().awmh_bg_owner(ctypes.c_uint64(n_total), ctypes.c_int(sample_rate), ctypes.c_int(world), ctypes.c_int(chunk), ctypes.c_uint64(index))
    if r < 0:
        raise ValueError("sharded get: sample rate %d Hz is outside the resampler's range" % sample_rate)
    return r


def balanced_input_range(n_total: int, rank: int, world: int, sample_rate=44100) -> tuple[int, int]:
    """stream frames [first, end) at sample_rate that rank `rank` of `world` has to hold for balanced_get: the union of its slices at
    44.1 kHz; at other rates every frame the resampler taps of that union read, plus one frame on each side.  (0, 0) for a rank
    without slices"""
    first, end = ctypes.c_uint64(), ctypes.c_uint64()
    if load().awmh_bg_input_range(ctypes.c_uint64(n_total), ctypes.c_int(rank), ctypes.c_int(world), ctypes.c_int(sample_rate), ctypes.byref(first),
                                  ctypes.byref(end)):
        raise ValueError("sharded get: sample rate %d Hz / rank %d of %d not supported" % (sample_rate, rank, world))
    return first.value, end.value


def engine_ctx() -> int:
    """awm_ctx* of the host library's GPU context (creates it; raises without a CUDA device)"""
    h = load().awmh_ctx()
    if not h:
        raise RuntimeError("no GPU context: a CUDA device is required, there is no CPU fallback")
    return int(h)


def key_slot(key=None) -> int:
    s = load().awmh_key_slot(_key(key))
    if s < 0:
        raise RuntimeError("key table upload failed")
    return s


def stage_select(peaks: np.ndarray, floor_q: float, clip_mode=False):
    """test aid (CPU): the candidate selection of `get` (select_candidates_from_peaks) on a peak list -> (candidates, complete)"""
    pk = np.ascontiguousarray(peaks, capi.SEARCH_SCORE)
    out = np.zeros(max(len(pk), 1), capi.SEARCH_SCORE)
    n, complete = ctypes.c_size_t(), ctypes.c_int()
    rc = load().awmh_stage_select(_ptr(pk), ctypes.c_size_t(len(pk)), ctypes.c_double(floor_q), ctypes.c_int(1 if clip_mode else 0),
                                  _ptr(out), ctypes.c_size_t(len(out)), ctypes.byref(n), ctypes.byref(complete))
    if rc:
        raise RuntimeError("awmh_stage_select failed (%d)" % rc)
    return out[:n.value].copy(), bool(complete.value)


def gpu_launches() -> int:
    return int(load().awmh_gpu_launches())


def gpu_stream() -> int:
    return int(load().awmh_gpu_stream() or 0)


def synchronize():
    """wait for the context stream (calls with DEVICE pointers are asynchronous)."""
    if load().awmh_synchronize():
        raise RuntimeError("no GPU context")


def profile_enable(on=True):
    if load().awmh_profile_enable(ctypes.c_int(1 if on else 0)):
        raise RuntimeError("no GPU context")


def profile_report() -> dict:
    buf = ctypes.create_string_buffer(1 << 16)
    if load().awmh_profile_report(buf, ctypes.c_size_t(len(buf))):
        raise RuntimeError("awmh_profile_report failed")
    return json.loads(buf.value.decode())


def shutdown():
    if _lib is not None:
        _lib.awmh_shutdown()
