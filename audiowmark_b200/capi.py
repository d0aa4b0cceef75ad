"""ctypes binding of the C ABI (include/awm_b200.h) exported by lib/libawm_b200.so.

Thin by design: arguments are numpy arrays (host) or raw device pointers (ints, e.g.
torch.Tensor.data_ptr()).  Nothing here computes; if the CUDA library is missing or no
device is usable every call fails loudly -- there is no CPU fallback.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libawm_b200.so")

FRAME = 1024
N_BANDS = 81
MODE_BLOCK, MODE_CLIP = 0, 1
BLOCK_A, BLOCK_B, BLOCK_AB = 0, 1, 2

SYNC_ENTRY = np.dtype([("frame", "<u2"), ("up", "u1", (30,)), ("down", "u1", (30,))])       # awm_sync_entry
MIX_ENTRY = np.dtype([("frame", "<u2"), ("up", "u1"), ("down", "u1")])                      # awm_mix_entry
SEARCH_SCORE = np.dtype([("index", "<u8"), ("raw_quality", "<f8"), ("local_mean", "<f8")])  # awm_search_score
BATCH_ITEM = np.dtype({"names": ["value_offset", "n_frames", "channels"], "formats": ["<u8", "<u8", "<i4"],
                       "offsets": [0, 8, 16], "itemsize": 24})                                 # awm_batch_item

EXPORTS = [
    "awm_create", "awm_destroy", "awm_last_error", "awm_launch_count", "awm_stream", "awm_synchronize",
    "awm_profile_enable", "awm_profile_report", "awm_host_alloc", "awm_host_free",
    "awm_fft_r2c", "awm_fft_c2r", "awm_set_embed_tables", "awm_set_sync_tables", "awm_set_mix_tables",
    "awm_pcm_bind", "awm_embed", "awm_sync_approx", "awm_sync_approx_enqueue", "awm_sync_use_slot", "awm_sync_have", "awm_sync_peaks", "awm_sync_refine", "awm_sync_refine_offsets", "awm_sync_refine_rescored", "awm_decode_blocks", "awm_viterbi",
    "awm_resample", "awm_pcm_push_resampled", "awm_pcm_pop", "awm_copy_to_host", "awm_copy", "awm_is_device_pointer", "awm_speed_scan", "awm_gather", "awm_pcm_bind_s16", "awm_pcm_device", "awm_embed_s16", "awm_embed_window", "awm_pcm_stage", "awm_pcm_stage_wait", "awm_dist_unique_id", "awm_dist_init", "awm_dist_world", "awm_dist_allgather",
    "awm_set_embed_roles", "awm_batch_validate", "awm_embed_batch", "awm_batch_rates_validate", "awm_embed_batch_rates",
    "awm_batch_offsets_validate", "awm_embed_batch_offsets", "awm_batch_rates_offsets_validate", "awm_embed_batch_rates_offsets",
    "awm_set_embed_roles_keys", "awm_get_embed_roles_keys", "awm_batch_keys_validate", "awm_embed_batch_keys",
    "awm_speed_mags", "awm_resampler_cache",
    "awm_resample_stream_available", "awm_resample_stream_frames", "awm_resample_taps", "awm_resample_range_validate", "awm_resample_range",
    "awm_device_alloc", "awm_device_free", "awm_embed_window_rates", "awm_window_range_rates",
]

_lib = None


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(the CUDA extension is mandatory, there is no CPU fallback)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        lib.awm_last_error.restype = ctypes.c_char_p
        lib.awm_launch_count.restype = ctypes.c_uint64
        lib.awm_stream.restype = ctypes.c_void_p
        _lib = lib
    return _lib


def _ptr(x):
    """numpy array -> host pointer, int -> device pointer."""
    if x is None:
        return ctypes.c_void_p(0)
    if isinstance(x, (int, np.integer)):
        return ctypes.c_void_p(int(x))
    assert x.flags["C_CONTIGUOUS"]
    return x.ctypes.data_as(ctypes.c_void_p)


class AwmError(RuntimeError):
    pass


def batch_validate(items, n_values: int) -> str:
    """awm_batch_validate: '' if every (value_offset, n_frames, channels) item fits a packed buffer of n_values values, else the reason"""
    it = np.array([tuple(int(v) for v in t) for t in items], BATCH_ITEM)
    err = ctypes.create_string_buffer(256)
    rc = load().awm_batch_validate(_ptr(it), ctypes.c_size_t(len(it)), ctypes.c_size_t(n_values), err, ctypes.c_size_t(len(err)))
    return err.value.decode() if rc else ""


def batch_rates_validate(items, n_values: int, sample_rates, n_emit=None, mark_sample_rate: int = 44100) -> str:
    """awm_batch_rates_validate: '' if the items fit a packed buffer of n_values values and every rate (and n_emit, if given) is
    acceptable, else the reason"""
    it = np.array([tuple(int(v) for v in t) for t in items], BATCH_ITEM)
    rates = np.ascontiguousarray(sample_rates, np.int32)
    emit = None if n_emit is None else np.ascontiguousarray(n_emit, np.uint64)
    err = ctypes.create_string_buffer(256)
    rc = load().awm_batch_rates_validate(_ptr(it), ctypes.c_size_t(len(it)), ctypes.c_size_t(n_values), _ptr(rates), _ptr(emit),
                                         ctypes.c_int(mark_sample_rate), err, ctypes.c_size_t(len(err)))
    return err.value.decode() if rc else ""


MAX_STREAM_FRAMES = 1 << 48          # AWM_MAX_STREAM_FRAMES: longest stream (zero_frames + n_frames) a batch item may end


def batch_offsets_validate(items, n_values: int, zero_frames, sample_rate: int = 44100, mark_sample_rate: int = 44100) -> str:
    """awm_batch_offsets_validate: '' if the items fit a packed buffer of n_values values and every stream offset is acceptable at
    sample_rate, else the reason"""
    it = np.array([tuple(int(v) for v in t) for t in items], BATCH_ITEM)
    z = list(zero_frames)
    if len(z) != len(it):
        return "%d items but %d zero_frames" % (len(it), len(z))
    zf = np.array([int(v) for v in z], np.uint64)
    err = ctypes.create_string_buffer(256)
    rc = load().awm_batch_offsets_validate(_ptr(it), ctypes.c_size_t(len(it)), ctypes.c_size_t(n_values), _ptr(zf), ctypes.c_int(sample_rate),
                                           ctypes.c_int(mark_sample_rate), err, ctypes.c_size_t(len(err)))
    return err.value.decode() if rc else ""


def batch_rates_offsets_validate(items, n_values: int, sample_rates, zero_frames, n_emit=None, mark_sample_rate: int = 44100) -> str:
    """awm_batch_rates_offsets_validate: '' if awm_batch_rates_validate accepts the items and rates and every stream offset (frames at
    the item's rate) is acceptable, else the reason"""
    it = np.array([tuple(int(v) for v in t) for t in items], BATCH_ITEM)
    rates = np.ascontiguousarray(sample_rates, np.int32)
    emit = None if n_emit is None else np.ascontiguousarray(n_emit, np.uint64)
    z = list(zero_frames)
    if len(z) != len(it):
        return "%d items but %d zero_frames" % (len(it), len(z))
    zf = np.array([int(v) for v in z], np.uint64)
    err = ctypes.create_string_buffer(256)
    rc = load().awm_batch_rates_offsets_validate(_ptr(it), ctypes.c_size_t(len(it)), ctypes.c_size_t(n_values), _ptr(rates), _ptr(emit),
                                                 _ptr(zf), ctypes.c_int(mark_sample_rate), err, ctypes.c_size_t(len(err)))
    return err.value.decode() if rc else ""


def batch_keys_validate(items, n_values: int, key_index, n_keys: int, sample_rates=None, zero_frames=None, n_emit=None,
                        mark_sample_rate: int = 44100) -> str:
    """awm_batch_keys_validate: '' if the checks of the matching single-key validator pass and every key index (None: a NULL list) is
    below n_keys, else the reason"""
    it = np.array([tuple(int(v) for v in t) for t in items], BATCH_ITEM)
    rates = None if sample_rates is None else np.ascontiguousarray(sample_rates, np.int32)
    emit = None if n_emit is None else np.ascontiguousarray(n_emit, np.uint64)
    zf = None if zero_frames is None else np.array([int(v) for v in zero_frames], np.uint64)
    ki = None if key_index is None else np.array([int(v) for v in key_index], np.uint32)
    for name, arr in (("sample_rates", rates), ("zero_frames", zf), ("key_index", ki)):
        if arr is not None and len(arr) != len(it):
            return "%d items but %d %s" % (len(it), len(arr), name)
    err = ctypes.create_string_buffer(256)
    rc = load().awm_batch_keys_validate(_ptr(it), ctypes.c_size_t(len(it)), ctypes.c_size_t(n_values), _ptr(rates), _ptr(emit), _ptr(zf), _ptr(ki),
                                        ctypes.c_size_t(n_keys), ctypes.c_int(mark_sample_rate), err, ctypes.c_size_t(len(err)))
    return err.value.decode() if rc else ""


def resample_taps(n_in_total: int, ratio: float, out_first: int, out_frames: int, hlen: int = 16) -> tuple[int, int]:
    """awm_resample_taps: input frames [first, end) the taps of outputs [out_first, out_first + out_frames) read, inside the stream"""
    first, end = ctypes.c_uint64(), ctypes.c_uint64()
    load().awm_resample_taps(ctypes.c_uint64(n_in_total), ctypes.c_double(ratio), ctypes.c_int(hlen), ctypes.c_uint64(out_first),
                             ctypes.c_uint64(out_frames), ctypes.byref(first), ctypes.byref(end))
    return first.value, end.value


def window_range_rates(own_first: int, own_end: int, n_total: int, sample_rate: int, mark_sample_rate: int = 44100, limiter_ms: int = 1000,
                       hlen: int = 16) -> tuple[int, int]:
    """awm_window_range_rates: input frames [ext_first, ext_end) that make awm_embed_window_rates's outputs [own_first, own_end) exact
    (n_total = 2^64-1: the end is not known yet); ValueError for a range or rate the planner refuses"""
    first, end = ctypes.c_uint64(), ctypes.c_uint64()
    rc = load().awm_window_range_rates(ctypes.c_uint64(own_first), ctypes.c_uint64(own_end), ctypes.c_uint64(n_total), ctypes.c_int(sample_rate),
                                       ctypes.c_int(mark_sample_rate), ctypes.c_int(limiter_ms), ctypes.c_int(hlen), ctypes.byref(first), ctypes.byref(end))
    if rc:
        raise ValueError("awm_window_range_rates refuses own [%d, %d) of %d frames at %d Hz" % (own_first, own_end, n_total, sample_rate))
    return first.value, end.value


def resample_range_validate(in_first: int, in_frames: int, n_in_total: int, channels: int, ratio: float, out_first: int, out_frames: int,
                            hlen: int = 16) -> str:
    """awm_resample_range_validate: '' if awm_resample_range accepts the window, the ratio and the output range, else the reason"""
    err = ctypes.create_string_buffer(256)
    rc = load().awm_resample_range_validate(ctypes.c_uint64(in_first), ctypes.c_uint64(in_frames), ctypes.c_uint64(n_in_total), ctypes.c_int(channels),
                                            ctypes.c_double(ratio), ctypes.c_int(hlen), ctypes.c_uint64(out_first), ctypes.c_uint64(out_frames), err,
                                            ctypes.c_size_t(len(err)))
    return err.value.decode() if rc else ""


class Context:
    """One awm_ctx (device + stream)."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = ctypes.c_void_p()
        rc = self.lib.awm_create(ctypes.c_int(device), ctypes.byref(h))
        if rc != 0 or not h:
            raise AwmError("awm_create failed (rc=%d): no usable CUDA device; this package has no CPU fallback" % rc)
        self.h = h

    @classmethod
    def from_handle(cls, handle):
        """non-owning view of an existing awm_ctx* (the host library's engine context)"""
        self = cls.__new__(cls)
        self.lib = load()
        self.h = ctypes.c_void_p(handle)
        self._borrowed = True
        if not handle:
            raise AwmError("no GPU context (a CUDA device is required, there is no CPU fallback)")
        return self

    def close(self):
        if getattr(self, "h", None) and not getattr(self, "_borrowed", False):
            self.lib.awm_destroy(self.h)
        self.h = None

    __del__ = close

    def _ck(self, rc):
        if rc != 0:
            raise AwmError(self.lib.awm_last_error(self.h).decode())

    @property
    def launches(self) -> int:
        return int(self.lib.awm_launch_count(self.h))

    @property
    def stream(self) -> int:
        return int(self.lib.awm_stream(self.h) or 0)

    def synchronize(self):
        self._ck(self.lib.awm_synchronize(self.h))

    def profile_enable(self, on=True):
        self._ck(self.lib.awm_profile_enable(self.h, ctypes.c_int(1 if on else 0)))

    def profile_report(self) -> dict:
        import json
        buf = ctypes.create_string_buffer(1 << 16)
        self._ck(self.lib.awm_profile_report(self.h, buf, ctypes.c_size_t(len(buf))))
        return json.loads(buf.value.decode())

    # ---- FFTProcessor
    def fft_r2c(self, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, np.float32).reshape(-1, FRAME)
        out = np.empty((x.shape[0], FRAME + 2), np.float32)
        self._ck(self.lib.awm_fft_r2c(self.h, _ptr(x), _ptr(out), ctypes.c_size_t(x.shape[0]), ctypes.c_int(FRAME)))
        return out.view(np.complex64)

    def fft_c2r(self, spec: np.ndarray) -> np.ndarray:
        s = np.ascontiguousarray(spec, np.complex64).reshape(-1, FRAME // 2 + 1).view(np.float32)
        out = np.empty((s.shape[0], FRAME), np.float32)
        self._ck(self.lib.awm_fft_c2r(self.h, _ptr(s), _ptr(out), ctypes.c_size_t(s.shape[0]), ctypes.c_int(FRAME)))
        return out

    # ---- tables
    def set_embed_tables(self, frame_mod_ab: np.ndarray):
        fm = np.ascontiguousarray(frame_mod_ab, np.uint8)
        assert fm.ndim == 3 and fm.shape[0] == 2 and fm.shape[2] == 101
        self._ck(self.lib.awm_set_embed_tables(self.h, _ptr(fm), ctypes.c_int(fm.shape[1])))

    def set_embed_roles_keys(self, keys, layout):
        """awm_set_embed_roles_keys: build the role tables of keys (16-byte keys, or a uint8 array [n, 16]) on the device; layout: the 6
        ints of awm_role_layout (hostapi.role_layout())"""
        kb = np.ascontiguousarray(np.frombuffer(b"".join(bytes(k) for k in keys), np.uint8) if not isinstance(keys, np.ndarray) else keys, np.uint8)
        lay = np.ascontiguousarray(layout, np.int32)
        assert kb.size % 16 == 0 and lay.shape == (6,)
        self._ck(self.lib.awm_set_embed_roles_keys(self.h, _ptr(kb), ctypes.c_size_t(kb.size // 16), _ptr(lay)))

    def get_embed_roles_keys(self, first_key: int, n_keys: int, frames_per_block: int) -> np.ndarray:
        out = np.zeros((n_keys, frames_per_block, 101), np.uint16)
        self._ck(self.lib.awm_get_embed_roles_keys(self.h, ctypes.c_size_t(first_key), ctypes.c_size_t(n_keys), _ptr(out)))
        return out

    def set_sync_tables(self, key_slot: int, mode: int, entries: np.ndarray, bit_offsets: np.ndarray):
        e = np.ascontiguousarray(entries, SYNC_ENTRY)
        off = np.ascontiguousarray(bit_offsets, np.int32)
        self._ck(self.lib.awm_set_sync_tables(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), _ptr(e), ctypes.c_int(len(e)),
                                              _ptr(off), ctypes.c_int(len(off) - 1)))

    def set_mix_tables(self, key_slot: int, entries: np.ndarray, bit_order: np.ndarray, frames_per_bit: int, frames_per_block: int):
        e = np.ascontiguousarray(entries, MIX_ENTRY)
        o = np.ascontiguousarray(bit_order, np.uint16)
        self._ck(self.lib.awm_set_mix_tables(self.h, ctypes.c_int(key_slot), _ptr(e), ctypes.c_int(len(e)), _ptr(o), ctypes.c_int(len(o)),
                                             ctypes.c_int(frames_per_bit), ctypes.c_int(frames_per_block)))

    # ---- PCM
    def pcm_bind(self, pcm, n_frames: int | None = None, channels: int | None = None, pad_start: int = 0, pad_end: int = 0):
        if isinstance(pcm, np.ndarray) and pcm.dtype == np.int16:        # 16 bit PCM: converted on the device
            pcm = np.ascontiguousarray(pcm)
            n_frames, channels = pcm.shape
            self._keep = pcm
            self._ck(self.lib.awm_pcm_bind_s16(self.h, _ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                                               ctypes.c_size_t(pad_start), ctypes.c_size_t(pad_end)))
            self.synchronize()
            return
        if isinstance(pcm, np.ndarray):
            pcm = np.ascontiguousarray(pcm, np.float32)
            n_frames, channels = pcm.shape
            self._keep = pcm
        host = isinstance(pcm, np.ndarray)
        self._ck(self.lib.awm_pcm_bind(self.h, _ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                                       ctypes.c_size_t(pad_start), ctypes.c_size_t(pad_end)))
        if host or pad_start or pad_end:        # the asynchronous copy reads the caller's array; a device pointer is bound in place
            self.synchronize()

    # ---- embed
    def embed(self, pcm_in, pcm_out=None, n_frames=None, channels=None, first_frame_number=0, frames_pad_start=250,
              water_delta=0.01, limiter_block=44100, limiter_ceiling=0.99, want_snr=False):
        if isinstance(pcm_in, np.ndarray):
            pcm_in = np.ascontiguousarray(pcm_in, np.float32)
            n_frames, channels = pcm_in.shape
            if pcm_out is None:
                pcm_out = np.empty_like(pcm_in)
        snr = (ctypes.c_double * 2)()
        self._ck(self.lib.awm_embed(self.h, _ptr(pcm_in), _ptr(pcm_out), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                                    ctypes.c_uint64(first_frame_number), ctypes.c_int(frames_pad_start), ctypes.c_double(water_delta),
                                    ctypes.c_int(limiter_block), ctypes.c_float(limiter_ceiling), snr if want_snr else None))
        return (pcm_out, (snr[0], snr[1])) if want_snr else pcm_out

    def embed_s16(self, pcm_in, pcm_out=None, n_frames=None, channels=None, first_frame_number=0, frames_pad_start=250,
                  water_delta=0.01, limiter_block=44100, limiter_ceiling=0.99, want_snr=False):
        """awm_embed_s16: embed as awm_embed between 16 bit buffers (int16 numpy arrays or device pointers with sizes given)"""
        if isinstance(pcm_in, np.ndarray):
            pcm_in = np.ascontiguousarray(pcm_in, np.int16)
            n_frames, channels = pcm_in.shape
            if pcm_out is None:
                pcm_out = np.empty_like(pcm_in)
        snr = (ctypes.c_double * 2)()
        self._ck(self.lib.awm_embed_s16(self.h, _ptr(pcm_in), _ptr(pcm_out), ctypes.c_size_t(n_frames), ctypes.c_int(channels),
                                        ctypes.c_uint64(first_frame_number), ctypes.c_int(frames_pad_start), ctypes.c_double(water_delta),
                                        ctypes.c_int(limiter_block), ctypes.c_float(limiter_ceiling), snr if want_snr else None))
        return (pcm_out, (snr[0], snr[1])) if want_snr else pcm_out

    # ---- sync
    def sync_approx(self, key_slot=0, mode=MODE_BLOCK, wav_first=0, wav_last=None, water_delta=0.01) -> np.ndarray:
        if wav_last is None:
            wav_last = 0xFFFFFFFFFFFFFFF
        n = ctypes.c_size_t()
        self._ck(self.lib.awm_sync_approx(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first), ctypes.c_uint64(wav_last),
                                          ctypes.c_double(water_delta), None, ctypes.c_size_t(0), ctypes.byref(n)))
        out = np.zeros(n.value, SEARCH_SCORE)
        if n.value:
            self._ck(self.lib.awm_sync_approx(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first), ctypes.c_uint64(wav_last),
                                              ctypes.c_double(water_delta), _ptr(out), ctypes.c_size_t(n.value), ctypes.byref(n)))
        return out

    def sync_approx_run(self, key_slot=0, mode=MODE_BLOCK, wav_first=0, wav_last=None, water_delta=0.01) -> int:
        """run the search, keep the scores on the device (for sync_peaks); returns the number of scores"""
        if wav_last is None:
            wav_last = 0xFFFFFFFFFFFFFFF
        n = ctypes.c_size_t()
        self._ck(self.lib.awm_sync_approx(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first), ctypes.c_uint64(wav_last),
                                          ctypes.c_double(water_delta), None, ctypes.c_size_t(0), ctypes.byref(n)))
        return n.value

    def sync_approx_enqueue(self, slot: int, key_slot=0, mode=MODE_BLOCK, wav_first=0, wav_last=None, water_delta=0.01):
        """awm_sync_approx_enqueue: queue the search into approx slot `slot` (the bound PCM must be the caller's device memory)"""
        if wav_last is None:
            wav_last = 0xFFFFFFFFFFFFFFF
        self._ck(self.lib.awm_sync_approx_enqueue(self.h, ctypes.c_int(slot), ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first),
                                                  ctypes.c_uint64(wav_last), ctypes.c_double(water_delta)))

    def sync_use_slot(self, slot: int) -> int:
        """awm_sync_use_slot: make approx slot `slot` current; returns its number of scores"""
        n = ctypes.c_size_t()
        self._ck(self.lib.awm_sync_use_slot(self.h, ctypes.c_int(slot), ctypes.byref(n)))
        return n.value

    def sync_have(self) -> np.ndarray:
        """awm_sync_have: [4][frame_count - 1] bool, the frames the current slot's last search analysed"""
        n = ctypes.c_size_t()
        self._ck(self.lib.awm_sync_have(self.h, None, ctypes.c_size_t(0), ctypes.byref(n)))
        out = np.zeros((4, n.value), np.uint8)
        if n.value:
            self._ck(self.lib.awm_sync_have(self.h, _ptr(out), ctypes.c_size_t(out.size), ctypes.byref(n)))
        return out.astype(bool)

    def sync_peaks(self, min_abs_quality: float, max_peaks: int = 65536):
        """local maxima above a floor of the LAST sync_approx call; returns (peaks sorted by index, number found)."""
        out = np.empty(max_peaks, SEARCH_SCORE)
        n = ctypes.c_size_t()
        self._ck(self.lib.awm_sync_peaks(self.h, ctypes.c_double(min_abs_quality), _ptr(out), ctypes.c_size_t(max_peaks), ctypes.byref(n)))
        return out[:min(n.value, max_peaks)].copy(), n.value

    def sync_refine(self, scores: np.ndarray, key_slot=0, mode=MODE_BLOCK, wav_first=0, wav_last=None, water_delta=0.01) -> np.ndarray:
        if wav_last is None:
            wav_last = 0xFFFFFFFFFFFFFFF
        s = np.ascontiguousarray(scores, SEARCH_SCORE).copy()
        self._ck(self.lib.awm_sync_refine(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first), ctypes.c_uint64(wav_last),
                                          ctypes.c_double(water_delta), _ptr(s), ctypes.c_size_t(len(s))))
        return s

    def sync_refine_offsets(self, scores: np.ndarray, exact: bool, key_slot=0, mode=MODE_BLOCK, wav_first=0, wav_last=None, water_delta=0.01):
        """per-offset qualities of search_refine's 65 fine offsets: sliding-DFT ranking (exact=False) or fresh transforms (exact=True)"""
        if wav_last is None:
            wav_last = 0xFFFFFFFFFFFFFFF
        s = np.ascontiguousarray(scores, SEARCH_SCORE)
        q = np.zeros((len(s), 65), np.float64)
        valid = np.zeros((len(s), 65), np.uint8)
        self._ck(self.lib.awm_sync_refine_offsets(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first), ctypes.c_uint64(wav_last),
                                                  ctypes.c_double(water_delta), _ptr(s), ctypes.c_size_t(len(s)), ctypes.c_int(1 if exact else 0), _ptr(q), _ptr(valid)))
        return q, valid.astype(bool)

    def sync_refine_rescored(self, scores: np.ndarray, key_slot=0, mode=MODE_BLOCK, wav_first=0, wav_last=None, water_delta=0.01):
        """[n][65] bool: the fine offsets awm_sync_refine scores again exactly, as the device ranking picks them"""
        if wav_last is None:
            wav_last = 0xFFFFFFFFFFFFFFF
        s = np.ascontiguousarray(scores, SEARCH_SCORE)
        out = np.zeros((len(s), 65), np.uint8)
        self._ck(self.lib.awm_sync_refine_rescored(self.h, ctypes.c_int(key_slot), ctypes.c_int(mode), ctypes.c_uint64(wav_first), ctypes.c_uint64(wav_last),
                                                   ctypes.c_double(water_delta), _ptr(s), ctypes.c_size_t(len(s)), _ptr(out)))
        return out.astype(bool)

    # ---- decode
    def decode_blocks(self, indices, n_coded: int, key_slot=0):
        idx = np.ascontiguousarray(indices, np.uint64)
        raw = np.zeros((len(idx), n_coded), np.float32)
        valid = np.zeros(len(idx), np.int32)
        self._ck(self.lib.awm_decode_blocks(self.h, ctypes.c_int(key_slot), _ptr(idx), ctypes.c_size_t(len(idx)), _ptr(raw), _ptr(valid)))
        return raw, valid

    def viterbi(self, jobs, block_types, n_msg_bits=128, hard=False):
        """jobs: list of 1-D float arrays (or a 2-D array) of raw soft bits, one per code word (mixed A/B/AB allowed)."""
        jobs = [np.ascontiguousarray(j, np.float32).reshape(-1) for j in jobs]
        bt = np.ascontiguousarray(block_types, np.int32).reshape(-1)
        assert len(jobs) == len(bt)
        for j, t in zip(jobs, bt):
            assert len(j) == (12 if t == BLOCK_AB else 6) * (n_msg_bits + 15)
        raw = np.concatenate(jobs) if jobs else np.zeros(0, np.float32)
        bits = np.zeros((len(jobs), n_msg_bits), np.uint8)
        err = np.zeros(len(jobs), np.float32)
        self._ck(self.lib.awm_viterbi(self.h, _ptr(raw), ctypes.c_size_t(len(jobs)), ctypes.c_int(n_msg_bits), _ptr(bt), ctypes.c_int(1 if hard else 0),
                                      _ptr(bits), _ptr(err)))
        return bits, err

    def resample(self, pcm, ratio: float, n_out: int | None = None, hlen: int = 16, n_frames=None, channels=None, out=None):
        """awm_resample: numpy [n, ch] -> numpy [n_out, ch] (n_out defaults to lrint(n * ratio)); device pointers with sizes given"""
        if isinstance(pcm, np.ndarray):
            pcm = np.ascontiguousarray(pcm, np.float32)
            n_frames, channels = pcm.shape
        if n_out is None:
            n_out = int(np.rint(n_frames * ratio))
        res = np.zeros((n_out, channels), np.float32) if out is None else out
        self._ck(self.lib.awm_resample(self.h, _ptr(pcm), ctypes.c_size_t(n_frames), ctypes.c_int(channels), ctypes.c_double(ratio), ctypes.c_int(hlen),
                                       _ptr(res), ctypes.c_size_t(n_out)))
        return res

    def resample_range(self, window, in_first: int, n_in_total: int, ratio: float, out, out_first: int, out_frames: int, hlen: int = 16,
                       in_frames=None, channels=None):
        """awm_resample_range: outputs [out_first, out_first + out_frames) of resampling a stream of n_in_total frames, read from the
        window of stream frames [in_first, in_first + in_frames) (numpy [n, ch], or a device pointer with in_frames / channels given),
        written to the device pointer out"""
        if isinstance(window, np.ndarray):
            window = np.ascontiguousarray(window, np.float32)
            in_frames, channels = window.shape
        self._ck(self.lib.awm_resample_range(self.h, _ptr(window), ctypes.c_uint64(in_first), ctypes.c_uint64(in_frames), ctypes.c_uint64(n_in_total),
                                             ctypes.c_int(channels), ctypes.c_double(ratio), ctypes.c_int(hlen), _ptr(out), ctypes.c_uint64(out_first),
                                             ctypes.c_uint64(out_frames)))

    def pcm_push_resampled(self, ratio: float, n_out: int, hlen: int = 16):
        self._ck(self.lib.awm_pcm_push_resampled(self.h, ctypes.c_double(ratio), ctypes.c_int(hlen), ctypes.c_size_t(n_out)))

    def pcm_pop(self):
        self._ck(self.lib.awm_pcm_pop(self.h))

    def speed_scan(self, clip, seconds: float, centers, relative_speeds, key_slot=0, sample_rate=44100, water_delta=0.01,
                   n_frames=None, channels=None) -> np.ndarray:
        """awm_speed_scan: relative_speeds [n_centers][n_rel] -> quality [n_centers][n_rel]"""
        if isinstance(clip, np.ndarray):
            clip = np.ascontiguousarray(clip, np.float32)
            n_frames, channels = clip.shape
        centers = np.ascontiguousarray(centers, np.float64).reshape(-1)
        rel = np.ascontiguousarray(relative_speeds, np.float64).reshape(len(centers), -1)
        out = np.zeros(rel.shape, np.float64)
        self._ck(self.lib.awm_speed_scan(self.h, ctypes.c_int(key_slot), _ptr(clip), ctypes.c_size_t(n_frames), ctypes.c_int(channels), ctypes.c_int(sample_rate),
                                         ctypes.c_double(seconds), _ptr(centers), ctypes.c_int(len(centers)), _ptr(rel), ctypes.c_int(rel.shape[1]),
                                         ctypes.c_double(water_delta), _ptr(out)))
        return out

    def speed_mags(self, center: int) -> np.ndarray:
        """awm_speed_mags: the MagMatrix of centre `center` of the last speed_scan, float32 [n_entries][rows][2] (umag, dmag), entries in
        table order"""
        rows, n_ent = ctypes.c_int(), ctypes.c_int()
        self._ck(self.lib.awm_speed_mags(self.h, ctypes.c_int(center), None, ctypes.c_size_t(0), ctypes.byref(rows), ctypes.byref(n_ent)))
        out = np.zeros((n_ent.value, rows.value, 2), np.float32)
        if out.size:
            self._ck(self.lib.awm_speed_mags(self.h, ctypes.c_int(center), _ptr(out), ctypes.c_size_t(out.size // 2), ctypes.byref(rows),
                                             ctypes.byref(n_ent)))
        return out

    def resampler_cache(self) -> tuple[int, int]:
        """awm_resampler_cache: (filter tables held, tables held before the cache is emptied)"""
        size, cap = ctypes.c_size_t(), ctypes.c_size_t()
        self._ck(self.lib.awm_resampler_cache(self.h, ctypes.byref(size), ctypes.byref(cap)))
        return size.value, cap.value
