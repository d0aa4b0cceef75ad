"""Plan functions of the multi-GPU run of one long stream (one process per GPU, torch.distributed).

The sharded `get` itself is C++ (host/awm_balanced.cc: every rank searches an equal slice of the start frames of every chunk its span
of positions overlaps; three ncclAllGather exchanges of small lists; hostapi.balanced_get).  What lives here is what bench.py and the
CPU tests need around it: the reference's chunk walk (WavChunkLoader: 30 min, 134.4 s overlap; src/wavchunkloader.cc:54-163), the
slices of a rank (a mirror of the C++ planner, tests/test_sharding_cpu.py holds the two equal), the range a rank has to embed so that
its slices read exactly what the unsharded `add` would have written (`add` shards by frame blocks with a recomputed halo: one
1024-frame for the synthesis window tails, two limiter blocks for the gain ramp), and the blob helpers of the chunk-granular variant.
"""
from __future__ import annotations

import os
import struct

FRAME = 1024


def chunk_plan(n_frames: int, max_frames: int, overlap: int, rate: int = 44100):
    """[(first_frame, n_frames_in_chunk, time_offset_seconds)] exactly as get_watermark_buffer walks a stream."""
    if n_frames <= 0:
        return []
    out = []
    start, end, toff = 0, min(max_frames, n_frames), 0.0
    eof = end < max_frames
    while True:
        out.append((start, end - start, toff))
        if eof:
            break
        toff += float(end - start - overlap) / rate
        start = end - overlap
        new_end = min(start + max_frames, n_frames)
        eof = (new_end - start) < max_frames
        end = new_end
    return out


def assign_chunks(n_chunks: int, world: int):
    """contiguous, balanced: rank r gets chunks [lo, hi)."""
    base, extra = divmod(n_chunks, world)
    out, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < extra else 0)
        out.append((lo, hi))
        lo = hi
    return out


def embed_range(own_start: int, own_end: int, n_frames: int, limiter_block: int):
    """Extended range [ext_start, ext_end) a rank has to embed so that [own_start, own_end) comes out exactly as in the
    unsharded run.  ext_start is a multiple of 1024 (-> first_frame_number); returns (ext_start, ext_end, first_frame_number).
    44.1 kHz only: at any sample rate a rank takes its range from hostapi.window_range and marks it with hostapi.add_window."""
    if own_start <= 0:
        ext_start = 0
    else:
        b = own_start // limiter_block                     # first owned limiter block
        lo = max(b - 1, 0) * limiter_block                 # the block before it must be complete
        ext_start = max((lo // FRAME) * FRAME - FRAME, 0)  # + one frame for the synthesis-window tail
    if own_end >= n_frames:
        ext_end = n_frames
    else:
        b = (own_end - 1) // limiter_block                 # last owned limiter block
        hi = (b + 2) * limiter_block                       # the block after it must be complete
        ext_end = ext_start + -(-(hi - ext_start) // FRAME) * FRAME + FRAME
        ext_end = min(ext_end, n_frames)
    return ext_start, ext_end, ext_start // FRAME


def rank_ranges(n_frames: int, rank: int, world: int, max_frames: int, overlap: int, rate: int = 44100):
    """chunks of this rank and the PCM range [lo, hi) they cover."""
    plan = chunk_plan(n_frames, max_frames, overlap, rate)
    lo_c, hi_c = assign_chunks(len(plan), world)[rank]
    mine = plan[lo_c:hi_c]
    if not mine:
        return plan, (lo_c, hi_c), None
    return plan, (lo_c, hi_c), (mine[0][0], mine[-1][0] + mine[-1][1])


# ---- gathering chunk results ---------------------------------------------------------------------------------------

def pack_blobs(blobs) -> bytes:
    """[(chunk_index, bytes)] -> one byte string."""
    out = struct.pack("<I", len(blobs))
    for idx, b in blobs:
        out += struct.pack("<II", idx, len(b)) + b
    return out


def unpack_blobs(data: bytes):
    n, = struct.unpack_from("<I", data, 0)
    pos, out = 4, []
    for _ in range(n):
        idx, ln = struct.unpack_from("<II", data, pos)
        pos += 8
        out.append((idx, bytes(data[pos:pos + ln])))
        pos += ln
    return out


def gather_blobs(blobs, device=None):
    """all ranks -> list over ranks of [(chunk_index, bytes)].  Uses tensor collectives (all_gather of sizes, then of
    padded byte tensors) so it runs on NCCL (device = cuda) and on gloo (device = None / cpu)."""
    import torch
    import torch.distributed as dist
    payload = pack_blobs(blobs)
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return [unpack_blobs(payload)]
    world = dist.get_world_size()
    dev = device if device is not None else torch.device("cpu")
    size = torch.tensor([len(payload)], dtype=torch.int64, device=dev)
    sizes = [torch.zeros_like(size) for _ in range(world)]
    dist.all_gather(sizes, size)
    cap = int(max(int(s.item()) for s in sizes))
    buf = torch.zeros(cap, dtype=torch.uint8, device=dev)
    buf[:len(payload)] = torch.frombuffer(bytearray(payload), dtype=torch.uint8).to(dev)
    bufs = [torch.zeros_like(buf) for _ in range(world)]
    dist.all_gather(bufs, buf)
    return [unpack_blobs(bytes(b[:int(s.item())].cpu().numpy().tobytes())) for b, s in zip(bufs, sizes)]


# =====================================================================================================================
# Frame-balanced `get` across ranks: the driver is C++ (audiowmark_b200/host/awm_balanced.cc, reached through
# hostapi.balanced_get; exchanges = ncclAllGather on the context stream).  Chunk sharding above is exact but coarse
# (30-minute units); there every rank owns an equal span of stream POSITIONS and searches, for each chunk that overlaps its
# span, the slice of the chunk's start frames it owns.  The plan functions below restate the C++ ones: bench.py uses them to
# decide which part of the stream a rank has to hold (and embed), tests/test_sharding_cpu.py checks that both agree.
# =====================================================================================================================

import math

import numpy as np

MARK_RATE = 44100              # the watermark rate: a stream at another rate is planned after resampling to it
T_BLOCK = 2226                 # frames per block (payload 128 bit): sync pattern length in BLOCK mode
MARGIN = 6                     # start frames of margin on each side of a slice (local mean uses +-20 scores = +-5 frames)


def owner_span(n_total: int, world: int) -> int:
    per = -(-n_total // world)
    return -(-per // FRAME) * FRAME


class Slice:
    __slots__ = ("chunk", "sa", "sb", "a", "b", "lo", "hi")

    def __init__(self, chunk, sa, sb, a, b, lo, hi):
        self.chunk, self.sa, self.sb, self.a, self.b, self.lo, self.hi = chunk, sa, sb, a, b, lo, hi


def rank_slices(plan, rank: int, world: int, n_total: int):
    """slices (chunk, owned start frames [sa,sb), searched [a,b), stream PCM range [lo,hi)) of one rank"""
    span = owner_span(n_total, world)
    out = []
    for c, (cs, cn, _) in enumerate(plan):
        n_starts = max(cn // FRAME - T_BLOCK - 1, 0)
        if n_starts == 0:
            continue
        # start frame s sits at stream position cs + s*1024; owner = position // span (last rank takes the remainder)
        def first_s(pos):                       # smallest s with cs + s*1024 >= pos
            return max(0, -(-(pos - cs) // FRAME))
        sa = min(first_s(rank * span), n_starts)
        sb = n_starts if rank == world - 1 else min(first_s((rank + 1) * span), n_starts)
        if sb <= sa:
            continue
        a, b = max(sa - MARGIN, 0), min(sb + MARGIN, n_starts)
        hi = cs + cn if b == n_starts else cs + (b + T_BLOCK + 1) * FRAME     # the last slice keeps the chunk's partial tail frame
        out.append(Slice(c, sa, sb, a, b, cs + a * FRAME, hi))
    return out


def index_owners(plan, n_total: int, world: int, chunk: int, indices) -> np.ndarray:
    """rank that owns each chunk-relative sample index (by the start frame it falls into): the rank whose slice of `chunk`
    contains that start frame in [sa, sb) (rank_slices uses the same position rule)"""
    cs, cn, _ = plan[chunk]
    n_starts = max(cn // FRAME - T_BLOCK - 1, 0)
    s = np.clip(np.asarray(indices, np.int64) // FRAME, 0, max(n_starts - 1, 0))
    span = owner_span(n_total, world)
    return np.minimum((cs + s * FRAME) // span, world - 1)


def rank_input_range(slices, n_total: int, sample_rate: int):
    """stream frames [first, end) at sample_rate that a rank with these slices (rank_slices of the stream at the watermark rate, of
    hostapi.resample_stream_frames(n_total, 44100 / sample_rate) frames) has to hold: at 44.1 kHz the union [min lo, max hi) of its
    slices; at other rates every input frame a resampler tap of that union reads -- output n has taps c(n) - 2h + 2 .. c(n) + 1,
    c(n) = floor((h - 1) + n * step) -- plus one frame on each side, inside [0, n_total).  (0, 0) without slices."""
    if not slices:
        return 0, 0
    lo, hi = min(sl.lo for sl in slices), max(sl.hi for sl in slices)
    if sample_rate == MARK_RATE:
        return lo, hi
    ratio = MARK_RATE / sample_rate
    h = int(math.ceil(16 / min(ratio, 1.0)))
    step = 1.0 / ratio

    def c(n):
        return math.floor(float(h - 1) + float(n) * step)
    first = min(max(c(lo) - 2 * h + 2 - 1, 0), n_total)
    end = min(max(c(hi - 1) + 2 + 1, first), n_total)
    return first, end
