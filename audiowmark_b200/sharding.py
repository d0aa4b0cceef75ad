"""Plan functions of the multi-GPU run of one long stream (one process per GPU).

The sharded `get` itself is C++ (host/awm_balanced.cc, reached through hostapi.balanced_get): the reference's 30-minute chunks are
kept, every rank owns an equal span of stream positions and searches, for each chunk that overlaps its span, the slice of the chunk's
start frames it owns; three ncclAllGather exchanges of small lists on the context stream.  What lives here is what bench.py and the
CPU tests need around it: the reference's chunk walk (WavChunkLoader: 30 min, 134.4 s overlap; src/wavchunkloader.cc:54-163), the
slices of a rank and the owner of an index (a mirror of the C++ planner, tests/test_sharding_cpu.py holds the two equal), the input
range a rank holds, and the range a rank has to embed so that its slices read exactly what the unsharded `add` would have written
(`add` shards by frame blocks with a recomputed halo: one 1024-frame for the synthesis window tails, two limiter blocks for the gain
ramp).
"""
from __future__ import annotations

import math

import numpy as np

FRAME = 1024
MARK_RATE = 44100              # the watermark rate: a stream at another rate is planned after resampling to it
T_BLOCK = 2226                 # frames per block (payload 128 bit): sync pattern length in BLOCK mode
MARGIN = 6                     # start frames of margin on each side of a slice (local mean uses +-20 scores = +-5 frames)


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
