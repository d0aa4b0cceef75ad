"""The approximate sync search (awm_sync_approx: spectrogram + entry sums + per-bit gather + quality + local mean), awm_sync_peaks and
the sync table checks, against a float64 reference of the same operation written here in plain numpy.

The reference (`search_ref`) takes arbitrary tables: windowed frames (O.analysis_window) -> np.fft.rfft per channel in float64 ->
band dB (-96 for a power of exactly zero) summed over channels -> per entry U / D -> per-bit sums over the frames that were analysed
-> bit quality -> normalisation by min(water_delta, 0.08) * 2.9 -> local mean over j = -20..20, |j| >= 4 of the index-sorted list.
test_reference_matches_oracle pins it to O.SyncFinder.search_approx on real tables.

Error bound of a score (`search_ref` returns it next to the score).  Every dB term i carries a magnitude
    m_i = sum over channels of ( |dB| + (20 / ln 10) log2(1024) ||x w|| / |X_k| + (10 / ln 10) 2^-149 / (|X_k|^2 u) )
the dB value itself, its condition with respect to the fp32 FFT of the frame, and the spacing of fp32 denormals at the bin's power,
all in units of u = 2^-24.  A bit sums n = 30 * (frames analysed) terms into u and into d; recursive fp32 summation of n terms has an
error that grows like sqrt(n) u sum |term| (probabilistic bound, Higham and Mary 2019), so
    du <= LAMBDA sqrt(n) u sum_i m_i,        raw bit 1 - u/d:  dr <= du / |d| + |u| dd / d^2   (d/u - 1 symmetrically)
    dq <= sum_bits cnt_b dr_b / sum_bits cnt_b / (min(water_delta, 0.08) 2.9)
and the local mean's bound is the mean of its neighbours' bounds.  LAMBDA = 3.  The default kernel is held to the simt kernel
(the same per-entry sums on the fp32 pipes) with TIGHT = 1/4 of that bound: the two differ by the fp16 hi + lo representation of
each term (at most 2^-22 = 4u relative, so at most 4 u sum m <= 4 / (LAMBDA sqrt(30)) < 1/4 of the bound for any entry) and the
order of the additions, so a lost fp16 low term (2^-12 relative per term) shows there long before it shows against the reference.
Largest observed |error| / bound over the whole matrix on an H100 (NVIDIA H100 80GB HBM3, 700 W power limit): 0.014 for the ring
kernel and 0.059 for every kernel including the dynamic-range cases; default against simt 0.24 of the TIGHT bound (the 1-entry
table).  The tests print the running maxima with -s.
"""
import os

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi

P = O.Params()
U = 2.0 ** -24
LAMBDA = 3.0
TIGHT = 0.25
N = 1024
KEYS = (O.Key(), O.Key.test_key(7))
SYN = 9                                  # key slot of the synthetic tables
KERNELS = ("default", "simt", "ring")
RATIOS = {}


# ------------------------------------------------------------------------------------------------ float64 reference

def frame_db(x, shift, nfr):
    """channel-summed band dB [nfr][81] and per-term error magnitude m [nfr][81] (units of u) of the frames shift + f * 1024"""
    C = x.shape[1]
    win = O.analysis_window(N).astype(np.float64)
    db = np.zeros((nfr, P.n_bands))
    mag = np.zeros((nfr, P.n_bands))
    for f0 in range(0, nfr, 512):
        f = np.arange(f0, min(nfr, f0 + 512))
        idx = shift + f[:, None] * N + np.arange(N)[None, :]
        for ch in range(C):
            xw = x[idx, ch].astype(np.float64) * win
            X = np.fft.rfft(xw, axis=1)[:, P.min_band:P.max_band + 1]
            pw = X.real ** 2 + X.imag ** 2
            pos = pw > 0
            d = np.where(pos, 10 * np.log10(np.where(pos, pw, 1.0)), -96.0)
            nx = np.sqrt((xw * xw).sum(axis=1))[:, None]
            with np.errstate(divide="ignore", invalid="ignore"):
                cond = np.where(pos, (20 / np.log(10)) * 10 * nx / np.sqrt(np.where(pos, pw, 1.0))
                                + (10 / np.log(10)) * 2.0 ** -125 / np.where(pos, pw, 1.0), 0.0)
            db[f] += d
            mag[f] += np.abs(d) + cond
    return db, mag


def band_matrix(bands, n_ent):
    """[81][n_ent] count of each band in each entry's list (a repeated band counts every time it appears)"""
    M = np.zeros((P.n_bands, n_ent))
    np.add.at(M, (np.asarray(bands).reshape(n_ent, -1), np.arange(n_ent)[:, None]), 1.0)
    return M


def search_ref(x, entries, offsets, total, wav_first=0, wav_last=None, water_delta=0.01, clip=False):
    """float64 search_approx: (index [n], q [n], local mean [n], bound of q [n], bound of the local mean [n], have [4][n_out])"""
    x = np.ascontiguousarray(x, np.float32)
    n, C = x.shape
    if wav_last is None:
        wav_last = n * C
    fc = n // N
    nfr = max(fc - 1, 0)
    n_starts = max(fc - total - 1, 0)
    n_ent = len(entries)
    fr = entries["frame"].astype(np.int64)
    Mu, Md = band_matrix(entries["up"], n_ent), band_matrix(entries["down"], n_ent)
    n_bits = len(offsets) - 1
    norm = min(water_delta, 0.08) * 2.9
    q = np.zeros((n_starts, 4))
    qb = np.zeros((n_starts, 4))
    have_all = np.zeros((4, nfr), bool)
    s = np.arange(n_starts)
    for shift in range(4):
        start = shift * 256 + np.arange(nfr) * N
        have = ~(((start + N) * C < wav_first) | (start * C > wav_last))
        have_all[shift] = have
        if n_starts == 0:
            continue
        db, mag = frame_db(x, shift * 256, nfr)
        db[~have] = 0
        mag[~have] = 0
        Ue, De, Au, Ad = db @ Mu, db @ Md, mag @ Mu, mag @ Md
        sq = np.zeros(n_starts)
        sb = np.zeros(n_starts)
        bc = np.zeros(n_starts)
        for b in range(n_bits):
            u = np.zeros(n_starts); d = np.zeros(n_starts); au = np.zeros(n_starts); ad = np.zeros(n_starts)
            cnt = np.zeros(n_starts)
            for e in range(offsets[b], offsets[b + 1]):
                rows = s + fr[e]
                h = have[rows] if clip else np.ones(n_starts, bool)
                u += np.where(h, Ue[rows, e], 0); d += np.where(h, De[rows, e], 0)
                au += np.where(h, Au[rows, e], 0); ad += np.where(h, Ad[rows, e], 0)
                cnt += h
            with np.errstate(divide="ignore", invalid="ignore"):
                zero = (u == 0) | (d == 0)
                lt = u < d
                raw = np.where(zero, 0.0, np.where(lt, 1 - u / d, d / u - 1))
                grow = LAMBDA * np.sqrt(30 * cnt) * U
                du, dd = grow * au, grow * ad
                dr = np.where(zero, 0.0, np.where(lt, du / np.abs(d) + np.abs(u) * dd / d ** 2, dd / np.abs(u) + np.abs(d) * du / u ** 2))
            sq += (raw if b & 1 else -raw) * cnt
            sb += dr * cnt
            bc += cnt
        q[:, shift] = np.where(bc > 0, sq / np.maximum(bc, 1), sq) / norm
        qb[:, shift] = np.where(bc > 0, sb / np.maximum(bc, 1), sb) / norm
    idx = (s[:, None] * N + np.arange(4)[None, :] * 256).reshape(-1)
    q, qb = q.reshape(-1), qb.reshape(-1)
    lm, lmb = local_mean(q), local_mean(qb)
    return idx, q, lm, qb, lmb, have_all


def local_mean(q):
    m = len(q)
    acc = np.zeros(m)
    cnt = np.zeros(m)
    for j in range(-20, 21):
        if abs(j) >= 4:
            lo, hi = max(0, -j), min(m, m - j)
            if hi > lo:
                acc[lo:hi] += q[lo + j:hi + j]
                cnt[lo:hi] += 1
    return np.where(cnt > 0, acc / np.maximum(cnt, 1), acc)


# ------------------------------------------------------------------------------------------------ tables

def real_tables(key, mode):
    ent, off = T.sync_entries(key, O.CLIP if mode == capi.MODE_CLIP else O.BLOCK, P)
    return ent, off


def synthetic_tables(n_ent, n_bits, total, seed, sizes=None):
    """n_ent entries over n_bits bits of uneven size (or `sizes`), frames sorted inside a bit, including frame 0 and total - 1, bands
    0 and 80; 30 distinct up and 30 distinct down bands per entry"""
    rng = np.random.default_rng(seed)
    if sizes is None:
        w = rng.random(n_bits) + 0.2
        sizes = np.floor(w / w.sum() * n_ent).astype(int)
        sizes[0] += n_ent - sizes.sum()
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    ent = np.zeros(n_ent, capi.SYNC_ENTRY)
    frames = rng.integers(0, total, n_ent)
    frames[0] = 0
    frames[-1] = total - 1
    for b in range(n_bits):
        frames[off[b]:off[b + 1]] = np.sort(frames[off[b]:off[b + 1]])
    ent["frame"] = frames
    for e in range(n_ent):
        perm = rng.permutation(P.n_bands)
        ent["up"][e] = perm[:30]
        ent["down"][e] = perm[30:60]
    ent["up"][0][0], ent["down"][-1][0] = 0, 80
    return fix_distinct(ent), off


def fix_distinct(ent):
    """replace repeated bands of a list (from forcing bands 0 and 80 in) by unused ones"""
    for e in range(len(ent)):
        for key in ("up", "down"):
            row = ent[key][e]
            if len(set(row.tolist())) != 30:
                free = [b for b in range(P.n_bands) if b not in set(row.tolist())]
                seen = set()
                for i, b in enumerate(row):
                    if b in seen:
                        row[i] = free.pop()
                    seen.add(int(row[i]))
                ent[key][e] = row
    return ent


def set_syn_fpb(ctx, fpb, slot=SYN):
    mix = np.zeros(30, capi.MIX_ENTRY)
    mix["up"] = np.arange(30) + 20
    mix["down"] = np.arange(30) + 60
    ctx.set_mix_tables(slot, mix, np.zeros(1, np.uint16), 1, fpb)


# ------------------------------------------------------------------------------------------------ GPU comparison

@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    for k, key in enumerate(KEYS):
        T.setup_ctx(c, key, P, key_slot=k)
    yield c
    c.close()


def run_kernel(ctx, kernel, slot, mode, wav_first, wav_last, water_delta=0.01):
    old = os.environ.get("AWM_APPROX")
    try:
        if kernel == "default":
            os.environ.pop("AWM_APPROX", None)
        else:
            os.environ["AWM_APPROX"] = kernel
        got = ctx.sync_approx(slot, mode, wav_first, wav_last, water_delta)
    finally:
        if old is None:
            os.environ.pop("AWM_APPROX", None)
        else:
            os.environ["AWM_APPROX"] = old
    return got, ctx.sync_have()


def check_search(ctx, name, x, ent, off, slot, mode, total, bind, wav_first=0, wav_last=None, kernels=KERNELS):
    """every kernel against the float64 reference (count and indices exact, have exact, values within the bound) and the default
    kernel against simt within TIGHT times the bound"""
    n, C = x.shape
    if wav_last is None:
        wav_last = n * C
    clip = mode == capi.MODE_CLIP
    idx, q, lm, qb, lmb, have = search_ref(x, ent, off, total, wav_first, wav_last, clip=clip)
    out = {}
    for kernel in kernels:
        bind()
        got, ghave = run_kernel(ctx, kernel, slot, mode, wav_first, wav_last)
        assert len(got) == len(idx), (name, kernel, len(got), len(idx))
        assert np.array_equal(got["index"], idx.astype(np.uint64)), (name, kernel)
        if len(idx) == 0:                      # nothing searched, nothing analysed
            assert ghave.shape == (4, 0), (name, kernel)
        else:
            assert ghave.shape == have.shape and np.array_equal(ghave, have), (name, kernel, np.argwhere(ghave != have)[:8])
        if len(idx):
            eq = np.abs(got["raw_quality"] - q)
            em = np.abs(got["local_mean"] - lm)
            rq, rm = (eq / np.maximum(qb, 1e-300)).max(), (em / np.maximum(lmb, 1e-300)).max()
            RATIOS[kernel] = max(RATIOS.get(kernel, 0.0), rq, rm)
            bad = np.nonzero(eq > qb)[0]
            assert len(bad) == 0, (name, kernel, "raw_quality", bad[:5], eq[bad[:5]], qb[bad[:5]])
            bad = np.nonzero(em > lmb)[0]
            assert len(bad) == 0, (name, kernel, "local_mean", bad[:5], em[bad[:5]], lmb[bad[:5]])
        out[kernel] = got
    if "default" in out and "simt" in out and len(idx):
        a, b = out["default"], out["simt"]
        for f, bound in (("raw_quality", qb), ("local_mean", lmb)):
            e = np.abs(a[f] - b[f])
            RATIOS["default vs simt"] = max(RATIOS.get("default vs simt", 0.0), (e / np.maximum(TIGHT * bound, 1e-300)).max())
            bad = np.nonzero(e > TIGHT * bound)[0]
            assert len(bad) == 0, (name, f, bad[:5], e[bad[:5]], bound[bad[:5]])
    print("%-40s %6d scores  max err/bound %s" % (name, len(idx), {k: "%.3g" % v for k, v in RATIOS.items()}))
    return out


def host_bind(ctx, x):
    return lambda: ctx.pcm_bind(x)


def device_bind(ctx, x, byte_offset):
    """x as a device buffer starting byte_offset bytes past a 16-byte boundary"""
    torch = pytest.importorskip("torch")
    n, C = x.shape
    pad = byte_offset // 4
    buf = torch.zeros(n * C + pad + 4, dtype=torch.float32, device="cuda")
    view = buf[pad:pad + n * C]
    view.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(-1)))
    torch.cuda.synchronize()
    assert view.data_ptr() % 16 == byte_offset
    bind = lambda: ctx.pcm_bind(view.data_ptr(), n_frames=n, channels=C)
    bind.keep = buf
    return bind


def signal(n_frames, C, seed, amp=0.5):
    rng = np.random.default_rng(seed)
    return ((rng.random((n_frames, C), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ the reference itself

def test_reference_matches_oracle():
    """search_ref against O.SyncFinder.search_approx on the real tables, BLOCK and CLIP (with silence edges), to the 2e-4 of the
    existing parity tests -- this pins the reference, no GPU involved"""
    fpb = O.frames_per_block(P)
    for mode, total, C in ((O.BLOCK, fpb, 2), (O.CLIP, 2 * fpb, 1)):
        x = signal((total + 1 + 12) * N + 300, C, seed=3 + mode)
        sf = O.SyncFinder(P)
        sf.first, sf.last = (0, x.size) if mode == O.BLOCK else (5000 * C + 1, x.size - 7000 * C)
        want = sf.search_approx(O.get_sync_bits(O.Key(), mode, P), x, mode)
        ent, off = T.sync_entries(O.Key(), mode, P)
        idx, q, lm, qb, lmb, _ = search_ref(x, ent, off, total, sf.first, sf.last, clip=mode == O.CLIP)
        assert len(want) == len(idx) == 4 * 12
        assert np.array_equal(idx, [w.index for w in want])
        assert np.abs(q - [w.raw_quality for w in want]).max() < 2e-4
        assert np.abs(lm - [w.local_mean for w in want]).max() < 2e-4
        # the fp32 oracle is itself within the bound of the float64 reference
        assert (np.abs(q - [w.raw_quality for w in want]) <= qb).all()


# ------------------------------------------------------------------------------------------------ approximate search matrix

@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 1])
@pytest.mark.parametrize("mode", [capi.MODE_BLOCK, capi.MODE_CLIP])
def test_real_tables(ctx, k, mode):
    """the real tables of two keys (510 entries in BLOCK, 1020 in CLIP mode): stereo from the host, then mono at a 4-byte offset"""
    fpb = O.frames_per_block(P)
    total = fpb * (2 if mode == capi.MODE_CLIP else 1)
    ent, off = real_tables(KEYS[k], mode)
    x = signal((total + 1 + 40) * N + 777, 2, seed=10 + 2 * k + mode)
    check_search(ctx, "real key %d mode %d stereo" % (k, mode), x, ent, off, k, mode, total, host_bind(ctx, x))
    xm = np.ascontiguousarray(x[:, :1])
    check_search(ctx, "real key %d mode %d mono" % (k, mode), xm, ent, off, k, mode, total, device_bind(ctx, xm, 4))


FPB = 24
# (entries, bits, explicit bit sizes or None)
TABLES = [(1, 1, None), (47, 6, None), (48, 6, [8, 0, 20, 1, 9, 10]), (49, 2, None), (96, 6, None), (97, 5, None), (1024, 6, None),
          (1025, 6, None), (1, 6, [0, 0, 0, 0, 0, 1]), (200, 1, None)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [capi.MODE_BLOCK, capi.MODE_CLIP])
@pytest.mark.parametrize("table", range(len(TABLES)))
def test_synthetic_tables(ctx, table, mode):
    """synthetic tables of every entry count around the tensor-core kernel's 48-entry mask chunks, past the gather limit (1025 takes
    k_stft_db + k_sync_approx), 1 and 6 bits of uneven size, entries at frame 0 and total - 1 and bands 0 and 80"""
    n_ent, n_bits, sizes = TABLES[table]
    total = FPB * (2 if mode == capi.MODE_CLIP else 1)
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(n_ent, n_bits, total, seed=100 + table, sizes=sizes)
    ctx.set_sync_tables(SYN, mode, ent, off)
    C = (1, 2, 3)[table % 3]
    x = signal((total + 1 + 37 + table) * N + 1 + 511 * table, C, seed=200 + table + 50 * mode)
    check_search(ctx, "synthetic %d entries %d bits C=%d mode %d" % (n_ent, n_bits, C, mode), x, ent, off, SYN, mode, total, host_bind(ctx, x))


@pytest.mark.gpu
@pytest.mark.parametrize("C,placement", [(1, "host"), (2, "host"), (3, "host"), (4, "host"), (6, "host"),
                                         (2, "device+8"), (1, "device+4"), (3, "device+4")])
@pytest.mark.parametrize("n_out_mod", [0, 1, 127])
def test_channels_and_lengths(ctx, C, placement, n_out_mod):
    """1 to 6 channels, PCM from the host (stereo: bulk copies) or in place on the device (the load path); frame counts with
    n_out mod 128 = 0, 1, 127 (the last 128-frame tile full, one frame, one frame short) and sample counts off the frame grid"""
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(97, 6, FPB, seed=7)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    n_out = 128 + n_out_mod if n_out_mod else 256
    extra = {0: 1, 1: 1023, 127: 0}[n_out_mod]
    x = signal((n_out + 1) * N + extra, C, seed=C * 1000 + n_out_mod)
    bind = host_bind(ctx, x) if placement == "host" else device_bind(ctx, x, int(placement.split("+")[1]))
    check_search(ctx, "C=%d %s n_out=%d" % (C, placement, n_out), x, ent, off, SYN, capi.MODE_BLOCK, FPB, bind)


@pytest.mark.gpu
@pytest.mark.parametrize("n_starts", [0, 1, 2])
def test_few_start_frames(ctx, n_starts):
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(49, 6, FPB, seed=8)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    x = signal((FPB + 1 + n_starts) * N + 5, 2, seed=40 + n_starts)
    check_search(ctx, "n_starts=%d" % n_starts, x, ent, off, SYN, capi.MODE_BLOCK, FPB, host_bind(ctx, x))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3])
def test_clip_silence_edges(ctx, C):
    """CLIP mode: a frame ending exactly at wav_first is analysed, one ending a value before it is not; a frame starting exactly at
    wav_last is analysed, one starting a value after it is not.  wav_first / wav_last are off the channel grid in one of the two
    runs each.  Then the full range on the same PCM: every frame analysed again, the last one of every shift included."""
    total = 2 * FPB
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(96, 6, total, seed=9)
    ctx.set_sync_tables(SYN, capi.MODE_CLIP, ent, off)
    fc = total + 1 + 60
    x = signal(fc * N + 3, C, seed=60 + C)
    bind = host_bind(ctx, x)
    f_lo, f_hi = 9, fc - 14                   # frames (shift 1) at the two edges
    end_lo = (256 + f_lo * N + N) * C         # f_last of frame f_lo
    start_hi = (256 + f_hi * N) * C           # f_first of frame f_hi
    for wav_first, wav_last, kept in ((end_lo, start_hi - 1, (True, False)), (end_lo + 1, start_hi, (False, True))):
        out = check_search(ctx, "CLIP edges C=%d first %d last %d" % (C, wav_first, wav_last), x, ent, off, SYN, capi.MODE_CLIP, total,
                           bind, wav_first, wav_last)
        have = ctx.sync_have()
        assert (have[1][f_lo], have[1][f_hi]) == kept
        assert len(out["default"])
    check_search(ctx, "CLIP full range C=%d" % C, x, ent, off, SYN, capi.MODE_CLIP, total, bind)


@pytest.mark.gpu
def test_dynamic_range(ctx):
    """outside the |channel-summed dB| < 256 the fp16 hi/lo split is laid out for: six channels of full-scale tones over a faint
    noise floor (bins far from a tone near -100 dB per channel), quiet audio (1e-6) with a 1e-20 stretch, and a BLOCK-mode
    interior stretch of digital silence (power exactly zero: -96 per channel)"""
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(97, 6, FPB, seed=11)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    n = (FPB + 1 + 70) * N + 100
    t = np.arange(n) / 44100.0
    tones = np.stack([np.sin(2 * np.pi * (700 + 330 * c) * t + c) * (0.999 if c % 2 else 0.7) for c in range(6)], axis=1)
    loud = (tones + signal(n, 6, seed=12, amp=1e-4)).astype(np.float32)
    quiet = signal(n, 2, seed=13, amp=1e-6)
    quiet[30 * N:40 * N] *= np.float32(1e-14)
    silent = signal(n, 3, seed=14)
    silent[20 * N:50 * N] = 0
    for name, x in (("loud 6ch tones", loud), ("quiet 1e-6 / 1e-20", quiet), ("silent stretch", silent)):
        check_search(ctx, name, x, ent, off, SYN, capi.MODE_BLOCK, FPB, host_bind(ctx, x))
    print("max |error| / bound:", RATIOS)


# ------------------------------------------------------------------------------------------------ pipelined search

@pytest.mark.gpu
def test_enqueued_search_equals_direct(ctx):
    """awm_sync_approx_enqueue into slot 0 and slot 1, then awm_sync_use_slot: the peaks of each slot (floor -1: every local maximum)
    are bit-identical to those of awm_sync_approx on the same PCM"""
    fpb = O.frames_per_block(P)
    xs = [signal((fpb + 1 + 30) * N, 2, seed=70 + i) for i in range(2)]
    binds = [device_bind(ctx, x, 0) for x in xs]
    want = []
    for b in binds:
        b()
        ctx.sync_approx(0, capi.MODE_BLOCK)
        want.append(ctx.sync_peaks(-1.0))
    for slot, b in enumerate(binds):
        b()
        ctx.sync_approx_enqueue(slot, 0, capi.MODE_BLOCK)
    for slot in (1, 0):
        n = ctx.sync_use_slot(slot)
        assert n == 4 * 30
        got = ctx.sync_peaks(-1.0)
        assert got[1] == want[slot][1] and got[0].tobytes() == want[slot][0].tobytes(), slot
    ctx.sync_use_slot(0)


# ------------------------------------------------------------------------------------------------ peaks

def peaks_rule(scores, floor_q):
    """k_peaks: |q - mean| > floor, >= both neighbours, 0 beyond the ends"""
    a = np.abs(scores["raw_quality"] - scores["local_mean"])
    prev = np.concatenate([[0.0], a[:-1]])
    nxt = np.concatenate([a[1:], [0.0]])
    return scores[(a > floor_q) & (a >= prev) & (a >= nxt)]


@pytest.mark.gpu
def test_sync_peaks(ctx):
    """awm_sync_peaks against the rule of k_peaks applied to the GPU's own scores: floors -1, 0 and a typical threshold; more than
    2048 peaks (the second copy); max_peaks below the count; max_peaks = 0; digital silence, where every score is 0 and every score
    is a maximum with equal neighbours"""
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(96, 6, FPB, seed=15)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    x = signal((FPB + 1 + 2000) * N, 2, seed=16)
    ctx.pcm_bind(x)
    scores = ctx.sync_approx(SYN, capi.MODE_BLOCK)
    for floor_q in (-1.0, 0.0, P.sync_threshold2 * 0.75 * 0.15, P.sync_threshold2 * 0.75):
        want = peaks_rule(scores, floor_q)
        got, n = ctx.sync_peaks(floor_q)
        assert n == len(want) and got.tobytes() == want.tobytes(), (floor_q, n, len(want))
    want = peaks_rule(scores, -1.0)
    assert len(want) > 2048
    got, n = ctx.sync_peaks(-1.0, max_peaks=100)
    assert n == len(want) and len(got) == 100
    assert np.all(np.diff(got["index"].astype(np.int64)) > 0) and np.isin(got["index"], want["index"]).all()
    for g in got:
        w = want[np.searchsorted(want["index"], g["index"])]
        assert g.tobytes() == w.tobytes()
    got, n = ctx.sync_peaks(-1.0, max_peaks=0)
    assert n == len(want) and len(got) == 0
    z = np.zeros_like(x)
    ctx.pcm_bind(z)
    scores = ctx.sync_approx(SYN, capi.MODE_BLOCK)
    assert (scores["raw_quality"] == 0).all() and (scores["local_mean"] == 0).all()
    got, n = ctx.sync_peaks(-1.0, max_peaks=len(scores))
    assert n == len(scores) and got.tobytes() == scores.tobytes()
    assert ctx.sync_peaks(0.0)[1] == 0


# ------------------------------------------------------------------------------------------------ sync table checks

def bad_tables(ent, off):
    """tables awm_set_sync_tables must refuse: 7 bits, decreasing offsets, a repeated up band, a repeated down band, band 81"""
    out = []
    e7 = np.concatenate([ent, ent[:1]])
    out.append(("7 bits", e7, np.concatenate([off, [len(e7)]]).astype(np.int32)))
    o = off.copy()
    o[2], o[3] = o[3], o[2]
    out.append(("decreasing offsets", ent, o))
    for key in ("up", "down"):
        e = ent.copy()
        e[key][3][7] = e[key][3][2]
        out.append(("repeated %s band" % key, e, off))
    e = ent.copy()
    e["down"][0][0] = 81
    out.append(("band 81", e, off))
    return out


@pytest.mark.gpu
def test_rejected_tables_keep_previous(ctx):
    """a rejected table changes nothing: the slot searches with its previous table, bit for bit"""
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(96, 6, FPB, seed=17)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    x = signal((FPB + 1 + 50) * N, 2, seed=18)
    ctx.pcm_bind(x)
    before = ctx.sync_approx(SYN, capi.MODE_BLOCK)
    other, other_off = synthetic_tables(96, 6, FPB, seed=19)
    for name, e, o in bad_tables(other, other_off):
        with pytest.raises(capi.AwmError):
            ctx.set_sync_tables(SYN, capi.MODE_BLOCK, e, o)
        after = ctx.sync_approx(SYN, capi.MODE_BLOCK)
        assert after.tobytes() == before.tobytes(), name


@pytest.mark.gpu
def test_repeated_band_rejected(ctx):
    ent, off = synthetic_tables(48, 6, FPB, seed=20)
    ent["up"][5][29] = ent["up"][5][0]
    with pytest.raises(capi.AwmError, match="repeats a band"):
        ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)


@pytest.mark.gpu
def test_entry_frame_past_block_rejected_at_search(ctx):
    """an entry frame equal to the search length (frames_per_block, set later with the mix tables) fails the search; the same table
    passes in CLIP mode, whose search covers two blocks"""
    set_syn_fpb(ctx, FPB)
    ent, off = synthetic_tables(48, 6, FPB, seed=21)
    ent["frame"][-1] = FPB
    x = signal((FPB + 1 + 50) * N, 2, seed=22)
    ctx.pcm_bind(x)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    with pytest.raises(capi.AwmError, match="not inside"):
        ctx.sync_approx(SYN, capi.MODE_BLOCK)
    ctx.set_sync_tables(SYN, capi.MODE_CLIP, ent, off)
    assert len(ctx.sync_approx(SYN, capi.MODE_CLIP)) == 4 * (50 - FPB)
