"""The speed scan (awm_speed_scan: k_resample -> k_speed_mags -> k_speed_compare) against a float64 reference of the same operation
written here in plain numpy, at the shapes where the kernels take their edge paths.

The reference starts from the half-rate clip of O.resample_ratio_truncate (the resampler is bit exact against the oracle, see
test_gpu_speed.py) and follows SpeedSync::prepare_mags + compare: the 512-point window of O.gen_normalized_window, np.fft.rfft per
channel in float64, band dB (-96 where the power is exactly zero) summed over channels, up / down sums per entry (`mags_ref`); then
the 16.16 offsets of compare in exact integer arithmetic from the same truncated doubles, per-bit sums, bit quality, normalisation by
min(water_delta, 0.08) * 2.9, fabs, maximum over the pad_start offsets (`compare_ref`).  test_reference_matches_oracle pins both to
O.speed_prepare_mags / O.speed_compare on the real tables of two keys, without a GPU.

Three checks per case:
  * rows exact, every MagMatrix value within its bound;
  * the compare bit exact: `compare_f32` emulates k_speed_compare (float32 sums per bit in entry order, double accumulation of the
    bit qualities) on the GPU's own MagMatrix (awm_speed_mags) and must reproduce every quality bit for bit; on real tables it
    also equals O.speed_compare on that matrix.  This holds the compare kernel exactly, independent of the FFT's error;
  * end to end: each quality within the largest over the offsets of the propagated bound.

Error bound of a MagMatrix value.  k_speed_mags transforms two consecutive rows and two channels with one 1024-point fp32 FFT, so
the error of a bin scales with the norm of that whole packed input z (both rows, both channels, windowed).  Every dB term i
(one band of one channel) carries a magnitude
    m_i = |dB| + (20 / ln 10) ETA log2(1024) ||z|| / |X_k| + (10 / ln 10) 2^-149 / (|X_k|^2 u)
the dB value itself, its condition with respect to the packed fp32 FFT (ETA = 4 sqrt(2) + 1: the error of one radix-2 stage in units
of u, Higham, Accuracy and Stability of Numerical Algorithms, 24.1; log2(1024) stages), and the spacing of fp32 denormals at the
bin's power, in units of u = 2^-24.  The FFT term is a typical size, not a worst case: it spreads the FFT's 2-norm error bound
evenly over the 1024 bins, where a single bin could in the worst case carry sqrt(1024) times more.  A value sums n = 30 C such
terms (30 bands, C channels), and the whole is scaled like recursive fp32 summation in the probabilistic model of Higham and Mary
(2019), so the bound below is a probabilistic (LAMBDA standard deviations) bound, not a rigorous one:
    dU <= LAMBDA sqrt(30 C) u sum_i m_i + sum_i f_i,        LAMBDA = 3,
where f_i = |dB + 96| for a power below 2^-146, which fp32 may round to exactly zero (then the -96 floor applies), else 0.
Error bound of a quality.  A bit sums cnt MagMatrix values in fp32: du <= sum dU + LAMBDA sqrt(cnt) u sum |U|; the bit quality
1 - u/d has dr <= du / |d| + |u| dd / d^2 + 2u (d/u - 1 symmetrically), and
    dq <= sum_bits cnt_b dr_b / sum_bits cnt_b / (min(water_delta, 0.08) 2.9)
per offset; the scan keeps the largest |q| over the offsets, so its error is at most the largest dq over the offsets.
Largest observed |error| / bound on an H100 (NVIDIA H100 80GB HBM3, 700 W power limit): MagMatrix 0.77 (1e-20 audio, where fp32
powers fall into denormals), 0.013 for every other case; qualities 0.012.  The tests print the running maxima with -s.
"""
import math

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi
from audiowmark_b200 import hostapi as H
from test_gpu_sync_search import KEYS, SYN, ctx, set_syn_fpb, synthetic_tables  # noqa: F401  (ctx: the fixture, two keys set up)

P = O.Params()
U = 2.0 ** -24
LAMBDA = 3.0
ETA = 4 * math.sqrt(2) + 1               # error of one radix-2 FFT stage in units of u (Higham, Accuracy and Stability, 24.1)
SUB_FRAME, SUB_HOP = 512, 128
RATIOS = {}


# ------------------------------------------------------------------------------------------------ float64 reference

def n_rows(n_sub):
    return (n_sub - SUB_FRAME + SUB_HOP - 1) // SUB_HOP if n_sub > SUB_FRAME else 0


def sub_clip(clip, rate, center, seconds):
    return O.resample_ratio_truncate(np.ascontiguousarray(clip, np.float32), rate, center / 2, seconds / center)


def band_matrix(bands, n_ent):
    """[81][n_ent] count of each band in each entry's list"""
    M = np.zeros((P.n_bands, n_ent))
    np.add.at(M, (np.asarray(bands).reshape(n_ent, -1), np.arange(n_ent)[:, None]), 1.0)
    return M


def mags_ref(sub, ent):
    """float64 prepare_mags on the half-rate clip: (U [n_ent][rows], D, bound of U, bound of D) in table order"""
    sub = np.asarray(sub, np.float32)
    n_sub, C = sub.shape
    rows = n_rows(n_sub)
    n_ent = len(ent)
    if rows == 0:
        z = np.zeros((n_ent, 0))
        return z, z, z, z
    win = O.gen_normalized_window(SUB_FRAME).astype(np.float64)
    idx = np.arange(rows)[:, None] * SUB_HOP + np.arange(SUB_FRAME)[None, :]
    xw = sub[idx].astype(np.float64) * win[None, :, None]                  # [rows][512][C]
    e2 = (xw * xw).sum(axis=1)                                              # [rows][C] energy of each windowed row
    # packed input of k_speed_mags: rows 2j and 2j + 1 (a missing partner row is zero), channels 2i and 2i + 1
    partner = np.arange(rows) ^ 1
    pr = e2 + np.where((partner < rows)[:, None], e2[np.minimum(partner, rows - 1)], 0.0)     # [rows][C] energy of both rows
    db = np.zeros((rows, P.n_bands))
    mag = np.zeros((rows, P.n_bands))
    under = np.zeros((rows, P.n_bands))
    for ch in range(C):
        lo = ch - ch % 2
        nz = np.sqrt(pr[:, lo:lo + 2].sum(axis=1))[:, None]
        X = np.fft.rfft(xw[:, :, ch], axis=1)[:, P.min_band:P.max_band + 1]
        pw = X.real ** 2 + X.imag ** 2
        pos = pw > 0
        safe = np.where(pos, pw, 1.0)
        d = np.where(pos, 10 * np.log10(safe), -96.0)
        cond = np.where(pos, (20 / np.log(10)) * ETA * 10 * nz / np.sqrt(safe) + (10 / np.log(10)) * 2.0 ** -149 / (safe * U), 0.0)
        db += d
        mag += np.abs(d) + cond
        under += np.where(pw < 2.0 ** -146, np.abs(d + 96.0), 0.0)     # fp32 may round this power to 0, where -96 applies
    Mu, Md = band_matrix(ent["up"], n_ent), band_matrix(ent["down"], n_ent)
    grow = LAMBDA * math.sqrt(30 * C) * U
    return (db @ Mu).T, (db @ Md).T, (grow * (mag @ Mu) + under @ Mu).T, (grow * (mag @ Md) + under @ Md).T


def offsets(rs, fpb, frames):
    """the 16.16 start offsets [pad_start] and frame offsets [3][n_ent] of compare as exact integers: the reference's truncated doubles"""
    pad_start = fpb * 4 + 4
    off = np.trunc((np.arange(pad_start) - pad_start).astype(np.float64) * (65536.0 / rs)).astype(np.int64)
    inv = 1 / rs
    v = ((np.arange(3)[:, None] * fpb + np.asarray(frames, np.int64)[None, :]) * 4).astype(np.float64)
    fo = np.trunc((v * inv + 0.5) * 65536.0).astype(np.int64)
    return off, fo


def window(off, fo, rows):
    """one block and entry: (valid [pad_start] mask, row index [pad_start]) -- the iterator window of compare_bits"""
    s = off + fo
    valid = (s >= 0) & ((s >> 16) < rows)
    return valid, np.where(valid, s >> 16, 0)


def compare_ref(Um, Dm, BU, BD, ent, off_bits, fpb, rs, water_delta):
    """float64 compare for one relative speed on a float64 MagMatrix with its bound: (quality, bound of the quality)"""
    rows = Um.shape[1]
    off, fo = offsets(rs, fpb, ent["frame"])
    pad_start = len(off)
    sq = np.zeros(pad_start)
    sb = np.zeros(pad_start)
    bc = np.zeros(pad_start)
    for b in range(len(off_bits) - 1):
        u = np.zeros(pad_start); d = np.zeros(pad_start); au = np.zeros(pad_start); ad = np.zeros(pad_start); aa = np.zeros(pad_start)
        cnt = np.zeros(pad_start)
        for B in range(3):
            for e in range(off_bits[b], off_bits[b + 1]):
                h, i = window(off, fo[B, e], rows)
                if not h.any():
                    continue
                uu, dd = (Dm, Um) if B & 1 else (Um, Dm)
                bu, bd = (BD, BU) if B & 1 else (BU, BD)
                u += np.where(h, uu[e, i], 0); d += np.where(h, dd[e, i], 0)
                au += np.where(h, bu[e, i], 0); ad += np.where(h, bd[e, i], 0)
                aa += np.where(h, np.abs(uu[e, i]) + np.abs(dd[e, i]), 0)
                cnt += h
        with np.errstate(divide="ignore", invalid="ignore"):
            g = LAMBDA * np.sqrt(cnt) * U * aa
            du, dd = au + g, ad + g
            zero = (u == 0) | (d == 0)
            lt = u < d
            raw = np.where(zero, 0.0, np.where(lt, 1 - u / d, d / u - 1))
            dr = np.where(zero, 0.0, np.where(lt, du / np.abs(d) + np.abs(u) * dd / d ** 2, dd / np.abs(u) + np.abs(d) * du / u ** 2) + 2 * U)
        sq += (raw if b & 1 else -raw) * cnt
        sb += dr * cnt
        bc += cnt
    norm = min(water_delta, 0.08) * 2.9
    has = bc > 0
    q = np.where(has, np.abs(sq / np.maximum(bc, 1) / norm), 0.0)
    qb = np.where(has, sb / np.maximum(bc, 1) / norm, 0.0)
    return q.max(), qb.max()


def compare_f32(M, ent, off_bits, fpb, rs, water_delta):
    """k_speed_compare's arithmetic on a float32 MagMatrix [n_ent][rows][2] (table order): float32 sums per bit over blocks 0..2 and
    the bit's entries in table order, bit qualities in float32, accumulated in double; max |quality| over the offsets"""
    rows = M.shape[1]
    off, fo = offsets(rs, fpb, ent["frame"])
    pad_start = len(off)
    sq = np.zeros(pad_start)
    bc = np.zeros(pad_start, np.int64)
    one = np.float32(1)
    for b in range(len(off_bits) - 1):
        um = np.zeros(pad_start, np.float32)
        dm = np.zeros(pad_start, np.float32)
        cnt = np.zeros(pad_start, np.int64)
        for B in range(3):
            for e in range(off_bits[b], off_bits[b + 1]):
                h, i = window(off, fo[B, e], rows)
                if not h.any():
                    continue
                m = M[e, i]
                x, y = (m[:, 1], m[:, 0]) if B & 1 else (m[:, 0], m[:, 1])
                um = np.where(h, um + x, um)
                dm = np.where(h, dm + y, dm)
                cnt += h
        with np.errstate(divide="ignore", invalid="ignore"):
            raw = np.where((um == 0) | (dm == 0), np.float32(0),
                           np.where(um < dm, one - um / dm, dm / um - one)).astype(np.float64)
        sq = sq + (raw if b & 1 else -raw) * cnt
        bc += cnt
    norm_div = water_delta if water_delta < 0.080 else 0.080
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(bc > 0, np.abs(sq / bc / norm_div / 2.9), 0.0)
    return q.max()


# ------------------------------------------------------------------------------------------------ tables and signals

def oracle_entries(ent, off):
    """table-order entries -> the oracle's (frame, bit, up, down), sorted by frame, and the permutation that sorts them"""
    bit = np.zeros(len(ent), np.int32)
    for b in range(len(off) - 1):
        bit[off[b]:off[b + 1]] = b
    order = np.argsort(ent["frame"], kind="stable")
    return ((np.ascontiguousarray(ent["frame"][order], np.int32), np.ascontiguousarray(bit[order]),
             np.ascontiguousarray(ent["up"][order], np.int32), np.ascontiguousarray(ent["down"][order], np.int32)), order)


def signal(n_frames, C, seed, amp=0.5):
    rng = np.random.default_rng(seed)
    return ((rng.random((n_frames, C), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


def shaped(kind, n, C, seed, rate=44100):
    """test signals: noise, 1e-6 / 1e-20 audio, digital silence, loud tones, one channel at 1e-6 of the other, a level that jumps
    from one row to the next"""
    if kind == "noise":
        return signal(n, C, seed)
    if kind == "quiet":
        x = signal(n, C, seed, amp=1e-6)
        x[n // 3:2 * n // 3] *= np.float32(1e-14)            # a stretch at 1e-20
        return x
    if kind == "silence":
        return np.zeros((n, C), np.float32)
    if kind == "tones":
        t = np.arange(n) / float(rate)
        tones = np.stack([np.sin(2 * np.pi * (700 + 330 * c) * t + c) * (0.999 if c % 2 else 0.7) for c in range(C)], axis=1)
        return (tones + signal(n, C, seed, amp=1e-4)).astype(np.float32)
    if kind == "faint_channel":
        x = signal(n, C, seed)
        x[:, 1] *= np.float32(1e-6)
        return x
    if kind == "steps":
        x = signal(n, C, seed)
        lvl = np.where((np.arange(n) // 256) % 2 == 0, 1.0, 1e-5).astype(np.float32)    # 128 half-rate frames: one row hop
        return (x * lvl[:, None]).astype(np.float32)
    raise ValueError(kind)


def device_clip(x, byte_offset):
    """x as a device buffer starting byte_offset bytes past a 16-byte boundary: (pointer, keep-alive)"""
    torch = pytest.importorskip("torch")
    n, C = x.shape
    pad = byte_offset // 4
    buf = torch.zeros(n * C + pad + 4, dtype=torch.float32, device="cuda")
    view = buf[pad:pad + n * C]
    view.copy_(torch.from_numpy(np.ascontiguousarray(x).reshape(-1)))
    torch.cuda.synchronize()
    assert view.data_ptr() % 16 == byte_offset
    return view.data_ptr(), buf


# ------------------------------------------------------------------------------------------------ the reference itself

def test_reference_matches_oracle():
    """mags_ref / compare_ref against O.speed_prepare_mags / O.speed_compare on the real tables of two keys (stereo and mono, two
    centres): the oracle's fp32 MagMatrix lies inside the reference's bound, the fp32 qualities inside the propagated bound, and
    compare_f32 on the oracle's own matrix equals O.speed_compare bit for bit -- no GPU involved"""
    fpb = O.frames_per_block(P)
    for k, key in enumerate(KEYS):
        ent, off = T.sync_entries(key, O.BLOCK, P)
        oent, order = oracle_entries(ent, off)
        C = 2 - k
        clip = signal(int(12 * 44100), C, seed=30 + k)
        rel = [1.0007 ** p for p in (-5, 0, 5)] + [0.5, 2.0]
        for center in (1.0007 ** -308, 1.0):
            sub = sub_clip(clip, 44100, center, 10.0)
            Um, Dm, BU, BD = mags_ref(sub, ent)
            om = O.speed_prepare_mags(clip, 44100, center, 10.0, oent)          # [n_ent][rows][2] in frame order
            tm = np.empty_like(om)
            tm[order] = om                                                      # back to table order
            assert tm.shape[1] == Um.shape[1] == n_rows(sub.shape[0]) > 0
            assert (np.abs(tm[:, :, 0] - Um) <= BU).all() and (np.abs(tm[:, :, 1] - Dm) <= BD).all()
            want = O.speed_compare(om, oent, rel, P)
            for r, rs in enumerate(rel):
                assert compare_f32(tm, ent, off, fpb, rs, P.water_delta) == want[r], (k, center, rs)
                q, qb = compare_ref(Um, Dm, BU, BD, ent, off, fpb, rs, P.water_delta)
                assert abs(q - want[r]) <= qb, (k, center, rs, q, want[r], qb)


# ------------------------------------------------------------------------------------------------ GPU comparison

def check_scan(ctx, name, clip, rate, seconds, centers, rel, slot, ent, off, fpb, water_delta=0.01, oracle_P=None, clip_arg=None):
    """scan `clip` (or the device pointer clip_arg holding it) and hold every centre's MagMatrix and every quality to the reference;
    returns the qualities"""
    n, C = clip.shape
    rel = np.asarray(rel, np.float64).reshape(len(centers), -1)
    arg = clip if clip_arg is None else clip_arg
    got = ctx.speed_scan(arg, seconds, centers, rel, key_slot=slot, sample_rate=rate, water_delta=water_delta, n_frames=n, channels=C)
    oent, order = oracle_entries(ent, off) if oracle_P is not None else (None, None)
    for ci, c in enumerate(centers):
        sub = sub_clip(clip, rate, c, seconds)
        rows = n_rows(sub.shape[0])
        M = ctx.speed_mags(ci)
        assert M.shape == (len(ent), rows, 2), (name, c, M.shape, rows)
        if rows == 0:
            assert (got[ci] == 0).all(), (name, c)
            continue
        Um, Dm, BU, BD = mags_ref(sub, ent)
        eu, ed = np.abs(M[:, :, 0] - Um), np.abs(M[:, :, 1] - Dm)
        RATIOS["mags"] = max(RATIOS.get("mags", 0.0), (eu / np.maximum(BU, 1e-300)).max(), (ed / np.maximum(BD, 1e-300)).max())
        bad = np.argwhere((eu > BU) | (ed > BD))
        assert len(bad) == 0, (name, c, bad[:5], eu[tuple(bad[0])], BU[tuple(bad[0])])
        for r, rs in enumerate(rel[ci]):
            want = compare_f32(M, ent, off, fpb, rs, water_delta)
            assert got[ci, r] == want, (name, c, rs, got[ci, r], want)
            q, qb = compare_ref(Um, Dm, BU, BD, ent, off, fpb, rs, water_delta)
            e = abs(got[ci, r] - q)
            RATIOS["scores"] = max(RATIOS.get("scores", 0.0), e / max(qb, 1e-300))
            assert e <= qb, (name, c, rs, got[ci, r], q, qb)
        if oracle_P is not None:
            want = O.speed_compare(np.ascontiguousarray(M[order]), oent, rel[ci], oracle_P)
            assert np.array_equal(got[ci], want), (name, c, got[ci], want)
    print("%-44s max err/bound %s" % (name, {k: "%.3g" % v for k, v in RATIOS.items()}))
    return got


REL_TEST = [1.0007 ** -5, 1.0, 1.0007 ** 5, 0.5, 2.0]        # scan 1's ends and two far enough out to drop whole blocks
FPB = 24


def syn_setup(ctx, n_ent, n_bits, fpb, seed, sizes=None):
    set_syn_fpb(ctx, fpb)
    ent, off = synthetic_tables(n_ent, n_bits, fpb, seed=seed, sizes=sizes)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    return ent, off


def syn_clip_frames(rows, center=1.0, rate=44100):
    """clip frames whose half-rate clip at `center` has about `rows` rows"""
    return int((SUB_FRAME + SUB_HOP * rows) / (center / 2) * rate / 44100)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 6])
def test_channels(ctx, C):
    """1 to 6 channels (odd counts take the lone-channel half of the packed FFT and k_resample<0>); three centres in one call, two of
    them truncated to seconds / centre and one limited by the clip's end, so that they have different row counts; stereo with one
    channel at 1e-6 of the other; mono whose level jumps every row"""
    ent, off = syn_setup(ctx, 97, 6, FPB, seed=300 + C)
    kind = {1: "steps", 2: "faint_channel"}.get(C, "noise")
    x = shaped(kind, syn_clip_frames(420), C, seed=310 + C)
    centers = [1.0, 0.9, 1.0007 ** 308]
    seconds = x.shape[0] / 44100 * 0.95                  # centre 0.9 would keep 1.06 times the clip: it keeps all of it
    assert len({n_rows(sub_clip(x, 44100, c, seconds).shape[0]) for c in centers}) == 2
    check_scan(ctx, "C=%d %s" % (C, kind), x, 44100, seconds, centers, [REL_TEST] * 3, SYN, ent, off, FPB)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", [0, 1, 15, 16, 17, 31, 33])
def test_row_counts(ctx, rows):
    """0 rows (n_sub <= 512: all qualities 0), 1 row, around the 16-row CTA of k_speed_mags; centre 2 resamples 1:1, so the row count
    is exact, seconds <= 0 keeps the whole clip; a second centre in the same call has about half the rows"""
    ent, off = syn_setup(ctx, 49, 6, 6, seed=320)
    n = SUB_FRAME + SUB_HOP * (rows - 1) + 1 if rows else SUB_FRAME
    x = signal(n, 2 if rows % 2 else 1, seed=330 + rows)
    assert n_rows(n) == rows
    got = check_scan(ctx, "rows=%d" % rows, x, 44100, 0.0, [2.0, 1.0], [REL_TEST] * 2, SYN, ent, off, 6)
    if rows == 0:
        assert (got == 0).all()


SCANS = {  # name: (seconds, centre step, n_steps, centre steps) of SpeedScanParams, normal and patient
    "scan1": (25, 1.0007, 5, 28), "scan1-patient": (50, 1.00035, 11, 28),
    "scan2": (50, 1.00035, 1, 0), "scan2-patient": (50, 1.000175, 1, 0),
    "scan3": (50, 1.00005, 40, 0), "scan3-patient": (50, 1.00005, 40, 0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("scan,rate", [("scan1", 44100), ("scan1-patient", 48000), ("scan2", 32000), ("scan2-patient", 44100),
                                       ("scan3", 48000), ("scan3-patient", 32000)])
def test_real_scans(ctx, scan, rate):
    """the real tables of two keys at the ends of scans 1, 2 and 3 (normal and patient), full length (25 or 50 s) scans of a clip of
    1.3 times that, at 32, 44.1 and 48 kHz; qualities also equal O.speed_compare on the GPU's own matrix"""
    seconds, step, n_steps, n_center = SCANS[scan]
    k = len(scan) % 2
    ent, off = T.sync_entries(KEYS[k], O.BLOCK, P)
    speed = 1.0 if scan.startswith("scan1") else 1.01
    centers = [speed * step ** (c * (2 * n_steps + 1)) for c in ((-n_center, n_center) if n_center else (0,))]
    rel = [[step ** -n_steps, step ** n_steps]] * len(centers)
    x = signal(int(seconds * 1.3 * rate), 2, seed=500 + list(SCANS).index(scan))
    check_scan(ctx, "%s %d Hz key %d" % (scan, rate, k), x, rate, seconds, centers, rel, k, ent, off, O.frames_per_block(P), oracle_P=P)


BLOCK_PARAMS = {"short12": dict(payload_size=12, payload_short=True), "short16": dict(payload_size=16, payload_short=True),
                "short20": dict(payload_size=20, payload_short=True), "fpb1": dict(frames_per_bit=1), "fpb3": dict(frames_per_bit=3)}


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(BLOCK_PARAMS))
def test_block_lengths(ctx, params):
    """real tables at other block lengths (--short 12/16/20, --frames-per-bit 1 and 3), which move pad_start and the compare grid;
    --frames-per-bit 3 with the CLI's 50 s scan (its third block reaches 16.16 offsets past 2^30): equal to the oracle"""
    Pv = O.Params(**BLOCK_PARAMS[params])
    slot = 2
    ent, off = T.sync_entries(KEYS[0], O.BLOCK, Pv)
    ctx.set_sync_tables(slot, capi.MODE_BLOCK, ent, off)
    set_syn_fpb(ctx, O.frames_per_block(Pv), slot=slot)            # the scan reads frames_per_block of the mix tables only
    seconds = 50.0 if params == "fpb3" else 25.0
    x = signal(int(seconds * 1.3 * 44100), 1 + (params == "fpb1"), seed=340 + len(params))
    centers = [1.0007 ** -308, 1.0]
    check_scan(ctx, params, x, 44100, seconds, centers, [[1.0007 ** -5, 1.0, 1.0007 ** 5]] * 2, slot, ent, off, O.frames_per_block(Pv),
               oracle_P=Pv)


TABLES = {  # name: (entries, bits, explicit bit sizes or None, frames per block)
    "1 entry 1 bit": (1, 1, None, FPB), "6 uneven bits": (60, 6, [1, 20, 3, 15, 9, 12], FPB),
    "1024 entries pad 512": (1024, 6, None, 127), "97 entries pad 256": (97, 5, None, 63),
}


@pytest.mark.gpu
@pytest.mark.parametrize("table", list(TABLES))
@pytest.mark.parametrize("water_delta", [0.01, 0.1])
def test_synthetic_tables(ctx, table, water_delta):
    """synthetic tables: 1 entry of 1 bit, 6 bits of uneven size, exactly 1024 entries, entries at frames 0 and fpb - 1 and bands 0
    and 80; fpb 63 and 127, where pad_start is exactly 256 and 512; water_delta below and above the 0.08 cap"""
    n_ent, n_bits, sizes, fpb = TABLES[table]
    ent, off = syn_setup(ctx, n_ent, n_bits, fpb, seed=350 + n_ent, sizes=sizes)
    assert ent["frame"].max() == fpb - 1 and (n_ent == 1 or ent["frame"].min() == 0)
    x = signal(syn_clip_frames(4 * fpb * 3 + 40), 2, seed=360 + n_ent)
    check_scan(ctx, "%s wd %g" % (table, water_delta), x, 44100, 0.0, [1.0, 1.0007 ** -308], [REL_TEST] * 2, SYN, ent, off, fpb,
               water_delta=water_delta)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,C", [("silence", 2), ("quiet", 2), ("tones", 6), ("quiet", 1)])
def test_dynamic_range(ctx, kind, C):
    """digital silence (every power exactly zero: -96 dB), 1e-6 audio with a 1e-20 stretch, loud six-channel tones"""
    ent, off = syn_setup(ctx, 97, 6, FPB, seed=370)
    x = shaped(kind, syn_clip_frames(400), C, seed=380 + C)
    got = check_scan(ctx, "%s C=%d" % (kind, C), x, 44100, 0.0, [1.0], [REL_TEST], SYN, ent, off, FPB)
    if kind == "silence":
        assert (got == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 2, 3])
@pytest.mark.parametrize("byte_offset", [0, 4])
def test_device_clips(ctx, C, byte_offset):
    """a clip in device memory, taken 37 frames into a buffer that starts byte_offset bytes past a 16-byte boundary (stereo at 4 bytes:
    the float2 path of k_resample is not allowed there): MagMatrix and qualities bit-identical to the same clip from the host"""
    ent, off = syn_setup(ctx, 97, 6, FPB, seed=390)
    full = signal(syn_clip_frames(300) + 37, C, seed=400 + C)
    x = np.ascontiguousarray(full[37:])
    centers, rel = [1.0, 0.95], [REL_TEST] * 2
    want = check_scan(ctx, "host C=%d" % C, x, 44100, 0.0, centers, rel, SYN, ent, off, FPB)
    want_m = [ctx.speed_mags(i) for i in range(2)]
    ptr, keep = device_clip(full, byte_offset)
    p = ptr + 37 * C * 4
    got = ctx.speed_scan(p, 0.0, centers, rel, key_slot=SYN, n_frames=x.shape[0], channels=C)
    assert got.tobytes() == want.tobytes(), (C, byte_offset, got, want)
    for i in range(2):
        assert ctx.speed_mags(i).tobytes() == want_m[i].tobytes()
    del keep


@pytest.mark.gpu
@pytest.mark.parametrize("byte_offset", [4, 8])
def test_resample_unaligned_stereo(ctx, byte_offset):
    """awm_resample on a stereo device buffer 4 bytes past an 8-byte boundary (k_resample<0>) and on an aligned one (k_resample<2>):
    bit-identical to the host input, which the oracle pins"""
    x = signal(50001, 2, seed=410)
    want = ctx.resample(x, 44100 / 48000.0)
    assert np.array_equal(want.view(np.uint32), O.resample_ratio(x, 44100 / 48000.0).view(np.uint32))
    ptr, keep = device_clip(x, byte_offset)
    got = ctx.resample(ptr, 44100 / 48000.0, n_frames=x.shape[0], channels=2)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    del keep


# ------------------------------------------------------------------------------------------------ resampler table cache

@pytest.mark.gpu
def test_cache_eviction_inside_a_scan(ctx):
    """with the resampler table cache two tables short of its cap and 2 of a scan's 5 centres in it, the scan (3 new centres) empties
    it first and then fetches all 5 tables: qualities and MagMatrices bit-identical to the same scan on a fresh context, and the cache
    holds just those 5.  Then a scan of 1025 distinct centres, 5 of them cached (1020 new ones would fit an emptied cache, but the
    call needs all 1025 tables at once), is refused; one of exactly 1024 distinct centres runs and keeps the first 5 qualities"""
    ent, off = syn_setup(ctx, 97, 6, FPB, seed=420)
    x = signal(syn_clip_frames(300), 2, seed=421)
    centers = [1.0007 ** (11 * c) + 1e-7 for c in (-2, -1, 0, 1, 2)]      # ratios nobody asked for before
    ctx.speed_scan(x, 0.0, centers[:2], [REL_TEST] * 2, key_slot=SYN)
    size, cap = ctx.resampler_cache()
    one = np.zeros((1, 1), np.float32)
    k = 0
    while size < cap - 2:
        ctx.resample(one, 1.5 + 1e-4 * k, n_out=1)
        k += 1
        size, _ = ctx.resampler_cache()
    assert size == cap - 2
    got = ctx.speed_scan(x, 0.0, centers, [REL_TEST] * 5, key_slot=SYN)
    got_m = [ctx.speed_mags(i) for i in range(5)]
    assert ctx.resampler_cache() == (5, cap)
    fresh = capi.Context(0)
    try:
        set_syn_fpb(fresh, FPB)
        fresh.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
        want = fresh.speed_scan(x, 0.0, centers, [REL_TEST] * 5, key_slot=SYN)
        assert got.tobytes() == want.tobytes()
        for i in range(5):
            assert got_m[i].tobytes() == fresh.speed_mags(i).tobytes()
    finally:
        fresh.close()
    more = centers + [0.5 + 1e-4 * i for i in range(cap + 1 - 5)]
    with pytest.raises(capi.AwmError, match="1025 distinct centres exceed the resampler table cache"):
        ctx.speed_scan(x, 0.0, more, np.tile(REL_TEST[:1], (len(more), 1)), key_slot=SYN)
    assert ctx.resampler_cache() == (5, cap)
    more = more[:cap] + more[:3]                                            # repeats count once
    q = ctx.speed_scan(x, 0.0, more, np.tile(REL_TEST, (len(more), 1)), key_slot=SYN)
    assert ctx.resampler_cache() == (cap, cap)
    assert q[:5].tobytes() == got.tobytes() and q[-3:].tobytes() == got[:3].tobytes()


# ------------------------------------------------------------------------------------------------ argument checks and 16.16 limits

@pytest.mark.gpu
def test_refusals(ctx):
    """relative speeds that are not finite and > 0, more than 65535 jobs, and 1025 entries are refused with a message"""
    ent, off = syn_setup(ctx, 97, 6, FPB, seed=430)
    x = signal(syn_clip_frames(100), 1, seed=431)
    for bad in (0.0, -1.0, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(capi.AwmError, match="not finite and > 0"):
            ctx.speed_scan(x, 0.0, [1.0, 1.0], [[1.0, 1.0], [1.0, bad]], key_slot=SYN)
    with pytest.raises(capi.AwmError, match="exceed the limit 65535"):
        ctx.speed_scan(x, 0.0, [1.0, 1.0], np.ones((2, 32768)), key_slot=SYN)
    assert ctx.speed_scan(x, 0.0, [1.0], np.ones((1, 65535)) * 1.01, key_slot=SYN).shape == (1, 65535)
    ent, off = synthetic_tables(1025, 6, FPB, seed=432)
    ctx.set_sync_tables(SYN, capi.MODE_BLOCK, ent, off)
    with pytest.raises(capi.AwmError, match="exceed the kernel limit 1024"):
        ctx.speed_scan(x, 0.0, [1.0], [[1.0]], key_slot=SYN)


@pytest.mark.gpu
def test_offsets_past_31_bits(ctx):
    """seconds = 150 of a 160 s clip (25800 rows): at --frames-per-bit 3 (3084-frame blocks) entries of the third block that can still
    land in the matrix need 16.16 offsets above 2^31, and the scan is refused; with the default blocks the offsets fit although rows
    and start offsets reach past 2^31 together, and the scan equals the exact-integer emulation and the oracle bit for bit"""
    x = signal(160 * 44100, 1, seed=440)
    P3 = O.Params(frames_per_bit=3)
    assert O.frames_per_block(P3) == 3084
    T.setup_ctx(ctx, KEYS[0], P3, key_slot=3)
    with pytest.raises(capi.AwmError, match="more than 31 bits"):
        ctx.speed_scan(x, 150.0, [1.0], [[1.0]], key_slot=3)
    ent, off = T.sync_entries(KEYS[0], O.BLOCK, P)
    rel = [1.00005 ** -40, 1.0, 1.00005 ** 40]
    check_scan(ctx, "150 s of 160 s", x, 44100, 150.0, [1.0], [rel], 0, ent, off, O.frames_per_block(P), oracle_P=P)
    assert ctx.speed_mags(0).shape[1] > 25000


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 6])
def test_detect_speed_device_buffer(C):
    """detect_speed on mono, 3 and 6 channels: a device buffer gives the same speed and quality as the host buffer (the clip location
    is hashed from a sparse sample subset that awm_gather fetches from the device)"""
    torch = pytest.importorskip("torch")
    y = T.speed_changed(30, 1.01)
    x = np.ascontiguousarray(np.concatenate([y, 0.5 * y, -y], axis=1)[:, :C])
    H.set_params()
    want = H.detect_speed(x)
    d = torch.from_numpy(x.reshape(-1)).cuda()
    torch.cuda.synchronize()
    got = H.detect_speed(d.data_ptr(), n_frames=x.shape[0], channels=C)
    assert got == want, (C, got, want)
