"""The embed kernels (k_embed, k_embed_strip, k_embed_batch, k_limiter, k_limiter_batch, k_s16_to_f32, k_f32_to_s16) against a
float64 reference of the same operation written here in plain numpy, sample by sample, at the shapes where the kernels take their
edge paths.

`embed_ref` follows awm_embed: for every 1024-frame m in [0, ceil(n / 1024) + 1) the frame is windowed with
O.gen_normalized_window(1024) (its float32 values are the definition), transformed with np.fft.rfft per channel, and every marked bin
k of table row (frame_number0 + m) mod 2 fpb gets D_k = X_k (|X_k|^(-+water_delta) - 1) (up: -, down: +) where |X_k| > 1e-7, with
expm1 / log; the inverse is the unnormalised c2r (irfft * 1024).  Output frame m is ((wm[m-1] w2) + wm[m] w1) + wm[m+1] w0 with
O.synth_window, frames outside the buffer contribute nothing; y = wm + x.  The limiter takes block peaks over every emitted position
(the spill frame included) on the stream-global block grid, blocks -1 and past the end count as the ceiling, and ramps the gain
linearly as limiter.cc does.  Batch items at a stream offset z are embed_ref on zeros(z) ++ x from frame max(z // 1024 - 1, 0) on
(`embed_ref_offset`).  Tables always come from the oracle (O.init_frame_mod), so the device role build is checked as well.
test_reference_matches_oracle pins embed_ref to O.embed within the bound below, without a GPU.

Error bound of a sample (u = 2^-24, LAMBDA = 3, ETA = 4 sqrt(2) + 1: the error of one radix-2 FFT stage in units of u, Higham,
Accuracy and Stability of Numerical Algorithms, 24.1; log2(1024) = 10 stages):
  * forward FFT: the kernels transform a channel PAIR (a + i b) as one complex FFT, so a bin's error scales with the pair's windowed
    norm ||z||, not the channel's own:  eX = LAMBDA (ETA log2 N + 2) u ||z||  (the +2: the window product and the unpacking of the
    pair).  As in test_gpu_speed_scan.py this spreads the FFT's 2-norm bound evenly over the bins: a probabilistic bound.
  * the factor f = exp2f(e/2 log2f(|X|^2)) - 1 (no fast-math: log2f 1 ulp, exp2f 2 ulp, no flush to zero): with t = e log2|X|,
    dt <= |e|/2 (3u + 2u |log2 |X|^2|) + 2u |t|  (the power's fma, log2f, float(water_delta) and the product), and
    df <= |X|^e (4u + ln 2 dt) + u |f|;  the FFT's error propagates through X (|X|^e - 1), whose Jacobian is at most
    |f| + |e| |X|^e:  dD <= |X| df + eX (|f| + |e| |X|^e) + 2u |D|.
  * bins within eX + 4u 1e-7 of |X| = 1e-7 are ambiguous: D may be 0 or the full value there, so |X f| joins their dD.
  * the inverse transform (the pair again): every sample of channel c of frame m is off by at most
    E = 2 sum_k dD_c,k + 4u sum_k (|D_a,k| + |D_b,k|) + LAMBDA ETA log2 N u sqrt(2 sum_k (|D_a,k|^2 + |D_b,k|^2))
    (mirrored bins count twice; the sum of the pair's spectra rounds once per bin; FFT rounding as above).
  * synthesis ((p w2 + c w1) + n w0): E[m-1] w2 + E[m] w1 + E[m+1] w0 + 3u (sum of |terms|); the mix: u |y| where the watermark
    or its bound is nonzero.  Where every bin of the frames around a sample is unmarked or clearly below 1e-7 the bound is exactly 0
    and the output must equal the input bit for bit.
  * the limiter: a block peak moves by at most d, the largest sample bound in the block; with M = max(last, cur) (likewise
    max(cur, next)) the scale ceiling / M moves by at most ceiling d / (M max(M - d, ceiling)), the ramp adds 6u of roundings and
    the product u |out|:  dout <= dy scale + |y| ds + u |out|, where any of the three blocks could be engaged (peak + d > ceiling).
  * --snr: the watermark sum moves by at most sum (2 |wm| b + b^2), the signal sum is exact up to double rounding.
16 bit output must equal the conversion of the float64 result wherever that lies farther than its bound from a quantisation
boundary, and lie between the conversions of result - bound and result + bound elsewhere.

test_bound_is_sharp runs five mutated references (the other block's row at one frame, the 104-sample neighbour term dropped at one
frame, one block's peak given to its neighbour, water_delta * 1.01, the two channels of a pair swapped) and requires each to leave
the bound by at least 10x somewhere.  The GPU tests print the largest error / bound per case with -s.

Largest observed error / bound on an H100 (NVIDIA H100 80GB HBM3, 700 W power limit), 196 cases: 0.93 on a table that marks two
rows only, at a sample whose whole bound is the rounding of the mix (the watermark there is below half an ulp of the sample, and
fl(x + wm) - (x + wm) <= u |y| is rigorous); 0.39 on tones whose bins sit on |X| = 1e-7; at most 0.09 on every other case.
"""
import ctypes
import functools
import math

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import capi

P = O.Params()
N = 1024
U = 2.0 ** -24
LAMBDA = 3.0
ETA = 4 * math.sqrt(2) + 1
LOG2N = 10
MIN_MAG = float(np.float32(1e-7))        # the reference's float min_mag
WIN = O.gen_normalized_window(N).astype(np.float64)
SW = O.synth_window(P).astype(np.float64)
W0, W1, W2 = SW[:N], SW[N:2 * N], SW[2 * N:]
RATE = 44100
KEYS = [O.Key(), O.Key(bytes(range(1, 17)))]
CEIL = float(np.float32(0.99))


# ------------------------------------------------------------------------------------------------ float64 reference

def _spectrum_delta(X, rows, wd, nz, ex=0.0):
    """D and its bound dD for one channel: X [F][101] complex, rows [F][101] table bytes, nz [F] windowed norm of the channel's pair,
    ex [F] a bound of the error the input itself carries into every bin"""
    mag = np.abs(X)
    marked = rows != 0
    e = np.where(rows == 1, -wd, np.where(rows == 2, wd, 0.0))
    pos = mag > 0
    lmag = np.log(np.where(pos, mag, 1.0))
    with np.errstate(over="ignore", invalid="ignore"):
        f = np.where(marked & pos, np.expm1(e * lmag), 0.0)
        pw = f + 1.0                                                   # |X|^e
        above = marked & (mag > MIN_MAG)
        Dfull = X * f
        D = np.where(above, Dfull, 0)
        eX = (LAMBDA * (ETA * LOG2N + 2) * U * nz + ex)[:, None]
        L2 = 2 * lmag / math.log(2)                                    # log2 of the power
        t = e * lmag / math.log(2)
        dt = np.abs(e) / 2 * (3 * U + 2 * U * np.abs(L2)) + 2 * U * np.abs(t)
        df = pw * (4 * U + math.log(2) * dt) + U * np.abs(f)
        dD = mag * df + eX * (np.abs(f) + np.abs(e) * pw) + 2 * U * np.abs(Dfull)
        amb = marked & pos & (np.abs(mag - MIN_MAG) <= eX + 4 * U * MIN_MAG)
        dD = np.where(above, dD, 0.0) + np.where(amb, np.abs(Dfull) + dD, 0.0)
    return D, np.where(np.isfinite(dD), dD, 0.0)


def embed_ref(x, fm, frame_number0, wd=0.01, limiter_block=0, ceiling=CEIL, stream_pos0=0, snr_pos=(0, None), mutate=None, m0=1,
              dx=None, delta_only=False):
    """float64 awm_embed of x [n][C] with FrameMod table fm [2][fpb][101]: (out [n][C], bound [n][C], (sum wm^2, sum x^2, bound of
    the first)).  mutate: one of 'row', 'neighbour', 'peak', 'delta', 'swap' (test_bound_is_sharp), applied at frame / block m0.
    dx [n][C]: a bound of the error x itself carries (x is then a float64 value the GPU only approximates); it enters every bin of
    channel c of frame m as sum_i WIN_i dx_c,i (the transform is linear, so an input error reaches its own channel's spectrum only;
    the rounding the pair shares is the FFT term).  delta_only: the watermark signal alone (k_embed_batch's delta_only), n_proc * 1024
    frames with the spill frame, no mix, no limiter."""
    x = np.asarray(x, np.float64)
    n, C = x.shape
    if n == 0:
        return np.zeros((0, C)), np.zeros((0, C)), (0.0, 0.0, 0.0)
    fpb = fm.shape[1]
    n_real = -(-n // N)
    n_proc = n_real + 1
    Ln = n_proc * N
    ext = np.zeros((Ln, C))
    ext[:n] = x
    fr = ext[:n_real * N].reshape(n_real, N, C)
    r = (frame_number0 + np.arange(n_real, dtype=np.int64)) % (2 * fpb)
    if mutate == "row" and m0 < n_real:
        r[m0] = (r[m0] + fpb) % (2 * fpb)
    rows = fm.reshape(2 * fpb, 101)[r]
    assert not rows[:, :P.min_band].any() and rows.max(initial=0) <= 2
    wd_used = wd * 1.01 if mutate == "delta" else wd
    X, e2, ed = [], [], []
    if dx is not None:
        extd = np.zeros((n_real * N, C))
        extd[:n] = dx
        frd = extd.reshape(n_real, N, C)
    for c in range(C):
        xw = fr[:, :, c] * WIN
        e2.append((xw * xw).sum(axis=1))
        X.append(np.fft.rfft(xw, axis=1)[:, :101])
        ed.append((frd[:, :, c] * WIN).sum(axis=1) if dx is not None else np.zeros(n_real))
    D, dD, nz = [], [], []
    for c in range(C):
        lo = c - c % 2
        nz.append(np.sqrt(e2[lo] + (e2[lo + 1] if lo + 1 < C else 0.0)))
        src = c ^ 1 if (mutate == "swap" and C >= 2 and c < 2) else c
        d, b = _spectrum_delta(X[src], rows, wd_used, nz[c], ed[c])
        D.append(d)
        dD.append(b)
    y = np.zeros((Ln, C))
    by = np.zeros((Ln, C))
    snr_d = snr_s = snr_b = 0.0
    snr_frames = n_proc if limiter_block > 0 else n_real
    p_lo, p_hi = snr_pos[0], min(snr_pos[1] if snr_pos[1] is not None else Ln, snr_frames * N)
    for c in range(C):
        lo = c - c % 2
        hi = lo + 1 if lo + 1 < C else lo
        pair_abs = np.abs(D[lo]).sum(axis=1) + (np.abs(D[hi]).sum(axis=1) if hi != lo else 0)
        pair_sq = (np.abs(D[lo]) ** 2).sum(axis=1) + ((np.abs(D[hi]) ** 2).sum(axis=1) if hi != lo else 0)
        E = 2 * dD[c].sum(axis=1) + 4 * U * pair_abs + LAMBDA * ETA * LOG2N * U * np.sqrt(2 * pair_sq)
        spec = np.zeros((n_real, N // 2 + 1), complex)
        spec[:, :101] = D[c]
        wmf = np.zeros((n_proc + 2, N))
        wmf[1:n_real + 1] = np.fft.irfft(spec, n=N, axis=1) * N
        Ez = np.zeros(n_proc + 2)
        Ez[1:n_real + 1] = E
        t1, t2, t3 = wmf[0:n_proc] * W2, wmf[1:n_proc + 1] * W1, wmf[2:n_proc + 2] * W0
        if mutate == "neighbour" and m0 < n_proc:
            t1[m0] = 0
        wm = ((t1 + t2) + t3).reshape(-1)
        bt = Ez[0:n_proc, None] * W2 + Ez[1:n_proc + 1, None] * W1 + Ez[2:n_proc + 2, None] * W0
        bwm = (bt + 3 * U * (np.abs(t1) + np.abs(t2) + np.abs(t3) + bt)).reshape(-1)
        if delta_only:
            y[:, c], by[:, c] = wm, bwm
            continue
        y[:, c] = wm + ext[:, c]
        by[:, c] = bwm + np.where(np.abs(wm) + bwm > 0, U * (np.abs(y[:, c]) + bwm), 0.0)
        w = wm[p_lo:p_hi]
        snr_d += float((w * w).sum())
        snr_s += float((ext[p_lo:p_hi, c] ** 2).sum())
        snr_b += float((2 * np.abs(w) * bwm[p_lo:p_hi] + bwm[p_lo:p_hi] ** 2).sum())
    if delta_only:
        return y, by, None
    out, bound = y, by
    if limiter_block > 0:
        out, bound = limiter_ref(y, by, limiter_block, ceiling, stream_pos0, move_peak=m0 if mutate == "peak" else None)
    return out[:n], bound[:n], (snr_d, snr_s, snr_b)


def limiter_ref(y, by, block, ceiling, stream_pos0, move_peak=None):
    """the limiter on y [n][C] (bound by) at stream positions stream_pos0 + i, on the stream's grid of `block`-frame blocks: the
    blocks before and after y count as the ceiling.  move_peak = b: block b's peak is given to block b + 1 (test_bound_is_sharp)."""
    B = block
    g = stream_pos0 + np.arange(len(y), dtype=np.int64)
    rel = g // B - stream_pos0 // B
    starts = np.concatenate([[0], np.flatnonzero(np.diff(rel)) + 1])
    pk = np.maximum.reduceat(np.abs(y).max(axis=1), starts)
    dpk = np.maximum.reduceat(by.max(axis=1), starts)
    if move_peak is not None and move_peak + 1 < len(pk):
        pk[move_peak + 1] = max(pk[move_peak + 1], pk[move_peak])
        pk[move_peak] = 0.0
    bm = np.concatenate([[ceiling], np.maximum(ceiling, pk), [ceiling]])     # bm[b + 1] = block b
    db = np.concatenate([[0.0], dpk, [0.0]])
    pe = np.concatenate([[False], pk + dpk > ceiling, [False]])              # the GPU could see this block above the ceiling
    # per block b (index b + 1 of bm): gain at its start and end, their bound, whether the GPU could ramp at all
    Ms, Me = np.maximum(bm[:-2], bm[1:-1]), np.maximum(bm[1:-1], bm[2:])
    dMs, dMe = np.maximum(db[:-2], db[1:-1]), np.maximum(db[1:-1], db[2:])
    s0, s1 = ceiling / Ms, ceiling / Me
    ds = np.maximum(ceiling * dMs / (Ms * np.maximum(Ms - dMs, ceiling)), ceiling * dMe / (Me * np.maximum(Me - dMe, ceiling))) + 6 * U
    eng = pe[:-2] | pe[1:-1] | pe[2:]
    scale = s0[rel] + (g % B) * ((s1 - s0) / B)[rel]
    del g
    out = y * scale[:, None]
    dsp, ep = ds[rel][:, None], eng[rel][:, None]
    bound = np.where(ep, by * (scale[:, None] + dsp) + np.abs(y) * dsp + U * np.abs(out), by)
    return out, bound


def embed_ref_offset(x, fm, z, pad=250, wd=0.01, limiter_block=44100, ceiling=CEIL, **kw):
    """a stream segment at offset z (awm_embed_batch_offsets): embed_ref on zeros(z) ++ x from frame f0 = max(z // 1024 - 1, 0)"""
    x = np.asarray(x, np.float32)
    fpb = fm.shape[1]
    f0 = max(z // N - 1, 0)
    lead = z - f0 * N
    assert f0 == 0 or lead >= N          # frames before f0 (and f0 - 1, whose spill reaches f0) are silent: they carry no watermark
    xz = np.concatenate([np.zeros((lead, x.shape[1]), np.float32), x])
    out, b, snr = embed_ref(xz, fm, 2 * fpb - pad + f0, wd, limiter_block, ceiling, stream_pos0=f0 * N, snr_pos=(lead, None), **kw)
    return out[lead:], b[lead:], snr


@functools.lru_cache(maxsize=None)
def oracle_fm(key_i=0, payload=T.PAYLOAD, **pkw):
    Pp = O.Params(**pkw)
    bv = O.parse_payload(payload, Pp)
    key = KEYS[key_i] if isinstance(key_i, int) else key_i
    fm = np.stack([O.init_frame_mod(key, 0, bv, Pp), O.init_frame_mod(key, 1, bv, Pp)])
    fm.setflags(write=False)
    return fm


def q16(v):
    """k_f32_to_s16 / float_to_int_clip<32> >> 16 on float64 values"""
    s = np.asarray(v, np.float64) * 2.0 ** 31
    t = np.where(s >= 2.0 ** 31, 2 ** 31 - 1, np.where(s <= -2.0 ** 31, -2 ** 31, np.trunc(np.clip(s, -2.0 ** 31, 2.0 ** 31)))).astype(np.int64)
    return (t >> 16).astype(np.int16)


# ------------------------------------------------------------------------------------------------ comparison

MAXR = {}


def check(name, got, want, bound):
    got = np.asarray(got, np.float64).reshape(want.shape)
    err = np.abs(got - want)
    zero = bound == 0
    assert np.array_equal(got[zero], want[zero]), "%s: %d samples with a zero bound differ" % (name, int((got[zero] != want[zero]).sum()))
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(zero, 0.0, err / np.where(zero, 1.0, bound))
    worst = float(r.max(initial=0.0))
    MAXR[name] = worst
    print("%-48s max error / bound %.3g  (max error %.3g, max bound %.3g, %d zero-bound samples)" % (
        name, worst, float(err.max(initial=0)), float(bound.max(initial=0)), int(zero.sum())))
    if worst > 1:
        i = np.unravel_index(int(np.argmax(r)), r.shape)
        raise AssertionError("%s: error %.3g > bound %.3g at %s (got %r, want %r)" % (name, err[i], bound[i], i, got[i], want[i]))


def check_snr(name, got, snr):
    d, s, bd = snr
    assert abs(got[1] - s) <= 1e-9 * s + 1e-300, (name, got, snr)
    assert abs(got[0] - d) <= bd + 1e-9 * d, (name, got, snr)


def check_s16(name, got, want, bound):
    got = np.asarray(got).astype(np.int64)
    lo, hi, mid = q16(want - bound).astype(np.int64), q16(want + bound).astype(np.int64), q16(want).astype(np.int64)
    sure = lo == hi
    assert np.array_equal(got[sure], mid[sure]), (name, int((got[sure] != mid[sure]).sum()))
    assert ((got >= lo) & (got <= hi)).all(), name
    print("%-48s 16 bit: %d of %d samples near a quantisation boundary" % (name, int((~sure).sum()), got.size))


def tone(n, C, amp, bins, seed=0):
    t = np.arange(n)[:, None]
    ph = np.random.default_rng(seed).random((len(bins), C)) * 2 * np.pi
    return sum(amp * np.cos(2 * np.pi * k * t / N + ph[j]) for j, k in enumerate(bins)).astype(np.float32)


def varied(seconds, C, seed, amps):
    """noise whose level changes every 4096 frames through amps: neighbouring limiter blocks of 4096 get different peaks"""
    x = T.noise(seconds, C, seed=seed, amp=1.0)
    lvl = np.asarray(amps, np.float32)[(np.arange(len(x)) // 4096) % len(amps)]
    return (x * lvl[:, None]).astype(np.float32)


# ------------------------------------------------------------------------------------------------ CPU: the reference itself

@pytest.mark.parametrize("case", [(0, 1, True, 0), (1, 2, False, 0), (0, 3, True, 0), (1, 2, True, 5000), (0, 1, False, 3 * RATE + 7)])
def test_reference_matches_oracle(case):
    """embed_ref against O.embed (float32, the reference's arithmetic) within the bound: real tables of two keys, 1 to 3 channels,
    limiter on and off, a zero prefix; and the --snr sums"""
    key_i, C, limiter, z = case
    Pl = O.Params(test_no_limiter=not limiter)
    x = T.noise(4.0, C, seed=40 + C, amp=1.0 if limiter else 0.5)
    xz = np.concatenate([np.zeros((z, C), np.float32), x])
    want = O.embed(xz, KEYS[key_i], T.PAYLOAD, Pl)
    fm = oracle_fm(key_i)
    if z:
        out, b, snr = embed_ref_offset(x, fm, z, limiter_block=RATE if limiter else 0)
    else:
        out, b, snr = embed_ref(x, fm, 2 * fm.shape[1] - 250, 0.01, RATE if limiter else 0)
    check("oracle key %d C=%d limiter=%d z=%d" % case, want.samples[z:], out, b)
    if not z:
        assert abs(10 * math.log10(snr[1] / snr[0]) - want.snr_db) < 1e-6 + 10 / math.log(10) * snr[2] / snr[0]


def test_bound_is_sharp():
    """each of five injected errors leaves the bound by at least 10x somewhere"""
    x = varied(3.0, 2, 51, [0.3, 0.9, 0.6, 1.0])
    fm = oracle_fm(0)
    kw = dict(frame_number0=2 * fm.shape[1] - 250, wd=0.01, limiter_block=4096, ceiling=float(np.float32(0.5)))
    out, b, _ = embed_ref(x, fm, **kw)
    assert (b > 0).all()
    for mutate, m0 in (("row", 40), ("neighbour", 40), ("peak", 9), ("delta", 0), ("swap", 0)):
        mo, _, _ = embed_ref(x, fm, mutate=mutate, m0=m0, **kw)
        ratio = float((np.abs(mo - out) / b).max())
        print("mutation %-10s largest deviation / bound %.3g" % (mutate, ratio))
        assert ratio >= 10, (mutate, ratio)


def test_zero_bound_where_nothing_is_marked():
    """an all-keep table, and audio under 1e-7 everywhere: the bound is exactly 0 (the GPU tests then demand identical bits)"""
    fm = np.zeros((2, 7, 101), np.uint8)
    x = T.noise(1.0, 3, seed=3)
    assert not embed_ref(x, fm, 0)[1].any()
    x = T.noise(1.0, 2, seed=3, amp=1e-12)
    assert not embed_ref(x, oracle_fm(0), 100)[1].any()


# ------------------------------------------------------------------------------------------------ GPU

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context()
    yield c
    c.close()
    if MAXR:
        print("\nlargest error / bound over %d cases: %.3g (%s)" % (len(MAXR), max(MAXR.values()), max(MAXR, key=MAXR.get)))


def run_single(ctx, name, x, fm, ffn=0, pad=250, wd=0.01, block=RATE, ceiling=CEIL, device=None, out_dev=None):
    """ctx.embed with the oracle table fm, compared with embed_ref (device: the byte offsets of in and out in device buffers)"""
    ctx.set_embed_tables(fm)
    fpb = fm.shape[1]
    want, b, snr = embed_ref(x, fm, ffn % (2 * fpb) + 2 * fpb - pad, wd, block, ceiling, stream_pos0=ffn * N)
    kw = dict(first_frame_number=ffn, frames_pad_start=pad, water_delta=wd, limiter_block=block, limiter_ceiling=ceiling, want_snr=True)
    if device is None:
        got, s = ctx.embed(x, **kw)
    else:
        torch = pytest.importorskip("torch")
        n, C = x.shape
        raw_in = torch.zeros(n * C * 4 + 64, dtype=torch.uint8, device="cuda")
        raw_out = torch.zeros(n * C * 4 + 64, dtype=torch.uint8, device="cuda")
        assert raw_in.data_ptr() % 256 == 0 and raw_out.data_ptr() % 256 == 0
        oi, oo = device, device if out_dev is None else out_dev
        raw_in[oi:oi + n * C * 4].copy_(torch.from_numpy(x.reshape(-1).view(np.uint8).copy()).cuda())
        torch.cuda.synchronize()
        _, s = ctx.embed(raw_in.data_ptr() + oi, raw_out.data_ptr() + oo, n_frames=n, channels=C, **kw)
        ctx.synchronize()
        got = raw_out[oo:oo + n * C * 4].cpu().numpy().view(np.float32).reshape(n, C)
    check(name, got, want, b)
    check_snr(name, s, snr)
    return got


LENGTHS = [0, 1, 1023, 1024, 1025, 2049, 3 * RATE, 61 * RATE]


@gpu
@pytest.mark.parametrize("C", [1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("n", LENGTHS)
def test_channels_and_lengths(ctx, C, n):
    x = T.noise(n / RATE, C, seed=1000 + n % 997 + C) if n else np.zeros((0, C), np.float32)
    x = x[:n] if len(x) >= n else np.concatenate([x, T.noise(1.0, C, seed=5)[:n - len(x)]])
    run_single(ctx, "host C=%d n=%d" % (C, n), x, oracle_fm(C % 2))


@gpu
@pytest.mark.parametrize("offsets", [(0, 0), (16, 16), (8, 8), (4, 4), (4, 12), (0, 4), (0, 8)])
def test_device_buffers_at_offsets(ctx, offsets):
    """stereo device buffers at 16-, 8- and 4-byte offsets and with only out misaligned: k_embed_strip only for a 16-byte aligned
    input with an 8-byte aligned output, k_embed<VEC2> only where both allow float2, k_embed<false> otherwise"""
    x = T.noise(3.0, 2, seed=61, amp=1.0)
    run_single(ctx, "device stereo in+%d out+%d" % offsets, x, oracle_fm(0), device=offsets[0], out_dev=offsets[1])


@gpu
@pytest.mark.parametrize("C,off", [(1, 4), (3, 4), (3, 8)])
def test_device_buffers_multichannel(ctx, C, off):
    x = T.noise(2.0, C, seed=62 + C)
    run_single(ctx, "device C=%d in+%d" % (C, off), x, oracle_fm(1), device=off)


@gpu
def test_long_device_stereo(ctx):
    """600 s of stereo on the device: strip_len = ceil(25 841 / (132 SMs * 12 warps)) = 17 > 16"""
    x = T.noise(600.0, 2, seed=63, amp=0.9)
    run_single(ctx, "device stereo 600 s", x, oracle_fm(0), device=0)


@gpu
@pytest.mark.parametrize("C", [1, 2, 3])
def test_pipelined_pieces(ctx, C, monkeypatch):
    """60 s from the host in 1024-frame pieces: the copies, halos and the per-piece limiter cross piece boundaries"""
    monkeypatch.setenv("AWM_PIECE", "1024")
    x = varied(60.0, C, 64 + C, [0.4, 1.0, 0.7])
    run_single(ctx, "pieces of 1024 frames C=%d" % C, x, oracle_fm(1), ceiling=float(np.float32(0.5)))


@gpu
@pytest.mark.parametrize("pad", [0, 250, "2fpb"])
@pytest.mark.parametrize("ffn", [0, 1, "fpb-1", "2fpb-1", 1000, 2 ** 38 - 200])
def test_stream_position(ctx, ffn, pad):
    fm = oracle_fm(0)
    fpb = fm.shape[1]
    ffn = {"fpb-1": fpb - 1, "2fpb-1": 2 * fpb - 1}.get(ffn, ffn)
    pad = 2 * fpb if pad == "2fpb" else pad
    x = T.noise(3.0, 2, seed=70, amp=1.0)
    run_single(ctx, "first frame %d pad %d" % (ffn, pad), x, fm, ffn=ffn, pad=pad)
    run_single(ctx, "first frame %d pad %d mono" % (ffn, pad), x[:, :1].copy(), fm, ffn=ffn, pad=pad)


def synthetic_fm(kind, fpb=7):
    fm = np.zeros((2, fpb, 101), np.uint8)
    if kind == "all":
        k = np.arange(P.min_band, 101)
        for ab in range(2):
            for f in range(fpb):
                fm[ab, f, P.min_band:] = np.where((k + f + ab) % 2, 1, 2)
    elif kind == "some-keep":
        fm[0, 1, P.min_band:] = 1
        fm[1, 4, 50:] = 2
    return fm


@gpu
@pytest.mark.parametrize("table", ["fpbit1", "fpbit3", "short12", "short16", "short20", "linear", "all", "keep", "some-keep"])
def test_tables(ctx, table):
    pkw = {"fpbit1": dict(frames_per_bit=1), "fpbit3": dict(frames_per_bit=3), "short12": dict(payload_size=12, payload_short=True),
           "short16": dict(payload_size=16, payload_short=True), "short20": dict(payload_size=20, payload_short=True),
           "linear": dict(mix=False)}.get(table)
    if pkw is not None:
        fm, pad = oracle_fm(1, T.PAYLOAD[:pkw.get("payload_size", 128) // 4], **pkw), 250
    else:
        fm, pad = synthetic_fm(table), 3
    x = T.noise(5.0, 3, seed=80)
    got = run_single(ctx, "table %s" % table, x, fm, pad=pad, block=0)
    if table == "keep":
        assert np.array_equal(got, x)


@gpu
@pytest.mark.parametrize("wd", [0.001, 0.01, 0.1])
def test_strength(ctx, wd):
    x = T.noise(4.0, 2, seed=81)
    run_single(ctx, "water_delta %g" % wd, x, oracle_fm(0), wd=wd)
    run_single(ctx, "water_delta %g synthetic" % wd, x[:, :1].copy(), synthetic_fm("all"), wd=wd, pad=5)


@gpu
@pytest.mark.parametrize("block", [0, 1024, 1025, 44100, 2 ** 18])
@pytest.mark.parametrize("ceiling", [0.99, 0.5])
def test_limiter(ctx, block, ceiling):
    x = varied(8.0, 2, 90, [0.2, 0.6, 1.0, 0.45])
    c = float(np.float32(ceiling))
    run_single(ctx, "limiter block %d ceiling %g" % (block, ceiling), x, oracle_fm(0), block=block, ceiling=c)
    run_single(ctx, "limiter block %d ceiling %g C=3" % (block, ceiling), x[:, [0, 1, 0]].copy(), oracle_fm(1), ffn=77, block=block, ceiling=c)


@gpu
def test_full_scale(ctx):
    x = np.sign(T.noise(5.0, 2, seed=91)).astype(np.float32)
    run_single(ctx, "full-scale square noise", x, oracle_fm(0))
    run_single(ctx, "full-scale, no limiter", x, oracle_fm(0), block=0)


def signal(kind):
    n = 3 * RATE + 500
    if kind == "silence":
        return np.zeros((n, 2), np.float32)
    if kind == "1e-20":
        return T.noise(n / RATE, 2, seed=92, amp=1e-20)
    if kind == "-80dBFS":
        return T.noise(n / RATE, 2, seed=93, amp=1e-4)
    if kind == "tone-1e-7":             # a cosine of amplitude A at bin k gives |X_k| = A (the window sums to 2)
        return tone(n, 2, 1e-7, range(20, 101, 3), seed=94)
    if kind == "loud+quiet":
        x = T.noise(n / RATE, 2, seed=95, amp=1.0)
        x[:, 1] *= 1e-4
        return x
    if kind == "dc":
        return np.full((n, 3), 0.25, np.float32)
    if kind == "impulse":
        x = np.zeros((n, 2), np.float32)
        x[40 * N, :] = 0.8
        x[41 * N - 1, 0] = -0.6
        return x
    raise KeyError(kind)


@gpu
@pytest.mark.parametrize("kind", ["silence", "1e-20", "-80dBFS", "tone-1e-7", "loud+quiet", "dc", "impulse"])
def test_signals(ctx, kind):
    x = signal(kind)
    got = run_single(ctx, "signal %s" % kind, x, oracle_fm(0))
    run_single(ctx, "signal %s, no limiter" % kind, x, oracle_fm(1), block=0)
    if kind in ("silence", "1e-20"):
        assert np.array_equal(got, x)


def s16_of(x):
    return np.clip(np.round(x * 32768), -32768, 32767).astype(np.int16)


@gpu
@pytest.mark.parametrize("where", ["host", "device", "device+2"])
@pytest.mark.parametrize("C", [1, 2, 3])
def test_s16(ctx, where, C):
    """awm_embed_s16 on host and device buffers (a 2-byte offset: the scalar conversion path), with +-32768 clipping (limiter off)"""
    x16 = s16_of(T.noise(3.0, C, seed=100 + C, amp=0.6))
    x16[1000:1400] = 32767
    x16[5000:5400] = -32768
    for block in (RATE, 0):
        fm = oracle_fm(0)
        ctx.set_embed_tables(fm)
        x = x16.astype(np.float32) / 32768
        want, b, _ = embed_ref(x, fm, 2 * fm.shape[1] - 250, 0.01, block)
        if where == "host":
            got = ctx.embed_s16(x16, limiter_block=block)
        else:
            torch = pytest.importorskip("torch")
            off = 2 if where == "device+2" else 0
            n = len(x16)
            ri = torch.zeros(x16.size * 2 + 64, dtype=torch.uint8, device="cuda")
            ro = torch.zeros(x16.size * 2 + 64, dtype=torch.uint8, device="cuda")
            ri[off:off + x16.size * 2].copy_(torch.from_numpy(x16.reshape(-1).view(np.uint8).copy()).cuda())
            torch.cuda.synchronize()
            ctx.embed_s16(ri.data_ptr() + off, ro.data_ptr() + off, n_frames=n, channels=C, limiter_block=block)
            ctx.synchronize()
            got = ro[off:off + x16.size * 2].cpu().numpy().view(np.int16).reshape(n, C)
        check_s16("s16 %s C=%d block %d" % (where, C, block), got, want, b)
        if block == 0:
            assert (got == 32767).any() and (got == -32768).any()


@gpu
def test_pcm_bind_s16_odd_offset(ctx):
    """awm_pcm_bind_s16 with pad_start * channels odd converts into an odd float offset: the scalar conversion path"""
    x16 = s16_of(T.noise(0.5, 1, seed=7))
    ctx.pcm_bind(x16, pad_start=1, pad_end=2)
    nf, ch = ctypes.c_size_t(), ctypes.c_int()
    ctx.lib.awm_pcm_device.restype = ctypes.c_void_p
    p = ctx.lib.awm_pcm_device(ctx.h, ctypes.byref(nf), ctypes.byref(ch))
    got = np.zeros(nf.value * ch.value, np.float32)
    ctx._ck(ctx.lib.awm_copy_to_host(ctx.h, capi._ptr(got), ctypes.c_void_p(p), ctypes.c_size_t(got.nbytes)))
    want = np.concatenate([[0], x16[:, 0].astype(np.float32) / 32768, [0, 0]]).astype(np.float32)
    assert np.array_equal(got, want)


# ---- batched embed (hostapi: the library builds its own tables; the reference uses the oracle's)

def batch_refs(pcms, payloads, zs, keys):
    out = []
    for x, pay, z, k in zip(pcms, payloads, zs, keys):
        fm = oracle_fm(O.Key(bytes(k)), pay)
        x = np.asarray(x, np.float32)
        out.append(embed_ref_offset(x, fm, z) if x.shape[0] else (np.zeros(x.shape), np.zeros(x.shape), None))
    return out


def payloads_for(n, seed):
    rng = np.random.default_rng(seed)
    return ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in range(n)]


ZERO_FRAMES = [0, 1, 1023, 1024, 2047, 2048, RATE - 1, RATE + 1, 3 * RATE - 1, 3 * RATE + 1, 2 ** 40]


@gpu
@pytest.mark.parametrize("mode", ["host", "s16", "offsets", "keys", "rates"])
def test_batch(mode):
    from audiowmark_b200 import hostapi as H
    H.set_params()
    lens = [0, 1, 1023, 1025, 2 * RATE + 3, 5 * RATE]
    pcms = [T.noise(n / RATE, 1 + i % 3, seed=300 + i, amp=0.9)[:n] if n else np.zeros((0, 1 + i % 3), np.float32) for i, n in enumerate(lens)]
    pcms = [p if len(p) == n else np.concatenate([p, np.zeros((n - len(p), p.shape[1]), np.float32)]) for p, n in zip(pcms, lens)]
    if mode == "offsets" or mode == "keys":
        pcms = [T.noise(1.3, 1 + i % 2, seed=400 + i, amp=0.9) for i in range(len(ZERO_FRAMES))]
    pays = payloads_for(len(pcms), 11)
    zs = ZERO_FRAMES if mode in ("offsets", "keys") else [0] * len(pcms)
    keys = [bytes([i % 4]) * 16 for i in range(len(pcms))] if mode == "keys" else [bytes(16)] * len(pcms)
    refs = batch_refs(pcms, pays, zs, keys)
    if mode == "s16":
        p16 = [s16_of(p) for p in pcms]
        outs = H.add_batch(p16, pays)
        for i, (o, (w, b, _)) in enumerate(zip(outs, batch_refs([p.astype(np.float32) / 32768 for p in p16], pays, zs, keys))):
            check_s16("batch s16 item %d" % i, o, w, b)
        return
    if mode == "rates":
        from test_gpu_resample_ref import add_rates_ref
        rates = [RATE if i % 2 == 0 else 48000 for i in range(len(pcms))]
        outs = H.add_batch_rates(pcms, pays, rates)
        for i, (o, (w, b, _)) in enumerate(zip(outs, refs)):
            if rates[i] == RATE:
                check("batch rates item %d (44.1 kHz)" % i, o, w, b)
            else:
                w, b, _, _ = add_rates_ref(pcms[i], rates[i], oracle_fm(O.Key(bytes(keys[i])), pays[i]))
                check("batch rates item %d (48 kHz)" % i, o, w, b)
        return
    kw = dict(zero_frames=zs) if mode in ("offsets", "keys") else {}
    if mode == "keys":
        kw["keys"] = keys
    outs = H.add_batch(pcms, pays, **kw)
    for i, (o, (w, b, _)) in enumerate(zip(outs, refs)):
        check("batch %s item %d z=%d" % (mode, i, zs[i]), o, w, b)


@gpu
def test_batch_device_odd_value_offsets():
    """stereo items at odd value offsets of a packed device buffer take embed_tile<false>"""
    torch = pytest.importorskip("torch")
    from audiowmark_b200 import hostapi as H
    H.set_params()
    pcms = [T.noise(s, 2, seed=500 + i, amp=0.9) for i, s in enumerate([1.5, 2.0, 0.7])]
    off, items = 1, []
    for p in pcms:
        items.append((off, len(p), 2))
        off += p.size + 1                      # every stereo item starts at an odd value
    flat = np.zeros(off, np.float32)
    for (o, n, c), p in zip(items, pcms):
        flat[o:o + n * c] = p.reshape(-1)
    pays = payloads_for(len(pcms), 12)
    outs = H.add_batch(torch.from_numpy(flat).cuda(), pays, items=items)
    for i, (o, (w, b, _)) in enumerate(zip(outs, batch_refs(pcms, pays, [0] * 3, [bytes(16)] * 3))):
        check("batch device item %d at value %d" % (i, items[i][0]), o.cpu().numpy(), w, b)


# ---- refused arguments: nothing runs, and the context still embeds correctly afterwards

def _expect_refusal(fn, what):
    with pytest.raises(capi.AwmError) as e:
        fn()
    assert what in str(e.value), str(e.value)


@gpu
def test_refused_embed_arguments(ctx):
    fm = oracle_fm(0)
    fpb = fm.shape[1]
    ctx.set_embed_tables(fm)
    x = T.noise(1.0, 2, seed=600)
    for pad in (-1, 2 * fpb + 1):
        _expect_refusal(lambda: ctx.embed(x, frames_pad_start=pad), "frames_pad_start")
        _expect_refusal(lambda: ctx.embed_s16(s16_of(x), frames_pad_start=pad), "frames_pad_start")
    for block in (-1, 1, 1023, 2 ** 18 + 1):
        _expect_refusal(lambda: ctx.embed(x, limiter_block=block), "limiter block")
    max_ffn = (capi.MAX_STREAM_FRAMES - len(x)) // N
    _expect_refusal(lambda: ctx.embed(x, first_frame_number=max_ffn + 1), "stream length")
    _expect_refusal(lambda: ctx.embed(x, first_frame_number=2 ** 63 - 5), "stream length")
    _expect_refusal(lambda: ctx.embed(x, first_frame_number=2 ** 64 - 1), "stream length")
    snr = (ctypes.c_double * 2)()
    rc = ctx.lib.awm_embed_window(ctx.h, capi._ptr(x), capi._ptr(np.empty_like(x)), ctypes.c_size_t(len(x)), ctypes.c_int(2),
                                  ctypes.c_uint64(2 ** 62), ctypes.c_int(250), ctypes.c_double(0.01), ctypes.c_int(RATE), ctypes.c_float(0.99),
                                  ctypes.c_uint64(0), ctypes.c_uint64(len(x)), snr)
    assert rc != 0 and b"stream length" in ctx.lib.awm_last_error(ctx.h)
    run_single(ctx, "after refusals", x, fm)
    run_single(ctx, "last stream position", x, fm, ffn=max_ffn)


@gpu
def test_refused_embed_tables(ctx):
    fm = oracle_fm(1)
    ctx.set_embed_tables(fm)
    bad = fm.copy()
    bad[1, 5, 60] = 3
    _expect_refusal(lambda: ctx.set_embed_tables(bad), "entries are 0 keep")
    bad = fm.copy()
    bad[0, 9, 19] = 1
    _expect_refusal(lambda: ctx.set_embed_tables(bad), "bins below")
    x = T.noise(2.0, 1, seed=601)
    want, b, _ = embed_ref(x, fm, 2 * fm.shape[1] - 250, 0.01, RATE)     # the refused calls left the previous table in place
    check("table kept after refusals", ctx.embed(x), want, b)


def _batch_call(ctx, fn_name, x, items, coded, **kw):
    """the batched C entry points with explicit limiter / pad arguments; returns (rc, message)"""
    lib = ctx.lib
    it = np.array(items, capi.BATCH_ITEM)
    out = np.empty_like(x)
    n = ctypes.c_size_t(x.size)
    pad = ctypes.c_int(kw.get("pad", 250))
    wd, ceil = ctypes.c_double(0.01), ctypes.c_float(0.99)
    rates = np.full(len(items), 44100, np.int32)
    emit = np.array([t[1] for t in items], np.uint64)
    zeros = np.zeros(len(items), np.uint64)
    keyi = np.zeros(len(items), np.uint32)
    if fn_name == "awm_embed_batch":
        rc = lib.awm_embed_batch(ctx.h, capi._ptr(x), capi._ptr(out), 0, n, capi._ptr(it), ctypes.c_size_t(len(it)), capi._ptr(coded), pad, wd,
                                 ctypes.c_int(kw["block"]), ceil, None)
    elif fn_name == "awm_embed_batch_offsets":
        rc = lib.awm_embed_batch_offsets(ctx.h, capi._ptr(x), capi._ptr(out), 0, n, capi._ptr(it), ctypes.c_size_t(len(it)), capi._ptr(zeros),
                                         capi._ptr(coded), pad, wd, ctypes.c_int(kw["block"]), ceil, None)
    elif fn_name == "awm_embed_batch_rates":
        rc = lib.awm_embed_batch_rates(ctx.h, capi._ptr(x), capi._ptr(out), 0, n, capi._ptr(it), ctypes.c_size_t(len(it)), capi._ptr(coded),
                                       capi._ptr(rates), capi._ptr(emit), 44100, pad, wd, ctypes.c_int(kw["ms"]), ceil, None, ctypes.c_size_t(0))
    elif fn_name == "awm_embed_batch_rates_offsets":
        rc = lib.awm_embed_batch_rates_offsets(ctx.h, capi._ptr(x), capi._ptr(out), 0, n, capi._ptr(it), ctypes.c_size_t(len(it)), capi._ptr(coded),
                                               capi._ptr(rates), capi._ptr(emit), capi._ptr(zeros), 44100, pad, wd, ctypes.c_int(kw["ms"]), ceil,
                                               None, ctypes.c_size_t(0))
    else:
        rc = lib.awm_embed_batch_keys(ctx.h, capi._ptr(x), capi._ptr(out), 0, n, capi._ptr(it), ctypes.c_size_t(len(it)), capi._ptr(coded),
                                      None, None, None, capi._ptr(keyi), 44100, pad, wd, ctypes.c_int(kw["ms"]), ceil, None, ctypes.c_size_t(0))
    return rc, (lib.awm_last_error(ctx.h).decode() if rc else ""), out.reshape(-1, 2)


@gpu
@pytest.mark.parametrize("fn_name", ["awm_embed_batch", "awm_embed_batch_offsets", "awm_embed_batch_rates", "awm_embed_batch_rates_offsets",
                                     "awm_embed_batch_keys"])
def test_refused_batch_arguments(ctx, fn_name):
    from audiowmark_b200 import hostapi as H
    H.set_params()
    key = bytes(16)
    roles = np.ascontiguousarray(H.embed_roles(key))
    ctx._ck(ctx.lib.awm_set_embed_roles(ctx.h, capi._ptr(roles), ctypes.c_int(roles.shape[0]), ctypes.c_int(H.n_coded_bits())))
    ctx.set_embed_roles_keys([key], H.role_layout())
    x = T.noise(2.0, 2, seed=602)
    flat = np.ascontiguousarray(x.reshape(-1))
    items = [(0, len(x), 2)]
    coded = np.ascontiguousarray(H.coded_bits(key, T.PAYLOAD)[None])
    fpb = roles.shape[0]
    per_ms = fn_name != "awm_embed_batch" and fn_name != "awm_embed_batch_offsets"
    bad_blocks = [dict(ms=10), dict(ms=6000)] if per_ms else [dict(block=1023), dict(block=2 ** 18 + 1), dict(block=-5)]
    for b in bad_blocks:
        rc, msg, _ = _batch_call(ctx, fn_name, flat, items, coded, **b)
        assert rc and "limiter block" in msg, (b, msg)
    good = dict(ms=1000) if per_ms else dict(block=RATE)
    for pad in (-1, 2 * fpb + 1):
        rc, msg, _ = _batch_call(ctx, fn_name, flat, items, coded, pad=pad, **good)
        assert rc and "frames_pad_start" in msg, (pad, msg)
    rc, msg, got = _batch_call(ctx, fn_name, flat, items, coded, **good)
    assert rc == 0, msg
    w, b, _ = embed_ref(x, oracle_fm(O.Key(key), T.PAYLOAD), 2 * fpb - 250, 0.01, RATE)
    check("%s after refusals" % fn_name, got, w, b)
