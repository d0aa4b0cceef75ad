"""The resampler kernels (k_resample behind awm_resample / awm_resample_range, and k_resample_batch, k_resample_mix_batch and
k_limiter_rates behind `add` at any sample rate) against a float64 restatement of the filter as include/awm_b200.h defines it:

  out[n] = sum_i in[i] g (i - n / ratio),   g (d) = fc sinc (fc d) w (d / h),   w (x) = 0.384 + 0.5 cos (pi x) + 0.116 cos (2 pi x)
  (0 for |x| >= 1),   fc = min (1, ratio),   h = ceil (hlen / fc),   256 phases, linear interpolation between phase rows.

`resample_ref` takes output n's position as the definition does, t = (h - 1) + n step in double (step = 1 / ratio; one product, then
one sum, not fused), c = floor t, p = floor (256 (t - c)), alpha = 256 (t - c) - p, and sums the 2h inputs c - 2h + 2 + j with the
weights W_j = (1 - alpha) g (d_j - p / 256) + alpha g (d_j - (p + 1) / 256), d_j = j - (h - 1), g evaluated in float64 (not from a
float32 table).  Inputs outside [0, n_in) are 0; outputs whose c lies past n_stop + h - 2 (a stream's post-roll) are 0.
test_reference_matches_oracle pins it to O.resample_ratio within the bound below, without a GPU.

`add_rates_ref` restates O.embed_resampled (and awm_embed_batch_rates_offsets for a stream offset z) on top of it: the input is
resampled to 44.1 kHz from a 1024-frame before the first output whose taps reach the item (the stream is exactly silent before), the
watermark signal is embed_ref of test_gpu_embed_ref.py on that (delta_only), resampled back for the stream's n_emit frames (n_emit and
the WatermarkGen run count from O.resampled_add_plan: `add_plan` skips the loop's iterations before EOF, test_add_plan_matches_oracle),
mixed into the input and limited on the item's own block grid of rate * 1000 / 1000 frames (limiter_ref), with the --snr sums.

Error bound of an output (u = 2^-24, LAMBDA = 3 as in the other reference tests):
  * a weight: the kernel forms w = fl (fl (b T0) + fl (a T1)) from float32 table entries T = g (1 + theta), |theta| <= u, a = fl
    (alpha), |a - alpha| <= u alpha, and b = fl (1 - a), |b - (1 - alpha)| <= u alpha + u (1 - alpha + u alpha) =: eb.  With B0 = 1 -
    alpha + eb >= |b| and B1 = alpha (1 + u) >= |a|:
      |w - W| <= eW = (2u + u^2)(1 + u)(B0 |g0| + B1 |g1|)  (the two products and the sum)
                    + u (B0 |g0| + B1 |g1|)                 (the table entries)
                    + eb |g0| + u alpha |g1|                (a and b).
  * the dot product of 2h float products accumulated in tap order: LAMBDA sqrt(2h) u sum_j |x_j| (|W_j| + eW_j) (probabilistic, as
    the FFT terms of the other reference tests), plus sum_j |x_j| eW_j.
  * an input that carries a bound dx (the resampled add's second stage): |x_j| becomes |x_j| + dx_j above, plus sum_j |W_j| dx_j.
Where every tap is 0 or reads a zero input the bound is exactly 0, and the GPU must return 0 bit for bit.
The resampled add chains the bounds: the in-resampler's bound dx enters every bin of a watermark frame as sum_i WIN_i dx_i
(embed_ref's dx), the watermark's bound passes through the out-resampler as sum_j |W_j| b_j plus that resampler's own rounding, the
mix adds u |y|, and limiter_ref and the --snr sums propagate it as in test_gpu_embed_ref.py.

test_bound_is_sharp runs five mutated references (rows p and p + 1 swapped, the taps one frame off, fc = 1 when downsampling, h =
floor (hlen / fc), a Blackman window 0.42 / 0.5 / 0.08) and requires each to leave the bound by at least 10x somewhere.  The GPU
tests print the largest error / bound per case with -s.

Largest observed error / bound on an H100 (NVIDIA H100 80GB HBM3, 700 W power limit), about 200 cases, the file taking about 2.5
minutes: 0.89 on a 1025-frame stereo item at 2 822 399 Hz and 0.59 on a 36-frame item of 3 channels at 48 kHz (short batch
items); 0.40 for k_resample (phase 255 at hlen 96, and stereo 4 bytes off alignment); 0.30 for the second grid-stride pass; 0.28
for windows far into a stream; at most 0.034 for items at stream offsets and 0.004 for a window.
Sabotage check (each change in a scratch build, caught by the tests named): a and b swapped in resample_pos -> every k_resample
test but test_ratios at 1/64 + 1 ulp with hlen 96; k_resample_mix_batch's scratch index one frame off -> test_stream_offsets,
test_window_cuts_limiter_block; k_limiter_rates given z for i0 -> test_stream_offsets.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
import test_gpu_embed_ref as E
from audiowmark_b200 import capi
from test_gpu_embed_ref import CEIL, LAMBDA, N, U, check, check_s16, check_snr, embed_ref, limiter_ref, oracle_fm, payloads_for, s16_of

PHASES = 256
MARK = 44100
WINDOW = (0.384, 0.5, 0.116)
NEVER = None                    # n_stop of a resampler that keeps being fed zeros


# ------------------------------------------------------------------------------------------------ float64 reference

def filter_shape(ratio, hlen, mutate=None):
    fc = min(1.0, ratio)
    h = math.floor(hlen / fc) if mutate == "floor" else math.ceil(hlen / fc)
    return (1.0 if mutate == "fc1" else fc), h


def _g_rows(fc, h, win):
    """g (d_j - p / 256) for p = 0 .. 256 and j = 0 .. 2h - 1, float64: [257][2h]"""
    d = (np.arange(2 * h, dtype=np.float64) - (h - 1))[None, :] - np.arange(PHASES + 1, dtype=np.float64)[:, None] / PHASES
    x = np.abs(d / h)
    w = np.where(x >= 1, 0.0, win[0] + win[1] * np.cos(np.pi * x) + win[2] * np.cos(2 * np.pi * x))
    return fc * np.sinc(fc * d) * w


def resample_at(x, ratio, hlen, idx, in_first=0, n_stop=NEVER, dx=None, mutate=None):
    """outputs idx (stream output indices) of resampling the stream whose frames [in_first, in_first + len(x)) are x [n][C] and which is
    0 elsewhere: (out [len(idx)][C], bound).  dx: a bound of the error x carries.  mutate: 'swap', 'shift', 'fc1', 'floor', 'blackman'
    (test_bound_is_sharp)."""
    x = np.asarray(x, np.float64)
    nw, C = x.shape
    idx = np.asarray(idx, np.int64)
    out, bound = np.zeros((len(idx), C)), np.zeros((len(idx), C))
    fc, h = filter_shape(ratio, hlen, mutate)
    K = 2 * h
    t = (h - 1) + idx.astype(np.float64) * (1.0 / ratio)         # one product, one sum: numpy does not fuse them
    cf = np.floor(t)
    frac = (t - cf) * PHASES
    p = frac.astype(np.int64)
    al = frac - p
    c = cf.astype(np.int64)
    i0 = c - 2 * h + 2 - in_first + (1 if mutate == "shift" else 0)
    if mutate == "swap":
        al = 1.0 - al
    live = np.ones(len(idx), bool) if n_stop is NEVER else c <= n_stop + h - 2
    dxa = np.zeros_like(x) if dx is None else np.asarray(dx, np.float64)
    nzr = np.flatnonzero((x != 0).any(axis=1) | (dxa > 0).any(axis=1))
    if not len(nzr):
        return out, bound
    sel = np.flatnonzero(live & (i0 + K - 1 >= nzr[0]) & (i0 <= nzr[-1]))     # outputs whose taps reach a nonzero input
    G = _g_rows(fc, h, (0.42, 0.5, 0.08) if mutate == "blackman" else WINDOW)
    j = np.arange(K)
    m = max(1, 3_000_000 // (K * C))
    for s in range(0, len(sel), m):
        q = sel[s:s + m]
        ii = i0[q][:, None] + j
        ok = ((ii >= 0) & (ii < nw))[..., None]
        iic = np.clip(ii, 0, nw - 1)
        xv, dv = np.where(ok, x[iic], 0.0), np.where(ok, dxa[iic], 0.0)
        g0, g1 = G[p[q]], G[p[q] + 1]
        a = al[q][:, None]
        W = (1 - a) * g0 + a * g1
        eb = U * a + U * (1 - a + U * a)
        B0, B1 = 1 - a + eb, a * (1 + U)
        A = B0 * np.abs(g0) + B1 * np.abs(g1)
        eW = (2 * U + U * U) * (1 + U) * A + U * A + eb * np.abs(g0) + U * a * np.abs(g1)
        out[q] = np.einsum("mk,mkc->mc", W, xv)
        xa = np.abs(xv) + dv
        bound[q] = (np.einsum("mk,mkc->mc", eW, xa) + np.einsum("mk,mkc->mc", np.abs(W), dv)
                    + LAMBDA * math.sqrt(K) * U * np.einsum("mk,mkc->mc", np.abs(W) + eW, xa))
    return out, bound


def resample_ref(x, ratio, hlen, n_out, first_out=0, in_first=0, n_stop=NEVER, dx=None, mutate=None):
    """outputs [first_out, first_out + n_out) of resampling a stream (see resample_at)"""
    return resample_at(x, ratio, hlen, np.arange(first_out, first_out + n_out, dtype=np.int64), in_first, n_stop, dx, mutate)


def add_plan(n, rate, limiter=True):
    """O.resampled_add_plan (n_emit, WatermarkGen runs) without the loop's iterations before EOF: until then the loop cannot stop and
    nothing it computes is returned, so it starts at the first iteration that feeds less than a frame"""
    r_in, r_out, bs = MARK / rate, rate / MARK, rate * 1000 // 1000

    def it(j):
        runs = O.stream_avail(N * (j + 1), r_in) // N
        em = O.stream_avail(runs * N, r_out) if runs else 0
        return em, runs, (max(em // bs - 1, 0) * bs if limiter else em)
    j = n // N
    em = runs = total_out = 0
    if j:
        em, runs, lim = it(j - 1)
        total_out = min(lim, N * j)
    while total_out != n:
        em, runs, lim = it(j)
        total_out = min(lim, n)
        j += 1
    return em, runs


def data_blocks(runs, fpb, pad=250):
    f0 = 2 * fpb - pad
    return max((f0 + runs) // fpb - f0 // fpb - 1, 0)


def add_rates_ref(x, rate, fm, z=0, limiter=True, snr=None, wd=0.01, pad=250, ceiling=CEIL):
    """float64 `add` of x [n][C] at `rate` as frames [z, z + n) of a stream that is silent before: (out [n][C], bound, (sum wm^2,
    sum x^2, bound of the first) over stream positions snr = [s0, s1) (default [z, stream n_emit)), WatermarkGen runs)"""
    x = np.asarray(x, np.float32)
    n, C = x.shape
    end, runs = add_plan(z + n, rate, limiter)
    if n == 0:
        return np.zeros((0, C)), np.zeros((0, C)), (0.0, 0.0, 0.0), runs
    r_in, r_out = MARK / rate, rate / MARK
    h_in, h_out = filter_shape(r_in, 16)[1], filter_shape(r_out, 16)[1]
    n44 = ((math.floor((end - 1) * (1.0 / r_out)) + h_out) // N + 1) * N          # up to the out-resampler's highest tap
    # 44.1 kHz outputs before m_lo read only silence (their last tap c + 1 < z): start one 1024-frame before m_lo's frame
    m_lo = max(0, math.floor((z - h_in - 2) / (1.0 / r_in)) - 2)
    w0 = max(m_lo // N - 1, 0) * N
    x44, b44 = resample_ref(x, r_in, 16, n44 - w0, first_out=w0, in_first=z)
    fpb = fm.shape[1]
    wm44, bwm44, _ = embed_ref(x44, fm, 2 * fpb - pad + w0 // N, wd, dx=b44, delta_only=True)
    B = rate * 1000 // 1000
    p0 = max((z // B - 1) * B, 0) if limiter else z                               # the block before the item's first counts
    wm, bwm = resample_ref(wm44[:n44 - w0], r_out, 16, end - p0, first_out=p0, in_first=w0, dx=bwm44[:n44 - w0])
    ext = np.zeros((end - p0, C))
    ext[z - p0:z - p0 + n] = x
    y = wm + ext
    by = bwm + np.where(np.abs(wm) + bwm > 0, U * (np.abs(y) + bwm), 0.0)
    s0, s1 = snr if snr is not None else (z, end)
    w, bw = wm[s0 - p0:s1 - p0], bwm[s0 - p0:s1 - p0]
    sums = (float((w * w).sum()), float((ext[s0 - p0:s1 - p0] ** 2).sum()), float((2 * np.abs(w) * bw + bw * bw).sum()))
    if limiter:
        y, by = limiter_ref(y, by, B, ceiling, p0)
    return y[z - p0:z - p0 + n], by[z - p0:z - p0 + n], sums, runs


# ------------------------------------------------------------------------------------------------ comparison

SEEN = set()


def chk(name, got, want, bound):
    SEEN.add(name)
    check(name, got, want, bound)


def check_snr_db(name, got_db, sums):
    """a --snr value in dB against the reference sums: 10 log10 (signal / watermark) moves by at most 10 / ln 10 * bound / watermark"""
    d, s, bd = sums
    if d == 0 or s == 0:
        return
    want = 10 * math.log10(s / d)
    assert abs(got_db - want) <= 10 / math.log(10) * bd / max(d - bd, 1e-300) + 1e-9 * abs(want), (name, got_db, want)


def noise(n, C, seed, amp=0.5):
    rng = np.random.default_rng(seed)
    return ((rng.random((n, C), dtype=np.float32) - 0.5) * (2 * amp)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ CPU: the reference itself

@pytest.mark.parametrize("ratio", [44100 / 48000, 48000 / 44100, 1 / 1.01, 0.49, 63.9, 1 / 63.9])
@pytest.mark.parametrize("hlen", [8, 16, 96])
def test_reference_matches_oracle(ratio, hlen):
    """resample_ref against O.resample_ratio (float32, the oracle's own filter table) within the bound, trailing zeros included"""
    h = filter_shape(ratio, hlen)[1]
    n = max(int(40 * h / min(ratio, 1)), 4000) if ratio >= 1 else 8 * h + 3000
    x = noise(n, 2, seed=hlen + int(ratio * 1000))
    n_out = O.stream_out_count(n, ratio, hlen) + 3
    want = O.resample_ratio(x, ratio, n_out=n_out, hlen=hlen)
    got, b = resample_ref(x, ratio, hlen, n_out, n_stop=n)
    chk("oracle ratio %.6g hlen %d" % (ratio, hlen), want, got, b)
    assert not got[-3:].any() and not b[-3:].any()


def test_bound_is_sharp():
    """each of five injected errors leaves the bound by at least 10x somewhere"""
    ratio, hlen = 44100 / 48000, 16
    x = noise(20000, 1, seed=5)
    out, b = resample_ref(x, ratio, hlen, 15000, n_stop=len(x))
    live = b > 0
    assert live[100:-100].all()
    for mutate in ("swap", "shift", "fc1", "floor", "blackman"):
        mo, _ = resample_ref(x, ratio, hlen, 15000, n_stop=len(x), mutate=mutate)
        r = float((np.abs(mo - out)[live] / b[live]).max())
        print("mutation %-9s largest deviation / bound %.3g" % (mutate, r))
        assert r >= 10, (mutate, r)


def test_zero_bound_on_silence():
    """outputs whose taps read only zeros have a zero bound: the GPU tests then demand +0 exactly"""
    x = np.zeros((5000, 2), np.float32)
    x[2000] = 0.5
    out, b = resample_ref(x, 48000 / 44100, 16, 5000, n_stop=5000)
    zero = ~(b > 0).any(axis=1)
    assert zero[:2000].any() and zero[2300:].any() and not out[zero].any()


@pytest.mark.parametrize("rate", [690, 8000, 48000, 192000, 2822399])
@pytest.mark.parametrize("limiter", [True, False])
def test_add_plan_matches_oracle(rate, limiter):
    P = O.Params(test_no_limiter=not limiter)
    for n in (0, 1, 1023, 1024, 1025, 5000, 3 * rate // 2 + 17):
        assert add_plan(n, rate, limiter) == O.resampled_add_plan(n, rate, P), (rate, n)


@pytest.mark.parametrize("case", [(48000, 1, True), (22050, 2, True), (8000, 3, False), (192000, 2, False)])
def test_add_reference_matches_oracle(case):
    """add_rates_ref against O.embed_resampled (float32 throughout) within the bound, and its --snr"""
    rate, C, limiter = case
    x = noise(int(2.2 * rate), C, seed=rate + C, amp=1.0 if limiter else 0.5)
    P = O.Params(test_no_limiter=not limiter)
    want = O.embed(x, O.Key(), T.PAYLOAD, P, rate=rate)
    out, b, sums, runs = add_rates_ref(x, rate, oracle_fm(0), limiter=limiter)
    chk("oracle add %d Hz C=%d limiter=%d" % case, want.samples, out, b)
    check_snr_db("oracle add %d Hz" % rate, want.snr_db, sums)
    assert data_blocks(runs, oracle_fm(0).shape[1]) == want.data_blocks


# ------------------------------------------------------------------------------------------------ GPU: k_resample

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context()
    yield c
    c.close()
    got = {k: E.MAXR[k] for k in SEEN if k in E.MAXR}
    if got:
        print("\nlargest error / bound over %d cases: %.3g (%s)" % (len(got), max(got.values()), max(got, key=got.get)))


def run_resample(ctx, name, x, ratio, hlen, n_out):
    got = ctx.resample(x, ratio, n_out=n_out, hlen=hlen)
    want, b = resample_ref(x, ratio, hlen, n_out, n_stop=len(x))
    chk(name, got, want, b)
    return got


PHASE255 = 256000 / 255999         # step = 1 - 1 / 256000: outputs 1 .. 999 sit on phase 255, alpha = 1 - n / 1000
RATIOS = [np.nextafter(1 / 64, 1.0), np.nextafter(64.0, 0.0), 44100 / 48000, 48000 / 44100, 8000 / 44100, 44100 / 8000, 192000 / 44100,
          44100 / 192000, 1.0, 2.0, PHASE255, 0.8]


@gpu
@pytest.mark.parametrize("hlen", [8, 16, 96])
@pytest.mark.parametrize("ratio", RATIOS)
def test_ratios(ctx, ratio, hlen):
    """stereo from the host (k_resample<2>) at the range limits, the common rate pairs, the integer ratios (positions on input
    frames reproduce them exactly), phase 255 with alpha close to 1 (row 256 is read) and alpha = 0 (ratio 0.8: step 1.25)"""
    fc, h = filter_shape(ratio, hlen)
    n_out = min(6000, int(200 * h * ratio / fc) + 2000) if ratio > 1 else max(int(3_000_000 / (2 * h)) // 8, 300)
    n = int(n_out / ratio) + 2 * h + 5
    x = noise(n, 2, seed=int(ratio * 997) + hlen)
    got = run_resample(ctx, "ratio %.9g hlen %d" % (ratio, hlen), x, ratio, hlen, n_out)
    if ratio in (1.0, 2.0):
        k = int(ratio)
        on = x[:(n_out + k - 1) // k]
        big = np.abs(on) > 1e-6
        assert np.array_equal(got[::k][:len(on)][big], on[big])
    if ratio == PHASE255:
        t = (h - 1) + np.arange(1, 1000) * (1.0 / ratio)
        fr = (t - np.floor(t)) * PHASES
        assert (fr.astype(int) == 255).all() and (fr - 255).max() > 0.99
    if ratio == 0.8:
        t = (h - 1) + np.arange(n_out) * (1.0 / ratio)
        assert ((t - np.floor(t)) * PHASES % 1 == 0).all()


@gpu
@pytest.mark.parametrize("C", [1, 3, 6])
@pytest.mark.parametrize("ratio", [44100 / 48000, 48000 / 44100])
def test_channels(ctx, C, ratio):
    x = noise(30000, C, seed=10 + C)
    run_resample(ctx, "C=%d ratio %.6g" % (C, ratio), x, ratio, 16, int(len(x) * ratio))


@gpu
@pytest.mark.parametrize("ratio", [44100 / 48000, 2.0])
def test_unaligned_stereo_device(ctx, ratio):
    """stereo in and out 4 bytes off 8-byte alignment: k_resample<0> instead of <2>, the same values"""
    torch = pytest.importorskip("torch")
    x = noise(40000, 2, seed=21)
    n_out = int(len(x) * ratio)
    xd = torch.zeros(x.size + 2, dtype=torch.float32, device="cuda")
    yd = torch.zeros(n_out * 2 + 2, dtype=torch.float32, device="cuda")
    xd[1:1 + x.size] = torch.from_numpy(x.reshape(-1)).cuda()
    torch.cuda.synchronize()
    assert (xd.data_ptr() + 4) % 8 == 4 and (yd.data_ptr() + 4) % 8 == 4
    ctx.resample(xd.data_ptr() + 4, ratio, n_out=n_out, n_frames=len(x), channels=2, out=yd.data_ptr() + 4)
    ctx.synchronize()
    got = yd[1:1 + 2 * n_out].cpu().numpy().reshape(n_out, 2)
    want, b = resample_ref(x, ratio, 16, n_out, n_stop=len(x))
    chk("device stereo +4 ratio %.6g" % ratio, got, want, b)


@gpu
@pytest.mark.parametrize("ratio", [44100 / 48000, 48000 / 44100, 1 / 63.9, 63.9])
@pytest.mark.parametrize("C", [1, 2, 3])
def test_short_inputs(ctx, ratio, C):
    """inputs of 1, 2, 2h - 1 and 2h frames, and outputs past the post-roll: they must be +0 exactly"""
    h = filter_shape(ratio, 16)[1]
    for n in (1, 2, 2 * h - 1, 2 * h):
        x = noise(n, C, seed=n + C)
        n_out = O.stream_out_count(n, ratio) + 7
        got = run_resample(ctx, "n=%d C=%d ratio %.6g" % (n, C, ratio), x, ratio, 16, n_out)
        assert not got[-7:].any()


def _rounds_up_onto_integer(ratio, h, near, span=200_000):
    """an output index n >= near whose t = (h - 1) + n step is an integer in double although the exact value lies below it"""
    step = 1.0 / ratio
    n = near + np.arange(span, dtype=np.int64)
    t = (h - 1) + n.astype(np.float64) * step
    for k in np.flatnonzero(t == np.floor(t)):
        if Fraction(int(n[k])) * Fraction(step) + (h - 1) < Fraction(float(t[k])):
            return int(n[k])
    raise AssertionError("no output rounds up onto an integer near %d" % near)


@gpu
@pytest.mark.parametrize("C", [1, 2])
@pytest.mark.parametrize("ratio,where", [(r, w) for r in (44100 / 48000, 48000 / 44100) for w in (2 ** 31 - 3, 2 ** 32 - 1000, 2 ** 40 + 11)]
                         + [(48000 / 44100, "up")])
def test_range_at_stream_positions(ctx, ratio, where, C):
    """awm_resample_range windows far into a stream: only the window is allocated; "up": an output whose position rounds up onto an
    input frame in double (a fused multiply-add would land on the frame before, phase 255).  Near 2^40 only step = 1 / (48000 /
    44100) has such outputs: the double step of the other direction rounds every near-integer position down."""
    torch = pytest.importorskip("torch")
    h = filter_shape(ratio, 16)[1]
    out_first = _rounds_up_onto_integer(ratio, h, 2 ** 40) - 100 if where == "up" else where
    out_frames = 3000
    n_total = int((out_first + out_frames) / ratio) + 10 * h
    first, end = capi.resample_taps(n_total, ratio, out_first, out_frames)
    x = noise(end - first, C, seed=C + out_first % 1000)
    yd = torch.zeros(out_frames * C, dtype=torch.float32, device="cuda")
    ctx.resample_range(x, first, n_total, ratio, yd.data_ptr(), out_first, out_frames)
    ctx.synchronize()
    got = yd.cpu().numpy().reshape(out_frames, C)
    want, b = resample_ref(x, ratio, 16, out_frames, first_out=out_first, in_first=first, n_stop=n_total)
    chk("range at %d C=%d ratio %.6g" % (out_first, C, ratio), got, want, b)


# ------------------------------------------------------------------------------------------------ GPU: the rates kernels

RATES = [690, 8000, 11025, 22050, 32000, 48000, 96000, 192000, 2822399]


@pytest.fixture
def hapi():
    from audiowmark_b200 import hostapi as H
    H.set_params()
    yield H
    H.set_params()


def rate_items(rate, seed):
    """lengths 0, 1, 2 h_in, 1023, 1025 and a longer one; channels 1, 2, 3, 6; quiet and loud (the limiter engages)"""
    h_in = filter_shape(MARK / rate, 16)[1]
    long = int(2.5 * rate) if rate <= 192000 else 20000
    lens = [0, 1, 2 * h_in, 1023, 1025, long, long // 3]
    chans = [1, 2, 3, 6, 2, 2, 3]
    amps = [0.5, 1.0, 0.05, 1.0, 0.3, 1.0, 0.02]
    return [noise(n, c, seed + i, a) for i, (n, c, a) in enumerate(zip(lens, chans, amps))]


def check_item(name, got, x, rate, pay, z=0, limiter=True, snr_db=None, blocks=None):
    fm = oracle_fm(O.Key(bytes(16)), pay)
    want, b, sums, runs = add_rates_ref(x, rate, fm, z=z, limiter=limiter)
    chk(name, got, want, b)
    if snr_db is not None:
        check_snr_db(name, snr_db, sums)
    if blocks is not None:
        assert blocks == data_blocks(runs, fm.shape[1]), (name, blocks)


@gpu
@pytest.mark.parametrize("rate", RATES)
def test_batch_rates(hapi, rate):
    """one add_batch_rates call per rate: every item against add_rates_ref, with its --snr and data blocks"""
    pcms = rate_items(rate, seed=rate % 1000)
    pays = payloads_for(len(pcms), rate % 97)
    outs, blocks, snrs = hapi.add_batch_rates(pcms, pays, [rate] * len(pcms), want_stats=True)
    for i, (o, x) in enumerate(zip(outs, pcms)):
        check_item("batch %d Hz item %d n=%d C=%d" % (rate, i, x.shape[0], x.shape[1]), o, x, rate, pays[i], snr_db=snrs[i], blocks=blocks[i])


@gpu
@pytest.mark.parametrize("rate", [690, 48000, 2822399])
def test_single_add_without_limiter(hapi, rate):
    hapi.set_params(test_no_limiter=True)
    x = noise(int(1.5 * rate) if rate < 10 ** 6 else 30000, 2, seed=7, amp=1.0)
    y, blocks, snr = hapi.add(x, T.PAYLOAD, sample_rate=rate, want_stats=True)
    check_item("add %d Hz no limiter" % rate, y, x, rate, T.PAYLOAD, limiter=False, snr_db=snr, blocks=blocks)


@gpu
@pytest.mark.parametrize("rate", [22050, 48000])
def test_batch_rates_s16(hapi, rate):
    """16 bit items (add_s16 takes 44.1 kHz only): k_s16_to_f32, the float path, k_f32_to_s16; a full-scale run clips"""
    x16 = [s16_of(noise(2 * rate, C, seed=8 + C, amp=0.9)) for C in (1, 2)]
    for x in x16:
        x[1000:1400] = 32767
    pays = payloads_for(2, 9)
    outs = hapi.add_batch_rates(x16, pays, [rate] * 2)
    for i, (o, x) in enumerate(zip(outs, x16)):
        want, b, _, _ = add_rates_ref(x.astype(np.float32) / 32768, rate, oracle_fm(O.Key(bytes(16)), pays[i]))
        check_s16("s16 %d Hz C=%d" % (rate, x.shape[1]), o, want, b)


@gpu
def test_odd_value_offsets(hapi):
    """stereo items at odd values of a packed device buffer: rate_vec2 is off, the scalar path must give the same values"""
    torch = pytest.importorskip("torch")
    pcms = [noise(int(s * 48000), 2, seed=30 + i, amp=a) for i, (s, a) in enumerate([(1.2, 1.0), (0.4, 0.3), (2.1, 0.9)])]
    off, items = 1, []
    for p in pcms:
        items.append((off, len(p), 2))
        off += p.size + 1
    flat = np.zeros(off, np.float32)
    for (o, n, c), p in zip(items, pcms):
        flat[o:o + n * c] = p.reshape(-1)
    pays = payloads_for(len(pcms), 31)
    outs = hapi.add_batch_rates(torch.from_numpy(flat).cuda(), pays, [48000] * len(pcms), items=items)
    for i, (o, x) in enumerate(zip(outs, pcms)):
        check_item("packed 48 kHz item %d at value %d" % (i, items[i][0]), o.cpu().numpy(), x, 48000, pays[i])


@gpu
@pytest.mark.parametrize("rate", [48000, 8000])
def test_stream_offsets(hapi, rate):
    """items continuing a silent stream: offsets just past the start, a block -+ 1 (the limiter grid), and beyond 2^32 and at 2^40"""
    zs = [1, 1023, rate - 1, rate + 1, 2 * rate - 1, 2 ** 32 + 7, 2 ** 40]
    pcms = [noise(int(0.7 * rate) + 5 * i, 1 + i % 3, seed=50 + i, amp=1.0 if i % 2 else 0.4) for i in range(len(zs))]
    pays = payloads_for(len(pcms), 52)
    outs, blocks, snrs = hapi.add_batch_rates(pcms, pays, [rate] * len(pcms), zero_frames=zs, want_stats=True)
    for i, (o, x) in enumerate(zip(outs, pcms)):
        check_item("%d Hz z=%d C=%d" % (rate, zs[i], x.shape[1]), o, x, rate, pays[i], z=zs[i], snr_db=snrs[i], blocks=blocks[i])


@gpu
def test_window_cuts_limiter_block(hapi):
    """add_window whose owned range cuts a 48 kHz limiter block, and its --snr sums, against the whole stream's reference"""
    rate, n_total = 48000, 4 * 48000 + 333
    x = noise(n_total, 2, seed=60, amp=1.0)
    own0, own1 = 70000, 130001
    e0, e1 = hapi.window_range(own0, own1, n_total, sample_rate=rate)
    y, sd, ss = hapi.add_window(x[e0:e1], T.PAYLOAD, e0, n_total, own0, own1, sample_rate=rate, want_stats=True)
    fm = oracle_fm(O.Key(bytes(16)), T.PAYLOAD)
    want, b, sums, _ = add_rates_ref(x, rate, fm, snr=(own0, own1))
    chk("window [%d, %d) of 48 kHz" % (own0, own1), y[own0 - e0:own1 - e0], want[own0:own1], b[own0:own1])
    check_snr("window [%d, %d) of 48 kHz" % (own0, own1), (sd, ss), sums)


@gpu
def test_grid_stride_second_pass(ctx):
    """one call of more than 2^28 outputs: k_resample's grid (at most 2^20 CTAs of 256) covers them in a second pass of its
    grid-stride loop; checked on a strided subset, the first frames and the whole second pass"""
    torch = pytest.importorskip("torch")
    ratio = 63.9
    n_out = 2 ** 28 + 4099
    n = int(n_out / ratio) + 40
    x = noise(n, 1, seed=70)
    xd = torch.from_numpy(x).cuda()
    yd = torch.empty(n_out, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.resample(xd.data_ptr(), ratio, n_out=n_out, n_frames=n, channels=1, out=yd.data_ptr())
    ctx.synchronize()
    idx = np.unique(np.concatenate([np.arange(0, n_out, 65537), np.arange(2000), np.arange(2 ** 28 - 100, n_out)]))
    got = yd[torch.from_numpy(idx).cuda()].cpu().numpy().reshape(-1, 1)
    del yd, xd
    want, b = resample_at(x, ratio, 16, idx, n_stop=n)
    chk("2^28 + 4099 outputs", got, want, b)
