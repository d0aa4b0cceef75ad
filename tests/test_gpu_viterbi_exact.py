"""k_viterbi against the oracle's conv_decode_soft (orc_viterbi, exact float32): decoded bits identical and the error metric
bit-equal, for every block type, soft and hard, from clean to heavily corrupted words.

The kernel skips the trellis words that cannot matter at both ends of the trellis (states not yet reachable from state 0,
states that can no longer reach it); message lengths below 15 bits make the two ends overlap.  Hard input produces many exact
ties between the two candidates of a state, which the strict '<' rule must break as the reference does.

A state's new metric is summed once, from the better predecessor; both candidates are summed and compared only when the two
predecessors are close enough for the rounding of the sums to merge them.  Soft words whose bits are +-1 with a tiny jitter make
the competing path metrics differ by a few ulps again and again, so that comparison runs in almost every step."""
import numpy as np
import pytest

import awm_oracle as O
from audiowmark_b200 import capi

pytestmark = pytest.mark.gpu

TYPES = ((O.A, capi.BLOCK_A), (O.B, capi.BLOCK_B), (O.AB, capi.BLOCK_AB))
NOISE = (0.0, 0.6, 1.5, 4.0)
SHORT_LENGTHS = sorted(n for n, _ in O.SHORT_CODES.values())          # conv message lengths of --short 12 / 16 / 20


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def words(bt, n_msg, rng, noise_levels=NOISE):
    """one received word per noise level: +-1 for the coded bits plus Gaussian noise"""
    msg = [int(b) for b in rng.integers(0, 2, n_msg)]
    coded = np.array(O.conv_encode(bt, msg), np.float32)
    return msg, [((coded * 2 - 1) + s * rng.standard_normal(len(coded))).astype(np.float32) for s in noise_levels]


def check(bits, err, jobs, types, n_msg, hard):
    P = O.Params(hard=hard)
    for j, (raw, bt) in enumerate(zip(jobs, types)):
        wb, we = O.conv_decode_soft(bt, O.normalize_soft_bits(raw, P))
        assert list(bits[j]) == wb, (bt, n_msg, hard, j)
        assert np.float32(err[j]).tobytes() == np.float32(we).tobytes(), (bt, n_msg, hard, j, float(err[j]), we)


@pytest.mark.parametrize("n_msg", [128] + SHORT_LENGTHS + [1, 6, 14, 15, 20])
@pytest.mark.parametrize("hard", [False, True])
def test_viterbi_exact(ctx, n_msg, hard):
    rng = np.random.default_rng(1000 + n_msg)
    for bt, cbt in TYPES:
        msg, jobs = words(bt, n_msg, rng)
        bits, err = ctx.viterbi(jobs, [cbt] * len(jobs), n_msg_bits=n_msg, hard=hard)
        check(bits, err, jobs, [bt] * len(jobs), n_msg, hard)
        assert list(bits[0]) == msg


@pytest.mark.parametrize("hard", [False, True])
def test_viterbi_exact_mixed_split_and_silence(ctx, hard):
    """mixed block types in one call, more jobs than one launch takes (512), and all-zero words (digital silence)"""
    n_msg = 10
    rng = np.random.default_rng(7)
    jobs, types, ctypes_ = [], [], []
    for i in range(530):
        bt, cbt = TYPES[i % 3]
        if i in (3, 517):
            raw = np.zeros(O.conv_code_size(bt, n_msg), np.float32)
        else:
            _, (raw,) = words(bt, n_msg, rng, (NOISE[i % len(NOISE)],))
        jobs.append(raw)
        types.append(bt)
        ctypes_.append(cbt)
    bits, err = ctx.viterbi(jobs, ctypes_, n_msg_bits=n_msg, hard=hard)
    check(bits, err, jobs, types, n_msg, hard)
    if not hard:
        for i in (3, 517):
            assert not bits[i].any() and err[i] == np.float32(-1.0 / len(jobs[i])), (i, err[i])


@pytest.mark.parametrize("jitter", [2.0 ** -22, 2.0 ** -16, 2.0 ** -10])
@pytest.mark.parametrize("n_msg", [128, 14])
def test_viterbi_exact_near_ties(ctx, jitter, n_msg):
    """soft words of +-1 with bit errors and a relative jitter of a few ulps: near-ties between the two candidates everywhere"""
    rng = np.random.default_rng(int(n_msg + 1 / jitter))
    for bt, cbt in TYPES:
        jobs = []
        for flip in (0.0, 0.05, 0.2, 0.4):
            msg = [int(b) for b in rng.integers(0, 2, n_msg)]
            coded = np.array(O.conv_encode(bt, msg), np.float32) * 2 - 1
            sign = np.where(rng.random(len(coded)) < flip, -1.0, 1.0)
            jobs.append((coded * sign * (1 + jitter * rng.standard_normal(len(coded)))).astype(np.float32))
        bits, err = ctx.viterbi(jobs, [cbt] * len(jobs), n_msg_bits=n_msg)
        check(bits, err, jobs, [bt] * len(jobs), n_msg, False)


# An A word of 2 message bits (soft bits +-1, half of them flipped, jitter 2^-20) on which the two candidates of a state on the
# decoded path are summed from predecessors that differ, and round to the same metric: the reference keeps ps0 there, so taking
# the smaller predecessor without comparing the sums decodes [1, 1] instead of [1, 0].
MERGED_TIE_A2 = np.array([
    0x3f7fffdd, 0x3f800004, 0xbf800002, 0xbf7ffff7, 0x3f800003, 0xbf800001, 0xbf7ffffe, 0xbf7fffe6,
    0xbf7ffffc, 0xbf7ffff6, 0xbf7ffff5, 0x3f7ffff1, 0xbf7ffffb, 0xbf800000, 0xbf800008, 0xbf7fffef,
    0x3f7fffe6, 0xbf800006, 0xbf7ffff9, 0xbf7ffffe, 0x3f80000c, 0x3f800000, 0x3f7ffffd, 0xbf7ffffc,
    0xbf7ffffb, 0xbf80000b, 0x3f7ffff1, 0x3f80000d, 0xbf7fffea, 0x3f7fffff, 0xbf7fffed, 0x3f800003,
    0x3f7ffff4, 0xbf800008, 0x3f800013, 0x3f80000e, 0x3f7ffff4, 0x3f80000b, 0x3f800007, 0xbf7ffffa,
    0x3f800006, 0x3f7ffff3, 0x3f800002, 0xbf800007, 0xbf7ffff9, 0x3f7ffffd, 0xbf800007, 0x3f800004,
    0xbf800003, 0x3f800001, 0xbf7ffffc, 0x3f7ffffb, 0xbf7ffffe, 0x3f800002, 0x3f800006, 0x3f7ffff1,
    0xbf7ffff9, 0xbf7fffd7, 0x3f7ffff8, 0x3f7fffe7, 0xbf800004, 0x3f7ffffd, 0xbf7fffff, 0xbf7ffffa,
    0xbf7ffff1, 0xbf7ffffb, 0xbf7ffffd, 0x3f7fffef, 0xbf800003, 0x3f800007, 0xbf800006, 0x3f800000,
    0xbf7fffe4, 0x3f7ffffb, 0x3f7ffff3, 0xbf7ffffe, 0x3f800004, 0xbf7ffff9, 0xbf7fffff, 0xbf800007,
    0x3f800001, 0x3f7fffe3, 0x3f7ffff8, 0x3f7ffffe, 0x3f7ffff0, 0xbf7ffff4, 0x3f800002, 0x3f800000,
    0x3f7ffffb, 0xbf80000e, 0x3f800002, 0x3f800010, 0xbf800003, 0xbf7ffff2, 0xbf800005, 0xbf7fffe9,
    0x3f80000f, 0x3f800009, 0x3f80000e, 0xbf7ffff2, 0xbf800002, 0xbf7fffeb,
], np.uint32).view(np.float32)


def test_viterbi_exact_merged_tie(ctx):
    bits, err = ctx.viterbi([MERGED_TIE_A2], [capi.BLOCK_A], n_msg_bits=2)
    check(bits, err, [MERGED_TIE_A2], [O.A], 2, False)
    assert list(bits[0]) == [1, 0]
