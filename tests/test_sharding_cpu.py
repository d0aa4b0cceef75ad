"""CPU: the multi-GPU host logic -- chunk plan, the Python plan functions against the C++ planner, embed ranges -- and the C++
merge, sort and print of per-chunk pattern records against the oracle's ResultSet."""
import struct

import numpy as np
import pytest

import awm_oracle as O
from audiowmark_b200 import hostapi as H, sharding as S

P = O.Params()


def test_chunk_plan_matches_reference_geometry():
    H.set_params()
    mx, ov = H.chunk_geometry(44100)
    assert (mx, ov) == (79380000, 5926502)                      # 30 min; lrint(2 * 51.6876 s * 1.3 * 44100)
    for n in (0, 1000, mx - 1, mx, mx + 1, 158760000, 8 * 158760000):
        want = O.chunk_ranges(n, P)
        got = S.chunk_plan(n, mx, ov)
        assert [(a, b) for a, b, _ in got] == [(a, b) for a, b, _ in want]
        assert np.allclose([t for _, _, t in got], [t for _, _, t in want], rtol=0, atol=1e-9)
    assert len(S.chunk_plan(158760000, mx, ov)) == 3           # 1 h: 1800 s, 1800 s, 268.8 s
    assert len(S.chunk_plan(8 * 158760000, mx, ov)) == 18       # 8 h (SURVEY 8e)


def test_embed_ranges_cover_rank_slices():
    """the range bench.py embeds on each rank (embed_range of the union of its slices) starts on a 1024-frame, stays inside the stream
    and carries the halo the limiter and the synthesis window need around it, for every world size the bench runs"""
    H.set_params()
    mx, ov = H.chunk_geometry(44100)
    n = 4 * 158760000
    plan = S.chunk_plan(n, mx, ov)
    for world in (1, 2, 3, 4, 8):
        for r in range(world):
            sl = S.rank_slices(plan, r, world, n)
            if not sl:
                continue
            lo, hi = min(s.lo for s in sl), max(s.hi for s in sl)
            e0, e1, ffn = S.embed_range(lo, hi, n, 44100)
            assert e0 % 1024 == 0 and ffn * 1024 == e0 and e0 <= lo and e1 >= hi and 0 <= e0 and e1 <= n
            if lo > 0:       # one complete limiter block + one frame before the first owned block
                assert e0 + 1024 <= (lo // 44100 - 1) * 44100
            if hi < n:
                assert e1 - 1024 >= ((hi - 1) // 44100 + 2) * 44100


def _records(patterns, key_index=0):
    out = b""
    for (time, quality, idx, err, bt, ty, speed, bits) in patterns:
        out += struct.pack("<iddQfBBdH", key_index, time, quality, idx, err, bt, ty, speed, len(bits)) + bytes(bits)
    return out


def test_merge_chunks_matches_oracle_resultset():
    """C++ merge/sort/print of chunk records == the oracle's ResultSet (src/wmget.cc:252-316)."""
    rng = np.random.default_rng(0)
    key = O.Key()
    payload = O.parse_payload("0123456789abcdef0011223344556677", P)
    other = [int(b) for b in rng.integers(0, 2, 128)]
    chunks, offs = [], [0.0, 1665.6122, 3331.2244]
    want = O.ResultSet()
    for c, toff in enumerate(offs):
        pats, crs = [], O.ResultSet()
        for k in range(6):
            t = 5.8 + 51.688 * k
            bits = payload if k % 3 else other
            bt = k & 1
            q = float(rng.uniform(0.3, 1.4))
            err = float(np.float32(rng.uniform(0.05, 0.4)))
            pats.append((t, q, int(t * 44100), err, bt, 0, 1.0, bits))
            crs.add_pattern(key, t, O.Score(int(t * 44100), q, bt), bits, err, O.TYPE_BLOCK)
        pats.append((0.0, 1.1, 0, 0.1, 0, 2, 1.0, payload))                       # "all"
        crs.add_pattern(key, 0.0, O.Score(0, 1.1, O.A), payload, np.float32(0.1), O.TYPE_ALL)
        # a duplicate of the previous chunk's overlap region: same block seen again with the shifted time
        if c > 0:
            t_dup = (5.8 + 51.688 * 5) + offs[c - 1] - toff
            pats.append((t_dup, 0.9, 1, 0.2, 1, 0, 1.0, payload))
            crs.add_pattern(key, t_dup, O.Score(1, 0.9, O.B), payload, np.float32(0.2), O.TYPE_BLOCK)
        chunks.append(_records(pats))
        crs.apply_time_offset(toff)
        want.merge(crs)
    want.sort([key])
    doc = H.merge_chunks(chunks, offs, 3600.0)
    wdoc = want.json_doc(3600)
    assert doc["length"] == wdoc["length"] and len(doc["matches"]) == len(wdoc["matches"])
    for g, w in zip(doc["matches"], wdoc["matches"]):
        assert (g["pos"], g["bits"], g["type"]) == (w["pos"], w["bits"], w["type"])
        assert "%.5f" % g["quality"] == w["quality"] and "%.6f" % g["error"] == w["error"] and "%.5f" % g["rating"] == w["rating"]


def test_every_start_frame_has_exactly_one_owner_up_to_8_ranks():
    """frame-balanced get: the position rule that deals candidates / blocks to ranks (index_owners) and the slices the ranks
    search (rank_slices) must agree for every world size the bench runs (1, 2, 4, 8) and for ragged stream lengths"""
    rng = np.random.default_rng(5)
    for hours, world in ((1, 1), (2, 2), (4, 4), (8, 8), (1.37, 3), (0.2, 8), (8, 5)):
        n_total = int(hours * 3600 * 44100)
        mx = int(round(30.0 * 60 * 44100))
        ov = int(round(2 * (2226 * 1024 / 44100.0) * 1.3 * 44100))
        plan = S.chunk_plan(n_total, mx, ov)
        slices = [S.rank_slices(plan, r, world, n_total) for r in range(world)]
        for c, (cs, cn, _) in enumerate(plan):
            n_starts = max(cn // S.FRAME - S.T_BLOCK - 1, 0)
            if n_starts == 0:
                assert not any(sl.chunk == c for per in slices for sl in per)
                continue
            # the owned ranges [sa, sb) of all ranks tile [0, n_starts) without gaps or overlaps
            owned = sorted((sl.sa, sl.sb, r) for r, per in enumerate(slices) for sl in per if sl.chunk == c)
            assert owned[0][0] == 0 and owned[-1][1] == n_starts
            assert all(a[1] == b[0] for a, b in zip(owned, owned[1:]))
            # ... and index_owners sends every index to the rank whose range holds its start frame
            idx = np.concatenate([rng.integers(0, cn, 200), np.array([0, cn - 1, (n_starts - 1) * S.FRAME, n_starts * S.FRAME + 5])])
            own = S.index_owners(plan, n_total, world, c, idx)
            s = np.clip(idx // S.FRAME, 0, n_starts - 1)
            for si, r in zip(s, own):
                assert any(a <= si < b and rr == r for a, b, rr in owned), (hours, world, c, int(si), int(r))
            # every slice carries the PCM its searched range [a, b) needs: b + one block + one frame, inside the chunk
            for per in slices:
                for sl in per:
                    if sl.chunk == c:
                        assert sl.lo == cs + sl.a * S.FRAME and sl.hi <= cs + cn and sl.hi >= min(cs + (sl.b + S.T_BLOCK + 1) * S.FRAME, cs + cn)


def test_cpp_plan_functions_agree_with_their_python_restatement():
    """the C++ driver of the sharded get (host/awm_balanced.cc) and bench.py's Python plan functions must cut the stream the same
    way: chunks, slices of every rank and the owner of an index, for the world sizes the bench runs and ragged lengths"""
    H.set_params()
    mx, ov = H.chunk_geometry(44100)
    rng = np.random.default_rng(6)
    for hours, world in ((1, 1), (2, 2), (4, 4), (8, 8), (1.37, 3), (0.2, 8)):
        n_total = int(hours * 3600 * 44100)
        plan = S.chunk_plan(n_total, mx, ov)
        for r in range(world):
            chunks, slices = H.balanced_plan(n_total, r, world)
            assert [(a, b) for a, b, _ in chunks] == [(a, b) for a, b, _ in plan]
            assert np.allclose([t for _, _, t in chunks], [t for _, _, t in plan], rtol=0, atol=1e-9)
            want = [(sl.chunk, sl.sa, sl.sb, sl.a, sl.b, sl.lo, sl.hi) for sl in S.rank_slices(plan, r, world, n_total)]
            assert slices == want, (hours, world, r)
        for c, (cs, cn, _) in enumerate(plan):
            idx = rng.integers(0, cn, 20)
            own = S.index_owners(plan, n_total, world, c, idx)
            assert [H.balanced_owner(n_total, world, c, int(i)) for i in idx] == [int(o) for o in own]


@pytest.mark.parametrize("frames_per_bit,short", [(2, 0), (3, 0), (2, 12), (2, 20), (1, 16)])
def test_cpp_planner_follows_the_block_length_of_the_parameters(frames_per_bit, short):
    """--frames-per-bit and --short change the block length (sync + data frames); the C++ planner of the sharded get takes it from the
    parameters: for every world size the owned start-frame ranges of the ranks tile every chunk exactly, every slice carries the PCM
    its searched range needs (one block + one frame beyond it), and the owner rule sends an index to the rank whose range holds it"""
    H.set_params(frames_per_bit=frames_per_bit)
    H.set_short_payload(short)
    try:
        T_blk = H.frames_per_block()
        if short == 0:
            assert T_blk == 85 * 6 + 858 * frames_per_bit       # 510 sync frames + one data frame group per coded bit
        rng = np.random.default_rng(7)
        for hours, world in ((1, 1), (2, 2), (3.3, 4), (8, 8), (0.4, 3)):
            n_total = int(hours * 3600 * 44100)
            per_rank = [H.balanced_plan(n_total, r, world) for r in range(world)]
            chunks = per_rank[0][0]
            for c, (cs, cn, _) in enumerate(chunks):
                n_starts = max(int(cn) // 1024 - T_blk - 1, 0)
                owned = sorted((sl[1], sl[2], r) for r, (_, sls) in enumerate(per_rank) for sl in sls if sl[0] == c)
                if n_starts == 0:
                    assert not owned
                    continue
                assert owned[0][0] == 0 and owned[-1][1] == n_starts, (frames_per_bit, short, hours, world, c)
                assert all(a[1] == b[0] for a, b in zip(owned, owned[1:]))
                for r, (_, sls) in enumerate(per_rank):
                    for chunk, sa, sb, a, b, lo, hi in sls:
                        if chunk == c:
                            assert a <= sa < sb <= b and lo == cs + a * 1024
                            assert hi <= cs + cn and hi >= min(cs + (b + T_blk + 1) * 1024, cs + cn)
                for i in rng.integers(0, int(cn), 12):
                    s = min(int(i) // 1024, n_starts - 1)
                    r = H.balanced_owner(n_total, world, c, int(i))
                    assert any(x <= s < y and rr == r for x, y, rr in owned)
    finally:
        H.set_short_payload(0)
        H.set_params()
