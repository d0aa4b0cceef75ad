"""GPU: sharded runs reproduce the single-process result exactly (simulated ranks on one GPU whose exchanges run in lock step in
one process; the ncclAllGather exchange of real ranks runs in bench.py)."""
import json

import numpy as np
import pytest

import awm_oracle as O
import awm_testlib as T
from audiowmark_b200 import hostapi as H, sharding as S

pytestmark = pytest.mark.gpu


def test_sharded_embed_is_bit_identical():
    x = T.noise(130.0, 2, seed=21, amp=1.0)                 # full-scale noise: the limiter works on every block
    H.set_params()
    full = H.add(x, T.PAYLOAD)
    n = x.shape[0]
    for cuts in ([0, n // 2, n], [0, 1234567, 2999999, n], [0, 44100 * 50, 44100 * 51, n]):
        for lo, hi in zip(cuts, cuts[1:]):
            e0, e1, ffn = S.embed_range(lo, hi, n, 44100)
            part = H.add(x[e0:e1], T.PAYLOAD, first_frame_number=ffn)
            assert np.array_equal(part[lo - e0:hi - e0], full[lo:hi]), (lo, hi, e0, e1)


def test_pipelined_host_paths_equal_device_paths():
    """awm_embed splits long HOST buffers into pieces to overlap H2D / kernels / D2H, and `get` stages its whole input piece by piece
    (awm_pcm_stage) and binds each chunk's slice once its pieces have arrived: both must give exactly what the one-shot device-pointer
    path gives."""
    torch = pytest.importorskip("torch")
    x = T.noise(600.0, 2, seed=23, amp=1.0)                 # 10 min: three pieces of 12288 frames, limiter active
    H.set_params(chunk_size_min=4.0)
    xd = torch.from_numpy(x).cuda()
    yd = torch.empty_like(xd)
    torch.cuda.synchronize()                                # the context has its own (non-blocking) stream
    H.add(xd.data_ptr(), T.PAYLOAD, None, yd.data_ptr(), x.shape[0], 2)
    H.synchronize()                                         # device-pointer calls are asynchronous
    want = yd.cpu().numpy()
    xp = torch.from_numpy(x).pin_memory()
    yp = torch.empty_like(xp).pin_memory()
    H.add(xp.numpy(), T.PAYLOAD, None, yp.numpy())
    assert np.array_equal(yp.numpy(), want)
    assert np.array_equal(H.add(x, T.PAYLOAD), want)        # pageable host memory
    doc_dev = H.get(yd.data_ptr(), n_frames=x.shape[0], channels=2)
    assert H.get(yp.numpy()) == doc_dev
    assert H.get(want) == doc_dev
    H.set_params()



def test_host_gets_back_to_back_read_only_their_own_upload():
    """two host `get`s in a row on one context, the second on a shorter buffer, each over several chunks: every upload replaces the
    staged stream (16 bit pieces are converted again), so each document equals the device-pointer `get` of the same audio"""
    torch = pytest.importorskip("torch")
    H.set_params(chunk_size_min=4.0)
    try:
        audio = [O.quantize_sndfile16(H.add(T.noise(seconds, 2, seed=seed), T.PAYLOAD)) for seconds, seed in ((600.0, 31), (380.0, 32))]
        want = []
        for y16 in audio:
            yd = torch.from_numpy(O.int16_to_float(y16)).cuda()
            torch.cuda.synchronize()
            want.append(H.get(yd.data_ptr(), n_frames=y16.shape[0], channels=2))
            assert any(m["bits"] == T.PAYLOAD for m in want[-1]["matches"])
        assert [H.get(O.int16_to_float(y16)) for y16 in audio] == want
        assert [H.get_s16(y16) for y16 in audio] == want
    finally:
        H.set_params()


def test_try_speed_on_host_input_equals_device_input():
    """--try-speed on host float and 16 bit input searches the staged device copy of each chunk, over several chunks and on a clip
    short enough for the clip decoder, after which the chunk is bound again (here once per key): the documents equal the
    device-input one"""
    torch = pytest.importorskip("torch")
    H.set_params(chunk_size_min=4.0)
    H.set_speed_params(try_speed=T.cli_float(1.01))
    try:
        for seconds, keys in ((600.0, None), (100.0, [bytes(16), bytes(range(1, 17))])):
            y = H.add(T.noise(seconds, 2, seed=33), T.PAYLOAD)
            y16 = O.quantize_sndfile16(H.resample(y, 1 / T.cli_float(1.01)))
            yf = O.int16_to_float(y16)
            yd = torch.from_numpy(yf).cuda()
            torch.cuda.synchronize()
            want = H.get(yd.data_ptr(), keys=keys, n_frames=yf.shape[0], channels=2)
            assert any(m["bits"] == T.PAYLOAD for m in want["matches"]), seconds
            assert H.get(yf, keys=keys) == want
            assert H.get_s16(y16, keys=keys) == want
    finally:
        H.set_speed_params()
        H.set_params()

@pytest.mark.parametrize("world", [1, 2, 3])
def test_frame_balanced_get_equals_single_process(world):
    """every rank searches an equal share of the start frames of every chunk; per-chunk decisions are taken on the
    gathered lists -- the merged result must be the single-process one, digit for digit.  The C++ driver
    (host/awm_balanced.cc) runs here stage by stage, the exchanges are simulated in lock step (the product path uses
    ncclAllGather; bench.py checks that one on real ranks)."""
    x = T.noise(700.0, 2, seed=22)
    H.set_params(chunk_size_min=4.0)
    y = H.add(x, T.PAYLOAD)
    doc = H.get(y)
    n = y.shape[0]
    torch = pytest.importorskip("torch")
    ranks, keep = [], []
    for r in range(world):
        _, slices = H.balanced_plan(n, r, world)
        lo, hi = min(s[5] for s in slices), max(s[6] for s in slices)
        part = torch.from_numpy(np.ascontiguousarray(y[lo:hi])).cuda()      # every simulated rank holds its own device copy
        keep.append(part)
        torch.cuda.synchronize()
        ranks.append(H.BalancedStages(r, world, n, part.data_ptr(), hi - lo, 2, lo))
    try:
        pay = [rk.stage(0) for rk in ranks]                          # peaks
        retry = [rk.stage(1, pay) for rk in ranks]                   # select
        assert all(rt == retry[0] for rt in retry)
        if retry[0]:
            pay = [rk.stage(2, [retry[0]]) for rk in ranks]
            assert all(rk.stage(1, pay) == b"" for rk in ranks)
        pay = [rk.stage(3) for rk in ranks]                          # refine + soft bits
        pay = [rk.stage(4, pay) for rk in ranks]                     # viterbi (the sharers of a chunk deal its jobs out among themselves)
        docs = [json.loads(rk.stage(5, pay).decode()) for rk in ranks]
        assert all(d == doc for d in docs)
    finally:
        for rk in ranks:
            rk.close()
        H.set_params()


def test_balanced_get_entry_point_single_rank():
    """hostapi.balanced_get without a communicator is a world of one: same document as hostapi.get, for float and 16 bit PCM"""
    x = T.noise(300.0, 2, seed=24)
    H.set_params(chunk_size_min=4.0)
    try:
        y = H.add(x, T.PAYLOAD)
        assert H.balanced_get(y, 0, y.shape[0]) == H.get(y)
        import awm_oracle as O
        y16 = O.quantize_sndfile16(y)
        assert H.balanced_get(y16, 0, y16.shape[0]) == H.get_s16(y16)
    finally:
        H.set_params()


@pytest.mark.parametrize("short,frames_per_bit", [(16, 2), (0, 3)])
def test_balanced_get_with_other_block_lengths(short, frames_per_bit):
    """--short / --frames-per-bit change the block length; the sharded driver takes it from the parameters (host/awm_balanced.cc:
    frames_per_block): same document as the single GPU get, three simulated ranks"""
    payload = "beef" if short else T.PAYLOAD
    H.set_params(chunk_size_min=4.0, frames_per_bit=frames_per_bit)
    H.set_short_payload(short)
    torch = pytest.importorskip("torch")
    ranks, keep = [], []
    try:
        y = H.add(T.noise(500.0, 2, seed=26), payload)
        doc = H.get(y)
        assert sum(m["bits"] == payload for m in doc["matches"]) >= 3
        n, world = y.shape[0], 3
        for r in range(world):
            _, slices = H.balanced_plan(n, r, world)
            lo, hi = min(s[5] for s in slices), max(s[6] for s in slices)
            part = torch.from_numpy(np.ascontiguousarray(y[lo:hi])).cuda()
            keep.append(part)
            torch.cuda.synchronize()
            ranks.append(H.BalancedStages(r, world, n, part.data_ptr(), hi - lo, 2, lo))
        pay = [rk.stage(0) for rk in ranks]
        retry = [rk.stage(1, pay) for rk in ranks]
        assert all(rt == retry[0] for rt in retry)
        if retry[0]:
            pay = [rk.stage(2, [retry[0]]) for rk in ranks]
            assert all(rk.stage(1, pay) == b"" for rk in ranks)
        pay = [rk.stage(3) for rk in ranks]
        pay = [rk.stage(4, pay) for rk in ranks]
        assert json.loads(ranks[0].stage(5, pay).decode()) == doc
    finally:
        for rk in ranks:
            rk.close()
        H.set_short_payload(0)
        H.set_params()


def test_balanced_get_refuses_clip_sized_input():
    """inputs under 3.1 blocks go through the reference's ClipDecoder (src/wmget.cc:764-884), which the sharded driver does not run:
    it must refuse them loudly instead of returning a document without CLIP patterns"""
    y = T.noise(100.0, 2, seed=25)
    with pytest.raises(RuntimeError):
        H.balanced_get(y, 0, y.shape[0])
    assert any(m["type"].startswith("CLIP") for m in H.get(H.add(y, T.PAYLOAD))["matches"])    # the single GPU get does run it


@pytest.mark.parametrize("limiter", [True, False])
def test_streaming_add_equals_whole_stream_add(limiter):
    """`audiowmark add` reads, embeds and writes window by window (bounded memory, first output long before EOF; reference loop
    src/wmadd.cc:520-589): identical bits, the same "Data Blocks" and --snr figures as embedding the whole stream at once, for
    windows that are whole blocks, ragged, and shorter than a limiter block"""
    x = T.noise(130.0, 2, seed=31, amp=1.0)
    H.set_params(test_no_limiter=not limiter)
    try:
        whole, blocks, snr = H.add(x, T.PAYLOAD, want_stats=True)
        for window in (0, 1000, 37, 3):
            out, wblocks, wsnr = H.add_windowed(x, T.PAYLOAD, window_frames=window)
            assert np.array_equal(out, whole), window
            assert wblocks == blocks and abs(wsnr - snr) < 1e-9, (window, wblocks, blocks, wsnr, snr)
    finally:
        H.set_params()


def test_streaming_add_with_stream_offset():
    """zero_frames (HLS segments, src/wmadd.cc:504-519): the input continues a stream that began with that much silence -- the result is
    what embedding silence + input gives, minus the silent part"""
    x = T.noise(70.0, 2, seed=32)
    H.set_params()
    for zero_frames in (1024 * 300, 1024 * 300 + 517, 100):
        full = H.add(np.concatenate([np.zeros((zero_frames, 2), np.float32), x]), T.PAYLOAD)
        out, _, _ = H.add_windowed(x, T.PAYLOAD, zero_frames=zero_frames, window_frames=500)
        assert np.array_equal(out, full[zero_frames:]), zero_frames
