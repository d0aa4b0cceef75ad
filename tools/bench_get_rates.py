#!/usr/bin/env python
"""bench_get_rates.py -- detection of 1 h of 48 kHz stereo: the single GPU `get` against the sharded `get`, which resamples each
rank's part on its device instead of going through the host.

get_dev_ms        hostapi.get(sample_rate=48000) on the stream in HBM (float)
get_s16_ms        hostapi.get_s16(sample_rate=48000) on the stream as 16 bit host PCM
balanced_dev_ms   hostapi.balanced_get(sample_rate=48000), world 1, on the same device buffer
balanced_s16_ms   hostapi.balanced_get(sample_rate=48000), world 1, on the same 16 bit host buffer
resample_range_ms awm_resample_range alone: the whole stream to 44.1 kHz, device to device, CUDA events on the context stream

Each is the median over --steps calls after --warmup calls, host clock around calls that return a finished document.  The documents
of each input kind must be equal (exit status 1 otherwise).  Under torchrun on N > 1 GPUs every rank also holds only its
balanced_input_range of the same stream in HBM and runs the real sharded path over NCCL (sharded_dev_ms on rank 0, which checks
the document against get); with one process the multi-GPU figure is reported as not measured.  Prints one JSON line with the
card's name and power limit.

python tools/bench_get_rates.py [--minutes M] [--steps K] [--warmup W]
torchrun --nproc_per_node N tools/bench_get_rates.py ...
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle")]
RATE = 48000
PAYLOAD = "0123456789abcdef0011223344556677"


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def timed(fn, steps, warmup):
    for _ in range(warmup):
        out = fn()
    ts = []
    for _ in range(steps):
        t = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t) * 1e3)
    return round(median(ts), 3), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    import numpy as np
    import torch
    import torch.distributed as dist
    from audiowmark_b200 import capi as C, hostapi as H
    from bench_batch import gpu_card

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    H.set_params(gpu_device=local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
        H.dist_init_from_torch()

    n, ch = int(args.minutes * 60 * RATE), 2
    # uniform noise at -6 dBFS in blocks of 2^22 frames seeded by block number: every rank builds the same stream
    x = torch.empty((n, ch), device=dev, dtype=torch.float32)
    g = torch.Generator(device=dev)
    blk_frames = 1 << 22
    for b in range((n - 1) // blk_frames + 1):
        g.manual_seed(4800 + b)
        hi = min(n, (b + 1) * blk_frames)
        x[b * blk_frames:hi] = torch.rand((hi - b * blk_frames, ch), device=dev, generator=g, dtype=torch.float32) - 0.5
    y = torch.empty_like(x)
    H.add(x.data_ptr(), PAYLOAD, None, y.data_ptr(), n, ch, sample_rate=RATE)
    H.synchronize()
    del x
    torch.cuda.synchronize()
    res = {"card": gpu_card(), "workload": "get of %g min stereo at 48 kHz, marked by add" % args.minutes, "steps": args.steps,
           "warmup": args.warmup, "world": world}
    same = True

    if rank == 0:
        import awm_oracle as O
        y16 = O.quantize_sndfile16(y.cpu().numpy())
        res["get_dev_ms"], doc = timed(lambda: H.get(y.data_ptr(), n_frames=n, channels=ch, sample_rate=RATE, parse=False), args.steps, args.warmup)
        res["get_s16_ms"], doc16 = timed(lambda: H.get_s16(y16, sample_rate=RATE, parse=False), args.steps, args.warmup)
        if world == 1:
            res["balanced_dev_ms"], bdoc = timed(lambda: H.balanced_get(y.data_ptr(), 0, n, n_frames=n, channels=ch, sample_rate=RATE, parse=False),
                                                 args.steps, args.warmup)
            res["balanced_s16_ms"], bdoc16 = timed(lambda: H.balanced_get(y16, 0, n, sample_rate=RATE, parse=False), args.steps, args.warmup)
            same = bdoc == doc and bdoc16 == doc16
        res["patterns_found"] = sum(m["bits"] == PAYLOAD for m in json.loads(doc)["matches"])

        ctx = C.Context(local)
        ratio = 44100 / RATE
        n_mark = H.resample_stream_frames(n, ratio)
        out = torch.empty((n_mark, ch), device=dev, dtype=torch.float32)
        stream = torch.cuda.ExternalStream(ctx.stream, device=dev)
        ts = []
        for i in range(args.warmup + args.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ctx.resample_range(y.data_ptr(), 0, n, ratio, out.data_ptr(), 0, n_mark, in_frames=n, channels=ch)
            e1.record(stream)
            torch.cuda.synchronize()
            if i >= args.warmup:
                ts.append(e0.elapsed_time(e1))
        res["resample_range_ms"] = round(median(ts), 3)
        # the stream read once and the watermark-rate stream written once
        res["resample_range_gb_per_s"] = round((n + n_mark) * ch * 4 / (res["resample_range_ms"] * 1e-3) / 1e9, 1)
        ctx.close()

    if world > 1:
        lo, hi = H.balanced_input_range(n, rank, world, RATE)
        part = y[lo:hi].contiguous()
        torch.cuda.synchronize()
        if rank != 0:
            del y
        ms, sdoc = timed(lambda: H.balanced_get(part.data_ptr(), lo, n, n_frames=hi - lo, channels=ch, sample_rate=RATE, parse=False),
                         args.steps, args.warmup)
        if rank == 0:
            res["sharded_dev_ms"] = ms
            same = same and sdoc == doc
        dist.barrier()
    else:
        res["sharded_dev_ms"] = "not measured (one GPU)"
    if rank == 0:
        res["same_documents"] = same
        print(json.dumps(res), flush=True)
    if world > 1:
        dist.destroy_process_group()
    sys.exit(0 if same else 1)


if __name__ == "__main__":
    main()
