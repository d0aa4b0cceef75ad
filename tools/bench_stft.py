#!/usr/bin/env python
"""bench_stft.py -- k_stft_mags_tc, the sync search's spectrogram + entry-sum kernel, timed on its own.

Input: one 30-minute chunk of stereo 44.1 kHz noise in HBM (the chunk length `get` searches at a time), bench.py's noise generator,
the default key's block-mode sync tables.  Each step is one awm_sync_approx (k_stft_mags_tc, then the gather, quality and local
mean kernels); the per-kernel CUDA events of the library (awm_profile_*) give k_stft_mags_tc's time per launch over all timed steps.

--dirs A [B ...] times the library built in each directory (a checkout in which __graft_entry__.build() has run), alternating
the directories round by round, each in a fresh process.  The approx scores of the last step (index, raw quality, local mean of
every start position and shift) are hashed; exit status 1 if the directories disagree.  Prints one JSON line with the card's name
and power limit, read in the same run.

python tools/bench_stft.py [--dirs DIR ...] [--rounds R] [--steps K] [--warmup W]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATE = 44100
CHUNK_MINUTES = 30


def worker(lib_dir, steps, warmup):
    # the oracle (sync tables) from this checkout, the library under test from lib_dir
    for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests"), lib_dir):
        sys.path.insert(0, p)
    import numpy as np
    import torch
    import awm_oracle as O
    import awm_testlib as T
    from audiowmark_b200 import capi

    n, ch = CHUNK_MINUTES * 60 * RATE, 2
    dev = torch.device("cuda", 0)
    # bench.py's input: uniform noise at -6 dBFS in blocks of 2^22 frames seeded by block number
    blk_frames = 1 << 22
    x = torch.empty((n, ch), device=dev, dtype=torch.float32)
    g = torch.Generator(device=dev)
    for b in range((n - 1) // blk_frames + 1):
        g.manual_seed(1234 + b)
        blk = torch.rand((blk_frames, ch), device=dev, generator=g, dtype=torch.float32) - 0.5
        hi = min(n, (b + 1) * blk_frames)
        x[b * blk_frames:hi] = blk[:hi - b * blk_frames]
    del blk
    torch.cuda.synchronize()
    ctx = capi.Context(0)
    T.setup_ctx(ctx, O.Key(), O.Params())
    ctx.pcm_bind(x.data_ptr(), n_frames=n, channels=ch)
    for _ in range(warmup):
        ctx.sync_approx_run(0, capi.MODE_BLOCK)
    ctx.synchronize()
    ctx.profile_enable(True)
    for _ in range(steps):
        ctx.sync_approx_run(0, capi.MODE_BLOCK)
    prof = ctx.profile_report()
    ctx.profile_enable(False)
    k = prof["k_stft_mags_tc"]
    scores = ctx.sync_approx(0, capi.MODE_BLOCK)
    ctx.close()
    return {"stft_ms": round(k["ms"] / k["launches"], 4), "launches": k["launches"],
            "scores_sha1": hashlib.sha1(np.ascontiguousarray(scores).tobytes()).hexdigest(), "n_scores": int(len(scores))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dirs", nargs="+", default=[ROOT])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--worker", metavar="DIR", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        print(json.dumps(worker(os.path.abspath(args.worker), args.steps, args.warmup)), flush=True)
        return
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_batch import gpu_card
    dirs = [os.path.abspath(d) for d in args.dirs]
    runs = {d: [] for d in dirs}
    for _ in range(args.rounds):
        for d in dirs:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", d, "--steps", str(args.steps), "--warmup", str(args.warmup)],
                                 check=True, capture_output=True, text=True).stdout
            runs[d].append(json.loads(out.strip().splitlines()[-1]))
    result = {"card": gpu_card(), "workload": "awm_sync_approx on 30 min of stereo 44.1 kHz noise in HBM, block mode", "steps": args.steps,
              "builds": {}}
    for d, rs in runs.items():
        ms = sorted(r["stft_ms"] for r in rs)
        result["builds"][d] = {"stft_ms": [r["stft_ms"] for r in rs], "stft_ms_median": ms[len(ms) // 2],
                               "launches": rs[-1]["launches"], "n_scores": rs[-1]["n_scores"], "scores_sha1": rs[-1]["scores_sha1"]}
    shas = {r["scores_sha1"] for rs in runs.values() for r in rs}
    result["same_scores"] = len(shas) == 1
    print(json.dumps(result), flush=True)
    sys.exit(0 if len(shas) == 1 else 1)


if __name__ == "__main__":
    main()
