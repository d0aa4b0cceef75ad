#!/usr/bin/env python
"""bench_viterbi.py -- the Viterbi decoder (awm_viterbi, kernel k_viterbi) on the job mix of bench.py's `get`: about 108 code
words of 128 message bits per call, 37 A, 37 B and 34 AB words, soft decoding.  The words are seeded noisy encodings of random
messages; one call decodes all of them in one launch, as `get` does after its last chunk.

kernel_ms    CUDA-event time of k_viterbi per call (awm_profile_*: events recorded around the launch on the context stream)
call_ms      host time of one awm_viterbi call (uploads, launch, downloads; the call ends in a stream synchronise), profiler off

--dirs A [B ...] times the library built in each directory (a checkout in which __graft_entry__.build() has run), alternating
the directories round by round, each in a fresh process; the decoded bits and errors of all directories are compared (exit
status 1 if they differ).  Prints one JSON line with the card's name and power limit.

python tools/bench_viterbi.py [--dirs DIR ...] [--rounds R] [--calls K] [--warmup W]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_MSG = 128
MIX = (37, 37, 34)            # A, B, AB words per call


def worker(lib_dir, calls, warmup):
    sys.path.insert(0, lib_dir)
    sys.path.insert(0, os.path.join(lib_dir, "oracle"))
    import numpy as np
    import awm_oracle as O
    from audiowmark_b200 import capi
    rng = np.random.default_rng(2024)
    jobs, types = [], []
    for bt, cbt, count in ((O.A, capi.BLOCK_A, MIX[0]), (O.B, capi.BLOCK_B, MIX[1]), (O.AB, capi.BLOCK_AB, MIX[2])):
        for _ in range(count):
            msg = [int(b) for b in rng.integers(0, 2, N_MSG)]
            coded = np.array(O.conv_encode(bt, msg), np.float32)
            jobs.append(((coded * 2 - 1) + rng.uniform(0.3, 1.5) * rng.standard_normal(len(coded))).astype(np.float32))
            types.append(cbt)
    ctx = capi.Context(0)
    for _ in range(warmup):
        ctx.viterbi(jobs, types, N_MSG)
    t0 = time.perf_counter()
    for _ in range(calls):
        bits, err = ctx.viterbi(jobs, types, N_MSG)
    call_ms = (time.perf_counter() - t0) * 1e3 / calls
    ctx.profile_enable(True)
    for _ in range(calls):
        ctx.viterbi(jobs, types, N_MSG)
    ctx.synchronize()
    prof = ctx.profile_report()
    ctx.profile_enable(False)
    ctx.close()
    kernel_ms = prof["k_viterbi"]["ms"] / calls
    digest = hashlib.sha1(bits.tobytes() + err.tobytes()).hexdigest()
    return {"kernel_ms": round(kernel_ms, 4), "call_ms": round(call_ms, 4), "sha1": digest}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dirs", nargs="+", default=[ROOT])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--worker", metavar="DIR", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        print(json.dumps(worker(os.path.abspath(args.worker), args.calls, args.warmup)), flush=True)
        return
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_batch import gpu_card
    dirs = [os.path.abspath(d) for d in args.dirs]
    runs = {d: [] for d in dirs}
    for _ in range(args.rounds):
        for d in dirs:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", d, "--calls", str(args.calls), "--warmup", str(args.warmup)],
                                 check=True, capture_output=True, text=True).stdout
            runs[d].append(json.loads(out.strip().splitlines()[-1]))
    result = {"card": gpu_card(), "workload": "awm_viterbi, %d A + %d B + %d AB words of %d bits, soft" % (MIX + (N_MSG,)), "calls": args.calls,
              "builds": {}}
    for d, rs in runs.items():
        km = sorted(r["kernel_ms"] for r in rs)
        result["builds"][d] = {"kernel_ms": [r["kernel_ms"] for r in rs], "kernel_ms_median": km[len(km) // 2],
                               "call_ms": [r["call_ms"] for r in rs], "sha1": rs[-1]["sha1"]}
    shas = {r["sha1"] for rs in runs.values() for r in rs}
    result["same_results"] = len(shas) == 1
    print(json.dumps(result), flush=True)
    sys.exit(0 if len(shas) == 1 else 1)


if __name__ == "__main__":
    main()
