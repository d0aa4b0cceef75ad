#!/usr/bin/env python
"""bench_get_pipeline.py -- how busy `get` keeps the GPU: the resident `get` of bench.py's flagship input (1 h stereo 44.1 kHz,
PCM in HBM) against the sum of its kernel times.

get_ms       CUDA-event time of one `get` on the context stream, profiler off (mean over the timed steps)
kernel_ms    sum of the per-kernel CUDA-event times (awm_profile_*) of one `get`, from a separate profiled run of the same steps
idle_ms      get_ms - kernel_ms: time in which the context stream has no kernel running (copies, synchronisations, host work,
             launch latency).  Kernels of a second stream that run at the same time as those of the context stream are counted
             in full, so with overlapping streams idle_ms is a lower bound and can become negative.
idle_frac    idle_ms / get_ms
idle_vs_first_ms / idle_vs_first_frac
             get_ms - the median kernel_ms of the first directory: for builds that run the same kernels as the first one, but on
             overlapping streams, this is the time the GPU runs none of them

--dirs A [B ...] times the library built in each directory (a checkout in which __graft_entry__.build() has run), alternating
the directories round by round, each in a fresh process; the `get --json` documents of all directories are compared (exit
status 1 if they differ).  Prints one JSON line with the card's name and power limit.

python tools/bench_get_pipeline.py [--dirs DIR ...] [--rounds R] [--steps K] [--warmup W]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATE = 44100
PAYLOAD = "0123456789abcdef0011223344556677"


def worker(lib_dir, steps, warmup):
    sys.path.insert(0, lib_dir)
    import torch
    from audiowmark_b200 import hostapi as H
    n, ch = 60 * 60 * RATE, 2
    H.set_params()
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
    y = torch.empty_like(x)
    H.add(x.data_ptr(), PAYLOAD, None, y.data_ptr(), n, ch)
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(H.gpu_stream(), device=dev)

    def run(profile):
        torch.cuda.synchronize()
        if profile:
            H.profile_enable(True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        doc = None
        for _ in range(steps):
            doc = H.get(y.data_ptr(), n_frames=n, channels=ch, parse=False)
        e1.record(stream)
        torch.cuda.synchronize()
        prof = H.profile_report() if profile else None
        if profile:
            H.profile_enable(False)
        return e0.elapsed_time(e1) / steps, doc, prof

    for _ in range(warmup):
        H.get(y.data_ptr(), n_frames=n, channels=ch, parse=False)
    get_ms, doc, _ = run(False)
    prof_get_ms, _, prof = run(True)
    kernel_ms = sum(r["ms"] for r in prof.values()) / steps
    top = sorted(((r["ms"] / steps, k) for k, r in prof.items()), reverse=True)[:6]
    return {"get_ms": round(get_ms, 4), "kernel_ms": round(kernel_ms, 4), "idle_ms": round(get_ms - kernel_ms, 4),
            "idle_frac": round((get_ms - kernel_ms) / get_ms, 4), "profiled_get_ms": round(prof_get_ms, 4),
            "top_kernels_ms": {k: round(v, 4) for v, k in top},
            "doc_sha1": hashlib.sha1(doc.encode() if isinstance(doc, str) else json.dumps(doc, sort_keys=True).encode()).hexdigest()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dirs", nargs="+", default=[ROOT])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
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
    result = {"card": gpu_card(), "workload": "resident get of 1 h stereo 44.1 kHz (bench.py input, marked by add)", "steps": args.steps,
              "builds": {}}
    for d, rs in runs.items():
        gm = sorted(r["get_ms"] for r in rs)
        result["builds"][d] = {"get_ms": [r["get_ms"] for r in rs], "get_ms_median": gm[len(gm) // 2],
                               "kernel_ms": [r["kernel_ms"] for r in rs], "idle_ms": [r["idle_ms"] for r in rs],
                               "idle_frac": [r["idle_frac"] for r in rs], "profiled_get_ms": [r["profiled_get_ms"] for r in rs],
                               "top_kernels_ms": rs[-1]["top_kernels_ms"], "doc_sha1": rs[-1]["doc_sha1"]}
    km = sorted(r["kernel_ms"] for r in runs[dirs[0]])
    ref_kernel_ms = km[len(km) // 2]
    for d, rs in runs.items():
        result["builds"][d]["idle_vs_first_ms"] = [round(r["get_ms"] - ref_kernel_ms, 4) for r in rs]
        result["builds"][d]["idle_vs_first_frac"] = [round((r["get_ms"] - ref_kernel_ms) / r["get_ms"], 4) for r in rs]
    shas = {r["doc_sha1"] for rs in runs.values() for r in rs}
    result["same_documents"] = len(shas) == 1
    print(json.dumps(result), flush=True)
    sys.exit(0 if len(shas) == 1 else 1)


if __name__ == "__main__":
    main()
