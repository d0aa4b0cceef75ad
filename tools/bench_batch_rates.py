#!/usr/bin/env python
"""bench_batch_rates.py -- batched embed of many items, each at its own sample rate with its own payload (hostapi.add_batch_rates /
awm_embed_batch_rates, INTEGRATION §4b), against a loop of per-item hostapi.add(..., sample_rate=r) over the same items.

workloads  1024 x 10 s mono at 48 kHz (short clips: per-call overhead), 128 x 3 min stereo at 48 kHz (long clips: bandwidth, several
           scratch waves), 384 x 30 s stereo split evenly over 32 / 44.1 / 48 kHz (a mixed-rate library), 1 x 60 min stereo at 48 kHz
           (one long soundtrack: the single `add` is a one-item batch, so loop and batch run the same path); uniform noise at -6 dBFS,
           a random payload per item
residency  PCM resident in HBM (one packed float32 tensor; the loop passes device pointers into it)
timing     host wall time around each pass; both passes end in a synchronise; the two alternate within every step
checked    the outputs of the batch and of the loop are compared bit for bit (exit status 1 if they differ)
prints     one JSON line: items/s and PCM frames/s of both, per workload, with the card's name and power limit

python tools/bench_batch_rates.py [--steps K] [--warmup W]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batch import gpu_card  # noqa: E402

WORKLOADS = [("1024x10s_mono_48k", 1024, 10.0, 1, (48000,)),
             ("128x3min_stereo_48k", 128, 180.0, 2, (48000,)),
             ("384x30s_stereo_32k_44k_48k", 384, 30.0, 2, (32000, 44100, 48000)),
             ("1x60min_stereo_48k", 1, 3600.0, 2, (48000,))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    import torch
    from audiowmark_b200 import hostapi as H

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    H.set_params()
    rng = np.random.default_rng(7)
    results = []
    for name, n_items, seconds, ch, rate_set in WORKLOADS:
        rates = [rate_set[i * len(rate_set) // n_items] for i in range(n_items)]      # even split, in runs of one rate
        items, off = [], 0
        for r in rates:
            n = int(seconds * r)
            items.append((off, n, ch))
            off += n * ch
        payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in range(n_items)]
        g = torch.Generator(device=dev)
        g.manual_seed(4321)
        x = torch.rand(off, device=dev, generator=g, dtype=torch.float32) - 0.5
        y_batch, y_loop = torch.empty_like(x), torch.empty_like(x)
        torch.cuda.synchronize()
        es = x.element_size()

        def run_batch():
            H.add_batch_rates(x, payloads, rates, items=items, out=y_batch)

        def run_loop():
            for (o, nf, c), p, r in zip(items, payloads, rates):
                H.add(x.data_ptr() + o * es, p, None, y_loop.data_ptr() + o * es, nf, c, sample_rate=r)
            H.synchronize()

        t = {"batch": [], "loop": []}
        for step in range(args.warmup + args.steps):
            order = (("batch", run_batch), ("loop", run_loop)) if step % 2 == 0 else (("loop", run_loop), ("batch", run_batch))
            for leg, fn in order:
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if step >= args.warmup:
                    t[leg].append(dt)
        equal = bool(torch.equal(y_batch, y_loop))
        frames = sum(n for _, n, _ in items)
        tb, tl = float(np.median(t["batch"])), float(np.median(t["loop"]))
        results.append({"workload": name, "items": n_items, "seconds_per_item": seconds, "channels": ch, "rates": list(rate_set),
                        "pcm_frames": frames, "batch_s": tb, "loop_s": tl, "batch_items_per_s": n_items / tb, "loop_items_per_s": n_items / tl,
                        "batch_frames_per_s": frames / tb, "loop_frames_per_s": frames / tl, "speedup": tl / tb,
                        "batch_s_all": t["batch"], "loop_s_all": t["loop"], "outputs_equal": equal})
        del x, y_batch, y_loop
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "batch_rates_embed_items_per_s", "steps": args.steps, "warmup": args.warmup, "residency": "device",
                      "gpu": gpu_card(), "workloads": results}), flush=True)
    if not all(r["outputs_equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
