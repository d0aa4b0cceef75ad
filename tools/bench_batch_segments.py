#!/usr/bin/env python
"""bench_batch_segments.py -- batched embed of HLS segments at their stream offsets (hostapi.add_batch(zero_frames=...) /
awm_embed_batch_offsets, INTEGRATION §4b) against a loop of per-item hostapi.add_windowed(zero_frames=...) over the same items.

workloads  live fan-out: 1024 viewers x one 12 s stereo item (6 s segment + 3 s of context on each side) about 40 min into the
           stream, one payload per viewer;  VOD: 1 h of stereo as 600 such items at their own offsets, one payload
residency  host float32 arrays (add_windowed takes host buffers); both passes read and write host memory
timing     host wall time around each pass; the two alternate within every step
checked    the outputs of the batch and of the loop are compared bit for bit (exit status 1 if they differ)
prints     one JSON line: items/s and PCM frames/s of both, per workload, with the card's name and power limit

python tools/bench_batch_segments.py [--steps K] [--warmup W]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from bench_batch import gpu_card  # noqa: E402

RATE = 44100
SEG, CTX = 6 * RATE, 3 * RATE


def workloads(np):
    rng = np.random.default_rng(9)
    pay = lambda: "".join("%x" % v for v in rng.integers(0, 16, 32))
    # live fan-out: segment 400 (40 min in) with its context, the same audio for every viewer
    start = 400 * SEG
    item = ((rng.random((SEG + 2 * CTX, 2), dtype=np.float32) - 0.5) * 0.5).astype(np.float32)
    yield "live_1024x12s_stereo_at40min", [item] * 1024, [start - CTX] * 1024, [pay() for _ in range(1024)]
    # VOD: one hour cut into 600 segments with their context, one payload
    stream = ((rng.random((3600 * RATE, 2), dtype=np.float32) - 0.5) * 0.5).astype(np.float32)
    items, zs = [], []
    for s in range(0, stream.shape[0], SEG):
        prev, nxt = min(s, CTX), min(stream.shape[0] - s - SEG, CTX)
        items.append(stream[s - prev:s + SEG + nxt])
        zs.append(s - prev)
    p = pay()
    yield "vod_600x12s_stereo_1h", items, zs, [p] * len(items)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    from audiowmark_b200 import hostapi as H

    H.set_params()
    results = []
    for name, items, zs, payloads in workloads(np):
        out = {}

        def run_batch():
            out["batch"] = H.add_batch(items, payloads, zero_frames=zs)

        def run_loop():
            out["loop"] = [H.add_windowed(x, p, zero_frames=z)[0] for x, z, p in zip(items, zs, payloads)]

        t = {"batch": [], "loop": []}
        for step in range(args.warmup + args.steps):
            order = (("batch", run_batch), ("loop", run_loop)) if step % 2 == 0 else (("loop", run_loop), ("batch", run_batch))
            for leg, fn in order:
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if step >= args.warmup:
                    t[leg].append(dt)
        equal = all(np.array_equal(a, b) for a, b in zip(out["batch"], out["loop"]))
        frames = sum(x.shape[0] for x in items)
        tb, tl = float(np.median(t["batch"])), float(np.median(t["loop"]))
        results.append({"workload": name, "items": len(items), "pcm_frames": frames, "max_zero_frames": int(max(zs)),
                        "batch_s": tb, "loop_s": tl, "batch_items_per_s": len(items) / tb, "loop_items_per_s": len(items) / tl,
                        "batch_frames_per_s": frames / tb, "loop_frames_per_s": frames / tl, "speedup": tl / tb,
                        "batch_s_all": t["batch"], "loop_s_all": t["loop"], "outputs_equal": bool(equal)})
        out.clear()
    print(json.dumps({"metric": "batch_segments_items_per_s", "steps": args.steps, "warmup": args.warmup, "residency": "host",
                      "gpu": gpu_card(), "workloads": results}), flush=True)
    if not all(r["outputs_equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
