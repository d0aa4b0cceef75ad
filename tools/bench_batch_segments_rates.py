#!/usr/bin/env python
"""bench_batch_segments_rates.py -- batched embed of 48 kHz HLS segments at their stream offsets (hostapi.add_batch_rates(
zero_frames=...) / awm_embed_batch_rates_offsets, INTEGRATION §4b).

workloads  live fan-out: 1024 viewers x one 12 s stereo item (6 s segment + 3 s of context on each side) 40 min into a 48 kHz
           stream, one payload per viewer, against a per-viewer baseline that materialises the silent prefix (add_batch_rates of
           zeros (z) ++ item, one call per viewer): that baseline is timed on --baseline-items viewers only and its figure for
           1024 viewers is an EXTRAPOLATION (labelled so in the output);
           VOD: 1 h of 48 kHz stereo as 600 such items at their own offsets, one payload, against one whole-stream
           add(sample_rate=48000)
residency  host float32 arrays; every pass reads and writes host memory
timing     host wall time around each pass; batch and baseline alternate within every step
checked    live: the baseline items equal the batch's bit for bit; VOD: the trimmed segments equal the whole-stream add (exit status 1
           if either differs)
prints     one JSON line: seconds and items/s per workload, with the card's name and power limit

python tools/bench_batch_segments_rates.py [--steps K] [--warmup W] [--baseline-items N]
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

RATE = 48000
SEG, CTX = 6 * RATE, 3 * RATE


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--baseline-items", type=int, default=2)
    args = ap.parse_args()

    import numpy as np
    from audiowmark_b200 import hostapi as H

    H.set_params()
    rng = np.random.default_rng(9)
    pay = lambda: "".join("%x" % v for v in rng.integers(0, 16, 32))
    results = []

    def timed(legs):
        t = {k: [] for k in legs}
        for step in range(args.warmup + args.steps):
            order = list(legs.items()) if step % 2 == 0 else list(legs.items())[::-1]
            for leg, fn in order:
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if step >= args.warmup:
                    t[leg].append(dt)
        return t

    # live fan-out: segment 400 (40 min in) with its context, the same audio for every viewer
    z = 400 * SEG - CTX
    item = ((rng.random((SEG + 2 * CTX, 2), dtype=np.float32) - 0.5) * 0.5).astype(np.float32)
    viewers = [pay() for _ in range(1024)]
    nb = max(1, min(args.baseline_items, len(viewers)))
    ext = np.concatenate([np.zeros((z, 2), np.float32), item])
    out = {}

    def live_batch():
        out["batch"] = H.add_batch_rates([item] * len(viewers), viewers, [RATE] * len(viewers), zero_frames=[z] * len(viewers))

    def live_baseline():
        out["base"] = [H.add_batch_rates([ext], [p], [RATE])[0][z:] for p in viewers[:nb]]

    t = timed({"batch": live_batch, "baseline": live_baseline})
    tb, tl = float(np.median(t["batch"])), float(np.median(t["baseline"]))
    equal = all(np.array_equal(a, b) for a, b in zip(out["batch"][:nb], out["base"]))
    results.append({"workload": "live_1024x12s_stereo_48k_at40min", "items": len(viewers), "zero_frames": z, "batch_s": tb,
                    "batch_items_per_s": len(viewers) / tb, "baseline_items_timed": nb, "baseline_s_for_timed_items": tl,
                    "baseline_s_for_1024_items_EXTRAPOLATED": tl / nb * len(viewers), "batch_s_all": t["batch"],
                    "baseline_s_all": t["baseline"], "outputs_equal": bool(equal)})
    out.clear()
    del ext

    # VOD: one hour cut into 600 segments with their context, one payload, against the whole stream's add
    stream = ((rng.random((3600 * RATE, 2), dtype=np.float32) - 0.5) * 0.5).astype(np.float32)
    segs = []
    for s in range(0, stream.shape[0], SEG):
        prev, nxt = min(s, CTX), min(stream.shape[0] - s - SEG, CTX)
        segs.append((s, prev, stream[s - prev:s + SEG + nxt]))
    p = pay()

    def vod_batch():
        out["batch"] = H.add_batch_rates([x for _, _, x in segs], [p] * len(segs), [RATE] * len(segs), zero_frames=[s - prev for s, prev, _ in segs])

    def vod_whole():
        out["whole"] = H.add(stream, p, sample_rate=RATE)

    t = timed({"batch": vod_batch, "whole": vod_whole})
    trimmed = np.concatenate([y[prev:prev + SEG] for (s, prev, _), y in zip(segs, out["batch"])])
    equal = np.array_equal(trimmed, out["whole"])
    tb, tw = float(np.median(t["batch"])), float(np.median(t["whole"]))
    results.append({"workload": "vod_600x12s_stereo_48k_1h", "items": len(segs), "batch_s": tb, "whole_stream_add_s": tw,
                    "batch_s_all": t["batch"], "whole_s_all": t["whole"], "outputs_equal": bool(equal)})
    print(json.dumps({"metric": "batch_segments_rates_s", "steps": args.steps, "warmup": args.warmup, "residency": "host",
                      "gpu": gpu_card(), "workloads": results}), flush=True)
    if not all(r["outputs_equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
