#!/usr/bin/env python
"""bench_add_windowed.py -- `add` of 1 h of stereo from host float arrays: the whole stream in one call against the bounded-memory
window loop that `audiowmark add` streams through.

whole_ms     hostapi.add(sample_rate=R): the whole stream as one item (device scratch 2 x n44 x C floats + in / out images)
windowed_ms  hostapi.add_windowed(sample_rate=R) with the default window (4096 1024-frames): each window with its halo, one at a time

Rows at 48 kHz and, as a control, at 44.1 kHz.  Each figure is the median over --steps calls after --warmup calls, host clock around
calls that return finished host arrays.  The two outputs of a row must be bit identical (exit status 1 otherwise).  Prints one JSON
line with the card's name and power limit, read in the same run.

python tools/bench_add_windowed.py [--minutes M] [--steps K] [--warmup W]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
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
    return round(median(ts), 1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    from audiowmark_b200 import hostapi as H
    from bench_batch import gpu_card

    H.set_params()
    rows, ok = [], True
    for rate in (48000, 44100):
        n = int(args.minutes * 60 * rate)
        rng = np.random.default_rng(7)
        x = ((rng.random((n, 2), dtype=np.float32) - 0.5) * 0.5).astype(np.float32)
        whole_ms, y0 = timed(lambda: H.add(x, PAYLOAD, sample_rate=rate), args.steps, args.warmup)
        win_ms, y1 = timed(lambda: H.add_windowed(x, PAYLOAD, sample_rate=rate)[0], args.steps, args.warmup)
        same = bool(np.array_equal(y0, y1))
        ok = ok and same
        rows.append({"rate": rate, "frames": n, "channels": 2, "whole_ms": whole_ms, "windowed_ms": win_ms,
                     "windowed_over_whole": round(win_ms / whole_ms, 3), "bit_identical": same})
        del x, y0, y1
    print(json.dumps({"bench": "add_windowed", "minutes": args.minutes, "steps": args.steps, "card": gpu_card(), "rows": rows}))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
