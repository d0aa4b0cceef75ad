#!/usr/bin/env python
"""bench_batch_keys.py -- batched embed with a key per item (hostapi.add_batch(keys=...) / awm_embed_batch_keys, INTEGRATION §4b),
against the alternative without it: one add_batch (key=...) per distinct key over the same items.

workloads  1024 x 10 s mono, 44.1 kHz, uniform noise at -6 dBFS, a random payload per item, with 1024 distinct keys and with 16 keys
           (items of a key are contiguous in the packed buffer, so each per-key call covers one slice of it)
residency  PCM resident in HBM (one packed float32 tensor)
timing     host wall time around each pass; both passes end in a synchronise; the two alternate within every step.  The keyed
           pass includes building the role tables of its keys on the device, the per-key passes the host's gen_embed_roles of each
           key (the role table of the previous call is reused when the key repeats, which never happens here)
checked    the outputs of the two passes are compared bit for bit (exit status 1 if they differ)
roles      also: the device role build of 1024 keys (awm_set_embed_roles_keys, median of the steps) next to the host's
           gen_embed_roles (hostapi.embed_roles) of the same 1024 keys, measured once
prints     one JSON line with the card's name and power limit

python tools/bench_batch_keys.py [--steps K] [--warmup W]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.bench_batch import gpu_card  # noqa: E402

RATE = 44100
N_ITEMS, SECONDS = 1024, 10.0
KEY_COUNTS = [1024, 16]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()

    import numpy as np
    import torch
    from audiowmark_b200 import capi, hostapi as H

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    H.set_params()
    rng = np.random.default_rng(11)
    n = int(SECONDS * RATE)
    items = [(i * n, n, 1) for i in range(N_ITEMS)]
    payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in range(N_ITEMS)]
    g = torch.Generator(device=dev)
    g.manual_seed(4321)
    x = torch.rand(N_ITEMS * n, device=dev, generator=g, dtype=torch.float32) - 0.5
    y_keys, y_per_key = torch.empty_like(x), torch.empty_like(x)
    torch.cuda.synchronize()
    results = []
    for n_keys in KEY_COUNTS:
        keys = [bytes(rng.integers(0, 256, 16, dtype=np.uint8)) for _ in range(n_keys)]
        item_keys = [keys[i * n_keys // N_ITEMS] for i in range(N_ITEMS)]
        groups = [(k * N_ITEMS // n_keys, (k + 1) * N_ITEMS // n_keys) for k in range(n_keys)]

        def run_keys():
            H.add_batch(x, payloads, keys=item_keys, items=items, out=y_keys)

        def run_per_key():
            for k, (a, b) in enumerate(groups):
                H.add_batch(x[a * n:b * n], payloads[a:b], key=keys[k], items=[(o - a * n, f, c) for o, f, c in items[a:b]], out=y_per_key[a * n:b * n])
            H.synchronize()

        t = {"keys": [], "per_key": []}
        for step in range(args.warmup + args.steps):
            order = (("keys", run_keys), ("per_key", run_per_key)) if step % 2 == 0 else (("per_key", run_per_key), ("keys", run_keys))
            for leg, fn in order:
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if step >= args.warmup:
                    t[leg].append(dt)
        equal = bool(torch.equal(y_keys, y_per_key))
        tk, tp = float(np.median(t["keys"])), float(np.median(t["per_key"]))
        results.append({"workload": "%dx10s_mono_%dkeys" % (N_ITEMS, n_keys), "items": N_ITEMS, "keys": n_keys, "pcm_frames": N_ITEMS * n,
                        "keys_s": tk, "per_key_s": tp, "keys_items_per_s": N_ITEMS / tk, "per_key_items_per_s": N_ITEMS / tp, "speedup": tp / tk,
                        "keys_s_all": t["keys"], "per_key_s_all": t["per_key"], "outputs_equal": equal})
    del x, y_keys, y_per_key
    torch.cuda.empty_cache()

    # role tables of 1024 keys: one device build against the host's builder, key by key
    keys = [bytes(rng.integers(0, 256, 16, dtype=np.uint8)) for _ in range(1024)]
    ctx = capi.Context.from_handle(H.engine_ctx())
    layout = H.role_layout()
    dev_s = []
    for step in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        ctx.set_embed_roles_keys(keys, layout)             # returns after the build (it checks the tables' error flags)
        dt = time.perf_counter() - t0
        if step >= args.warmup:
            dev_s.append(dt)
    t0 = time.perf_counter()
    for k in keys:
        H.embed_roles(k)
    host_s = time.perf_counter() - t0
    roles = {"keys": len(keys), "device_s": float(np.median(dev_s)), "device_s_all": dev_s, "host_gen_embed_roles_s": host_s,
             "host_ms_per_key": 1000 * host_s / len(keys), "host_over_device": host_s / float(np.median(dev_s))}
    print(json.dumps({"metric": "batch_keys_embed_items_per_s", "steps": args.steps, "warmup": args.warmup, "residency": "device",
                      "gpu": gpu_card(), "workloads": results, "role_build": roles}), flush=True)
    if not all(r["outputs_equal"] for r in results):
        sys.exit(1)


if __name__ == "__main__":
    main()
