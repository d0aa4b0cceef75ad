#!/usr/bin/env python
"""batch_digest.py -- what every route of the batched `add` computes and launches, in a form two builds can be compared by.

routes     add_batch (plain, zero_frames), add_batch_rates (with and without zero_frames), keys= on both (all four list combinations),
           and the one-item batch that `add` at 48 kHz runs; each in float32 and int16, with host arrays and with one packed device
           tensor, with the limiter on and off, with and without statistics
inputs     seeded: uniform noise at -6 dBFS, 1 to 3 channels, 0 to 7 s per item, random payloads and keys
prints     one JSON line per case: SHA-256 of the output bytes, the per-item data blocks, the per-item SNR to 9 significant digits (the
           device sums it with atomics, so its last bits depend on the order blocks finish), the kernels in first-launch order with
           their launch counts (profile_report), and the launch count of the call (gpu_launches)

Two builds compute the same thing when their outputs are equal line for line:
  python tools/batch_digest.py > a.jsonl; (other build) python tools/batch_digest.py > b.jsonl; cmp a.jsonl b.jsonl
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# (sample rate, frames, channels) per item: several rates, an empty item and one long enough for several limiter blocks
ITEMS = [(44100, 3 * 44100 + 517, 2), (48000, 5 * 48000 + 3, 1), (44100, 0, 2), (32000, 7 * 32000, 3), (22050, 2 * 22050 + 11, 2),
         (44100, 44100 // 3, 1)]
OFFSETS = [(1 << 40) + 3, 4 * 48000 + 5, 1024, 7 * 32000, 0, 300 * 1024 + 517]


def snr9(values):
    return [float("%.9g" % v) for v in values]


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(a.tobytes())
    return h.hexdigest()


def main():
    import numpy as np
    import torch
    from audiowmark_b200 import hostapi as H

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    rng = np.random.default_rng(20261018)
    pcm = [(rng.random((n, c), np.float32) - 0.5) for _, n, c in ITEMS]
    payloads = ["".join("%x" % v for v in rng.integers(0, 16, 32)) for _ in ITEMS]
    keys = [bytes(rng.integers(0, 256, 16, np.uint8)) for _ in range(2)]
    key_list = [keys[i % 2] for i in range(len(ITEMS))]
    key_list[-1] = keys[0]
    rates = [r for r, _, _ in ITEMS]
    at44 = [i for i, r in enumerate(rates) if r == 44100]

    def cases():
        for limiter, stats in ((True, True), (False, True), (True, False)):
            yield limiter, stats, "plain", at44, {}
            yield limiter, stats, "offsets", at44, {"zero_frames": [OFFSETS[i] for i in at44]}
            yield limiter, stats, "rates", None, {"sample_rates": rates}
            yield limiter, stats, "rates_offsets", None, {"sample_rates": rates, "zero_frames": OFFSETS}
            yield limiter, stats, "keys", at44, {"keys": [key_list[i] for i in at44]}
            yield limiter, stats, "keys_offsets", at44, {"keys": [key_list[i] for i in at44], "zero_frames": [OFFSETS[i] for i in at44]}
            yield limiter, stats, "keys_rates", None, {"keys": key_list, "sample_rates": rates}
            yield limiter, stats, "keys_rates_offsets", None, {"keys": key_list, "sample_rates": rates, "zero_frames": OFFSETS}
            yield limiter, stats, "keys_one_item", [1], {"keys": [keys[1]], "sample_rates": [rates[1]]}

    for limiter, stats, route, sel, kw in cases():
        H.set_params(test_no_limiter=not limiter)
        sel = list(range(len(ITEMS))) if sel is None else sel
        if "sample_rates" in kw and len(kw["sample_rates"]) != len(sel):
            kw = dict(kw, sample_rates=[rates[i] for i in sel])
        fn = H.add_batch_rates if "sample_rates" in kw else H.add_batch
        key = None if "keys" in kw else keys[0]
        for dtype in (np.float32, np.int16):
            xs = [pcm[i] if dtype == np.float32 else np.round(pcm[i] * 32767).astype(np.int16) for i in sel]
            pays = [payloads[i] for i in sel]
            for residency in ("host", "device"):
                if residency == "host":
                    args, extra = (xs,), {}
                else:
                    items, off = [], 0
                    for x in xs:
                        items.append((off, x.shape[0], x.shape[1]))
                        off += x.size
                    packed = torch.from_numpy(np.concatenate([x.reshape(-1) for x in xs])).to(dev)
                    args, extra = (packed,), {"items": items}
                torch.cuda.synchronize()
                H.profile_enable(True)
                n0 = H.gpu_launches()
                res = fn(*args, pays, key=key, want_stats=stats, **kw, **extra)
                outs, blocks, snr = res if stats else (res, [], [])
                launches = H.gpu_launches() - n0
                prof = H.profile_report()
                H.profile_enable(False)
                outs = [o.cpu().numpy() if residency == "device" else o for o in outs]
                print(json.dumps({"route": route, "limiter": limiter, "stats": stats, "dtype": np.dtype(dtype).name, "residency": residency,
                                  "out_sha256": sha(*outs), "data_blocks": blocks, "snr_db": snr9(snr),
                                  "kernels": [[k, v["launches"]] for k, v in prof.items()], "launches": launches}), flush=True)
    # `add` at another rate: a one-item batch
    for limiter in (True, False):
        H.set_params(test_no_limiter=not limiter)
        H.profile_enable(True)
        n0 = H.gpu_launches()
        y, blocks, snr = H.add(pcm[1], payloads[1], keys[0], sample_rate=rates[1], want_stats=True)
        launches = H.gpu_launches() - n0
        prof = H.profile_report()
        H.profile_enable(False)
        print(json.dumps({"route": "add_48k", "limiter": limiter, "dtype": "float32", "residency": "host",
                          "out_sha256": sha(y), "data_blocks": [blocks], "snr_db": snr9([snr]),
                          "kernels": [[k, v["launches"]] for k, v in prof.items()], "launches": launches}), flush=True)
    H.set_params()


if __name__ == "__main__":
    main()
