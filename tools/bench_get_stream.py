#!/usr/bin/env python
"""bench_get_stream.py -- `get` of a long stream: wall time and peak host memory of the CLI on files and pipes, and the library call
at 48 kHz, for this tree and for a build of another tree (the parent commit), alternating the two in one run.

cli_<rate>_<file|pipe>   `bin/audiowmark get` of --minutes of stereo 16 bit noise marked at <rate>: from the WAV on tmpfs, or the same
                         bytes through a pipe (`cat in.wav | audiowmark get -`).  Wall time from fork to exit and peak RSS of the
                         audiowmark process (os.wait4 in a small launcher process).  Whether each tree printed the same stdout as the other is reported.
lib_get_dev48_ms         hostapi.get(sample_rate=48000) of the same length of 48 kHz stereo float in HBM (median of --steps calls after
                         one warm-up), in a fresh process per tree.

Each figure is the median over --reps alternated runs of each tree.  Prints one JSON line with the card's name and power limit.  Without
a GPU nothing is measured: every figure is reported as not measured.

python tools/bench_get_stream.py --other DIR [--minutes M] [--reps R] [--steps K]
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tools")]
PAYLOAD = "0123456789abcdef0011223344556677"


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


# A child's peak RSS counts the memory of the process it was forked from (Linux carries the forked copy's high-water mark across exec),
# so the CLI is started by a small launcher and measured there, not by this process, which holds the test audio.
LAUNCHER = r"""
import json, os, sys, time
t = time.perf_counter()
pid = os.fork()
if pid == 0:
    os.execv(sys.argv[2], sys.argv[2:])
_, status, usage = os.wait4(pid, 0)
with open(sys.argv[1], "w") as f:
    json.dump({"wall": time.perf_counter() - t, "maxrss": usage.ru_maxrss * 1024, "rc": os.waitstatus_to_exitcode(status)}, f)
"""


def run_cli(cli, wav, pipe, report):
    """(wall s, peak RSS bytes, exit code, stdout) of `audiowmark get` on wav, read from the file or through a pipe"""
    args = [sys.executable, "-c", LAUNCHER, report, cli, "get", "-" if pipe else wav]
    if pipe:
        cat = subprocess.Popen(["cat", wav], stdout=subprocess.PIPE)
        p = subprocess.run(args, stdin=cat.stdout, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
        cat.stdout.close()
        cat.wait()
    else:
        p = subprocess.run(args, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    with open(report) as f:
        r = json.load(f)
    return r["wall"], r["maxrss"], r["rc"], p.stdout


LIB_CHILD = r"""
import json, sys, time
sys.path.insert(0, sys.argv[1])
import numpy as np, torch
from audiowmark_b200 import hostapi as H
n, steps = int(sys.argv[2]), int(sys.argv[3])
g = torch.Generator(device="cuda"); g.manual_seed(7)
x = torch.rand((n, 2), device="cuda", generator=g) - 0.5
y = torch.empty_like(x)
H.add(x.data_ptr(), sys.argv[4], None, y.data_ptr(), n, 2, sample_rate=48000)
H.synchronize()
ts = []
for i in range(steps + 1):
    t = time.perf_counter()
    doc = H.get(y.data_ptr(), n_frames=n, channels=2, sample_rate=48000, parse=False)
    ts.append((time.perf_counter() - t) * 1e3)
print(json.dumps({"ms": sorted(ts[1:])[len(ts[1:]) // 2], "doc": doc}))
"""


def run_lib(tree, n, steps):
    p = subprocess.run([sys.executable, "-c", LIB_CHILD, tree, str(n), str(steps), PAYLOAD], capture_output=True, text=True)
    if p.returncode:
        raise RuntimeError(p.stderr[-2000:])
    return json.loads(p.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="root of another built tree (the parent commit) to alternate with")
    ap.add_argument("--minutes", type=float, default=60.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    from bench_batch import gpu_card

    trees = {"other": os.path.abspath(args.other), "this": ROOT}
    result = {"card": gpu_card(), "minutes": args.minutes, "trees": trees}
    if not os.path.exists("/dev/nvidiactl"):
        result["figures"] = "not measured: no GPU"
        print(json.dumps(result))
        return

    import numpy as np
    sys.path.insert(0, ROOT)
    from audiowmark_b200 import hostapi as H
    import torch                                                            # noqa: F401  (CUDA for the marking below)

    tmp = tempfile.mkdtemp(prefix="awm_gs_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None)
    wavs = {}
    try:
        for rate in (44100, 48000):
            n = int(args.minutes * 60 * rate)
            rng = np.random.default_rng(rate)
            x = (rng.random((n, 2), dtype=np.float32) - 0.5).astype(np.float32)
            y = H.add(x, PAYLOAD, sample_rate=rate)
            pcm = np.clip(np.floor(y * 32768), -32768, 32767).astype(np.int16)
            path = os.path.join(tmp, "%d.wav" % rate)
            with open(path, "wb") as f:
                data = pcm.size * 2
                f.write(b"RIFF" + struct.pack("<I", 36 + data) + b"WAVEfmt " + struct.pack("<IHHIIHH", 16, 1, 2, rate, rate * 4, 4, 16)
                        + b"data" + struct.pack("<I", data))
                f.write(pcm.tobytes())
            wavs[rate] = path
            del x, y, pcm
        H.shutdown()

        samples, outs = {}, {}
        for rep in range(args.reps):
            for name, tree in (("other", trees["other"]), ("this", trees["this"])) if rep % 2 == 0 else (("this", trees["this"]), ("other", trees["other"])):
                cli = os.path.join(tree, "audiowmark_b200", "bin", "audiowmark")
                for rate, wav in wavs.items():
                    for pipe in (False, True):
                        key = "cli_%d_%s" % (rate, "pipe" if pipe else "file")
                        wall, rss, rc, out = run_cli(cli, wav, pipe, os.path.join(tmp, "report.json"))
                        samples.setdefault((name, key), []).append((wall, rss, rc))
                        outs.setdefault(key, {})[name] = out
                lib = run_lib(tree, int(args.minutes * 60 * 48000), args.steps)
                samples.setdefault((name, "lib_get_dev48_ms"), []).append((lib["ms"], 0, 0))
                outs.setdefault("lib_get_dev48_ms", {})[name] = lib["doc"].encode()
        figures = {}
        for (name, key), v in samples.items():
            f = figures.setdefault(key, {})
            if key.startswith("cli"):
                f[name] = {"wall_s": round(median([w for w, _, _ in v]), 3), "wall_s_all": [round(w, 3) for w, _, _ in v],
                           "peak_rss_mb": round(median([r for _, r, _ in v]) / 2**20, 1), "exit": sorted({c for _, _, c in v})}
            else:
                f[name] = {"ms": round(median([w for w, _, _ in v]), 1), "ms_all": [round(w, 1) for w, _, _ in v]}
        for key, o in outs.items():
            figures[key]["same_output"] = o.get("this") == o.get("other")
        result["figures"] = figures
    finally:
        for p in list(wavs.values()) + [os.path.join(tmp, "report.json")]:
            if os.path.exists(p):
                os.remove(p)
        os.rmdir(tmp)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
