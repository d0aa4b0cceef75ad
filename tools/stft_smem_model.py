#!/usr/bin/env python
"""stft_smem_model.py -- shared-memory bytes per 128-frame tile of k_stft_mags_tc, counted from the kernel's shapes (no GPU).

FFT warps, per frame on the bulk-copy path (awm_approx_tc.cuh + fft1024_warp in awm_fft.cuh; the instruction counts are those of
the frame loop in `cuobjdump -sass`):
  landing buffer read   32 LDS.64 (float2 per lane)              twiddles   32 LDS.64
  window                32 LDS    (float per lane)               transpose  32 STS.64 + 32 LDS.64
  A operand             8 STS.U16 (hi and lo of 4 bands per lane; counted as whole warp-wide accesses)
  PCM landing           one 8 KB bulk copy (UBLKCP) written into the transpose buffer
MMA warpgroup, per tile: the wgmma read A (64 rows x 16 K x 2 B = 2 KB per wgmma) and B (N columns x 16 K x 2 B) from shared
memory; the mask chunks arrive by bulk copy (18 KB each).  Two MMA structures are counted:
  blocks  per chunk and 64-row half, 3 column blocks of m64n32k16, each 2 (hi, lo) x 6 (K steps) wgmma
  wide    per chunk and 64-row half, 1 m64n96k16 accumulator, 2 x 6 wgmma

--ms T [--sms 132] [--clock-ghz 1.98] also prints the share of the 128 B/clk/SM shared-memory bandwidth that a kernel time of
T ms per launch (30-minute chunk, four shifts) would imply.

python tools/stft_smem_model.py [--ms T] [--sms N] [--clock-ghz F]
"""
import argparse
import json

TILE, K, WARP = 128, 96, 32
N_ENT, CHUNK_ENT = 510, 48
N_CHUNKS = (N_ENT + CHUNK_ENT - 1) // CHUNK_ENT
K_STEPS, TERMS = K // 16, 2                     # wgmma K steps per operand term, fp16 terms (hi, lo)
SMEM_BYTES_PER_CLK = 128


def fft_bytes_per_frame():
    lds64, lds32, sts64, sts16 = 32 + 32 + 32, 32, 32, 8
    return {"lds": lds64 * WARP * 8 + lds32 * WARP * 4, "sts": sts64 * WARP * 8 + sts16 * WARP * 2, "bulk_pcm": 1024 * 2 * 4}


def mma_bytes_per_tile(n_cols):
    wgmma = N_CHUNKS * 2 * (2 * CHUNK_ENT // n_cols) * TERMS * K_STEPS
    return {"wgmma": wgmma, "a": wgmma * 64 * 16 * 2, "b": wgmma * n_cols * 16 * 2, "bulk_masks": N_CHUNKS * 2 * CHUNK_ENT * K * 2}


def model():
    f = fft_bytes_per_frame()
    fft_tile = {k: v * TILE for k, v in f.items()}
    out = {"per_frame_fft": f, "per_tile_fft": fft_tile, "structures": {}}
    for name, n in (("blocks_m64n32k16", 32), ("wide_m64n96k16", 96)):
        m = mma_bytes_per_tile(n)
        total = sum(fft_tile.values()) + m["a"] + m["b"] + m["bulk_masks"]
        out["structures"][name] = dict(m, mma_operand_bytes=m["a"] + m["b"], total_bytes=total,
                                       smem_clk_per_tile=total // SMEM_BYTES_PER_CLK)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ms", type=float, help="measured k_stft_mags_tc time per launch on a 30-minute chunk")
    ap.add_argument("--sms", type=int, default=132)
    ap.add_argument("--clock-ghz", type=float, default=1.98)
    args = ap.parse_args()
    out = model()
    if args.ms:
        frames = 30 * 60 * 44100 // 1024
        tiles_per_sm = 4 * ((frames + TILE - 1) // TILE) / args.sms
        clk_per_tile = args.ms * 1e-3 * args.clock_ghz * 1e9 / tiles_per_sm
        out["at_ms"] = {"ms": args.ms, "tiles_per_sm": round(tiles_per_sm, 2), "clk_per_tile": round(clk_per_tile),
                        "smem_busy": {k: round(s["smem_clk_per_tile"] / clk_per_tile, 3) for k, s in out["structures"].items()}}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
