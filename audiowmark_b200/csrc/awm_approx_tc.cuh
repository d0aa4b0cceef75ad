// awm_approx_tc.cuh -- k_stft_mags_tc: SyncFinder::sync_fft for the four 256-sample shifts (src/syncfinder.cc:560-657) plus the
// inner sums of sync_decode (:116-153) as ONE persistent, warp-specialised Hopper kernel.
//
// What it computes is what k_stft_mags (awm_approx_mags.cuh) computes: for every frame f of a shift the channel-summed band dB
// values dB[f][0..80], and from them, for every sync entry e (a sync frame with 30 "up" and 30 "down" bands),
//     U_e(f) = sum_{u in up(e)} dB[f][u],   D_e(f) = sum_{d in down(e)} dB[f][d]      -> mags[shift][e][f] = (U, D)
// The second step is the contraction  [128 frames x 96 bands] . [96 bands x 2 n_ent 0/1 columns].  On the fp32 pipes it costs
// 30 600 shared-memory reads + adds per frame.  Here it runs on the tensor cores (wgmma):
//   * A operand = the dB tile, written by the FFT warps straight into the K-major operand layout (awm_tc.cuh) as TWO fp16 terms
//     hi = fp16 (v), lo = fp16 (v - hi): |v| < 256, so hi + lo carries v to 2^-16 absolute -- the resolution fp32 itself has there;
//     every product with a 0/1 mask element is exact, accumulation is fp32
//   * B operand = the 0/1 masks of 48 entries (96 columns: U and D of an entry side by side), prepared once per key on the host in
//     operand layout and fetched chunk by chunk with the bulk-copy engine (TMA, cp.async.bulk -> mbarrier complete_tx)
//   * D = one 64 x 96 fp32 accumulator per 64-row half of the tile and chunk (48 registers per thread) in the registers of the
//     MMA warpgroup, which writes it to `mags` itself; the stores of the second half run under the bulk copy of the next mask chunk
// Warp roles (one CTA per SM, CTAs walk the (frame tile, shift) list with stride gridDim.x):
//   warps 0 .. 11      FFT: frame (PCM prefetched by TMA into the warp's transpose buffer) -> packed 1024-point FFT -> dB ->
//                      fp16 hi/lo into A[buf]                                                     (a_empty -> a_full)
//   warps 12 .. 15     one warpgroup: B chunk loads (thread 0), 2 x 12 m64n96k16 wgmma per chunk, stores
//                                                                                                 (a_full, b_full -> a_empty)
// All hand-offs are mbarriers; the FFT of tile i + 1 overlaps the MMAs and the stores of tile i.
// Shared memory (225.25 KB of the 227 KB an SM grants one CTA):
//   twiddles 8 KB | window 4 KB | 12 transpose / PCM landing buffers of 8448 B (99 KB) | 2 A buffers of 48 KB (hi 24 KB + lo 24 KB)
//   | 1 B buffer of 18 KB (one mask chunk) | mbarriers (256 B)
// A second B buffer does not fit, so the next chunk's masks are fetched into the one buffer once the chunk's last wgmma retired.
// Operand bytes per wgmma: A 2 KB (64 rows x 16 K), B 3 KB (96 columns x 16 K); per 128-frame tile 11 chunks x 24 wgmma read
// 22 x 12 A blocks (0.53 MB) and 11 x 24 B blocks (0.79 MB) -- tools/stft_smem_model.py counts them against the FFT warps' bytes.
#pragma once
#include "awm_kernels.cuh"
#include "awm_tc.cuh"
#include <cuda_fp16.h>

namespace awm {

constexpr int kTcTile = 128;                 // frames per tile (two 64-row wgmma halves)
constexpr int kTcK = 96;                     // 81 bands padded to a multiple of the wgmma K (16)
constexpr uint32_t kTcASplit = kTcTile * kTcK * 2;        // bytes of one fp16 term of the A tile (24 KB)
constexpr uint32_t kTcABytes = 2 * kTcASplit;             // hi + lo
constexpr int kTcEpiWarps = 4;             // the MMA warpgroup
constexpr int kTcFftWarps = 12;
constexpr int kTcABufs = 2;                // the FFT of tile i + 1 fills one A buffer while the MMAs read tile i from the other
// sync entries per B chunk -> N = 2 kTcChunkEnt columns (U and D column of every entry), chunk of N x 96 fp16 (18 KB): small
// enough to leave room for twelve FFT warps AND two A buffers
constexpr int kTcChunkEnt = 48;
constexpr int kTcN = 2 * kTcChunkEnt;
constexpr uint32_t kTcBBytes = uint32_t (kTcN) * kTcK * 2;
constexpr size_t kTcSmemBytes = fft_smem_bytes (kTcFftWarps) + size_t (kTcABufs) * kTcABytes + kTcBBytes + 256;
static_assert (kTcFftWarps % 4 == 0, "the MMA warpgroup has to start at a warp index divisible by four");
static_assert (kTcN == 96, "one m64n96k16 wgmma covers the columns of a chunk");

// host side: the 0/1 masks of all entries in operand layout, chunk after chunk ([ceil (n_ent / kTcChunkEnt)][kTcBBytes])
inline void
tc_build_masks (const awm_sync_entry *ent, int n_ent, std::vector<unsigned char>& out)
{
  const int n_chunks = (n_ent + kTcChunkEnt - 1) / kTcChunkEnt;
  out.assign (size_t (n_chunks) * kTcBBytes, 0);
  const uint16_t one = 0x3c00;               // 1.0 in fp16
  for (int e = 0; e < n_ent; e++)
    {
      unsigned char *chunk = out.data() + size_t (e / kTcChunkEnt) * kTcBBytes;
      const int col = 2 * (e % kTcChunkEnt);
      for (int i = 0; i < kUD; i++)
        {
          memcpy (chunk + tc::operand_offset (kTcN, col, ent[e].up[i]), &one, 2);
          memcpy (chunk + tc::operand_offset (kTcN, col + 1, ent[e].down[i]), &one, 2);
        }
    }
}

__global__ void __launch_bounds__ ((kTcFftWarps + kTcEpiWarps) * 32, 1)
k_stft_mags_tc (const float *__restrict__ pcm, long long n_frames, int C, int n_out, int ld,
                const unsigned char *__restrict__ masks /* [n_chunks][kTcBBytes] */, int n_ent, int n_chunks,
                float2 *__restrict__ mags /* [4][n_ent][ld] */, unsigned char *__restrict__ have,
                long long wav_first, long long wav_last, const float2 *g_tw, const float *g_win, int tma_ok /* stereo, pcm 16-byte aligned */)
{
  using namespace tc;
  extern __shared__ __align__ (16) unsigned char smem[];
  FftSmem s = fft_smem_setup (smem, g_tw, g_win, kTcFftWarps);
  unsigned char *abuf = reinterpret_cast<unsigned char *> (s.extra);
  unsigned char *bbuf = abuf + size_t (kTcABufs) * kTcABytes;
  uint64_t *bars = reinterpret_cast<uint64_t *> (bbuf + kTcBBytes);
  uint64_t *a_full = bars, *a_empty = bars + 2, *b_full = bars + 4;
  uint64_t *pcm_bars = bars + 5;                                   // one per FFT warp: its next frame has landed in its transpose buffer
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;

  if (threadIdx.x == 0)
    {
      for (int i = 0; i < 2; i++)
        {
          mbar_init (&a_full[i], kTcFftWarps);
          mbar_init (&a_empty[i], kTcEpiWarps);
        }
      mbar_init (b_full, 1);
      for (int i = 0; i < kTcFftWarps; i++)
        mbar_init (&pcm_bars[i], 1);
      fence_mbar_init();
    }
  // band columns 81 .. 95 of A are never written again and must be finite: clear everything once
  for (uint32_t i = threadIdx.x; i < kTcABufs * kTcABytes / 16; i += blockDim.x)
    reinterpret_cast<uint4 *> (abuf)[i] = make_uint4 (0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();
  const int n_tiles = 4 * ((n_out + kTcTile - 1) / kTcTile);

  if (w < kTcFftWarps)
    {
      // ===================================================================================== FFT warps
      // The PCM of a frame reaches the warp through the bulk-copy engine: while the second butterfly pass of frame i runs, the
      // 8 KB of frame i + 1 (1024 stereo sample-frames, contiguous and 16-byte aligned in the interleaved stream) land in the
      // warp's transpose buffer, which is idle from that point on; the next iteration finds them in shared memory (mbarrier
      // complete_tx) instead of waiting ~1 us for 32 global loads per lane.  Frames the copy cannot serve -- mono / multichannel
      // audio, the ragged end of the stream, an unaligned caller buffer -- take the global-load path of frame_db_sum.
      uint64_t *pcm_bar = pcm_bars + w;
      uint32_t pcm_phase = 0;
      struct Frame { int t, r; };
      auto frame_start = [&] (Frame fr) { return (long long) (fr.t & 3) * 256 + (long long) ((fr.t >> 2) * kTcTile + fr.r) * kFrame; };
      auto exists = [&] (Frame fr) { return fr.t < n_tiles; };
      auto wanted = [&] (Frame fr)          // sync_fft computes this frame: inside the output range and not in leading / trailing digital silence
        {
          const long long start = frame_start (fr);
          const long long f_first = start * C, f_last = (start + kFrame) * C;
          return (fr.t >> 2) * kTcTile + fr.r < n_out && !(f_last < wav_first || f_first > wav_last);
        };
      auto by_tma = [&] (Frame fr) { return tma_ok && exists (fr) && wanted (fr) && frame_start (fr) + kFrame <= n_frames; };
      auto next_of = [&] (Frame fr)
        {
          fr.r += kTcFftWarps;
          if (fr.r >= kTcTile)
            {
              fr.r = w;
              fr.t += gridDim.x;
            }
          return fr;
        };
      auto prefetch = [&] (Frame fr)        // caller: after __syncwarp, every lane is done with the transpose buffer
        {
          if (lane == 0)
            {
              fence_proxy_async();          // the lanes' generic-proxy accesses to xbuf are ordered before the engine's writes
              mbar_arrive_expect_tx (pcm_bar, kFrame * 2 * sizeof (float));
              bulk_load (s.xbuf, pcm + frame_start (fr) * 2, kFrame * 2 * sizeof (float), pcm_bar);
            }
        };
      Frame cur { int (blockIdx.x), w };
      if (by_tma (cur))
        prefetch (cur);
      int it = 0;
      for (; exists (cur); it++)
        {
          const int shift_idx = cur.t & 3, f0 = (cur.t >> 2) * kTcTile;
          const int a = it % kTcABufs, use = it / kTcABufs;
          mbar_wait_relaxed (&a_empty[a], (use & 1) ^ 1);         // the MMAs that read this buffer last time are done
          unsigned char *A = abuf + size_t (a) * kTcABytes;
          const int t_now = cur.t;
          for (; cur.t == t_now; )
            {
              const int r = cur.r, f = f0 + r;
              const Frame nxt = next_of (cur);
              const bool ok = wanted (cur), nxt_tma = by_tma (nxt);
              float acc[4] = { 0.f, 0.f, 0.f, 0.f };
              if (by_tma (cur))
                {
                  float re[32], im[32];
                  mbar_wait (pcm_bar, pcm_phase);
                  pcm_phase ^= 1;
                  const float2 *xp = reinterpret_cast<const float2 *> (s.xbuf) + lane;
#pragma unroll
                  for (int j = 0; j < 32; j++)
                    {
                      const float2 v = xp[32 * j];
                      const float wn = s.win[32 * j + lane];
                      re[j] = __fmul_rn (v.x, wn);
                      im[j] = __fmul_rn (v.y, wn);
                    }
                  __syncwarp();                                   // all lanes hold their samples before the transposes reuse the buffer
                  fft1024_warp (re, im, s.tw, s.xbuf, lane, [&] { if (nxt_tma) prefetch (nxt); });
                  // dB with MUFU.LG2 (__log2f): its error (~2e-7 relative) is two orders below the 2^-16 absolute resolution the
                  // value is about to be stored with (fp16 hi + lo)
                  auto db = [] (float re_, float im_) { const float a2 = __fmaf_rn (re_, re_, __fmul_rn (im_, im_)); return a2 > 0.0f ? __log2f (a2) * 3.01029995663981f : -96.f; };
                  float ar, ai, br, bi;
                  unpack_pair<0> (re, im, lane, ar, ai, br, bi);
                  acc[0] = db (ar, ai) + db (br, bi);
                  unpack_pair<1> (re, im, lane, ar, ai, br, bi);
                  acc[1] = db (ar, ai) + db (br, bi);
                  unpack_pair<2> (re, im, lane, ar, ai, br, bi);
                  acc[2] = db (ar, ai) + db (br, bi);
                  unpack_pair<3> (re, im, lane, ar, ai, br, bi);
                  acc[3] = db (ar, ai) + db (br, bi);
                }
              else
                {
                  if (ok)
                    frame_db_sum (pcm, n_frames, C, frame_start (cur), s, lane, acc);
                  __syncwarp();
                  if (nxt_tma)
                    prefetch (nxt);
                }
#pragma unroll
              for (int k2 = 0; k2 < 4; k2++)
                {
                  const int band = lane + 32 * k2 - kMinBand;
                  if (band >= 0 && band < kBands)
                    {
                      const __half hi = __float2half_rn (acc[k2]);
                      const __half lo = __float2half_rn (acc[k2] - __half2float (hi));
                      const uint32_t o = operand_offset (kTcTile, r, band);
                      *reinterpret_cast<__half *> (A + o) = hi;
                      *reinterpret_cast<__half *> (A + kTcASplit + o) = lo;
                    }
                }
              if (lane == 0 && f < n_out)
                have[(size_t) shift_idx * ld + f] = ok ? 1 : 0;
              cur = nxt;
            }
          fence_proxy_async();                                    // st.shared above -> visible to wgmma (async proxy)
          __syncwarp();
          if (lane == 0)
            mbar_arrive (&a_full[a]);
        }
    }
  else
    {
      // ===================================================================================== MMA warpgroup
      // Per chunk and 64-row half: ONE 64 x 96 accumulator (all 48 entries of the chunk), built by 2 (hi, lo) x 6 (K steps)
      // m64n96k16 wgmma in that order, so an element sees the same products in the same order as in any narrower split of the
      // columns.  Half 0 is computed and stored, then half 1; once half 1 has retired nothing reads the mask chunk any more,
      // thread 0 starts the bulk copy of the next chunk into the one B buffer, and half 1 is stored while it lands.  (Keeping both
      // halves in flight -- 96 accumulators, half 0 stored under the MMAs of half 1 -- measured slower: the extra registers cost
      // the FFT warps spills in their frame loop.)
      const int wt = threadIdx.x - kTcFftWarps * 32, wi = wt >> 5;                  // thread / warp within the warpgroup
      const uint32_t b_addr = smem_u32 (bbuf);
      auto load_b = [&] (int c)
        {
          mbar_arrive_expect_tx (b_full, kTcBBytes);
          bulk_load (bbuf, masks + size_t (c) * kTcBBytes, kTcBBytes, b_full);
        };
      // the descriptors of all 24 wgmma of a chunk are one base descriptor per operand plus a constant (the start address sits in
      // the low bits, in units of 16 bytes, and never carries out of its field).  The A base is re-derived behind an empty asm in
      // every chunk, so the compiler does not keep 24 loop-invariant descriptors live next to the accumulators.
      auto mma_half = [&] (float (&d)[kTcN / 2], uint64_t da, uint64_t db, int mh)
        {
#pragma unroll
          for (int sp = 0; sp < 2; sp++)
#pragma unroll
            for (int j = 0; j < kTcK / 16; j++)
              wgmma_m64n96k16_f16 (d, da + ((sp * kTcASplit + j * 2 * (kTcTile * 16) + mh * (64 / 8) * 128) >> 4),
                                   db + ((j * 2 * (kTcN * 16)) >> 4), (sp | j) != 0);
          wgmma_commit();
        };
      auto store_half = [&] (float (&d)[kTcN / 2], int shift_idx, int f0, int c, int mh)
        {
#pragma unroll
          for (int i = 0; i < kTcN / 2; i++)
            wgmma_fence_operand (d[i]);
          asm volatile ("" : "+r"(c));              // the addresses are formed here, after the wait, not held across the MMAs
          const int e_base = c * kTcChunkEnt + (lane & 3);
          const int f = f0 + mh * 64 + wi * 16 + (lane >> 2);                   // f + 8 < ld always (ld multiple of 128)
#pragma unroll
          for (int q = 0; q < kTcN / 8; q++)
            {
              const int e = e_base + 4 * q;
              if (e < n_ent)
                {
                  // streaming stores (evict first): the 1.27 GB of entry sums per chunk pass through L2 without pushing out the
                  // PCM frames and mask chunks that the bulk copies read again
                  float2 *row = mags + ((size_t) shift_idx * n_ent + e) * ld + f;
                  __stcs (row, make_float2 (d[4 * q], d[4 * q + 1]));
                  __stcs (row + 8, make_float2 (d[4 * q + 2], d[4 * q + 3]));
                }
            }
        };
      if (wt == 0 && blockIdx.x < n_tiles && n_chunks > 0)
        load_b (0);
      int it = 0, g = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, it++)
        {
          const int a = it % kTcABufs, use = it / kTcABufs;
          const int shift_idx = t & 3, f0 = (t >> 2) * kTcTile;
          const uint32_t a_addr = smem_u32 (abuf + size_t (a) * kTcABytes);
          mbar_wait_relaxed (&a_full[a], use & 1);                                // all FFT warps have delivered their rows of the tile
          if (n_chunks == 0)
            {
              __syncwarp();
              if (lane == 0)
                mbar_arrive (&a_empty[a]);
            }
          for (int c = 0; c < n_chunks; c++, g++)
            {
              float d[kTcN / 2];
#pragma unroll
              for (int i = 0; i < kTcN / 2; i++)
                d[i] = 0.f;
              mbar_wait_relaxed (b_full, g & 1);
              uint32_t a_base = a_addr;
              asm volatile ("" : "+r"(a_base));
              const uint64_t da = smem_desc_kmajor (a_base, kTcTile * 16, 128), db = smem_desc_kmajor (b_addr, kTcN * 16, 128);
              wgmma_fence();
              mma_half (d, da, db, 0);
              wgmma_wait<0>();
              store_half (d, shift_idx, f0, c, 0);
              wgmma_fence();
              mma_half (d, da, db, 1);
              wgmma_wait<0>();
              // every wgmma of the chunk has retired: this warp no longer reads A (last chunk) or B
              __syncwarp();
              if (c == n_chunks - 1 && lane == 0)
                mbar_arrive (&a_empty[a]);
              asm volatile ("bar.sync 1, %0;" :: "n"(kTcEpiWarps * 32) : "memory");      // the whole warpgroup is past B
              if (wt == 0)
                {
                  if (c + 1 < n_chunks)
                    load_b (c + 1);
                  else if (t + int (gridDim.x) < n_tiles)
                    load_b (0);
                }
              store_half (d, shift_idx, f0, c, 1);
            }
        }
    }
}

} // namespace awm
