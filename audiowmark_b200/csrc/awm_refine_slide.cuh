// awm_refine_slide.cuh -- SyncFinder::search_refine (src/syncfinder.cc:393-458) with a sliding DFT.
//
// search_refine scores 65 fine offsets (8 samples apart) per candidate; for each of them the reference transforms all
// wanted sync frames again (sync_fft, :560-605) although consecutive offsets share 1016 of the 1024 samples of every frame.
// Here one warp owns one (candidate, sync frame) pair and walks the 65 offsets:
//   offset 0     : one 1024-point FFT of the un-windowed frame (left + i right) -> rectangular-window spectrum R[k], k = 19..102
//   offset m+1   : R'[k] = W^(-8k) (R[k] + sum_{j<8} (x[P+1024+j] - x[P+j]) W^(jk)),  W = exp (-2 pi i / 1024)
//   Hann window  : the reference's window w[n] = (0.5 - 0.5 cos (2 pi n / 1024)) / 256 acts in the frequency domain as
//                  X[k] = (R[k] - (R[k-1] + R[k+1]) / 2) / 512
//   dB of bins 20..100 summed over the channels, up / down band sums of this sync frame (warp reduction)
// The sample differences of all 64 slides are staged once in the warp's transpose buffer; the band sums of four offsets are
// reduced together.  207 warp instructions per offset in stereo (117 mono) instead of ~1700 for a fresh transform.  A second kernel adds the per-frame sums of each
// sync bit in frame order.  Numerics: a float sliding update carries an error of a few 1e-6 relative to the largest
// bins after 64 steps, the same order as a float FFT's own rounding (DESIGN.md section 6); tests hold it to the
// same bars as the FFT path (quality 2e-4, index within one 8-sample step).
// Lane l keeps bins 19 + 3l .. 21 + 3l (lanes 0..27), so the Hann neighbours are one shuffle away.
#pragma once
#include "awm_kernels.cuh"

namespace awm {

constexpr int kSlideWarps = 8;
constexpr int kSlideBins = 3;
constexpr int kSlideGroup = 4;                          // offsets whose band sums are reduced together
constexpr int kSlideStage = 8 * (kOffsets - 1);         // staged sample differences: 64 slides of 8
constexpr float kSlideScale = 1.0f / 512.0f;            // the Hann window's 1/512, applied to the spectrum (exact: a power of two)
constexpr float kSlideDbPerLog2 = 3.01029995663981f;    // 10 log10 (2): dB of |X|^2 = 10 log10 2 * log2 |X|^2
constexpr float kSlideSilenceLog2 = -96.0f / kSlideDbPerLog2;

template<int C> __global__ void __launch_bounds__ (kSlideWarps * 32, 2)
k_refine_slide (const float *__restrict__ pcm, long long n_frames,
                const long long *__restrict__ cand_start, const int *__restrict__ cand_noff, int n_cand,
                const awm_sync_entry *__restrict__ g_ent, int n_ent, int total_frame_count,
                long long wav_first, long long wav_last,
                float2 *__restrict__ ent_ud /* [cand][65][n_ent] */, unsigned char *__restrict__ ent_flag,
                const float2 *g_tw, const float2 *__restrict__ tw1024)
{
  extern __shared__ __align__ (16) unsigned char smem[];
  FftSmem s = fft_smem_setup (smem, g_tw, nullptr, kSlideWarps);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long job = (long long) blockIdx.x * kSlideWarps + w;
  if (job >= (long long) n_cand * n_ent)
    return;
  const int c = int (job / n_ent), e = int (job % n_ent);
  const awm_sync_entry *en = g_ent + e;
  const long long p0 = cand_start[c] + (long long) en->frame * kFrame;      // first sample of this sync frame at offset 0
  // offsets whose block would read past the end yield no result (sync_fft returns nothing): same rule as k_refine_reduce
  long long n_valid = cand_noff[c];
  {
    const long long room = n_frames - (long long) total_frame_count * kFrame - cand_start[c];
    n_valid = room < 0 ? 0 : (n_valid < room / 8 + 1 ? n_valid : room / 8 + 1);
  }
  float2 *out = ent_ud + ((size_t) c * kOffsets) * n_ent + e;
  unsigned char *flag = ent_flag + ((size_t) c * kOffsets) * n_ent + e;
  if (n_valid <= 0)
    return;

  // ---- offset 0: rectangular-window spectrum by one FFT, scaled by 1/512 (exact: a power of two)
  float rl_re[kSlideBins], rl_im[kSlideBins], rr_re[kSlideBins], rr_im[kSlideBins];
  {
    float re[32], im[32];
    if (C == 2)
      {
        const float2 *p = reinterpret_cast<const float2 *> (pcm) + p0 + lane;
#pragma unroll
        for (int j = 0; j < 32; j++)
          {
            const float2 v = __ldg (p + 32 * j);
            re[j] = v.x;
            im[j] = v.y;
          }
      }
    else
      {
#pragma unroll
        for (int j = 0; j < 32; j++)
          {
            re[j] = __ldg (pcm + p0 + 32 * j + lane);
            im[j] = 0.f;
          }
      }
    fft1024_warp (re, im, s.tw, s.xbuf, lane);
    float4 *sc = reinterpret_cast<float4 *> (s.xbuf);           // the transpose buffer is free again: [128] (Lre, Lim, Rre, Rim)
    float ar, ai, br, bi;
    unpack_pair<0> (re, im, lane, ar, ai, br, bi); sc[lane]      = make_float4 (ar, ai, br, bi);
    unpack_pair<1> (re, im, lane, ar, ai, br, bi); sc[lane + 32] = make_float4 (ar, ai, br, bi);
    unpack_pair<2> (re, im, lane, ar, ai, br, bi); sc[lane + 64] = make_float4 (ar, ai, br, bi);
    unpack_pair<3> (re, im, lane, ar, ai, br, bi); sc[lane + 96] = make_float4 (ar, ai, br, bi);
    __syncwarp();
#pragma unroll
    for (int b = 0; b < kSlideBins; b++)
      {
        const int k = (19 + kSlideBins * lane + b) & 127;
        const float4 v = sc[k];
        rl_re[b] = v.x * kSlideScale; rl_im[b] = v.y * kSlideScale; rr_re[b] = v.z * kSlideScale; rr_im[b] = v.w * kSlideScale;
      }
    __syncwarp();
  }
  if (n_valid > 1 && p0 + 8 * (n_valid - 2) + kFrame + 8 > n_frames)       // cannot happen (n_valid is cut to the stream above); keeps the loads in bounds
    return;
  // ---- the transpose buffer is free again: it takes the differences x[P + 1024 + n] - x[P + n] (scaled by 1/512 like the spectrum)
  // of every slide, kSlideStage of them, zero past the last slide that exists.  Loaded once, coalesced; each slide then reads its 8
  // (stereo: 8 x 2) as broadcast LDS.128 instead of every lane loading the same 16 samples from L2.
  {
    const int n_slide = int (8 * (n_valid - 1));
    if (C == 2)
      {
        const float2 *po = reinterpret_cast<const float2 *> (pcm) + p0;
        float2 *xb = reinterpret_cast<float2 *> (s.xbuf);
#pragma unroll
        for (int t = 0; t < kSlideStage / 32; t++)
          {
            const int i = 32 * t + lane;
            float2 v = make_float2 (0.f, 0.f);
            if (i < n_slide)
              {
                const float2 xo = __ldg (po + i), xi = __ldg (po + kFrame + i);
                v = make_float2 ((xi.x - xo.x) * kSlideScale, (xi.y - xo.y) * kSlideScale);
              }
            xb[i] = v;
          }
      }
    else
      {
#pragma unroll
        for (int t = 0; t < kSlideStage / 32; t++)
          {
            const int i = 32 * t + lane;
            s.xbuf[i] = i < n_slide ? (__ldg (pcm + p0 + kFrame + i) - __ldg (pcm + p0 + i)) * kSlideScale : 0.f;
          }
      }
    __syncwarp();
  }
  // ---- per-lane constants: W^(jk) for the 7 entering / leaving samples j = 1..7 (W^0 = 1 is an add), the rotation W^(-8k), band membership
  float wr[kSlideBins][7], wi[kSlideBins][7], rot_c[kSlideBins], rot_s[kSlideBins], m_up[kSlideBins], m_dn[kSlideBins];
#pragma unroll
  for (int b = 0; b < kSlideBins; b++)
    {
      const int k = 19 + kSlideBins * lane + b;
#pragma unroll
      for (int j = 1; j < 8; j++)
        {
          const float2 t = __ldg (tw1024 + ((j * k) & 1023));
          wr[b][j - 1] = t.x;
          wi[b][j - 1] = t.y;
        }
      const float2 r = __ldg (tw1024 + ((8 * k) & 1023));
      rot_c[b] = r.x;
      rot_s[b] = -r.y;                     // conj: W^(-8k)
      const int band = k - kMinBand;
      float mu = 0.f, md = 0.f;
      if (band >= 0 && band < kBands)
        for (int i = 0; i < kUD; i++)
          {
            if (en->up[i] == band) mu = 1.f;
            if (en->down[i] == band) md = 1.f;
          }
      m_up[b] = mu;
      m_dn[b] = md;
    }

  // log2 |X|^2 for RANKING the offsets: MUFU.LG2 (abs. error ~1e-7 on these magnitudes -- an order below the float sliding DFT's own
  // error) instead of the ~22-instruction log2f; the offsets that matter are scored again exactly by k_refine_exact_*.  A bin of
  // exactly zero energy stands for -96 dB as in the reference.  The flush-to-zero MUFU alone is right for every normal energy; a lane
  // that meets a zero or subnormal one takes the rule of __log2f (which scales subnormals first) on all six.  The band sums are
  // turned into dB (x 10 log10 2) once, after the reduction.
  auto lg_ftz = [] (float x) { float r; asm ("lg2.approx.ftz.f32 %0, %1;" : "=f" (r) : "f" (x)); return r; };
  // per-lane part of the up / down band sums of the current spectrum: Hann in the frequency domain, log2 |X|^2 of both channels
  auto band_partials = [&] (float& u, float& d)
    {
      const float ll_re = __shfl_up_sync (0xffffffffu, rl_re[2], 1), ll_im = __shfl_up_sync (0xffffffffu, rl_im[2], 1);
      const float nl_re = __shfl_down_sync (0xffffffffu, rl_re[0], 1), nl_im = __shfl_down_sync (0xffffffffu, rl_im[0], 1);
      float lr_re = 0, lr_im = 0, nr_re = 0, nr_im = 0;
      if (C == 2)
        {
          lr_re = __shfl_up_sync (0xffffffffu, rr_re[2], 1); lr_im = __shfl_up_sync (0xffffffffu, rr_im[2], 1);
          nr_re = __shfl_down_sync (0xffffffffu, rr_re[0], 1); nr_im = __shfl_down_sync (0xffffffffu, rr_im[0], 1);
        }
      float e[C][kSlideBins];              // |X|^2 per channel and bin
#pragma unroll
      for (int b = 0; b < kSlideBins; b++)
        {
          const float pl_re = b == 0 ? ll_re : rl_re[b - 1], pl_im = b == 0 ? ll_im : rl_im[b - 1];
          const float ql_re = b == kSlideBins - 1 ? nl_re : rl_re[b + 1], ql_im = b == kSlideBins - 1 ? nl_im : rl_im[b + 1];
          const float hl_re = rl_re[b] - 0.5f * (pl_re + ql_re), hl_im = rl_im[b] - 0.5f * (pl_im + ql_im);
          e[0][b] = hl_re * hl_re + hl_im * hl_im;
          if (C == 2)
            {
              const float pr_re = b == 0 ? lr_re : rr_re[b - 1], pr_im = b == 0 ? lr_im : rr_im[b - 1];
              const float qr_re = b == kSlideBins - 1 ? nr_re : rr_re[b + 1], qr_im = b == kSlideBins - 1 ? nr_im : rr_im[b + 1];
              const float hr_re = rr_re[b] - 0.5f * (pr_re + qr_re), hr_im = rr_im[b] - 0.5f * (pr_im + qr_im);
              e[C - 1][b] = hr_re * hr_re + hr_im * hr_im;
            }
        }
      float l2[C][kSlideBins], lo = e[0][0];
#pragma unroll
      for (int c = 0; c < C; c++)
#pragma unroll
        for (int b = 0; b < kSlideBins; b++)
          {
            l2[c][b] = lg_ftz (e[c][b]);
            lo = fminf (lo, e[c][b]);
          }
      if (lo < 1.17549435e-38f)            // FLT_MIN
        {
#pragma unroll
          for (int c = 0; c < C; c++)
#pragma unroll
            for (int b = 0; b < kSlideBins; b++)
              l2[c][b] = e[c][b] > 0.0f ? __log2f (e[c][b]) : kSlideSilenceLog2;
        }
      u = 0.f;
      d = 0.f;
#pragma unroll
      for (int b = 0; b < kSlideBins; b++)
        {
          const float l = C == 2 ? l2[0][b] + l2[C - 1][b] : l2[0][b];
          u = fmaf (l, m_up[b], u);
          d = fmaf (l, m_dn[b], d);
        }
    };
  // slide m: offset m -> m + 1, the 8 (stereo: 8 x 2) sample differences read from the stage as broadcast LDS.128
  auto slide = [&] (int m)
    {
      float dl[8], dr[8];
      if (C == 2)
        {
          const float4 *q = reinterpret_cast<const float4 *> (s.xbuf) + 4 * m;
#pragma unroll
          for (int t = 0; t < 4; t++)
            {
              const float4 v = q[t];
              dl[2 * t] = v.x; dr[2 * t] = v.y; dl[2 * t + 1] = v.z; dr[2 * t + 1] = v.w;
            }
        }
      else
        {
          const float4 *q = reinterpret_cast<const float4 *> (s.xbuf) + 2 * m;
#pragma unroll
          for (int t = 0; t < 2; t++)
            {
              const float4 v = q[t];
              dl[4 * t] = v.x; dl[4 * t + 1] = v.y; dl[4 * t + 2] = v.z; dl[4 * t + 3] = v.w;
              dr[4 * t] = dr[4 * t + 1] = dr[4 * t + 2] = dr[4 * t + 3] = 0.f;
            }
        }
#pragma unroll
      for (int b = 0; b < kSlideBins; b++)
        {
          float tr = rl_re[b] + dl[0], ti = rl_im[b];
#pragma unroll
          for (int j = 1; j < 8; j++)
            {
              tr = fmaf (dl[j], wr[b][j - 1], tr);
              ti = fmaf (dl[j], wi[b][j - 1], ti);
            }
          rl_re[b] = tr * rot_c[b] - ti * rot_s[b];
          rl_im[b] = tr * rot_s[b] + ti * rot_c[b];
          if (C == 2)
            {
              float sr = rr_re[b] + dr[0], si = rr_im[b];
#pragma unroll
              for (int j = 1; j < 8; j++)
                {
                  sr = fmaf (dr[j], wr[b][j - 1], sr);
                  si = fmaf (dr[j], wi[b][j - 1], si);
                }
              rr_re[b] = sr * rot_c[b] - si * rot_s[b];
              rr_im[b] = sr * rot_s[b] + si * rot_c[b];
            }
        }
    };
  // frames in digital silence are not counted (src/syncfinder.cc:573-580)
  auto counted = [&] (int m) -> unsigned char
    {
      const long long start = p0 + 8LL * m;
      const long long f_first = start * C, f_last = (start + kFrame) * C;
      return !(f_last < wav_first || f_first > wav_last);
    };

  // ---- offset 0
  {
    float u, d;
    band_partials (u, d);
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1)
      {
        u += __shfl_xor_sync (0xffffffffu, u, sh);
        d += __shfl_xor_sync (0xffffffffu, d, sh);
      }
    if (lane == 0)
      {
        out[0] = make_float2 (u * kSlideDbPerLog2, d * kSlideDbPerLog2);
        flag[0] = counted (0);
      }
  }
  // ---- offsets 1..64 in groups of four.  The 8 per-lane partial sums of a group (u, d of each offset) are reduced together by a
  // reduce-scatter: three halving exchanges (lanes 16, 8, 4 apart) leave lane l with value l >> 2 summed over 8 lanes, two butterflies
  // finish it -- 10 shuffles per group instead of 10 per offset.  Lane 4g then holds u of offset m0 + g, lane 16 + 4g its d.
  // Slides past the last valid offset read zero differences (the stage is zero there) and their sums are not stored.
  static_assert (kSlideGroup == 4 && (kOffsets - 1) % kSlideGroup == 0, "the reduce-scatter below is written for groups of four");
  for (int m0 = 1; m0 < n_valid; m0 += kSlideGroup)
    {
      float v[2 * kSlideGroup];
#pragma unroll
      for (int g = 0; g < kSlideGroup; g++)
        {
          slide (m0 + g - 1);
          band_partials (v[g], v[kSlideGroup + g]);
        }
      const bool h16 = lane & 16, h8 = lane & 8, h4 = lane & 4;
      float a[4], b[2];
#pragma unroll
      for (int i = 0; i < 4; i++)
        a[i] = (h16 ? v[i + 4] : v[i]) + __shfl_xor_sync (0xffffffffu, h16 ? v[i] : v[i + 4], 16);
#pragma unroll
      for (int i = 0; i < 2; i++)
        b[i] = (h8 ? a[i + 2] : a[i]) + __shfl_xor_sync (0xffffffffu, h8 ? a[i] : a[i + 2], 8);
      float r = (h4 ? b[1] : b[0]) + __shfl_xor_sync (0xffffffffu, h4 ? b[0] : b[1], 4);
      r += __shfl_xor_sync (0xffffffffu, r, 2);
      r += __shfl_xor_sync (0xffffffffu, r, 1);
      const int g = (lane >> 2) & 3, m = m0 + g;
      if ((lane & 3) == 0 && m < n_valid)
        {
          reinterpret_cast<float *> (out + (size_t) m * n_ent)[lane >> 4] = r * kSlideDbPerLog2;
          if (lane < 16)
            flag[(size_t) m * n_ent] = counted (m);
        }
    }
}

// per (candidate, offset, sync bit): add the per-frame sums in frame order, count the frames that were used
// -> out_ud[((c*65 + o)*n_bits + bit)*2 + {0,1}] = umag, dmag; out_cnt = frames used; out_valid[c*65 + o]
__global__ void
k_refine_reduce (const float2 *__restrict__ ent_ud, const unsigned char *__restrict__ ent_flag, int n_cand, int n_ent,
                 const int *__restrict__ g_bit_off, int n_bits, const long long *__restrict__ cand_start, const int *__restrict__ cand_noff,
                 long long n_frames, int total_frame_count,
                 float *__restrict__ out_ud, int *__restrict__ out_cnt, unsigned char *__restrict__ out_valid)
{
  const long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long) n_cand * kOffsets * n_bits)
    return;
  const int c = int (i / (kOffsets * n_bits)), o = int ((i / n_bits) % kOffsets), bit = int (i % n_bits);
  const long long fine = cand_start[c] + 8LL * o;
  const bool valid = o < cand_noff[c] && fine + (long long) total_frame_count * kFrame <= n_frames;
  if (bit == 0)
    out_valid[c * kOffsets + o] = valid ? 1 : 0;
  if (!valid)
    return;
  const float2 *ud = ent_ud + ((size_t) c * kOffsets + o) * n_ent;
  const unsigned char *fl = ent_flag + ((size_t) c * kOffsets + o) * n_ent;
  float umag = 0.f, dmag = 0.f;
  int cnt = 0;
  for (int e = g_bit_off[bit]; e < g_bit_off[bit + 1]; e++)
    if (fl[e])
      {
        const float2 v = ud[e];
        umag += v.x;
        dmag += v.y;
        cnt++;
      }
  const size_t ob = ((size_t) c * kOffsets + o) * n_bits + bit;
  out_ud[ob * 2] = umag;
  out_ud[ob * 2 + 1] = dmag;
  out_cnt[ob] = cnt;
}

} // namespace awm

namespace awm {

// ---- exact scoring of a list of (candidate, offset) pairs: the ones the sliding pass picks, or every valid offset --------------
// The transforms run in parallel (warp = one pair x one sync frame, time-domain window and arithmetic of frame_db_sum, i.e. of the
// reference's sync_fft) and only the additions stay serial: k_refine_exact_sum_n adds the stored band values of a bit in the
// reference's order (frames ascending, 30 up / 30 down bands each).  The list's length is written by the device (k_refine_rank) or
// the host; a fixed grid walks the jobs.
constexpr int kExactWarps = 8;

/* one (pair, sync frame) job of k_refine_exact_fft_n */
__device__ __forceinline__ void
refine_exact_fft_job (const float *__restrict__ pcm, long long n_frames, int C, const long long *__restrict__ pair_start,
                      const awm_sync_entry *__restrict__ g_ent, int n_ent, float *__restrict__ vals, const FftSmem& s, float *sband,
                      int lane, long long job)
{
  const int p = int (job / n_ent), e = int (job % n_ent);
  const awm_sync_entry *en = g_ent + e;
  const long long start = pair_start[p] + (long long) en->frame * kFrame;
  float acc[4];
  frame_db_sum (pcm, n_frames, C, start, s, lane, acc);
  bands_to_array (acc, lane, sband, 1);
  __syncwarp();
  float *o = vals + ((size_t) p * n_ent + e) * (2 * kUD);
  if (lane < kUD)
    {
      o[lane] = sband[en->up[lane]];
      o[kUD + lane] = sband[en->down[lane]];
    }
}

__global__ void __launch_bounds__ (kExactWarps * 32, 2)
k_refine_exact_fft_n (const float *__restrict__ pcm, long long n_frames, int C, const long long *__restrict__ pair_start, const int *__restrict__ n_pairs,
                      const awm_sync_entry *__restrict__ g_ent, int n_ent, float *__restrict__ vals, const float2 *g_tw, const float *g_win)
{
  extern __shared__ __align__ (16) unsigned char smem[];
  FftSmem s = fft_smem_setup (smem, g_tw, g_win, kExactWarps);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float *sband = s.extra + w * 96;
  const long long n_jobs = (long long) *n_pairs * n_ent;
  for (long long job = (long long) blockIdx.x * kExactWarps + w; job < n_jobs; job += (long long) gridDim.x * kExactWarps)
    {
      __syncwarp();                               // the previous job's band values are read from sband
      refine_exact_fft_job (pcm, n_frames, C, pair_start, g_ent, n_ent, vals, s, sband, lane, job);
    }
}

// One warp per (pair, sync bit, up / down): the 30 band values of every frame of the bit are first staged in shared memory by the
// whole warp (coalesced), then lane 0 adds them one after the other in the reference's order -- the chain of ~2550 dependent float
// additions is what this kernel's time consists of, the loads no longer sit between them.
constexpr int kExactSumWarps = 4;

/* one (pair, sync bit, up / down) job of k_refine_exact_sum_n */
__device__ __forceinline__ void
refine_exact_sum_job (const float *__restrict__ vals, const long long *__restrict__ pair_start, long long n_frames, int C,
                      const awm_sync_entry *__restrict__ g_ent, int n_ent, const int *__restrict__ g_bit_off, int n_bits, int total_frame_count,
                      long long wav_first, long long wav_last, float *__restrict__ out_ud, int *__restrict__ out_cnt,
                      unsigned char *__restrict__ out_valid, float *stage, int lane, int i)
{
  const int p = i / (n_bits * 2), bit = (i / 2) % n_bits, which = i & 1;       // which: 0 = up bands, 1 = down bands
  const long long fine = pair_start[p];
  const bool valid = fine + (long long) total_frame_count * kFrame <= n_frames;
  if (bit == 0 && which == 0 && lane == 0)
    out_valid[p] = valid ? 1 : 0;
  if (!valid)
    return;
  const int e0 = g_bit_off[bit], e1 = g_bit_off[bit + 1];
  for (int k = lane; k < (e1 - e0) * kUD; k += 32)
    stage[k] = __ldg (vals + ((size_t) p * n_ent + e0 + k / kUD) * (2 * kUD) + which * kUD + k % kUD);
  __syncwarp();
  if (lane != 0)
    return;
  float mag = 0.f;
  int cnt = 0;
  for (int e = e0; e < e1; e++)
    {
      const long long start = fine + (long long) g_ent[e].frame * kFrame;
      const long long f_first = start * C, f_last = (start + kFrame) * C;
      if (f_last < wav_first || f_first > wav_last)        // frames in digital silence are not counted
        continue;
      const float *v = stage + (e - e0) * kUD;
#pragma unroll
      for (int k = 0; k < kUD; k++)
        mag = __fadd_rn (mag, v[k]);
      cnt++;
    }
  out_ud[((size_t) p * n_bits + bit) * 2 + which] = mag;
  if (which == 0)
    out_cnt[(size_t) p * n_bits + bit] = cnt;
}

__global__ void __launch_bounds__ (kExactSumWarps * 32)
k_refine_exact_sum_n (const float *__restrict__ vals, const long long *__restrict__ pair_start, const int *__restrict__ n_pairs, long long n_frames, int C,
                      const awm_sync_entry *__restrict__ g_ent, int n_ent, const int *__restrict__ g_bit_off, int n_bits, int total_frame_count,
                      long long wav_first, long long wav_last, int max_bit_frames,
                      float *__restrict__ out_ud, int *__restrict__ out_cnt, unsigned char *__restrict__ out_valid)
{
  extern __shared__ __align__ (16) unsigned char smem[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float *stage = reinterpret_cast<float *> (smem) + size_t (w) * max_bit_frames * kUD;
  const int n_jobs = *n_pairs * n_bits * 2;
  for (int i = blockIdx.x * kExactSumWarps + w; i < n_jobs; i += gridDim.x * kExactSumWarps)
    {
      __syncwarp();                               // lane 0 of the previous job has finished reading the stage
      refine_exact_sum_job (vals, pair_start, n_frames, C, g_ent, n_ent, g_bit_off, n_bits, total_frame_count, wav_first, wav_last,
                            out_ud, out_cnt, out_valid, stage, lane, i);
    }
}


// ---- which offsets the exact kernels re-score --------------------------------------------------------------------------------
// The rule of awm_sync_refine on the sums of k_refine_reduce, without a host round trip: per candidate the sync_decode quality of
// every valid sliding offset (the host's quality_of, src/syncfinder.cc:94-114,144-152, in double and in the same order of
// operations: float ratio, then the double products and sums unfused), every offset whose -|q - local_mean| lies within `margin`
// of the smallest one, and the offset of the approx index if it is valid.  Output: the (start, candidate, offset) list in
// candidate order, offsets ascending, and its length.  One CTA: warps own candidates, thread 0 places them one after the other.
constexpr int kRankWarps = 32;

__device__ __forceinline__ double
rank_quality (const float *__restrict__ ud, const int *__restrict__ cnt, size_t base, int n_bits, double norm_div)
{
  double sync_quality = 0;
  int bit_count = 0;
  for (int bit = 0; bit < n_bits; bit++)
    {
      const size_t ob = base * n_bits + bit;
      const float umag = ud[ob * 2], dmag = ud[ob * 2 + 1];
      double raw_bit;
      if (umag == 0 || dmag == 0)
        raw_bit = 0;
      else if (umag < dmag)
        raw_bit = __fsub_rn (1.f, __fdiv_rn (umag, dmag));
      else
        raw_bit = __fsub_rn (__fdiv_rn (dmag, umag), 1.f);
      sync_quality = __dadd_rn (sync_quality, __dmul_rn ((bit & 1) ? raw_bit : -raw_bit, double (cnt[ob])));
      bit_count += cnt[ob];
    }
  if (bit_count)
    sync_quality = __ddiv_rn (sync_quality, double (bit_count));
  return __ddiv_rn (__ddiv_rn (sync_quality, norm_div), 2.9);
}

__global__ void __launch_bounds__ (kRankWarps * 32)
k_refine_rank (const float *__restrict__ ud, const int *__restrict__ cnt, const unsigned char *__restrict__ valid,
               const awm_search_score *__restrict__ cand, const long long *__restrict__ cand_start, const int *__restrict__ cand_noff,
               int nc, int n_bits, double norm_div, double margin, unsigned *__restrict__ keep /* [nc][3] */, int *__restrict__ first /* [nc] */,
               long long *__restrict__ out_start, int *__restrict__ out_cand, int *__restrict__ out_off, int *__restrict__ out_n)
{
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int c = w; c < nc; c += kRankWarps)
    {
      double key[3];
      bool ok[3];
      double best = __longlong_as_double (0x7ff0000000000000LL);      // +inf
      for (int k = 0; k < 3; k++)
        {
          const int o = lane + 32 * k;
          ok[k] = o < cand_noff[c] && valid[(size_t) c * kOffsets + o];
          key[k] = ok[k] ? -fabs (__dsub_rn (rank_quality (ud, cnt, (size_t) c * kOffsets + o, n_bits, norm_div), cand[c].local_mean)) : 0.0;
          if (ok[k] && key[k] < best)
            best = key[k];
        }
      for (int d = 16; d; d >>= 1)
        best = fmin (best, __shfl_xor_sync (0xffffffffu, best, d));
      const double limit = __dadd_rn (best, margin);
      const int o_self = int (((long long) cand[c].index - cand_start[c]) / 8);
      for (int k = 0; k < 3; k++)
        {
          const int o = lane + 32 * k;
          const bool kept = ok[k] && (key[k] <= limit || o == o_self);
          const unsigned m = __ballot_sync (0xffffffffu, kept);
          if (lane == 0)
            keep[c * 3 + k] = m;
        }
    }
  __syncthreads();
  if (threadIdx.x == 0)
    {
      int n = 0;
      for (int c = 0; c < nc; c++)
        {
          first[c] = n;
          n += __popc (keep[c * 3]) + __popc (keep[c * 3 + 1]) + __popc (keep[c * 3 + 2]);
        }
      *out_n = n;
    }
  __syncthreads();
  for (int c = w; c < nc; c += kRankWarps)
    {
      int pos = first[c];
      for (int k = 0; k < 3; k++)
        {
          const unsigned m = keep[c * 3 + k];
          if (m >> lane & 1)
            {
              const int at = pos + __popc (m & ((1u << lane) - 1));
              const int o = lane + 32 * k;
              out_start[at] = cand_start[c] + 8LL * o;
              out_cand[at] = c;
              out_off[at] = o;
            }
          pos += __popc (m);
        }
    }
}

} // namespace awm
