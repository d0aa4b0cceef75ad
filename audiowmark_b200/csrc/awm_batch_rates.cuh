// awm_batch_rates.cuh -- batched embed of items at any sample rate (awm_embed_batch_rates in awm_capi.cu): the add loop with a
// WatermarkResampler (src/wmadd.cc:353-430, 548-566) for many items of one packed buffer, each at its own rate, with one launch per step.
//
//   k_resample_batch      in-resampler (:392-393): item PCM -> the item at the watermark rate (scratch, zero extended as the loop
//                         keeps feeding zero frames: n_stop "never")
//   (k_embed_batch)       WatermarkGen::run on it (:394-399), delta_only: the watermark signal alone (scratch)
//   k_resample_mix_batch  out-resampler (:401-406) fused with the mixer (:548-566): for every frame the add loop emits, the watermark
//                         resampled back to the item's rate + the input, the item's limiter block peaks and --snr sums
//   k_limiter_rates       k_limiter per item with the item's own block size
//
// Work lists as in k_embed_batch: all CTAs of a launch cost the same (256 output frames of one resampling job, 4096 limiter
// positions), every item contributes its own number of them, a CTA finds its item by binary search over the items' first CTA.
//
// OFFSETS = true (awm_embed_batch_rates_offsets): the item continues a stream that began z frames earlier with silence.  Both
// resamplers run at stream positions, so t = (h-1) + n step is the whole stream's, while the item and the scratch are indexed at
// stream position minus their origin and read as zero outside.  The scratch holds the stream at the watermark rate from w0 on
// (a whole 1024-frame before the first frame that can see the item: the whole stream's x44 and watermark are exactly zero before
// it); the mixer starts at i0, the first position whose watermark can be non-zero, so positions [i0, z) count for the limiter
// block peaks of the stream's block grid without being written.  OFFSETS = false is the stream-start case alone.
#pragma once
#include "awm_kernels.cuh"
#include "awm_speed.cuh"

namespace awm {

struct RateItem
{
  const float *in;             // the item in the packed input: n_frames x C
  float *out;                  // the item in the packed output
  float *x44, *wm44;           // scratch: the item at the watermark rate and its watermark signal, n44 x C each
  long long n_frames, n_emit, n44;
  int C, item;                 // item: index in the caller's list (--snr slot)
  double step_in, step_out;    // input frames per output frame of the in- and out-resampler
  int h_in, h_out;
  const float *coef_in, *coef_out;
  int limiter_block;           // sample_rate * ms / 1000 of this item; 0 = off
  long long peak0, n_blocks;   // its limiter block peaks: peaks[peak0 .. peak0 + n_blocks)
  long long rs0, mix0, lim0;   // first CTA of the item in k_resample_batch / k_resample_mix_batch / k_limiter_rates
  // stream origin (OFFSETS only; all 0 for an item that starts its stream): n44 counts from w0, n_emit from i0, peaks from blk0
  long long z;                 // stream position of the item's first frame (input rate)
  long long w0;                // stream position (watermark rate) of the scratch's first frame, a multiple of 1024
  long long i0;                // first stream position (input rate) whose watermark can be non-zero, <= z
  long long blk0;              // i0 / limiter_block: the limiter block of peaks[peak0]
  long long snr0, snr1;        // stream positions [snr0, snr1) the --snr sums count (OFFSETS only): [z, z + n_emit) unless a window narrows them
};

constexpr int kRateCta = 256;  // threads (= output frames) per resampling CTA

enum { kRateRs, kRateMix, kRateLim };

// the last item whose first CTA is <= cta (items without CTAs of this kind repeat the next item's first CTA)
template<int KIND> __device__ __forceinline__ const RateItem&
rate_item_of (const RateItem *__restrict__ items, int n_items, long long cta)
{
  int lo = 0, hi = n_items - 1;
  while (lo < hi)
    {
      const int mid = (lo + hi + 1) >> 1;
      const RateItem& m = items[mid];
      if ((KIND == kRateRs ? m.rs0 : KIND == kRateMix ? m.mix0 : m.lim0) <= cta)
        lo = mid;
      else
        hi = mid - 1;
    }
  return items[lo];
}

// stereo as float2 where both buffers allow it (an item at an odd value of the packed buffer does not); same values either way
__device__ __forceinline__ bool
rate_vec2 (int C, const void *a, const void *b)
{
  return C == 2 && ((reinterpret_cast<uintptr_t> (a) | reinterpret_cast<uintptr_t> (b)) & 7) == 0;
}

template<bool OFFSETS> __global__ void __launch_bounds__ (kRateCta)
k_resample_batch (const RateItem *__restrict__ items, int n_items)
{
  const RateItem& it = rate_item_of<kRateRs> (items, n_items, blockIdx.x);
  ResampleJob J;
  J.in = it.in;
  J.out = it.x44;
  J.n_in = it.n_frames;
  J.n_out = it.n44;
  J.n_stop = LLONG_MAX / 4;
  J.step = it.step_in;
  J.h = it.h_in;
  J.coef = it.coef_in;
  const long long n = ((long long) blockIdx.x - it.rs0) * kRateCta + threadIdx.x;
  if (n >= J.n_out)
    return;
  const int C = it.C;
  float *o = J.out + n * C;
  ResamplePos P;
  if (!resample_pos (J, OFFSETS ? it.w0 + n : n, P))
    {
      for (int ch = 0; ch < C; ch++)
        o[ch] = 0.0f;
      return;
    }
  if (OFFSETS)
    P.i0 -= it.z;                                           // stream input frame -> frame of the item
  if (rate_vec2 (C, J.in, J.out))
    reinterpret_cast<float2 *> (J.out)[n] = resample_dot2 (J, P);
  else
    for (int ch = 0; ch < C; ch++)
      o[ch] = resample_dot (J, P, C, ch);
}

// frame i < n_emit of an item: y = wm + orig (orig is zero beyond n_frames), stored for i < n_frames; peak of |y| per limiter block
// of the item (only peaks above the ceiling matter, Limiter::block_max starts at the ceiling); --snr sums of wm and orig.  The
// watermark is resampled by the operations of k_resample and stays in registers.  OFFSETS: stream position i = i0 + thread's frame
// is the item's frame i - z; positions before z are not stored, and only positions in [snr0, snr1) are summed for --snr.
template<bool OFFSETS> __global__ void __launch_bounds__ (kRateCta)
k_resample_mix_batch (const RateItem *__restrict__ items, int n_items, float ceiling, unsigned *__restrict__ peaks, double *__restrict__ snr)
{
  const RateItem& it = rate_item_of<kRateMix> (items, n_items, blockIdx.x);
  ResampleJob J;
  J.in = it.wm44;
  J.out = nullptr;
  J.n_in = it.n44;
  J.n_out = it.n_emit;
  J.n_stop = LLONG_MAX / 4;
  J.step = it.step_out;
  J.h = it.h_out;
  J.coef = it.coef_out;
  const long long k = ((long long) blockIdx.x - it.mix0) * kRateCta + threadIdx.x;
  const long long i = OFFSETS ? it.i0 + k : k;              // stream position
  const long long q = OFFSETS ? i - it.z : i;               // frame of the item
  const int C = it.C;
  const bool own = OFFSETS ? q >= 0 && q < it.n_frames : i < it.n_frames;
  const bool counts = !OFFSETS || (i >= it.snr0 && i < it.snr1);   // --snr: the item's own positions, or a window's owned part
  double sd = 0, ss = 0;
  if (k < J.n_out)
    {
      ResamplePos P;
      const bool live = resample_pos (J, i, P);
      if (OFFSETS)
        P.i0 -= it.w0;                                      // stream frame at the watermark rate -> frame of the scratch
      float mx = 0.f;
      auto mix = [&] (int c, float w)
        {
          const float o = own ? __ldg (it.in + q * C + c) : 0.f;
          const float y = __fadd_rn (w, o);
          if (own)
            it.out[q * C + c] = y;
          mx = fmaxf (mx, fabsf (y));
          if (counts)
            {
              sd += double (w) * double (w);
              ss += double (o) * double (o);
            }
        };
      if (rate_vec2 (C, J.in, J.in))
        {
          const float2 w = live ? resample_dot2 (J, P) : make_float2 (0.0f, 0.0f);
          mix (0, w.x);
          mix (1, w.y);
        }
      else
        for (int c = 0; c < C; c++)
          mix (c, live ? resample_dot (J, P, C, c) : 0.0f);
      if (it.limiter_block > 0 && mx > ceiling)
        atomicMax (peaks + it.peak0 + (OFFSETS ? i / it.limiter_block - it.blk0 : i / it.limiter_block), __float_as_uint (mx));
    }
  if (snr)
    {
      for (int d = 16; d > 0; d >>= 1)
        {
          sd += __shfl_xor_sync (0xffffffffu, sd, d);
          ss += __shfl_xor_sync (0xffffffffu, ss, d);
        }
      if ((threadIdx.x & 31) == 0 && (sd != 0 || ss != 0))
        {
          atomicAdd (snr + 2 * it.item, sd);
          atomicAdd (snr + 2 * it.item + 1, ss);
        }
    }
}

// OFFSETS: positions count from i0 on the stream's block grid; the item's own frames begin at z - i0
template<bool OFFSETS> __global__ void
k_limiter_rates (const RateItem *__restrict__ items, int n_items, float ceiling, const unsigned *__restrict__ peaks)
{
  const RateItem& it = rate_item_of<kRateLim> (items, n_items, blockIdx.x);
  const long long first = ((long long) blockIdx.x - it.lim0) * blockDim.x * kLimiterIter;
  if (OFFSETS)
    {
      const long long lead = it.z - it.i0;
      limiter_cta (it.out, lead + first, lead + it.n_frames, it.C, it.limiter_block, ceiling, peaks + it.peak0, it.n_blocks, it.i0, lead);
    }
  else
    limiter_cta (it.out, first, it.n_frames, it.C, it.limiter_block, ceiling, peaks + it.peak0, it.n_blocks, 0);
}

} // namespace awm
