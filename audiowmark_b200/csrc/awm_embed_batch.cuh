// awm_embed_batch.cuh -- batched embed: many items of one packed buffer, one payload per item (and with awm_embed_batch_keys one key
// per item), in one launch of k_embed_batch and one of k_limiter_batch (awm_embed_batch / awm_embed_batch_offsets in awm_capi.cu).
//
// Work list: every item with at least one sample-frame contributes ceil((F+1)/14) tiles of k_embed's shape (14 output frames +
// one halo frame on each side) and ceil(F/4096) limiter CTAs; a CTA finds its item by binary search over the items' first tile
// (first limiter CTA).  All tiles cost the same, so the grid is balanced over the SMs whatever the item lengths.  A tile runs
// k_embed's code (embed_tile) on its item as if the item were the end of a stream that began zero_frames (z) earlier with
// silence (add_stream_watermark with zero_frames, src/wmadd.cc:501-580): table rows, synthesis and limiter blocks are those of
// the whole stream, own --snr sums over the item's own positions, the item's end is the stream's end.  z = 0 is awm_embed with
// first_frame_number 0.  The silent prefix is never in memory: the processed range starts at stream frame frame0 =
// max (floor (z / 1024) - 1, 0) -- the frame before the item's first one receives that frame's synthesis spill, which the limiter
// block peaks must see -- and its first lead = z - 1024 * frame0 positions read as zero and are not written.  Earlier frames of
// the stream are silent and carry no watermark.  The frame-mod row of a frame is formed per warp in shared memory from the key's
// role table and the item's coded bits (role_frame_mod); no per-item table exists.
#pragma once
#include "awm_kernels.cuh"
#include "awm_roles.hh"

namespace awm {

struct BatchItem
{
  long long v0;                // first value of the item in the packed buffer
  long long n_frames;          // > 0
  int C;
  int item;                    // index in the caller's list: coded bits and --snr slot
  long long tile0;             // first k_embed_batch CTA of the item
  long long lim0;              // first k_limiter_batch CTA of the item
  long long peak0, n_blocks;   // the item's limiter block peaks: peaks[peak0 .. peak0 + n_blocks)
  long long frame0;            // stream 1024-frame where the processed range starts (0 for z < 2048)
  long long lead;              // processed positions before the item's first sample: z - 1024 * frame0, in [0, 2048)
  long long blk0;              // limiter block of stream position 1024 * frame0: peaks[peak0] belongs to it
  int role_table;              // the item's role table: roles [role_table] (0 with one key per batch; awm_embed_batch_keys: its key's)
};

constexpr int kBatchRow = 104;           // per-warp frame-mod row in shared memory (101 bins, padded)
constexpr size_t kEmbedBatchSmem = kEmbedSmem + size_t (kEmbedWarps) * kBatchRow;

// index of the item a CTA belongs to: the last one whose first CTA is <= cta (first CTAs strictly increase)
template<bool LIMITER> __device__ __forceinline__ int
batch_item_of (const BatchItem *__restrict__ items, int n_items, long long cta)
{
  int lo = 0, hi = n_items - 1;
  while (lo < hi)
    {
      const int mid = (lo + hi + 1) >> 1;
      if ((LIMITER ? items[mid].lim0 : items[mid].tile0) <= cta)
        lo = mid;
      else
        hi = mid - 1;
    }
  return lo;
}

// base: the fields all items share (tables, strength, limiter block, peaks / snr base pointers, frame_number0 of a stream start);
// in / out point to the packed buffer.  A tile's frames count from the item's frame0, positions from frame0 * 1024.
// OFFSETS = false: every item starts its stream (frame0 = lead = blk0 = 0), the code of that case alone (awm_embed_batch).
// KEYS = true: every item reads its own role table roles [role_table] (awm_embed_batch_keys); false: all read roles [0].
template<bool OFFSETS, bool KEYS> __global__ void __launch_bounds__ (kEmbedWarps * 32, 1)
k_embed_batch (EmbedArgs base, const BatchItem *__restrict__ items, int n_items, const uint16_t *__restrict__ roles,
               const uint8_t *__restrict__ coded, int n_coded)
{
  extern __shared__ __align__ (16) unsigned char smem[];
  const long long cta = blockIdx.x;
  const BatchItem it = items[batch_item_of<false> (items, n_items, cta)];
  EmbedArgs A = base;
  A.in = base.in + it.v0;
  A.out = base.out + it.v0;
  A.n_frames = OFFSETS ? it.lead + it.n_frames : it.n_frames;   // the processed range ends with the stream
  A.C = it.C;
  A.n_proc = (A.n_frames + kFrame - 1) / kFrame + 1;
  A.frame_begin = 0;
  A.frame_end = A.n_proc;
  if (OFFSETS)
    {
      A.frame_number0 = base.frame_number0 + it.frame0;
      A.stream_pos0 = it.frame0 * kFrame;
      A.blk0 = it.blk0;
      A.snr_pos0 = it.lead;                                 // in / out begin here; --snr counts the item's own positions (awm_embed_window)
    }
  A.peaks = base.peaks + it.peak0;
  A.snr = base.snr ? base.snr + 2 * it.item : nullptr;
  A.snr_frames = A.limiter_block > 0 ? A.n_proc : A.n_proc - 1;   // as awm_embed: frames the reference loop emits
  uint8_t *row = smem + kEmbedSmem + (threadIdx.x >> 5) * kBatchRow;
  const uint8_t *item_coded = coded + (size_t) it.item * 2 * n_coded;
  const int lane = threadIdx.x & 31;
  auto fm_row = [&] (long long r)
    {
      const int ab = r >= A.fpb;                            // rows [0,fpb) = A, [fpb,2fpb) = B
      const uint16_t *role = roles + (size_t) (r + (long long) ((KEYS ? it.role_table : 0) - ab) * A.fpb) * (kMaxBand + 1);
      for (int k = lane; k <= kMaxBand; k += 32)
        row[k] = role_frame_mod (role[k], ab, item_coded + ab * n_coded);
      __syncwarp();
      return (const uint8_t *) row;
    };
  /* a stereo item that starts at an odd value of the packed buffer cannot be read as float2 */
  if (((reinterpret_cast<uintptr_t> (A.in) | reinterpret_cast<uintptr_t> (A.out)) & 7) == 0)
    embed_tile<true, OFFSETS> (A, (cta - it.tile0) * kEmbedTile, smem, fm_row);
  else
    embed_tile<false, OFFSETS> (A, (cta - it.tile0) * kEmbedTile, smem, fm_row);
}

// k_limiter over every item's own positions and block peaks, on the stream's block grid; out is the packed buffer
__global__ void
k_limiter_batch (float *__restrict__ out, const BatchItem *__restrict__ items, int n_items, int block, float ceiling, const unsigned *__restrict__ peaks)
{
  const long long cta = blockIdx.x;
  const BatchItem it = items[batch_item_of<true> (items, n_items, cta)];
  limiter_cta (out + it.v0, it.lead + (cta - it.lim0) * blockDim.x * kLimiterIter, it.lead + it.n_frames, it.C, block, ceiling, peaks + it.peak0,
               it.n_blocks, it.frame0 * kFrame, it.lead);
}

} // namespace awm
