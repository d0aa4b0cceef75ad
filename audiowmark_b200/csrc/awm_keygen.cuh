// awm_keygen.cuh -- role tables of many keys built on the device (awm_set_embed_roles_keys): k_embed_roles_keys writes, for each
// of n_keys 16-byte AES keys, exactly the table gen_embed_roles (host/awm_tables.cc) builds on the host, uint16 [fpb][101].
//
// The keyed generator is Random (host/awm_random.cc): draw i after seed (s, stream) is big-endian u64 word i % 2 of
// AES_k (ctr0 + i / 2), ctr0 = AES_k (be64 (s) || stream || 0^7), the counter one 128-bit big-endian integer.  Every draw can
// therefore be computed on its own; only the swaps of a Fisher-Yates shuffle (j = i + r % (n - i)) are serial.  One CTA per key:
//   1. S-box (inverse in GF(2^8) + affine map), one T-table, the key schedule and the two counter blocks in shared memory;
//   2. the whole CTA computes the j of every swap of BitPosGen (stream frame_position, fpb slots) and of the mix shuffle
//      (stream mix, data_frames * 30 entries) into global scratch;
//   3. warp 1 lane 0 applies the mix swaps to an index array in shared memory (u16; in global memory past 65536 entries) while
//      warp 0 lane 0 applies the BitPosGen swaps and then, with warps 2.., shuffles the 81 bands of every frame (UpDownGen:
//      streams sync_up_down / data_up_down, one reseed per frame), one warp per frame with the bands in registers (lane l
//      holds positions l, l + 32, l + 64; only the first 60 swaps decide the 30 up and 30 down bands);
//   4. sync frames and, without mix, data entries are written as they are found; with mix every entry e reads the entry it
//      came from (index array) and its bands (scratch) and takes coded bit e / 30 / frames_per_bit.
// A (frame, bin) written twice (16-bit atomicCAS on a zeroed table) sets the key's error flag, as gen_embed_roles reports it.
#pragma once
#include "awm_roles.hh"
#include <stdint.h>

namespace awm {

constexpr int kKeygenThreads = 512;
constexpr int kKeygenBands = AWM_MAX_BAND - AWM_MIN_BAND + 1;      // UpDownGen shuffles bands 20..100
constexpr int kKeygenUpDown = 2 * AWM_BANDS_PER_FRAME;             // swaps that decide the up and down bands
constexpr int kKeygenSmemIdxMax = 65536;                           // mix entries whose index array is u16 in shared memory
constexpr int kKeygenStreamDataUpDown = 1, kKeygenStreamSyncUpDown = 2, kKeygenStreamMix = 4, kKeygenStreamFramePosition = 6;

struct KeygenLayout
{
  int sync_frames, sync_frames_per_bit, data_frames, frames_per_bit, mix;
  int fpb, n_mix;              // sync_frames + data_frames; data_frames * AWM_BANDS_PER_FRAME
  long long j_stride;          // u32 j values per key in the scratch: BitPosGen's, then the mix's, each padded to 16
  int j_mix0;                  // offset of the mix's j values
};

// shared memory: T0 [256] u32 | key schedule [44] u32 | counter blocks [2][4] u32 | S-box [256] | pos [fpb] u16 | mix index [n_mix] u16
constexpr size_t kKeygenSmemFixed = 256 * 4 + 44 * 4 + 8 * 4 + 256;
__host__ __device__ inline size_t keygen_pos_bytes (int fpb) { return (size_t (fpb) * 2 + 15) & ~size_t (15); }
inline size_t keygen_smem (int fpb, int n_mix, bool smem_idx) { return kKeygenSmemFixed + keygen_pos_bytes (fpb) + (smem_idx ? size_t (n_mix) * 2 : 0); }

__device__ __forceinline__ uint32_t kg_bswap (uint32_t x) { return __byte_perm (x, 0, 0x0123); }
__device__ __forceinline__ uint8_t kg_xtime (uint32_t x) { return uint8_t ((x << 1) ^ ((x & 0x80) ? 0x1B : 0)); }

__device__ __forceinline__ uint8_t
kg_gf_mul (uint32_t a, uint32_t b)
{
  uint32_t r = 0;
  for (int i = 0; i < 8; i++)
    {
      if (b & 1)
        r ^= a;
      a = kg_xtime (a);
      b >>= 1;
    }
  return uint8_t (r);
}

// AES S-box entry: x^254 (the inverse, 0 for 0) through the affine map
__device__ __forceinline__ uint8_t
kg_sbox (uint32_t x)
{
  uint32_t r = 1, base = x;
  for (int e = 254; e; e >>= 1)
    {
      if (e & 1)
        r = kg_gf_mul (r, base);
      base = kg_gf_mul (base, base);
    }
  const uint32_t q = r | (r << 8);
  const uint32_t s = q ^ (q >> 7) ^ (q >> 6) ^ (q >> 5) ^ (q >> 4);     // q ^ rotl (q, 1..4) in the low byte
  return uint8_t ((s ^ 0x63) & 0xff);
}

// one AES-128 block; state and result as little-endian column words (byte (r, c) in bits 8r.. of word c), as encrypt_block
__device__ __forceinline__ void
kg_aes (const uint32_t *T0, const uint8_t *sb, const uint32_t *rk, uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3)
{
  c0 ^= rk[0]; c1 ^= rk[1]; c2 ^= rk[2]; c3 ^= rk[3];
#pragma unroll 1
  for (int round = 1; round < 10; round++)
    {
      const uint32_t *k = rk + 4 * round;
      const uint32_t n0 = T0[c0 & 0xff] ^ __funnelshift_l (T0[(c1 >> 8) & 0xff], T0[(c1 >> 8) & 0xff], 8) ^
                          __funnelshift_l (T0[(c2 >> 16) & 0xff], T0[(c2 >> 16) & 0xff], 16) ^ __funnelshift_l (T0[c3 >> 24], T0[c3 >> 24], 24) ^ k[0];
      const uint32_t n1 = T0[c1 & 0xff] ^ __funnelshift_l (T0[(c2 >> 8) & 0xff], T0[(c2 >> 8) & 0xff], 8) ^
                          __funnelshift_l (T0[(c3 >> 16) & 0xff], T0[(c3 >> 16) & 0xff], 16) ^ __funnelshift_l (T0[c0 >> 24], T0[c0 >> 24], 24) ^ k[1];
      const uint32_t n2 = T0[c2 & 0xff] ^ __funnelshift_l (T0[(c3 >> 8) & 0xff], T0[(c3 >> 8) & 0xff], 8) ^
                          __funnelshift_l (T0[(c0 >> 16) & 0xff], T0[(c0 >> 16) & 0xff], 16) ^ __funnelshift_l (T0[c1 >> 24], T0[c1 >> 24], 24) ^ k[2];
      const uint32_t n3 = T0[c3 & 0xff] ^ __funnelshift_l (T0[(c0 >> 8) & 0xff], T0[(c0 >> 8) & 0xff], 8) ^
                          __funnelshift_l (T0[(c1 >> 16) & 0xff], T0[(c1 >> 16) & 0xff], 16) ^ __funnelshift_l (T0[c2 >> 24], T0[c2 >> 24], 24) ^ k[3];
      c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    }
  auto last = [&] (uint32_t a, uint32_t b, uint32_t c, uint32_t d, uint32_t k)
    {
      return (uint32_t (sb[a & 0xff]) | (uint32_t (sb[(b >> 8) & 0xff]) << 8) | (uint32_t (sb[(c >> 16) & 0xff]) << 16) |
              (uint32_t (sb[d >> 24]) << 24)) ^ k;
    };
  const uint32_t o0 = last (c0, c1, c2, c3, rk[40]), o1 = last (c1, c2, c3, c0, rk[41]);
  const uint32_t o2 = last (c2, c3, c0, c1, rk[42]), o3 = last (c3, c0, c1, c2, rk[43]);
  c0 = o0; c1 = o1; c2 = o2; c3 = o3;
}

// counter block of seed (s, stream): AES (be64 (s) || stream || 0^7)
__device__ __forceinline__ void
kg_seed (const uint32_t *T0, const uint8_t *sb, const uint32_t *rk, unsigned long long s, int stream, uint32_t ctr[4])
{
  uint32_t c0 = kg_bswap (uint32_t (s >> 32)), c1 = kg_bswap (uint32_t (s)), c2 = uint32_t (stream), c3 = 0;
  kg_aes (T0, sb, rk, c0, c1, c2, c3);
  ctr[0] = c0; ctr[1] = c1; ctr[2] = c2; ctr[3] = c3;
}

// draws 2b and 2b + 1 after the seed whose counter block is ctr: AES (ctr + b), read as two big-endian u64
__device__ __forceinline__ void
kg_draws (const uint32_t *T0, const uint8_t *sb, const uint32_t *rk, const uint32_t ctr[4], unsigned long long b,
          unsigned long long& r0, unsigned long long& r1)
{
  const unsigned long long hi = (static_cast<unsigned long long> (kg_bswap (ctr[0])) << 32) | kg_bswap (ctr[1]);
  const unsigned long long lo = (static_cast<unsigned long long> (kg_bswap (ctr[2])) << 32) | kg_bswap (ctr[3]);
  const unsigned long long lo2 = lo + b, hi2 = hi + (lo2 < lo ? 1 : 0);
  uint32_t c0 = kg_bswap (uint32_t (hi2 >> 32)), c1 = kg_bswap (uint32_t (hi2)), c2 = kg_bswap (uint32_t (lo2 >> 32)), c3 = kg_bswap (uint32_t (lo2));
  kg_aes (T0, sb, rk, c0, c1, c2, c3);
  r0 = (static_cast<unsigned long long> (kg_bswap (c0)) << 32) | kg_bswap (c1);
  r1 = (static_cast<unsigned long long> (kg_bswap (c2)) << 32) | kg_bswap (c3);
}

// the swaps of a Fisher-Yates shuffle of v [n] with precomputed j (16-byte aligned, readable up to a multiple of 4 entries), by one
// thread; the j loads run 32 swaps ahead of their use
template<class IDX> __device__ __forceinline__ void
kg_serial_shuffle (IDX *v, const uint32_t *__restrict__ j, int n)
{
  const uint4 *jq = reinterpret_cast<const uint4 *> (j);
  const int nq = (n + 3) / 4;
  uint4 q[8];
#pragma unroll
  for (int k = 0; k < 8; k++)
    q[k] = k < nq ? jq[k] : make_uint4 (0, 0, 0, 0);
  for (int base = 0; base < nq; base += 8)
#pragma unroll
    for (int k = 0; k < 8; k++)
      {
        const uint4 cur = q[k];
        const int g = base + k;
        q[k] = g + 8 < nq ? jq[g + 8] : make_uint4 (0, 0, 0, 0);
        const uint32_t js[4] = { cur.x, cur.y, cur.z, cur.w };
#pragma unroll
        for (int m = 0; m < 4; m++)
          {
            const int i = 4 * g + m;
            if (i < n)
              {
                const IDX a = v[i], b = v[js[m]];
                v[i] = b;
                v[js[m]] = a;
              }
          }
      }
}

__device__ __forceinline__ void
kg_set (uint16_t *R, int frame, int bin, uint16_t code, int *err)
{
  if (atomicCAS (reinterpret_cast<unsigned short *> (R + size_t (frame) * (AWM_MAX_BAND + 1) + bin), (unsigned short) 0, (unsigned short) code))
    *err = 1;
}

// one CTA per key.  keys16 [n_keys][16]; roles [n_keys][fpb][101]; jscr [n_keys][j_stride]; ud [n_keys][2][n_mix] (mix only);
// gidx [n_keys][n_mix] (mix with !SMEM_IDX only); err [n_keys] (zeroed by the caller)
template<bool SMEM_IDX> __global__ void __launch_bounds__ (kKeygenThreads, 2)
k_embed_roles_keys (const uint8_t *__restrict__ keys16, KeygenLayout L, uint16_t *__restrict__ roles, uint32_t *__restrict__ jscr,
                    uint8_t *__restrict__ ud, uint32_t *__restrict__ gidx, int *__restrict__ err)
{
  extern __shared__ __align__ (16) unsigned char smem[];
  uint32_t *T0 = reinterpret_cast<uint32_t *> (smem);
  uint32_t *rk = T0 + 256;
  uint32_t *ctr = rk + 44;                      // [0]: frame_position, [1]: mix
  uint8_t *sb = reinterpret_cast<uint8_t *> (ctr + 8);
  uint16_t *pos = reinterpret_cast<uint16_t *> (sb + 256);
  uint16_t *sidx = reinterpret_cast<uint16_t *> (reinterpret_cast<unsigned char *> (pos) + keygen_pos_bytes (L.fpb));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long key = blockIdx.x;
  const size_t n_roles = size_t (L.fpb) * (AWM_MAX_BAND + 1);
  uint16_t *R = roles + key * n_roles;
  uint32_t *jpos = jscr + key * L.j_stride, *jmix = jpos + L.j_mix0;
  uint8_t *ud_up = ud + key * 2 * L.n_mix, *ud_down = ud_up + L.n_mix;
  int *kerr = err + key;

  for (size_t i = tid; i < n_roles; i += kKeygenThreads)
    R[i] = 0;
  if (tid < 256)
    sb[tid] = kg_sbox (tid);
  for (int i = tid; i < L.fpb; i += kKeygenThreads)
    pos[i] = uint16_t (i);
  if (L.mix)
    for (int i = tid; i < L.n_mix; i += kKeygenThreads)
      {
        if (SMEM_IDX)
          sidx[i] = uint16_t (i);
        else
          gidx[key * L.n_mix + i] = uint32_t (i);
      }
  __syncthreads();
  if (tid < 256)
    {
      const uint32_t s = sb[tid], s2 = kg_xtime (s), s3 = s2 ^ s;
      T0[tid] = s2 | (s << 8) | (s << 16) | (s3 << 24);          // bytes (2s, s, s, 3s): SubBytes + MixColumns of one column
    }
  if (tid == 0)
    {
      /* key expansion (FIPS-197 5.2) on little-endian words: word i = bytes 4i .. 4i + 3 */
      const uint8_t *k = keys16 + key * 16;
      for (int i = 0; i < 4; i++)
        rk[i] = uint32_t (k[4 * i]) | (uint32_t (k[4 * i + 1]) << 8) | (uint32_t (k[4 * i + 2]) << 16) | (uint32_t (k[4 * i + 3]) << 24);
      uint32_t rcon = 1;
      for (int i = 4; i < 44; i++)
        {
          uint32_t t = rk[i - 1];
          if (i % 4 == 0)
            {
              t = (uint32_t (sb[(t >> 8) & 0xff]) ^ rcon) | (uint32_t (sb[(t >> 16) & 0xff]) << 8) | (uint32_t (sb[t >> 24]) << 16) |
                  (uint32_t (sb[t & 0xff]) << 24);
              rcon = kg_xtime (rcon);
            }
          rk[i] = rk[i - 4] ^ t;
        }
    }
  __syncthreads();
  if (tid < 2)
    kg_seed (T0, sb, rk, 0, tid == 0 ? kKeygenStreamFramePosition : kKeygenStreamMix, ctr + 4 * tid);
  __syncthreads();

  /* the j of every swap of BitPosGen and of the mix shuffle: one AES block gives two */
  const long long blocks_pos = (L.fpb + 1) / 2, blocks_mix = L.mix ? (L.n_mix + 1) / 2 : 0;
  for (long long b = tid; b < blocks_pos + blocks_mix; b += kKeygenThreads)
    {
      const bool m = b >= blocks_pos;
      const long long bb = m ? b - blocks_pos : b;
      const unsigned long long n = m ? L.n_mix : L.fpb;
      uint32_t *out = m ? jmix : jpos;
      unsigned long long r0, r1;
      kg_draws (T0, sb, rk, ctr + (m ? 4 : 0), bb, r0, r1);
      const unsigned long long i = 2 * bb;
      out[i] = uint32_t (i + r0 % (n - i));
      if (i + 1 < n)
        out[i + 1] = uint32_t (i + 1 + r1 % (n - i - 1));
    }
  __syncthreads();

  if (warp == 1)
    {
      if (lane == 0 && L.mix)
        {
          if (SMEM_IDX)
            kg_serial_shuffle (sidx, jmix, L.n_mix);
          else
            kg_serial_shuffle (gidx + key * L.n_mix, jmix, L.n_mix);
        }
      __syncwarp();
    }
  else
    {
      if (tid == 0)
        kg_serial_shuffle (pos, jpos, L.fpb);
      __syncwarp();
      asm volatile ("bar.sync 1, %0;" :: "r" (kKeygenThreads - 32));        // every warp but warp 1: pos is final
      const int n_ud_warps = kKeygenThreads / 32 - 1, w = warp ? warp - 1 : 0;
      for (int g = w; g < L.fpb; g += n_ud_warps)
        {
          const bool sync = g < L.sync_frames;
          uint32_t c[4];
          kg_seed (T0, sb, rk, sync ? g : g - L.sync_frames, sync ? kKeygenStreamSyncUpDown : kKeygenStreamDataUpDown, c);
          unsigned ja = 0, jb = 0;
          if (lane < kKeygenUpDown / 2)
            {
              unsigned long long r0, r1;
              kg_draws (T0, sb, rk, c, lane, r0, r1);
              ja = 2 * lane + unsigned (r0 % (unsigned long long) (kKeygenBands - 2 * lane));
              jb = 2 * lane + 1 + unsigned (r1 % (unsigned long long) (kKeygenBands - 2 * lane - 1));
            }
          int v0 = lane, v1 = lane + 32, v2 = lane + 64;       // band - 20 at positions lane, lane + 32, lane + 64
#pragma unroll 4
          for (int i = 0; i < kKeygenUpDown; i++)
            {
              const int j = __shfl_sync (0xffffffffu, (i & 1) ? jb : ja, i >> 1);
              const int si = i >> 5, sj = j >> 5;
              const int vi = __shfl_sync (0xffffffffu, si == 0 ? v0 : si == 1 ? v1 : v2, i & 31);
              const int vj = __shfl_sync (0xffffffffu, sj == 0 ? v0 : sj == 1 ? v1 : v2, j & 31);
              if (lane == (i & 31))
                {
                  if (si == 0) v0 = vj; else if (si == 1) v1 = vj; else v2 = vj;
                }
              if (lane == (j & 31))
                {
                  if (sj == 0) v0 = vi; else if (sj == 1) v1 = vi; else v2 = vi;
                }
            }
          const int vals[2] = { v0, v1 };
#pragma unroll
          for (int s = 0; s < 2; s++)                      // positions >= 64 are neither up nor down bands
            {
              const int p = lane + 32 * s;
              if (p >= kKeygenUpDown)
                continue;
              const bool down = p >= AWM_BANDS_PER_FRAME;
              const int band = vals[s] + AWM_MIN_BAND, slot = down ? p - AWM_BANDS_PER_FRAME : p;
              if (sync)
                kg_set (R, pos[g], band, uint16_t (AWM_ROLE_MARK | AWM_ROLE_SYNC | (down ? AWM_ROLE_DOWN : 0) |
                                                   ((g / L.sync_frames_per_bit) << AWM_ROLE_SHIFT)), kerr);
              else
                {
                  const int d = g - L.sync_frames, k = d * AWM_BANDS_PER_FRAME + slot;
                  if (L.mix)
                    (down ? ud_down : ud_up)[k] = uint8_t (band);
                  else        /* --linear: entry k keeps its place */
                    kg_set (R, pos[g], band, uint16_t (AWM_ROLE_MARK | (down ? AWM_ROLE_DOWN : 0) |
                                                       ((k / AWM_BANDS_PER_FRAME / L.frames_per_bit) << AWM_ROLE_SHIFT)), kerr);
                }
            }
        }
    }
  __syncthreads();
  if (!L.mix)
    return;
  /* with mixing the coded bit of an entry follows from its position after the shuffle, its frame and bands from where it came from */
  const uint32_t *gi = gidx + key * L.n_mix;
  for (int e = tid; e < L.n_mix; e += kKeygenThreads)
    {
      const int k = SMEM_IDX ? int (sidx[e]) : int (gi[e]);
      const int frame = pos[L.sync_frames + k / AWM_BANDS_PER_FRAME];
      const int bit = e / AWM_BANDS_PER_FRAME / L.frames_per_bit;
      kg_set (R, frame, ud_up[k], uint16_t (AWM_ROLE_MARK | (bit << AWM_ROLE_SHIFT)), kerr);
      kg_set (R, frame, ud_down[k], uint16_t (AWM_ROLE_MARK | AWM_ROLE_DOWN | (bit << AWM_ROLE_SHIFT)), kerr);
    }
}

} // namespace awm
