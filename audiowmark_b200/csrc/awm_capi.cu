// awm_capi.cu -- implementation of the C ABI declared in include/awm_b200.h.
//
// One context = one device + one stream + growable device buffers.  Host pointers are staged
// through context-owned device memory; device pointers are used in place.  There is no CPU
// fallback: every entry point launches the sm_90a kernels of awm_kernels.cuh or fails.
#include "awm_kernels.cuh"
#include "awm_speed.cuh"
#include "awm_refine_slide.cuh"
#include "awm_approx_mags.cuh"
#include <vector>
#include <time.h>
#include <string.h>
#include "awm_approx_tc.cuh"
#include "awm_embed_strip.cuh"
#include "awm_embed_batch.cuh"
#include "awm_batch_rates.cuh"
#include "awm_keygen.cuh"

#include <cuda_runtime.h>
#include <dlfcn.h>
#include <algorithm>
#include <cmath>
#include <map>
#include <set>
#include <thread>
#include <limits.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>

using namespace awm;

namespace {

struct DevBuf
{
  void  *p = nullptr;
  size_t cap = 0;
  cudaError_t
  reserve (size_t bytes)
  {
    if (bytes <= cap)
      return cudaSuccess;
    if (p)
      cudaFree (p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc (&p, want);
    if (e == cudaSuccess)
      cap = want;
    return e;
  }
  void
  release()
  {
    if (p)
      cudaFree (p);
    p = nullptr;
    cap = 0;
  }
  template<class T> T *as() { return static_cast<T *> (p); }
};

/* page-locked staging memory for the small lists that go back and forth between the stages of a `get` (candidate lists, per-offset
 * sums, soft bits, code words): copies from / to pageable memory are staged by the driver and block the host; with pinned memory
 * the copies of a stage are queued back to back and cost one synchronisation.  Bump allocator, reset at the start of an API call. */
struct PinArena
{
  struct Chunk { unsigned char *p; size_t cap; };
  std::vector<Chunk> chunks;
  size_t cur = 0, off = 0;
  void reset() { cur = 0; off = 0; }
  void *alloc (size_t n)
  {
    n = (n + 63) & ~size_t (63);
    for (;;)
      {
        if (cur < chunks.size() && off + n <= chunks[cur].cap)
          {
            void *r = chunks[cur].p + off;
            off += n;
            return r;
          }
        if (cur + 1 < chunks.size())
          {
            cur++;
            off = 0;
            continue;
          }
        Chunk c { nullptr, std::max<size_t> (n, size_t (4) << 20) };
        if (cudaMallocHost (reinterpret_cast<void **> (&c.p), c.cap) != cudaSuccess)
          return nullptr;
        chunks.push_back (c);
        cur = chunks.size() - 1;
        off = 0;
      }
  }
  template<class T> T *get (size_t count) { return static_cast<T *> (alloc (std::max<size_t> (count, 1) * sizeof (T))); }
  void release()
  {
    for (auto& c : chunks)
      cudaFreeHost (c.p);
    chunks.clear();
    reset();
  }
};

inline double
wall_now()
{
  timespec ts;
  clock_gettime (CLOCK_MONOTONIC, &ts);
  return double (ts.tv_sec) + 1e-9 * double (ts.tv_nsec);
}

struct SyncTab
{
  DevBuf ent, off, sorted, groups;
  DevBuf masks;                       // 0/1 band masks of the entries as wgmma B operand chunks of 48 entries (awm_approx_tc.cuh)
  int n_chunks = 0;
  int n_groups = 0;
  int n_ent = 0, n_bits = 0, total_frames = 0;
  int max_frame = 0;                  // largest entry frame: a search needs it inside the block (frames_per_block, twice that in CLIP mode)
  std::vector<awm_sync_entry> h_ent;
  std::vector<int> h_off;
};

struct KeyTab
{
  SyncTab sync[2];
  DevBuf mix, order;
  int n_mix = 0, n_coded = 0, frames_per_bit = 0, fpb = 0;
};

} // namespace

struct awm_ctx
{
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t s_in = nullptr, s_out = nullptr;      // copy streams of the pipelined host paths
  std::string err;
  uint64_t launches = 0;
  int n_sms = 0;
  bool profiling = false;
  struct ProfRec { const char *name; cudaEvent_t e0, e1; double bytes; };
  std::vector<ProfRec> prof;

  DevBuf tw, win, synth;             // constant tables
  DevBuf frame_mod; int embed_fpb = 0;
  DevBuf roles; int roles_fpb = 0, roles_n_coded = 0;         // batched embed: role table of one key
  DevBuf batch_items, batch_coded;
  /* batched embed with a key per item: role tables of n_keys keys built on the device (awm_set_embed_roles_keys) and the builder's
   * scratch (j values, bands of the data entries, index array of a mix too large for shared memory, per-key error flags) */
  DevBuf key_roles, keygen_keys, keygen_j, keygen_ud, keygen_idx, keygen_err;
  size_t key_roles_n = 0; int key_roles_fpb = 0, key_roles_n_coded = 0;
  DevBuf rate_items, rate_scratch;                           // batched embed at other sample rates: work list, per-wave scratch
  KeyTab keys[AWM_MAX_KEYS];

  // bound PCM
  const float *pcm = nullptr; size_t pcm_frames = 0; int pcm_ch = 0;
  DevBuf pcm_own, pcm16_own;
  /* awm_pcm_stage: a host stream on its way into `staged` piece by piece */
  DevBuf staged, staged16;
  std::vector<cudaEvent_t> stage_done;           // one per piece, recorded on s_in
  size_t stage_piece = 0, stage_frames = 0, stage_converted = 0;
  int stage_ch = 0;
  bool stage_s16 = false;

  /* approx: the per-call state of awm_sync_approx lives in a slot, so that the search of the next chunk can run
   * (awm_sync_approx_enqueue, on s_approx) while peaks / refine / decode of the current one read theirs */
  struct ApproxSlot
  {
    DevBuf have, q, scores, a_ud, a_cnt;
    size_t n_scores = 0;
    long long n_have = 0; int ld_have = 0;                                // have[4][ld_have]: frames per shift written by the search
    const float *pcm = nullptr; size_t pcm_frames = 0; int pcm_ch = 0;    // the PCM view the search ran on
    cudaEvent_t done = nullptr;                                           // recorded after k_local_mean
  };
  ApproxSlot aslot[2];
  int cur_aslot = 0;
  cudaStream_t s_approx = nullptr;
  DevBuf dbT, peaks_out, peaks_cnt, a_mags;   // a_mags is shared: every slot's gather runs before the next search overwrites it
  DevBuf cand_start, cand_noff, r_ud, r_cnt, rvalid, r_ent_ud, r_ent_flag, tw1024;   // refine
  DevBuf cand_score, rank_keep, rank_first, ex_start, ex_cand, ex_off, ex_n;         // offsets picked for exact re-scoring (k_refine_rank)
  DevBuf blk_start, D, raw;          // decode
  DevBuf vit_raw, vit_off, vit_types, vit_delta, vit_dec, vit_bits, vit_err;
  DevBuf emb_in, emb_out, emb_in16, emb_out16, peaks, snr;

  PinArena pin;

  // multi-GPU exchange (awm_dist_*): NCCL communicator of the sharded run + staging buffers
  void *nccl_comm = nullptr;
  int dist_rank = 0, dist_world = 1;
  DevBuf dist_send, dist_recv;
  unsigned char *dist_hsend = nullptr, *dist_hhdr = nullptr;
  size_t dist_hsend_cap = 0;

  // resampler / speed scan
  struct CoefTab { DevBuf buf; int h = 0; };
  std::map<std::pair<double, int>, CoefTab> coef_cache;          // (ratio, hlen) -> filter table
  DevBuf rs_in, rs_out, rs_jobs, pcm_rs;
  const float *saved_pcm = nullptr; size_t saved_frames = 0; int saved_ch = 0; bool pushed = false;
  DevBuf win512, sp_clip, sp_sub, sp_mags, sp_mag_jobs, sp_cmp_jobs, sp_best;
  std::vector<MagJob> sp_last;                                   // the MagMatrix of every centre of the last scan (awm_speed_mags)
  int sp_last_ent = 0;
};

namespace {

int
fail (awm_ctx *ctx, const char *fmt, ...)
{
  char buf[512];
  va_list ap;
  va_start (ap, fmt);
  vsnprintf (buf, sizeof (buf), fmt, ap);
  va_end (ap);
  if (ctx)
    ctx->err = buf;
  return 1;
}

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail (ctx, "%s: %s", #call, cudaGetErrorString (e_)); } while (0)
#define LAUNCH_CHECK(name) do { ctx->launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) return fail (ctx, "launch %s: %s", name, cudaGetErrorString (e_)); prof_end (ctx, name); } while (0)
/* PROF (ctx) goes right before a kernel launch, LAUNCH_CHECK right after it */
#define PROF(ctx) prof_begin (ctx)

void
prof_begin (awm_ctx *ctx)
{
  if (!ctx->profiling)
    return;
  awm_ctx::ProfRec r;
  r.name = nullptr;
  r.bytes = 0;
  cudaEventCreate (&r.e0);
  cudaEventCreate (&r.e1);
  cudaEventRecord (r.e0, ctx->stream);
  ctx->prof.push_back (r);
}

void
prof_end (awm_ctx *ctx, const char *name)
{
  if (!ctx->profiling || ctx->prof.empty() || ctx->prof.back().name)
    return;
  ctx->prof.back().name = name;
  cudaEventRecord (ctx->prof.back().e1, ctx->stream);
}

/* measurement aid: algorithmic bytes of the launch that was just recorded (the compulsory traffic of the work it was given;
 * only kernels whose volume depends on run-time counts report it here, the others are sized by the caller from the input) */
void
prof_bytes (awm_ctx *ctx, double bytes)
{
  if (ctx->profiling && !ctx->prof.empty())
    ctx->prof.back().bytes = bytes;
}

bool
is_device_ptr (const void *p)
{
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes (&a, p) != cudaSuccess)
    {
      cudaGetLastError();
      return false;
    }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

double
window_cos (double x)    // von Hann, reference src/wmcommon.hh:187-193
{
  if (fabs (x) > 1)
    return 0;
  return 0.5 * cos (x * M_PI) + 0.5;
}

int
init_tables (awm_ctx *ctx)
{
  // twiddles exp(-2 pi i k1 t / 1024) at [k1*32 + t]
  std::vector<float2> tw (1024);
  for (int k1 = 0; k1 < 32; k1++)
    for (int t = 0; t < 32; t++)
      {
        const double a = -2.0 * M_PI * double (k1 * t) / 1024.0;
        tw[k1 * 32 + t] = make_float2 (float (cos (a)), float (sin (a)));
      }
  // FFTAnalyzer::gen_normalized_window (src/wmcommon.cc:68-89)
  std::vector<float> win (kFrame);
  double weight = 0;
  for (int i = 0; i < kFrame; i++)
    {
      const double w = window_cos ((i - kFrame / 2.0) / (kFrame / 2.0));
      win[i] = w;
      weight += w;
    }
  for (int i = 0; i < kFrame; i++)
    win[i] *= 2.0 / weight;
  // WatermarkSynth::generate_window (src/wmadd.cc:177-206)
  std::vector<float> synth (3 * kFrame);
  for (int i = 0; i < 3 * kFrame; i++)
    {
      const double overlap = 0.1;
      double norm_pos = (double (i) - kFrame) / kFrame;
      if (norm_pos > 0.5)
        norm_pos = 1 - norm_pos;
      double tri;
      if (norm_pos < -overlap)
        tri = 0;
      else if (norm_pos < overlap)
        tri = 0.5 + norm_pos / (2 * overlap);
      else
        tri = 1;
      synth[i] = (cos (tri * M_PI + M_PI) + 1) * 0.5;
    }
  CK (ctx->tw.reserve (tw.size() * sizeof (float2)));
  CK (ctx->win.reserve (win.size() * sizeof (float)));
  CK (ctx->synth.reserve (synth.size() * sizeof (float)));
  CK (cudaMemcpy (ctx->tw.p, tw.data(), tw.size() * sizeof (float2), cudaMemcpyHostToDevice));
  CK (cudaMemcpy (ctx->win.p, win.data(), win.size() * sizeof (float), cudaMemcpyHostToDevice));
  CK (cudaMemcpy (ctx->synth.p, synth.data(), synth.size() * sizeof (float), cudaMemcpyHostToDevice));
  return 0;
}

template<class K> int
set_smem (awm_ctx *ctx, K kernel, size_t bytes)
{
  /* the attribute sticks to the function: one driver call per kernel (and size), not one per launch */
  static std::map<std::pair<const void *, int>, size_t> done;
  size_t& have = done[{ reinterpret_cast<const void *> (kernel), ctx->device }];
  if (have >= bytes && have)
    return 0;
  CK (cudaFuncSetAttribute (kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int (bytes)));
  have = bytes;
  return 0;
}

} // namespace

void nccl_destroy (void *comm);       // defined with the awm_dist_* functions below

extern "C" {

int
awm_create (int device, awm_ctx **out)
{
  if (!out)
    return 1;
  *out = nullptr;
  int n_dev = 0;
  if (cudaGetDeviceCount (&n_dev) != cudaSuccess || n_dev <= 0)
    return 2;          // no CUDA device: the product has no CPU fallback
  if (device < 0 || device >= n_dev)
    return 3;
  awm_ctx *ctx = new awm_ctx();
  ctx->device = device;
  if (cudaSetDevice (device) != cudaSuccess || cudaStreamCreateWithFlags (&ctx->stream, cudaStreamNonBlocking) != cudaSuccess)
    {
      delete ctx;
      return 4;
    }
  if (init_tables (ctx))
    {
      fprintf (stderr, "awm_create: %s\n", ctx->err.c_str());
      delete ctx;
      return 5;
    }
  *out = ctx;
  return 0;
}

void
awm_destroy (awm_ctx *ctx)
{
  if (!ctx)
    return;
  cudaSetDevice (ctx->device);
  cudaStreamSynchronize (ctx->stream);
  if (ctx->s_approx)
    cudaStreamSynchronize (ctx->s_approx);
  DevBuf *bufs[] = { &ctx->tw, &ctx->win, &ctx->synth, &ctx->frame_mod, &ctx->roles, &ctx->batch_items, &ctx->batch_coded, &ctx->key_roles, &ctx->keygen_keys, &ctx->keygen_j, &ctx->keygen_ud, &ctx->keygen_idx, &ctx->keygen_err, &ctx->rate_items, &ctx->rate_scratch, &ctx->pcm_own, &ctx->pcm16_own, &ctx->staged, &ctx->staged16, &ctx->dbT, &ctx->peaks_out, &ctx->peaks_cnt, &ctx->a_mags,
                     &ctx->cand_start, &ctx->cand_noff, &ctx->r_ud, &ctx->r_cnt, &ctx->rvalid, &ctx->r_ent_ud, &ctx->r_ent_flag, &ctx->tw1024,
                     &ctx->cand_score, &ctx->rank_keep, &ctx->rank_first, &ctx->ex_start, &ctx->ex_cand, &ctx->ex_off, &ctx->ex_n, &ctx->vit_off, &ctx->blk_start, &ctx->D, &ctx->raw,
                     &ctx->vit_raw, &ctx->vit_types, &ctx->vit_delta, &ctx->vit_dec, &ctx->vit_bits, &ctx->vit_err,
                     &ctx->emb_in, &ctx->emb_out, &ctx->emb_in16, &ctx->emb_out16, &ctx->peaks, &ctx->snr, &ctx->rs_in, &ctx->rs_out, &ctx->rs_jobs, &ctx->pcm_rs,
                     &ctx->win512, &ctx->sp_clip, &ctx->sp_sub, &ctx->sp_mags, &ctx->sp_mag_jobs, &ctx->sp_cmp_jobs, &ctx->sp_best };
  for (DevBuf *b : bufs)
    b->release();
  ctx->pin.release();
  ctx->dist_send.release();
  ctx->dist_recv.release();
  if (ctx->dist_hsend) cudaFreeHost (ctx->dist_hsend);
  if (ctx->dist_hhdr) cudaFreeHost (ctx->dist_hhdr);
  if (ctx->nccl_comm)
    nccl_destroy (ctx->nccl_comm);
  for (auto& ct : ctx->coef_cache)
    ct.second.buf.release();
  for (KeyTab& k : ctx->keys)
    {
      for (SyncTab& s : k.sync)
        {
          s.ent.release();
          s.masks.release();
          s.off.release();
          s.sorted.release();
          s.groups.release();
        }
      k.mix.release();
      k.order.release();
    }
  for (auto& s : ctx->aslot)
    {
      DevBuf *sb[] = { &s.have, &s.q, &s.scores, &s.a_ud, &s.a_cnt };
      for (DevBuf *b : sb)
        b->release();
      if (s.done)
        cudaEventDestroy (s.done);
    }
  for (cudaEvent_t e : ctx->stage_done)
    cudaEventDestroy (e);
  if (ctx->s_approx)
    cudaStreamDestroy (ctx->s_approx);
  if (ctx->s_in)
    cudaStreamDestroy (ctx->s_in);
  if (ctx->s_out)
    cudaStreamDestroy (ctx->s_out);
  cudaStreamDestroy (ctx->stream);
  delete ctx;
}

const char *
awm_last_error (const awm_ctx *ctx)
{
  return ctx ? ctx->err.c_str() : "no context (is a CUDA device present? there is no CPU fallback)";
}

uint64_t
awm_launch_count (const awm_ctx *ctx)
{
  return ctx ? ctx->launches : 0;
}

void *
awm_stream (awm_ctx *ctx)
{
  return ctx ? (void *) ctx->stream : nullptr;
}

int
awm_synchronize (awm_ctx *ctx)
{
  CK (cudaSetDevice (ctx->device));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

void *
awm_host_alloc (size_t bytes)
{
  void *p = nullptr;
  if (cudaHostAlloc (&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess)
    {
      cudaGetLastError();
      return nullptr;
    }
  return p;
}

void
awm_host_free (void *p)
{
  if (p)
    cudaFreeHost (p);
}

int
awm_profile_enable (awm_ctx *ctx, int on)
{
  ctx->profiling = on != 0;
  return 0;
}

int
awm_profile_report (awm_ctx *ctx, char *json_out, size_t json_cap)
{
  CK (cudaSetDevice (ctx->device));
  CK (cudaStreamSynchronize (ctx->stream));
  struct Acc { std::string name; int n; double ms; double bytes; };
  std::vector<Acc> acc;
  for (auto& r : ctx->prof)
    {
      float ms = 0;
      if (r.name && cudaEventElapsedTime (&ms, r.e0, r.e1) == cudaSuccess)
        {
          bool found = false;
          for (auto& a : acc)
            if (a.name == r.name)
              {
                a.n++;
                a.ms += ms;
                a.bytes += r.bytes;
                found = true;
              }
          if (!found)
            acc.push_back ({ r.name, 1, ms, r.bytes });
        }
      cudaEventDestroy (r.e0);
      cudaEventDestroy (r.e1);
    }
  ctx->prof.clear();
  std::string js = "{";
  for (size_t i = 0; i < acc.size(); i++)
    {
      char buf[256];
      snprintf (buf, sizeof (buf), "%s\"%s\": {\"launches\": %d, \"ms\": %.6f, \"algo_bytes\": %.0f}", i ? ", " : "", acc[i].name.c_str(), acc[i].n, acc[i].ms, acc[i].bytes);
      js += buf;
    }
  js += "}";
  if (json_out && json_cap)
    {
      if (js.size() + 1 > json_cap)
        return fail (ctx, "awm_profile_report: buffer too small");
      memcpy (json_out, js.c_str(), js.size() + 1);
    }
  return 0;
}

/* ---------------------------------------------------------------- FFTProcessor */

static int
fft_batch (awm_ctx *ctx, const float *in, float *out, size_t count, int n, bool inverse)
{
  if (n != kFrame)
    return fail (ctx, "awm_fft: only n = 1024 is supported (got %d)", n);
  if (count == 0)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const size_t in_elems = count * (inverse ? kFrame + 2 : kFrame), out_elems = count * (inverse ? kFrame : kFrame + 2);
  const float *d_in = in;
  float *d_out = out;
  const bool in_dev = is_device_ptr (in), out_dev = is_device_ptr (out);
  if (!in_dev)
    {
      CK (ctx->emb_in.reserve (in_elems * sizeof (float)));
      CK (cudaMemcpyAsync (ctx->emb_in.p, in, in_elems * sizeof (float), cudaMemcpyHostToDevice, ctx->stream));
      d_in = ctx->emb_in.as<float>();
    }
  if (!out_dev)
    {
      CK (ctx->emb_out.reserve (out_elems * sizeof (float)));
      d_out = ctx->emb_out.as<float>();
    }
  const size_t smem = fft_smem_bytes (kFftWarps);
  const unsigned grid = unsigned (((count + 1) / 2 + kFftWarps - 1) / kFftWarps);
  if (inverse)
    {
      if (set_smem (ctx, k_fft_c2r, smem)) return 1;
      PROF (ctx);
      k_fft_c2r<<<grid, kFftWarps * 32, smem, ctx->stream>>> (d_in, d_out, (long long) count, ctx->tw.as<float2>());
    }
  else
    {
      if (set_smem (ctx, k_fft_r2c, smem)) return 1;
      PROF (ctx);
      k_fft_r2c<<<grid, kFftWarps * 32, smem, ctx->stream>>> (d_in, d_out, (long long) count, ctx->tw.as<float2>());
    }
  LAUNCH_CHECK ("k_fft");
  if (!out_dev)
    CK (cudaMemcpyAsync (out, d_out, out_elems * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

int awm_fft_r2c (awm_ctx *ctx, const float *in, float *out, size_t count, int n) { return fft_batch (ctx, in, out, count, n, false); }
int awm_fft_c2r (awm_ctx *ctx, const float *in, float *out, size_t count, int n) { return fft_batch (ctx, in, out, count, n, true); }

/* ---------------------------------------------------------------- tables */

int
awm_set_embed_tables (awm_ctx *ctx, const uint8_t *frame_mod_ab, int frames_per_block)
{
  if (!frame_mod_ab || frames_per_block <= 0)
    return fail (ctx, "awm_set_embed_tables: bad arguments");
  const size_t bytes = size_t (2) * frames_per_block * (kMaxBand + 1);
  for (size_t i = 0; i < bytes; i++)               /* the kernels read bins kMinBand .. kMaxBand, and 1 as up, anything else as down */
    if (frame_mod_ab[i] > 2 || (frame_mod_ab[i] && int (i % (kMaxBand + 1)) < kMinBand))
      return fail (ctx, "awm_set_embed_tables: entry %zu (row %zu, bin %d) is %d: entries are 0 keep, 1 up, 2 down, and bins below %d are kept",
                   i, i / (kMaxBand + 1), int (i % (kMaxBand + 1)), int (frame_mod_ab[i]), kMinBand);
  CK (cudaSetDevice (ctx->device));
  CK (ctx->frame_mod.reserve (bytes));
  CK (cudaMemcpyAsync (ctx->frame_mod.p, frame_mod_ab, bytes, cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  ctx->embed_fpb = frames_per_block;
  return 0;
}

int
awm_set_embed_roles (awm_ctx *ctx, const uint16_t *roles, int frames_per_block, int n_coded_bits)
{
  if (!roles || frames_per_block <= 0 || n_coded_bits <= 0 || n_coded_bits > AWM_ROLE_MAX_INDEX + 1)
    return fail (ctx, "awm_set_embed_roles: bad arguments");
  const size_t n = size_t (frames_per_block) * (kMaxBand + 1);
  for (size_t i = 0; i < n; i++)                         /* k_embed_batch reads coded bits at these indices */
    if ((roles[i] & AWM_ROLE_MARK) && !(roles[i] & AWM_ROLE_SYNC) && (roles[i] >> AWM_ROLE_SHIFT) >= n_coded_bits)
      return fail (ctx, "awm_set_embed_roles: role %zu names coded bit %d of %d", i, roles[i] >> AWM_ROLE_SHIFT, n_coded_bits);
  CK (cudaSetDevice (ctx->device));
  CK (ctx->roles.reserve (n * sizeof (uint16_t)));
  CK (cudaMemcpyAsync (ctx->roles.p, roles, n * sizeof (uint16_t), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  ctx->roles_fpb = frames_per_block;
  ctx->roles_n_coded = n_coded_bits;
  return 0;
}

int
awm_set_embed_roles_keys (awm_ctx *ctx, const uint8_t *keys16, size_t n_keys, const awm_role_layout *layout)
{
  ctx->key_roles_n = 0;
  if (!keys16 || !n_keys || n_keys > INT_MAX || !layout)
    return fail (ctx, "awm_set_embed_roles_keys: bad arguments");
  const awm_role_layout& l = *layout;
  if (l.sync_frames <= 0 || l.sync_frames_per_bit <= 0 || l.sync_frames % l.sync_frames_per_bit || l.frames_per_bit <= 0 || l.n_coded_bits <= 0 ||
      l.n_coded_bits > AWM_ROLE_MAX_INDEX + 1 || l.sync_frames / l.sync_frames_per_bit > AWM_ROLE_MAX_INDEX + 1 ||
      (long long) l.n_coded_bits * l.frames_per_bit != l.data_frames || (long long) l.sync_frames + l.data_frames > 65536)
    return fail (ctx, "awm_set_embed_roles_keys: bad layout (sync frames %d, %d per bit, data frames %d, %d per bit, %d coded bits)",
                 l.sync_frames, l.sync_frames_per_bit, l.data_frames, l.frames_per_bit, l.n_coded_bits);
  KeygenLayout L;
  L.sync_frames = l.sync_frames;
  L.sync_frames_per_bit = l.sync_frames_per_bit;
  L.data_frames = l.data_frames;
  L.frames_per_bit = l.frames_per_bit;
  L.mix = l.mix != 0;
  L.fpb = l.sync_frames + l.data_frames;
  L.n_mix = l.data_frames * AWM_BANDS_PER_FRAME;
  L.j_mix0 = (L.fpb + 15) & ~15;
  L.j_stride = L.j_mix0 + (L.mix ? (L.n_mix + 15) & ~15 : 0);
  const bool smem_idx = !L.mix || L.n_mix <= kKeygenSmemIdxMax;      /* a larger mix keeps its index array in global memory */
  const size_t smem = keygen_smem (L.fpb, L.n_mix, L.mix && smem_idx);
  CK (cudaSetDevice (ctx->device));
  int smem_max = 0;
  CK (cudaDeviceGetAttribute (&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
  if (smem > size_t (smem_max))
    return fail (ctx, "awm_set_embed_roles_keys: %d frames per block need %zu bytes of shared memory (%d available)", L.fpb, smem, smem_max);
  const size_t n_roles = n_keys * size_t (L.fpb) * (kMaxBand + 1);
  CK (ctx->key_roles.reserve (n_roles * sizeof (uint16_t)));
  CK (ctx->keygen_keys.reserve (n_keys * 16));
  CK (ctx->keygen_j.reserve (n_keys * size_t (L.j_stride) * sizeof (uint32_t)));
  CK (ctx->keygen_ud.reserve (L.mix ? n_keys * 2 * size_t (L.n_mix) : 16));
  CK (ctx->keygen_idx.reserve (L.mix && !smem_idx ? n_keys * size_t (L.n_mix) * sizeof (uint32_t) : 16));
  CK (ctx->keygen_err.reserve (n_keys * sizeof (int)));
  CK (cudaMemcpyAsync (ctx->keygen_keys.p, keys16, n_keys * 16, cudaMemcpyDefault, ctx->stream));
  CK (cudaMemsetAsync (ctx->keygen_err.p, 0, n_keys * sizeof (int), ctx->stream));
  auto kernel = smem_idx ? k_embed_roles_keys<true> : k_embed_roles_keys<false>;
  if (set_smem (ctx, kernel, smem)) return 1;
  PROF (ctx);
  kernel<<<unsigned (n_keys), kKeygenThreads, smem, ctx->stream>>> (ctx->keygen_keys.as<uint8_t>(), L, ctx->key_roles.as<uint16_t>(), ctx->keygen_j.as<uint32_t>(),
                                                                    ctx->keygen_ud.as<uint8_t>(), ctx->keygen_idx.as<uint32_t>(), ctx->keygen_err.as<int>());
  LAUNCH_CHECK ("k_embed_roles_keys");
  std::vector<int> errs (n_keys);
  CK (cudaMemcpyAsync (errs.data(), ctx->keygen_err.p, n_keys * sizeof (int), cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  for (size_t k = 0; k < n_keys; k++)
    if (errs[k])
      return fail (ctx, "awm_set_embed_roles_keys: key %zu: a (frame, bin) entry is assigned twice", k);
  ctx->key_roles_n = n_keys;
  ctx->key_roles_fpb = L.fpb;
  ctx->key_roles_n_coded = l.n_coded_bits;
  return 0;
}

int
awm_get_embed_roles_keys (awm_ctx *ctx, size_t first_key, size_t n_keys, uint16_t *out)
{
  if (first_key > ctx->key_roles_n || n_keys > ctx->key_roles_n - first_key || (n_keys && !out))
    return fail (ctx, "awm_get_embed_roles_keys: keys %zu .. %zu of a role set of %zu keys", first_key, first_key + n_keys, ctx->key_roles_n);
  if (!n_keys)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const size_t per_key = size_t (ctx->key_roles_fpb) * (kMaxBand + 1);
  CK (cudaMemcpyAsync (out, ctx->key_roles.as<uint16_t>() + first_key * per_key, n_keys * per_key * sizeof (uint16_t), cudaMemcpyDefault, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

int
awm_set_sync_tables (awm_ctx *ctx, int key_slot, int mode, const awm_sync_entry *entries, int n_entries,
                     const int *bit_offsets, int n_bits)
{
  if (key_slot < 0 || key_slot >= AWM_MAX_KEYS || mode < 0 || mode > 1 || !entries || n_entries <= 0 || !bit_offsets || n_bits <= 0)
    return fail (ctx, "awm_set_sync_tables: bad arguments");
  /* every check comes before the slot is touched: a rejected table leaves the previous one in place, whole */
  if (n_bits > 6)
    return fail (ctx, "awm_set_sync_tables: at most 6 sync bits are supported");
  if (bit_offsets[0] != 0 || bit_offsets[n_bits] != n_entries)
    return fail (ctx, "awm_set_sync_tables: bit_offsets must run from 0 to n_entries");
  for (int b = 0; b < n_bits; b++)
    if (bit_offsets[b + 1] < bit_offsets[b])
      return fail (ctx, "awm_set_sync_tables: bit_offsets must not decrease (bit %d)", b);
  int max_frame = 0;
  for (int i = 0; i < n_entries; i++)
    {
      /* the tensor-core kernel sums an entry's bands through a 0/1 mask, so a band can count only once per list */
      uint32_t seen_up[3] = { 0, 0, 0 }, seen_down[3] = { 0, 0, 0 };
      for (int j = 0; j < kUD; j++)
        {
          const int u = entries[i].up[j], d = entries[i].down[j];
          if (u >= kBands || d >= kBands)
            return fail (ctx, "awm_set_sync_tables: band index out of range");
          if ((seen_up[u >> 5] >> (u & 31)) & 1 || (seen_down[d >> 5] >> (d & 31)) & 1)
            return fail (ctx, "awm_set_sync_tables: entry %d repeats a band in its up or down list", i);
          seen_up[u >> 5] |= 1u << (u & 31);
          seen_down[d >> 5] |= 1u << (d & 31);
        }
      max_frame = std::max (max_frame, int (entries[i].frame));
    }
  CK (cudaSetDevice (ctx->device));
  SyncTab& t = ctx->keys[key_slot].sync[mode];
  CK (t.ent.reserve (sizeof (awm_sync_entry) * n_entries));
  CK (t.off.reserve (sizeof (int) * (n_bits + 1)));
  CK (cudaMemcpyAsync (t.ent.p, entries, sizeof (awm_sync_entry) * n_entries, cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaMemcpyAsync (t.off.p, bit_offsets, sizeof (int) * (n_bits + 1), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  /* k_sync_approx walks all entries in ascending frame order (per-bit order is kept: frames are sorted inside a bit) */
  std::vector<ApproxEntry> sorted (n_entries);
  {
    std::vector<int> idx (n_entries), bit_of (n_entries);
    for (int b = 0; b < n_bits; b++)
      for (int e = bit_offsets[b]; e < bit_offsets[b + 1]; e++)
        bit_of[e] = b;
    for (int i = 0; i < n_entries; i++)
      idx[i] = i;
    std::stable_sort (idx.begin(), idx.end(), [&] (int a, int b) { return entries[a].frame < entries[b].frame; });
    for (int i = 0; i < n_entries; i++)
      {
        const awm_sync_entry& src = entries[idx[i]];
        sorted[i].frame = src.frame;
        sorted[i].bit = bit_of[idx[i]];
        sorted[i].pad = 0;
        memcpy (sorted[i].up, src.up, kUD);
        memcpy (sorted[i].down, src.down, kUD);
      }
  }
  std::vector<int> group_end;
  for (int i = 0; i < n_entries; )
    {
      int j = i;
      while (j < n_entries && j - i < 16 && sorted[j].frame - sorted[i].frame <= kApproxMaxSpan)
        j++;
      group_end.push_back (j);
      i = j;
    }
  CK (t.sorted.reserve (sorted.size() * sizeof (ApproxEntry)));
  CK (t.groups.reserve (group_end.size() * sizeof (int)));
  CK (cudaMemcpyAsync (t.sorted.p, sorted.data(), sorted.size() * sizeof (ApproxEntry), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaMemcpyAsync (t.groups.p, group_end.data(), group_end.size() * sizeof (int), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  {
    std::vector<unsigned char> masks;
    tc_build_masks (entries, n_entries, masks);
    CK (t.masks.reserve (masks.size()));
    CK (cudaMemcpyAsync (t.masks.p, masks.data(), masks.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK (cudaStreamSynchronize (ctx->stream));
    t.n_chunks = int (masks.size() / kTcBBytes);
  }
  t.n_groups = int (group_end.size());
  t.n_ent = n_entries;
  t.n_bits = n_bits;
  t.max_frame = max_frame;
  t.h_ent.assign (entries, entries + n_entries);
  t.h_off.assign (bit_offsets, bit_offsets + n_bits + 1);
  return 0;
}

int
awm_set_mix_tables (awm_ctx *ctx, int key_slot, const awm_mix_entry *entries, int n_entries,
                    const uint16_t *bit_order, int n_coded_bits, int frames_per_bit, int frames_per_block)
{
  if (key_slot < 0 || key_slot >= AWM_MAX_KEYS || !entries || !bit_order || n_coded_bits <= 0 || frames_per_bit <= 0
      || n_entries != n_coded_bits * frames_per_bit * kUD || frames_per_block <= 0)
    return fail (ctx, "awm_set_mix_tables: bad arguments");
  for (int i = 0; i < n_entries; i++)
    if (entries[i].frame >= frames_per_block || entries[i].up < kMinBand || entries[i].up > kMaxBand
        || entries[i].down < kMinBand || entries[i].down > kMaxBand)
      return fail (ctx, "awm_set_mix_tables: entry %d out of range", i);
  for (int i = 0; i < n_coded_bits; i++)
    if (bit_order[i] >= n_coded_bits)
      return fail (ctx, "awm_set_mix_tables: bit_order out of range");
  CK (cudaSetDevice (ctx->device));
  KeyTab& k = ctx->keys[key_slot];
  CK (k.mix.reserve (sizeof (awm_mix_entry) * n_entries));
  CK (k.order.reserve (sizeof (uint16_t) * n_coded_bits));
  CK (cudaMemcpyAsync (k.mix.p, entries, sizeof (awm_mix_entry) * n_entries, cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaMemcpyAsync (k.order.p, bit_order, sizeof (uint16_t) * n_coded_bits, cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  k.n_mix = n_entries;
  k.n_coded = n_coded_bits;
  k.frames_per_bit = frames_per_bit;
  k.fpb = frames_per_block;
  return 0;
}

/* ---------------------------------------------------------------- PCM */

namespace {

/* awm_pcm_bind / awm_pcm_bind_s16 */
int
pcm_bind_any (awm_ctx *ctx, const void *pcm_v, bool s16, size_t n_frames, int channels, size_t pad_start, size_t pad_end)
{
  if (channels <= 0 || (!pcm_v && n_frames))
    return fail (ctx, "awm_pcm_bind: bad arguments");
  CK (cudaSetDevice (ctx->device));
  ctx->pushed = false;                           // a new bind replaces whatever awm_pcm_push_resampled saved
  const float *pcm = s16 ? nullptr : static_cast<const float *> (pcm_v);
  const bool dev = pcm_v && is_device_ptr (pcm_v);
  if (dev && !s16 && pad_start == 0 && pad_end == 0)
    {
      ctx->pcm = pcm;
    }
  else
    {
      const size_t total = (pad_start + n_frames + pad_end) * channels;
      CK (ctx->pcm_own.reserve (std::max<size_t> (total, 1) * sizeof (float)));
      float *d = ctx->pcm_own.as<float>();
      if (pad_start)
        CK (cudaMemsetAsync (d, 0, pad_start * channels * sizeof (float), ctx->stream));
      if (n_frames && !s16)
        CK (cudaMemcpyAsync (d + pad_start * channels, pcm, n_frames * channels * sizeof (float),
                             dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, ctx->stream));
      if (n_frames && s16)
        {
          const int16_t *src16 = static_cast<const int16_t *> (pcm_v);
          const long long n_val = (long long) (n_frames * channels);
          if (!dev)
            {
              CK (ctx->pcm16_own.reserve (n_val * sizeof (int16_t)));
              CK (cudaMemcpyAsync (ctx->pcm16_own.p, src16, n_val * sizeof (int16_t), cudaMemcpyHostToDevice, ctx->stream));
              src16 = ctx->pcm16_own.as<int16_t>();
            }
          PROF (ctx);
          s16_to_f32_kernel (src16, d + pad_start * channels)<<<unsigned (((n_val + 1) / 2 + 255) / 256), 256, 0, ctx->stream>>> (src16, d + pad_start * channels, n_val);
          LAUNCH_CHECK ("k_s16_to_f32");
        }
      if (pad_end)
        CK (cudaMemsetAsync (d + (pad_start + n_frames) * channels, 0, pad_end * channels * sizeof (float), ctx->stream));
      ctx->pcm = d;
    }
  ctx->pcm_frames = pad_start + n_frames + pad_end;
  ctx->pcm_ch = channels;
  return 0;
}

} // namespace

int awm_pcm_bind (awm_ctx *ctx, const float *pcm, size_t n_frames, int channels, size_t pad_start, size_t pad_end) { return pcm_bind_any (ctx, pcm, false, n_frames, channels, pad_start, pad_end); }
int awm_pcm_bind_s16 (awm_ctx *ctx, const int16_t *pcm, size_t n_frames, int channels, size_t pad_start, size_t pad_end) { return pcm_bind_any (ctx, pcm, true, n_frames, channels, pad_start, pad_end); }

/* awm_pcm_stage / awm_pcm_stage_wait: see include/awm_b200.h */
int
awm_pcm_stage (awm_ctx *ctx, const void *pcm, int is_s16, size_t n_frames, int channels, size_t piece_frames, const float **device_out)
{
  if (!ctx || !pcm || !n_frames || channels <= 0 || !piece_frames || !device_out)
    return fail (ctx, "awm_pcm_stage: bad arguments");
  CK (cudaSetDevice (ctx->device));
  if (is_device_ptr (pcm))
    return fail (ctx, "awm_pcm_stage: the stream is already in device memory");
  if (!ctx->s_in)
    {
      CK (cudaStreamCreateWithFlags (&ctx->s_in, cudaStreamNonBlocking));
      CK (cudaStreamCreateWithFlags (&ctx->s_out, cudaStreamNonBlocking));
    }
  /* kernels in flight may still read the previous contents of the staging buffer: order the copies behind them */
  cudaEvent_t busy;
  CK (cudaEventCreateWithFlags (&busy, cudaEventDisableTiming));
  CK (cudaEventRecord (busy, ctx->stream));
  CK (cudaStreamWaitEvent (ctx->s_in, busy, 0));
  CK (cudaEventDestroy (busy));
  const size_t n_val = n_frames * channels;
  CK (ctx->staged.reserve (n_val * sizeof (float)));
  if (is_s16)
    CK (ctx->staged16.reserve (n_val * sizeof (int16_t)));
  piece_frames = (piece_frames + 1) & ~size_t (1);               // even: the conversion kernel stores float pairs
  const size_t n_pieces = (n_frames + piece_frames - 1) / piece_frames;
  while (ctx->stage_done.size() < n_pieces)
    {
      cudaEvent_t e;
      CK (cudaEventCreateWithFlags (&e, cudaEventDisableTiming));
      ctx->stage_done.push_back (e);
    }
  for (size_t p = 0; p < n_pieces; p++)
    {
      const size_t f0 = p * piece_frames, f1 = std::min (f0 + piece_frames, n_frames);
      const size_t v0 = f0 * channels, nv = (f1 - f0) * channels;
      if (is_s16)       /* copies only on the copy stream; a piece becomes float on the context stream when somebody waits for it */
        CK (cudaMemcpyAsync (ctx->staged16.as<int16_t>() + v0, static_cast<const int16_t *> (pcm) + v0, nv * sizeof (int16_t), cudaMemcpyHostToDevice, ctx->s_in));
      else
        CK (cudaMemcpyAsync (ctx->staged.as<float>() + v0, static_cast<const float *> (pcm) + v0, nv * sizeof (float), cudaMemcpyHostToDevice, ctx->s_in));
      CK (cudaEventRecord (ctx->stage_done[p], ctx->s_in));
    }
  ctx->stage_piece = piece_frames;
  ctx->stage_frames = n_frames;
  ctx->stage_ch = channels;
  ctx->stage_s16 = is_s16 != 0;
  ctx->stage_converted = 0;
  *device_out = ctx->staged.as<float>();
  return 0;
}

int
awm_pcm_stage_wait (awm_ctx *ctx, size_t n_frames)
{
  if (!ctx || !ctx->stage_piece || n_frames > ctx->stage_frames)
    return fail (ctx, "awm_pcm_stage_wait: nothing staged / beyond the staged stream");
  if (!n_frames)
    return 0;
  const size_t last = (n_frames - 1) / ctx->stage_piece;
  CK (cudaStreamWaitEvent (ctx->stream, ctx->stage_done[last], 0));
  for (; ctx->stage_s16 && ctx->stage_converted <= last; ctx->stage_converted++)
    {
      const size_t f0 = ctx->stage_converted * ctx->stage_piece, f1 = std::min (f0 + ctx->stage_piece, ctx->stage_frames);
      const size_t v0 = f0 * ctx->stage_ch;
      const long long nv = (long long) ((f1 - f0) * ctx->stage_ch);
      PROF (ctx);
      s16_to_f32_kernel (ctx->staged16.as<int16_t>() + v0, ctx->staged.as<float>() + v0)<<<unsigned (((nv + 1) / 2 + 255) / 256), 256, 0, ctx->stream>>> (ctx->staged16.as<int16_t>() + v0, ctx->staged.as<float>() + v0, nv);
      LAUNCH_CHECK ("k_s16_to_f32");
    }
  return 0;
}

/* the device copy of the bound PCM (float, [frames][channels]): lets a caller that bound 16 bit or host audio run device-pointer
 * entry points (awm_speed_scan, awm_gather) on it without another transfer */
const float *
awm_pcm_device (awm_ctx *ctx, size_t *n_frames, int *channels)
{
  if (!ctx || !ctx->pcm_ch)
    return nullptr;
  if (n_frames)
    *n_frames = ctx->pcm_frames;
  if (channels)
    *channels = ctx->pcm_ch;
  return ctx->pcm;
}

/* ---------------------------------------------------------------- embed */

namespace {

/* the arguments every entry point that reaches k_embed* shares.  The table row of a stream's first frame is 2*fpb - frames_pad_start,
 * which must not be negative.  A 1024-frame span touches at most two limiter blocks (k_embed keeps two peaks, k_embed_strip one
 * boundary per span), and the pipelined limiter of piece p - 1 runs after piece p's embed, so a block may reach at most half a piece
 * (AWM_PIECE >= 1024 frames) past its end: limiter_block is 0 (off) or in [AWM_MIN_LIMITER_BLOCK, AWM_MAX_LIMITER_BLOCK]. */
int
embed_args_check (awm_ctx *ctx, const char *name, int frames_pad_start, int fpb, int limiter_block)
{
  if (frames_pad_start < 0 || frames_pad_start > 2 * fpb)
    return fail (ctx, "%s: frames_pad_start %d outside [0, 2 * frames_per_block = %d]", name, frames_pad_start, 2 * fpb);
  if (limiter_block != 0 && (limiter_block < AWM_MIN_LIMITER_BLOCK || limiter_block > AWM_MAX_LIMITER_BLOCK))
    return fail (ctx, "%s: limiter block %d frames outside [%d, %d] (0 disables the limiter)", name, limiter_block, AWM_MIN_LIMITER_BLOCK,
                 AWM_MAX_LIMITER_BLOCK);
  return 0;
}

/* awm_embed / awm_embed_s16: `s16` selects 16 bit PCM buffers (in16 / out16) that are converted on the device */
int
embed_any (awm_ctx *ctx, const void *in_v, void *out_v, bool s16, size_t n_frames, int channels,
           uint64_t first_frame_number, int frames_pad_start, double water_delta,
           int limiter_block, float limiter_ceiling, double *snr_power, long long snr_pos0 = 0, long long snr_pos1 = LLONG_MAX)
{
  const float *in = s16 ? nullptr : static_cast<const float *> (in_v);
  float *out = s16 ? nullptr : static_cast<float *> (out_v);
  const int16_t *in16 = s16 ? static_cast<const int16_t *> (in_v) : nullptr;
  int16_t *out16 = s16 ? static_cast<int16_t *> (out_v) : nullptr;
  if (!ctx->embed_fpb)
    return fail (ctx, "awm_embed: awm_set_embed_tables has not been called");
  if (channels <= 0 || (n_frames && (!in_v || !out_v)))
    return fail (ctx, "awm_embed: bad arguments");
  if (embed_args_check (ctx, "awm_embed", frames_pad_start, ctx->embed_fpb, limiter_block))
    return 1;
  if (first_frame_number > AWM_MAX_STREAM_FRAMES / kFrame || first_frame_number * kFrame + n_frames > AWM_MAX_STREAM_FRAMES)
    return fail (ctx, "awm_embed: first_frame_number %llu * 1024 + n_frames %zu exceeds the stream length limit of 2^48 frames",
                 (unsigned long long) first_frame_number, n_frames);
  if (snr_power)
    snr_power[0] = snr_power[1] = 0;
  if (n_frames == 0)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const size_t n_val = n_frames * channels;
  /* 16 bit buffers always go through the float staging buffers; a device resident 16 bit buffer is converted in place of a copy */
  const bool in16_dev = s16 && is_device_ptr (in16), out16_dev = s16 && is_device_ptr (out16);
  const bool in_dev = !s16 && is_device_ptr (in), out_dev = !s16 && is_device_ptr (out);
  const float *d_in = in;
  float *d_out = out;
  if (!in_dev)
    {
      CK (ctx->emb_in.reserve (n_val * sizeof (float)));
      d_in = ctx->emb_in.as<float>();
    }
  if (!out_dev)
    {
      CK (ctx->emb_out.reserve (n_val * sizeof (float)));
      d_out = ctx->emb_out.as<float>();
    }
  const int16_t *d_in16 = in16;
  int16_t *d_out16 = out16;
  if (s16 && !in16_dev)
    {
      CK (ctx->emb_in16.reserve (n_val * sizeof (int16_t)));
      d_in16 = ctx->emb_in16.as<int16_t>();
    }
  if (s16 && !out16_dev)
    {
      CK (ctx->emb_out16.reserve (n_val * sizeof (int16_t)));
      d_out16 = ctx->emb_out16.as<int16_t>();
    }
  auto to_float = [&] (long long v0, long long v1, cudaStream_t st) -> int     /* values [v0, v1) of the 16 bit input -> emb_in */
    {
      if (v1 <= v0)
        return 0;
      if (st == ctx->stream)          /* the profile events live on the context stream */
        PROF (ctx);
      s16_to_f32_kernel (d_in16 + v0, ctx->emb_in.as<float>() + v0)<<<unsigned (((v1 - v0 + 1) / 2 + 255) / 256), 256, 0, st>>> (d_in16 + v0, ctx->emb_in.as<float>() + v0, v1 - v0);
      LAUNCH_CHECK ("k_s16_to_f32");
      return 0;
    };
  auto to_s16 = [&] (long long v0, long long v1, cudaStream_t st) -> int
    {
      if (v1 <= v0)
        return 0;
      if (st == ctx->stream)
        PROF (ctx);
      f32_to_s16_kernel (d_out + v0, d_out16 + v0)<<<unsigned (((v1 - v0 + 1) / 2 + 255) / 256), 256, 0, st>>> (d_out + v0, d_out16 + v0, v1 - v0);
      LAUNCH_CHECK ("k_f32_to_s16");
      return 0;
    };
  const long long n_real = (long long) ((n_frames + kFrame - 1) / kFrame);
  const long long n_proc = n_real + 1;
  long long n_blocks = 0;
  if (limiter_block > 0)
    {
      n_blocks = (n_proc * kFrame + limiter_block - 1) / limiter_block + 2;   // + partial first block of a mid-stream shard
      CK (ctx->peaks.reserve (n_blocks * sizeof (unsigned)));
      CK (cudaMemsetAsync (ctx->peaks.p, 0, n_blocks * sizeof (unsigned), ctx->stream));
    }
  if (snr_power)
    {
      CK (ctx->snr.reserve (2 * sizeof (double)));
      CK (cudaMemsetAsync (ctx->snr.p, 0, 2 * sizeof (double), ctx->stream));
    }
  EmbedArgs A;
  A.in = d_in;
  A.out = d_out;
  A.n_frames = (long long) n_frames;
  A.C = channels;
  A.n_proc = n_proc;
  A.fpb = ctx->embed_fpb;
  A.frame_number0 = (long long) (first_frame_number % (2ull * A.fpb)) + 2LL * A.fpb - frames_pad_start;   // WatermarkGen starts at 2*fpb - pad (src/wmadd.cc:295)
  A.frame_mod = ctx->frame_mod.as<uint8_t>();
  A.pow_up = 0.5f * float (-water_delta * 1);       // powf (mag, -Params::water_delta * data_bit_sign), src/wmadd.cc:79
  A.pow_down = 0.5f * float (-water_delta * -1);
  A.limiter_block = limiter_block;
  A.stream_pos0 = (long long) first_frame_number * kFrame;
  A.blk0 = limiter_block > 0 ? A.stream_pos0 / limiter_block : 0;
  A.peaks = ctx->peaks.as<unsigned>();
  A.snr = snr_power ? ctx->snr.as<double>() : nullptr;
  A.snr_frames = limiter_block > 0 ? n_proc : n_real;   // frames the reference loop emits (src/wmadd.cc:539-546)
  A.snr_pos0 = snr_pos0;
  A.snr_pos1 = snr_pos1;
  A.delta_only = 0;
  A.tw = ctx->tw.as<float2>();
  A.win = ctx->win.as<float>();
  A.synth = ctx->synth.as<float>();
  const size_t smem = kEmbedSmem;
  /* stereo audio in a 16-byte aligned buffer (bulk copies) with an 8-byte aligned output (float2 stores) streams through
   * k_embed_strip (awm_embed_strip.cuh); anything else takes k_embed, with float2 accesses where both buffers allow them */
  const uintptr_t in_a = reinterpret_cast<uintptr_t> (A.in), out_a = reinterpret_cast<uintptr_t> (A.out);
  const auto k_embed_any = ((in_a | out_a) & 7) == 0 ? k_embed<true> : k_embed<false>;
  if (set_smem (ctx, k_embed_any, smem)) return 1;
  const bool use_strip = channels == 2 && (in_a & 15) == 0 && (out_a & 7) == 0;
  if (use_strip)
    {
      if (!ctx->n_sms)
        CK (cudaDeviceGetAttribute (&ctx->n_sms, cudaDevAttrMultiProcessorCount, ctx->device));
      if (set_smem (ctx, k_embed_strip, kStripSmem)) return 1;
    }

  /* The buffer is processed in pieces of kPiece frames so that, for host buffers, the H2D copy of piece p+1, the
   * kernels of piece p and the D2H copy of piece p-1 overlap (three streams, events in between).  The arithmetic is
   * the same as for one launch: a piece only restricts which frames a launch emits, halo frames are read from the
   * (already copied) neighbour pieces, the limiter of a piece runs once the block peaks after it are final. */
  long long kPiece = 6144;                                   // 1024-frames per piece (6.3 M sample-frames, 25 MB of 16 bit stereo): measured best of 3072 .. 24576
  if (const char *e = getenv ("AWM_PIECE"))                  // measurement aid: other piece sizes
    kPiece = std::max (1024LL, atoll (e));
  const bool pipelined = !in_dev && !out_dev && !in16_dev && !out16_dev && n_proc > 2 * kPiece;
  const int n_pieces = pipelined ? int ((n_proc + kPiece - 1) / kPiece) : 1;
  auto piece_frames = [&] (int p, long long& fb, long long& fe) { fb = pipelined ? p * kPiece : 0; fe = pipelined ? std::min<long long> (fb + kPiece, n_proc) : n_proc; };
  auto piece_samples = [&] (int p, long long& s0, long long& s1) { long long fb, fe; piece_frames (p, fb, fe); s0 = std::min<long long> (fb * kFrame, n_frames); s1 = std::min<long long> (fe * kFrame, n_frames); };
  std::vector<cudaEvent_t> ev_in (n_pieces), ev_out (n_pieces);
  const bool trace_pipe = pipelined && getenv ("AWM_TRACE");     // device-side timeline of the three streams
  cudaEvent_t tr[4] = { nullptr, nullptr, nullptr, nullptr };
  const double t_host0 = wall_now();
  if (pipelined)
    {
      if (!ctx->s_in)
        {
          CK (cudaStreamCreateWithFlags (&ctx->s_in, cudaStreamNonBlocking));
          CK (cudaStreamCreateWithFlags (&ctx->s_out, cudaStreamNonBlocking));
        }
      for (int p = 0; p < n_pieces; p++)
        {
          CK (cudaEventCreateWithFlags (&ev_in[p], cudaEventDisableTiming));
          CK (cudaEventCreateWithFlags (&ev_out[p], cudaEventDisableTiming));
        }
      cudaEvent_t ev_start;
      CK (cudaEventCreateWithFlags (&ev_start, cudaEventDisableTiming));
      CK (cudaEventRecord (ev_start, ctx->stream));          // copies must not overtake earlier work on the context stream
      CK (cudaStreamWaitEvent (ctx->s_in, ev_start, 0));
      CK (cudaEventDestroy (ev_start));
      if (trace_pipe)
        {
          for (cudaEvent_t& e : tr)
            CK (cudaEventCreate (&e));
          CK (cudaEventRecord (tr[0], ctx->s_in));
        }
      for (int p = 0; p < n_pieces; p++)
        {
          long long s0, s1;
          piece_samples (p, s0, s1);
          if (s1 > s0 && !s16)
            CK (cudaMemcpyAsync (ctx->emb_in.as<float>() + s0 * channels, in + s0 * channels, size_t (s1 - s0) * channels * sizeof (float),
                                 cudaMemcpyHostToDevice, ctx->s_in));
          if (s1 > s0 && s16)
            {
              /* only the copy goes to the copy stream: a conversion kernel between two copies would leave the copy engine idle
               * while it runs (13 gaps per hour of audio); the conversion happens on the context stream once the piece is there */
              CK (cudaMemcpyAsync (ctx->emb_in16.as<int16_t>() + s0 * channels, in16 + s0 * channels, size_t (s1 - s0) * channels * sizeof (int16_t),
                                   cudaMemcpyHostToDevice, ctx->s_in));
            }
          CK (cudaEventRecord (ev_in[p], ctx->s_in));
        }
      if (trace_pipe)
        CK (cudaEventRecord (tr[1], ctx->s_in));
    }
  else if (s16)
    {
      if (!in16_dev)
        CK (cudaMemcpyAsync (ctx->emb_in16.p, in16, n_val * sizeof (int16_t), cudaMemcpyHostToDevice, ctx->stream));
      if (to_float (0, (long long) n_val, ctx->stream))
        return 1;
    }
  else if (!in_dev)
    CK (cudaMemcpyAsync (ctx->emb_in.p, in, n_val * sizeof (float), cudaMemcpyHostToDevice, ctx->stream));

  auto launch_limiter = [&] (int p) -> int
    {
      long long s0, s1;
      piece_samples (p, s0, s1);
      if (limiter_block > 0 && s1 > s0)
        {
          PROF (ctx);
          k_limiter<<<unsigned ((s1 - s0 + 256 * kLimiterIter - 1) / (256 * kLimiterIter)), 256, 0, ctx->stream>>> (d_out, s0, s1, channels, limiter_block, limiter_ceiling,
                                                                           ctx->peaks.as<unsigned>(), n_blocks, (long long) first_frame_number * kFrame);
          LAUNCH_CHECK ("k_limiter");
        }
      if (pipelined)
        {
          if (s1 > s0 && s16 && to_s16 (s0 * channels, s1 * channels, ctx->stream))      // the copy stream carries copies only
            return 1;
          CK (cudaEventRecord (ev_out[p], ctx->stream));
          CK (cudaStreamWaitEvent (ctx->s_out, ev_out[p], 0));
          if (s1 > s0 && !s16)
            CK (cudaMemcpyAsync (out + s0 * channels, d_out + s0 * channels, size_t (s1 - s0) * channels * sizeof (float),
                                 cudaMemcpyDeviceToHost, ctx->s_out));
          if (s1 > s0 && s16)
            CK (cudaMemcpyAsync (out16 + s0 * channels, d_out16 + s0 * channels, size_t (s1 - s0) * channels * sizeof (int16_t),
                                 cudaMemcpyDeviceToHost, ctx->s_out));
        }
      return 0;
    };
  int n_converted = 0;                                       // pieces of 16 bit input already turned into floats
  for (int p = 0; p < n_pieces; p++)
    {
      if (pipelined)
        {
          const int need = std::min (p + 1, n_pieces - 1);    // halo frame of the next piece
          CK (cudaStreamWaitEvent (ctx->stream, ev_in[need], 0));
          for (; s16 && n_converted <= need; n_converted++)
            {
              long long s0, s1;
              piece_samples (n_converted, s0, s1);
              if (to_float (s0 * channels, s1 * channels, ctx->stream))
                return 1;
            }
        }
      piece_frames (p, A.frame_begin, A.frame_end);
      if (use_strip)
        {
          /* strips long enough to make the two halo frames cheap, short enough to give every SM's warps one */
          const long long n_emit = A.frame_end - A.frame_begin;
          const int strip_len = int (std::max<long long> (16, (n_emit + (long long) ctx->n_sms * kStripWarps - 1) / ((long long) ctx->n_sms * kStripWarps)));
          const long long n_strips = (n_emit + strip_len - 1) / strip_len;
          PROF (ctx);
          k_embed_strip<<<unsigned ((n_strips + kStripWarps - 1) / kStripWarps), kStripWarps * 32, kStripSmem, ctx->stream>>> (A, strip_len);
          LAUNCH_CHECK ("k_embed_strip");
          prof_bytes (ctx, double (std::min<long long> (A.frame_end * kFrame, (long long) n_frames) - std::min<long long> (A.frame_begin * kFrame, (long long) n_frames)) * channels * 2 * sizeof (float));
          if (p > 0 && launch_limiter (p - 1))
            return 1;
          continue;
        }
      const unsigned grid = unsigned ((A.frame_end - A.frame_begin + kEmbedTile - 1) / kEmbedTile);
      PROF (ctx);
      k_embed_any<<<grid, kEmbedWarps * 32, smem, ctx->stream>>> (A);
      LAUNCH_CHECK ("k_embed");
      if (p > 0 && launch_limiter (p - 1))                     // peaks of the blocks after piece p-1 are final now
        return 1;
    }
  if (launch_limiter (n_pieces - 1))
    return 1;
  if (pipelined)
    {
      if (trace_pipe)
        {
          CK (cudaEventRecord (tr[2], ctx->stream));
          CK (cudaEventRecord (tr[3], ctx->s_out));
        }
      CK (cudaStreamSynchronize (ctx->s_out));
      if (trace_pipe)
        {
          float t_in = 0, t_k = 0, t_out = 0;
          cudaEventElapsedTime (&t_in, tr[0], tr[1]);
          cudaEventElapsedTime (&t_k, tr[0], tr[2]);
          cudaEventElapsedTime (&t_out, tr[0], tr[3]);
          fprintf (stderr, "[trace] embed pipeline (%d pieces): last H2D done %.2f ms, last kernel %.2f ms, last D2H %.2f ms, host issue %.2f ms\n",
                   n_pieces, t_in, t_k, t_out, (wall_now() - t_host0) * 1e3);
          for (cudaEvent_t e : tr)
            cudaEventDestroy (e);
        }
      for (int p = 0; p < n_pieces; p++)
        {
          cudaEventDestroy (ev_in[p]);
          cudaEventDestroy (ev_out[p]);
        }
    }
  else if (s16)
    {
      if (to_s16 (0, (long long) n_val, ctx->stream))
        return 1;
      if (!out16_dev)
        CK (cudaMemcpyAsync (out16, d_out16, n_val * sizeof (int16_t), cudaMemcpyDeviceToHost, ctx->stream));
    }
  else if (!out_dev)
    CK (cudaMemcpyAsync (out, d_out, n_val * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
  if (snr_power)
    CK (cudaMemcpyAsync (snr_power, ctx->snr.p, 2 * sizeof (double), cudaMemcpyDeviceToHost, ctx->stream));
  if ((s16 ? !out16_dev : !out_dev) || snr_power)
    CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

} // namespace

int
awm_embed (awm_ctx *ctx, const float *in, float *out, size_t n_frames, int channels,
           uint64_t first_frame_number, int frames_pad_start, double water_delta,
           int limiter_block, float limiter_ceiling, double *snr_power)
{
  return embed_any (ctx, in, out, false, n_frames, channels, first_frame_number, frames_pad_start, water_delta, limiter_block, limiter_ceiling, snr_power);
}

int
awm_embed_window (awm_ctx *ctx, const float *in, float *out, size_t n_frames, int channels,
                  uint64_t first_frame_number, int frames_pad_start, double water_delta,
                  int limiter_block, float limiter_ceiling, uint64_t snr_first, uint64_t snr_last, double *snr_power)
{
  return embed_any (ctx, in, out, false, n_frames, channels, first_frame_number, frames_pad_start, water_delta, limiter_block, limiter_ceiling, snr_power,
                    (long long) std::min<uint64_t> (snr_first, LLONG_MAX), (long long) std::min<uint64_t> (snr_last, LLONG_MAX));
}

int
awm_embed_s16 (awm_ctx *ctx, const int16_t *in, int16_t *out, size_t n_frames, int channels,
               uint64_t first_frame_number, int frames_pad_start, double water_delta,
               int limiter_block, float limiter_ceiling, double *snr_power)
{
  return embed_any (ctx, in, out, true, n_frames, channels, first_frame_number, frames_pad_start, water_delta, limiter_block, limiter_ceiling, snr_power);
}

int
awm_batch_validate (const awm_batch_item *items, size_t n_items, size_t n_values, char *err, size_t err_cap)
{
  auto bad = [&] (size_t i, const char *why)
    {
      if (err && err_cap)
        snprintf (err, err_cap, "batch item %zu: %s", i, why);
      return 1;
    };
  if (n_items && !items)
    return bad (0, "item list is NULL");
  for (size_t i = 0; i < n_items; i++)
    {
      const awm_batch_item& it = items[i];
      if (it.channels <= 0)
        return bad (i, "channels must be >= 1");
      if (it.n_frames > (n_values - std::min<uint64_t> (it.value_offset, n_values)) / uint64_t (it.channels) || it.value_offset > n_values)
        return bad (i, "extends past the end of the buffer");
    }
  if (err && err_cap)
    err[0] = 0;
  return 0;
}

namespace {

/* float images of a packed batch buffer: the caller's own buffers where they are float device memory, else the context's staging
 * buffers, which receive the input (16 bit input converted on the device) */
int
batch_images (awm_ctx *ctx, const void *in_v, void *out_v, bool s16, size_t n_values, const float **d_in_out, float **d_out_out)
{
  const bool in_dev = is_device_ptr (in_v), out_dev = is_device_ptr (out_v);
  const float *d_in = !s16 && in_dev ? static_cast<const float *> (in_v) : nullptr;
  float *d_out = !s16 && out_dev ? static_cast<float *> (out_v) : nullptr;
  if (!d_in)
    {
      CK (ctx->emb_in.reserve (n_values * sizeof (float)));
      d_in = ctx->emb_in.as<float>();
    }
  if (!d_out)
    {
      CK (ctx->emb_out.reserve (n_values * sizeof (float)));
      d_out = ctx->emb_out.as<float>();
    }
  if (s16)
    {
      const int16_t *d_in16 = static_cast<const int16_t *> (in_v);
      if (!in_dev)
        {
          CK (ctx->emb_in16.reserve (n_values * sizeof (int16_t)));
          CK (cudaMemcpyAsync (ctx->emb_in16.p, in_v, n_values * sizeof (int16_t), cudaMemcpyHostToDevice, ctx->stream));
          d_in16 = ctx->emb_in16.as<int16_t>();
        }
      PROF (ctx);
      s16_to_f32_kernel (d_in16, ctx->emb_in.as<float>())<<<unsigned (((n_values + 1) / 2 + 255) / 256), 256, 0, ctx->stream>>> (d_in16, ctx->emb_in.as<float>(), (long long) n_values);
      LAUNCH_CHECK ("k_s16_to_f32");
    }
  else if (!in_dev)
    CK (cudaMemcpyAsync (ctx->emb_in.p, in_v, n_values * sizeof (float), cudaMemcpyHostToDevice, ctx->stream));
  *d_in_out = d_in;
  *d_out_out = d_out;
  return 0;
}

/* the float image d_out of batch_images into out_v (16 bit output converted on the device), the --snr sums into snr_power */
int
batch_finish (awm_ctx *ctx, void *out_v, bool s16, size_t n_values, const float *d_out, double *snr_power, size_t n_snr)
{
  const bool out_dev = is_device_ptr (out_v);
  if (s16)
    {
      int16_t *d_out16 = static_cast<int16_t *> (out_v);
      if (!out_dev)
        {
          CK (ctx->emb_out16.reserve (n_values * sizeof (int16_t)));
          d_out16 = ctx->emb_out16.as<int16_t>();
        }
      PROF (ctx);
      f32_to_s16_kernel (d_out, d_out16)<<<unsigned (((n_values + 1) / 2 + 255) / 256), 256, 0, ctx->stream>>> (d_out, d_out16, (long long) n_values);
      LAUNCH_CHECK ("k_f32_to_s16");
      if (!out_dev)
        CK (cudaMemcpyAsync (out_v, d_out16, n_values * sizeof (int16_t), cudaMemcpyDeviceToHost, ctx->stream));
    }
  else if (!out_dev)
    CK (cudaMemcpyAsync (out_v, d_out, n_values * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
  if (snr_power && n_snr)
    CK (cudaMemcpyAsync (snr_power, ctx->snr.p, 2 * n_snr * sizeof (double), cudaMemcpyDeviceToHost, ctx->stream));
  if (!out_dev || snr_power)
    CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

/* k_embed_batch work list entry of a non-empty item with awm_embed's geometry (limiter_block 0: no block peaks); advances the
 * launch's tile / limiter CTA counters and the flat peak array.  zero_frames: the item ends a stream that began that many
 * sample-frames earlier with silence (awm_embed_batch_offsets); its processed range starts one frame before the item's first
 * frame (awm_embed_batch.cuh) */
BatchItem
batch_entry (long long v0, long long n_frames, int C, int item, int limiter_block, long long& n_tiles, long long& n_lim, long long& n_peaks,
             long long zero_frames = 0, int role_table = 0)
{
  BatchItem b;
  b.role_table = role_table;
  b.v0 = v0;
  b.n_frames = n_frames;
  b.C = C;
  b.item = item;
  b.frame0 = zero_frames >= 2 * kFrame ? zero_frames / kFrame - 1 : 0;
  b.lead = zero_frames - b.frame0 * kFrame;
  b.blk0 = limiter_block > 0 ? b.frame0 * kFrame / limiter_block : 0;
  const long long n_proc = (b.lead + b.n_frames + kFrame - 1) / kFrame + 1;
  b.tile0 = n_tiles;
  b.lim0 = n_lim;
  b.peak0 = n_peaks;
  b.n_blocks = limiter_block > 0 ? (n_proc * kFrame + limiter_block - 1) / limiter_block + 2 : 0;   // as awm_embed's
  n_tiles += (n_proc + kEmbedTile - 1) / kEmbedTile;
  n_lim += (b.n_frames + 256 * kLimiterIter - 1) / (256 * kLimiterIter);
  n_peaks += b.n_blocks;
  return b;
}

/* the role tables a batch reads: one key's (awm_set_embed_roles) or a key set's (awm_set_embed_roles_keys), [role_table][fpb][101] */
struct RoleSet { const uint16_t *p; int fpb, n_coded; bool per_item; };

/* k_embed_batch over the n_list items at d_items (v0 relative to in / out), then k_limiter_batch when limiter_block > 0.
 * Peaks go to ctx->peaks (zeroed by the caller), --snr sums to d_snr (null: none); delta_only: write the watermark signal alone */
int
launch_embed_batch (awm_ctx *ctx, const RoleSet& rs, const float *in, float *out, const BatchItem *d_items, int n_list, long long n_tiles, long long n_lim,
                    int frames_pad_start, double water_delta, int limiter_block, float limiter_ceiling, double *d_snr, int delta_only,
                    bool offsets = false)
{
  EmbedArgs A = {};
  A.in = in;
  A.out = out;
  A.fpb = rs.fpb;
  A.frame_number0 = 2LL * A.fpb - frames_pad_start;       // of a stream start; each item adds its frame0
  A.pow_up = 0.5f * float (-water_delta * 1);
  A.pow_down = 0.5f * float (-water_delta * -1);
  A.limiter_block = limiter_block;
  A.peaks = ctx->peaks.as<unsigned>();
  A.snr = d_snr;
  A.snr_pos1 = LLONG_MAX;
  A.delta_only = delta_only;
  A.tw = ctx->tw.as<float2>();
  A.win = ctx->win.as<float>();
  A.synth = ctx->synth.as<float>();
  /* items at stream offsets take their own instance: the offset arithmetic costs the stream-start case registers and spills; so does
   * a role table per item, whose batches always take the offsets instance (zero offsets give the stream-start result) */
  auto kernel = rs.per_item ? k_embed_batch<true, true> : offsets ? k_embed_batch<true, false> : k_embed_batch<false, false>;
  if (set_smem (ctx, kernel, kEmbedBatchSmem)) return 1;
  PROF (ctx);
  kernel<<<unsigned (n_tiles), kEmbedWarps * 32, kEmbedBatchSmem, ctx->stream>>> (A, d_items, n_list, rs.p, ctx->batch_coded.as<uint8_t>(),
                                                                                 rs.n_coded);
  LAUNCH_CHECK ("k_embed_batch");
  if (limiter_block > 0)
    {
      PROF (ctx);
      k_limiter_batch<<<unsigned (n_lim), 256, 0, ctx->stream>>> (out, d_items, n_list, limiter_block, limiter_ceiling, ctx->peaks.as<unsigned>());
      LAUNCH_CHECK ("k_limiter_batch");
    }
  return 0;
}

/* awm_batch_validate plus the offset list of awm_embed_batch_offsets (NULL: all zero) */
int
batch_offsets_check (const awm_batch_item *items, size_t n_items, size_t n_values, const uint64_t *zero_frames, bool need_list, char *err, size_t err_cap)
{
  if (awm_batch_validate (items, n_items, n_values, err, err_cap))
    return 1;
  if (!zero_frames)
    {
      if (need_list && n_items)
        {
          if (err && err_cap)
            snprintf (err, err_cap, "zero_frames list is NULL");
          return 1;
        }
      return 0;
    }
  for (size_t i = 0; i < n_items; i++)
    if (zero_frames[i] > AWM_MAX_STREAM_FRAMES || items[i].n_frames > AWM_MAX_STREAM_FRAMES - zero_frames[i])
      {
        if (err && err_cap)
          snprintf (err, err_cap, "batch item %zu: zero_frames %llu + n_frames %llu exceeds the stream length limit of 2^48 frames", i,
                    (unsigned long long) zero_frames[i], (unsigned long long) items[i].n_frames);
        return 1;
      }
  return 0;
}

} // namespace

int
awm_batch_offsets_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const uint64_t *zero_frames, int sample_rate,
                            int mark_sample_rate, char *err, size_t err_cap)
{
  if (batch_offsets_check (items, n_items, n_values, zero_frames, true, err, err_cap))
    return 1;
  if (sample_rate != mark_sample_rate)
    for (size_t i = 0; i < n_items; i++)
      if (zero_frames[i])
        {
          if (err && err_cap)
            snprintf (err, err_cap, "batch item %zu: stream offsets are only supported at %d Hz", i, mark_sample_rate);
          return 1;
        }
  if (err && err_cap)
    err[0] = 0;
  return 0;
}

/* ---------------------------------------------------------------- sync search */

namespace {

/* the search of awm_sync_approx on the bound PCM into approx slot `s`, on ctx->stream */
int
approx_launch (awm_ctx *ctx, awm_ctx::ApproxSlot& s, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last,
               double water_delta, awm_search_score *scores_out, size_t max_scores, size_t *n_scores)
{
  if (key_slot < 0 || key_slot >= AWM_MAX_KEYS || mode < 0 || mode > 1 || !n_scores)
    return fail (ctx, "awm_sync_approx: bad arguments");
  SyncTab& t = ctx->keys[key_slot].sync[mode];
  const int fpb = ctx->keys[key_slot].fpb;
  if (!t.n_ent || !fpb)
    return fail (ctx, "awm_sync_approx: tables for key slot %d / mode %d not set", key_slot, mode);
  if (!ctx->pcm_ch)
    return fail (ctx, "awm_sync_approx: no PCM bound");
  CK (cudaSetDevice (ctx->device));
  const int total = fpb * (mode == AWM_MODE_CLIP ? 2 : 1);
  /* start frame s reads frame s + entry frame: past the block it would read the scores of a later start frame, or another entry's row */
  if (t.max_frame >= total)
    return fail (ctx, "awm_sync_approx: sync entry frame %d is not inside the %d frames of a search (frames_per_block %d)", t.max_frame, total, fpb);
  const long long fc = (long long) (ctx->pcm_frames / kFrame);           // frame_count (wav_data)
  const long long n_out = fc > 0 ? fc - 1 : 0;                           // sync_fft_parallel: frame_count - 1 frames per shift
  const long long n_starts = fc - total - 1 > 0 ? fc - total - 1 : 0;    // (start + total) * n_bands < fft_db.size()
  *n_scores = size_t (n_starts) * 4;
  s.n_scores = 0;
  s.n_have = 0;
  s.pcm = ctx->pcm;
  s.pcm_frames = ctx->pcm_frames;
  s.pcm_ch = ctx->pcm_ch;
  if (!s.done)
    CK (cudaEventCreateWithFlags (&s.done, cudaEventDisableTiming));
  if (n_starts == 0)
    {
      CK (cudaEventRecord (s.done, ctx->stream));
      return 0;
    }
  if (scores_out && max_scores < size_t (n_starts) * 4)
    return fail (ctx, "awm_sync_approx: scores_out too small (%zu < %lld)", max_scores, n_starts * 4);
  const int ld = int ((n_out + 127) / 128 * 128);
  CK (s.have.reserve (size_t (4) * ld));
  CK (s.q.reserve (size_t (n_starts) * 4 * sizeof (double)));
  CK (s.a_ud.reserve (size_t (n_starts) * 4 * t.n_bits * 2 * sizeof (float)));
  CK (s.a_cnt.reserve (size_t (n_starts) * 4 * t.n_bits * sizeof (int)));
  CK (s.scores.reserve (size_t (n_starts) * 4 * sizeof (awm_search_score)));
  const double norm_div = water_delta < 0.080 ? water_delta : 0.080;     // normalize_sync_quality, src/syncfinder.cc:90
  /* default: entry sums on the tensor cores (k_stft_mags_tc, awm_approx_tc.cuh) + one streaming gather.  AWM_APPROX selects the
   * test references: simt = the same entry sums on the fp32 pipes (k_stft_mags, awm_approx_mags.cuh); ring = the kernel that walks
   * the dB matrix per start frame in the reference's exact summation order.  Read per call: tests compare the kernels in one process */
  const char *env_approx = getenv ("AWM_APPROX");
  const bool force_ring = env_approx && !strcmp (env_approx, "ring"), force_simt = env_approx && !strcmp (env_approx, "simt");
  if (!force_ring && t.n_ent <= kGatherMaxEntries)
    {
      CK (ctx->a_mags.reserve (size_t (4) * t.n_ent * ld * sizeof (float2)));
      if (!force_simt)
        {
          if (!ctx->n_sms)
            CK (cudaDeviceGetAttribute (&ctx->n_sms, cudaDevAttrMultiProcessorCount, ctx->device));
          const int n_tiles = 4 * int ((n_out + kTcTile - 1) / kTcTile);
          const unsigned grid = unsigned (std::min (n_tiles, ctx->n_sms));
          /* stereo PCM in a 16-byte aligned buffer reaches the FFT warps by bulk copies, anything else by global loads */
          const int tma_ok = ctx->pcm_ch == 2 && (reinterpret_cast<uintptr_t> (ctx->pcm) & 15) == 0;
          if (set_smem (ctx, k_stft_mags_tc, kTcSmemBytes)) return 1;
          PROF (ctx);
          k_stft_mags_tc<<<grid, (kTcFftWarps + kTcEpiWarps) * 32, kTcSmemBytes, ctx->stream>>> (ctx->pcm, (long long) ctx->pcm_frames,
            ctx->pcm_ch, int (n_out), ld, t.masks.as<unsigned char>(), t.n_ent, t.n_chunks, ctx->a_mags.as<float2>(),
            s.have.as<unsigned char>(), (long long) wav_first, (long long) wav_last, ctx->tw.as<float2>(), ctx->win.as<float>(), tma_ok);
          LAUNCH_CHECK ("k_stft_mags_tc");
          prof_bytes (ctx, double (ctx->pcm_frames) * ctx->pcm_ch * sizeof (float) + double (4) * t.n_ent * n_out * sizeof (float2));   /* PCM in, entry sums out */
        }
      else
      {
        const size_t smem = kMagSmem2;
        if (set_smem (ctx, k_stft_mags, smem)) return 1;
        const unsigned grid = 4u * unsigned ((n_out + kMagTile - 1) / kMagTile);
        PROF (ctx);
        k_stft_mags<<<grid, kMagWarps2 * 32, smem, ctx->stream>>> (ctx->pcm, (long long) ctx->pcm_frames, ctx->pcm_ch, int (n_out), ld,
                                                                  t.ent.as<awm_sync_entry>(), t.n_ent, ctx->a_mags.as<float2>(), s.have.as<unsigned char>(),
                                                                  (long long) wav_first, (long long) wav_last, ctx->tw.as<float2>(), ctx->win.as<float>());
        LAUNCH_CHECK ("k_stft_mags");
        prof_bytes (ctx, double (ctx->pcm_frames) * ctx->pcm_ch * sizeof (float) + double (4) * t.n_ent * n_out * sizeof (float2));   /* PCM in, entry sums out */
      }
      dim3 grid (unsigned ((n_starts + 255) / 256), 4);
      PROF (ctx);
      if (mode == AWM_MODE_CLIP)
        k_sync_gather<true><<<grid, 256, 0, ctx->stream>>> (ctx->a_mags.as<float2>(), s.have.as<unsigned char>(), ld, int (n_starts), t.ent.as<awm_sync_entry>(), t.n_ent,
                                                            t.off.as<int>(), t.n_bits, s.a_ud.as<float>(), s.a_cnt.as<int>());
      else
        k_sync_gather<false><<<grid, 256, 0, ctx->stream>>> (ctx->a_mags.as<float2>(), s.have.as<unsigned char>(), ld, int (n_starts), t.ent.as<awm_sync_entry>(), t.n_ent,
                                                             t.off.as<int>(), t.n_bits, s.a_ud.as<float>(), s.a_cnt.as<int>());
      LAUNCH_CHECK ("k_sync_gather");
      /* every (start frame, entry) pair reads its float2 once; the per-bit sums are written once */
      prof_bytes (ctx, double (4) * n_starts * t.n_ent * sizeof (float2) + double (4) * n_starts * t.n_bits * 12.0);
    }
  else
    {
      CK (ctx->dbT.reserve (size_t (4) * kBands * ld * sizeof (float)));
      {
        const size_t smem = fft_smem_bytes (kStftWarps) + kBands * (kStftWarps + 1) * sizeof (float);
        if (set_smem (ctx, k_stft_db, smem)) return 1;
        const unsigned grid = 4u * unsigned ((n_out + kStftWarps - 1) / kStftWarps);
        PROF (ctx);
        k_stft_db<<<grid, kStftWarps * 32, smem, ctx->stream>>> (ctx->pcm, (long long) ctx->pcm_frames, ctx->pcm_ch, int (n_out), ld,
                                                                ctx->dbT.as<float>(), s.have.as<unsigned char>(),
                                                                (long long) wav_first, (long long) wav_last,
                                                                ctx->tw.as<float2>(), ctx->win.as<float>());
        LAUNCH_CHECK ("k_stft_db");
      }
      {
        const size_t smem = kApproxSmem;
        dim3 grid (unsigned ((n_starts + kApproxCands - 1) / kApproxCands), 4);
        if (mode == AWM_MODE_CLIP)
          {
            if (set_smem (ctx, k_sync_approx<true>, smem)) return 1;
            PROF (ctx);
            k_sync_approx<true><<<grid, kApproxThreads, smem, ctx->stream>>> (ctx->dbT.as<float>(), s.have.as<unsigned char>(), ld, int (n_out), int (n_starts),
                                                                            t.sorted.as<ApproxEntry>(), t.groups.as<int>(), t.n_groups, t.n_bits,
                                                                            s.a_ud.as<float>(), s.a_cnt.as<int>());
          }
        else
          {
            if (set_smem (ctx, k_sync_approx<false>, smem)) return 1;
            PROF (ctx);
            k_sync_approx<false><<<grid, kApproxThreads, smem, ctx->stream>>> (ctx->dbT.as<float>(), s.have.as<unsigned char>(), ld, int (n_out), int (n_starts),
                                                                             t.sorted.as<ApproxEntry>(), t.groups.as<int>(), t.n_groups, t.n_bits,
                                                                             s.a_ud.as<float>(), s.a_cnt.as<int>());
          }
        LAUNCH_CHECK ("k_sync_approx");
      }
    }
  {
    PROF (ctx);
    k_sync_quality<<<unsigned ((n_starts * 4 + 255) / 256), 256, 0, ctx->stream>>> (s.a_ud.as<float>(), s.a_cnt.as<int>(), int (n_starts), t.n_bits,
                                                                                norm_div, s.q.as<double>());
    LAUNCH_CHECK ("k_sync_quality");
  }
  {
    const long long n = n_starts * 4;
    PROF (ctx);
    k_local_mean<<<unsigned ((n + 255) / 256), 256, 0, ctx->stream>>> (s.q.as<double>(), n, s.scores.as<awm_search_score>());
    LAUNCH_CHECK ("k_local_mean");
  }
  s.n_scores = size_t (n_starts) * 4;
  s.n_have = n_out;
  s.ld_have = ld;
  CK (cudaEventRecord (s.done, ctx->stream));
  if (scores_out)
    {
      CK (cudaMemcpyAsync (scores_out, s.scores.p, size_t (n_starts) * 4 * sizeof (awm_search_score), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaStreamSynchronize (ctx->stream));
    }
  return 0;
}

} // namespace

int
awm_sync_approx (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last,
                 double water_delta, awm_search_score *scores_out, size_t max_scores, size_t *n_scores)
{
  /* searches still running on s_approx write a_mags: the search below waits for them */
  for (auto& s : ctx->aslot)
    if (s.done)
      CK (cudaStreamWaitEvent (ctx->stream, s.done, 0));
  return approx_launch (ctx, ctx->aslot[ctx->cur_aslot], key_slot, mode, wav_first, wav_last, water_delta, scores_out, max_scores, n_scores);
}

int
awm_sync_approx_enqueue (awm_ctx *ctx, int slot, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta)
{
  if (slot < 0 || slot > 1)
    return fail (ctx, "awm_sync_approx_enqueue: bad slot %d", slot);
  /* the slot keeps a pointer to the bound PCM until it is used: a buffer of the context would be overwritten by the next bind or
   * stage in the meantime */
  const void *own[] = { ctx->pcm_own.p, ctx->staged.p, ctx->pcm_rs.p };
  for (const void *b : own)
    if (b && ctx->pcm == b)
      return fail (ctx, "awm_sync_approx_enqueue: the bound PCM must be the caller's device memory, not a buffer of the context");
  CK (cudaSetDevice (ctx->device));
  if (!ctx->s_approx)
    CK (cudaStreamCreateWithFlags (&ctx->s_approx, cudaStreamNonBlocking));
  /* the PCM may have been written, and the slot's buffers may still be read, by work queued on the context stream */
  cudaEvent_t busy;
  CK (cudaEventCreateWithFlags (&busy, cudaEventDisableTiming));
  CK (cudaEventRecord (busy, ctx->stream));
  CK (cudaStreamWaitEvent (ctx->s_approx, busy, 0));
  CK (cudaEventDestroy (busy));
  /* the launch code queues its kernels and profiling records on ctx->stream */
  cudaStream_t main_stream = ctx->stream;
  ctx->stream = ctx->s_approx;
  size_t n_scores = 0;
  const int r = approx_launch (ctx, ctx->aslot[slot], key_slot, mode, wav_first, wav_last, water_delta, nullptr, 0, &n_scores);
  ctx->stream = main_stream;
  return r;
}

int
awm_sync_use_slot (awm_ctx *ctx, int slot, size_t *n_scores)
{
  if (slot < 0 || slot > 1 || !ctx->aslot[slot].done)
    return fail (ctx, "awm_sync_use_slot: nothing searched in slot %d", slot);
  awm_ctx::ApproxSlot& s = ctx->aslot[slot];
  CK (cudaSetDevice (ctx->device));
  CK (cudaStreamWaitEvent (ctx->stream, s.done, 0));
  ctx->cur_aslot = slot;
  ctx->pcm = s.pcm;
  ctx->pcm_frames = s.pcm_frames;
  ctx->pcm_ch = s.pcm_ch;
  if (n_scores)
    *n_scores = s.n_scores;
  return 0;
}

int
awm_sync_have (awm_ctx *ctx, unsigned char *out, size_t max, size_t *n_frames)
{
  if (!n_frames || (max && !out))
    return fail (ctx, "awm_sync_have: bad arguments");
  const awm_ctx::ApproxSlot& s = ctx->aslot[ctx->cur_aslot];
  *n_frames = size_t (s.n_have);
  if (!s.n_have || !max)
    return 0;
  if (max < size_t (4) * s.n_have)
    return fail (ctx, "awm_sync_have: out too small (%zu < %lld)", max, 4 * s.n_have);
  CK (cudaSetDevice (ctx->device));
  CK (cudaMemcpy2DAsync (out, size_t (s.n_have), s.have.p, size_t (s.ld_have), size_t (s.n_have), 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

int
awm_sync_peaks (awm_ctx *ctx, double min_abs_quality, awm_search_score *out, size_t max, size_t *n)
{
  if (!n || (max && !out))
    return fail (ctx, "awm_sync_peaks: bad arguments");
  *n = 0;
  awm_ctx::ApproxSlot& s = ctx->aslot[ctx->cur_aslot];
  if (!s.n_scores)
    return 0;
  CK (cudaSetDevice (ctx->device));
  /* counter and entries share one buffer ([u64 count, u64 pad][entries]) so that the usual case -- a few dozen peaks -- comes back
   * with ONE device-to-host copy and one synchronisation instead of two of each */
  constexpr size_t kHead = 16, kFirst = 2048;
  CK (ctx->peaks_out.reserve (kHead + std::max<size_t> (max, 1) * sizeof (awm_search_score)));
  unsigned char *base = ctx->peaks_out.as<unsigned char>();
  CK (cudaMemsetAsync (base, 0, kHead, ctx->stream));
  const long long ns = (long long) s.n_scores;
  PROF (ctx);
  k_peaks<<<unsigned ((ns + 255) / 256), 256, 0, ctx->stream>>> (s.scores.as<awm_search_score>(), ns, min_abs_quality,
                                                                reinterpret_cast<awm_search_score *> (base + kHead), (unsigned long long) max,
                                                                reinterpret_cast<unsigned long long *> (base));
  LAUNCH_CHECK ("k_peaks");
  const size_t first = std::min (max, kFirst);
  ctx->pin.reset();
  unsigned char *stage = ctx->pin.get<unsigned char> (kHead + first * sizeof (awm_search_score));
  if (!stage)
    return fail (ctx, "awm_sync_peaks: out of page-locked memory");
  CK (cudaMemcpyAsync (stage, base, kHead + first * sizeof (awm_search_score), cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  unsigned long long cnt = 0;
  memcpy (&cnt, stage, sizeof (cnt));
  *n = size_t (cnt);
  const size_t got = std::min<size_t> (cnt, max);
  if (got)
    {
      memcpy (out, stage + kHead, std::min (got, first) * sizeof (awm_search_score));
      if (got > first)
        {
          CK (cudaMemcpyAsync (out + first, base + kHead + first * sizeof (awm_search_score), (got - first) * sizeof (awm_search_score), cudaMemcpyDeviceToHost, ctx->stream));
          CK (cudaStreamSynchronize (ctx->stream));
        }
      std::sort (out, out + got, [] (const awm_search_score& a, const awm_search_score& b) { return a.index < b.index; });
    }
  return 0;
}

/* what a refine call hands back */
enum class RefineOut
{
  Refined,          // the best fine offset of every candidate (awm_sync_refine)
  Exact,            // the exact quality of every fine offset (awm_sync_refine_offsets, exact = 1)
  Sliding,          // the sliding quality of every fine offset, the exact one above two channels (awm_sync_refine_offsets, exact = 0)
  Rescored,         // the fine offsets that are scored exactly (awm_sync_refine_rescored)
};

/* Up to two channels a sliding DFT ranks the 65 fine offsets of every candidate and only the offsets it picks are scored exactly;
 * above two channels, and for the exact per-offset qualities, every valid offset is.  Refined is written to `refined`, Exact and
 * Sliding to q_out / valid_out ([n_scores][65], invalid offsets 0), Rescored to rescored_out ([n_scores][65], 1 = scored exactly). */
static int
refine_impl (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta,
             const awm_search_score *scores, size_t n_scores, RefineOut want, awm_search_score *refined, double *q_out,
             unsigned char *valid_out, unsigned char *rescored_out)
{
  if (key_slot < 0 || key_slot >= AWM_MAX_KEYS || mode < 0 || mode > 1 || (n_scores && !scores))
    return fail (ctx, "awm_sync_refine: bad arguments");
  SyncTab& t = ctx->keys[key_slot].sync[mode];
  const int fpb = ctx->keys[key_slot].fpb;
  if (!t.n_ent || !fpb)
    return fail (ctx, "awm_sync_refine: tables for key slot %d / mode %d not set", key_slot, mode);
  if (!ctx->pcm_ch)
    return fail (ctx, "awm_sync_refine: no PCM bound");
  if (n_scores == 0)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const int total = fpb * (mode == AWM_MODE_CLIP ? 2 : 1);
  const double norm_div = water_delta < 0.080 ? water_delta : 0.080;

  const size_t nc = n_scores;
  const size_t np_max = nc * kOffsets;
  const int n_bits = t.n_bits;
  CK (ctx->cand_start.reserve (nc * sizeof (long long)));
  CK (ctx->cand_noff.reserve (nc * sizeof (int)));
  CK (ctx->r_ud.reserve (nc * kOffsets * n_bits * 2 * sizeof (float)));
  CK (ctx->r_cnt.reserve (nc * kOffsets * n_bits * sizeof (int)));
  CK (ctx->rvalid.reserve (nc * kOffsets));
  ctx->pin.reset();
  long long *h_start = ctx->pin.get<long long> (nc);
  int *h_noff = ctx->pin.get<int> (nc);
  if (!h_start || !h_noff)
    return fail (ctx, "awm_sync_refine: out of page-locked memory");
  for (size_t c = 0; c < nc; c++)
    {
      // int start = max (int (index) - sync_search_step, 0); end = index + sync_search_step; step sync_search_fine
      const long long idx = (long long) scores[c].index;
      const long long start = std::max<long long> (idx - 256, 0), end = idx + 256;
      h_start[c] = start;
      h_noff[c] = int (std::min<long long> ((end - start) / 8 + 1, kOffsets));
    }
  CK (cudaMemcpyAsync (ctx->cand_start.p, h_start, nc * sizeof (long long), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaMemcpyAsync (ctx->cand_noff.p, h_noff, nc * sizeof (int), cudaMemcpyHostToDevice, ctx->stream));
  const bool slide = ctx->pcm_ch <= 2 && want != RefineOut::Exact;        // the sliding pass is written for one and two channels
  /* a float2 per (candidate, offset, entry) from the sliding pass, 2 x kUD band values per (pair, entry) from the exact re-score of up
   * to all 65 offsets (k_refine_exact_fft_n): no reallocation between the kernels */
  CK (ctx->r_ent_ud.reserve (np_max * t.n_ent * 2 * kUD * sizeof (float)));
  if (slide)
    {
      if (!ctx->tw1024.p)
        {
          std::vector<float2> tw (1024);
          for (int p = 0; p < 1024; p++)
            {
              const double a = -2.0 * M_PI * double (p) / 1024.0;
              tw[p] = make_float2 (float (cos (a)), float (sin (a)));
            }
          CK (ctx->tw1024.reserve (tw.size() * sizeof (float2)));
          CK (cudaMemcpy (ctx->tw1024.p, tw.data(), tw.size() * sizeof (float2), cudaMemcpyHostToDevice));
        }
      CK (ctx->r_ent_flag.reserve (np_max * t.n_ent));
      const size_t smem = fft_smem_bytes (kSlideWarps);
      const long long jobs = (long long) nc * t.n_ent;
      const unsigned grid = unsigned ((jobs + kSlideWarps - 1) / kSlideWarps);
      PROF (ctx);
      if (ctx->pcm_ch == 2)
        {
          if (set_smem (ctx, k_refine_slide<2>, smem)) return 1;
          k_refine_slide<2><<<grid, kSlideWarps * 32, smem, ctx->stream>>> (ctx->pcm, (long long) ctx->pcm_frames, ctx->cand_start.as<long long>(), ctx->cand_noff.as<int>(), int (nc),
            t.ent.as<awm_sync_entry>(), t.n_ent, total, (long long) wav_first, (long long) wav_last, ctx->r_ent_ud.as<float2>(), ctx->r_ent_flag.as<unsigned char>(),
            ctx->tw.as<float2>(), ctx->tw1024.as<float2>());
        }
      else
        {
          if (set_smem (ctx, k_refine_slide<1>, smem)) return 1;
          k_refine_slide<1><<<grid, kSlideWarps * 32, smem, ctx->stream>>> (ctx->pcm, (long long) ctx->pcm_frames, ctx->cand_start.as<long long>(), ctx->cand_noff.as<int>(), int (nc),
            t.ent.as<awm_sync_entry>(), t.n_ent, total, (long long) wav_first, (long long) wav_last, ctx->r_ent_ud.as<float2>(), ctx->r_ent_flag.as<unsigned char>(),
            ctx->tw.as<float2>(), ctx->tw1024.as<float2>());
        }
      LAUNCH_CHECK ("k_refine_slide");
      /* what the kernel has to read: of every candidate's block only the SYNC frames (n_ent of the 2226), each with the 512 samples the
       * 64 slides walk over -- not the whole block */
      prof_bytes (ctx, double (nc) * double (t.n_ent) * (double (kFrame) + 512.0) * ctx->pcm_ch * sizeof (float));
      const long long n_red = (long long) nc * kOffsets * n_bits;
      PROF (ctx);
      k_refine_reduce<<<unsigned ((n_red + 127) / 128), 128, 0, ctx->stream>>> (ctx->r_ent_ud.as<float2>(), ctx->r_ent_flag.as<unsigned char>(), int (nc), t.n_ent,
        t.off.as<int>(), n_bits, ctx->cand_start.as<long long>(), ctx->cand_noff.as<int>(), (long long) ctx->pcm_frames, total,
        ctx->r_ud.as<float>(), ctx->r_cnt.as<int>(), ctx->rvalid.as<unsigned char>());
      LAUNCH_CHECK ("k_refine_reduce");
    }
  // sync_decode epilogue (src/syncfinder.cc:94-114,144-152) from the per-bit float sums
  auto quality_of = [&] (const float *ud, const int *cnt, size_t base) -> double
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
            raw_bit = 1 - umag / dmag;
          else
            raw_bit = dmag / umag - 1;
          sync_quality += ((bit & 1) ? raw_bit : -raw_bit) * cnt[ob];
          bit_count += cnt[ob];
        }
      if (bit_count)
        sync_quality /= bit_count;
      return sync_quality / norm_div / 2.9;
    };
  /* the pair list (start, candidate, offset) and its length, and the sums of up to np_max pairs: those of k_refine_reduce
   * ([candidate][65]) or those of the exact re-score (in list order) */
  int *e_n = ctx->pin.get<int> (1);
  int *e_cand = ctx->pin.get<int> (np_max);
  int *e_off = ctx->pin.get<int> (np_max);
  float *e_ud = ctx->pin.get<float> (np_max * n_bits * 2);
  int *e_cnt = ctx->pin.get<int> (np_max * n_bits);
  unsigned char *e_valid = ctx->pin.get<unsigned char> (np_max);
  if (!e_n || !e_cand || !e_off || !e_ud || !e_cnt || !e_valid)
    return fail (ctx, "awm_sync_refine: out of page-locked memory");
  auto fetch_list = [&] () -> int
    {
      CK (cudaMemcpyAsync (e_n, ctx->ex_n.p, sizeof (int), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaMemcpyAsync (e_cand, ctx->ex_cand.p, np_max * sizeof (int), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaMemcpyAsync (e_off, ctx->ex_off.p, np_max * sizeof (int), cudaMemcpyDeviceToHost, ctx->stream));
      return 0;
    };
  auto fetch_sums = [&] () -> int
    {
      CK (cudaMemcpyAsync (e_ud, ctx->r_ud.p, np_max * n_bits * 2 * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaMemcpyAsync (e_cnt, ctx->r_cnt.p, np_max * n_bits * sizeof (int), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaMemcpyAsync (e_valid, ctx->rvalid.p, np_max, cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaStreamSynchronize (ctx->stream));
      return 0;
    };
  // Exact / Sliding: the quality of the sums at `p` goes to offset `at` ([candidate][65]); offsets not written stay invalid
  auto put_quality = [&] (size_t p, size_t at)
    {
      valid_out[at] = e_valid[p];
      q_out[at] = e_valid[p] ? quality_of (e_ud, e_cnt, p) : 0.0;
    };
  if (q_out)
    {
      std::fill (valid_out, valid_out + np_max, 0);
      std::fill (q_out, q_out + np_max, 0.0);
    }
  if (slide && want == RefineOut::Sliding)
    {
      if (fetch_sums()) return 1;
      for (size_t c = 0; c < nc; c++)
        for (int o = 0; o < h_noff[c]; o++)
          put_quality (c * kOffsets + o, c * kOffsets + o);
      return 0;
    }
  CK (ctx->ex_start.reserve (np_max * sizeof (long long)));
  CK (ctx->ex_cand.reserve (np_max * sizeof (int)));
  CK (ctx->ex_off.reserve (np_max * sizeof (int)));
  CK (ctx->ex_n.reserve (sizeof (int)));
  if (slide)
    {
      /* The sliding DFT only RANKS the 65 offsets: every offset whose sliding score S lies within kVerifyMargin of the best sliding
       * score is scored again with fresh FFTs in the reference's summation order (k_refine_exact_fft_n / _sum_n below), and the
       * reference's rule picks among those exact values E.  If |S - E| <= d for all offsets, the exact arg-max o* satisfies
       * S(o*) >= E(o*) - d >= E(o') - d >= S(o') - 2d for the sliding arg-max o', so with kVerifyMargin >= 2d the exact arg-max is
       * always re-scored and index / quality are those of the exact re-score of every offset.  d is measured by
       * tests/test_gpu_stages.py::test_sync_refine_vs_oracle (asserted < kVerifyMargin / 4 on all 65 offsets of every golden
       * candidate); neighbouring offsets of a real peak differ by ~3e-3, so usually one or two offsets are re-scored.  The offset of the approx index itself is always re-scored: in the
       * reference the search starts from the approx quality, which there IS the exact value of that offset (same transforms, same
       * order of additions); ours comes from the entry-sum formulation and differs by ~1e-5 relative, so the exact value takes its
       * place below.  k_refine_rank picks the offsets on the device (the same rule as tests/test_gpu_refine_rank.py applies on the
       * host), so the sliding sums never leave the GPU. */
      constexpr double kVerifyMargin = 1e-3;
      CK (ctx->cand_score.reserve (nc * sizeof (awm_search_score)));
      CK (ctx->rank_keep.reserve (nc * 3 * sizeof (unsigned)));
      CK (ctx->rank_first.reserve (nc * sizeof (int)));
      awm_search_score *h_sc = ctx->pin.get<awm_search_score> (nc);
      if (!h_sc)
        return fail (ctx, "awm_sync_refine: out of page-locked memory");
      std::copy (scores, scores + nc, h_sc);
      CK (cudaMemcpyAsync (ctx->cand_score.p, h_sc, nc * sizeof (awm_search_score), cudaMemcpyHostToDevice, ctx->stream));
      PROF (ctx);
      k_refine_rank<<<1, kRankWarps * 32, 0, ctx->stream>>> (ctx->r_ud.as<float>(), ctx->r_cnt.as<int>(), ctx->rvalid.as<unsigned char>(),
        ctx->cand_score.as<awm_search_score>(), ctx->cand_start.as<long long>(), ctx->cand_noff.as<int>(), int (nc), n_bits, norm_div, kVerifyMargin,
        ctx->rank_keep.as<unsigned>(), ctx->rank_first.as<int>(), ctx->ex_start.as<long long>(), ctx->ex_cand.as<int>(), ctx->ex_off.as<int>(), ctx->ex_n.as<int>());
      LAUNCH_CHECK ("k_refine_rank");
    }
  else
    {
      /* every offset that gets a result (sync_fft returns nothing for a window past the end), in candidate order, offsets ascending;
       * the exact kernels read the starts and the length */
      long long *e_start = ctx->pin.get<long long> (np_max);
      if (!e_start)
        return fail (ctx, "awm_sync_refine: out of page-locked memory");
      int n = 0;
      for (size_t c = 0; c < nc; c++)
        for (int o = 0; o < h_noff[c]; o++)
          if (h_start[c] + 8LL * o + (long long) total * kFrame <= (long long) ctx->pcm_frames)
            {
              e_start[n] = h_start[c] + 8LL * o;
              e_cand[n] = int (c);
              e_off[n] = o;
              n++;
            }
      *e_n = n;
      CK (cudaMemcpyAsync (ctx->ex_start.p, e_start, n * sizeof (long long), cudaMemcpyHostToDevice, ctx->stream));
      CK (cudaMemcpyAsync (ctx->ex_n.p, e_n, sizeof (int), cudaMemcpyHostToDevice, ctx->stream));
    }
  if (want == RefineOut::Rescored)
    {
      if (slide && fetch_list()) return 1;
      CK (cudaStreamSynchronize (ctx->stream));
      std::fill (rescored_out, rescored_out + np_max, 0);
      for (int p = 0; p < *e_n; p++)
        rescored_out[size_t (e_cand[p]) * kOffsets + e_off[p]] = 1;
      return 0;
    }
  if (!ctx->n_sms)
    CK (cudaDeviceGetAttribute (&ctx->n_sms, cudaDevAttrMultiProcessorCount, ctx->device));
  const size_t smem = fft_smem_bytes (kExactWarps) + kExactWarps * 96 * sizeof (float);
  if (set_smem (ctx, k_refine_exact_fft_n, smem)) return 1;
  const long long jobs_max = (long long) np_max * t.n_ent;
  PROF (ctx);
  k_refine_exact_fft_n<<<unsigned (std::min<long long> ((jobs_max + kExactWarps - 1) / kExactWarps, 4LL * ctx->n_sms)), kExactWarps * 32, smem, ctx->stream>>> (
    ctx->pcm, (long long) ctx->pcm_frames, ctx->pcm_ch, ctx->ex_start.as<long long>(), ctx->ex_n.as<int>(), t.ent.as<awm_sync_entry>(), t.n_ent,
    ctx->r_ent_ud.as<float>(), ctx->tw.as<float2>(), ctx->win.as<float>());
  LAUNCH_CHECK ("k_refine_exact_fft_n");
  /* the re-scored offsets of a candidate lie within 512 samples of each other: its sync frames are compulsory traffic once
   * (and were read by the sliding pass a moment ago: they come from L2) */
  prof_bytes (ctx, double (nc) * double (t.n_ent) * (double (kFrame) + 512.0) * ctx->pcm_ch * sizeof (float));
  int max_bit_frames = 1;
  for (int b = 0; b < n_bits; b++)
    max_bit_frames = std::max (max_bit_frames, t.h_off[b + 1] - t.h_off[b]);
  const size_t sum_smem = size_t (kExactSumWarps) * max_bit_frames * kUD * sizeof (float);
  if (set_smem (ctx, k_refine_exact_sum_n, sum_smem)) return 1;
  const long long sum_jobs_max = (long long) np_max * n_bits * 2;
  PROF (ctx);
  k_refine_exact_sum_n<<<unsigned (std::min<long long> ((sum_jobs_max + kExactSumWarps - 1) / kExactSumWarps, 16LL * ctx->n_sms)), kExactSumWarps * 32, sum_smem, ctx->stream>>> (
    ctx->r_ent_ud.as<float>(), ctx->ex_start.as<long long>(), ctx->ex_n.as<int>(), (long long) ctx->pcm_frames, ctx->pcm_ch, t.ent.as<awm_sync_entry>(), t.n_ent,
    t.off.as<int>(), n_bits, total, (long long) wav_first, (long long) wav_last, max_bit_frames, ctx->r_ud.as<float>(), ctx->r_cnt.as<int>(), ctx->rvalid.as<unsigned char>());
  LAUNCH_CHECK ("k_refine_exact_sum_n");
  if (slide && fetch_list()) return 1;          // one round trip: the list the device wrote and the exact sums
  if (fetch_sums()) return 1;
  const size_t np = size_t (*e_n);
  if (want != RefineOut::Refined)
    {
      for (size_t p = 0; p < np; p++)
        put_quality (p, size_t (e_cand[p]) * kOffsets + e_off[p]);
      return 0;
    }
  std::vector<double> best_quality (nc);
  std::vector<uint64_t> best_index (nc);
  for (size_t c = 0; c < nc; c++)
    {
      best_quality[c] = scores[c].raw_quality;
      best_index[c] = scores[c].index;
    }
  for (size_t p = 0; p < np; p++)               // starting value: the exact quality at the approx index
    if (e_valid[p] && uint64_t (h_start[e_cand[p]] + 8LL * e_off[p]) == scores[e_cand[p]].index)
      best_quality[e_cand[p]] = quality_of (e_ud, e_cnt, p);
  for (size_t p = 0; p < np; p++)               // per candidate in ascending offset order
    if (e_valid[p])
      {
        const size_t c = size_t (e_cand[p]);
        const double q = quality_of (e_ud, e_cnt, p);
        if (fabs (q - scores[c].local_mean) > fabs (best_quality[c] - scores[c].local_mean))   // src/syncfinder.cc:436-440
          {
            best_quality[c] = q;
            best_index[c] = uint64_t (h_start[c] + 8LL * e_off[p]);
          }
      }
  for (size_t c = 0; c < nc; c++)
    {
      refined[c] = scores[c];
      refined[c].index = best_index[c];
      refined[c].raw_quality = best_quality[c];
    }
  return 0;
}

int
awm_sync_refine (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last,
                 double water_delta, awm_search_score *scores, size_t n_scores)
{
  return refine_impl (ctx, key_slot, mode, wav_first, wav_last, water_delta, scores, n_scores, RefineOut::Refined, scores, nullptr, nullptr, nullptr);
}

int
awm_sync_refine_rescored (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta,
                          const awm_search_score *scores, size_t n_scores, unsigned char *rescored_out)
{
  if (!rescored_out)
    return fail (ctx, "awm_sync_refine_rescored: bad arguments");
  return refine_impl (ctx, key_slot, mode, wav_first, wav_last, water_delta, scores, n_scores, RefineOut::Rescored, nullptr, nullptr, nullptr,
                      rescored_out);
}

int
awm_sync_refine_offsets (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta,
                         const awm_search_score *scores, size_t n_scores, int exact, double *quality_out, unsigned char *valid_out)
{
  if (!quality_out || !valid_out)
    return fail (ctx, "awm_sync_refine_offsets: bad arguments");
  return refine_impl (ctx, key_slot, mode, wav_first, wav_last, water_delta, scores, n_scores, exact ? RefineOut::Exact : RefineOut::Sliding,
                      nullptr, quality_out, valid_out, nullptr);
}

/* ---------------------------------------------------------------- multi-GPU exchange
 * NCCL is loaded on first use (dlopen), so that single-GPU users of the library do not depend on it. */
namespace {

struct NcclUniqueId { char internal[128]; };
struct NcclApi
{
  void *lib = nullptr;
  int (*GetUniqueId) (NcclUniqueId *) = nullptr;
  int (*CommInitRank) (void **, int, NcclUniqueId, int) = nullptr;
  int (*AllGather) (const void *, void *, size_t, int, void *, cudaStream_t) = nullptr;
  int (*CommDestroy) (void *) = nullptr;
  const char *(*GetErrorString) (int) = nullptr;
  std::string error;
};

NcclApi&
nccl_api()
{
  static NcclApi api;
  if (api.lib || !api.error.empty())
    return api;
  for (const char *name : { "libnccl.so.2", "libnccl.so" })
    if ((api.lib = dlopen (name, RTLD_NOW | RTLD_GLOBAL)))
      break;
  if (!api.lib)
    {
      api.error = std::string ("cannot load libnccl.so.2: ") + dlerror();
      return api;
    }
  auto sym = [&] (const char *n) { void *p = dlsym (api.lib, n); if (!p) api.error = std::string ("libnccl: missing symbol ") + n; return p; };
  api.GetUniqueId = reinterpret_cast<decltype (api.GetUniqueId)> (sym ("ncclGetUniqueId"));
  api.CommInitRank = reinterpret_cast<decltype (api.CommInitRank)> (sym ("ncclCommInitRank"));
  api.AllGather = reinterpret_cast<decltype (api.AllGather)> (sym ("ncclAllGather"));
  api.CommDestroy = reinterpret_cast<decltype (api.CommDestroy)> (sym ("ncclCommDestroy"));
  api.GetErrorString = reinterpret_cast<decltype (api.GetErrorString)> (sym ("ncclGetErrorString"));
  return api;
}

} // namespace

} // extern "C"

void
nccl_destroy (void *comm)
{
  NcclApi& n = nccl_api();
  if (n.CommDestroy)
    n.CommDestroy (comm);
}

extern "C" {

int
awm_dist_unique_id (unsigned char id_out[128])
{
  NcclApi& n = nccl_api();
  if (!n.error.empty() || !id_out)
    return 1;
  NcclUniqueId id;
  if (n.GetUniqueId (&id))
    return 1;
  memcpy (id_out, id.internal, 128);
  return 0;
}

int
awm_dist_init (awm_ctx *ctx, int rank, int world, const unsigned char id[128])
{
  if (!ctx || !id || world < 1 || rank < 0 || rank >= world)
    return fail (ctx, "awm_dist_init: bad arguments");
  NcclApi& n = nccl_api();
  if (!n.error.empty())
    return fail (ctx, "awm_dist_init: %s", n.error.c_str());
  CK (cudaSetDevice (ctx->device));
  if (ctx->nccl_comm)
    {
      n.CommDestroy (ctx->nccl_comm);
      ctx->nccl_comm = nullptr;
    }
  NcclUniqueId uid;
  memcpy (uid.internal, id, 128);
  const int rc = n.CommInitRank (&ctx->nccl_comm, world, uid, rank);
  if (rc)
    return fail (ctx, "ncclCommInitRank: %s", n.GetErrorString (rc));
  ctx->dist_rank = rank;
  ctx->dist_world = world;
  return 0;
}

int
awm_dist_world (const awm_ctx *ctx, int *rank, int *world)
{
  if (!ctx)
    return 1;
  if (rank) *rank = ctx->dist_rank;
  if (world) *world = ctx->nccl_comm ? ctx->dist_world : 1;
  return 0;
}

int
awm_dist_allgather (awm_ctx *ctx, const void *send, size_t send_bytes, size_t slot_bytes, void *recv, size_t *recv_bytes)
{
  if (!ctx || (send_bytes && !send) || !recv || !recv_bytes || slot_bytes < 16 || slot_bytes % 16)
    return fail (ctx, "awm_dist_allgather: bad arguments");
  const int world = ctx->nccl_comm ? ctx->dist_world : 1;
  if (world == 1)
    {
      if (send_bytes + 8 > slot_bytes)
        return fail (ctx, "awm_dist_allgather: payload of %zu bytes does not fit a slot of %zu", send_bytes, slot_bytes);
      memcpy (recv, send, send_bytes);
      recv_bytes[0] = send_bytes;
      return 0;
    }
  NcclApi& n = nccl_api();
  CK (cudaSetDevice (ctx->device));
  CK (ctx->dist_send.reserve (slot_bytes));
  CK (ctx->dist_recv.reserve (slot_bytes * world));
  if (ctx->dist_hsend_cap < slot_bytes)
    {
      if (ctx->dist_hsend) cudaFreeHost (ctx->dist_hsend);
      if (ctx->dist_hhdr) cudaFreeHost (ctx->dist_hhdr);
      ctx->dist_hsend = ctx->dist_hhdr = nullptr;
      ctx->dist_hsend_cap = 0;
      CK (cudaMallocHost (reinterpret_cast<void **> (&ctx->dist_hsend), slot_bytes));
      CK (cudaMallocHost (reinterpret_cast<void **> (&ctx->dist_hhdr), 8 * 1024));
      ctx->dist_hsend_cap = slot_bytes;
    }
  /* slot = [u64 payload length | payload]; a payload that does not fit is announced by its length alone, every rank then sees
   * the same lengths and reports the same failure (the caller repeats the exchange with a larger slot) */
  const uint64_t len = send_bytes;
  const bool fits = send_bytes + 8 <= slot_bytes;
  memcpy (ctx->dist_hsend, &len, 8);
  if (fits && send_bytes)
    memcpy (ctx->dist_hsend + 8, send, send_bytes);
  CK (cudaMemcpyAsync (ctx->dist_send.p, ctx->dist_hsend, fits ? 8 + send_bytes : 8, cudaMemcpyHostToDevice, ctx->stream));
  const int rc = n.AllGather (ctx->dist_send.p, ctx->dist_recv.p, slot_bytes, 0 /* ncclChar */, ctx->nccl_comm, ctx->stream);
  if (rc)
    return fail (ctx, "ncclAllGather: %s", n.GetErrorString (rc));
  ctx->launches++;
  CK (cudaMemcpy2DAsync (ctx->dist_hhdr, 8, ctx->dist_recv.p, slot_bytes, 8, world, cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  bool all_fit = true;
  for (int r = 0; r < world; r++)
    {
      uint64_t l;
      memcpy (&l, ctx->dist_hhdr + 8 * r, 8);
      recv_bytes[r] = size_t (l);
      all_fit = all_fit && l + 8 <= slot_bytes;
    }
  if (!all_fit)
    return 2;                                   /* recv_bytes holds the lengths: repeat with slot_bytes >= max + 8 */
  for (int r = 0; r < world; r++)
    if (recv_bytes[r])
      CK (cudaMemcpyAsync (static_cast<unsigned char *> (recv) + size_t (r) * slot_bytes, ctx->dist_recv.as<unsigned char>() + size_t (r) * slot_bytes + 8,
                           recv_bytes[r], cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

/* ---------------------------------------------------------------- block decode */

int
awm_decode_blocks (awm_ctx *ctx, int key_slot, const uint64_t *indices, size_t n_blocks, float *raw_bits_out, int *valid_out)
{
  if (key_slot < 0 || key_slot >= AWM_MAX_KEYS || (n_blocks && (!indices || !raw_bits_out || !valid_out)))
    return fail (ctx, "awm_decode_blocks: bad arguments");
  KeyTab& k = ctx->keys[key_slot];
  if (!k.n_mix)
    return fail (ctx, "awm_decode_blocks: mix tables for key slot %d not set", key_slot);
  if (!ctx->pcm_ch)
    return fail (ctx, "awm_decode_blocks: no PCM bound");
  if (n_blocks == 0)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const int C = ctx->pcm_ch;
  std::vector<long long> starts;
  std::vector<size_t> which;
  for (size_t i = 0; i < n_blocks; i++)
    {
      // fft_range: empty result if samples.size() < (start_index + frame_count * frame_size) * n_channels
      const bool ok = indices[i] + uint64_t (k.fpb) * kFrame <= ctx->pcm_frames;
      valid_out[i] = ok ? 1 : 0;
      if (ok)
        {
          starts.push_back ((long long) indices[i]);
          which.push_back (i);
        }
    }
  const size_t per_blk = size_t (k.fpb) * C * kBands * sizeof (float);
  size_t batch = std::max<size_t> (1, (size_t (1) << 30) / per_blk);
  const size_t smem = fft_smem_bytes (kDecodeWarps);
  if (set_smem (ctx, k_decode_fft, smem)) return 1;
  ctx->pin.reset();
  for (size_t b0 = 0; b0 < starts.size(); b0 += batch)
    {
      const size_t nb = std::min (batch, starts.size() - b0);
      long long *h_starts = ctx->pin.get<long long> (nb);
      float *h_raw = ctx->pin.get<float> (nb * k.n_coded);
      if (!h_starts || !h_raw)
        return fail (ctx, "awm_decode_blocks: out of page-locked memory");
      std::copy (starts.begin() + b0, starts.begin() + b0 + nb, h_starts);
      CK (ctx->D.reserve (nb * per_blk));
      CK (ctx->blk_start.reserve (nb * sizeof (long long)));
      CK (ctx->raw.reserve (nb * k.n_coded * sizeof (float)));
      CK (cudaMemcpyAsync (ctx->blk_start.p, h_starts, nb * sizeof (long long), cudaMemcpyHostToDevice, ctx->stream));
      const int pairs = (C + 1) / 2;
      const long long jobs = (long long) nb * k.fpb * pairs;
      PROF (ctx);
      k_decode_fft<<<unsigned ((jobs + kDecodeWarps - 1) / kDecodeWarps), kDecodeWarps * 32, smem, ctx->stream>>> (
        ctx->pcm, (long long) ctx->pcm_frames, C, ctx->blk_start.as<long long>(), int (nb), k.fpb, ctx->D.as<float>(),
        ctx->tw.as<float2>(), ctx->win.as<float>());
      LAUNCH_CHECK ("k_decode_fft");
      prof_bytes (ctx, double (nb) * k.fpb * (double (kFrame) * C * sizeof (float) + double (C) * kBands * sizeof (float)));   /* block PCM in, band dB out */
      dim3 grid (unsigned ((k.n_coded + 127) / 128), unsigned (nb));
      PROF (ctx);
      k_mix_decode<<<grid, 128, 0, ctx->stream>>> (ctx->D.as<float>(), int (nb), C, k.fpb, k.mix.as<awm_mix_entry>(), k.frames_per_bit,
                                                   k.n_coded, k.order.as<uint16_t>(), ctx->raw.as<float>());
      LAUNCH_CHECK ("k_mix_decode");
      CK (cudaMemcpyAsync (h_raw, ctx->raw.p, nb * k.n_coded * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaStreamSynchronize (ctx->stream));
      for (size_t b = 0; b < nb; b++)
        memcpy (raw_bits_out + which[b0 + b] * k.n_coded, h_raw + b * k.n_coded, k.n_coded * sizeof (float));
    }
  return 0;
}

/* ---------------------------------------------------------------- Viterbi */

int
awm_viterbi (awm_ctx *ctx, const float *raw_bits, size_t n_jobs, int n_msg_bits, const int *block_types,
             int hard, uint8_t *bits_out, float *error_out)
{
  if (n_jobs == 0)
    return 0;
  if (!raw_bits || !block_types || !bits_out || !error_out || n_msg_bits <= 0 || n_msg_bits > 4096)
    return fail (ctx, "awm_viterbi: bad arguments");
  const int steps = n_msg_bits + AWM_VITERBI_ORDER;
  std::vector<long long> off (n_jobs + 1, 0);
  for (size_t j = 0; j < n_jobs; j++)
    {
      if (block_types[j] < 0 || block_types[j] > 2)
        return fail (ctx, "awm_viterbi: bad block type %d", block_types[j]);
      off[j + 1] = off[j] + (long long) steps * (block_types[j] == AWM_BLOCK_AB ? 12 : 6);
    }
  CK (cudaSetDevice (ctx->device));
  const size_t max_jobs = 512;
  const size_t smem = viterbi_smem_bytes (steps);
  if (smem > 220 * 1024)
    return fail (ctx, "awm_viterbi: %d message bits are more than the kernel holds in shared memory", n_msg_bits);
  if (set_smem (ctx, k_viterbi, smem)) return 1;
  for (size_t j0 = 0; j0 < n_jobs; j0 += max_jobs)
    {
      const size_t nj = std::min (max_jobs, n_jobs - j0);
      const long long base = off[j0], n_raw = off[j0 + nj] - base;
      std::vector<long long> rel (nj);
      for (size_t j = 0; j < nj; j++)
        rel[j] = off[j0 + j] - base;
      CK (ctx->vit_raw.reserve (n_raw * sizeof (float)));
      CK (ctx->vit_off.reserve (nj * sizeof (long long)));
      CK (ctx->vit_types.reserve (nj * sizeof (int)));
      CK (ctx->vit_dec.reserve (nj * steps * kVitWords * sizeof (uint32_t)));
      CK (ctx->vit_bits.reserve (nj * n_msg_bits));
      CK (ctx->vit_err.reserve (nj * sizeof (float)));
      /* host inputs / outputs pass through page-locked staging: the three uploads, the launch and the two downloads queue up
       * without the host waiting in between */
      ctx->pin.reset();
      const bool raw_on_device = is_device_ptr (raw_bits);
      float *h_in = raw_on_device ? nullptr : ctx->pin.get<float> (size_t (n_raw));
      long long *h_rel = ctx->pin.get<long long> (nj);
      int *h_types = ctx->pin.get<int> (nj);
      unsigned char *h_bits = ctx->pin.get<unsigned char> (nj * n_msg_bits);
      float *h_err = ctx->pin.get<float> (nj);
      if ((!raw_on_device && !h_in) || !h_rel || !h_types || !h_bits || !h_err)
        return fail (ctx, "awm_viterbi: out of page-locked memory");
      if (h_in)
        memcpy (h_in, raw_bits + base, size_t (n_raw) * sizeof (float));
      std::copy (rel.begin(), rel.end(), h_rel);
      std::copy (block_types + j0, block_types + j0 + nj, h_types);
      CK (cudaMemcpyAsync (ctx->vit_raw.p, h_in ? h_in : raw_bits + base, n_raw * sizeof (float), cudaMemcpyDefault, ctx->stream));
      CK (cudaMemcpyAsync (ctx->vit_off.p, h_rel, nj * sizeof (long long), cudaMemcpyHostToDevice, ctx->stream));
      CK (cudaMemcpyAsync (ctx->vit_types.p, h_types, nj * sizeof (int), cudaMemcpyHostToDevice, ctx->stream));
      PROF (ctx);
      k_viterbi<<<unsigned (nj), kVitThreads, smem, ctx->stream>>> (ctx->vit_raw.as<float>(), ctx->vit_off.as<long long>(), n_msg_bits, ctx->vit_types.as<int>(), hard,
                                                                  steps, ctx->vit_dec.as<uint32_t>(),
                                                                  ctx->vit_bits.as<unsigned char>(), ctx->vit_err.as<float>());
      LAUNCH_CHECK ("k_viterbi");
      CK (cudaMemcpyAsync (h_bits, ctx->vit_bits.p, nj * n_msg_bits, cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaMemcpyAsync (h_err, ctx->vit_err.p, nj * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaStreamSynchronize (ctx->stream));
      memcpy (bits_out + j0 * n_msg_bits, h_bits, nj * n_msg_bits);
      memcpy (error_out + j0, h_err, nj * sizeof (float));
    }
  return 0;
}

} // extern "C"

/* ---------------------------------------------------------------- resampler */

namespace {

double
rs_sinc (double x)
{
  x = fabs (x);
  if (x < 1e-9)
    return 1;
  x *= M_PI;
  return sin (x) / x;
}

double
rs_window (double x)        /* three-term cosine window on [-1, 1] */
{
  x = fabs (x);
  if (x >= 1)
    return 0;
  x *= M_PI;
  return 0.384 + 0.5 * cos (x) + 0.116 * cos (2 * x);
}

/* filter table for one conversion ratio: g(d) = fc sinc (fc d) w (d / h), fc = min (1, ratio), h = ceil (hlen / fc) input
 * frames to each side; row p holds the 2h taps for a fractional position of p / 256.  Built on the host in double (a
 * few ms, cached per ratio) so that every implementation that evaluates the same formula has the same float table. */
constexpr size_t kCoefCacheCap = 1024;

/* room for n_new filter tables: the cache is emptied when it would grow past kCoefCacheCap (data dependent ratios accumulate in
 * long running hosts) */
int
coef_cache_room (awm_ctx *ctx, size_t n_new)
{
  if (ctx->coef_cache.size() + n_new <= kCoefCacheCap)
    return 0;
  CK (cudaStreamSynchronize (ctx->stream));
  for (auto& ct : ctx->coef_cache)
    ct.second.buf.release();
  ctx->coef_cache.clear();
  return 0;
}

bool
resample_ratio_ok (double ratio)
{
  return ratio > 1.0 / 64 && ratio < 64;
}

int
coef_table (awm_ctx *ctx, double ratio, int hlen, const float **coef, int *h_out)
{
  if (!resample_ratio_ok (ratio) || hlen < 8 || hlen > 96)
    return fail (ctx, "resampler: ratio %g / hlen %d not supported", ratio, hlen);
  auto key = std::make_pair (ratio, hlen);
  auto it = ctx->coef_cache.find (key);
  if (it == ctx->coef_cache.end())
    {
      if (coef_cache_room (ctx, 1))
        return 1;
      const double fc = ratio < 1 ? ratio : 1;
      const int h = int (ceil (hlen / fc));
      const int taps = 2 * h, rows = kResamplePhases + 1;
      std::vector<float> tab (size_t (rows) * taps);
      auto fill = [&] (int p0, int p1)
        {
          for (int p = p0; p < p1; p++)
            for (int j = 0; j < taps; j++)
              {
                const double d = (j - (h - 1)) - double (p) / kResamplePhases;
                tab[size_t (j) * rows + p] = float (fc * rs_sinc (fc * d) * rs_window (d / h));     /* tap major, see ResampleJob */
              }
        };
      const int n_thr = 8;
      std::vector<std::thread> thr;
      for (int t = 0; t < n_thr; t++)
        thr.emplace_back (fill, rows * t / n_thr, rows * (t + 1) / n_thr);
      for (auto& t : thr)
        t.join();
      awm_ctx::CoefTab& ct = ctx->coef_cache[key];
      ct.h = h;
      CK (ct.buf.reserve (tab.size() * sizeof (float)));
      CK (cudaMemcpy (ct.buf.p, tab.data(), tab.size() * sizeof (float), cudaMemcpyHostToDevice));
      it = ctx->coef_cache.find (key);
    }
  *coef = it->second.buf.as<float>();
  *h_out = it->second.h;
  return 0;
}

/* frames at the watermark rate a resampled item of awm_embed_batch_rates needs: up to the highest tap of output n_emit - 1 (> 0), in
 * whole 1024-frames */
long long
resampled_n44 (uint64_t n_emit, double step_out, int h_out)
{
  const long long top = (long long) floor (double (n_emit - 1) * step_out) + h_out;
  return (top / kFrame + 1) * kFrame;
}

int
launch_resample (awm_ctx *ctx, const std::vector<ResampleJob>& jobs, int channels)
{
  if (jobs.empty())
    return 0;
  long long max_out = 0;
  for (const auto& j : jobs)
    max_out = std::max (max_out, j.n_out);
  if (max_out == 0)
    return 0;
  CK (ctx->rs_jobs.reserve (jobs.size() * sizeof (ResampleJob)));
  CK (cudaMemcpyAsync (ctx->rs_jobs.p, jobs.data(), jobs.size() * sizeof (ResampleJob), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));             /* jobs is a caller-owned host vector */
  const dim3 grid (unsigned (std::min<long long> ((max_out + 255) / 256, 1 << 20)), unsigned (jobs.size()));
  /* float2 loads and stores only where every job's input and output are 8-byte aligned (a device clip may start at any float);
   * k_resample<0> produces the same bits, resample_dot and resample_dot2 share the arithmetic */
  bool aligned8 = true;
  for (const auto& j : jobs)
    aligned8 = aligned8 && uintptr_t (j.in) % 8 == 0 && uintptr_t (j.out) % 8 == 0;
  PROF (ctx);
  if (channels == 2 && aligned8)
    k_resample<2><<<grid, 256, 0, ctx->stream>>> (ctx->rs_jobs.as<ResampleJob>(), channels);
  else if (channels == 1)
    k_resample<1><<<grid, 256, 0, ctx->stream>>> (ctx->rs_jobs.as<ResampleJob>(), channels);
  else
    k_resample<0><<<grid, 256, 0, ctx->stream>>> (ctx->rs_jobs.as<ResampleJob>(), channels);
  LAUNCH_CHECK ("k_resample");
  return 0;
}

} // namespace

int
awm_resample (awm_ctx *ctx, const float *in, size_t n_in, int channels, double ratio, int hlen, float *out, size_t n_out)
{
  if (channels <= 0 || (n_in && !in) || (n_out && !out))
    return fail (ctx, "awm_resample: bad arguments");
  if (n_out == 0)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const float *coef;
  int h;
  if (coef_table (ctx, ratio, hlen, &coef, &h))
    return 1;
  const bool in_dev = n_in == 0 || is_device_ptr (in), out_dev = is_device_ptr (out);
  ResampleJob J;
  J.in = in;
  J.out = out;
  if (!in_dev)
    {
      CK (ctx->rs_in.reserve (n_in * channels * sizeof (float)));
      CK (cudaMemcpyAsync (ctx->rs_in.p, in, n_in * channels * sizeof (float), cudaMemcpyHostToDevice, ctx->stream));
      J.in = ctx->rs_in.as<float>();
    }
  if (!out_dev)
    {
      CK (ctx->rs_out.reserve (n_out * channels * sizeof (float)));
      J.out = ctx->rs_out.as<float>();
    }
  J.n_in = (long long) n_in;
  J.n_stop = J.n_in;
  J.n_out = (long long) n_out;
  J.step = 1.0 / ratio;
  J.h = h;
  J.coef = coef;
  if (launch_resample (ctx, { J }, channels))
    return 1;
  if (!out_dev)
    {
      CK (cudaMemcpyAsync (out, J.out, n_out * channels * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
      CK (cudaStreamSynchronize (ctx->stream));
    }
  return 0;
}

uint64_t
awm_resample_stream_available (uint64_t fed, double ratio, int hlen)
{
  const double fc = ratio < 1 ? ratio : 1;
  const int h = int (ceil (hlen / fc));
  const double step = 1.0 / ratio;
  if ((long long) fed - 2 < h - 1)
    return 0;
  const double limit = double (fed) - 2;            /* centre tap (in pre-roll coordinates) of the last output that fits */
  long long n = (long long) ((double (fed) - 1 - h) * ratio) - 2;
  if (n < 0)
    n = 0;
  while (n > 0 && floor ((h - 1) + double (n - 1) * step) > limit)
    n--;
  while (floor ((h - 1) + double (n) * step) <= limit)
    n++;
  return uint64_t (n);
}

uint64_t
awm_resample_stream_frames (uint64_t n_in, double ratio, int hlen)
{
  const double fc = ratio < 1 ? ratio : 1;
  return awm_resample_stream_available (n_in + uint64_t (ceil (hlen / fc)), ratio, hlen);
}

void
awm_resample_taps (uint64_t n_in_total, double ratio, int hlen, uint64_t out_first, uint64_t out_frames, uint64_t *first, uint64_t *end)
{
  *first = *end = 0;
  if (!out_frames)
    return;
  const double fc = ratio < 1 ? ratio : 1;
  const long long h = (long long) ceil (hlen / fc);
  const double step = 1.0 / ratio;
  /* c (n) of resample_pos, rounded the same way: a product and a sum, not fused */
  auto centre = [&] (uint64_t n) { volatile double p = double (n) * step; return (long long) floor (double (h - 1) + p); };
  const long long lo = centre (out_first) - 2 * h + 2, hi = centre (out_first + out_frames - 1) + 2;
  *first = uint64_t (std::min<long long> (std::max (lo, 0LL), (long long) n_in_total));
  *end = uint64_t (std::min<long long> (std::max (hi, (long long) *first), (long long) n_in_total));
}

int
awm_resample_range_validate (uint64_t in_first, uint64_t in_frames, uint64_t n_in_total, int channels, double ratio, int hlen,
                             uint64_t out_first, uint64_t out_frames, char *err, size_t err_cap)
{
  char why[240] = "";
  uint64_t t0 = 0, t1 = 0;
  if (channels <= 0)
    snprintf (why, sizeof (why), "channels %d must be > 0", channels);
  else if (!resample_ratio_ok (ratio) || hlen < 8 || hlen > 96)
    snprintf (why, sizeof (why), "ratio %g / hlen %d not supported (ratio in (1/64, 64), hlen in [8, 96])", ratio, hlen);
  else if (n_in_total > AWM_MAX_STREAM_FRAMES || out_first > AWM_MAX_STREAM_FRAMES || out_frames > AWM_MAX_STREAM_FRAMES
           || in_first > AWM_MAX_STREAM_FRAMES || in_frames > AWM_MAX_STREAM_FRAMES)
    snprintf (why, sizeof (why), "frame counts and positions must be at most 2^48");
  else if (out_first + out_frames > awm_resample_stream_frames (n_in_total, ratio, hlen))
    snprintf (why, sizeof (why), "outputs [%llu, %llu) end past the %llu frames of the resampled stream", (unsigned long long) out_first,
              (unsigned long long) (out_first + out_frames), (unsigned long long) awm_resample_stream_frames (n_in_total, ratio, hlen));
  else
    {
      awm_resample_taps (n_in_total, ratio, hlen, out_first, out_frames, &t0, &t1);
      if (t0 < t1 && (t0 < in_first || t1 > in_first + in_frames))
        snprintf (why, sizeof (why), "outputs [%llu, %llu) read input frames [%llu, %llu), the window holds [%llu, %llu)", (unsigned long long) out_first,
                  (unsigned long long) (out_first + out_frames), (unsigned long long) t0, (unsigned long long) t1, (unsigned long long) in_first,
                  (unsigned long long) (in_first + in_frames));
    }
  if (err && err_cap)
    snprintf (err, err_cap, "%s", why);
  return why[0] ? 1 : 0;
}

int
awm_resample_range (awm_ctx *ctx, const float *in, uint64_t in_first, uint64_t in_frames, uint64_t n_in_total, int channels, double ratio, int hlen,
                    float *out, uint64_t out_first, uint64_t out_frames)
{
  char why[240];
  if (awm_resample_range_validate (in_first, in_frames, n_in_total, channels, ratio, hlen, out_first, out_frames, why, sizeof (why)))
    return fail (ctx, "awm_resample_range: %s", why);
  if ((in_frames && !in) || (out_frames && !out))
    return fail (ctx, "awm_resample_range: bad arguments");
  if (!out_frames)
    return 0;
  CK (cudaSetDevice (ctx->device));
  if (!is_device_ptr (out))
    return fail (ctx, "awm_resample_range: out must be device memory");
  const float *coef;
  int h;
  if (coef_table (ctx, ratio, hlen, &coef, &h))
    return 1;
  ResampleJob J;
  J.in = in;
  J.out = out;
  if (in_frames && !is_device_ptr (in))
    {
      CK (ctx->rs_in.reserve (in_frames * channels * sizeof (float)));
      CK (cudaMemcpyAsync (ctx->rs_in.p, in, in_frames * channels * sizeof (float), cudaMemcpyHostToDevice, ctx->stream));
      J.in = ctx->rs_in.as<float>();
    }
  J.n0 = (long long) out_first;
  J.in0 = (long long) in_first;
  J.n_in = (long long) n_in_total - J.in0;               /* the window-relative tap test i < n_in is the stream's i < n_in_total */
  J.n_stop = (long long) n_in_total;
  J.n_out = (long long) out_frames;
  J.step = 1.0 / ratio;
  J.h = h;
  J.coef = coef;
  return launch_resample (ctx, { J }, channels);
}

int
awm_device_alloc (awm_ctx *ctx, size_t bytes, void **out)
{
  if (!ctx || !out)
    return fail (ctx, "awm_device_alloc: bad arguments");
  *out = nullptr;
  if (!bytes)
    return 0;
  CK (cudaSetDevice (ctx->device));
  CK (cudaMalloc (out, bytes));
  return 0;
}

int
awm_device_free (awm_ctx *ctx, void *p)
{
  if (!ctx)
    return 1;
  if (!p)
    return 0;
  CK (cudaSetDevice (ctx->device));
  CK (cudaStreamSynchronize (ctx->stream));              /* kernels queued on the context stream may still read it */
  CK (cudaFree (p));
  return 0;
}

int
awm_pcm_push_resampled (awm_ctx *ctx, double ratio, int hlen, size_t n_out)
{
  if (!ctx->pcm_ch)
    return fail (ctx, "awm_pcm_push_resampled: no PCM bound");
  if (ctx->pushed)
    return fail (ctx, "awm_pcm_push_resampled: a resampled binding is already active");
  CK (cudaSetDevice (ctx->device));
  const float *coef;
  int h;
  if (coef_table (ctx, ratio, hlen, &coef, &h))
    return 1;
  CK (ctx->pcm_rs.reserve (std::max<size_t> (n_out, 1) * ctx->pcm_ch * sizeof (float)));
  ResampleJob J;
  J.in = ctx->pcm;
  J.out = ctx->pcm_rs.as<float>();
  J.n_in = (long long) ctx->pcm_frames;
  J.n_stop = J.n_in;
  J.n_out = (long long) n_out;
  J.step = 1.0 / ratio;
  J.h = h;
  J.coef = coef;
  if (launch_resample (ctx, { J }, ctx->pcm_ch))
    return 1;
  ctx->saved_pcm = ctx->pcm;
  ctx->saved_frames = ctx->pcm_frames;
  ctx->saved_ch = ctx->pcm_ch;
  ctx->pushed = true;
  ctx->pcm = J.out;
  ctx->pcm_frames = n_out;
  return 0;
}

int
awm_pcm_pop (awm_ctx *ctx)
{
  if (!ctx->pushed)
    return fail (ctx, "awm_pcm_pop: nothing to restore");
  ctx->pcm = ctx->saved_pcm;
  ctx->pcm_frames = ctx->saved_frames;
  ctx->pcm_ch = ctx->saved_ch;
  ctx->pushed = false;
  return 0;
}

int
awm_gather (awm_ctx *ctx, const float *src, const uint64_t *indices, size_t n, float *dst_host)
{
  if (!src || !indices || !dst_host)
    return fail (ctx, "awm_gather: bad arguments");
  if (!n)
    return 0;
  CK (cudaSetDevice (ctx->device));
  CK (ctx->rs_jobs.reserve (n * sizeof (uint64_t)));
  CK (ctx->rs_out.reserve (n * sizeof (float)));
  CK (cudaMemcpyAsync (ctx->rs_jobs.p, indices, n * sizeof (uint64_t), cudaMemcpyHostToDevice, ctx->stream));
  PROF (ctx);
  k_gather<<<unsigned ((n + 255) / 256), 256, 0, ctx->stream>>> (src, ctx->rs_jobs.as<unsigned long long>(), (long long) n, ctx->rs_out.as<float>());
  LAUNCH_CHECK ("k_gather");
  CK (cudaMemcpyAsync (dst_host, ctx->rs_out.p, n * sizeof (float), cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

int
awm_is_device_pointer (const void *p)
{
  return p && is_device_ptr (p) ? 1 : 0;
}

int
awm_copy_to_host (awm_ctx *ctx, void *dst, const void *src, size_t bytes)
{
  CK (cudaSetDevice (ctx->device));
  CK (cudaMemcpyAsync (dst, src, bytes, cudaMemcpyDefault, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

int
awm_copy (awm_ctx *ctx, void *dst, const void *src, size_t bytes)
{
  if (!ctx || (bytes && (!dst || !src)))
    return fail (ctx, "awm_copy: bad arguments");
  if (!bytes)
    return 0;
  CK (cudaSetDevice (ctx->device));
  CK (cudaMemcpyAsync (dst, src, bytes, cudaMemcpyDefault, ctx->stream));
  if (!is_device_ptr (src))
    CK (cudaStreamSynchronize (ctx->stream));       /* a pinned host source is read asynchronously: the caller may reuse it next */
  return 0;
}

/* ---------------------------------------------------------------- batched embed */

namespace {

constexpr size_t kBatchMaxRates = 256;                          // different resampled rates per call: two filter tables each
constexpr size_t kBatchDefaultScratch = size_t (4) << 30;       // per-wave scratch when the caller passes 0

} // namespace

int
awm_batch_rates_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const int *sample_rates, const uint64_t *n_emit,
                          int mark_sample_rate, char *err, size_t err_cap)
{
  if (awm_batch_validate (items, n_items, n_values, err, err_cap))
    return 1;
  char why[200] = "";
  std::vector<int> rates;
  if (mark_sample_rate <= 0)
    snprintf (why, sizeof (why), "mark sample rate %d must be > 0", mark_sample_rate);
  else if (n_items && !sample_rates)
    snprintf (why, sizeof (why), "sample rate list is NULL");
  for (size_t i = 0; i < n_items && !why[0]; i++)
    {
      const int r = sample_rates[i];
      if (r <= 0)
        snprintf (why, sizeof (why), "batch item %zu: sample rate %d must be > 0", i, r);
      else if (r == mark_sample_rate)
        continue;
      else if (!resample_ratio_ok (double (mark_sample_rate) / r) || !resample_ratio_ok (double (r) / mark_sample_rate))
        snprintf (why, sizeof (why), "batch item %zu: sample rate %d is outside the resampler's range (%d Hz / 64 .. %d Hz * 64, exclusive)",
                  i, r, mark_sample_rate, mark_sample_rate);
      else if (n_emit && n_emit[i] < items[i].n_frames)
        snprintf (why, sizeof (why), "batch item %zu: n_emit %llu is less than n_frames %llu", i, (unsigned long long) n_emit[i],
                  (unsigned long long) items[i].n_frames);
      else
        rates.push_back (r);
    }
  std::sort (rates.begin(), rates.end());
  rates.erase (std::unique (rates.begin(), rates.end()), rates.end());
  if (!why[0] && rates.size() > kBatchMaxRates)
    snprintf (why, sizeof (why), "%zu different sample rates (at most %zu per call)", rates.size(), kBatchMaxRates);
  if (err && err_cap)
    snprintf (err, err_cap, "%s", why);
  return why[0] ? 1 : 0;
}

int
awm_batch_rates_offsets_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const int *sample_rates, const uint64_t *n_emit,
                                  const uint64_t *zero_frames, int mark_sample_rate, char *err, size_t err_cap)
{
  if (awm_batch_rates_validate (items, n_items, n_values, sample_rates, n_emit, mark_sample_rate, err, err_cap) ||
      batch_offsets_check (items, n_items, n_values, zero_frames, true, err, err_cap))
    return 1;
  /* the stream at the watermark rate, (z + n) * mark / rate frames, must fit the limit too (at 8 kHz it is 5.5 times longer) */
  for (size_t i = 0; i < n_items; i++)
    {
      const unsigned __int128 end = (unsigned __int128) (zero_frames[i] + items[i].n_frames);
      if (end * unsigned (mark_sample_rate) > (unsigned __int128) AWM_MAX_STREAM_FRAMES * unsigned (sample_rates[i]))
        {
          if (err && err_cap)
            snprintf (err, err_cap, "batch item %zu: zero_frames %llu + n_frames %llu at %d Hz exceeds the stream length limit of 2^48 frames at %d Hz",
                      i, (unsigned long long) zero_frames[i], (unsigned long long) items[i].n_frames, sample_rates[i], mark_sample_rate);
          return 1;
        }
    }
  if (err && err_cap)
    err[0] = 0;
  return 0;
}

int
awm_batch_keys_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const int *sample_rates, const uint64_t *n_emit,
                         const uint64_t *zero_frames, const uint32_t *key_index, size_t n_keys, int mark_sample_rate, char *err, size_t err_cap)
{
  if (sample_rates ? (zero_frames ? awm_batch_rates_offsets_validate (items, n_items, n_values, sample_rates, n_emit, zero_frames, mark_sample_rate, err, err_cap)
                                  : awm_batch_rates_validate (items, n_items, n_values, sample_rates, n_emit, mark_sample_rate, err, err_cap))
                   : batch_offsets_check (items, n_items, n_values, zero_frames, false, err, err_cap))
    return 1;
  char why[160] = "";
  if (n_items && !key_index)
    snprintf (why, sizeof (why), "key index list is NULL");
  else if (n_items && !n_keys)
    snprintf (why, sizeof (why), "the role set has no keys");
  for (size_t i = 0; i < n_items && !why[0]; i++)
    if (key_index[i] >= n_keys)
      snprintf (why, sizeof (why), "batch item %zu: key index %u is out of range (%zu keys)", i, key_index[i], n_keys);
  if (err && err_cap)
    snprintf (err, err_cap, "%s", why);
  return why[0] ? 1 : 0;
}

namespace {

/* awm_embed_batch, awm_embed_batch_offsets, awm_embed_batch_rates, awm_embed_batch_rates_offsets and awm_embed_batch_keys after their
 * own argument checks (name: the error prefix).  sample_rates NULL: every item is at mark_sample_rate; zero_frames NULL: every item
 * starts a stream; key_index NULL: every item uses the role table of awm_set_embed_roles, else item i that of key key_index[i] of
 * the role set of awm_set_embed_roles_keys.  Items at mark_sample_rate use limiter_block44, the others rate * limiter_ms / 1000;
 * n_emit[i] counts from the item's first frame.  The --snr sums of a resampled item at a stream offset count its positions
 * [snr_first, snr_last) (from its first frame) inside [0, n_emit[i]): all of them by default, a window's owned part for
 * awm_embed_window_rates. */
int
embed_batch (const char *name, awm_ctx *ctx, const void *in_v, void *out_v, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
             const uint8_t *coded_bits, const uint64_t *zero_frames, const int *sample_rates, const uint64_t *n_emit, int mark_sample_rate,
             int frames_pad_start, double water_delta, int limiter_block44, int limiter_ms, float limiter_ceiling, double *snr_power,
             size_t scratch_bytes, const uint32_t *key_index = nullptr, uint64_t snr_first = 0, uint64_t snr_last = UINT64_MAX)
{
  RoleSet rs { ctx->roles.as<uint16_t>(), ctx->roles_fpb, ctx->roles_n_coded, false };
  if (key_index)
    {
      if (!ctx->key_roles_n)
        return fail (ctx, "%s: awm_set_embed_roles_keys has not been called", name);
      rs = { ctx->key_roles.as<uint16_t>(), ctx->key_roles_fpb, ctx->key_roles_n_coded, true };
    }
  else if (!ctx->roles_fpb)
    return fail (ctx, "%s: awm_set_embed_roles has not been called", name);
  auto role_table = [&] (size_t i) { return key_index ? int (key_index[i]) : 0; };
  if ((n_items && (!coded_bits || (sample_rates && !n_emit))) || (n_values && (!in_v || !out_v)) || limiter_ms < 0)
    return fail (ctx, "%s: bad arguments", name);
  /* the limiter block reaches k_embed_batch only through the items at mark_sample_rate; the others' blocks go to k_limiter_rates */
  bool any44 = !sample_rates;
  for (size_t i = 0; i < n_items && !any44; i++)
    any44 = sample_rates[i] == mark_sample_rate;
  if (embed_args_check (ctx, name, frames_pad_start, rs.fpb, any44 ? limiter_block44 : 0))
    return 1;
  if (snr_power)
    std::fill (snr_power, snr_power + 2 * n_items, 0.0);
  if (n_values == 0)
    return 0;
  CK (cudaSetDevice (ctx->device));
  const bool s16 = is_s16 != 0;
  const float *d_in;
  float *d_out;
  if (batch_images (ctx, in_v, out_v, s16, n_values, &d_in, &d_out))
    return 1;
  auto resampled = [&] (size_t i) { return sample_rates && sample_rates[i] != mark_sample_rate; };
  auto block_of = [&] (int rate) { return int ((long long) rate * limiter_ms / 1000); };      // add_watermark_buffer's limiter block

  /* filter tables of every resampled rate, all fetched before any is used: coef_table empties its cache when it is full */
  struct Filters { const float *coef_in = nullptr, *coef_out = nullptr; int h_in = 0, h_out = 0; };
  std::map<int, Filters> filters;
  for (size_t i = 0; i < n_items; i++)
    if (items[i].n_frames && resampled (i))
      filters[sample_rates[i]];
  if (coef_cache_room (ctx, 2 * filters.size()))
    return 1;
  for (auto& f : filters)
    if (coef_table (ctx, double (mark_sample_rate) / f.first, 16, &f.second.coef_in, &f.second.h_in) ||
        coef_table (ctx, double (f.first) / mark_sample_rate, 16, &f.second.coef_out, &f.second.h_out))
      return 1;

  /* work lists.  Items at the watermark rate: one k_embed_batch pass, with their stream offsets.  The others: consecutive waves whose
   * scratch (input and watermark signal at the watermark rate, 2 x n44 x C floats per item) stays within scratch_bytes; an item
   * larger than that runs alone.  A wave's scratch holds the inputs of all its items, then their watermark signals. */
  struct Wave { size_t b0 = 0, r0 = 0, r1 = 0, values = 0; long long n_tiles = 0, n_rs = 0, n_mix = 0, n_lim = 0; };
  std::vector<BatchItem> blist;
  std::vector<RateItem> rlist;
  std::vector<size_t> soff;                 // offset of rlist[k] in its wave's input half of the scratch
  std::vector<Wave> waves;
  long long n_tiles44 = 0, n_lim44 = 0, n_peaks = 0, unused = 0;
  uint64_t covered = 0;
  for (size_t i = 0; i < n_items; i++)
    {
      covered += items[i].n_frames * uint64_t (items[i].channels);
      if (items[i].n_frames && !resampled (i))
        blist.push_back (batch_entry ((long long) items[i].value_offset, (long long) items[i].n_frames, items[i].channels, int (i), limiter_block44,
                                      n_tiles44, n_lim44, n_peaks, zero_frames ? (long long) zero_frames[i] : 0, role_table (i)));
    }
  const size_t n_list44 = blist.size();
  const size_t cap = scratch_bytes ? scratch_bytes : kBatchDefaultScratch;
  size_t max_values = 0;
  for (size_t i = 0; i < n_items; i++)
    {
      const awm_batch_item& bi = items[i];
      if (!bi.n_frames || !resampled (i))
        continue;
      const int rate = sample_rates[i];
      const Filters& f = filters[rate];
      RateItem R = {};
      R.in = d_in + bi.value_offset;
      R.out = d_out + bi.value_offset;
      R.n_frames = (long long) bi.n_frames;
      R.n_emit = (long long) n_emit[i];
      R.C = bi.channels;
      R.item = int (i);
      R.step_in = 1.0 / (double (mark_sample_rate) / rate);      // 1 / r_in, 1 / r_out: the ratios of the add loop's two resamplers
      R.step_out = 1.0 / (double (rate) / mark_sample_rate);
      R.h_in = f.h_in;
      R.h_out = f.h_out;
      R.coef_in = f.coef_in;
      R.coef_out = f.coef_out;
      R.limiter_block = block_of (rate);
      {
        const long long z = zero_frames ? (long long) zero_frames[i] : 0;
        R.snr0 = z + (long long) std::min<uint64_t> (snr_first, n_emit[i]);
        R.snr1 = z + (long long) std::min<uint64_t> (snr_last, n_emit[i]);
      }
      if (zero_frames && zero_frames[i])
        {
          /* the stream of this item ends at z + n_emit, its x44 at n44 of that.  Everything before the first input frame the
           * in-resampler's taps reach is silent: x44 is exactly +0 up to about (z - h_in) / step_in, the watermark up to one
           * 1024-frame before that (the synthesis spill), so the scratch may start at w_hi or earlier.  It starts `span` frames
           * before the end, a length that holds [w_hi, n44) for every z (bounds taken 16 frames early, rounding included): the
           * scratch of an item does not depend on its offset.  The mixer starts where the out-resampler's taps reach w0. */
          const long long z = (long long) zero_frames[i], end = z + R.n_emit;
          const long long x_lo = std::max (0LL, (long long) floor (double (z - R.h_in - 16) / R.step_in));
          const long long w_hi = std::max (x_lo / kFrame - 1, 0LL) * kFrame;
          const long long n44 = resampled_n44 (uint64_t (end), R.step_out, R.h_out);
          const long long span = ((long long) ceil ((double (R.n_emit + R.h_in + 32) * R.step_out + R.h_out) / kFrame) + 4) * kFrame;
          R.z = z;
          R.w0 = std::max (0LL, std::min (w_hi, n44 - span));
          R.i0 = std::min (z, std::max (0LL, (long long) floor (double (R.w0 - R.h_out - 16) / R.step_out)));
          R.blk0 = R.limiter_block > 0 ? R.i0 / R.limiter_block : 0;
          R.n44 = n44 - R.w0;
          R.n_emit = end - R.i0;
          R.n_blocks = R.limiter_block > 0 ? (end - 1) / R.limiter_block - R.blk0 + 2 : 0;   // every block the mixer reaches
        }
      else
        {
          R.n44 = resampled_n44 (n_emit[i], R.step_out, R.h_out);
          R.n_blocks = R.limiter_block > 0 ? (R.n_emit + R.limiter_block - 1) / R.limiter_block + 1 : 0;   // every block the mixer reaches
        }
      R.peak0 = n_peaks;
      n_peaks += R.n_blocks;
      const size_t values = size_t (R.n44) * size_t (R.C);
      if (waves.empty() || (waves.back().r1 > waves.back().r0 && 2 * (waves.back().values + values) * sizeof (float) > cap))
        {
          Wave w;
          w.b0 = blist.size();
          w.r0 = w.r1 = rlist.size();
          waves.push_back (w);
        }
      Wave& w = waves.back();
      R.rs0 = w.n_rs;
      R.mix0 = w.n_mix;
      R.lim0 = w.n_lim;
      w.n_rs += (R.n44 + kRateCta - 1) / kRateCta;
      w.n_mix += (R.n_emit + kRateCta - 1) / kRateCta;
      if (R.limiter_block > 0)
        w.n_lim += (R.n_frames + 256 * kLimiterIter - 1) / (256 * kLimiterIter);
      /* WatermarkGen::run on every 1024-frame of the scratch copy (src/wmadd.cc:394-399): n_frames = n44, no limiter, no --snr */
      blist.push_back (batch_entry ((long long) w.values, R.n44, R.C, int (i), 0, w.n_tiles, unused, unused, R.w0, role_table (i)));
      soff.push_back (w.values);
      w.values += values;
      rlist.push_back (R);
      w.r1 = rlist.size();
      max_values = std::max (max_values, w.values);
    }
  bool too_large = n_tiles44 >= INT_MAX || n_lim44 >= INT_MAX || blist.size() >= size_t (INT_MAX);
  for (const Wave& w : waves)
    too_large = too_large || std::max ({ w.n_tiles, w.n_rs, w.n_mix, w.n_lim }) >= INT_MAX;
  if (too_large)
    return fail (ctx, "%s: batch too large for one launch per step", name);
  if (covered < n_values)               /* values between items pass through unchanged */
    CK (cudaMemcpyAsync (d_out, d_in, n_values * sizeof (float), cudaMemcpyDeviceToDevice, ctx->stream));
  if (!blist.empty())
    {
      if (!rlist.empty())
        {
          CK (ctx->rate_scratch.reserve (2 * max_values * sizeof (float)));
          for (const Wave& w : waves)
            for (size_t k = w.r0; k < w.r1; k++)
              {
                rlist[k].x44 = ctx->rate_scratch.as<float>() + soff[k];
                rlist[k].wm44 = rlist[k].x44 + w.values;
              }
          CK (ctx->rate_items.reserve (rlist.size() * sizeof (RateItem)));
          CK (cudaMemcpyAsync (ctx->rate_items.p, rlist.data(), rlist.size() * sizeof (RateItem), cudaMemcpyHostToDevice, ctx->stream));
        }
      const size_t coded_bytes = n_items * 2 * size_t (rs.n_coded);
      CK (ctx->batch_items.reserve (blist.size() * sizeof (BatchItem)));
      CK (ctx->batch_coded.reserve (coded_bytes));
      CK (cudaMemcpyAsync (ctx->batch_items.p, blist.data(), blist.size() * sizeof (BatchItem), cudaMemcpyHostToDevice, ctx->stream));
      CK (cudaMemcpyAsync (ctx->batch_coded.p, coded_bits, coded_bytes, cudaMemcpyHostToDevice, ctx->stream));
      if (n_peaks)
        {
          CK (ctx->peaks.reserve (n_peaks * sizeof (unsigned)));
          CK (cudaMemsetAsync (ctx->peaks.p, 0, n_peaks * sizeof (unsigned), ctx->stream));
        }
      if (snr_power)
        {
          CK (ctx->snr.reserve (2 * n_items * sizeof (double)));
          CK (cudaMemsetAsync (ctx->snr.p, 0, 2 * n_items * sizeof (double), ctx->stream));
        }
      double *d_snr = snr_power ? ctx->snr.as<double>() : nullptr;
      const BatchItem *d_b = ctx->batch_items.as<BatchItem>();
      if (n_list44 && launch_embed_batch (ctx, rs, d_in, d_out, d_b, int (n_list44), n_tiles44, n_lim44, frames_pad_start, water_delta, limiter_block44,
                                          limiter_ceiling, d_snr, 0, zero_frames != nullptr))
        return 1;
      for (const Wave& w : waves)
        {
          const RateItem *d_r = ctx->rate_items.as<RateItem>() + w.r0;
          const int n_r = int (w.r1 - w.r0);
          float *x44 = ctx->rate_scratch.as<float>();
          /* items at stream offsets take their own instances, as k_embed_batch<true> does */
          const bool offsets = zero_frames != nullptr;
          PROF (ctx);
          (offsets ? k_resample_batch<true> : k_resample_batch<false>)<<<unsigned (w.n_rs), kRateCta, 0, ctx->stream>>> (d_r, n_r);
          LAUNCH_CHECK ("k_resample_batch");
          if (launch_embed_batch (ctx, rs, x44, x44 + w.values, d_b + w.b0, n_r, w.n_tiles, 0, frames_pad_start, water_delta, 0, limiter_ceiling, nullptr, 1,
                                  offsets))
            return 1;
          PROF (ctx);
          (offsets ? k_resample_mix_batch<true> : k_resample_mix_batch<false>)<<<unsigned (w.n_mix), kRateCta, 0, ctx->stream>>> (
            d_r, n_r, limiter_ceiling, ctx->peaks.as<unsigned>(), d_snr);
          LAUNCH_CHECK ("k_resample_mix_batch");
          if (w.n_lim)
            {
              PROF (ctx);
              (offsets ? k_limiter_rates<true> : k_limiter_rates<false>)<<<unsigned (w.n_lim), 256, 0, ctx->stream>>> (
                d_r, n_r, limiter_ceiling, ctx->peaks.as<unsigned>());
              LAUNCH_CHECK ("k_limiter_rates");
            }
        }
    }
  return batch_finish (ctx, out_v, s16, n_values, d_out, snr_power, blist.empty() ? 0 : n_items);
}

} // namespace

int
awm_embed_batch (awm_ctx *ctx, const void *in_v, void *out_v, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                 const uint8_t *coded_bits, int frames_pad_start, double water_delta, int limiter_block, float limiter_ceiling,
                 double *snr_power)
{
  char why[160];
  if (awm_batch_validate (items, n_items, n_values, why, sizeof (why)))
    return fail (ctx, "awm_embed_batch: %s", why);
  return embed_batch ("awm_embed_batch", ctx, in_v, out_v, is_s16, n_values, items, n_items, coded_bits, nullptr, nullptr, nullptr, 0,
                      frames_pad_start, water_delta, limiter_block, 0, limiter_ceiling, snr_power, 0);
}

int
awm_embed_batch_offsets (awm_ctx *ctx, const void *in_v, void *out_v, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                         const uint64_t *zero_frames, const uint8_t *coded_bits, int frames_pad_start, double water_delta, int limiter_block,
                         float limiter_ceiling, double *snr_power)
{
  if (n_items && !zero_frames)
    return fail (ctx, "awm_embed_batch_offsets: zero_frames list is NULL");
  char why[160];
  if (batch_offsets_check (items, n_items, n_values, zero_frames, false, why, sizeof (why)))
    return fail (ctx, "awm_embed_batch_offsets: %s", why);
  return embed_batch ("awm_embed_batch_offsets", ctx, in_v, out_v, is_s16, n_values, items, n_items, coded_bits, zero_frames, nullptr, nullptr, 0,
                      frames_pad_start, water_delta, limiter_block, 0, limiter_ceiling, snr_power, 0);
}

int
awm_embed_batch_rates (awm_ctx *ctx, const void *in_v, void *out_v, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                       const uint8_t *coded_bits, const int *sample_rates, const uint64_t *n_emit, int mark_sample_rate, int frames_pad_start,
                       double water_delta, int limiter_ms, float limiter_ceiling, double *snr_power, size_t scratch_bytes)
{
  char why[240];
  if (awm_batch_rates_validate (items, n_items, n_values, sample_rates, n_emit, mark_sample_rate, why, sizeof (why)))
    return fail (ctx, "awm_embed_batch_rates: %s", why);
  return embed_batch ("awm_embed_batch_rates", ctx, in_v, out_v, is_s16, n_values, items, n_items, coded_bits, nullptr, sample_rates, n_emit,
                      mark_sample_rate, frames_pad_start, water_delta, int ((long long) mark_sample_rate * limiter_ms / 1000), limiter_ms,
                      limiter_ceiling, snr_power, scratch_bytes);
}

int
awm_embed_batch_rates_offsets (awm_ctx *ctx, const void *in_v, void *out_v, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                               const uint8_t *coded_bits, const int *sample_rates, const uint64_t *n_emit, const uint64_t *zero_frames,
                               int mark_sample_rate, int frames_pad_start, double water_delta, int limiter_ms, float limiter_ceiling,
                               double *snr_power, size_t scratch_bytes)
{
  char why[240];
  if (awm_batch_rates_offsets_validate (items, n_items, n_values, sample_rates, n_emit, zero_frames, mark_sample_rate, why, sizeof (why)))
    return fail (ctx, "awm_embed_batch_rates_offsets: %s", why);
  return embed_batch ("awm_embed_batch_rates_offsets", ctx, in_v, out_v, is_s16, n_values, items, n_items, coded_bits, zero_frames, sample_rates,
                      n_emit, mark_sample_rate, frames_pad_start, water_delta, int ((long long) mark_sample_rate * limiter_ms / 1000), limiter_ms,
                      limiter_ceiling, snr_power, scratch_bytes);
}

int
awm_embed_batch_keys (awm_ctx *ctx, const void *in_v, void *out_v, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                      const uint8_t *coded_bits, const int *sample_rates, const uint64_t *n_emit, const uint64_t *zero_frames, const uint32_t *key_index,
                      int mark_sample_rate, int frames_pad_start, double water_delta, int limiter_ms, float limiter_ceiling, double *snr_power,
                      size_t scratch_bytes)
{
  if (!ctx->key_roles_n)
    return fail (ctx, "awm_embed_batch_keys: awm_set_embed_roles_keys has not been called");
  if (mark_sample_rate <= 0)
    return fail (ctx, "awm_embed_batch_keys: mark sample rate %d must be > 0", mark_sample_rate);
  char why[240];
  if (awm_batch_keys_validate (items, n_items, n_values, sample_rates, n_emit, zero_frames, key_index, ctx->key_roles_n, mark_sample_rate, why, sizeof (why)))
    return fail (ctx, "awm_embed_batch_keys: %s", why);
  return embed_batch ("awm_embed_batch_keys", ctx, in_v, out_v, is_s16, n_values, items, n_items, coded_bits, zero_frames, sample_rates, n_emit,
                      mark_sample_rate, frames_pad_start, water_delta, int ((long long) mark_sample_rate * limiter_ms / 1000), limiter_ms, limiter_ceiling,
                      snr_power, scratch_bytes, key_index);
}

int
awm_embed_window_rates (awm_ctx *ctx, const float *in, float *out, size_t n_frames, int channels, const uint8_t *coded_bits, int sample_rate,
                        int mark_sample_rate, uint64_t stream_first, uint64_t n_emit, int frames_pad_start, double water_delta, int limiter_ms,
                        float limiter_ceiling, uint64_t snr_first, uint64_t snr_last, double *snr_power)
{
  if (sample_rate == mark_sample_rate)
    return fail (ctx, "awm_embed_window_rates: the input is at the watermark rate %d Hz (use awm_embed_window)", mark_sample_rate);
  if (snr_first > snr_last)
    return fail (ctx, "awm_embed_window_rates: --snr range [%llu, %llu) is reversed", (unsigned long long) snr_first, (unsigned long long) snr_last);
  if (channels <= 0 || n_frames > AWM_MAX_STREAM_FRAMES)
    return fail (ctx, "awm_embed_window_rates: channels %d must be > 0 and n_frames %zu at most 2^48", channels, n_frames);
  const awm_batch_item item = { 0, n_frames, channels };
  const size_t n_values = n_frames * size_t (channels);
  char why[240];
  if (awm_batch_rates_offsets_validate (&item, 1, n_values, &sample_rate, &n_emit, &stream_first, mark_sample_rate, why, sizeof (why)))
    return fail (ctx, "awm_embed_window_rates: %s", why);
  return embed_batch ("awm_embed_window_rates", ctx, in, out, 0, n_values, &item, 1, coded_bits, &stream_first, &sample_rate, &n_emit, mark_sample_rate,
                      frames_pad_start, water_delta, int ((long long) mark_sample_rate * limiter_ms / 1000), limiter_ms, limiter_ceiling, snr_power, 0,
                      nullptr, snr_first, snr_last);
}

int
awm_window_range_rates (uint64_t own_first, uint64_t own_end, uint64_t n_total, int sample_rate, int mark_sample_rate, int limiter_ms, int hlen,
                        uint64_t *ext_first, uint64_t *ext_end)
{
  if (sample_rate <= 0 || mark_sample_rate <= 0 || !resample_ratio_ok (double (mark_sample_rate) / sample_rate) ||
      !resample_ratio_ok (double (sample_rate) / mark_sample_rate) || hlen < 8 || hlen > 96 || limiter_ms <= 0 || own_first >= own_end ||
      own_end > n_total || own_end > AWM_MAX_STREAM_FRAMES)
    return 1;
  const uint64_t N = kFrame, far = AWM_MAX_STREAM_FRAMES * 64;   // "no end": beyond every stream at either rate
  const uint64_t L = std::max<uint64_t> (uint64_t (sample_rate) * uint64_t (limiter_ms) / 1000, 1);
  /* 1. the limiter gain of an owned frame reads the peaks of its own block and of the blocks before and after it */
  const uint64_t b0 = own_first / L, b1 = (own_end - 1) / L;
  const uint64_t m0 = b0 ? (b0 - 1) * L : 0, m1 = (b1 + 2) * L;
  /* 2. every frame of those blocks reads the watermark at the watermark rate through the out-resampler's taps */
  uint64_t w0, w1;
  awm_resample_taps (far, double (sample_rate) / mark_sample_rate, hlen, m0, m1 - m0, &w0, &w1);
  /* 3. a watermark sample reads the 1024-frames before and after its own (the synthesis window) */
  const uint64_t x0 = (w0 / N ? w0 / N - 1 : 0) * N, x1 = ((std::max (w1, w0 + 1) - 1) / N + 2) * N;
  /* 4. those frames read the input through the in-resampler's taps */
  uint64_t e0, e1;
  awm_resample_taps (far, double (mark_sample_rate) / sample_rate, hlen, x0, x1 - x0, &e0, &e1);
  /* 5. one frame of margin on each side (the float positions of the taps are rounded), 6. inside the stream */
  e0 = std::min (e0, m0);
  e1 = std::max (e1, m1);
  *ext_first = e0 ? e0 - 1 : 0;
  *ext_end = std::min (e1 + 1, n_total);
  return 0;
}

/* ---------------------------------------------------------------- speed scan */

int
awm_speed_scan (awm_ctx *ctx, int key_slot, const float *clip, size_t clip_frames, int channels, int sample_rate,
                double seconds, const double *centers, int n_centers, const double *relative_speeds, int n_relative,
                double water_delta, double *quality_out)
{
  if (key_slot < 0 || key_slot >= AWM_MAX_KEYS || channels <= 0 || !clip || !centers || !relative_speeds || !quality_out || n_centers < 0 || n_relative < 0)
    return fail (ctx, "awm_speed_scan: bad arguments");
  SyncTab& t = ctx->keys[key_slot].sync[AWM_MODE_BLOCK];
  const int fpb = ctx->keys[key_slot].fpb;
  if (!t.n_ent || !fpb)
    return fail (ctx, "awm_speed_scan: tables for key slot %d not set", key_slot);
  if (t.n_ent > kCmpMaxEntries)
    return fail (ctx, "awm_speed_scan: %d sync entries exceed the kernel limit %d", t.n_ent, kCmpMaxEntries);
  const size_t n_jobs = size_t (n_centers) * n_relative;
  if (n_jobs > 65535)
    return fail (ctx, "awm_speed_scan: %d centres x %d relative speeds = %zu jobs exceed the limit 65535", n_centers, n_relative, n_jobs);
  for (size_t i = 0; i < n_jobs; i++)
    if (!(std::isfinite (relative_speeds[i]) && relative_speeds[i] > 0))
      return fail (ctx, "awm_speed_scan: relative speed %g (job %zu) is not finite and > 0", relative_speeds[i], i);
  for (size_t i = 0; i < n_jobs; i++)
    quality_out[i] = 0;
  ctx->sp_last.clear();
  ctx->sp_last_ent = t.n_ent;
  if (!n_jobs)
    return 0;
  CK (cudaSetDevice (ctx->device));
  /* geometry per centre: resample_ratio_truncate (in_data, center / 2, ..., seconds / center), src/wmspeed.cc:206 + src/resample.cc:100-125 */
  std::vector<ResampleJob> rj (n_centers);
  std::vector<MagJob> mj (n_centers);
  std::vector<CmpJob> cj (n_jobs);
  size_t sub_total = 0, mag_total = 0;
  int max_rows = 0;
  for (int c = 0; c < n_centers; c++)
    {
      const double ratio = centers[c] / 2;
      if (!resample_ratio_ok (ratio))
        return fail (ctx, "awm_speed_scan: centre %g not supported", centers[c]);
      const double max_in_seconds = seconds / centers[c];
      size_t in_trunc = clip_frames;
      if (max_in_seconds > 0)
        in_trunc = std::min<size_t> (in_trunc, size_t (lrint (sample_rate * max_in_seconds)));
      const long long n_sub = lrint (double (in_trunc) * ratio);
      const int rows = n_sub > kSpeedFrame ? int ((n_sub - kSpeedFrame + kSpeedHop - 1) / kSpeedHop) : 0;
      rj[c].n_in = (long long) in_trunc;
      rj[c].n_stop = rj[c].n_in;
      rj[c].n_out = n_sub;
      rj[c].step = 1.0 / ratio;
      mj[c].n_sub = n_sub;
      mj[c].rows = rows;
      sub_total += size_t (n_sub) * channels;
      mag_total += size_t (rows) * t.n_ent;
      max_rows = std::max (max_rows, rows);
    }
  /* SpeedSync::compare: offsets -pad_start .. -1, pad_start = one block + one frame in search steps (src/wmspeed.cc:331) */
  const int pad_start = fpb * 4 + 4;
  for (int c = 0; c < n_centers; c++)
    for (int r = 0; r < n_relative; r++)
      {
        CmpJob& J = cj[size_t (c) * n_relative + r];
        const double rs = relative_speeds[size_t (c) * n_relative + r];
        J.rows = mj[c].rows;
        J.inv = 1 / rs;                              /* relative_speed_inv, src/wmspeed.cc:274 */
        J.off_scale = (1 << 16) / rs;                /* src/wmspeed.cc:341 */
        /* the 16.16 contract of k_speed_compare: the most negative offset and every frame offset below fo_cut fit in 31 bits */
        const double off_min = double (-pad_start) * J.off_scale;
        if (!(off_min > -2147483647.0))
          return fail (ctx, "awm_speed_scan: relative speed %g: start offsets need more than 31 bits in 16.16", rs);
        J.fo_cut = 65536.0 * J.rows - double (int (off_min));
        if (J.fo_cut <= 2147483648.0)                /* every frame offset below fo_cut fits (always so for scans of <= 50 s) */
          continue;
        for (int B = 0; B < 3; B++)
          for (const auto& e : t.h_ent)
            {
              const double f = (double ((B * (long long) fpb + e.frame) * 4) * J.inv + 0.5) * 65536.0;
              if (f < J.fo_cut && f >= 2147483648.0)
                return fail (ctx, "awm_speed_scan: relative speed %g, %d rows: an entry of block %d at frame %d needs a 16.16 offset of more "
                             "than 31 bits", rs, J.rows, B, int (e.frame));
            }
      }
  /* every filter table this scan needs, fetched after making room for all new ones at once: coef_table empties a full cache,
   * which would free the tables of the centres already collected.  Making room may empty the cache, after which every distinct
   * centre of the call is fetched anew, so all of them (not only the new ones) must fit: then no fetch below empties it again */
  {
    std::set<double> ratios;
    size_t n_new = 0;
    for (int c = 0; c < n_centers; c++)
      if (ratios.insert (centers[c] / 2).second && !ctx->coef_cache.count (std::make_pair (centers[c] / 2, 16)))
        n_new++;
    if (ratios.size() > kCoefCacheCap)
      return fail (ctx, "awm_speed_scan: %zu distinct centres exceed the resampler table cache (%zu)", ratios.size(), kCoefCacheCap);
    if (coef_cache_room (ctx, n_new))
      return 1;
  }
  for (int c = 0; c < n_centers; c++)
    if (coef_table (ctx, centers[c] / 2, 16, &rj[c].coef, &rj[c].h))
      return 1;
  if (!ctx->win512.p)
    {
      /* FFTAnalyzer::gen_normalized_window (sub_frame_size), src/wmcommon.cc:68-89 */
      std::vector<float> win (kSpeedFrame);
      double weight = 0;
      for (int i = 0; i < kSpeedFrame; i++)
        {
          const double w = window_cos ((i - kSpeedFrame / 2.0) / (kSpeedFrame / 2.0));
          win[i] = w;
          weight += w;
        }
      for (int i = 0; i < kSpeedFrame; i++)
        win[i] *= 2.0 / weight;
      CK (ctx->win512.reserve (win.size() * sizeof (float)));
      CK (cudaMemcpy (ctx->win512.p, win.data(), win.size() * sizeof (float), cudaMemcpyHostToDevice));
    }
  const float *d_clip = clip;
  if (!is_device_ptr (clip))
    {
      CK (ctx->sp_clip.reserve (clip_frames * channels * sizeof (float)));
      CK (cudaMemcpyAsync (ctx->sp_clip.p, clip, clip_frames * channels * sizeof (float), cudaMemcpyHostToDevice, ctx->stream));
      d_clip = ctx->sp_clip.as<float>();
    }
  for (int c = 0; c < n_centers; c++)
    rj[c].in = d_clip;
  CK (ctx->sp_sub.reserve (std::max<size_t> (sub_total, 1) * sizeof (float)));
  CK (ctx->sp_mags.reserve (std::max<size_t> (mag_total, 1) * sizeof (float2)));
  {
    size_t so = 0, mo = 0;
    for (int c = 0; c < n_centers; c++)
      {
        rj[c].out = ctx->sp_sub.as<float>() + so;
        mj[c].sub = rj[c].out;
        mj[c].mags = ctx->sp_mags.as<float2>() + mo;
        so += size_t (rj[c].n_out) * channels;
        mo += size_t (mj[c].rows) * t.n_ent;
        for (int r = 0; r < n_relative; r++)
          cj[size_t (c) * n_relative + r].mags = mj[c].mags;
      }
  }
  if (launch_resample (ctx, rj, channels))
    return 1;
  CK (ctx->sp_mag_jobs.reserve (mj.size() * sizeof (MagJob)));
  CK (ctx->sp_cmp_jobs.reserve (cj.size() * sizeof (CmpJob)));
  CK (ctx->sp_best.reserve (n_jobs * sizeof (unsigned long long)));
  CK (cudaMemcpyAsync (ctx->sp_mag_jobs.p, mj.data(), mj.size() * sizeof (MagJob), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaMemcpyAsync (ctx->sp_cmp_jobs.p, cj.data(), cj.size() * sizeof (CmpJob), cudaMemcpyHostToDevice, ctx->stream));
  CK (cudaMemsetAsync (ctx->sp_best.p, 0, n_jobs * sizeof (unsigned long long), ctx->stream));
  if (max_rows > 0)
    {
      if (set_smem (ctx, k_speed_mags, kMagSmemBytes)) return 1;
      const dim3 grid (unsigned ((max_rows + kMagRows - 1) / kMagRows), unsigned (n_centers));
      PROF (ctx);
      k_speed_mags<<<grid, kMagWarps * 32, kMagSmemBytes, ctx->stream>>> (ctx->sp_mag_jobs.as<MagJob>(), channels, t.ent.as<awm_sync_entry>(), t.n_ent,
                                                                          ctx->tw.as<float2>(), ctx->win512.as<float>());
      LAUNCH_CHECK ("k_speed_mags");
      const double norm_div = water_delta < 0.080 ? water_delta : 0.080;
      const dim3 cgrid (unsigned ((pad_start + 255) / 256), unsigned (n_jobs));
      PROF (ctx);
      k_speed_compare<<<cgrid, 256, 0, ctx->stream>>> (ctx->sp_cmp_jobs.as<CmpJob>(), t.ent.as<awm_sync_entry>(), t.off.as<int>(), t.n_bits, t.n_ent,
                                                       fpb, pad_start, norm_div, ctx->sp_best.as<unsigned long long>());
      LAUNCH_CHECK ("k_speed_compare");
    }
  static_assert (sizeof (double) == sizeof (unsigned long long), "quality bits");
  CK (cudaMemcpyAsync (quality_out, ctx->sp_best.p, n_jobs * sizeof (double), cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  ctx->sp_last = mj;
  return 0;
}

int
awm_speed_mags (awm_ctx *ctx, int center, float *out, size_t max, int *rows, int *n_entries)
{
  if (!rows || !n_entries || center < 0 || size_t (center) >= ctx->sp_last.size())
    return fail (ctx, "awm_speed_mags: bad arguments (centre %d of %zu)", center, ctx->sp_last.size());
  const MagJob& m = ctx->sp_last[center];
  *rows = m.rows;
  *n_entries = ctx->sp_last_ent;
  const size_t n = size_t (m.rows) * ctx->sp_last_ent;
  if (!out || !n)
    return 0;
  if (max < n)
    return fail (ctx, "awm_speed_mags: out too small (%zu < %zu)", max, n);
  CK (cudaSetDevice (ctx->device));
  CK (cudaMemcpyAsync (out, m.mags, n * sizeof (float2), cudaMemcpyDeviceToHost, ctx->stream));
  CK (cudaStreamSynchronize (ctx->stream));
  return 0;
}

int
awm_resampler_cache (awm_ctx *ctx, size_t *size, size_t *cap)
{
  if (!size || !cap)
    return fail (ctx, "awm_resampler_cache: bad arguments");
  *size = ctx->coef_cache.size();
  *cap = kCoefCacheCap;
  return 0;
}
