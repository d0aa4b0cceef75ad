// awm_get.cc -- `audiowmark get / cmp`: chunk loop, BlockDecoder, ClipDecoder, ResultSet
// (reference src/wmget.cc:163-1013, src/wavchunkloader.cc:54-239).  FFTs, soft-bit extraction and the
// Viterbi decoder run on the GPU through the C ABI; pairing / combining logic stays on the host.
#include "awm_results.hh"
#include "awm_get_internal.hh"
#include "awm_balanced.hh"
#include "awm_speed.hh"
#include "awm_engine.hh"
#include "awm_tables.hh"
#include "awm_util.hh"

#include <algorithm>
#include <map>
#include <memory>
#include <math.h>
#include <string.h>
#include <stdlib.h>

using std::string;
using std::vector;
using std::max;
using std::min;

int
frame_count (const WavData& wav_data)
{
  return wav_data.n_values() / wav_data.n_channels() / Params::frame_size;
}

/* ---------------------------------------------------------------- GPU helpers */

namespace get_detail {

/* code_decode_soft for a set of code words (A, B and AB mixed) in ONE awm_viterbi launch */
bool
viterbi_decode (const vector<const VitJob *>& jobs, vector<uint8_t>& bits, vector<float>& err)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return false;
  const int n_msg = int (code_message_bits());        /* the block code word in short payload mode */
  bits.assign (jobs.size() * n_msg, 0);
  err.assign (jobs.size(), 0.f);
  if (jobs.empty())
    return true;
  vector<float> raw;
  vector<int> types (jobs.size());
  for (size_t j = 0; j < jobs.size(); j++)
    {
      raw.insert (raw.end(), jobs[j]->soft.begin(), jobs[j]->soft.end());
      types[j] = jobs[j]->block_type == ConvBlockType::a ? AWM_BLOCK_A : jobs[j]->block_type == ConvBlockType::b ? AWM_BLOCK_B : AWM_BLOCK_AB;
    }
  if (awm_viterbi (ctx, raw.data(), jobs.size(), n_msg, types.data(), Params::hard ? 1 : 0, bits.data(), err.data()))
    {
      error ("audiowmark: viterbi decoder failed: %s\n", awm_last_error (ctx));
      return false;
    }
  return true;
}

void
add_decoded_pattern (const VitJob& job, const uint8_t *bits, float err, ResultSet& chunk_result)
{
  const int n_msg = int (code_message_bits());
  vector<int> bit_vec (bits, bits + n_msg);
  if (Params::payload_short)
    {
      bit_vec = short_decode_blk (bit_vec);        /* code_decode_soft, src/shortcode.cc:129-133 */
      if (bit_vec.empty())
        return;
    }
  chunk_result.add_pattern (job.key, job.time, job.score, bit_vec, err, job.type, job.speed);
}

/* every pending code word of a `get` run (all chunks and keys) in one launch; the decoded patterns go to the result set of the
 * chunk they came from */
bool
run_viterbi_jobs (vector<VitJob>& jobs, vector<ResultSet>& chunk_results)
{
  vector<const VitJob *> list;
  for (const auto& j : jobs)
    list.push_back (&j);
  vector<uint8_t> bits;
  vector<float> err;
  if (!viterbi_decode (list, bits, err))
    return false;
  const int n_msg = int (code_message_bits());
  for (size_t j = 0; j < jobs.size(); j++)
    add_decoded_pattern (jobs[j], bits.data() + j * n_msg, err[j], chunk_results[jobs[j].chunk]);
  jobs.clear();
  return true;
}

/* fft_range + mix_decode + randomize_bit_order (decode) for several block start positions */
bool
decode_raw_bits (const Key& key, const vector<uint64_t>& indices, vector<vector<float>>& raw, vector<int>& valid)
{
  awm_ctx *ctx = Engine::ctx();
  const int slot = ctx ? Engine::key_slot (key) : -1;
  if (slot < 0)
    return false;
  const size_t n_coded = code_size (ConvBlockType::a, Params::payload_size);
  vector<float> flat (indices.size() * n_coded);
  valid.assign (indices.size(), 0);
  if (awm_decode_blocks (ctx, slot, indices.data(), indices.size(), flat.data(), valid.data()))
    {
      error ("audiowmark: block decode failed: %s\n", awm_last_error (ctx));
      return false;
    }
  raw.resize (indices.size());
  for (size_t i = 0; i < indices.size(); i++)
    raw[i].assign (flat.begin() + i * n_coded, flat.begin() + (i + 1) * n_coded);
  return true;
}

/* What BlockDecoder::run does once the soft bits of the synchronised blocks are known (src/wmget.cc:539-701), as three separate
 * steps over one list of decoded blocks (in sync-score order = ascending position):
 *   single blocks   every valid block is a code word of its own type
 *   AB pairs        a B block together with the A block that starts one block length before it
 *   "all"           the longest-scoring chain of alternating blocks, soft bits averaged per type
 * The selection rules (tolerances, strict comparisons, float accumulation of the chain score) are the reference's: they decide
 * which patterns are printed. */
struct DecodedBlock
{
  size_t               index;
  double               quality;
  ConvBlockType        type;
  const vector<float> *soft;
};

ConvBlockType
other_type (ConvBlockType t)
{
  return t == ConvBlockType::a ? ConvBlockType::b : ConvBlockType::a;
}

/* position in `blocks` of the block of type `want` nearest to sample `target`, among positions >= first and < last, nearer than
 * `tolerance` samples (the earliest of equally near blocks); -1 if there is none */
int
nearest_block (const vector<DecodedBlock>& blocks, size_t first, size_t last, ConvBlockType want, int target, int tolerance)
{
  int found = -1, nearest = tolerance;
  for (size_t j = first; j < last; j++)
    {
      const int dist = std::abs (target - int (blocks[j].index));
      if (blocks[j].type == want && dist < nearest)
        {
          found = int (j);
          nearest = dist;
        }
    }
  return found;
}

/* chain of alternating blocks that starts at block `head`: after the last member, the block expected k block lengths later
 * (type flips with odd k) is looked for with k = 1, 2, ... and a tolerance that grows with k; a hit restarts at k = 1 */
vector<size_t>
alternating_chain (const vector<DecodedBlock>& blocks, size_t head, size_t block_len)
{
  const size_t k_max = lrint (blocks.back().index / double (block_len) + 0.5);
  vector<size_t> chain { head };
  for (size_t k = 1; k <= k_max; )
    {
      const DecodedBlock& tail = blocks[chain.back()];
      const int next = nearest_block (blocks, chain.back(), blocks.size(), (k & 1) ? other_type (tail.type) : tail.type,
                                      int (tail.index + k * block_len), int (k * Params::frame_size / 2));
      if (next >= 0)
        {
          chain.push_back (next);
          k = 1;
        }
      else
        k++;
    }
  return chain;
}

float
chain_score (const vector<DecodedBlock>& blocks, const vector<size_t>& chain)
{
  float sum = 0;                                  /* single precision like the reference: it breaks near ties the same way */
  for (size_t b : chain)
    sum += blocks[b].quality;
  return sum;
}

void
build_block_jobs (const Key& key, const vector<SyncFinder::Score>& sync_scores, const vector<vector<float>>& raw, const vector<int>& valid,
                  int sample_rate, int chunk, double speed, vector<VitJob>& pending)
{
  const size_t block_len = (mark_sync_frame_count() + mark_data_frame_count()) * Params::frame_size;
  auto queue = [&] (const vector<float>& soft, ConvBlockType code, double time, SyncFinder::Score score, ResultSet::Type type)
    {
      pending.push_back (VitJob { soft, code, time, score, type, key, chunk, speed });
    };
  vector<DecodedBlock> blocks;
  for (size_t i = 0; i < sync_scores.size(); i++)
    if (valid[i])
      {
        blocks.push_back ({ sync_scores[i].index, sync_scores[i].quality, sync_scores[i].block_type, &raw[i] });
        queue (raw[i], sync_scores[i].block_type, double (sync_scores[i].index) / sample_rate, sync_scores[i], ResultSet::Type::BLOCK);
      }
  /* ---- AB pairs */
  for (size_t i = 0; i < blocks.size(); i++)
    {
      if (blocks[i].type != ConvBlockType::b)
        continue;
      const int partner = nearest_block (blocks, 0, i, ConvBlockType::a, int (blocks[i].index) - int (block_len), Params::frame_size / 2);
      if (partner < 0)
        continue;
      const vector<float>& sa = *blocks[partner].soft, &sb = *blocks[i].soft;
      vector<float> interleaved (sa.size() * 2);
      for (size_t k = 0; k < sa.size(); k++)
        {
          interleaved[2 * k] = sa[k];
          interleaved[2 * k + 1] = sb[k];
        }
      queue (interleaved, ConvBlockType::ab, double (blocks[i].index) / sample_rate,
             SyncFinder::Score { blocks[i].index, (blocks[partner].quality + blocks[i].quality) / 2, ConvBlockType::ab }, ResultSet::Type::BLOCK);
    }
  /* ---- "all": the chain with the largest quality sum (the first one among equals) */
  vector<size_t> best;
  for (size_t head = 0; head < blocks.size(); head++)
    {
      const vector<size_t> chain = alternating_chain (blocks, head, block_len);
      if (chain_score (blocks, chain) > chain_score (blocks, best))
        best = chain;
    }
  if (best.size() > 1)
    {
      vector<float> mean_soft (code_size (ConvBlockType::ab, Params::payload_size));
      int members[2] = { 0, 0 };
      double quality_sum = 0;
      for (size_t b : best)
        {
          const int slot = blocks[b].type == ConvBlockType::b ? 1 : 0;
          const vector<float>& soft = *blocks[b].soft;
          for (size_t k = 0; k < soft.size(); k++)
            mean_soft[2 * k + slot] += soft[k];
          members[slot]++;
          quality_sum += blocks[b].quality;
        }
      for (size_t k = 0; k < mean_soft.size(); k++)
        mean_soft[k] /= max (members[k & 1], 1);
      queue (mean_soft, ConvBlockType::ab, 0.0, SyncFinder::Score { 0, quality_sum / (members[0] + members[1]), ConvBlockType::a }, ResultSet::Type::ALL);
    }
}

/* ---------------------------------------------------------------- BlockDecoder (src/wmget.cc:492-735) */

class BlockDecoder
{
  int debug_sync_frame_count = 0;
  const double speed;
  vector<SyncFinder::KeyResult> key_results;
public:
  explicit BlockDecoder (double speed) : speed (speed) {}

  /* the PCM (n_frames x n_channels at sample_rate) is already bound to the GPU context, or searched in approx_slot (SyncFinder::search) */
  void
  run (const vector<Key>& key_list, size_t n_frames, int n_channels, int sample_rate, vector<VitJob>& pending, int chunk, int approx_slot = -1)
  {
    SyncFinder sync_finder;
    key_results = sync_finder.search (key_list, n_frames, n_channels, SyncFinder::Mode::BLOCK, 0, n_frames * n_channels, approx_slot);
    for (const auto& key_result : key_results)
      {
        const Key& key = key_result.key;
        vector<uint64_t> indices;
        for (const auto& s : key_result.sync_scores)
          indices.push_back (s.index);
        vector<vector<float>> raw;
        vector<int> valid;
        if (!indices.empty() && !decode_raw_bits (key, indices, raw, valid))
          continue;
        build_block_jobs (key, key_result.sync_scores, raw, valid, sample_rate, chunk, speed, pending);
      }
    debug_sync_frame_count = n_frames / Params::frame_size;
  }
  string
  debug_sync()
  {
    if (key_results.size() != 1)
      return "";
    const auto& sync_scores = key_results[0].sync_scores;
    const int expect0 = Params::frames_pad_start * Params::frame_size;
    const int expect_step = (mark_sync_frame_count() + mark_data_frame_count()) * Params::frame_size;
    const int expect_end = debug_sync_frame_count * Params::frame_size;
    int sync_match = 0;
    for (int expect_index = expect0; expect_index + expect_step < expect_end; expect_index += expect_step)
      for (auto sync_score : sync_scores)
        if (abs (int (sync_score.index + Params::test_cut) - expect_index) < int (Params::frame_size / 2))
          {
            sync_match++;
            break;
          }
    return string_printf ("sync_match %d %zd\n", sync_match, sync_scores.size());
  }
};

/* ---------------------------------------------------------------- ClipDecoder (src/wmget.cc:737-884) */

class ClipDecoder
{
  const int frames_per_blk;
  const double speed;

  enum class Pos { START, END };
  void
  run_block (const vector<Key>& key_list, const float *samples, size_t n_frames, int n_channels, int sample_rate, vector<VitJob>& pending, int chunk, Pos pos)
  {
    awm_ctx *ctx = Engine::ctx();
    if (!ctx)
      return;
    const size_t n_values = n_frames * n_channels;
    const size_t n = size_t (frames_per_blk + 5) * Params::frame_size * n_channels;      // values of one padded block
    size_t first_sample, last_sample, pad_start = n, pad_end = n;
    if (pos == Pos::START)
      {
        first_sample = 0;
        last_sample = min (n, n_values);
        if (last_sample < n)                    // available samples + padding must always be one long block
          pad_start += n - last_sample;
      }
    else
      {
        if (n_values <= n)
          return;
        first_sample = n_values - n;
        last_sample = n_values;
      }
    const double time_offset = double (first_sample) / sample_rate / n_channels;
    /* scan_silence on the padded signal: [wav_first, wav_last) in value units */
    size_t nz_first = first_sample, nz_last = last_sample;
    while (nz_first < last_sample && samples[nz_first] == 0)
      nz_first++;
    while (nz_last > nz_first && samples[nz_last - 1] == 0)
      nz_last--;
    size_t wav_first, wav_last;
    const size_t ext_values = pad_start + (last_sample - first_sample) + pad_end;
    if (nz_first == last_sample)                // all zero
      wav_first = wav_last = ext_values;
    else
      {
        wav_first = pad_start + (nz_first - first_sample);
        wav_last = pad_start + (nz_last - first_sample);
      }
    const size_t ext_frames = ext_values / n_channels;
    if (awm_pcm_bind (ctx, samples + first_sample, (last_sample - first_sample) / n_channels, n_channels, pad_start / n_channels, pad_end / n_channels))
      {
        error ("audiowmark: %s\n", awm_last_error (ctx));
        return;
      }
    SyncFinder sync_finder;
    vector<SyncFinder::KeyResult> key_results = sync_finder.search (key_list, ext_frames, n_channels, SyncFinder::Mode::CLIP, wav_first, wav_last);
    const size_t count = mark_sync_frame_count() + mark_data_frame_count();
    for (const auto& key_result : key_results)
      {
        const Key& key = key_result.key;
        vector<uint64_t> indices;
        for (const auto& s : key_result.sync_scores)
          {
            indices.push_back (s.index);
            indices.push_back (s.index + count * Params::frame_size);
          }
        vector<vector<float>> raw;
        vector<int> valid;
        if (indices.empty() || !decode_raw_bits (key, indices, raw, valid))
          continue;
        for (size_t i = 0; i < key_result.sync_scores.size(); i++)
          if (valid[2 * i] && valid[2 * i + 1])
            {
              const auto& sync_score = key_result.sync_scores[i];
              const vector<float>& r1 = raw[2 * i], & r2 = raw[2 * i + 1];
              vector<float> raw_bit_vec (r1.size() * 2);
              for (size_t k = 0; k < r1.size(); k++)
                {
                  raw_bit_vec[2 * k]     = sync_score.block_type == ConvBlockType::a ? r1[k] : r2[k];
                  raw_bit_vec[2 * k + 1] = sync_score.block_type == ConvBlockType::a ? r2[k] : r1[k];
                }
              SyncFinder::Score sync_score_nopad = sync_score;
              sync_score_nopad.index = time_offset * sample_rate;
              pending.push_back (VitJob { raw_bit_vec, ConvBlockType::ab, time_offset, sync_score_nopad, ResultSet::Type::CLIP, key, chunk, speed });
            }
      }
  }
public:
  explicit ClipDecoder (double speed) : frames_per_blk (mark_sync_frame_count() + mark_data_frame_count()), speed (speed) {}
  bool wanted (size_t n_frames) const { return int (n_frames / Params::frame_size) < frames_per_blk * 3.1; }   /* clip decoder is only used for small inputs */
  void
  run (const vector<Key>& key_list, const float *samples, size_t n_frames, int n_channels, int sample_rate, vector<VitJob>& pending, int chunk)
  {
    const int wav_frames = n_frames / Params::frame_size;
    if (wav_frames < frames_per_blk * 3.1)       // clip decoder is only used for small inputs
      {
        run_block (key_list, samples, n_frames, n_channels, sample_rate, pending, chunk, Pos::START);
        run_block (key_list, samples, n_frames, n_channels, sample_rate, pending, chunk, Pos::END);
      }
  }
};

/* decode (src/wmget.cc:886-939) for one chunk: everything up to the soft bits; the Viterbi jobs are queued.
 * pcm: the chunk's float samples in device memory, bound in place.  host_pcm (optional): the same samples in host memory; else the
 * clip decoder, which cuts and pads on the host, copies them back (short inputs only).
 * approx_slot >= 0: one key, no speed detection; the chunk's approx search has been queued into that slot (awm_sync_approx_enqueue) */
int
decode_chunk (vector<VitJob>& pending, int chunk, string& debug_sync, const vector<Key>& key_list, const float *pcm, const float *host_pcm,
              size_t n_frames, int n_channels, int sample_rate, bool first_chunk, bool print_speed_results, int approx_slot)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  if (approx_slot < 0 && awm_pcm_bind (ctx, pcm, n_frames, n_channels, 0, 0))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return 1;
    }
  vector<float> host_storage;
  auto need_host = [&] () -> const float *
    {
      if (!host_pcm)
        {
          host_storage.resize (n_frames * n_channels);
          if (awm_copy_to_host (ctx, host_storage.data(), pcm, host_storage.size() * sizeof (float)))
            return nullptr;
          host_pcm = host_storage.data();
        }
      return host_pcm;
    };
  /* The strategy for integrating speed detection into decoding (src/wmget.cc:888-928):
   *  - the watermark is always decoded on the original data
   *  - if the detected speed is somewhat different from 1.0, stretched data is decoded as well
   *  - all normal and speed results are reported (the detected speed may be wrong on short clips) */
  if (Params::detect_speed || Params::detect_speed_patient || Params::try_speed > 0)
    {
      vector<DetectSpeedResult> speed_results;
      if (Params::detect_speed || Params::detect_speed_patient)
        speed_results = detect_speed (key_list, pcm, n_frames, n_channels, sample_rate, print_speed_results);
      else
        for (const auto& key : key_list)
          speed_results.push_back ({ key, Params::try_speed });
      bool rebind = false;
      for (const auto& speed_result : speed_results)
        {
          /* resample_ratio (wav_data, speed, mark_sample_rate * speed): the stretched chunk stays on the device */
          const size_t speed_frames = lrint (double (n_frames) * speed_result.speed);
          const int speed_rate = Params::mark_sample_rate * speed_result.speed;
          if (rebind && awm_pcm_bind (ctx, pcm, n_frames, n_channels, 0, 0))
            return 1;
          rebind = false;
          if (awm_pcm_push_resampled (ctx, speed_result.speed, 16, speed_frames))
            {
              error ("audiowmark: %s\n", awm_last_error (ctx));
              return 1;
            }
          BlockDecoder speed_block_decoder (speed_result.speed);
          speed_block_decoder.run ({ speed_result.key }, speed_frames, n_channels, speed_rate, pending, chunk);
          awm_pcm_pop (ctx);
          if (first_chunk && int (speed_frames / Params::frame_size) < (mark_sync_frame_count() + mark_data_frame_count()) * 3.1)
            {
              /* the clip decoder cuts and pads on the host: short inputs only, so the extra copy is small */
              vector<float> stretched;
              if (!need_host() || !resample_ratio (need_host(), n_frames, n_channels, speed_result.speed, stretched))
                return 1;
              ClipDecoder speed_clip_decoder (speed_result.speed);
              speed_clip_decoder.run ({ speed_result.key }, stretched.data(), speed_frames, n_channels, speed_rate, pending, chunk);
              rebind = true;
            }
        }
      if (rebind && awm_pcm_bind (ctx, pcm, n_frames, n_channels, 0, 0))
        return 1;
    }
  const double tb0 = get_time();
  BlockDecoder block_decoder (1);
  block_decoder.run (key_list, n_frames, n_channels, sample_rate, pending, chunk, approx_slot);
  if (getenv ("AWM_TRACE"))
    fprintf (stderr, "[trace] chunk %d: block decoder (sync + soft bits) %.3f ms\n", chunk, (get_time() - tb0) * 1e3);
  if (first_chunk)
    {
      ClipDecoder clip_decoder (1);
      if (clip_decoder.wanted (n_frames))
        {
          if (!need_host())
            return 1;
          clip_decoder.run (key_list, need_host(), n_frames, n_channels, sample_rate, pending, chunk);
        }
    }
  debug_sync = block_decoder.debug_sync();
  return 0;
}

} // namespace get_detail

using namespace get_detail;

/* chunk geometry of WavChunkLoader (src/wavchunkloader.cc:54-163): chunks of get_chunk_size minutes that
 * overlap by two blocks * 1.3 */
void
chunk_geometry (int sample_rate, size_t& max_frames, size_t& overlap_frames)
{
  max_frames = lrint (Params::get_chunk_size * 60 * sample_rate);
  const double block_seconds = (mark_sync_frame_count() + mark_data_frame_count()) * Params::frame_size / double (Params::mark_sample_rate);
  overlap_frames = lrint (2 * block_seconds * 1.3 * sample_rate);
}

/* ---------------------------------------------------------------- GetStream */

namespace {

constexpr size_t kInputWindow = size_t (1) << 20;      // input frames the window takes between two resampler launches

/* buf[0, n) = buf[from, from + n) (frames of `channels` floats, device memory) in context stream order, in copies that do not
 * overlap: each reads frames no earlier copy has written */
bool
move_to_front (awm_ctx *ctx, float *buf, size_t from, size_t n, int channels)
{
  for (size_t done = 0; done < n && from; )
    {
      const size_t k = min (n - done, from);
      if (awm_copy (ctx, buf + done * channels, buf + (from + done) * channels, k * channels * sizeof (float)))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return false;
        }
      done += k;
    }
  return true;
}

/* the end of a `get`: one Viterbi launch over the jobs of all chunks, then the reference's per-chunk merge in chunk order */
int
merge_chunk_results (vector<VitJob>& pending, const vector<GetStream::Chunk>& chunks, const vector<string>& debug_syncs, const vector<Key>& key_list,
                     ResultSet& result_set)
{
  vector<ResultSet> chunk_results (chunks.size());
  const double tv0 = get_time();
  const size_t n_jobs = pending.size();
  if (!run_viterbi_jobs (pending, chunk_results))
    return 1;
  if (getenv ("AWM_TRACE"))
    fprintf (stderr, "[trace] viterbi: %zu jobs %.3f ms\n", n_jobs, (get_time() - tv0) * 1e3);
  for (size_t c = 0; c < chunk_results.size(); c++)
    {
      chunk_results[c].set_debug_sync (debug_syncs[c]);
      chunk_results[c].apply_time_offset (chunks[c].time_offset);
      result_set.merge (chunk_results[c]);
    }
  result_set.sort (key_list);
  return 0;
}

}

GetStream::GetStream (const vector<Key>& key_list, int n_channels, int sample_rate, bool print_speed_results, size_t max_input_frames, bool dry_run) :
  m_keys (key_list), m_channels (n_channels), m_rate (sample_rate), m_print_speed (print_speed_results), m_dry (dry_run), m_max_input (max_input_frames)
{
  if (n_channels <= 0)
    {
      error ("audiowmark: get: %d channels\n", n_channels);
      return;
    }
  if (!balanced::rate_supported (sample_rate))
    {
      error ("audiowmark: get: sample rate %d Hz is not supported (%d Hz / 64 .. %d Hz * 64, exclusive)\n", sample_rate, Params::mark_sample_rate,
             Params::mark_sample_rate);
      return;
    }
  m_ratio = double (Params::mark_sample_rate) / sample_rate;
  chunk_geometry (Params::mark_sample_rate, m_max_frames, m_overlap);
  if (m_overlap >= m_max_frames)
    {
      error ("audiowmark: get: chunks of %zu frames cannot overlap by %zu frames\n", m_max_frames, m_overlap);
      return;
    }
  m_ok = true;
}

GetStream::~GetStream()
{
  if (m_chunk || m_in)
    {
      awm_device_free (Engine::ctx(), m_chunk);
      awm_device_free (Engine::ctx(), m_in);
    }
}

/* the chunk buffer (watermark rate, at most one chunk, or the whole announced stream if shorter) and at other rates the input window,
 * allocated once with the first fed frame: the stream's length does not change them */
bool
GetStream::ensure_buffers()
{
  if (m_chunk_cap)
    return true;
  m_chunk_cap = m_max_input == ~size_t (0) ? m_max_frames : min (m_max_frames, balanced::mark_frames (m_max_input, m_rate));
  if (m_rate != Params::mark_sample_rate)
    {
      /* the taps of the next output start at most 2h - 1 frames before the input's end (awm_resample_stream_available), plus one frame
       * of margin as in balanced::input_range */
      const size_t h = size_t (ceil (16 / std::min (1.0, m_ratio)));
      m_in_cap = min (kInputWindow, m_max_input) + 2 * h + 2;
    }
  m_peak_bytes = (m_chunk_cap + m_in_cap) * m_channels * sizeof (float);
  if (m_dry)
    return true;
  awm_ctx *ctx = Engine::ctx();
  void *chunk = nullptr, *in = nullptr;
  if (!ctx || awm_device_alloc (ctx, m_chunk_cap * m_channels * sizeof (float), &chunk)
      || (m_in_cap && awm_device_alloc (ctx, m_in_cap * m_channels * sizeof (float), &in)))
    {
      if (ctx)
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          awm_device_free (ctx, chunk);
        }
      return false;
    }
  m_chunk = static_cast<float *> (chunk);
  m_in = static_cast<float *> (in);
  return true;
}

/* decode the chunk buffer's m_fill frames as chunk number m_chunks.size() */
bool
GetStream::decode()
{
  const int chunk = int (m_chunks.size());
  m_chunks.push_back ({ m_start, m_fill, m_time_offset });
  string debug_sync;
  if (!m_dry && decode_chunk (m_pending, chunk, debug_sync, m_keys, m_chunk, nullptr, m_fill, m_channels, Params::mark_sample_rate, chunk == 0,
                              m_print_speed, -1))
    return false;
  m_debug_syncs.push_back (debug_sync);
  return true;
}

/* a full chunk is decoded; the next one starts with its last m_overlap frames */
bool
GetStream::chunk_full()
{
  if (!decode() || (!m_dry && !move_to_front (Engine::ctx(), m_chunk, m_max_frames - m_overlap, m_overlap, m_channels)))
    return false;
  m_fill = m_overlap;
  m_start += m_max_frames - m_overlap;
  m_time_offset += double (m_max_frames - m_overlap) / Params::mark_sample_rate;
  return true;
}

/* resample the watermark-rate frames [m_produced, until) into the chunk buffer from the input window; the caller guarantees that their
 * taps lie in [m_in_first, m_fed), so they are what awm_resample over the whole stream computes, whatever its final length */
bool
GetStream::produce (size_t until)
{
  awm_ctx *ctx = m_dry ? nullptr : Engine::ctx();
  while (m_produced < until)
    {
      const size_t n = min (until - m_produced, m_max_frames - m_fill);
      if (ctx && awm_resample_range (ctx, m_in, m_in_first, m_fed - m_in_first, m_fed, m_channels, m_ratio, 16, m_chunk + m_fill * m_channels, m_produced, n))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return false;
        }
      m_produced += n;
      m_fill += n;
      if (m_fill == m_max_frames && !chunk_full())
        return false;
    }
  return true;
}

int
GetStream::feed (const float *pcm, size_t n_frames)
{
  if (!m_ok || m_failed || m_finished || (!pcm && n_frames && !m_dry) || n_frames > m_max_input - min (m_fed, m_max_input))
    {
      error ("audiowmark: get: cannot feed %zu frames to this stream (%s)\n", n_frames, !m_ok ? "refused" : m_failed ? "failed before"
             : m_finished ? "finished" : !pcm ? "no samples" : "more frames than announced");
      m_failed = true;
      return 1;
    }
  if (n_frames && !ensure_buffers())
    {
      m_failed = true;
      return 1;
    }
  awm_ctx *ctx = m_dry ? nullptr : Engine::ctx();
  const size_t C = m_channels;
  while (n_frames)
    {
      size_t n;
      if (m_rate == Params::mark_sample_rate)
        {
          n = min (n_frames, m_max_frames - m_fill);
          if (ctx && awm_copy (ctx, m_chunk + m_fill * C, pcm, n * C * sizeof (float)))
            break;
          m_fed += n;
          m_produced += n;
          m_fill += n;
          if (m_fill == m_max_frames && !chunk_full())
            {
              m_failed = true;
              return 1;
            }
        }
      else
        {
          if (m_fed - m_in_first == m_in_cap)
            {
              /* the window is full: make every output it can, then keep only the input the taps of later outputs read */
              uint64_t t0, t1;
              if (!produce (resample_stream_available (m_fed, m_ratio)))
                {
                  m_failed = true;
                  return 1;
                }
              awm_resample_taps (m_fed, m_ratio, 16, m_produced, 1, &t0, &t1);
              const size_t keep = std::max (m_in_first, t0 ? size_t (t0) - 1 : 0);
              if (ctx && !move_to_front (ctx, m_in, keep - m_in_first, m_fed - keep, m_channels))
                {
                  m_failed = true;
                  return 1;
                }
              m_in_first = keep;
            }
          n = min (n_frames, m_in_cap - (m_fed - m_in_first));
          if (ctx && awm_copy (ctx, m_in + (m_fed - m_in_first) * C, pcm, n * C * sizeof (float)))
            break;
          m_fed += n;
        }
      if (pcm)
        pcm += n * C;
      n_frames -= n;
    }
  if (n_frames)
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      m_failed = true;
      return 1;
    }
  return 0;
}

int
GetStream::finish (ResultSet& result_set, size_t *mark_rate_frames)
{
  if (!m_ok || m_failed || m_finished)
    {
      error ("audiowmark: get: cannot finish this stream (%s)\n", !m_ok ? "refused" : m_failed ? "failed before" : "finished");
      return 1;
    }
  m_finished = true;
  /* at EOF the resampler delivers its trailing outputs: those of the whole stream, now that its length is known */
  if (m_rate != Params::mark_sample_rate && m_fed && !produce (balanced::mark_frames (m_fed, m_rate)))
    return 1;
  if ((!m_chunks.empty() || m_fill) && !decode())
    return 1;
  if (mark_rate_frames)
    *mark_rate_frames = m_produced;
  if (m_dry || m_chunks.empty())
    return 0;
  return merge_chunk_results (m_pending, m_chunks, m_debug_syncs, m_keys, result_set);
}

int
get_watermark_buffer (const vector<Key>& key_list, const float *samples, size_t n_frames, int n_channels, int sample_rate, ResultSet& result_set,
                      bool print_speed_results, size_t *mark_rate_frames)
{
  return get_watermark_pcm (key_list, samples, nullptr, n_frames, n_channels, sample_rate, result_set, print_speed_results, mark_rate_frames);
}

int
get_watermark_buffer_s16 (const vector<Key>& key_list, const int16_t *samples, size_t n_frames, int n_channels, int sample_rate, ResultSet& result_set,
                          bool print_speed_results, size_t *mark_rate_frames)
{
  return get_watermark_pcm (key_list, nullptr, samples, n_frames, n_channels, sample_rate, result_set, print_speed_results, mark_rate_frames);
}

int
get_watermark_pcm (const vector<Key>& key_list, const float *samples, const int16_t *samples16, size_t n_frames, int n_channels, int sample_rate,
                   ResultSet& result_set, bool print_speed_results, size_t *mark_rate_frames)
{
  if (sample_rate != Params::mark_sample_rate)
    {
      /* WavChunkLoader resamples the input to the watermark rate while it reads (src/wavchunkloader.cc:66-73, 196-221): the whole
       * buffer is one piece of a stream, resampled chunk by chunk on the device */
      vector<float> converted;
      if (samples16)
        {
          /* rare combination: convert on the host, then take the float path through the resampler */
          converted.resize (n_frames * n_channels);
          const float norm = 1.0 / 0x80000000LL;
          for (size_t i = 0; i < converted.size(); i++)
            converted[i] = (int (samples16[i]) << 16) * norm;
          samples = converted.data();
        }
      GetStream stream (key_list, n_channels, sample_rate, print_speed_results, n_frames);
      if (!stream.ok() || stream.feed (samples, n_frames))
        return 1;
      return stream.finish (result_set, mark_rate_frames);
    }
  if (mark_rate_frames)
    *mark_rate_frames = n_frames;
  size_t max_frames, overlap;
  chunk_geometry (sample_rate, max_frames, overlap);
  size_t start = 0, end = min (max_frames, n_frames);
  double time_offset = 0;
  bool eof = end < max_frames;
  if (n_frames == 0)
    return 0;
  /* pass 1: sync search + soft bits per chunk (GPU), Viterbi jobs of all chunks are collected */
  vector<VitJob> pending;
  vector<GetStream::Chunk> chunks;
  vector<string> debug_syncs;
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  /* host input crosses PCIe once, piece by piece: a chunk waits only for the pieces it reads, so the later chunks travel while the
   * first one is searched.  Device float input is bound in place. */
  const bool staged = samples16 || !Engine::is_device_pointer (samples);
  const float *pcm = samples;
  if (staged && awm_pcm_stage (ctx, samples16 ? static_cast<const void *> (samples16) : samples, samples16 ? 1 : 0, n_frames, n_channels,
                               kStagePiece, &pcm))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return 1;
    }
  const float *host_pcm = staged && !samples16 ? samples : nullptr;
  /* Device PCM of several chunks, one key, no speed detection: the approx search of chunk k + 1 is queued (on a second stream, into
   * the other approx slot) before chunk k's candidate selection, refine and decode, so that the GPU has work while the host makes
   * those decisions.  Every decision still runs per chunk, in the same order, on the same values.  Host PCM keeps the serial loop:
   * there the upload, not the GPU, sets the pace. */
  const bool speed = Params::detect_speed || Params::detect_speed_patient || Params::try_speed > 0;
  const int pipe_key = (!eof && key_list.size() == 1 && !speed && !Params::test_no_sync && !staged) ? Engine::key_slot (key_list[0]) : -1;
  auto enqueue_approx = [&] (size_t c0, size_t c1, int approx_slot)
    {
      if (awm_pcm_bind (ctx, pcm + c0 * n_channels, c1 - c0, n_channels, 0, 0)
          || awm_sync_approx_enqueue (ctx, approx_slot, pipe_key, AWM_MODE_BLOCK, 0, (c1 - c0) * n_channels, Params::water_delta))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return false;
        }
      return true;
    };
  if (pipe_key >= 0 && !enqueue_approx (start, end, 0))
    return 1;
  std::unique_ptr<void, void (*) (void *)> aligned_chunk (nullptr, [] (void *p) { awm_device_free (Engine::ctx(), p); });
  for (;;)
    {
      string debug_sync;
      const int chunk = int (chunks.size());
      if (!eof && pipe_key >= 0)
        {
          const size_t nstart = end - overlap, nend = min (nstart + max_frames, n_frames);
          if (!enqueue_approx (nstart, nend, (chunk + 1) & 1))
            return 1;
          if (getenv ("AWM_TRACE"))
            fprintf (stderr, "[trace] chunk %d: approx search of chunk %d queued ahead\n", chunk, chunk + 1);
        }
      if (staged && awm_pcm_stage_wait (ctx, end))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return 1;
        }
      const float *chunk_pcm = pcm + start * n_channels;
      /* The sync search reads stereo PCM at a 16-byte aligned address by bulk copies and at any other by global loads, whose sums
       * can differ in the last bits.  A staged chunk that starts at an odd frame (an odd chunk step, as with --frames-per-bit 3) is
       * searched from an aligned copy, so that a host `get` finds what GetStream finds, which searches every chunk from the start
       * of its own buffer. */
      if (staged && n_channels == 2 && (reinterpret_cast<uintptr_t> (chunk_pcm) & 15))
        {
          void *buf = nullptr;
          if (!aligned_chunk && awm_device_alloc (ctx, max_frames * n_channels * sizeof (float), &buf))
            {
              error ("audiowmark: %s\n", awm_last_error (ctx));
              return 1;
            }
          if (buf)
            aligned_chunk.reset (buf);
          if (awm_copy (ctx, aligned_chunk.get(), chunk_pcm, (end - start) * n_channels * sizeof (float)))
            {
              error ("audiowmark: %s\n", awm_last_error (ctx));
              return 1;
            }
          chunk_pcm = static_cast<const float *> (aligned_chunk.get());
        }
      if (decode_chunk (pending, chunk, debug_sync, key_list, chunk_pcm, host_pcm ? host_pcm + start * n_channels : nullptr, end - start,
                        n_channels, sample_rate, chunk == 0, print_speed_results, pipe_key >= 0 ? chunk & 1 : -1))
        return 1;
      chunks.push_back ({ start, end - start, time_offset });
      debug_syncs.push_back (debug_sync);
      if (eof)
        break;
      time_offset += double (end - start - overlap) / sample_rate;
      start = end - overlap;
      const size_t new_end = min (start + max_frames, n_frames);
      eof = (new_end - start) < max_frames;
      end = new_end;
    }
  return merge_chunk_results (pending, chunks, debug_syncs, key_list, result_set);
}

static int
report (ResultSet& result_set, size_t time_length, const vector<int>& orig_bits)
{
  if (!Params::json_output.empty())
    result_set.print_json (time_length, Params::json_output);
  if (Params::json_output != "-")
    result_set.print();
  if (!orig_bits.empty())
    {
      const int match_count = result_set.print_match_count (orig_bits);
      result_set.print_debug_sync();
      if (Params::expect_matches >= 0)
        {
          printf ("expect_matches %d\n", Params::expect_matches);
          if (match_count != Params::expect_matches)
            return 1;
        }
      else if (!match_count)
        return 1;
    }
  return 0;
}

int
get_watermark (const vector<Key>& key_list, const string& infile, const string& orig_pattern)
{
  vector<int> orig_bitvec;
  if (!orig_pattern.empty())
    {
      orig_bitvec = parse_payload (orig_pattern);
      if (orig_bitvec.empty())
        return 1;
    }
  Error err;
  std::unique_ptr<AudioInputStream> in = AudioInputStream::create (infile, err);
  if (err)
    {
      error ("audiowmark: error loading %s: %s\n", infile.c_str(), err.message());
      return 1;
    }
  /* --test-truncate: the first sample_rate * seconds frames */
  const size_t limit = Params::test_truncate ? size_t (in->sample_rate()) * Params::test_truncate : ~size_t (0);
  GetStream stream (key_list, in->n_channels(), in->sample_rate(), !orig_bitvec.empty(),
                    in->n_frames() == AudioInputStream::N_FRAMES_UNKNOWN ? limit : min (in->n_frames(), limit));
  if (!stream.ok())
    return 1;
  vector<float> piece;
  for (size_t frames = 0; frames < limit; )
    {
      err = in->read_frames (piece, min<size_t> (limit - frames, 1 << 18));
      if (err)
        {
          error ("audiowmark: error loading %s: %s\n", infile.c_str(), err.message());
          return 1;
        }
      if (piece.empty())
        break;
      const size_t n = piece.size() / in->n_channels();
      if (stream.feed (piece.data(), n))
        return 1;
      frames += n;
    }
  ResultSet result_set;
  size_t mark_rate_frames = 0;
  if (stream.finish (result_set, &mark_rate_frames))
    return 1;
  const size_t time_length = lrint (mark_rate_frames / double (Params::mark_sample_rate));
  return report (result_set, time_length, orig_bitvec);
}
