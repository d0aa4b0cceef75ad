// awm_add.cc -- `audiowmark add`: add_stream_watermark / add_watermark (reference src/wmadd.cc:448-657).
// The reference pulls 1024-frame blocks through WatermarkGen / WatermarkSynth / Limiter on one CPU
// thread; here the whole stream is handed to awm_embed, which reproduces the same stream semantics
// (frame numbering from 2*fpb - 250, zero padding of the tail, limiter on the zero-extended signal).
#include "awm_wm.hh"
#include "awm_speed.hh"
#include "awm_engine.hh"
#include "awm_tables.hh"
#include "awm_util.hh"

#include <math.h>
#include <functional>
#include <map>

using std::string;
using std::vector;

/* number of WatermarkGen::run calls the reference loop makes (src/wmadd.cc:520-589): zero frames are fed
 * after EOF until every input frame has been written; synth delays one frame (src/wmadd.cc:240-249) and the
 * limiter keeps one block of look-ahead (src/limiter.cc:53-58).  Only needed for the "Data Blocks" line. */
static size_t
gen_runs (size_t n_frames, bool limiter_on, size_t limiter_block)
{
  const size_t N = Params::frame_size;
  if (n_frames == 0)
    return 0;
  if (!limiter_on)
    return 1 + (n_frames + N - 1) / N;
  const size_t need = ((n_frames + limiter_block - 1) / limiter_block + 1) * limiter_block;
  return 1 + (need + N - 1) / N;
}

/* Frame counts of the add loop when the input is not at the watermark rate (src/wmadd.cc:520-589 with a
 * WatermarkResampler, :353-430).  Every iteration pushes one 1024-frame block (zero frames after EOF) into the input
 * resampler; whole 1024-frames at the watermark rate go through WatermarkGen::run and the output resampler; whatever
 * that has delivered is mixed, counted for --snr and handed to the limiter, which holds back until two complete blocks
 * are buffered (src/limiter.cc:53-58).  The loop stops at the first short read with everything written.
 *   n_emit: frames that went through the mixer;  gen_runs: WatermarkGen::run calls */
void
resampled_add_plan (size_t n_frames, int sample_rate, bool limiter_on, size_t limiter_block, size_t& n_emit, size_t& gen_runs_out)
{
  const size_t N = Params::frame_size;
  const double r_in = double (Params::mark_sample_rate) / sample_rate, r_out = double (sample_rate) / Params::mark_sample_rate;
  /* the state after `iteration` blocks were pushed; released (frames the limiter has let out) never decreases */
  auto state = [&] (size_t iteration, size_t& emit, size_t& runs)
    {
      runs = resample_stream_available (N * iteration, r_in) / N;
      emit = runs ? resample_stream_available (runs * N, r_out) : 0;
      if (!limiter_on)
        return emit;
      return emit / limiter_block >= 2 ? (emit / limiter_block - 1) * limiter_block : 0;
    };
  n_emit = gen_runs_out = 0;
  if (n_frames == 0)
    return;
  /* the loop stops after the first iteration k that has read all input (N k >= n_frames) and released all of it: the first k
   * at or after ceil (n_frames / N) with released (k) >= n_frames, found by doubling the step and then bisecting */
  size_t lo = (n_frames + N - 1) / N;
  if (state (lo, n_emit, gen_runs_out) < n_frames)
    {
      size_t step = 1, hi;
      while (state (lo + step, n_emit, gen_runs_out) < n_frames)
        {
          lo += step;
          step *= 2;
        }
      hi = lo + step;                 /* released (lo) < n_frames <= released (hi) */
      while (hi - lo > 1)
        {
          const size_t mid = lo + (hi - lo) / 2;
          if (state (mid, n_emit, gen_runs_out) < n_frames)
            lo = mid;
          else
            hi = mid;
        }
      state (hi, n_emit, gen_runs_out);
    }
}

/* the "Data Blocks" and --snr values of an add loop that made `runs` WatermarkGen::run calls with the given --snr sums */
static AddStats
add_stats (size_t runs, double snr_delta, double snr_signal)
{
  const size_t fpb = frames_per_block(), f0 = 2 * fpb - Params::frames_pad_start;
  const int blocks = int ((f0 + runs) / fpb - f0 / fpb);
  AddStats s;
  s.data_blocks = std::max (blocks - 1, 0);         // the first (partial B) block is padding
  s.snr_db = snr_delta > 0 ? 10 * log10 (snr_signal / snr_delta) : INFINITY;
  return s;
}

static void
info_format (const string& label, const RawFormat& format)
{
  const char *e = format.encoding() == Encoding::SIGNED ? "signed" : format.encoding() == Encoding::UNSIGNED ? "unsigned" : "float";
  info ("%-13s %d Hz, %d Channels, %d Bit (%s %s-endian)\n", (label + ":").c_str(), format.sample_rate(), format.n_channels(),
        format.bit_depth(), e, format.endian() == RawFormat::LITTLE ? "little" : "big");
}

int
add_watermark_buffer (const Key& key, const float *in, float *out, size_t n_frames, int n_channels, int sample_rate,
                      const string& bits, AddStats *stats, uint64_t first_frame_number)
{
  const vector<int> bitvec = parse_payload (bits);
  if (bitvec.empty())
    return 1;
  if (sample_rate != Params::mark_sample_rate)
    {
      if (first_frame_number)
        {
          error ("audiowmark: sharded embedding is only available at %d Hz\n", Params::mark_sample_rate);
          return 1;
        }
      /* a batch of one item: the embed at other rates exists in batched form only */
      const awm_batch_item item = { 0, n_frames, n_channels };
      vector<AddStats> item_stats;
      if (add_watermark_batch ({ key }, false, in, out, false, n_frames * size_t (n_channels), &item, 1, { bits }, sample_rate, &sample_rate,
                               nullptr, 0, stats ? &item_stats : nullptr))
        return 1;
      if (stats)
        *stats = item_stats[0];
      return 0;
    }
  awm_ctx *ctx = Engine::ctx();
  if (!ctx || !Engine::set_embed_tables (key, bitvec))
    return 1;
  const int limiter_block = Params::test_no_limiter ? 0 : int (sample_rate * int (Params::limiter_block_size_ms) / 1000);
  double snr_power[2] = { 0, 0 };
  if (awm_embed (ctx, in, out, n_frames, n_channels, first_frame_number, Params::frames_pad_start, Params::water_delta,
                 limiter_block, Params::limiter_ceiling, (Params::snr || stats) ? snr_power : nullptr))
    {
      error ("audiowmark: embedding failed: %s\n", awm_last_error (ctx));
      return 1;
    }
  if (stats)
    *stats = add_stats (gen_runs (n_frames, !Params::test_no_limiter, sample_rate * int (Params::limiter_block_size_ms) / 1000), snr_power[0], snr_power[1]);
  return 0;
}

/* `add` between two 16 bit PCM buffers in host memory (44.1 kHz): the int <-> float conversions of SFInputStream / SFOutputStream
 * run on the device (awm_embed_s16), only 2 + 2 bytes per sample cross PCIe */
int
add_watermark_buffer_s16 (const Key& key, const int16_t *in, int16_t *out, size_t n_frames, int n_channels, int sample_rate,
                          const string& bits, AddStats *stats, uint64_t first_frame_number)
{
  const vector<int> bitvec = parse_payload (bits);
  if (bitvec.empty())
    return 1;
  if (sample_rate != Params::mark_sample_rate)
    {
      error ("audiowmark: 16 bit buffers are only accepted at %d Hz (use the float entry point for other rates)\n", Params::mark_sample_rate);
      return 1;
    }
  awm_ctx *ctx = Engine::ctx();
  if (!ctx || !Engine::set_embed_tables (key, bitvec))
    return 1;
  const int limiter_block = Params::test_no_limiter ? 0 : int (sample_rate * int (Params::limiter_block_size_ms) / 1000);
  double snr_power[2] = { 0, 0 };
  if (awm_embed_s16 (ctx, in, out, n_frames, n_channels, first_frame_number, Params::frames_pad_start, Params::water_delta,
                     limiter_block, Params::limiter_ceiling, (Params::snr || stats) ? snr_power : nullptr))
    {
      error ("audiowmark: embedding failed: %s\n", awm_last_error (ctx));
      return 1;
    }
  if (stats)
    *stats = add_stats (gen_runs (n_frames, !Params::test_no_limiter, sample_rate * int (Params::limiter_block_size_ms) / 1000), snr_power[0], snr_power[1]);
  return 0;
}

int
add_watermark_batch (const vector<Key>& keys, bool per_item_keys, const void *in, void *out, bool s16, size_t n_values, const awm_batch_item *items,
                     size_t n_items, const vector<string>& bits, int sample_rate, const int *sample_rates, const uint64_t *zero_frames,
                     size_t scratch_bytes, vector<AddStats> *stats)
{
  const int mark = Params::mark_sample_rate;
  if (per_item_keys && (keys.size() != n_items || bits.size() != n_items))
    {
      error ("audiowmark: %zu items but %zu keys and %zu payloads\n", n_items, keys.size(), bits.size());
      return 2;
    }
  /* the distinct keys in order of first use; item i uses key_index[i] of them (0 with one key) */
  vector<uint32_t> key_index (n_items);
  vector<vector<unsigned char>> distinct;
  std::map<vector<unsigned char>, uint32_t> seen;
  for (size_t i = 0; i < keys.size(); i++)
    {
      const vector<unsigned char> kb (keys[i].aes_key(), keys[i].aes_key() + Key::SIZE);
      auto it = seen.find (kb);
      if (it == seen.end())
        {
          it = seen.emplace (kb, uint32_t (distinct.size())).first;
          distinct.push_back (kb);
        }
      if (per_item_keys)
        key_index[i] = it->second;
    }
  /* the validator of the C call the input goes to (see awm_wm.hh), all before any GPU work */
  char why[256];
  auto refuse = [&] { error ("audiowmark: %s\n", why); return 2; };
  if (per_item_keys)
    {
      if (awm_batch_keys_validate (items, n_items, n_values, sample_rates, nullptr, zero_frames, key_index.data(), distinct.size(), mark, why,
                                   sizeof (why)))
        return refuse();
    }
  else if (sample_rates)
    {
      if (zero_frames ? awm_batch_rates_offsets_validate (items, n_items, n_values, sample_rates, nullptr, zero_frames, mark, why, sizeof (why))
                      : awm_batch_rates_validate (items, n_items, n_values, sample_rates, nullptr, mark, why, sizeof (why)))
        return refuse();
    }
  else if (zero_frames && awm_batch_offsets_validate (items, n_items, n_values, zero_frames, sample_rate, mark, why, sizeof (why)))
    return refuse();                             // names an offset at another rate before the rate itself
  if (!sample_rates && sample_rate != mark)
    {
      error ("audiowmark: batched embedding is only available at %d Hz\n", mark);
      return 2;
    }
  if (!per_item_keys && !sample_rates && awm_batch_validate (items, n_items, n_values, why, sizeof (why)))
    return refuse();
  /* every payload encoded with its own key's bit order, computed once per distinct key */
  const size_t n_coded = code_size (ConvBlockType::a, Params::payload_size);
  vector<vector<unsigned>> orders;
  for (const auto& kb : distinct)
    {
      Key k;
      k.set_key (kb.data(), "");
      orders.push_back (bit_order (k, n_coded));
    }
  vector<uint8_t> coded;
  for (size_t i = 0; i < n_items; i++)
    {
      const vector<int> bitvec = parse_payload (bits[i]);
      if (bitvec.empty())
        return 2;
      const vector<uint8_t> c = gen_coded_bits (orders[key_index[i]], bitvec);
      coded.insert (coded.end(), c.begin(), c.end());
    }
  /* per item what add_watermark_buffer computes for its whole stream (silent prefix included, as add_watermark_windowed counts):
   * frames through the mixer (other rates; counted from the item's first frame) and WatermarkGen::run calls */
  vector<uint64_t> n_emit (n_items);
  vector<size_t> runs (n_items);
  for (size_t i = 0; i < n_items; i++)
    {
      const int rate = sample_rates ? sample_rates[i] : mark;
      const size_t block = size_t (rate) * size_t (Params::limiter_block_size_ms) / 1000;
      const size_t z = zero_frames ? zero_frames[i] : 0, n_stream = z + items[i].n_frames;
      if (rate == mark)
        {
          runs[i] = gen_runs (n_stream, !Params::test_no_limiter, block);
          continue;
        }
      size_t emit = 0;
      resampled_add_plan (n_stream, rate, !Params::test_no_limiter, block, emit, runs[i]);
      n_emit[i] = std::max<uint64_t> (emit, n_stream) - z;
    }
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  if (per_item_keys)
    {
      /* a call without items still needs a role set: that of the zero key, which no item reads */
      vector<unsigned char> keys16 (std::max<size_t> (distinct.size(), 1) * Key::SIZE, 0);
      for (size_t k = 0; k < distinct.size(); k++)
        std::copy (distinct[k].begin(), distinct[k].end(), keys16.begin() + k * Key::SIZE);
      const awm_role_layout layout = embed_role_layout();
      if (awm_set_embed_roles_keys (ctx, keys16.data(), keys16.size() / Key::SIZE, &layout))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return 1;
        }
    }
  else if (!Engine::set_embed_roles (keys[0]))
    return 1;
  vector<double> snr_power (2 * n_items);
  double *snr = (Params::snr || stats) ? snr_power.data() : nullptr;
  const int limiter_ms = Params::test_no_limiter ? 0 : int (Params::limiter_block_size_ms);
  const int limiter_block = limiter_ms * mark / 1000;
  const int is_s16 = s16 ? 1 : 0, pad = Params::frames_pad_start;
  const double wd = Params::water_delta;
  const float ceiling = Params::limiter_ceiling;
  int rc;
  if (per_item_keys)
    rc = awm_embed_batch_keys (ctx, in, out, is_s16, n_values, items, n_items, coded.data(), sample_rates, sample_rates ? n_emit.data() : nullptr,
                               zero_frames, key_index.data(), mark, pad, wd, limiter_ms, ceiling, snr, scratch_bytes);
  else if (sample_rates && zero_frames)
    rc = awm_embed_batch_rates_offsets (ctx, in, out, is_s16, n_values, items, n_items, coded.data(), sample_rates, n_emit.data(), zero_frames, mark,
                                        pad, wd, limiter_ms, ceiling, snr, scratch_bytes);
  else if (sample_rates)
    rc = awm_embed_batch_rates (ctx, in, out, is_s16, n_values, items, n_items, coded.data(), sample_rates, n_emit.data(), mark, pad, wd, limiter_ms,
                                ceiling, snr, scratch_bytes);
  else if (zero_frames)
    rc = awm_embed_batch_offsets (ctx, in, out, is_s16, n_values, items, n_items, zero_frames, coded.data(), pad, wd, limiter_block, ceiling, snr);
  else
    rc = awm_embed_batch (ctx, in, out, is_s16, n_values, items, n_items, coded.data(), pad, wd, limiter_block, ceiling, snr);
  if (rc)
    {
      error ("audiowmark: batched embedding failed: %s\n", awm_last_error (ctx));
      return 1;
    }
  if (stats)
    {
      stats->resize (n_items);
      for (size_t i = 0; i < n_items; i++)
        (*stats)[i] = add_stats (runs[i], snr_power[2 * i], snr_power[2 * i + 1]);
    }
  return 0;
}

/* Part of the stream a window has to embed so that [own_start, own_end) comes out exactly as in a run over the whole stream:
 * one 1024-frame before the first limiter block that influences the owned range (synthesis-window tail of the frame before) and
 * everything up to the end of the limiter block after the last owned one (the gain ramp looks one block ahead), rounded to whole
 * 1024-frames.  n_total = ~0 while the end of the stream is not known. */
static void
window_range (size_t own_start, size_t own_end, size_t n_total, size_t limiter_block, size_t& ext_start, size_t& ext_end)
{
  const size_t N = Params::frame_size;
  if (own_start == 0)
    ext_start = 0;
  else
    {
      const size_t b = own_start / limiter_block;                   // first owned limiter block
      const size_t lo = (b ? b - 1 : 0) * limiter_block;            // the block before it must be complete
      ext_start = lo / N * N >= N ? lo / N * N - N : 0;
    }
  if (own_end >= n_total)
    ext_end = n_total;
  else
    {
      const size_t hi = ((own_end - 1) / limiter_block + 2) * limiter_block;
      ext_end = std::min (ext_start + (hi - ext_start + N - 1) / N * N + N, n_total);
    }
}

int
add_window_range (size_t own_first, size_t own_end, size_t n_total, int sample_rate, size_t& ext_first, size_t& ext_end)
{
  if (own_first >= own_end || own_end > n_total)
    {
      error ("audiowmark: owned range [%zu, %zu) is empty or ends past the %zu frames of the stream\n", own_first, own_end, n_total);
      return 1;
    }
  if (sample_rate == Params::mark_sample_rate)
    {
      window_range (own_first, own_end, n_total, size_t (sample_rate) * size_t (Params::limiter_block_size_ms) / 1000, ext_first, ext_end);
      return 0;
    }
  uint64_t e0 = 0, e1 = 0;
  if (awm_window_range_rates (own_first, own_end, n_total, sample_rate, Params::mark_sample_rate, int (Params::limiter_block_size_ms), 16, &e0, &e1))
    {
      error ("audiowmark: sample rate %d is outside the resampler's range\n", sample_rate);
      return 1;
    }
  ext_first = e0;
  ext_end = e1;
  return 0;
}

int
add_watermark_window (const Key& key, const string& bits, const float *in, float *out, size_t ext_first, size_t ext_end, size_t n_total,
                      int n_channels, int sample_rate, size_t own_first, size_t own_end, double *snr_power)
{
  const vector<int> bitvec = parse_payload (bits);
  if (bitvec.empty())
    return 1;
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  const int mark = Params::mark_sample_rate;
  /* the --snr sums count the watermark signal before the limiter over the owned frames; a window that ends the stream also takes the
   * frames the add loop emits after the end of the input */
  const uint64_t snr_first = own_first - ext_first, snr_last = own_end >= n_total ? ~uint64_t (0) : own_end - ext_first;
  int rc;
  if (sample_rate == mark)
    {
      if (!Engine::set_embed_tables (key, bitvec))
        return 1;
      const int limiter_block = Params::test_no_limiter ? 0 : sample_rate * int (Params::limiter_block_size_ms) / 1000;
      rc = awm_embed_window (ctx, in, out, ext_end - ext_first, n_channels, ext_first / Params::frame_size, Params::frames_pad_start, Params::water_delta,
                             limiter_block, Params::limiter_ceiling, snr_first, snr_last, snr_power);
    }
  else
    {
      if (!Engine::set_embed_roles (key))
        return 1;
      /* a window that ends the stream emits what the whole stream's add loop emits after its first frame */
      uint64_t n_emit = ext_end - ext_first;
      if (ext_end >= n_total)
        {
          size_t emit = 0, runs = 0;
          resampled_add_plan (n_total, sample_rate, !Params::test_no_limiter, size_t (sample_rate) * size_t (Params::limiter_block_size_ms) / 1000, emit, runs);
          n_emit = std::max (emit, n_total) - ext_first;
        }
      const vector<uint8_t> coded = gen_coded_bits (key, bitvec);
      rc = awm_embed_window_rates (ctx, in, out, ext_end - ext_first, n_channels, coded.data(), sample_rate, mark, ext_first, n_emit,
                                   Params::frames_pad_start, Params::water_delta, Params::test_no_limiter ? 0 : int (Params::limiter_block_size_ms),
                                   Params::limiter_ceiling, snr_first, snr_last, snr_power);
    }
  if (rc)
    {
      error ("audiowmark: embedding failed: %s\n", awm_last_error (ctx));
      return 1;
    }
  return 0;
}

/* add_stream_watermark's loop (src/wmadd.cc:504-589) with bounded memory: the stream is embedded window by window through
 * add_watermark_window, each window with the halo add_window_range asks for, so the owned part of every window is bit identical
 * to a run over the whole stream.  Reads block only until one window and its look-ahead (about two limiter blocks) are buffered:
 * a pipe gets its first output after ~100 s of input, not at EOF.
 * zero_frames: the input continues a stream that began zero_frames earlier with silence (HLS segments, src/wmadd.cc:504-519):
 * positions, table rows, resamplers and limiter blocks count from there, nothing is written for the silent part.
 * window_frames = 0: default window (4096 1024-frames = 95 s at 44.1 kHz); tests pass small windows. */
int
add_watermark_windowed (const Key& key, const std::function<Error (vector<float>&, size_t)>& read, const std::function<Error (const vector<float>&)>& write,
                        int n_channels, int sample_rate, const string& bits, size_t zero_frames, size_t window_frames, AddStats *stats, size_t *frames_written)
{
  const size_t N = Params::frame_size, C = size_t (n_channels);
  const size_t L = size_t (sample_rate) * size_t (Params::limiter_block_size_ms) / 1000;
  const size_t W = (window_frames ? window_frames : 4096) * N;
  const size_t unknown = ~size_t (0);
  if (parse_payload (bits).empty())
    return 1;
  vector<float> pending;                         // stream positions [p0, p1), interleaved
  size_t p0 = 0, p1 = 0, own_start = zero_frames, written = 0;
  double snr_delta = 0, snr_signal = 0;
  {
    /* the silent prefix is never materialised beyond what the first window's halo reaches into */
    size_t e0, e1;
    if (add_window_range (own_start, own_start + 1, unknown, sample_rate, e0, e1))
      return 1;
    p0 = e0;
    p1 = zero_frames;
    pending.assign ((p1 - p0) * C, 0.f);
  }
  bool eof = false;
  vector<float> block, out;
  while (!eof || own_start < p1)
    {
      size_t e0, e1;
      if (add_window_range (own_start, own_start + W, unknown, sample_rate, e0, e1))
        return 1;
      while (!eof && p1 < e1)                    // the window and its look-ahead
        {
          const Error err = read (block, std::min<size_t> (e1 - p1, 1 << 16));
          if (err)
            {
              error ("audiowmark: input stream read failed: %s\n", err.message());
              return 1;
            }
          if (block.empty())
            eof = true;
          pending.insert (pending.end(), block.begin(), block.end());
          p1 += block.size() / C;
        }
      const size_t n_total = eof ? p1 : unknown;
      const size_t own_end = eof ? p1 : own_start + W;
      if (own_end <= own_start)
        break;
      if (add_window_range (own_start, own_end, n_total, sample_rate, e0, e1))
        return 1;
      out.resize ((e1 - e0) * C);
      double snr_power[2] = { 0, 0 };
      if (add_watermark_window (key, bits, pending.data() + (e0 - p0) * C, out.data(), e0, e1, n_total, n_channels, sample_rate, own_start, own_end,
                                (Params::snr || stats) ? snr_power : nullptr))
        return 1;
      snr_delta += snr_power[0];
      snr_signal += snr_power[1];
      const float *o = out.data() + (own_start - e0) * C;
      const Error err = write (vector<float> (o, o + (own_end - own_start) * C));
      if (err)
        {
          error ("audiowmark output write failed: %s\n", err.message());
          return 1;
        }
      written += own_end - own_start;
      own_start = own_end;
      if (eof)
        break;
      if (add_window_range (own_start, own_start + 1, unknown, sample_rate, e0, e1))   // what the next window still needs of the buffer
        return 1;
      pending.erase (pending.begin(), pending.begin() + (e0 - p0) * C);
      p0 = e0;
    }
  if (frames_written)
    *frames_written = written;
  if (stats)
    {
      size_t emit = 0, runs = gen_runs (p1, !Params::test_no_limiter, L);
      if (sample_rate != Params::mark_sample_rate)
        resampled_add_plan (p1, sample_rate, !Params::test_no_limiter, L, emit, runs);
      *stats = add_stats (runs, snr_delta, snr_signal);
    }
  return 0;
}

int
add_stream_watermark (const Key& key, AudioInputStream *in_stream, AudioOutputStream *out_stream, const string& bits, size_t zero_frames)
{
  auto bitvec = parse_payload (bits);
  if (bitvec.empty())
    return 1;
  if (in_stream->sample_rate() != out_stream->sample_rate())
    {
      error ("audiowmark: input sample rate (%d) and output sample rate (%d) don't match\n", in_stream->sample_rate(), out_stream->sample_rate());
      return 1;
    }
  if (in_stream->n_channels() != out_stream->n_channels())
    {
      error ("audiowmark: input channels (%d) and output channels (%d) don't match\n", in_stream->n_channels(), out_stream->n_channels());
      return 1;
    }
  info ("Message:      %s\n", bit_vec_to_str (bitvec).c_str());
  info ("Strength:     %.6g\n\n", Params::water_delta * 1000);
  if (in_stream->n_frames() == AudioInputStream::N_FRAMES_UNKNOWN)
    info ("Time:         unknown\n");
  else
    {
      const size_t orig_seconds = in_stream->n_frames() / in_stream->sample_rate();
      info ("Time:         %zd:%02zd\n", orig_seconds / 60, orig_seconds % 60);
    }
  info ("Sample Rate:  %d\n", in_stream->sample_rate());
  info ("Channels:     %d\n", in_stream->n_channels());

  AddStats stats;
  size_t total_output_frames = 0;
  Error err;
  auto read = [&] (vector<float>& samples, size_t count) { return in_stream->read_frames (samples, count); };
  auto write = [&] (const vector<float>& samples) { return out_stream->write_frames (samples); };
  if (add_watermark_windowed (key, read, write, in_stream->n_channels(), in_stream->sample_rate(), bits, zero_frames, 0, &stats, &total_output_frames))
    return 1;
  if (Params::snr)
    info ("SNR:          %f dB\n", stats.snr_db);
  info ("Data Blocks:  %d\n", stats.data_blocks);

  if (in_stream->n_frames() != AudioInputStream::N_FRAMES_UNKNOWN && total_output_frames != in_stream->n_frames())
    {
      auto msg = string_printf ("unexpected EOF; input frames (%zd) != output frames (%zd)", in_stream->n_frames(), total_output_frames);
      if (Params::strict)
        {
          error ("audiowmark: error: %s\n", msg.c_str());
          return 1;
        }
      warning ("audiowmark: warning: %s\n", msg.c_str());
    }
  err = out_stream->close();
  if (err)
    {
      error ("audiowmark: closing output stream failed: %s\n", err.message());
      return 1;
    }
  return 0;
}

int
add_watermark (const Key& key, const string& infile, const string& outfile, const string& bits)
{
  Error err;
  std::unique_ptr<AudioInputStream> in_stream = AudioInputStream::create (infile, err);
  if (err)
    {
      error ("audiowmark: error opening %s: %s\n", infile.c_str(), err.message());
      return 1;
    }
  /* output keeps the input's depth / encoding, but at least 16 bit signed */
  int out_bit_depth = in_stream->bit_depth();
  Encoding out_encoding = in_stream->encoding();
  if (in_stream->bit_depth() < 16)
    {
      out_bit_depth = 16;
      out_encoding = Encoding::SIGNED;
    }
  std::unique_ptr<AudioOutputStream> out_stream = AudioOutputStream::create (outfile, in_stream->n_channels(), in_stream->sample_rate(),
                                                                           out_bit_depth, out_encoding, in_stream->n_frames(), err);
  if (err)
    {
      error ("audiowmark: error writing to %s: %s\n", outfile.c_str(), err.message());
      return 1;
    }
  info ("Input:        %s\n", Params::input_label.size() ? Params::input_label.c_str() : infile.c_str());
  if (Params::input_format == Format::RAW)
    info_format ("Raw Input", Params::raw_input_format);
  info ("Output:       %s\n", Params::output_label.size() ? Params::output_label.c_str() : outfile.c_str());
  if (Params::output_format == Format::RAW)
    info_format ("Raw Output", Params::raw_output_format);
  return add_stream_watermark (key, in_stream.get(), out_stream.get(), bits, 0);
}
