// awm_hostapi.cc -- plain C entry points over the host-side C++ (tables, add, get) so that the parity
// tests and bench.py can drive exactly what the CLI runs.  Table functions are pure host code (no GPU).
#include "awm_results.hh"
#include "awm_balanced.hh"
#include "awm_speed.hh"
#include "awm_engine.hh"
#include "awm_tables.hh"
#include "awm_util.hh"

#include <algorithm>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static Key
make_key (const unsigned char *key16, const char *name)
{
  Key k;
  k.set_key (key16, name ? name : "");
  return k;
}

extern "C" {

void
awmh_set_params (double water_delta, int frames_per_bit, int mix, int hard, double sync_threshold2, int n_best,
                 double chunk_size_min, int test_no_limiter, int test_no_sync, int gpu_device, int quiet)
{
  Params::water_delta = water_delta;
  Params::frames_per_bit = frames_per_bit;
  Params::mix = mix != 0;
  Params::hard = hard != 0;
  Params::sync_threshold2 = sync_threshold2;
  Params::get_n_best = n_best;
  Params::get_chunk_size = chunk_size_min;
  Params::test_no_limiter = test_no_limiter != 0;
  Params::test_no_sync = test_no_sync != 0;
  Params::gpu_device = gpu_device;
  set_log_level (quiet ? Log::WARNING : Log::INFO);
}

/* --short <bits> (src/audiowmark.cc:665-674); bits = 0 returns to the 128 bit payload.  returns the block code length or -1 */
int
awmh_set_short_payload (int bits)
{
  if (bits == 0)
    {
      Params::payload_short = false;
      Params::payload_size = 128;
      return 0;
    }
  const size_t n = short_code_init (bits);
  if (!n)
    return -1;
  Params::payload_size = bits;
  Params::payload_short = true;
  return int (n);
}

/* --detect-speed / --detect-speed-patient / --try-speed / --test-speed of `audiowmark get` (src/audiowmark.cc:831-854) */
void
awmh_set_speed_params (int detect_speed, int detect_speed_patient, double try_speed, double test_speed)
{
  Params::detect_speed = detect_speed != 0;
  Params::detect_speed_patient = detect_speed_patient != 0;
  Params::try_speed = try_speed;
  Params::test_speed = test_speed;
}

/* detect_speed (src/wmspeed.cc:622-781) for one key on one chunk: best speed / quality as the reference would print
 * them, *accepted = 1 if the speed would be used for a second decode */
int
awmh_detect_speed (const unsigned char *key16, const float *pcm, size_t n_frames, int n_channels, int sample_rate,
                   double *speed, double *quality, int *accepted)
{
  DetectSpeedInfo info;
  const std::vector<DetectSpeedResult> r = detect_speed ({ make_key (key16, "") }, pcm, n_frames, n_channels, sample_rate, false, &info);
  if (!info.valid)
    return 1;
  if (speed)
    *speed = info.speed;
  if (quality)
    *quality = info.quality;
  if (accepted)
    *accepted = r.empty() ? 0 : 1;
  return 0;
}

/* resample_ratio (src/resample.cc:127-131) / the streaming frame count of BufferedResamplerImpl */
int
awmh_resample (const float *in, size_t n_in, int n_channels, double ratio, float *out, size_t n_out)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  if (awm_resample (ctx, in, n_in, n_channels, ratio, 16, out, n_out))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return 1;
    }
  return 0;
}

uint64_t awmh_resample_stream_frames (uint64_t n_in, double ratio) { return resample_stream_frames (n_in, ratio); }
uint64_t awmh_resample_stream_available (uint64_t fed, double ratio) { return resample_stream_available (fed, ratio); }

void
awmh_resampled_add_plan (uint64_t n_frames, int sample_rate, uint64_t *n_emit, uint64_t *gen_runs)
{
  size_t e = 0, r = 0;
  resampled_add_plan (n_frames, sample_rate, !Params::test_no_limiter, sample_rate * int (Params::limiter_block_size_ms) / 1000, e, r);
  *n_emit = e;
  *gen_runs = r;
}

int awmh_frames_per_block() { return int (frames_per_block()); }
int awmh_n_coded_bits()     { return int (code_size (ConvBlockType::a, Params::payload_size)); }

int
awmh_random_u64 (const unsigned char *key16, uint64_t seed, int stream, uint64_t *out, int n)
{
  Random r (make_key (key16, ""), seed, Random::Stream (stream));
  for (int i = 0; i < n; i++)
    out[i] = r();
  return 0;
}

int
awmh_gen_noise (const unsigned char *key16, float *out, size_t n_values)
{
  Random r (make_key (key16, ""), 0, Random::Stream::data_up_down);
  for (size_t i = 0; i < n_values; i++)
    out[i] = r.random_double() * 2 - 1;
  return 0;
}

int
awmh_sync_table (const unsigned char *key16, int mode, awm_sync_entry *out, int max_entries, int *bit_offsets /* [sync_bits + 1] */)
{
  const SyncTable t = gen_sync_table (make_key (key16, ""), mode);
  if (int (t.entries.size()) > max_entries)
    return -1;
  memcpy (out, t.entries.data(), t.entries.size() * sizeof (awm_sync_entry));
  memcpy (bit_offsets, t.bit_offsets.data(), t.bit_offsets.size() * sizeof (int));
  return int (t.entries.size());
}

int
awmh_mix_table (const unsigned char *key16, awm_mix_entry *out, int max_entries, uint16_t *order, int max_order)
{
  const Key key = make_key (key16, "");
  const std::vector<MixEntry> mix = gen_mix_entries (key);
  const std::vector<unsigned> ord = bit_order (key, code_size (ConvBlockType::a, Params::payload_size));
  if (int (mix.size()) > max_entries || int (ord.size()) > max_order)
    return -1;
  for (size_t i = 0; i < mix.size(); i++)
    {
      out[i].frame = mix[i].frame;
      out[i].up = mix[i].up;
      out[i].down = mix[i].down;
    }
  for (size_t i = 0; i < ord.size(); i++)
    order[i] = ord[i];
  return int (mix.size());
}

int
awmh_frame_mod (const unsigned char *key16, const char *payload_hex, uint8_t *out, size_t out_size)
{
  const std::vector<int> bitvec = parse_payload (payload_hex);
  if (bitvec.empty())
    return -1;
  const std::vector<uint8_t> fm = gen_frame_mod_ab (make_key (key16, ""), bitvec);
  if (fm.empty() || fm.size() > out_size)
    return -1;
  memcpy (out, fm.data(), fm.size());
  return int (fm.size());
}

/* the two halves of gen_frame_mod_ab: key-only role codes [frames_per_block][101] and one payload's coded bits [2][n_coded] */
int
awmh_embed_roles (const unsigned char *key16, uint16_t *out, size_t out_size)
{
  const std::vector<uint16_t> roles = gen_embed_roles (make_key (key16, ""));
  if (roles.empty() || roles.size() > out_size)
    return -1;
  memcpy (out, roles.data(), roles.size() * sizeof (uint16_t));
  return int (roles.size());
}

int
awmh_coded_bits (const unsigned char *key16, const char *payload_hex, uint8_t *out, size_t out_size)
{
  const std::vector<int> bitvec = parse_payload (payload_hex);
  if (bitvec.empty())
    return -1;
  const std::vector<uint8_t> coded = gen_coded_bits (make_key (key16, ""), bitvec);
  if (coded.size() > out_size)
    return -1;
  memcpy (out, coded.data(), coded.size());
  return int (coded.size());
}

int
awmh_conv_encode (int block_type, const uint8_t *bits, int n, uint8_t *out, int max_out)
{
  std::vector<int> in (bits, bits + n);
  const std::vector<int> enc = conv_encode (ConvBlockType (block_type), in);
  if (int (enc.size()) > max_out)
    return -1;
  for (size_t i = 0; i < enc.size(); i++)
    out[i] = enc[i];
  return int (enc.size());
}

/* short payload block code (src/shortcode.cc:136-213) under the current --short setting: encode k -> n bits, decode n -> k bits
 * (returns 0 when no code word matches) */
int
awmh_short_encode (const uint8_t *bits, int k, uint8_t *out, int max_out)
{
  if (!Params::payload_short || size_t (k) != Params::payload_size)
    return -1;
  const std::vector<int> enc = short_encode_blk (std::vector<int> (bits, bits + k));
  if (int (enc.size()) > max_out)
    return -1;
  for (size_t i = 0; i < enc.size(); i++)
    out[i] = enc[i];
  return int (enc.size());
}

int
awmh_short_decode (const uint8_t *coded, int n, uint8_t *out, int max_out)
{
  if (!Params::payload_short || size_t (n) != code_message_bits())
    return -1;
  const std::vector<int> dec = short_decode_blk (std::vector<int> (coded, coded + n));
  if (int (dec.size()) > max_out)
    return -1;
  for (size_t i = 0; i < dec.size(); i++)
    out[i] = dec[i];
  return int (dec.size());
}

/* add_stream_watermark on buffers (host or device pointers) */
int
awmh_add (const unsigned char *key16, const float *in, float *out, size_t n_frames, int n_channels, int sample_rate,
          const char *payload_hex, int *data_blocks, double *snr_db, uint64_t first_frame_number)
{
  AddStats stats;
  const int rc = add_watermark_buffer (make_key (key16, ""), in, out, n_frames, n_channels, sample_rate, payload_hex,
                                       (data_blocks || snr_db) ? &stats : nullptr, first_frame_number);
  if (data_blocks)
    *data_blocks = stats.data_blocks;
  if (snr_db)
    *snr_db = stats.snr_db;
  return rc;
}

/* add_watermark_batch on a packed buffer (is_s16: 16 bit PCM, else float; host or device): payload_hex[i] goes into items[i].
 * keys16: one 16-byte key, or with per_item_keys [n_items][16] with item i's key.  sample_rates (NULL: every item is at sample_rate)
 * and zero_frames (NULL: every item starts its stream): [n_items].  data_blocks / snr_db (optional): [n_items].  Returns 2 for
 * malformed input (checked before any GPU work), 1 for other errors. */
int
awmh_add_batch (const unsigned char *keys16, int per_item_keys, const void *in, void *out, int is_s16, size_t n_values, const awm_batch_item *items,
                size_t n_items, const char *const *payload_hex, int sample_rate, const int *sample_rates, const uint64_t *zero_frames,
                size_t scratch_bytes, int *data_blocks, double *snr_db)
{
  const size_t n_keys = per_item_keys ? n_items : 1;
  if ((n_keys && !keys16) || (n_items && !payload_hex))
    return 2;
  std::vector<Key> keys (n_keys);
  for (size_t i = 0; i < n_keys; i++)
    keys[i] = make_key (keys16 + i * Key::SIZE, "");
  std::vector<std::string> bits (n_items);
  for (size_t i = 0; i < n_items; i++)
    bits[i] = payload_hex[i] ? payload_hex[i] : "";
  std::vector<AddStats> stats;
  const int rc = add_watermark_batch (keys, per_item_keys != 0, in, out, is_s16 != 0, n_values, items, n_items, bits, sample_rate, sample_rates,
                                      zero_frames, scratch_bytes, (data_blocks || snr_db) ? &stats : nullptr);
  for (size_t i = 0; i < stats.size(); i++)
    {
      if (data_blocks)
        data_blocks[i] = stats[i].data_blocks;
      if (snr_db)
        snr_db[i] = stats[i].snr_db;
    }
  return rc;
}

/* the role layout of the current Params (what awm_set_embed_roles_keys takes) as 6 ints in awm_role_layout's field order */
void
awmh_role_layout (int *out)
{
  const awm_role_layout l = embed_role_layout();
  const int v[6] = { l.sync_frames, l.sync_frames_per_bit, l.data_frames, l.frames_per_bit, l.mix, l.n_coded_bits };
  memcpy (out, v, sizeof (v));
}

/* role tables [n_keys][frames_per_block][101] of keys16 [n_keys][16] built on the device under the current Params (the tables
 * awmh_embed_roles builds on the host one key at a time) */
int
awmh_embed_roles_device (const unsigned char *keys16, size_t n_keys, uint16_t *out, size_t out_size)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  const awm_role_layout l = embed_role_layout();
  if (n_keys * frames_per_block() * (Params::max_band + 1) > out_size)
    return 2;
  if (awm_set_embed_roles_keys (ctx, keys16, n_keys, &l) || awm_get_embed_roles_keys (ctx, 0, n_keys, out))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return 1;
    }
  return 0;
}

/* add / get between 16 bit PCM host buffers (the contents of a 16 bit WAV file): conversions run on the device */
int
awmh_add_s16 (const unsigned char *key16, const int16_t *in, int16_t *out, size_t n_frames, int n_channels, int sample_rate,
              const char *payload_hex, int *data_blocks, double *snr_db, uint64_t first_frame_number)
{
  AddStats stats;
  const int rc = add_watermark_buffer_s16 (make_key (key16, ""), in, out, n_frames, n_channels, sample_rate, payload_hex, (data_blocks || snr_db) ? &stats : nullptr,
                                           first_frame_number);
  if (data_blocks)
    *data_blocks = stats.data_blocks;
  if (snr_db)
    *snr_db = stats.snr_db;
  return rc;
}

/* add_stream_watermark's bounded-memory loop (add_watermark_windowed) between two host buffers: `in` is read in small blocks like a
 * pipe, the result is appended to `out` (n_frames frames); window_frames = 0 uses the default window.  zero_frames: the input continues
 * a stream that began that many frames earlier with silence (src/wmadd.cc:504-519). */
int
awmh_add_windowed (const unsigned char *key16, const float *in, float *out, size_t n_frames, int n_channels, int sample_rate, const char *payload_hex,
                   size_t zero_frames, size_t window_frames, int *data_blocks, double *snr_db)
{
  size_t rpos = 0, wpos = 0;
  auto read = [&] (std::vector<float>& samples, size_t count)
    {
      const size_t n = std::min (count, n_frames - rpos);
      samples.assign (in + rpos * n_channels, in + (rpos + n) * n_channels);
      rpos += n;
      return Error (Error::Code::NONE);
    };
  auto write = [&] (const std::vector<float>& samples)
    {
      if (wpos * n_channels + samples.size() > n_frames * n_channels)
        return Error ("output buffer too small");
      memcpy (out + wpos * n_channels, samples.data(), samples.size() * sizeof (float));
      wpos += samples.size() / n_channels;
      return Error (Error::Code::NONE);
    };
  AddStats stats;
  size_t written = 0;
  const int rc = add_watermark_windowed (make_key (key16, ""), read, write, n_channels, sample_rate, payload_hex, zero_frames, window_frames, &stats, &written);
  if (rc)
    return rc;
  if (data_blocks) *data_blocks = stats.data_blocks;
  if (snr_db) *snr_db = stats.snr_db;
  return written == n_frames ? 0 : -3;
}

/* add_window_range: the input frames a window needs for its owned frames (n_total = UINT64_MAX: the end is not known yet) */
int
awmh_window_range (uint64_t own_first, uint64_t own_end, uint64_t n_total, int sample_rate, uint64_t *ext_first, uint64_t *ext_end)
{
  size_t e0 = 0, e1 = 0;
  if (add_window_range (own_first, own_end, n_total, sample_rate, e0, e1))
    return 2;
  *ext_first = e0;
  *ext_end = e1;
  return 0;
}

/* add_watermark_window on a buffer (host or device) that holds stream frames [stream_first, stream_first + n_frames): the window
 * add_window_range names for [own_first, own_end) is embedded in place of the same frames of `out`, the rest of `out` is not
 * touched.  snr_power (optional): the --snr sums of the owned frames.  Returns 2, before any GPU work, for a malformed range or a
 * buffer that misses a frame of the window, 1 for other errors. */
int
awmh_add_window (const unsigned char *key16, const float *in, float *out, uint64_t stream_first, size_t n_frames, int n_channels, int sample_rate,
                 const char *payload_hex, uint64_t n_total, uint64_t own_first, uint64_t own_end, double *snr_power)
{
  size_t e0 = 0, e1 = 0;
  if (n_channels <= 0 || add_window_range (own_first, own_end, n_total, sample_rate, e0, e1))
    return 2;
  if (e0 < stream_first || e1 > stream_first + n_frames)
    {
      error ("audiowmark: the buffer holds stream frames [%llu, %llu), the window needs [%zu, %zu)\n", (unsigned long long) stream_first,
             (unsigned long long) (stream_first + n_frames), e0, e1);
      return 2;
    }
  const size_t off = (e0 - stream_first) * size_t (n_channels);
  return add_watermark_window (make_key (key16, ""), payload_hex, in + off, out + off, e0, e1, n_total, n_channels, sample_rate, own_first, own_end,
                               snr_power);
}

static int result_json (ResultSet& result_set, size_t mark_rate_frames, char *json_out, size_t json_cap, int *n_patterns);

int
awmh_get_s16 (const unsigned char *keys16, const char *const *names, int n_keys, const int16_t *pcm, size_t n_frames, int n_channels,
              int sample_rate, char *json_out, size_t json_cap, int *n_patterns)
{
  std::vector<Key> key_list;
  for (int k = 0; k < n_keys; k++)
    key_list.push_back (make_key (keys16 + 16 * k, names ? names[k] : ""));
  ResultSet result_set;
  size_t mark_rate_frames = n_frames;
  const int rc = get_watermark_buffer_s16 (key_list, pcm, n_frames, n_channels, sample_rate, result_set, false, &mark_rate_frames);
  if (rc)
    return rc;
  return result_json (result_set, mark_rate_frames, json_out, json_cap, n_patterns);
}

/* get_watermark on a buffer (host pointer; a device pointer is accepted for inputs longer than 3.1 blocks,
 * where the clip decoder is not used).  Writes the --json document into json_out. */
int
awmh_get (const unsigned char *keys16, const char *const *names, int n_keys, const float *pcm, size_t n_frames, int n_channels,
          int sample_rate, char *json_out, size_t json_cap, int *n_patterns)
{
  std::vector<Key> key_list;
  for (int k = 0; k < n_keys; k++)
    key_list.push_back (make_key (keys16 + 16 * k, names ? names[k] : ""));
  ResultSet result_set;
  size_t mark_rate_frames = n_frames;
  const int rc = get_watermark_buffer (key_list, pcm, n_frames, n_channels, sample_rate, result_set, false, &mark_rate_frames);
  if (rc)
    return rc;
  return result_json (result_set, mark_rate_frames, json_out, json_cap, n_patterns);
}

static std::vector<Key> make_key_list (const unsigned char *keys16, const char *const *names, int n_keys);

/* ---- streaming `get` (GetStream): a stream fed piece by piece in bounded memory -------------------------------------------------
 * awmh_gs_create returns NULL, with a message and without GPU work, for a sample rate outside the resampler's range or channels <= 0.
 * awmh_gs_feed takes interleaved float frames in host or device memory; awmh_gs_finish writes the --json document as awmh_get does.
 * After a failed feed, or after finish, the stream only accepts awmh_gs_destroy. */
void *
awmh_gs_create (const unsigned char *keys16, const char *const *names, int n_keys, int n_channels, int sample_rate, int print_speed_results)
{
  GetStream *s = new GetStream (make_key_list (keys16, names, n_keys), n_channels, sample_rate, print_speed_results != 0);
  if (!s->ok())
    {
      delete s;
      return nullptr;
    }
  return s;
}

int
awmh_gs_feed (void *h, const float *pcm, size_t n_frames)
{
  return static_cast<GetStream *> (h)->feed (pcm, n_frames);
}

int
awmh_gs_finish (void *h, char *json_out, size_t json_cap, int *n_patterns)
{
  ResultSet result_set;
  size_t mark_rate_frames = 0;
  const int rc = static_cast<GetStream *> (h)->finish (result_set, &mark_rate_frames);
  if (rc)
    return rc;
  return result_json (result_set, mark_rate_frames, json_out, json_cap, n_patterns);
}

void
awmh_gs_destroy (void *h)
{
  delete static_cast<GetStream *> (h);
}

/* device bytes the stream holds at most (chunk buffer + input window) */
uint64_t
awmh_gs_peak_bytes (void *h)
{
  return static_cast<GetStream *> (h)->peak_device_bytes();
}

/* test aid (CPU): the chunks GetStream decodes for a stream of n_total frames at sample_rate fed in pieces of piece_frames, without a
 * device (chunks [max][3]: first frame, frames, time offset, in watermark-rate frames); *mark_frames: the stream's watermark-rate length.
 * Returns 1 for a refused rate */
int
awmh_gs_plan (uint64_t n_total, uint64_t piece_frames, int sample_rate, double *chunks, int max_chunks, int *n_chunks, uint64_t *mark_frames)
{
  GetStream s ({}, 1, sample_rate, false, ~size_t (0), true);
  if (!s.ok() || !piece_frames)
    return 1;
  for (uint64_t fed = 0; fed < n_total; fed += piece_frames)
    if (s.feed (nullptr, std::min (piece_frames, n_total - fed)))
      return 1;
  ResultSet rs;
  size_t m = 0;
  if (s.finish (rs, &m))
    return 1;
  *mark_frames = m;
  *n_chunks = int (s.chunks().size());
  for (int c = 0; c < *n_chunks && c < max_chunks; c++)
    {
      chunks[3 * c] = double (s.chunks()[c].first);
      chunks[3 * c + 1] = double (s.chunks()[c].n_frames);
      chunks[3 * c + 2] = s.chunks()[c].time_offset;
    }
  return 0;
}

static int
result_json (ResultSet& result_set, size_t mark_rate_frames, char *json_out, size_t json_cap, int *n_patterns)
{
  if (n_patterns)
    *n_patterns = int (result_set.all().size());
  if (json_out && json_cap)
    {
      char *buf = nullptr;
      size_t len = 0;
      FILE *f = open_memstream (&buf, &len);
      result_set.print_json (f, size_t (lrint (double (mark_rate_frames) / Params::mark_sample_rate)));
      fclose (f);
      if (len + 1 > json_cap)
        {
          free (buf);
          return -2;
        }
      memcpy (json_out, buf, len + 1);
      free (buf);
    }
  return 0;
}

/* ---- test aid (CPU): ResultSet merge, sort and --json print of per-chunk pattern records ----------------------
 * awmh_merge_chunks takes the chunk results as the test writes them, so that the C++ ResultSet can be checked against the oracle's
 * without a GPU, printed digits included.  Record (little endian, packed): i32 key_index, f64 time, f64 quality, u64 sync_index,
 * f32 decode_error, u8 block_type, u8 type, f64 speed, u16 n_bits, n_bits bytes (0/1)
 */
static bool
deserialize (const unsigned char *b, size_t len, const std::vector<Key>& key_list, ResultSet& rs)
{
  size_t pos = 0;
  auto get = [&] (void *p, size_t n) { if (pos + n > len) return false; memcpy (p, b + pos, n); pos += n; return true; };
  while (pos < len)
    {
      int32_t ki; double time, quality, speed; uint64_t idx; float err; uint8_t bt, ty; uint16_t nb;
      if (!get (&ki, 4) || !get (&time, 8) || !get (&quality, 8) || !get (&idx, 8) || !get (&err, 4) || !get (&bt, 1) || !get (&ty, 1)
          || !get (&speed, 8) || !get (&nb, 2) || pos + nb > len || ki < 0 || size_t (ki) >= key_list.size() || bt > 2 || ty > 2)
        return false;
      std::vector<int> bits (b + pos, b + pos + nb);
      pos += nb;
      rs.add_pattern (key_list[ki], time, SyncFinder::Score { size_t (idx), quality, ConvBlockType (bt) }, bits, err, ResultSet::Type (ty), speed);
    }
  return true;
}

static std::vector<Key>
make_key_list (const unsigned char *keys16, const char *const *names, int n_keys)
{
  std::vector<Key> key_list;
  for (int k = 0; k < n_keys; k++)
    key_list.push_back (make_key (keys16 + 16 * k, names ? names[k] : ""));
  return key_list;
}

/* ResultSet::merge in chunk order + sort + --json document (src/wmget.cc:289-316,252-287,340-382) from chunk records */
int
awmh_merge_chunks (const unsigned char *keys16, const char *const *names, int n_keys, const unsigned char *const *blobs, const size_t *blob_lens,
                   const double *time_offsets, int n_chunks, double total_seconds, char *json_out, size_t json_cap)
{
  const std::vector<Key> key_list = make_key_list (keys16, names, n_keys);
  ResultSet result_set;
  for (int c = 0; c < n_chunks; c++)
    {
      ResultSet chunk;
      if (!deserialize (blobs[c], blob_lens[c], key_list, chunk))
        return -3;
      chunk.apply_time_offset (time_offsets[c]);
      result_set.merge (chunk);
    }
  result_set.sort (key_list);
  char *buf = nullptr;
  size_t len = 0;
  FILE *f = open_memstream (&buf, &len);
  result_set.print_json (f, size_t (lrint (total_seconds)));
  fclose (f);
  const bool fits = len + 1 <= json_cap;
  if (fits)
    memcpy (json_out, buf, len + 1);
  free (buf);
  return fits ? 0 : -2;
}

void
awmh_chunk_geometry (int sample_rate, uint64_t *max_frames, uint64_t *overlap_frames)
{
  size_t m, o;
  chunk_geometry (sample_rate, m, o);
  *max_frames = m;
  *overlap_frames = o;
}

/* ---- sharded `get`: one long stream over several GPUs (awm_balanced.hh) --------------------------------------------------- */

int
awmh_dist_unique_id (unsigned char id_out[128])
{
  return awm_dist_unique_id (id_out);
}

/* join the NCCL communicator of the job (the id comes from rank 0's awmh_dist_unique_id, handed round by the launcher) */
int
awmh_dist_init (int rank, int world, const unsigned char id[128])
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  if (awm_dist_init (ctx, rank, world, id))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return 1;
    }
  return 0;
}

/* every rank calls this with its part of the stream ([pcm_start, pcm_start + pcm_frames) of n_total frames; float or 16 bit PCM,
 * host or device memory); rank 0 receives the --json document (n_patterns >= 0), the other ranks n_patterns = -1 */
int
awmh_balanced_get (const unsigned char *key16, const void *pcm, int is_s16, uint64_t pcm_start, uint64_t pcm_frames, uint64_t n_total, int n_channels,
                   int sample_rate, char *json_out, size_t json_cap, int *n_patterns)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return 1;
  int rank = 0, world = 1;
  awm_dist_world (ctx, &rank, &world);
  balanced::Get job (rank, world, n_total, is_s16 ? nullptr : static_cast<const float *> (pcm), is_s16 ? static_cast<const int16_t *> (pcm) : nullptr,
                     pcm_start, pcm_frames, n_channels, sample_rate, make_key (key16, ""));
  if (!job.ok())
    return 1;
  std::vector<unsigned char> recv;
  std::vector<size_t> lens (world);
  /* bytes per rank in an exchange: the refined scores + soft bits of a rank's candidates are ~0.4 MB per hour of audio; a payload that
   * does not fit costs a second round, so the size that was needed once is kept for the following calls */
  static size_t slot = 1024 * 1024;
  auto exchange = [&] (const std::string& mine, std::vector<std::string>& all)
    {
      for (;;)
        {
          recv.resize (slot * world);
          const int rc = awm_dist_allgather (ctx, mine.data(), mine.size(), slot, recv.data(), lens.data());
          if (rc == 2)                               // somebody's payload did not fit: every rank saw the same lengths
            {
              slot = (*std::max_element (lens.begin(), lens.end()) + 8 + 4095) / 4096 * 4096;
              continue;
            }
          if (rc)
            {
              error ("audiowmark: %s\n", awm_last_error (ctx));
              return false;
            }
          break;
        }
      all.resize (world);
      for (int r = 0; r < world; r++)
        all[r].assign (reinterpret_cast<const char *> (recv.data()) + size_t (r) * slot, lens[r]);
      return true;
    };
  ResultSet result_set;
  if (!job.run (exchange, result_set))
    return 1;
  if (rank != 0)
    {
      if (n_patterns)
        *n_patterns = -1;
      return 0;
    }
  return result_json (result_set, job.n_mark(), json_out, json_cap, n_patterns);
}

/* the stages one by one, for tests that run several ranks in one process on one GPU (tests/test_gpu_sharding.py):
 * stage 0 peaks, 1 select (-> retry list), 2 peaks again for the retry list in in[0], 3 refine + soft bits, 4 viterbi, 5 merge (-> JSON;
 * its length is that of the watermark-rate stream the driver planned, awmh_bg_stage's n_total is not used) */
void *
awmh_bg_create (const unsigned char *key16, int rank, int world, const float *pcm, uint64_t pcm_start, uint64_t pcm_frames, uint64_t n_total, int n_channels, int sample_rate)
{
  balanced::Get *g = new balanced::Get (rank, world, n_total, pcm, nullptr, pcm_start, pcm_frames, n_channels, sample_rate, make_key (key16, ""));
  if (!g->ok())
    {
      delete g;
      return nullptr;
    }
  return g;
}

void
awmh_bg_destroy (void *h)
{
  delete static_cast<balanced::Get *> (h);
}

int
awmh_bg_stage (void *h, int stage, const unsigned char *const *in, const size_t *in_len, int n_in, uint64_t n_total, unsigned char *out, size_t cap, size_t *out_len)
{
  balanced::Get *g = static_cast<balanced::Get *> (h);
  std::vector<std::string> all;
  for (int i = 0; i < n_in; i++)
    all.emplace_back (reinterpret_cast<const char *> (in[i]), in_len[i]);
  std::string res;
  bool ok = false;
  auto parse_floors = [] (const std::string& s)
    {
      std::map<int, double> m;
      for (size_t pos = 0; pos + 12 <= s.size(); pos += 12)
        {
          int32_t c; double f;
          memcpy (&c, s.data() + pos, 4); memcpy (&f, s.data() + pos + 4, 8);
          m[c] = f;
        }
      return m;
    };
  switch (stage)
    {
    case 0: ok = g->stage_peaks ({}, res); break;
    case 1:
      {
        std::map<int, double> retry;
        ok = g->stage_select (all, retry);
        for (const auto& kv : retry)
          {
            const int32_t c = kv.first; const double f = kv.second;
            res.append (reinterpret_cast<const char *> (&c), 4);
            res.append (reinterpret_cast<const char *> (&f), 8);
          }
        break;
      }
    case 2: ok = g->stage_peaks (parse_floors (all.empty() ? std::string() : all[0]), res); break;
    case 3: ok = g->stage_refine_decode (res); break;
    case 4: ok = g->stage_viterbi (all, res); break;
    case 5:
      {
        ResultSet rs;
        ok = g->stage_merge (all, rs);
        if (ok)
          {
            char *buf = nullptr;
            size_t len = 0;
            FILE *f = open_memstream (&buf, &len);
            rs.print_json (f, size_t (lrint (double (g->n_mark()) / Params::mark_sample_rate)));
            fclose (f);
            res.assign (buf, len);
            free (buf);
          }
        break;
      }
    }
  if (!ok)
    return 1;
  *out_len = res.size();
  if (res.size() > cap)
    return -2;
  if (!res.empty())
    memcpy (out, res.data(), res.size());
  return 0;
}

/* the plan functions for CPU tests and launchers: chunk walk, slices of a rank, owner of an index, the input a rank holds.  A stream of
 * n_total frames at sample_rate is planned at the watermark rate, as the driver runs it (balanced::mark_frames); 1 for a sample rate
 * the sharded get refuses */
int
awmh_bg_plan (uint64_t n_total, int sample_rate, int rank, int world, double *chunks /* [max][3] first, count, time offset */, int max_chunks, int *n_chunks,
              int64_t *slices /* [max][7] chunk, sa, sb, a, b, lo, hi */, int max_slices, int *n_slices)
{
  if (!balanced::rate_supported (sample_rate))
    return 1;
  const size_t n_mark = balanced::mark_frames (n_total, sample_rate);
  const auto plan = balanced::chunk_plan (n_mark, Params::mark_sample_rate);
  *n_chunks = int (plan.size());
  for (int c = 0; c < int (plan.size()) && c < max_chunks; c++)
    {
      chunks[3 * c] = double (plan[c].first);
      chunks[3 * c + 1] = double (plan[c].count);
      chunks[3 * c + 2] = plan[c].time_offset;
    }
  const auto sl = balanced::rank_slices (plan, rank, world, n_mark);
  *n_slices = int (sl.size());
  for (int i = 0; i < int (sl.size()) && i < max_slices; i++)
    {
      const int64_t v[7] = { sl[i].chunk, sl[i].sa, sl[i].sb, sl[i].a, sl[i].b, int64_t (sl[i].lo), int64_t (sl[i].hi) };
      memcpy (slices + 7 * i, v, sizeof (v));
    }
  return 0;
}

int
awmh_bg_owner (uint64_t n_total, int sample_rate, int world, int chunk, uint64_t index)
{
  if (!balanced::rate_supported (sample_rate))
    return -1;
  const size_t n_mark = balanced::mark_frames (n_total, sample_rate);
  return balanced::owner_of (balanced::chunk_plan (n_mark, Params::mark_sample_rate), n_mark, world, chunk, index);
}

/* input frames [*first, *end) of the stream that rank `rank` of `world` has to hold (balanced::input_range of its slices) */
int
awmh_bg_input_range (uint64_t n_total, int rank, int world, int sample_rate, uint64_t *first, uint64_t *end)
{
  if (!balanced::rate_supported (sample_rate) || world < 1 || rank < 0 || rank >= world)
    return 1;
  const size_t n_mark = balanced::mark_frames (n_total, sample_rate);
  size_t f, e;
  balanced::input_range (balanced::rank_slices (balanced::chunk_plan (n_mark, Params::mark_sample_rate), rank, world, n_mark), n_total, sample_rate, f, e);
  *first = f;
  *end = e;
  return 0;
}

/* ---- the GPU context and its key slots ------------------------------------------------------------------------- */

void *
awmh_ctx()
{
  return Engine::ctx();
}

int
awmh_key_slot (const unsigned char *key16)
{
  return Engine::key_slot (make_key (key16, ""));
}

/* test aid (CPU): ResultSet::merge and ResultSet::sort against their literal definitions (src/wmget.cc:268-312: scan everything found so
 * far with approx_match; compare name / rating / all-last / time / A-B-AB / bits one after the other) on random chunk results: a few
 * payloads, positions that collide within a frame across chunks, combined patterns, stretched speeds, two keys.  Returns 0 when the
 * merged and sorted documents are identical, else the number of the first failing round + 1. */
int
awmh_selftest_results (uint64_t seed, int rounds)
{
  uint64_t state = seed * 6364136223846793005ull + 1442695040888963407ull;
  auto rnd = [&] (uint32_t n) { state = state * 6364136223846793005ull + 1442695040888963407ull; return uint32_t ((state >> 33) % n); };
  const double frame = Params::frame_size / double (Params::mark_sample_rate);
  Key keys[2];
  keys[0] = make_key (reinterpret_cast<const unsigned char *> ("0123456789abcdef"), "alpha");
  keys[1] = make_key (reinterpret_cast<const unsigned char *> ("fedcba9876543210"), "beta");
  size_t n_in = 0, n_kept = 0;
  for (int round = 0; round < rounds; round++)
    {
      std::vector<std::vector<int>> payloads (3 + rnd (3), std::vector<int> (16));
      for (auto& pl : payloads)
        for (int& b : pl)
          b = int (rnd (2));
      const int n_chunks = 2 + int (rnd (4));
      std::vector<ResultSet> chunks (n_chunks), chunks_copy;
      for (int c = 0; c < n_chunks; c++)
        for (int i = 0, n = int (rnd (40)); i < n; i++)
          {
            const ResultSet::Type type = rnd (10) == 0 ? ResultSet::Type::ALL : rnd (8) == 0 ? ResultSet::Type::CLIP : ResultSet::Type::BLOCK;
            const ConvBlockType bt = ConvBlockType (rnd (3));
            /* positions on a coarse grid + a jitter around one frame, so that patterns of neighbouring chunks fall inside and just outside the match window */
            /* + a unique 1e-7 s: no two patterns tie in every sort key (std::sort leaves the order of ties open, in the reference too) */
            const double time = double (rnd (12)) * 7.0 + (double (rnd (5)) - 2.0) * frame * 0.6 + 1e-7 * double (c * 64 + i);
            const double speed = rnd (6) == 0 ? 1.0 + (double (rnd (5)) - 2.0) * 0.006 : 1.0;
            chunks[c].add_pattern (keys[rnd (2)], time, SyncFinder::Score { size_t (rnd (100000)), double (rnd (1000)) / 1000.0, bt }, payloads[rnd (uint32_t (payloads.size()))],
                                   float (rnd (100)) / 100.f, type, speed);
          }
      chunks_copy = chunks;
      /* the library */
      ResultSet merged;
      for (int c = 0; c < n_chunks; c++)
        {
          chunks[c].apply_time_offset (0.4 * frame * c);
          merged.merge (chunks[c]);
        }
      merged.sort ({ keys[0], keys[1] });
      /* the definition */
      std::vector<ResultSet::Pattern> ref;
      for (int c = 0; c < n_chunks; c++)
        {
          chunks_copy[c].apply_time_offset (0.4 * frame * c);
          std::vector<ResultSet::Pattern> in = chunks_copy[c].all();
          std::stable_sort (in.begin(), in.end(), [] (const ResultSet::Pattern& a, const ResultSet::Pattern& b) { return a.time < b.time; });
          for (const auto& p : in)
            {
              bool is_new = true;
              for (const auto& have : ref)
                if (have.approx_match (p))
                  is_new = false;
              if (is_new)
                ref.push_back (p);
            }
        }
      for (const Key& key : keys)
        {
          std::map<std::string, float> rating;
          for (const auto& p : ref)
            if (p.key == key)
              rating[bit_vec_to_str (p.bit_vec)] += p.sync_score.quality * (p.type == ResultSet::Type::ALL ? 2.f : 1.f);
          for (auto& p : ref)
            if (p.key == key)
              p.rating = rating[bit_vec_to_str (p.bit_vec)];
        }
      auto rank_of = [] (const ResultSet::Pattern& p) { return p.sync_score.block_type == ConvBlockType::a ? 0 : p.sync_score.block_type == ConvBlockType::b ? 1 : 2; };
      std::sort (ref.begin(), ref.end(), [&] (const ResultSet::Pattern& a, const ResultSet::Pattern& b)
        {
          const int all_a = a.type == ResultSet::Type::ALL, all_b = b.type == ResultSet::Type::ALL;
          if (a.key.name() != b.key.name()) return a.key.name() < b.key.name();
          if (a.rating != b.rating) return a.rating > b.rating;
          if (all_a != all_b) return all_a < all_b;
          if (a.time != b.time) return a.time < b.time;
          if (rank_of (a) != rank_of (b)) return rank_of (a) < rank_of (b);
          return bit_vec_to_str (a.bit_vec) < bit_vec_to_str (b.bit_vec);
        });
      const auto& got = merged.all();
      bool same = got.size() == ref.size();
      for (size_t i = 0; same && i < ref.size(); i++)
        same = got[i].key == ref[i].key && got[i].time == ref[i].time && got[i].bit_vec == ref[i].bit_vec && got[i].type == ref[i].type
            && got[i].sync_score.block_type == ref[i].sync_score.block_type && got[i].sync_score.quality == ref[i].sync_score.quality
            && got[i].speed == ref[i].speed && got[i].rating == ref[i].rating && got[i].decode_error == ref[i].decode_error;
      if (!same)
        return round + 1;
      for (const ResultSet& cr : chunks_copy)
        n_in += cr.all().size();
      n_kept += ref.size();
    }
  /* the test has teeth only if the merge did drop detections and keep others */
  return (n_kept < n_in && n_kept * 10 > n_in) ? 0 : -1;
}

/* test aid: sync positions.  awmh_sync_trace (1) starts recording what every SyncFinder::search call returns, awmh_sync_trace_fetch
 * copies the records out as rows of 5 doubles {search number, mode (0 BLOCK / 1 CLIP), searched frames, -1, -1} (one header row per
 * search) and {search number, index, quality, block type (0 A / 1 B), 0} (one row per score) and clears the trace */
int
awmh_sync_trace (int on)
{
  SyncFinder::trace_enable (on != 0);
  return 0;
}

int
awmh_sync_trace_fetch (double *rows, size_t max_rows, size_t *n_rows)
{
  const auto trace = SyncFinder::trace_take();
  size_t n = 0;
  auto put = [&] (double a, double b, double c, double d, double e)
    {
      if (n < max_rows)
        {
          double *r = rows + 5 * n;
          r[0] = a; r[1] = b; r[2] = c; r[3] = d; r[4] = e;
        }
      n++;
    };
  for (size_t i = 0; i < trace.size(); i++)
    {
      put (double (i), trace[i].mode == SyncFinder::Mode::CLIP ? 1 : 0, double (trace[i].n_frames), -1, -1);
      for (const auto& sc : trace[i].scores)
        put (double (i), double (sc.index), sc.quality, sc.block_type == ConvBlockType::a ? 0 : 1, 0);
    }
  *n_rows = n;
  return n <= max_rows ? 0 : -2;
}

/* test aid (CPU): select_candidates_from_peaks, the selection of the single-GPU and the sharded `get`, on a peak list the test builds.
 * Candidates of one chunk from its (gathered) peak list, complete above floor_q; *complete = 0 -> ask again with a lower floor */
int
awmh_stage_select (const awm_search_score *peaks, size_t n, double floor_q, int clip_mode, awm_search_score *out, size_t max_out, size_t *n_out, int *complete)
{
  std::vector<awm_search_score> sel;
  const size_t n_max = clip_mode ? std::max (Params::get_n_best, 5) : 0;
  *complete = select_candidates_from_peaks (peaks, n, floor_q, Params::sync_threshold2 * 0.75, sel, n_max) > 0 ? 1 : 0;
  if (clip_mode)
    {
      std::sort (sel.begin(), sel.end(), [] (const awm_search_score& a, const awm_search_score& b) { return fabs (a.raw_quality - a.local_mean) > fabs (b.raw_quality - b.local_mean); });
      if (sel.size() > n_max)
        sel.resize (n_max);
    }
  *n_out = sel.size();
  if (sel.size() > max_out)
    return -2;
  if (!sel.empty())
    memcpy (out, sel.data(), sel.size() * sizeof (awm_search_score));
  return 0;
}

uint64_t
awmh_gpu_launches()
{
  awm_ctx *c = Engine::ctx();
  return c ? awm_launch_count (c) : 0;
}

void *
awmh_gpu_stream()
{
  awm_ctx *c = Engine::ctx();
  return c ? awm_stream (c) : nullptr;
}

/* device-pointer calls are stream ordered and return without waiting: synchronise before touching the results from
 * another stream / the host */
int
awmh_synchronize()
{
  awm_ctx *c = Engine::ctx();
  return c ? awm_synchronize (c) : 1;
}

int
awmh_profile_enable (int on)
{
  awm_ctx *c = Engine::ctx();
  return c ? awm_profile_enable (c, on) : 1;
}

int
awmh_profile_report (char *json_out, size_t cap)
{
  awm_ctx *c = Engine::ctx();
  return c ? awm_profile_report (c, json_out, cap) : 1;
}

void
awmh_shutdown()
{
  Engine::shutdown();
}

} // extern "C"
