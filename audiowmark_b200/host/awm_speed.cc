// awm_speed.cc -- speed detection driver (reference: src/wmspeed.cc) and the resampling entry points
// (reference: src/resample.cc:52-131).
//
// The reference fans SpeedSync::prepare_mags / compare jobs out over a thread pool, one MagMatrix per centre speed.
// Here the host only keeps the control flow of detect_speed (three scans, peak selection, smoothing); a whole scan --
// resampling the clip for every centre, the 512-point spectra, and every (centre, relative speed) comparison -- is
// one awm_speed_scan call, i.e. three kernel launches.
#include "awm_speed.hh"
#include "awm_engine.hh"
#include "awm_util.hh"

#include <math.h>
#include <string.h>
#include <algorithm>

using std::vector;
using std::min;
using std::max;

namespace {

/* ---- SHA-1 (FIPS 180-4) for Random::seed_from_hash (src/random.cc:184-190; the reference calls libgcrypt) ---- */
struct Sha1
{
  uint32_t h[5] = { 0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u };
  unsigned char block[64];
  size_t fill = 0;
  uint64_t total = 0;
  static uint32_t rol (uint32_t v, int s) { return (v << s) | (v >> (32 - s)); }
  void
  compress()
  {
    uint32_t w[80];
    for (int i = 0; i < 16; i++)
      w[i] = uint32_t (block[4 * i]) << 24 | uint32_t (block[4 * i + 1]) << 16 | uint32_t (block[4 * i + 2]) << 8 | block[4 * i + 3];
    for (int i = 16; i < 80; i++)
      w[i] = rol (w[i - 3] ^ w[i - 8] ^ w[i - 14] ^ w[i - 16], 1);
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
    for (int i = 0; i < 80; i++)
      {
        uint32_t f, k;
        if (i < 20)      { f = (b & c) | (~b & d);          k = 0x5A827999u; }
        else if (i < 40) { f = b ^ c ^ d;                   k = 0x6ED9EBA1u; }
        else if (i < 60) { f = (b & c) | (b & d) | (c & d); k = 0x8F1BBCDCu; }
        else             { f = b ^ c ^ d;                   k = 0xCA62C1D6u; }
        const uint32_t t = rol (a, 5) + f + e + k + w[i];
        e = d; d = c; c = rol (b, 30); b = a; a = t;
      }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
  }
  void
  update (const void *data, size_t n)
  {
    const unsigned char *p = static_cast<const unsigned char *> (data);
    total += n;
    while (n)
      {
        const size_t take = min (n, 64 - fill);
        memcpy (block + fill, p, take);
        fill += take; p += take; n -= take;
        if (fill == 64)
          {
            compress();
            fill = 0;
          }
      }
  }
  void
  finish (unsigned char out[20])
  {
    const uint64_t bits = total * 8;
    const unsigned char one = 0x80, zero = 0;
    update (&one, 1);
    while (fill != 56)
      update (&zero, 1);
    unsigned char len[8];
    for (int i = 0; i < 8; i++)
      len[i] = (unsigned char) (bits >> (56 - 8 * i));
    update (len, 8);
    for (int i = 0; i < 5; i++)
      for (int j = 0; j < 4; j++)
        out[4 * i + j] = (unsigned char) (h[i] >> (24 - 8 * j));
  }
};

uint64_t
seed_from_hash (const vector<float>& floats)
{
  Sha1 sha;
  sha.update (floats.data(), floats.size() * sizeof (float));
  unsigned char hash[20];
  sha.finish (hash);
  uint64_t v = 0;
  for (int i = 0; i < 8; i++)                    /* uint64_from_buffer: big endian */
    v = (v << 8) | hash[i];
  return v;
}

struct SpeedScanParams        /* src/wmspeed.cc:54-60 */
{
  double seconds        = 0;
  double step           = 0;
  int    n_steps        = 0;
  int    n_center_steps = 0;
};

struct Score { double speed = 0; double quality = 0; };

/* PCM of one chunk; samples is a host pointer, or a device pointer when on_device is set (then the few values the
 * host needs are fetched with awm_gather / awm_copy_to_host, the chunk itself never crosses PCIe) */
struct Pcm
{
  const float *samples;
  size_t       n_frames;
  int          n_channels;
  int          sample_rate;
  bool         on_device;
};

/* get_speed_clip (src/wmspeed.cc:33-52): [start, end) in frames */
void
speed_clip_range (double location, const Pcm& in, double clip_seconds, size_t& start_point, size_t& end_point)
{
  const double end_sec = double (in.n_frames) / in.sample_rate;
  double start_sec = location * (end_sec - clip_seconds);
  if (start_sec < 0)
    start_sec = 0;
  start_point = start_sec * in.sample_rate;
  end_point = min<size_t> (start_point + clip_seconds * in.sample_rate, in.n_frames);
}

vector<double>
get_clip_locations (const Key& key, const Pcm& in, int n)      /* src/wmspeed.cc:533-552 */
{
  Random rng (key, 0, Random::Stream::speed_clip);
  /* to improve performance, not all samples are hashed but just a few */
  const size_t n_values = in.n_frames * in.n_channels;
  vector<float> xsamples;
  if (in.on_device)
    {
      vector<uint64_t> positions;
      for (size_t p = 0; p < n_values; p += rng() % 1000)
        positions.push_back (p);
      xsamples.resize (positions.size());
      if (awm_gather (Engine::ctx(), in.samples, positions.data(), positions.size(), xsamples.data()))
        error ("audiowmark: %s\n", awm_last_error (Engine::ctx()));
    }
  else
    for (size_t p = 0; p < n_values; p += rng() % 1000)
      xsamples.push_back (in.samples[p]);
  rng.seed (seed_from_hash (xsamples), Random::Stream::speed_clip);
  vector<double> result;
  for (int c = 0; c < n; c++)
    result.push_back (rng.random_double());
  return result;
}

double
get_best_clip_location (const Key& key, const Pcm& in, double seconds, int candidates)    /* src/wmspeed.cc:554-575 */
{
  double clip_location = 0, best_energy = 0;
  for (auto location : get_clip_locations (key, in, candidates))
    {
      size_t s, e;
      speed_clip_range (location, in, seconds, s, e);
      const float *clip = in.samples + s * in.n_channels;
      vector<float> clip_copy;
      if (in.on_device)
        {
          clip_copy.resize ((e - s) * in.n_channels);
          if (awm_copy_to_host (Engine::ctx(), clip_copy.data(), clip, clip_copy.size() * sizeof (float)))
            error ("audiowmark: %s\n", awm_last_error (Engine::ctx()));
          clip = clip_copy.data();
        }
      double energy = 0;
      for (size_t i = 0; i < (e - s) * in.n_channels; i++)
        {
          const float v = clip[i];
          energy += v * v;
        }
      if (energy > best_energy)
        {
          best_energy = energy;
          clip_location = location;
        }
    }
  return clip_location;
}

/* SpeedSearch::get_jobs + run_search for one key (src/wmspeed.cc:459-484, 688-722): all centres of all speeds in one GPU call */
bool
run_search (const Key& key, const Pcm& in, double clip_location, const SpeedScanParams& scan, const vector<double>& speeds, vector<Score>& scores)
{
  scores.clear();
  awm_ctx *ctx = Engine::ctx();
  const int slot = Engine::key_slot (key);
  if (!ctx || slot < 0)
    return false;
  size_t s, e;
  speed_clip_range (clip_location, in, scan.seconds * 1.3, s, e);     /* speed is between 0.8 and 1.25: factor 1.3 provides enough samples */
  vector<double> centers, relative;
  const int n_rel = 2 * scan.n_steps + 1;
  for (auto speed : speeds)
    for (int c = -scan.n_center_steps; c <= scan.n_center_steps; c++)
      {
        const double center = speed * pow (scan.step, c * (scan.n_steps * 2 + 1));
        centers.push_back (center);
        for (int p = -scan.n_steps; p <= scan.n_steps; p++)
          relative.push_back (pow (scan.step, p) * center / center);    /* SpeedSync::get_jobs is called with speed == centre, :171-175 */
      }
  vector<double> quality (relative.size());
  if (awm_speed_scan (ctx, slot, in.samples + s * in.n_channels, e - s, in.n_channels, in.sample_rate, scan.seconds, centers.data(), int (centers.size()),
                      relative.data(), n_rel, Params::water_delta, quality.data()))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return false;
    }
  for (size_t c = 0; c < centers.size(); c++)
    for (int r = 0; r < n_rel; r++)
      scores.push_back (Score { relative[c * n_rel + r] * centers[c], quality[c * n_rel + r] });
  return true;
}

void
select_n_best_scores (vector<Score>& scores, size_t n)      /* src/wmspeed.cc:487-530 */
{
  std::stable_sort (scores.begin(), scores.end(), [] (const Score& a, const Score& b) { return a.speed < b.speed; });
  auto get_quality = [&] (int pos) { return (pos >= 0 && size_t (pos) < scores.size()) ? scores[pos].quality : 0.0; };
  vector<Score> lmax_scores;
  for (int x = 0; size_t (x) < scores.size(); x++)
    {
      /* single peak: larger than both neighbours; double peak: two equal values larger than their outer neighbours */
      const double q1 = get_quality (x - 1), q2 = get_quality (x), q3 = get_quality (x + 1);
      if (q1 <= q2 && q2 >= q3)
        {
          lmax_scores.push_back (scores[x]);
          x++;     /* the score with quality q3 cannot be a local maximum */
        }
    }
  std::stable_sort (lmax_scores.begin(), lmax_scores.end(), [] (const Score& a, const Score& b) { return a.quality > b.quality; });
  if (lmax_scores.size() > n)
    lmax_scores.resize (n);
  scores = lmax_scores;
}

double
window_cos (double x)
{
  if (fabs (x) > 1)
    return 0;
  return 0.5 * cos (x * M_PI) + 0.5;
}

/* smooth the (noisy) scores with a cosine window and take the maximum of the smooth function (src/wmspeed.cc:377-419) */
double
score_smooth_find_best (const vector<Score>& in_scores, double step, double distance)
{
  auto scores = in_scores;
  std::stable_sort (scores.begin(), scores.end(), [] (const Score& a, const Score& b) { return a.speed < b.speed; });
  double best_speed = 0, best_quality = 0;
  for (double speed = scores.front().speed; speed < scores.back().speed; speed += 0.000001)
    {
      double quality_sum = 0, quality_div = 0;
      for (const auto& s : scores)
        {
          const double w = window_cos ((s.speed - speed) / (step * distance));
          quality_sum += s.quality * w;
          quality_div += w;
        }
      quality_sum /= quality_div;
      if (quality_sum > best_quality)
        {
          best_speed = speed;
          best_quality = quality_sum;
        }
    }
  return best_speed;
}

} // namespace

vector<DetectSpeedResult>
detect_speed (const vector<Key>& key_list, const float *samples, size_t n_frames, int n_channels, int sample_rate, bool print_results, DetectSpeedInfo *info)
{
  vector<DetectSpeedResult> results;
  const double in_seconds = double (n_frames) / sample_rate;
  if (in_seconds < 0.25)          /* the algorithm does not work at all for very short inputs (src/wmspeed.cc:627-633) */
    return results;
  const bool patient = Params::detect_speed_patient;
  SpeedScanParams scan1, scan2, scan3;
  if (patient)
    {
      scan1.seconds = 50; scan1.step = 1.00035;  scan1.n_steps = 11; scan1.n_center_steps = 28;
      scan2.seconds = 50; scan2.step = 1.000175; scan2.n_steps = 1;
    }
  else
    {
      scan1.seconds = 25; scan1.step = 1.0007;   scan1.n_steps = 5;  scan1.n_center_steps = 28;   /* first pass: speed approximately 0.8..1.25 */
      scan2.seconds = 50; scan2.step = 1.00035;  scan2.n_steps = 1;                               /* second pass: improve approximation */
    }
  scan3.seconds = 50; scan3.step = 1.00005; scan3.n_steps = 40;                                   /* third pass: fast refine */
  const double scan3_smooth_distance = 20;
  const double speed_sync_threshold = 0.4;
  const size_t n_best = patient ? 15 : 5;
  const int clip_candidates = 5;

  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return results;
  const Pcm in { samples, n_frames, n_channels, sample_rate, Engine::is_device_pointer (samples) };
  for (const auto& key : key_list)
    {
      const double clip_location = get_best_clip_location (key, in, scan1.seconds, clip_candidates);
      vector<Score> scores;
      /* initial search using a grid */
      if (!run_search (key, in, clip_location, scan1, { 1.0 }, scores))
        break;
      /* improve the N best matches */
      select_n_best_scores (scores, n_best);
      vector<double> speeds;
      for (const auto& s : scores)
        speeds.push_back (s.speed);
      if (speeds.empty() || !run_search (key, in, clip_location, scan2, speeds, scores))
        break;
      /* improve the best match */
      select_n_best_scores (scores, 1);
      if (scores.empty() || !run_search (key, in, clip_location, scan3, { scores[0].speed }, scores))
        break;
      const double best_speed = score_smooth_find_best (scores, 1 - scan3.step, scan3_smooth_distance);
      double best_quality = 0;
      for (const auto& s : scores)
        best_quality = max (best_quality, s.quality);
      if (info)
        {
          info->valid = true;
          info->speed = best_speed;
          info->quality = best_quality;
        }
      if (print_results)
        {
          double delta = -1;
          if (Params::test_speed > 0)
            delta = 100 * fabs (best_speed - Params::test_speed) / Params::test_speed;
          printf ("detect_speed %f %f %.4f\n", best_speed, best_quality, delta);
        }
      if (best_quality > speed_sync_threshold)
        {
          /* speeds closer to 1.0 than this usually work without stretching before decode */
          if (best_speed < 0.9999 || best_speed > 1.0001)
            results.push_back ({ key, best_speed });
        }
    }
  return results;
}

/* resample / resample_ratio (src/resample.cc:52-131) on host buffers */
bool
resample_ratio (const float *in, size_t n_frames, int n_channels, double ratio, vector<float>& out)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx)
    return false;
  const size_t n_out = lrint (double (n_frames) * ratio);
  out.assign (n_out * n_channels, 0.f);
  if (awm_resample (ctx, in, n_frames, n_channels, ratio, 16, out.data(), n_out))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return false;
    }
  return true;
}

/* outputs a streaming resampler (BufferedResamplerImpl::write_frames, src/resample.cc:168-196) has delivered once `fed`
 * frames have been written after the k/2 - 1 frames of pre-roll: every output whose taps are buffered */
size_t
resample_stream_available (size_t fed, double ratio)
{
  return awm_resample_stream_available (fed, ratio, 16);
}

/* ... plus write_trailing_frames (k/2 zero frames, src/resample.cc:198-204): what WavChunkLoader gets for n_in input frames */
size_t
resample_stream_frames (size_t n_in, double ratio)
{
  return awm_resample_stream_frames (n_in, ratio, 16);
}
