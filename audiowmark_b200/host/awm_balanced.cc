// awm_balanced.cc -- see awm_balanced.hh
#include "awm_balanced.hh"
#include "awm_engine.hh"
#include "awm_speed.hh"
#include "awm_tables.hh"
#include "awm_util.hh"

#include <algorithm>
#include <math.h>
#include <string.h>
#include <stdlib.h>

using std::map;
using std::string;
using std::vector;
using namespace get_detail;

namespace balanced {

namespace {

constexpr long kMargin = 6;       // start frames searched beyond the owned ones: the local mean reaches +-20 scores = +-5 start frames

long frames_per_block() { return long (mark_sync_frame_count() + mark_data_frame_count()); }
/* start frames of a chunk: search_approx scores start frames whose block fits into frame_count - 1 analysed frames */
long chunk_starts (const Chunk& c) { return std::max<long> (long (c.count / Params::frame_size) - frames_per_block() - 1, 0); }

/* ---- byte strings: fixed-width little-endian fields, vectors as u32 count + raw elements */
struct Writer
{
  string s;
  template<class T> void put (const T& v) { s.append (reinterpret_cast<const char *> (&v), sizeof (T)); }
  template<class T> void put_vec (const vector<T>& v)
  {
    put (uint32_t (v.size()));
    if (!v.empty())
      s.append (reinterpret_cast<const char *> (v.data()), v.size() * sizeof (T));
  }
};
struct Reader
{
  const string& s;
  size_t pos = 0;
  bool bad = false;
  explicit Reader (const string& str) : s (str) {}
  bool done() const { return pos >= s.size(); }
  template<class T> T get()
  {
    T v {};
    if (pos + sizeof (T) > s.size())
      {
        bad = true;
        return v;
      }
    memcpy (&v, s.data() + pos, sizeof (T));
    pos += sizeof (T);
    return v;
  }
  template<class T> void skip_vec()
  {
    const uint32_t n = get<uint32_t>();
    if (bad || pos + size_t (n) * sizeof (T) > s.size())
      bad = true;
    else
      pos += size_t (n) * sizeof (T);
  }
  const char *raw (size_t n)
  {
    if (bad || pos + n > s.size())
      {
        bad = true;
        return nullptr;
      }
    const char *p = s.data() + pos;
    pos += n;
    return p;
  }
  template<class T> vector<T> get_vec()
  {
    const uint32_t n = get<uint32_t>();
    vector<T> v;
    if (bad || pos + size_t (n) * sizeof (T) > s.size())
      {
        bad = true;
        return v;
      }
    v.resize (n);
    if (n)
      memcpy (v.data(), s.data() + pos, size_t (n) * sizeof (T));
    pos += size_t (n) * sizeof (T);
    return v;
  }
};

} // namespace

vector<Chunk>
chunk_plan (size_t n_frames, int sample_rate)
{
  vector<Chunk> plan;
  if (!n_frames)
    return plan;
  size_t max_frames, overlap;
  chunk_geometry (sample_rate, max_frames, overlap);
  size_t start = 0, end = std::min (max_frames, n_frames);
  double time_offset = 0;
  bool eof = end < max_frames;
  for (;;)
    {
      plan.push_back (Chunk { start, end - start, time_offset });
      if (eof)
        break;
      time_offset += double (end - start - overlap) / sample_rate;
      start = end - overlap;
      const size_t new_end = std::min (start + max_frames, n_frames);
      eof = (new_end - start) < max_frames;
      end = new_end;
    }
  return plan;
}

size_t
owner_span (size_t n_total, int world)
{
  const size_t per = (n_total + world - 1) / world, F = Params::frame_size;
  return (per + F - 1) / F * F;
}

vector<Slice>
rank_slices (const vector<Chunk>& plan, int rank, int world, size_t n_total)
{
  const long F = Params::frame_size, T = frames_per_block();
  const long long span = owner_span (n_total, world);
  vector<Slice> out;
  for (size_t c = 0; c < plan.size(); c++)
    {
      const long n_starts = chunk_starts (plan[c]);
      if (!n_starts)
        continue;
      const long long cs = plan[c].first;
      /* start frame s sits at stream position cs + s * 1024; a position belongs to rank position / span (the last rank takes the rest) */
      auto first_start_at = [&] (long long pos) { return pos <= cs ? 0L : long ((pos - cs + F - 1) / F); };
      Slice sl;
      sl.chunk = int (c);
      sl.sa = std::min (first_start_at ((long long) rank * span), n_starts);
      sl.sb = rank == world - 1 ? n_starts : std::min (first_start_at ((long long) (rank + 1) * span), n_starts);
      if (sl.sb <= sl.sa)
        continue;
      sl.a = std::max (sl.sa - kMargin, 0L);
      sl.b = std::min (sl.sb + kMargin, n_starts);
      sl.lo = size_t (cs + sl.a * F);
      sl.hi = sl.b == n_starts ? size_t (cs) + plan[c].count : size_t (cs + (sl.b + T + 1) * F);     // the last slice keeps the chunk's partial tail frame
      out.push_back (sl);
    }
  return out;
}

int
owner_of (const vector<Chunk>& plan, size_t n_total, int world, int chunk, uint64_t index)
{
  const long n_starts = chunk_starts (plan[chunk]);
  const long s = std::min<long> (long (index / Params::frame_size), std::max (n_starts - 1, 0L));
  const size_t pos = plan[chunk].first + size_t (s) * Params::frame_size;
  return int (std::min<size_t> (pos / owner_span (n_total, world), world - 1));
}

bool
rate_supported (int sample_rate)
{
  if (sample_rate <= 0)
    return false;
  const double up = double (Params::mark_sample_rate) / sample_rate, down = double (sample_rate) / Params::mark_sample_rate;
  return up > 1.0 / 64 && up < 64 && down > 1.0 / 64 && down < 64;
}

size_t
mark_frames (size_t n_total, int sample_rate)
{
  return sample_rate == Params::mark_sample_rate ? n_total : resample_stream_frames (n_total, double (Params::mark_sample_rate) / sample_rate);
}

void
input_range (const vector<Slice>& slices, size_t n_total, int sample_rate, size_t& first, size_t& end)
{
  first = end = 0;
  if (slices.empty())
    return;
  size_t lo = slices[0].lo, hi = slices[0].hi;
  for (const Slice& sl : slices)
    {
      lo = std::min (lo, sl.lo);
      hi = std::max (hi, sl.hi);
    }
  if (sample_rate == Params::mark_sample_rate)
    {
      first = lo;
      end = hi;
      return;
    }
  uint64_t t0, t1;
  awm_resample_taps (n_total, double (Params::mark_sample_rate) / sample_rate, 16, lo, hi - lo, &t0, &t1);
  /* one frame on each side: the range stays whole even if a build evaluates the tap positions with a fused multiply-add */
  first = t0 ? size_t (t0) - 1 : 0;
  end = std::min<size_t> (size_t (t1) + 1, n_total);
}

/* ---------------------------------------------------------------------------------------------------------------- Get */

Get::Get (int rank, int world, size_t n_total, const float *pcm, const int16_t *pcm16, size_t pcm_start, size_t pcm_frames, int channels,
          int sample_rate, const Key& key) :
  m_rank (rank), m_world (world), m_channels (channels), m_rate (sample_rate), m_n_total (n_total), m_pcm_start (pcm_start), m_pcm_frames (pcm_frames), m_key (key)
{
  awm_ctx *ctx = Engine::ctx();
  if (!ctx || !rate_supported (sample_rate) || (!pcm && !pcm16))
    {
      error ("audiowmark: sharded get needs a CUDA device and input at a sample rate of %d Hz / 64 .. %d Hz * 64 (exclusive), not %d Hz\n",
             Params::mark_sample_rate, Params::mark_sample_rate, sample_rate);
      return;
    }
  m_slot = Engine::key_slot (key);
  if (m_slot < 0)
    return;
  const bool resampled = sample_rate != Params::mark_sample_rate;
  const double ratio = double (Params::mark_sample_rate) / sample_rate;
  m_n_mark = mark_frames (n_total, sample_rate);
  /* inputs short enough for the reference's ClipDecoder (src/wmget.cc:764-884: fewer than 3.1 blocks) are a few seconds of work on one
   * GPU; the sharded driver only runs the block decoder, so it refuses them instead of returning a document without CLIP patterns */
  if (double (m_n_mark / Params::frame_size) < double (frames_per_block()) * 3.1)
    {
      error ("audiowmark: sharded get: input of %zu frames (%zu at %d Hz) is clip sized (under 3.1 blocks); use the single GPU get\n", n_total,
             m_n_mark, Params::mark_sample_rate);
      return;
    }
  m_plan = chunk_plan (m_n_mark, Params::mark_sample_rate);
  m_slices = rank_slices (m_plan, rank, world, m_n_mark);
  for (int r = 0; r < world; r++)                // which ranks search a slice of which chunk (ascending rank order)
    for (const Slice& sl : rank_slices (m_plan, r, world, m_n_mark))
      m_sharers[sl.chunk].push_back (r);
  if (!resampled)
    {
      for (const Slice& sl : m_slices)
        if (sl.lo < pcm_start || sl.hi > pcm_start + pcm_frames)
          {
            error ("audiowmark: sharded get: rank %d needs stream frames [%zu, %zu), its buffer holds [%zu, %zu)\n", rank, sl.lo, sl.hi, pcm_start, pcm_start + pcm_frames);
            return;
          }
    }
  else if (!m_slices.empty())
    {
      size_t first, end;
      input_range (m_slices, n_total, sample_rate, first, end);
      if (first < pcm_start || end > pcm_start + pcm_frames)
        {
          error ("audiowmark: sharded get: rank %d needs stream frames [%zu, %zu) at %d Hz, its buffer holds [%zu, %zu)\n", rank, first, end, sample_rate,
                 pcm_start, pcm_start + pcm_frames);
          return;
        }
      size_t lo = m_slices[0].lo, hi = m_slices[0].hi;        // chunks overlap: a later slice can begin before an earlier one
      for (const Slice& sl : m_slices)
        {
          lo = std::min (lo, sl.lo);
          hi = std::max (hi, sl.hi);
        }
      m_mark_lo = m_mark_done = lo;
      char why[240];
      if (awm_resample_range_validate (pcm_start, pcm_frames, n_total, channels, ratio, 16, m_mark_lo, hi - m_mark_lo, why, sizeof (why)))
        {
          error ("audiowmark: sharded get: %s\n", why);
          return;
        }
      void *buf = nullptr;
      if (awm_device_alloc (ctx, (hi - m_mark_lo) * channels * sizeof (float), &buf))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return;
        }
      m_mark = static_cast<float *> (buf);
    }
  /* one upload for all stages, piece by piece: the stages bind slices of the device copy, a slice waits only for the pieces it reads */
  if (pcm && Engine::is_device_pointer (pcm))
    m_dev = pcm;
  else
    {
      if (awm_pcm_stage (ctx, pcm16 ? static_cast<const void *> (pcm16) : pcm, pcm16 ? 1 : 0, pcm_frames, channels, kStagePiece, &m_dev))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return;
        }
      m_staged = true;
    }
  m_ok = true;
}

Get::~Get()
{
  if (m_mark)
    awm_device_free (Engine::ctx(), m_mark);
}

const Slice *
Get::my_slice (int chunk) const
{
  for (const Slice& sl : m_slices)
    if (sl.chunk == chunk)
      return &sl;
  return nullptr;
}

bool
Get::bind (const Slice& sl)
{
  awm_ctx *ctx = Engine::ctx();
  if (!m_mark)
    {
      if ((m_staged && awm_pcm_stage_wait (ctx, sl.hi - m_pcm_start))
          || awm_pcm_bind (ctx, m_dev + (sl.lo - m_pcm_start) * m_channels, sl.hi - sl.lo, m_channels, 0, 0))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return false;
        }
      return true;
    }
  /* [m_mark_lo, m_mark_done) is resampled: compute only the outputs no earlier bind produced, after the input pieces their taps
   * read have arrived */
  if (sl.hi > m_mark_done)
    {
      const double ratio = double (Params::mark_sample_rate) / m_rate;
      uint64_t t0, t1;
      awm_resample_taps (m_n_total, ratio, 16, m_mark_done, sl.hi - m_mark_done, &t0, &t1);
      if ((m_staged && awm_pcm_stage_wait (ctx, std::max<size_t> (t1, m_pcm_start) - m_pcm_start))
          || awm_resample_range (ctx, m_dev, m_pcm_start, m_pcm_frames, m_n_total, m_channels, ratio, 16, m_mark + (m_mark_done - m_mark_lo) * m_channels,
                                 m_mark_done, sl.hi - m_mark_done))
        {
          error ("audiowmark: %s\n", awm_last_error (ctx));
          return false;
        }
      m_mark_done = sl.hi;
    }
  if (awm_pcm_bind (ctx, m_mark + (sl.lo - m_mark_lo) * m_channels, sl.hi - sl.lo, m_channels, 0, 0))
    {
      error ("audiowmark: %s\n", awm_last_error (ctx));
      return false;
    }
  return true;
}

namespace {
/* AWM_TRACE=2: time stamps inside the stages (rank 0) */
struct FineTrace
{
  bool on;
  double t;
  explicit FineTrace (int rank) : on (rank == 0 && getenv ("AWM_TRACE") && atoi (getenv ("AWM_TRACE")) >= 2), t (get_time()) {}
  void mark (const char *what, long detail = -1)
  {
    if (!on)
      return;
    const double now = get_time();
    fprintf (stderr, "[trace]     %s%s %.3f ms\n", what, detail >= 0 ? string_printf (" %ld", detail).c_str() : "", (now - t) * 1e3);
    t = now;
  }
};
}

/* ---- stage 1: approximate search on my slices -> the local maxima above an (adaptive) floor, in chunk coordinates
 * payload: per slice { i32 chunk, f64 floor, vec<awm_search_score> peaks } */
bool
Get::stage_peaks (const map<int, double>& floors, string& out)
{
  awm_ctx *ctx = Engine::ctx();
  const double thr1 = Params::sync_threshold2 * 0.75;
  const size_t F = Params::frame_size;
  static vector<awm_search_score> buf (size_t (1) << 18);
  Writer w;
  FineTrace ft (m_rank);
  for (const Slice& sl : m_slices)
    {
      if (!floors.empty() && !floors.count (sl.chunk))
        continue;                                               // a retry concerns some chunks only
      if (!bind (sl))
        return false;
      size_t n_scores = 0;
      if (awm_sync_approx (ctx, m_slot, AWM_MODE_BLOCK, 0, (sl.hi - sl.lo) * m_channels, Params::water_delta, nullptr, 0, &n_scores))
        {
          error ("audiowmark: sync search failed: %s\n", awm_last_error (ctx));
          return false;
        }
      ft.mark ("approx launched, slice of chunk", sl.chunk);
      /* lowered step by step until the slice has three times n-best maxima above the floor (the selection keeps everything above the
       * threshold, or the n best: with that many in hand it can decide; if masking leaves too few the run asks again for all maxima).
       * The steps are fine enough that a list does not jump from a few dozen watermark peaks to thousands of noise peaks -- every rank
       * sorts and scans the gathered lists of ALL chunks, so short lists keep that replicated work small */
      vector<double> seq = { thr1, thr1 * 0.8, thr1 * 0.6, thr1 * 0.5, thr1 * 0.4, thr1 * 0.35, thr1 * 0.3, thr1 * 0.25, thr1 * 0.2, thr1 * 0.15, thr1 * 0.1,
                             thr1 * 0.05, -1.0 };
      const size_t enough = size_t (std::max (3 * Params::get_n_best, 24));
      if (floors.count (sl.chunk))
        seq = { floors.at (sl.chunk) };
      vector<awm_search_score> own;
      double used = -1;
      for (double floor_q : seq)
        {
          size_t n = 0;
          if (awm_sync_peaks (ctx, floor_q, buf.data(), buf.size(), &n) || n > buf.size())
            {
              error ("audiowmark: sync search failed: too many peaks above floor %g\n", floor_q);
              return false;
            }
          own.clear();
          const uint64_t lo = uint64_t (sl.sa - sl.a) * F, hi = uint64_t (sl.sb - sl.a) * F;
          for (size_t i = 0; i < n; i++)
            if (buf[i].index >= lo && buf[i].index < hi)
              own.push_back (buf[i]);
          used = floor_q;
          ft.mark ("peaks above floor:", long (n));
          if (own.size() >= enough || floor_q < 0)
            break;
        }
      for (auto& p : own)
        p.index += uint64_t (sl.a) * F;
      w.put (int32_t (sl.chunk));
      w.put (used);
      w.put_vec (own);
    }
  out.swap (w.s);
  return true;
}

/* ---- stage 2: candidate selection per chunk from everybody's peaks (identical on every rank); chunks whose lists were too short
 * are named in retry_floors (ask for all maxima and select again) */
bool
Get::stage_select (const vector<string>& all, map<int, double>& retry_floors)
{
  map<int, std::pair<double, vector<awm_search_score>>> per_chunk;
  for (const string& payload : all)
    {
      Reader r (payload);
      while (!r.done())
        {
          const int chunk = r.get<int32_t>();
          const double floor_q = r.get<double>();
          const vector<awm_search_score> pk = r.get_vec<awm_search_score>();
          if (r.bad)
            return false;
          auto it = per_chunk.find (chunk);
          if (it == per_chunk.end())
            per_chunk[chunk] = { floor_q, pk };
          else
            {
              it->second.first = std::max (it->second.first, floor_q);
              it->second.second.insert (it->second.second.end(), pk.begin(), pk.end());
            }
        }
    }
  retry_floors.clear();
  for (auto& kv : per_chunk)
    {
      vector<awm_search_score>& pk = kv.second.second;
      std::stable_sort (pk.begin(), pk.end(), [] (const awm_search_score& x, const awm_search_score& y) { return x.index < y.index; });
      vector<awm_search_score> sel;
      const int r = select_candidates_from_peaks (pk.data(), pk.size(), kv.second.first, Params::sync_threshold2 * 0.75, sel);
      if (r <= 0 && kv.second.first >= 0)
        retry_floors[kv.first] = -1.0;
      m_cands[kv.first] = sel;
    }
  return true;
}

/* ---- stage 3: refine the candidates I own and decode them to soft bits right away (the threshold2 / n-best selection that
 * follows needs everybody's refined scores; decoding the few candidates it will drop costs less than another exchange)
 * payload: per chunk { i32 chunk, vec<u32> position in the candidate list, vec<awm_search_score> refined, vec<i32> valid, vec<f32> soft bits } */
bool
Get::stage_refine_decode (string& out)
{
  awm_ctx *ctx = Engine::ctx();
  const size_t F = Params::frame_size;
  const size_t n_coded = code_size (ConvBlockType::a, Params::payload_size);
  Writer w;
  for (const auto& kv : m_cands)
    {
      const int chunk = kv.first;
      const Slice *sl = my_slice (chunk);
      if (!sl)
        continue;
      vector<uint32_t> mine;
      vector<awm_search_score> part;
      for (size_t i = 0; i < kv.second.size(); i++)
        if (owner_of (m_plan, m_n_mark, m_world, chunk, kv.second[i].index) == m_rank)
          {
            mine.push_back (uint32_t (i));
            part.push_back (kv.second[i]);
          }
      if (mine.empty())
        continue;
      if (!bind (*sl))
        return false;
      const uint64_t shift = uint64_t (sl->a) * F;            // chunk coordinates -> slice coordinates
      for (auto& p : part)
        p.index -= shift;
      if (awm_sync_refine (ctx, m_slot, AWM_MODE_BLOCK, 0, (sl->hi - sl->lo) * m_channels, Params::water_delta, part.data(), part.size()))
        {
          error ("audiowmark: sync search failed: %s\n", awm_last_error (ctx));
          return false;
        }
      vector<uint64_t> idx (part.size());
      for (size_t i = 0; i < part.size(); i++)
        idx[i] = part[i].index;
      vector<float> soft (part.size() * n_coded);
      vector<int32_t> valid (part.size());
      /* fft_range validity is decided against the CHUNK length: a slice either reaches the chunk end or is long enough */
      if (awm_decode_blocks (ctx, m_slot, idx.data(), idx.size(), soft.data(), valid.data()))
        {
          error ("audiowmark: block decode failed: %s\n", awm_last_error (ctx));
          return false;
        }
      for (auto& p : part)
        p.index += shift;
      w.put (int32_t (chunk));
      w.put_vec (mine);
      w.put_vec (part);
      w.put_vec (valid);
      w.put_vec (soft);
    }
  out.swap (w.s);
  return true;
}

/* ---- stage 4: the final scores (threshold2 / n-best on the refined candidates) and the code words of the block decoder, for the
 * chunks this rank searched a slice of; the ranks that share a chunk build the same job list and deal it out among themselves
 * (job j of the chunk goes to the (j mod k)-th of its k ranks), so the host work of a rank does not grow with the length of the stream
 * and the Viterbi launches stay balanced.  What rank 0 needs to print a decoded word travels with it:
 * payload: per job { i32 chunk, u32 job number inside the chunk, f64 time, u64 index, f64 quality, u8 score block type, u8 pattern type,
 *                    u16 pad, f32 error, u8 bits[n_msg] } */
bool
Get::stage_viterbi (const vector<string>& all, string& out)
{
  const size_t n_coded = code_size (ConvBlockType::a, Params::payload_size);
  struct Refined { vector<awm_search_score> score; vector<vector<float>> soft; vector<int> valid; };
  map<int, Refined> refined;
  for (const Slice& sl : m_slices)
    {
      auto it = m_cands.find (sl.chunk);
      if (it == m_cands.end())
        continue;
      Refined& r = refined[sl.chunk];
      r.score = it->second;
      r.soft.assign (it->second.size(), vector<float>());
      r.valid.assign (it->second.size(), 0);
    }
  for (const string& payload : all)
    {
      Reader r (payload);
      while (!r.done())
        {
          const int chunk = r.get<int32_t>();
          if (!refined.count (chunk))               // not my chunk: step over the record
            {
              r.skip_vec<uint32_t>();
              r.skip_vec<awm_search_score>();
              r.skip_vec<int32_t>();
              r.skip_vec<float>();
              if (r.bad)
                return false;
              continue;
            }
          const vector<uint32_t> pos = r.get_vec<uint32_t>();
          const vector<awm_search_score> sc = r.get_vec<awm_search_score>();
          const vector<int32_t> valid = r.get_vec<int32_t>();
          const vector<float> soft = r.get_vec<float>();
          if (r.bad || sc.size() != pos.size() || valid.size() != pos.size() || soft.size() != pos.size() * n_coded)
            return false;
          Refined& dst = refined[chunk];
          for (size_t i = 0; i < pos.size(); i++)
            {
              if (pos[i] >= dst.score.size())
                return false;
              dst.score[pos[i]] = sc[i];
              dst.valid[pos[i]] = valid[i];
              dst.soft[pos[i]].assign (soft.begin() + i * n_coded, soft.begin() + (i + 1) * n_coded);
            }
        }
    }
  m_jobs.clear();
  vector<uint32_t> job_number;                   // position of m_jobs[i] in its chunk's job list
  for (auto& kv : refined)                       // chunk order
    {
      Refined& r = kv.second;
      vector<awm_search_score> scores = r.score;
      vector<SyncFinder::Score> final_scores;
      select_final_scores (scores, final_scores);
      /* a final score is one of the refined candidates: find its soft bits (same index, same |q - mean| and sign) */
      vector<vector<float>> soft (final_scores.size());
      vector<int> valid (final_scores.size(), 0);
      vector<char> taken (r.score.size(), 0);
      for (size_t f = 0; f < final_scores.size(); f++)
        for (size_t c = 0; c < r.score.size(); c++)
          {
            const double q = r.score[c].raw_quality - r.score[c].local_mean;
            if (!taken[c] && r.score[c].index == final_scores[f].index && fabs (q) == final_scores[f].quality
                && (q > 0 ? ConvBlockType::a : ConvBlockType::b) == final_scores[f].block_type)
              {
                taken[c] = 1;
                soft[f].swap (r.soft[c]);
                valid[f] = r.valid[c] && !soft[f].empty();
                break;
              }
          }
      vector<VitJob> chunk_jobs;
      build_block_jobs (m_key, final_scores, soft, valid, Params::mark_sample_rate, kv.first, 1.0, chunk_jobs);
      const vector<int>& sharers = m_sharers[kv.first];
      for (size_t j = 0; j < chunk_jobs.size(); j++)
        if (sharers[j % sharers.size()] == m_rank)
          {
            m_jobs.push_back (std::move (chunk_jobs[j]));
            job_number.push_back (uint32_t (j));
          }
    }
  vector<const VitJob *> mine;
  for (const VitJob& j : m_jobs)
    mine.push_back (&j);
  vector<uint8_t> bits;
  vector<float> err;
  if (!viterbi_decode (mine, bits, err))
    return false;
  const size_t n_msg = code_message_bits();
  Writer w;
  for (size_t i = 0; i < m_jobs.size(); i++)
    {
      const VitJob& j = m_jobs[i];
      w.put (int32_t (j.chunk));
      w.put (job_number[i]);
      w.put (double (j.time));
      w.put (uint64_t (j.score.index));
      w.put (double (j.score.quality));
      w.put (uint8_t (j.score.block_type == ConvBlockType::a ? AWM_BLOCK_A : j.score.block_type == ConvBlockType::b ? AWM_BLOCK_B : AWM_BLOCK_AB));
      w.put (uint8_t (j.type));
      w.put (uint16_t (0));
      w.put (float (err[i]));
      w.s.append (reinterpret_cast<const char *> (bits.data() + i * n_msg), n_msg);
    }
  out.swap (w.s);
  return true;
}

/* ---- stage 5 (rank 0): decoded words -> patterns per chunk, in the order the block decoder queued them -> the reference's merge in
 * chunk order */
bool
Get::stage_merge (const vector<string>& all, ResultSet& result)
{
  const size_t n_msg = code_message_bits();
  struct Word { int chunk; uint32_t number; VitJob job; float err; const uint8_t *bits; };
  vector<Word> words;
  for (const string& payload : all)
    {
      Reader r (payload);
      while (!r.done())
        {
          Word wd;
          wd.chunk = r.get<int32_t>();
          wd.number = r.get<uint32_t>();
          wd.job.time = r.get<double>();
          wd.job.score.index = size_t (r.get<uint64_t>());
          wd.job.score.quality = r.get<double>();
          const uint8_t bt = r.get<uint8_t>();
          wd.job.score.block_type = bt == AWM_BLOCK_A ? ConvBlockType::a : bt == AWM_BLOCK_B ? ConvBlockType::b : ConvBlockType::ab;
          wd.job.type = ResultSet::Type (r.get<uint8_t>());
          r.get<uint16_t>();
          wd.err = r.get<float>();
          wd.bits = reinterpret_cast<const uint8_t *> (r.raw (n_msg));
          if (r.bad || wd.chunk < 0 || wd.chunk >= int (m_plan.size()))
            return false;
          wd.job.block_type = wd.job.score.block_type;
          wd.job.key = m_key;
          wd.job.chunk = wd.chunk;
          wd.job.speed = 1.0;
          words.push_back (std::move (wd));
        }
    }
  std::stable_sort (words.begin(), words.end(), [] (const Word& x, const Word& y) { return x.chunk != y.chunk ? x.chunk < y.chunk : x.number < y.number; });
  vector<ResultSet> chunk_results (m_plan.size());
  for (const Word& wd : words)
    add_decoded_pattern (wd.job, wd.bits, wd.err, chunk_results[wd.chunk]);
  for (size_t c = 0; c < chunk_results.size(); c++)
    {
      chunk_results[c].apply_time_offset (m_plan[c].time_offset);
      result.merge (chunk_results[c]);
    }
  result.sort ({ m_key });
  return true;
}

bool
Get::run (const Exchange& exchange, ResultSet& result)
{
  if (!m_ok)
    return false;
  const bool trace = getenv ("AWM_TRACE") != nullptr;
  double t = get_time();
  auto mark = [&] (const char *what)
    {
      if (trace)
        {
          const double now = get_time();
          fprintf (stderr, "[trace] rank %d sharded get: %s %.2f ms\n", m_rank, what, (now - t) * 1e3);
          t = now;
        }
    };
  string mine;
  vector<string> all;
  map<int, double> retry;
  FineTrace ft (m_rank);
  if (!stage_peaks ({}, mine))
    return false;
  ft.mark ("stage_peaks, payload bytes", long (mine.size()));
  if (!exchange (mine, all))
    return false;
  ft.mark ("exchange");
  if (!stage_select (all, retry))
    return false;
  ft.mark ("stage_select, chunks to retry:", long (retry.size()));
  mark ("peaks + select");
  if (!retry.empty())                            // identical on every rank: all of them take part in the second round
    {
      map<int, double> none;
      if (!stage_peaks (retry, mine) || !exchange (mine, all) || !stage_select (all, none))
        return false;
      mark ("retry");
    }
  if (!stage_refine_decode (mine) || !exchange (mine, all))
    return false;
  mark ("refine + soft bits");
  if (!stage_viterbi (all, mine) || !exchange (mine, all))
    return false;
  mark ("viterbi");
  if (m_rank == 0 && !stage_merge (all, result))
    return false;
  mark ("merge");
  return true;
}

} // namespace balanced
