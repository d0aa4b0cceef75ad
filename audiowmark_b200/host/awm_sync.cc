// awm_sync.cc -- SyncFinder::search (reference src/syncfinder.cc:487-558): the scoring sweeps run on
// the GPU (awm_sync_approx = search_approx, awm_sync_refine = search_refine); candidate selection
// (local maxima, false-positive masking, threshold / n-best) stays on the host and follows the
// reference's comparison operators exactly (src/syncfinder.cc:258-391).
#include "awm_wm.hh"
#include "awm_engine.hh"
#include "awm_util.hh"

#include <algorithm>
#include <math.h>
#include <stdlib.h>

using std::vector;

namespace {

typedef awm_search_score SearchScore;
inline double abs_quality (const SearchScore& s) { return fabs (s.raw_quality - s.local_mean); }
constexpr int local_mean_distance = 20;

/* The selection chain of SyncFinder::search in the reference's own order of operations (src/syncfinder.cc:258-281 local maxima,
 * :292-332 false-positive mask, :364-383 threshold / n-best): build the list of maxima, filter it, sort the filtered list by
 * descending |q - mean| with std::sort, cut.  std::sort is not stable, so which of several EQUAL scores survive a cut by count
 * depends on the element sequence handed to it; feeding it the same sequence as the reference does (maxima in index order)
 * reproduces the reference's choice (same libstdc++).  This matters for degenerate input only -- digital silence gives
 * |q - mean| == 0 for every start frame -- and costs a few ms per chunk, so the lazy paths below are used whenever no tie
 * straddles the cut. */
void
select_from_maxima_reference_order (const vector<SearchScore>& maxima, double threshold, vector<SearchScore>& out)
{
  constexpr int reach = local_mean_distance + 3;  // in list positions and in search steps
  out.clear();
  const int nm = int (maxima.size());
  for (int i = 0; i < nm; i++)
    {
      const double qi = abs_quality (maxima[i]);
      const bool neg_i = maxima[i].raw_quality - maxima[i].local_mean < 0;
      bool drop = false;
      for (int j = std::max (0, i - reach); j <= std::min (nm - 1, i + reach) && !drop; j++)
        {
          if (j == i)
            continue;
          const int steps = std::abs (int (maxima[i].index) - int (maxima[j].index)) / Params::sync_search_step;
          const bool neg_j = maxima[j].raw_quality - maxima[j].local_mean < 0;
          drop = steps <= reach && neg_i != neg_j && abs_quality (maxima[j]) > qi * 3;
        }
      if (!drop)
        out.push_back (maxima[i]);
    }
  std::sort (out.begin(), out.end(), [] (const SearchScore& a, const SearchScore& b) { return abs_quality (a) > abs_quality (b); });
  size_t above = 0;
  while (above < out.size() && abs_quality (out[above]) > threshold)
    above++;
  if (int (above) >= Params::get_n_best)
    out.resize (above);
  else if (int (out.size()) > Params::get_n_best)
    out.resize (Params::get_n_best);
}

/* the same from the complete score list of a chunk (sorted by index) */
void
select_candidates_reference_order (const SearchScore *sc, size_t n, double threshold, vector<SearchScore>& out)
{
  vector<SearchScore> maxima;
  maxima.reserve (n / 2 + 1);
  for (size_t i = 0; i < n; i++)
    {
      const double q = abs_quality (sc[i]);
      const double before = i ? abs_quality (sc[i - 1]) : 0.0;
      const double after = i + 1 < n ? abs_quality (sc[i + 1]) : 0.0;
      if (q < before || q < after)
        continue;
      maxima.push_back (sc[i]);
      i++;                                        // its right neighbour is never examined
    }
  select_from_maxima_reference_order (maxima, threshold, out);
}

/* scores sorted by descending |q - mean|: equal scores on both sides of a cut after the first n */
bool
tie_at (const vector<SearchScore>& sorted, size_t n)
{
  return n && sorted.size() > n && abs_quality (sorted[n - 1]) == abs_quality (sorted[n]);
}

} // namespace

/* Candidate selection on a list of local maxima (sorted by index) that is complete above `floor_q`
 * (= sync_select_local_maxima + sync_mask_avg_false_positives + sync_select_threshold_and_n_best, src/syncfinder.cc:258-383).
 * Why looking at the strongest peaks only is enough: a peak can only be masked by a 3x stronger one, which is above the floor
 * as well; peaks within 23 search steps of each other are always within 23 list positions; and if the scan stops before it
 * would need a peak at or below the floor, every peak the reference would select has been seen.
 * Returns 1: `out` is final.  0: the list was too short, ask again with a lower floor.  -1: peaks of EQUAL strength sit on both
 * sides of the n-best cut, which of them the reference keeps is decided by std::sort on the full list of maxima -- ask for all
 * maxima (floor < 0); with a complete list the reference's order of operations is followed literally.
 * truncate_n > 0: the caller keeps only the truncate_n strongest of `out` (CLIP mode).  Which of several EQUAL scores on that cut
 * survive is again decided by std::sort, over the reference's own sequence, so a tie there also returns -1. */
int
select_candidates_from_peaks (const awm_search_score *peaks, size_t n, double floor_q, double threshold, vector<awm_search_score>& out,
                              size_t truncate_n)
{
  constexpr int    mask_distance = local_mean_distance + 3;
  constexpr double mask_factor   = 3;
  /* "skip the score after a maximum": of directly adjacent scores that are both maxima (equal quality) the one
   * right after a selected maximum is not looked at */
  vector<SearchScore> pk;
  pk.reserve (n);
  bool prev_taken = false;
  uint64_t prev_index = ~uint64_t (0);
  for (size_t i = 0; i < n; i++)
    {
      const bool adjacent = peaks[i].index == prev_index + Params::sync_search_step;
      const bool take = !(adjacent && prev_taken);
      if (take)
        pk.push_back (peaks[i]);
      prev_taken = take;
      prev_index = peaks[i].index;
    }
  if (floor_q < 0)
    {
      select_from_maxima_reference_order (pk, threshold, out);
      return 1;
    }
  const size_t np = pk.size();
  vector<uint32_t> order (np);
  for (size_t k = 0; k < np; k++)
    order[k] = k;
  std::sort (order.begin(), order.end(), [&] (uint32_t a, uint32_t b) { return abs_quality (pk[a]) > abs_quality (pk[b]); });
  auto sign = [&] (size_t k) { return (pk[k].raw_quality - pk[k].local_mean < 0) ? -1 : 1; };
  auto masked = [&] (int i)
    {
      const double q = abs_quality (pk[i]);
      bool mask = false;
      for (int j = i - 1; j >= 0 && !mask && int (pk[i].index - pk[j].index) / Params::sync_search_step <= mask_distance; j--)
        mask = abs_quality (pk[j]) > q * mask_factor && sign (j) != sign (i);
      for (int j = i + 1; j < int (np) && !mask && int (pk[j].index - pk[i].index) / Params::sync_search_step <= mask_distance; j++)
        mask = abs_quality (pk[j]) > q * mask_factor && sign (j) != sign (i);
      return mask;
    };
  out.clear();
  for (size_t k = 0; k < np; k++)
    {
      const int i = order[k];
      const double q = abs_quality (pk[i]);
      if (q <= threshold && int (out.size()) >= Params::get_n_best)
        {
          /* cut.  By value if more than n_best peaks lie above the threshold; by count otherwise -- then the next peak that
           * would have been taken must be strictly weaker than the last one kept */
          if (int (out.size()) == Params::get_n_best && q == abs_quality (out.back()) && abs_quality (out.back()) <= threshold)
            {
              for (size_t kk = k; kk < np && abs_quality (pk[order[kk]]) == q; kk++)
                if (!masked (order[kk]))
                  return -1;
            }
          return tie_at (out, truncate_n) ? -1 : 1;
        }
      if (q <= floor_q)
        return 0;                               // peaks at or below the floor may be missing from the list
      if (!masked (i))
        out.push_back (pk[i]);
    }
  /* list exhausted: it held only the peaks above the floor; final if n_best unmasked peaks lie above it */
  if (int (out.size()) < Params::get_n_best)
    return 0;
  return tie_at (out, truncate_n) ? -1 : 1;
}

namespace {

/* the local maxima come from the GPU (awm_sync_peaks); only those above a floor are transferred, the floor is lowered
 * until the selection is complete */
bool
select_candidates_gpu (awm_ctx *ctx, double threshold, size_t truncate_n, vector<SearchScore>& out)
{
  static SearchScore *peaks = nullptr;
  static const size_t max_peaks = 1 << 18;    // a 30 minute chunk has at most 150 584 local maxima
  if (!peaks)
    peaks = static_cast<SearchScore *> (awm_host_alloc (max_peaks * sizeof (SearchScore)));
  if (!peaks)
    return false;
  const double floors[] = { threshold, threshold * 0.6, threshold * 0.35, threshold * 0.15, 0.0, -1.0 };
  for (double floor_q : floors)
    {
      size_t n = 0;
      if (awm_sync_peaks (ctx, floor_q, peaks, max_peaks, &n))
        return false;
      if (n > max_peaks)
        return false;                             // caller falls back to the full score list
      const int r = select_candidates_from_peaks (peaks, n, floor_q, threshold, out, truncate_n);
      if (r > 0)
        return true;
      if (r < 0 && floor_q >= 0)                  // a tie on the cut: only the complete list of maxima decides it
        {
          if (awm_sync_peaks (ctx, -1.0, peaks, max_peaks, &n) || n > max_peaks)
            return false;
          return select_candidates_from_peaks (peaks, n, -1.0, threshold, out, truncate_n) > 0;
        }
    }
  return false;
}

void
select_threshold_and_n_best (vector<SearchScore>& scores, double threshold)
{
  std::sort (scores.begin(), scores.end(), [] (const SearchScore& a, const SearchScore& b) { return abs_quality (a) > abs_quality (b); });
  int i = 0;
  while (i < int (scores.size()) && abs_quality (scores[i]) > threshold)
    i++;
  if (i >= Params::get_n_best)
    scores.resize (i);                        // all matches above the threshold
  else if (int (scores.size()) > Params::get_n_best)
    scores.resize (Params::get_n_best);       // otherwise the n best
}

void
select_truncate_n (vector<SearchScore>& scores, size_t n)
{
  std::sort (scores.begin(), scores.end(), [] (const SearchScore& a, const SearchScore& b) { return abs_quality (a) > abs_quality (b); });
  if (scores.size() > n)
    scores.resize (n);
}

} // namespace

/* threshold2 / n-best selection of the refined scores + conversion to Score (src/syncfinder.cc:533-555) */
void
select_final_scores (vector<awm_search_score>& scores, vector<SyncFinder::Score>& out)
{
  std::sort (scores.begin(), scores.end(), [] (const SearchScore& a, const SearchScore& b) { return a.index < b.index; });
  select_threshold_and_n_best (scores, Params::sync_threshold2);
  std::sort (scores.begin(), scores.end(), [] (const SearchScore& a, const SearchScore& b) { return a.index < b.index; });
  out.clear();
  for (const auto& s : scores)
    {
      const double q = s.raw_quality - s.local_mean;
      out.push_back (SyncFinder::Score { size_t (s.index), fabs (q), q > 0 ? ConvBlockType::a : ConvBlockType::b });
    }
}

namespace {
bool sync_trace_on = false;
vector<SyncFinder::TraceRecord> sync_trace;
}

void
SyncFinder::trace_enable (bool on)
{
  sync_trace_on = on;
  sync_trace.clear();
}

vector<SyncFinder::TraceRecord>
SyncFinder::trace_take()
{
  vector<TraceRecord> t;
  t.swap (sync_trace);
  return t;
}

double
SyncFinder::normalize_sync_quality (double raw_quality)
{
  return raw_quality / std::min (Params::water_delta, 0.080) / 2.9;
}

vector<SyncFinder::KeyResult>
SyncFinder::search (const vector<Key>& key_list, size_t n_frames, int n_channels, Mode mode, size_t wav_first, size_t wav_last, int approx_slot)
{
  vector<KeyResult> key_results;
  awm_ctx *ctx = Engine::ctx();
  const int amode = mode == Mode::CLIP ? AWM_MODE_CLIP : AWM_MODE_BLOCK;

  if (Params::test_no_sync)               // fake_sync (src/syncfinder.cc:460-485): the positions a clean file has
    {
      vector<Score> result_scores;
      if (mode == Mode::BLOCK)
        {
          const size_t expect0 = Params::frames_pad_start * Params::frame_size;
          const size_t expect_step = (mark_sync_frame_count() + mark_data_frame_count()) * Params::frame_size;
          const size_t expect_end = (n_frames / Params::frame_size) * Params::frame_size;
          int ab = 0;
          for (size_t expect_index = expect0; expect_index + expect_step < expect_end; expect_index += expect_step)
            result_scores.push_back (Score { expect_index, 1.0, (ab++ & 1) ? ConvBlockType::b : ConvBlockType::a });
        }
      for (const auto& key : key_list)
        key_results.push_back (KeyResult { key, result_scores });
      return key_results;
    }
  if (mode == Mode::BLOCK)                 // no special treatment of silence in block mode
    {
      wav_first = 0;
      wav_last = n_frames * n_channels;
    }
  for (const auto& key : key_list)
    {
      KeyResult key_result;
      key_result.key = key;
      const int slot = ctx ? Engine::key_slot (key) : -1;
      vector<SearchScore> scores;
      static SearchScore *all = nullptr;       // page-locked staging buffer for the full score list of a chunk
      static size_t all_cap = 0;
      bool ok = slot >= 0;
      size_t n_all = 0;
      bool gpu_selected = false;
      const bool trace = getenv ("AWM_TRACE") != nullptr;
      const double t0 = get_time();
      double t1 = t0, t2 = t0, t3 = t0;
      if (ok)
        {
          size_t n_scores = 0;
          if (approx_slot >= 0)
            ok = awm_sync_use_slot (ctx, approx_slot, &n_scores) == 0;
          else
            ok = awm_sync_approx (ctx, slot, amode, wav_first, wav_last, Params::water_delta, nullptr, 0, &n_scores) == 0;
          /* the scores stay on the device; normally only the peaks that matter come back */
          const size_t truncate_n = mode == Mode::CLIP ? std::max (Params::get_n_best, 5) : 0;
          gpu_selected = ok && n_scores && select_candidates_gpu (ctx, Params::sync_threshold2 * 0.75, truncate_n, scores);
          if (gpu_selected)
            n_scores = 0;                         // nothing else to fetch
          if (ok && n_scores > all_cap)
            {
              awm_host_free (all);
              all_cap = n_scores + n_scores / 4;
              all = static_cast<SearchScore *> (awm_host_alloc (all_cap * sizeof (SearchScore)));
              if (!all)
                {
                  all_cap = 0;
                  ok = false;
                }
            }
          if (ok && n_scores)
            ok = awm_sync_approx (ctx, slot, amode, wav_first, wav_last, Params::water_delta, all, all_cap, &n_scores) == 0;
          n_all = ok ? n_scores : 0;
        }
      t1 = get_time();
      if (ok)
        {
          if (!gpu_selected)
            select_candidates_reference_order (all, n_all, Params::sync_threshold2 * 0.75, scores);
          if (mode == Mode::CLIP)               // ClipDecoder: at most n_best matches, but at least 5
            select_truncate_n (scores, std::max (Params::get_n_best, 5));
          t2 = get_time();
          ok = awm_sync_refine (ctx, slot, amode, wav_first, wav_last, Params::water_delta, scores.data(), scores.size()) == 0;
        }
      t3 = get_time();
      if (trace)
        fprintf (stderr, "[trace] sync search: approx %.3f ms, select %.3f ms, refine %.3f ms (%zu candidates)\n",
                 (t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3, scores.size());
      if (!ok)
        {
          error ("audiowmark: sync search failed: %s\n", Engine::last_error().c_str());
          key_results.push_back (key_result);
          continue;
        }
      select_final_scores (scores, key_result.sync_scores);
      key_results.push_back (key_result);
    }
  if (sync_trace_on)
    {
      TraceRecord rec { mode, n_frames, {} };
      for (const auto& kr : key_results)
        rec.scores.insert (rec.scores.end(), kr.sync_scores.begin(), kr.sync_scores.end());
      sync_trace.push_back (rec);
    }
  return key_results;
}
