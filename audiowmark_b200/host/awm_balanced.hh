// awm_balanced.hh -- `audiowmark get` for ONE long stream spread over several GPUs (one process per GPU).
//
// The reference decodes a long file chunk by chunk (WavChunkLoader: 30 minute chunks, 134.4 s overlap) and fans the work inside
// a chunk out to a thread pool (src/wmget.cc:971-1013, src/syncfinder.cc:171-256).  Here every rank owns an equal span of stream
// positions; for every chunk that overlaps its span it runs the GPU stages on the slice of the chunk's start frames it owns, and
// the per-chunk decisions (candidate selection, threshold / n-best, AB / "all" combination, merge) are taken on the gathered lists
// by every rank identically -- the result is the single-GPU document, pattern for pattern.  Three small exchanges per run:
//   peaks                    the local maxima of the approximate search above an adaptive floor
//   refined scores + bits    every candidate a rank owns, refined and decoded to soft bits
//   decoded words            the Viterbi results of the code words a rank decoded (the ranks that share a chunk deal its jobs out
//                            among themselves), with what rank 0 needs to print them
// No PCM crosses NVLink.  The exchange itself is a callback: NCCL (awm_dist_allgather) in production, an in-process stand-in when
// tests run several ranks on one GPU.
#pragma once
#include <functional>
#include <map>
#include <string>
#include <vector>
#include "awm_results.hh"
#include "awm_get_internal.hh"

namespace balanced {

struct Chunk { size_t first = 0, count = 0; double time_offset = 0; };
struct Slice                       // what a rank searches of one chunk
{
  int    chunk = 0;
  long   sa = 0, sb = 0;           // owned start frames [sa, sb)
  long   a = 0, b = 0;             // searched start frames [a, b): the owned ones plus a margin for local mean / peak test
  size_t lo = 0, hi = 0;           // stream sample-frames [lo, hi) the search of [a, b) reads
};

/* the reference's chunk walk over a stream of n_frames at the watermark rate */
std::vector<Chunk> chunk_plan (size_t n_frames, int sample_rate);
/* span of stream positions a rank owns (a multiple of the frame size) */
size_t owner_span (size_t n_total, int world);
std::vector<Slice> rank_slices (const std::vector<Chunk>& plan, int rank, int world, size_t n_total);
/* rank that owns a chunk-relative sample index (by the start frame it falls into) */
int owner_of (const std::vector<Chunk>& plan, size_t n_total, int world, int chunk, uint64_t index);

/* Input at another sample rate: the single GPU get resamples the stream to the watermark rate first and plans there, and so does
 * the sharded get -- chunk_plan, rank_slices and owner_of above all take the watermark-rate stream of mark_frames (n_total) frames. */
bool rate_supported (int sample_rate);       /* both resampling ratios inside the resampler's range (1/64, 64) */
size_t mark_frames (size_t n_total, int sample_rate);
/* input frames [first, end) of a stream of n_total frames at sample_rate that a rank with these slices reads: at the watermark
 * rate the union [min lo, max hi) of its slices, at other rates every frame the resampler taps of that union read, plus one frame
 * on each side, inside [0, n_total); [0, 0) without slices */
void input_range (const std::vector<Slice>& slices, size_t n_total, int sample_rate, size_t& first, size_t& end);

/* every rank contributes one byte string and receives everybody's, in rank order */
typedef std::function<bool (const std::string& mine, std::vector<std::string>& all)> Exchange;

class Get
{
public:
  /* pcm / pcm16: this rank's part of the stream of n_total frames at sample_rate (host or device memory; exactly one of the two),
   * starting at stream frame pcm_start; it must cover input_range of the rank's slices.  At another rate than the watermark rate
   * the rank resamples what its slices need into a buffer of its own as it binds them (host input is uploaded piece by piece, a
   * slice waits only for the pieces its taps read) */
  Get (int rank, int world, size_t n_total, const float *pcm, const int16_t *pcm16, size_t pcm_start, size_t pcm_frames, int channels,
       int sample_rate, const Key& key);
  ~Get();
  Get (const Get&) = delete;
  Get& operator= (const Get&) = delete;
  bool ok() const { return m_ok; }
  size_t n_mark() const { return m_n_mark; }      /* frames of the stream at the watermark rate */

  /* the stages, callable one by one (tests drive several ranks in one process) */
  bool stage_peaks (const std::map<int, double>& floors, std::string& out);
  bool stage_select (const std::vector<std::string>& all, std::map<int, double>& retry_floors);
  bool stage_refine_decode (std::string& out);
  bool stage_viterbi (const std::vector<std::string>& all, std::string& out);
  bool stage_merge (const std::vector<std::string>& all, ResultSet& result);

  /* all stages with the exchanges in between; `result` is filled on rank 0 */
  bool run (const Exchange& exchange, ResultSet& result);

private:
  bool bind (const Slice& sl);
  const Slice *my_slice (int chunk) const;

  int    m_rank, m_world, m_channels, m_rate, m_slot = -1;
  size_t m_n_total, m_n_mark = 0, m_pcm_start, m_pcm_frames;
  const float *m_dev = nullptr;    // device copy of this rank's PCM
  float *m_mark = nullptr;         // other rates: watermark-rate frames [m_mark_lo, max hi of the slices) of the stream
  size_t m_mark_lo = 0, m_mark_done = 0;    // ... of which [m_mark_lo, m_mark_done) are resampled
  Key    m_key;
  bool   m_ok = false, m_staged = false;
  std::vector<Chunk> m_plan;
  std::vector<Slice> m_slices;
  std::map<int, std::vector<awm_search_score>> m_cands;     // per chunk: selected candidates (identical on every rank)
  std::map<int, std::vector<int>> m_sharers;                // per chunk: the ranks that search a slice of it
  std::vector<get_detail::VitJob> m_jobs;                   // the code words this rank decodes
};

}
