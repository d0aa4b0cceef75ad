// awm_get_internal.hh -- pieces of awm_get.cc that the multi-GPU driver (awm_balanced.cc) shares with the single-GPU chunk loop
#pragma once
#include <vector>
#include "awm_results.hh"

namespace get_detail {

/* sample-frames per piece of a host upload (awm_pcm_stage), 32 MB of 16 bit stereo: a chunk waits only for the pieces it reads */
constexpr size_t kStagePiece = size_t (8) << 20;

/* one code word waiting for the Viterbi decoder */
struct VitJob
{
  std::vector<float> soft;        // raw (un-normalised) soft bits, normalisation happens on the GPU
  ConvBlockType      block_type;
  double             time;
  SyncFinder::Score  score;
  ResultSet::Type    type;
  Key                key;
  int                chunk = 0;
  double             speed = 1;
};

/* all pending code words in ONE awm_viterbi launch; patterns go to the result set of the chunk they came from */
bool run_viterbi_jobs (std::vector<VitJob>& jobs, std::vector<ResultSet>& chunk_results);
/* the same split in two: decode only (bits [job][n_msg], err [job]) / turn decoded words into patterns */
bool viterbi_decode (const std::vector<const VitJob *>& jobs, std::vector<uint8_t>& bits, std::vector<float>& err);
void add_decoded_pattern (const VitJob& job, const uint8_t *bits, float err, ResultSet& chunk_result);

/* single blocks, AB pairs and the "all" chain of one chunk's synchronised blocks -> jobs */
void build_block_jobs (const Key& key, const std::vector<SyncFinder::Score>& sync_scores, const std::vector<std::vector<float>>& raw,
                       const std::vector<int>& valid, int sample_rate, int chunk, double speed, std::vector<VitJob>& pending);

}
