// awm_wm.hh -- entry points of the watermark drivers, same names / argument meaning as the reference
// (src/wmcommon.hh:226-228, src/syncfinder.hh:71-121).
#pragma once
#include <functional>
#include <string>
#include <vector>
#include "awm_params.hh"
#include "awm_random.hh"
#include "awm_code.hh"
#include "awm_streams.hh"
#include "../../include/awm_b200.h"

int add_stream_watermark (const Key& key, AudioInputStream *in_stream, AudioOutputStream *out_stream, const std::string& bits, size_t zero_frames);
int add_watermark (const Key& key, const std::string& infile, const std::string& outfile, const std::string& bits);
int get_watermark (const std::vector<Key>& key_list, const std::string& infile, const std::string& orig_pattern);

/* buffer-level drivers used by the C host API (bench / tests): same computation without file I/O */
struct AddStats { int data_blocks = 0; double snr_db = 0; };
int add_watermark_buffer (const Key& key, const float *in, float *out, size_t n_frames, int n_channels, int sample_rate,
                          const std::string& bits, AddStats *stats, uint64_t first_frame_number = 0);

/* add_watermark_buffer for many items of one packed buffer (float or 16 bit PCM, host or device), one payload per item, in one pass
 * over the GPU; item i comes out bit identical to add_watermark_buffer[_s16] on it alone, stats (optional) gets one entry per item.
 *   keys: one key for every item, or with per_item_keys keys[i] for item i (keys.size() == n_items; the role tables of the distinct
 *     keys are built on the device once per call, each payload is encoded with its own key's bit order).
 *   sample_rates (optional, [n_items]): item i is at sample_rates[i] (16 bit items: converted to float and back around the add, as
 *     `audiowmark add` does for a 16 bit file).  Without it every item is at sample_rate, which must be 44.1 kHz.
 *   zero_frames (optional, [n_items], frames at the item's own rate): item i continues a stream that began zero_frames[i] frames
 *     earlier with silence (HLS segments): it comes out as add_watermark_buffer of zeros (z) ++ item with the first z frames dropped,
 *     Data Blocks counted over that stream, --snr over the item's own positions.
 *   scratch_bytes: the wave size of the calls with a rate list, 0 = their default.
 * The input picks the C call, and each call runs its own k_embed_batch instance:
 *   per-item keys: awm_embed_batch_keys;  one key: awm_embed_batch, _offsets, _rates or _rates_offsets by which lists are given.
 * Returns 2 for a malformed item list, key list, rate, offset list or payload (before any GPU work), 1 for other errors. */
int add_watermark_batch (const std::vector<Key>& keys, bool per_item_keys, const void *in, void *out, bool s16, size_t n_values,
                         const awm_batch_item *items, size_t n_items, const std::vector<std::string>& bits, int sample_rate, const int *sample_rates,
                         const uint64_t *zero_frames, size_t scratch_bytes, std::vector<AddStats> *stats);

/* add_stream_watermark's loop with bounded memory (window by window; see awm_add.cc); callbacks read / write interleaved frames */
int add_watermark_windowed (const Key& key, const std::function<Error (std::vector<float>&, size_t)>& read,
                            const std::function<Error (const std::vector<float>&)>& write, int n_channels, int sample_rate, const std::string& bits,
                            size_t zero_frames, size_t window_frames, AddStats *stats, size_t *frames_written);

/* The input frames [ext_first, ext_end) a window needs so that its owned frames [own_first, own_end) come out as in a run over the
 * whole stream of n_total frames (~0: not known yet): window_range at 44.1 kHz (ext_first a multiple of 1024, as awm_embed_window
 * needs), awm_window_range_rates at other rates.  Returns 1, with a message, for a bad range or rate. */
int add_window_range (size_t own_first, size_t own_end, size_t n_total, int sample_rate, size_t& ext_first, size_t& ext_end);
/* One window of a stream at any rate: in / out hold stream frames [ext_first, ext_end), the range add_window_range names for the
 * owned frames [own_first, own_end) of a stream of n_total frames (~0: not known yet, so the window does not end it).  The owned
 * frames of out come out bit identical to add_watermark_buffer of the whole stream.  snr_power (optional, 2 doubles) receives the
 * --snr sums of the owned frames; the window that ends the stream also takes the frames the add loop emits after the input. */
int add_watermark_window (const Key& key, const std::string& bits, const float *in, float *out, size_t ext_first, size_t ext_end, size_t n_total,
                          int n_channels, int sample_rate, size_t own_first, size_t own_end, double *snr_power);

/* frame counts of the add loop for inputs that are not at the watermark rate (see awm_add.cc) */
void resampled_add_plan (size_t n_frames, int sample_rate, bool limiter_on, size_t limiter_block, size_t& n_emit, size_t& gen_runs_out);

class ResultSet;
int get_watermark_buffer (const std::vector<Key>& key_list, const float *samples, size_t n_frames, int n_channels, int sample_rate,
                          ResultSet& result_set, bool print_speed_results = false, size_t *mark_rate_frames = nullptr);

/* 16 bit PCM in host memory (what a 16 bit WAV file holds): converted on the device, identical results at half the PCIe traffic */
int get_watermark_buffer_s16 (const std::vector<Key>& key_list, const int16_t *samples, size_t n_frames, int n_channels, int sample_rate,
                              ResultSet& result_set, bool print_speed_results = false, size_t *mark_rate_frames = nullptr);
int get_watermark_pcm (const std::vector<Key>& key_list, const float *samples, const int16_t *samples16, size_t n_frames, int n_channels, int sample_rate,
                       ResultSet& result_set, bool print_speed_results, size_t *mark_rate_frames);
int add_watermark_buffer_s16 (const Key& key, const int16_t *in, int16_t *out, size_t n_frames, int n_channels, int sample_rate,
                              const std::string& bits, AddStats *stats, uint64_t first_frame_number = 0);

/* the reference's chunks (WavChunkLoader geometry), which get_watermark_buffer and the sharded `get` both walk */
void chunk_geometry (int sample_rate, size_t& max_frames, size_t& overlap_frames);

namespace get_detail { struct VitJob; }

/* One `get` over a stream that arrives piece by piece (a pipe, a long file), in bounded memory: the chunk loop of WavChunkLoader
 * (src/wavchunkloader.cc:112-239).  Fed frames (interleaved float, host or device) go into one device chunk buffer of max_frames
 * frames at the watermark rate; at other rates they pass a small device input window and are resampled into it (awm_resample_range)
 * bit for bit as awm_resample of the whole stream would.  A chunk is decoded when it is full, the next one starts with its last
 * `overlap` frames, and the last one is only known at finish (a stream that exactly fills a chunk gives one more, overlap-only
 * chunk; an empty stream none).  finish runs the Viterbi decoder once over all chunks and merges their results in chunk order, as
 * get_watermark_buffer does.  max_input_frames (optional): the stream has at most that many frames, so a short stream gets a chunk
 * buffer of its own size.  dry_run: no device work at all, only the chunk decisions (chunks()), for tests without a GPU. */
class GetStream
{
public:
  struct Chunk { size_t first, n_frames; double time_offset; };     // watermark-rate frames

  GetStream (const std::vector<Key>& key_list, int n_channels, int sample_rate, bool print_speed_results,
             size_t max_input_frames = ~size_t (0), bool dry_run = false);
  ~GetStream();
  GetStream (const GetStream&) = delete;
  GetStream& operator= (const GetStream&) = delete;

  bool ok() const { return m_ok; }                 // false: refused at construction, with a message
  int  feed (const float *pcm, size_t n_frames);    // 0, or 1 with a message (the stream is then unusable)
  int  finish (ResultSet& result_set, size_t *mark_rate_frames);
  const std::vector<Chunk>& chunks() const { return m_chunks; }
  size_t peak_device_bytes() const { return m_peak_bytes; }

private:
  bool ensure_buffers();
  bool chunk_full();
  bool produce (size_t until);
  bool decode();

  std::vector<Key> m_keys;
  int    m_channels, m_rate;
  bool   m_print_speed, m_dry, m_ok = false, m_failed = false, m_finished = false;
  double m_ratio = 1;                    // watermark rate / input rate
  size_t m_max_frames = 0, m_overlap = 0, m_max_input = 0;
  size_t m_fill = 0, m_fed = 0, m_produced = 0;
  size_t m_start = 0;                    // watermark-rate frame of the chunk buffer's first frame
  double m_time_offset = 0;
  float *m_chunk = nullptr;              // [m_chunk_cap][channels], device
  size_t m_chunk_cap = 0;
  float *m_in = nullptr;                 // input window [m_in_cap][channels], device: stream frames [m_in_first, m_fed)
  size_t m_in_cap = 0, m_in_first = 0;
  size_t m_peak_bytes = 0;
  std::vector<Chunk> m_chunks;
  std::vector<std::string> m_debug_syncs;
  std::vector<get_detail::VitJob> m_pending;
};

int frame_count (const WavData& wav_data);

class SyncFinder
{
public:
  enum class Mode { BLOCK, CLIP };
  struct Score { size_t index; double quality; ConvBlockType block_type; };
  struct KeyResult { Key key; std::vector<Score> sync_scores; };
  /* searches the PCM currently bound to the GPU context; n_frames/n_channels describe it
   * (padded length for CLIP mode), wav_first/wav_last = non-silent value range.  approx_slot >= 0: one key, whose approx search
   * has been queued with awm_sync_approx_enqueue into that slot (on the PCM to search, which need not be bound) */
  std::vector<KeyResult> search (const std::vector<Key>& key_list, size_t n_frames, int n_channels, Mode mode,
                                 size_t wav_first, size_t wav_last, int approx_slot = -1);
  static double normalize_sync_quality (double raw_quality);

  /* test aid: when tracing is on every search() call appends what it returns (mode, length of the searched signal and per key
   * the final scores), so that tests can compare sync positions exactly with the reference's SyncFinder::search */
  struct TraceRecord { Mode mode; size_t n_frames; std::vector<Score> scores; };
  static void trace_enable (bool on);
  static std::vector<TraceRecord> trace_take();
};

/* stage functions of SyncFinder::search / BlockDecoder::run, used by get_watermark_buffer and by the sharded `get`
 * (host/awm_balanced.cc), which runs the GPU stages on slices of a chunk on different ranks */
int  select_candidates_from_peaks (const awm_search_score *peaks, size_t n, double floor_q, double threshold, std::vector<awm_search_score>& out,
                                  size_t truncate_n = 0);
void select_final_scores (std::vector<awm_search_score>& scores, std::vector<SyncFinder::Score>& out);

