/* awm_b200.h -- C ABI of the H100-native (sm_90a) spectral watermark hot path.
 *
 * The reference (swesterfeld/audiowmark) has no FFI: its hot path is reached through
 * C++ classes and three free functions.  This header is the boundary a maintainer would
 * bind instead; every entry point names the reference interface it replaces
 * (paths relative to the reference tree).  Plain pointers and sizes only.
 *
 * Conventions
 *  - every function returns 0 on success, nonzero on error; awm_last_error (ctx) gives the text
 *  - a context owns one CUDA device + stream; single-owner, calls are stream ordered
 *  - PCM is interleaved fp32 in [-1,1) (what AudioInputStream::read_frames delivers,
 *    src/audiostream.hh:41-52); pointers may be host or device memory
 *  - "frame" in argument names is one PCM sample-frame (one sample per channel)
 *  - there is NO CPU fallback: without a usable CUDA device awm_create fails
 */
#ifndef AWM_B200_H
#define AWM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct awm_ctx awm_ctx;

#define AWM_FRAME_SIZE   1024   /* Params::frame_size      src/wmcommon.hh:36 */
#define AWM_MIN_BAND     20     /* Params::min_band        src/wmcommon.hh:40 */
#define AWM_MAX_BAND     100    /* Params::max_band        src/wmcommon.hh:39 */
#define AWM_N_BANDS      81
#define AWM_BANDS_PER_FRAME 30  /* Params::bands_per_frame src/wmcommon.hh:38 */
#define AWM_VITERBI_ORDER 15    /* src/convcode.cc:49 */

enum { AWM_MODE_BLOCK = 0, AWM_MODE_CLIP = 1 };           /* SyncFinder::Mode, src/syncfinder.hh:71 */
enum { AWM_BLOCK_A = 0, AWM_BLOCK_B = 1, AWM_BLOCK_AB = 2 }; /* ConvBlockType, src/convcode.hh:24 */

/* One sync frame: SyncFinder::FrameBit (src/syncfinder.hh:78-83); band indices are bin - AWM_MIN_BAND */
typedef struct {
  uint16_t frame;
  uint8_t  up[AWM_BANDS_PER_FRAME];
  uint8_t  down[AWM_BANDS_PER_FRAME];
} awm_sync_entry;

/* One mix entry: MixEntry (src/wmcommon.hh:149-154); up/down are FFT bin numbers */
typedef struct {
  uint16_t frame;
  uint8_t  up;
  uint8_t  down;
} awm_mix_entry;

/* SyncFinder::SearchScore (src/syncfinder.hh:89-98) */
typedef struct {
  uint64_t index;
  double   raw_quality;
  double   local_mean;
} awm_search_score;

/* ---- lifetime ------------------------------------------------------------------------- */
int         awm_create (int device, awm_ctx **out);
void        awm_destroy (awm_ctx *ctx);
const char *awm_last_error (const awm_ctx *ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t    awm_launch_count (const awm_ctx *ctx);
/* CUDA stream (cudaStream_t) the context launches on, for event timing by the caller */
void       *awm_stream (awm_ctx *ctx);
int         awm_synchronize (awm_ctx *ctx);
/* measurement aid: when enabled every kernel launch is bracketed by CUDA events on the context stream;
 * awm_profile_report synchronises, writes {"kernel": {"launches": n, "ms": total}, ...} as JSON and resets */
/* page-locked host memory for buffers that cross PCIe (PCM, score lists); plain malloc'ed memory works too, only slower */
void       *awm_host_alloc (size_t bytes);
void        awm_host_free (void *p);
int         awm_profile_enable (awm_ctx *ctx, int on);
int         awm_profile_report (awm_ctx *ctx, char *json_out, size_t json_cap);

/* ---- FFTProcessor (src/fft.hh:25-44, src/fft.cc:82-118) ------------------------------------
 * batched r2c / unnormalised c2r, n must be 1024.  in/out layouts as FFTW:
 *   r2c: in [count][1024] real  -> out [count][1026] (513 complex, re/im interleaved)
 *   c2r: in [count][1026]       -> out [count][1024] (sum over the Hermitian extension, not divided by n)
 */
int awm_fft_r2c (awm_ctx *ctx, const float *in, float *out, size_t count, int n);
int awm_fft_c2r (awm_ctx *ctx, const float *in, float *out, size_t count, int n);

/* ---- key / payload derived tables (built on the host, the AES key never reaches the GPU) ----
 * embed : FrameMod table of init_frame_mod_vec (src/wmadd.cc:148-162): uint8 [2 (A,B)][frames_per_block][101],
 *         0 keep / 1 up / 2 down
 * sync  : SyncFinder::get_sync_bits (src/syncfinder.cc:30-77) flattened bit-major; bit b owns
 *         entries bit_offsets[b] .. bit_offsets[b+1]-1, entries sorted by frame inside a bit; at most 6 bits,
 *         offsets non-decreasing, bands < 81 and no band twice in one entry's up (or down) list, else the call
 *         fails and the slot keeps its previous table.  A search fails if an entry frame is not below
 *         frames_per_block (twice that in CLIP mode)
 * mix   : gen_mix_entries (src/wmcommon.cc:179-202) and the bit order permutation of
 *         randomize_bit_order (src/wmcommon.hh:165-185): out[bit_order[i]] = in[i] on decode
 * key_slot selects one of AWM_MAX_KEYS table sets (audiowmark get accepts several --key options).
 */
#define AWM_MAX_KEYS 16
/* frame_mod_ab: uint8 [2 (A, B)][frames_per_block][101], 0 keep, 1 up, 2 down.  A byte above 2, or a nonzero byte below bin 20
 * (the kernels mark bins 20 .. 100 only), fails the call and leaves the previous table in place. */
int awm_set_embed_tables (awm_ctx *ctx, const uint8_t *frame_mod_ab, int frames_per_block);
int awm_set_sync_tables (awm_ctx *ctx, int key_slot, int mode, const awm_sync_entry *entries, int n_entries,
                         const int *bit_offsets, int n_bits);
int awm_set_mix_tables (awm_ctx *ctx, int key_slot, const awm_mix_entry *entries, int n_entries,
                        const uint16_t *bit_order, int n_coded_bits, int frames_per_bit, int frames_per_block);

/* ---- PCM residency (WavData::samples, src/wavdata.hh:27-74) ---------------------------------
 * Binds the audio the following sync / decode calls work on.  A host pointer is copied to a
 * context-owned device buffer (pinned or pageable, async on the context stream); a device
 * pointer is used in place and must stay valid until the next bind.
 * pad_start/pad_end: that many zero sample-frames are logically prepended / appended
 * (ClipDecoder::run_block zero padding, src/wmget.cc:823-866) without the caller materialising them.
 */
int awm_pcm_bind (awm_ctx *ctx, const float *pcm, size_t n_frames, int channels, size_t pad_start, size_t pad_end);

/* 16 bit PCM variants: the buffers hold interleaved int16 (what a 16 bit WAV file holds); conversion to / from the float
 * pipeline happens on the device with the reference's rules -- reading: sample * 2^-15 (src/sfinputstream.cc:189-210),
 * writing: float_to_int_clip<32> (src/rawconverter.hh:34-50), 16 most significant bits kept (src/sfoutputstream.cc:148-155) --
 * so results are identical to converting on the host, at half the PCIe traffic. */
int awm_pcm_bind_s16 (awm_ctx *ctx, const int16_t *pcm, size_t n_frames, int channels, size_t pad_start, size_t pad_end);
/* A long HOST stream (float or 16 bit PCM) on its way to the device piece by piece, for callers that work on parts of it while the
 * rest is still crossing PCIe; it replaces the read-ahead of WavChunkLoader (src/wavchunkloader.cc:54-163).  Both `get` drivers
 * upload host input this way: get_watermark_buffer searches its first chunk while the later chunks arrive, and the sharded get
 * searches a rank's first chunk slice while its later slices arrive.  awm_pcm_stage starts the copies on a copy stream and
 * returns the device address of the float copy at once; awm_pcm_stage_wait (n) orders everything issued on the context stream
 * afterwards behind the arrival of the first n sample-frames (16 bit pieces become float on the context stream then).  Bind
 * parts with awm_pcm_bind (device pointer + offset).  A new stage reuses the buffer: parts of the previous one must not be read
 * after it. */
int awm_pcm_stage (awm_ctx *ctx, const void *pcm, int is_s16, size_t n_frames, int channels, size_t piece_frames, const float **device_out);
int awm_pcm_stage_wait (awm_ctx *ctx, size_t n_frames);
/* device copy (float) of the bound PCM incl. padding; NULL if nothing is bound */
const float *awm_pcm_device (awm_ctx *ctx, size_t *n_frames, int *channels);

/* ---- embed: add_stream_watermark main loop (src/wmadd.cc:520-589) = FFTAnalyzer::run_fft
 * (src/wmcommon.cc:91-121) + apply_frame_mod (src/wmadd.cc:61-84) + WatermarkSynth::run
 * (src/wmadd.cc:215-250) + mix + Limiter::process (src/limiter.cc:45-124), for a whole buffer
 * at 44.1 kHz.  in/out: [n_frames][channels]; first_frame_number = index of the first 1024-frame
 * of this buffer in the stream (0 unless the caller shards; WatermarkGen starts its table row
 * at 2*frames_per_block - frames_pad_start, src/wmadd.cc:295; limiter blocks are counted from the stream start
 * as well, so a shard that brings a halo of one frame + two limiter blocks on each side reproduces the
 * unsharded result exactly in its interior).  limiter_block = sample_rate *
 * 1000 / 1000 frames (src/limiter.cc:33-37); limiter_block = 0 disables the limiter
 * (--test-no-limiter).  snr_power (optional, 2 doubles) receives sum(delta^2), sum(orig^2)
 * as --snr accumulates them (src/wmadd.cc:553-563).
 * The call fails before any work, with a message, unless: frames_pad_start is in [0, 2 * frames_per_block];
 * first_frame_number * 1024 + n_frames <= AWM_MAX_STREAM_FRAMES; limiter_block is 0 or in [AWM_MIN_LIMITER_BLOCK,
 * AWM_MAX_LIMITER_BLOCK].  The same frames_pad_start and limiter block rules hold for every batched embed below (for the
 * *_rates and *_keys calls the block mark_sample_rate * limiter_ms / 1000, when an item is at mark_sample_rate).
 * in / out may be device buffers at any 4-byte alignment (2-byte for the 16 bit variant).
 */
#define AWM_MIN_LIMITER_BLOCK 1024          /* a 1024-frame span touches at most two limiter blocks */
#define AWM_MAX_LIMITER_BLOCK (1 << 18)     /* half of the smallest pipeline piece: a block's peak is final before it is applied */
int awm_embed (awm_ctx *ctx, const float *in, float *out, size_t n_frames, int channels,
               uint64_t first_frame_number, int frames_pad_start, double water_delta,
               int limiter_block, float limiter_ceiling, double *snr_power);
/* awm_embed for one WINDOW of a longer stream (streaming `add` with bounded memory, add_stream_watermark's loop src/wmadd.cc:520-589
 * taken window by window): the buffer holds the window plus its halo, first_frame_number places it in the stream; only positions
 * [snr_first, snr_last) of the buffer (the part the caller keeps) enter the --snr sums.  Everything else as awm_embed. */
int awm_embed_window (awm_ctx *ctx, const float *in, float *out, size_t n_frames, int channels,
                      uint64_t first_frame_number, int frames_pad_start, double water_delta,
                      int limiter_block, float limiter_ceiling, uint64_t snr_first, uint64_t snr_last, double *snr_power);
/* the same for 16 bit PCM in and out (see awm_pcm_bind_s16): what `audiowmark add in16.wav out16.wav` computes between the files */
int awm_embed_s16 (awm_ctx *ctx, const int16_t *in, int16_t *out, size_t n_frames, int channels,
                   uint64_t first_frame_number, int frames_pad_start, double water_delta,
                   int limiter_block, float limiter_ceiling, double *snr_power);

/* ---- batched embed: many items, one key, one payload per item ------------------------------------------------
 * The FrameMod table of one (key, payload) is a key-only ROLE per (frame, bin) combined with the payload's coded bits.
 * Role code (uint16): 0 = keep; otherwise bit 0 is set, bit 1 = down band (the bit is inverted), bit 2 = sync bit,
 * bits 3..15 = index: of a coded data bit (data frames, position after randomize_bit_order) or of a sync bit.
 * The bit of a role in block ab (0 = A, 1 = B) is coded[ab][index] for data, (index + ab) & 1 for sync
 * (sync frames carry 010101 in A blocks, 101010 in B blocks); 1 -> entry 1 (up), 0 -> entry 2 (down), after the inversion. */
#define AWM_ROLE_MARK   1
#define AWM_ROLE_DOWN   2
#define AWM_ROLE_SYNC   4
#define AWM_ROLE_SHIFT  3
#define AWM_ROLE_MAX_INDEX 8191

/* one item of a batch: n_frames sample-frames of `channels` interleaved channels starting at value value_offset of the
 * packed buffer (values, not frames: items of different channel counts share one buffer) */
typedef struct {
  uint64_t value_offset;
  uint64_t n_frames;
  int      channels;
} awm_batch_item;

/* role table uint16 [frames_per_block][101] of one key; n_coded_bits = coded data bits per block (every data index < it) */
int awm_set_embed_roles (awm_ctx *ctx, const uint16_t *roles, int frames_per_block, int n_coded_bits);
/* 0 if every item has channels >= 1 and lies inside a packed buffer of n_values values, else nonzero with the reason in err
 * (err may be NULL).  Needs no device; awm_embed_batch runs the same check. */
int awm_batch_validate (const awm_batch_item *items, size_t n_items, size_t n_values, char *err, size_t err_cap);
/* awm_embed (first_frame_number 0) for every item of a packed buffer in one pass: item i comes out bit identical to awm_embed /
 * awm_embed_s16 on that item alone with the FrameMod table of payload i.  in / out: n_values floats (is_s16 = 0) or int16
 * (is_s16 = 1), host or device; host buffers cross PCIe as one copy each way.  Items must not overlap.  Values of out that belong
 * to no item are copied from in.
 * coded_bits: uint8 [n_items][2 (A, B)][n_coded_bits] (randomize_bit_order (code_encode (A | B, payload))).
 * snr_power (optional): [n_items][2] as awm_embed's.  Roles come from awm_set_embed_roles; zero items and zero-length items are legal. */
int awm_embed_batch (awm_ctx *ctx, const void *in, void *out, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                     const uint8_t *coded_bits, int frames_pad_start, double water_delta, int limiter_block, float limiter_ceiling,
                     double *snr_power);
/* Longest stream a batch item may end: zero_frames + n_frames <= 2^48 sample-frames (about 200 years at 44.1 kHz), so every stream
 * position, limiter block boundary and interleaved value index of the embed kernels stays far inside their 64-bit arithmetic. */
#define AWM_MAX_STREAM_FRAMES (1ull << 48)
/* 0 if awm_batch_validate passes, zero_frames is not NULL (for n_items > 0), zero_frames[i] + n_frames of every item is at most
 * AWM_MAX_STREAM_FRAMES and, when sample_rate != mark_sample_rate, every zero_frames[i] is 0; else nonzero with the reason in err.
 * Needs no device. */
int awm_batch_offsets_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const uint64_t *zero_frames, int sample_rate,
                                int mark_sample_rate, char *err, size_t err_cap);
/* awm_embed_batch for items that are segments of longer streams (HLS segments: add_stream_watermark with zero_frames,
 * src/wmadd.cc:501-580).  Item i continues a stream that began zero_frames[i] sample-frames earlier with silence: it comes out bit
 * identical to awm_embed (first_frame_number 0) of zeros (zero_frames[i]) ++ item, with the first zero_frames[i] frames dropped.
 * Table rows, synthesis and limiter blocks are those of that stream; the silent prefix is never materialised, nothing outside an
 * item's own values is read or written.  snr_power[i] sums the item's own positions only, as awm_embed_window does for the part
 * it keeps.  zero_frames: [n_items], 44.1 kHz sample-frames; all zero gives exactly awm_embed_batch.  Everything else as
 * awm_embed_batch. */
int awm_embed_batch_offsets (awm_ctx *ctx, const void *in, void *out, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                             const uint64_t *zero_frames, const uint8_t *coded_bits, int frames_pad_start, double water_delta, int limiter_block,
                             float limiter_ceiling, double *snr_power);
/* 0 if awm_batch_validate passes, mark_sample_rate > 0, every sample_rates[i] > 0, every rate other than mark_sample_rate has both
 * resampling ratios (mark / rate, rate / mark) inside the resampler's range (1/64, 64), at most 256 such rates are distinct and, where
 * n_emit is not NULL, n_emit[i] >= n_frames of every resampled item; else nonzero with the reason in err.  Needs no device. */
int awm_batch_rates_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const int *sample_rates, const uint64_t *n_emit,
                              int mark_sample_rate, char *err, size_t err_cap);
/* awm_embed_batch for items that each have their own sample rate.  Item i comes out as `add` of that item alone: awm_embed for
 * sample_rates[i] == mark_sample_rate; for any other rate the add loop (src/wmadd.cc:520-589) with a WatermarkResampler (:353-430):
 * the input is resampled to mark_sample_rate, the watermark signal alone is generated there (WatermarkGen::run), resampled back and
 * added to the untouched input (:548-566), and the limiter runs at the input rate (limiter block sample_rates[i] * limiter_ms / 1000).
 * 16 bit items as the float path between k_s16_to_f32 and k_f32_to_s16.
 * n_emit: [n_items], n_emit[i] >= n_frames = frames the reference loop pushes through the mixer before it stops (zero frames are fed
 * after EOF until resamplers and limiter have delivered everything; resampled_add_plan on the host): they enter the --snr sums and
 * the limiter's block peaks.  Ignored at mark_sample_rate.
 * limiter_ms = 0 disables the limiter.  snr_power (optional): [n_items][2].  Items at other rates run in consecutive waves whose
 * scratch (2 x n44 x channels floats per item, n44 = its length at mark_sample_rate) stays within scratch_bytes (0: 4 GiB); an item
 * larger than that runs alone.  The bound PCM (awm_pcm_bind) stays valid.  Everything else as awm_embed_batch. */
int awm_embed_batch_rates (awm_ctx *ctx, const void *in, void *out, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                           const uint8_t *coded_bits, const int *sample_rates, const uint64_t *n_emit, int mark_sample_rate, int frames_pad_start,
                           double water_delta, int limiter_ms, float limiter_ceiling, double *snr_power, size_t scratch_bytes);
/* 0 if awm_batch_rates_validate passes, zero_frames is not NULL (for n_items > 0) and every item's stream, zero_frames[i] +
 * n_frames, is at most AWM_MAX_STREAM_FRAMES both at sample_rates[i] and at mark_sample_rate ((z + n) * mark / rate); else nonzero
 * with the reason in err.  Needs no device. */
int awm_batch_rates_offsets_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const int *sample_rates, const uint64_t *n_emit,
                                      const uint64_t *zero_frames, int mark_sample_rate, char *err, size_t err_cap);
/* awm_embed_batch_rates for items that are segments of longer streams at any sample rate (HLS segments of a 48 kHz master:
 * add_stream_watermark with zero_frames, src/wmadd.cc:501-580).  Item i continues a stream at sample_rates[i] that began
 * zero_frames[i] frames (at that rate) earlier with silence: it comes out bit identical to item 0 of awm_embed_batch_rates on
 * zeros (zero_frames[i]) ++ item, with the first zero_frames[i] frames dropped.  Both resamplers, the watermark frames and the
 * limiter blocks are those of that stream; the silent prefix is never allocated, read or resampled, and an item's scratch does not
 * grow with its offset.  n_emit[i] counts from the item's first frame: the whole stream's n_emit minus zero_frames[i].  snr_power[i]
 * sums the item's own positions [z, z + n_emit[i]) only.  Items at mark_sample_rate are those of awm_embed_batch_offsets.  All
 * offsets zero gives exactly awm_embed_batch_rates; every rate at mark_sample_rate gives exactly awm_embed_batch_offsets. */
int awm_embed_batch_rates_offsets (awm_ctx *ctx, const void *in, void *out, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                                   const uint8_t *coded_bits, const int *sample_rates, const uint64_t *n_emit, const uint64_t *zero_frames,
                                   int mark_sample_rate, int frames_pad_start, double water_delta, int limiter_ms, float limiter_ceiling,
                                   double *snr_power, size_t scratch_bytes);

/* awm_embed_window for input that is not at mark_sample_rate (streaming and sharded `add` of a 48 kHz master): in / out hold stream
 * frames [stream_first, stream_first + n_frames) (interleaved float, host or device, any 4-byte alignment) and come out exactly as
 * item 0 of awm_embed_batch_rates_offsets with zero_frames = stream_first and this n_emit: the stream is taken as silent before the
 * window.  n_emit counts from stream_first: the window's own length for a window that does not end the stream, the whole stream's
 * n_emit (resampled_add_plan) minus stream_first for the last one.  A window with the halo awm_window_range_rates names for its owned
 * frames reproduces those frames of the whole stream's `add` bit for bit.  Roles come from awm_set_embed_roles, coded_bits is uint8
 * [2 (A, B)][n_coded_bits] as for the batched calls.  Only buffer positions [snr_first, snr_last) (inside [0, n_emit)) enter the
 * --snr sums.  Refused before any work: sample_rate == mark_sample_rate (use awm_embed_window), snr_first > snr_last, and whatever
 * awm_batch_rates_offsets_validate refuses for this one item (n_emit < n_frames among it). */
int awm_embed_window_rates (awm_ctx *ctx, const float *in, float *out, size_t n_frames, int channels, const uint8_t *coded_bits, int sample_rate,
                            int mark_sample_rate, uint64_t stream_first, uint64_t n_emit, int frames_pad_start, double water_delta, int limiter_ms,
                            float limiter_ceiling, uint64_t snr_first, uint64_t snr_last, double *snr_power);
/* The smallest input range [*ext_first, *ext_end) of a stream at sample_rate that makes outputs [own_first, own_end) of
 * awm_embed_window_rates exact: the limiter blocks before, of and after the owned frames (block sample_rate * limiter_ms / 1000,
 * which sizes the halo even when the embed runs without limiter), the out-resampler's taps into the watermark, one 1024-frame of
 * synthesis window on each side, the in-resampler's taps into the input, one frame of margin, clamped to [0, n_total).
 * n_total = UINT64_MAX: the end of the stream is not known yet.  Any cut is valid, no alignment is needed.  Returns nonzero, and
 * sets nothing, for an empty owned range, one that ends past n_total or 2^48, a rate outside the resampler's range, hlen outside
 * [8, 96] or limiter_ms <= 0.  Needs no device. */
int awm_window_range_rates (uint64_t own_first, uint64_t own_end, uint64_t n_total, int sample_rate, int mark_sample_rate, int limiter_ms, int hlen,
                            uint64_t *ext_first, uint64_t *ext_end);

/* ---- batched embed with a key per item ----------------------------------------------------------------------------------
 * What the role table of a key (gen_embed_roles on the host: UpDownGen, BitPosGen and gen_mix_entries, src/wmcommon.cc:143-202)
 * depends on besides the key: the frame counts of one block, frames_per_bit, --linear and the code length. */
typedef struct {
  int sync_frames;             /* sync_bits * sync_frames_per_bit (510) */
  int sync_frames_per_bit;     /* 85 */
  int data_frames;             /* n_coded_bits * frames_per_bit */
  int frames_per_bit;          /* --frames-per-bit */
  int mix;                     /* 0: --linear */
  int n_coded_bits;            /* coded data bits per block: code_size (A, payload_size) */
} awm_role_layout;
/* builds the role tables uint16 [n_keys][sync_frames + data_frames][101] of n_keys 16-byte AES keys (keys16: [n_keys][16], host or
 * device) on the device, each byte identical to the host's gen_embed_roles under this layout, and makes them the context's role set
 * (replacing the previous one; awm_set_embed_roles's table is not touched).  Fails, leaving no role set, if a key's table would assign
 * a (frame, bin) entry twice, as the host's builder does. */
int awm_set_embed_roles_keys (awm_ctx *ctx, const uint8_t *keys16, size_t n_keys, const awm_role_layout *layout);
/* copies the role tables of keys first_key .. first_key + n_keys - 1 of the role set to out (host or device) */
int awm_get_embed_roles_keys (awm_ctx *ctx, size_t first_key, size_t n_keys, uint16_t *out);
/* 0 if the validator of the matching single-key call passes (sample_rates NULL: awm_batch_offsets_validate's checks at
 * mark_sample_rate with zero_frames optional; else awm_batch_rates_validate, or awm_batch_rates_offsets_validate when zero_frames is
 * not NULL), key_index is not NULL and n_keys > 0 (for n_items > 0) and every key_index[i] < n_keys; else nonzero with the reason in
 * err.  Needs no device. */
int awm_batch_keys_validate (const awm_batch_item *items, size_t n_items, size_t n_values, const int *sample_rates, const uint64_t *n_emit,
                             const uint64_t *zero_frames, const uint32_t *key_index, size_t n_keys, int mark_sample_rate, char *err, size_t err_cap);
/* awm_embed_batch_rates_offsets with a key per item: item i is embedded with role table key_index[i] of the role set
 * (awm_set_embed_roles_keys) and its coded bits coded_bits[i] (randomize_bit_order with its own key), and comes out bit identical to
 * the single-key call with that key.  sample_rates NULL: every item is at mark_sample_rate (n_emit is then ignored); zero_frames
 * NULL: every item starts its stream.  coded_bits: uint8 [n_items][2][n_coded_bits of the role set].  Everything else as
 * awm_embed_batch_rates_offsets. */
int awm_embed_batch_keys (awm_ctx *ctx, const void *in, void *out, int is_s16, size_t n_values, const awm_batch_item *items, size_t n_items,
                          const uint8_t *coded_bits, const int *sample_rates, const uint64_t *n_emit, const uint64_t *zero_frames,
                          const uint32_t *key_index, int mark_sample_rate, int frames_pad_start, double water_delta, int limiter_ms,
                          float limiter_ceiling, double *snr_power, size_t scratch_bytes);

/* ---- sync search on the bound PCM --------------------------------------------------------
 * awm_sync_approx = SyncFinder::search_approx (src/syncfinder.cc:171-256): for the four
 * 256-sample shifts the channel-summed dB spectrogram (sync_fft, :560-605), sync_decode (:116-153)
 * for every start frame, and the local mean (:234-254).  scores_out (device->host) receives
 * *n_scores entries sorted by index.  wav_first/wav_last: non-silent value range
 * [first,last) as scan_silence computes it (:155-169) in interleaved-value units of the padded
 * signal; pass 0 / n_values for BLOCK mode.
 * Passing scores_out = NULL runs the search, keeps the scores on the device (for awm_sync_peaks) and returns the count.
 */
int awm_sync_approx (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last,
                     double water_delta, awm_search_score *scores_out, size_t max_scores, size_t *n_scores);

/* The search of awm_sync_approx without waiting for it: it is queued on a second stream of the context, behind everything queued on
 * the context stream so far, and keeps its scores and its PCM view in approx slot `slot` (0 or 1), so that the search of the next
 * chunk runs while the current chunk's peaks / refine / decode work on the other slot.  The bound PCM must stay valid (device
 * memory of the caller) until the slot is used.  awm_sync_use_slot makes a slot current: the context stream waits for its search,
 * the slot's PCM view becomes the bound PCM, awm_sync_peaks reads its scores; *n_scores as awm_sync_approx returns it.
 * awm_sync_approx itself works on the current slot. */
int awm_sync_approx_enqueue (awm_ctx *ctx, int slot, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta);
int awm_sync_use_slot (awm_ctx *ctx, int slot, size_t *n_scores);

/* The frames the last search of the current approx slot computed: out[shift][frame] = 1 where sync_fft analysed the frame, 0 where it
 * lies in leading / trailing digital silence (CLIP mode); 4 rows of *n_frames (frame_count - 1) each.  With max = 0 only *n_frames is
 * returned.  For tests of the spectrogram kernels. */
int awm_sync_have (awm_ctx *ctx, unsigned char *out, size_t max, size_t *n_frames);

/* awm_sync_peaks = sync_select_local_maxima (src/syncfinder.cc:258-281) on the score list of the current
 * approx slot (kept on the device), restricted to peaks with |raw_quality - local_mean| > min_abs_quality:
 * only those can pass the threshold / n-best selection that follows, so the host never has to look at the
 * several hundred thousand scores of a 30 minute chunk.  out: sorted by index; *n = number found (may exceed max,
 * then only max entries were written and the caller should raise min_abs_quality or use awm_sync_approx's full list).
 */
int awm_sync_peaks (awm_ctx *ctx, double min_abs_quality, awm_search_score *out, size_t max, size_t *n);

/* awm_sync_refine = SyncFinder::search_refine (src/syncfinder.cc:393-458): for each candidate the
 * fine offsets max(index-256,0) .. index+256 step 8 are scored with fresh FFTs of the wanted
 * sync frames; in/out: index, raw_quality are replaced by the best offset (strict '>' on
 * |q - local_mean|, earlier offset wins ties), local_mean is kept.
 */
int awm_sync_refine (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last,
                     double water_delta, awm_search_score *scores, size_t n_scores);

/* measurement aid for the parity tests: the sync_decode quality of each of the 65 fine offsets search_refine looks at
 * (src/syncfinder.cc:428-434), as the sliding-DFT kernel ranks them (exact = 0) or from fresh transforms in the reference's
 * summation order (exact = 1).  quality_out / valid_out: [n_scores][65]; offsets the reference gets no result for
 * (sync_fft returns nothing past the end of the signal) have valid 0.  awm_sync_refine re-scores every offset whose sliding
 * quality is within 1e-3 of the best exactly, so its result is that of the exact kernel as long as the two differ by < 5e-4.
 * On more than two channels there is no sliding pass: exact = 0 returns the exact qualities as well. */
int awm_sync_refine_offsets (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta,
                             const awm_search_score *scores, size_t n_scores, int exact, double *quality_out, unsigned char *valid_out);

/* measurement aid for the parity tests: the fine offsets awm_sync_refine re-scores exactly, as its ranking kernel picks them on the
 * device from the sliding qualities (every valid offset whose -|q - local_mean| is within 1e-3 of the smallest, plus the offset of the
 * approx index if it is valid).  On more than two channels every valid offset is scored exactly and flagged.
 * rescored_out: [n_scores][65], 1 = re-scored; scores is only read. */
int awm_sync_refine_rescored (awm_ctx *ctx, int key_slot, int mode, uint64_t wav_first, uint64_t wav_last, double water_delta,
                              const awm_search_score *scores, size_t n_scores, unsigned char *rescored_out);

/* ---- block decode: FFTAnalyzer::fft_range (src/wmcommon.cc:123-141) + mix_decode
 * (src/wmget.cc:67-108) + randomize_bit_order(decode) for blocks starting at indices[i]
 * (sample-frames of the padded signal).  raw_bits_out: [n_blocks][n_coded_bits] floats;
 * valid_out[i] = 0 when the block would read past the end (fft_range returns empty).
 */
int awm_decode_blocks (awm_ctx *ctx, int key_slot, const uint64_t *indices, size_t n_blocks,
                       float *raw_bits_out, int *valid_out);

/* ---- Viterbi: normalize_soft_bits (src/wmget.cc:40-65) + conv_decode_soft (src/convcode.cc:128-213)
 * for n_jobs independent code words in one launch.  block_types[j] in AWM_BLOCK_*: A / B words carry
 * 6 * (n_msg_bits + 15) soft bits, AB words 12 * (n_msg_bits + 15); raw_bits holds the jobs back to back
 * (un-normalised soft bits as mix_decode delivers them); hard != 0 => --hard.
 * bits_out: [n_jobs][n_msg_bits] bytes (0/1), error_out[j] = final path metric / coded bits.
 */
int awm_viterbi (awm_ctx *ctx, const float *raw_bits, size_t n_jobs, int n_msg_bits, const int *block_types,
                 int hard, uint8_t *bits_out, float *error_out);

/* ---- resampler: process_resampler / resample / resample_ratio_truncate (src/resample.cc:27-131) -------------
 * The reference delegates to zita-resampler (third party, not part of its tree); this library defines the filter itself:
 *   out[n] = sum_i in[i] g (i - n / ratio),   g (d) = fc sinc (fc d) w (d / h),   fc = min (1, ratio),   h = ceil (hlen / fc),
 *   w = 0.384 + 0.5 cos (pi x) + 0.116 cos (2 pi x) on [-1, 1];  256 phases, linear interpolation between phase rows,
 *   float accumulation in tap order; in is zero outside [0, n_in), outputs whose taps would pass h frames beyond the
 *   input are 0 (where a streaming resampler fed h - 1 frames of pre-roll and h of post-roll stops).
 * in/out: interleaved, host or device.  hlen = 16 everywhere in the reference.
 */
int awm_resample (awm_ctx *ctx, const float *in, size_t n_in, int channels, double ratio, int hlen, float *out, size_t n_out);

/* Frames a streaming resampler (the reference's BufferedResamplerImpl) has delivered after `fed` input frames (pre-roll excluded),
 * and after n_in frames plus its trailing frames: the length of the resampled stream.  hlen = 16 in the reference.  Needs no device. */
uint64_t awm_resample_stream_available (uint64_t fed, double ratio, int hlen);
uint64_t awm_resample_stream_frames (uint64_t n_in, double ratio, int hlen);
/* Input frames [*first, *end) of a stream of n_in_total frames that the taps of outputs [out_first, out_first + out_frames) of
 * awm_resample read, clamped to the stream (taps outside it read zero).  Needs no device. */
void awm_resample_taps (uint64_t n_in_total, double ratio, int hlen, uint64_t out_first, uint64_t out_frames, uint64_t *first, uint64_t *end);
/* Outputs [out_first, out_first + out_frames) of awm_resample over a whole stream of n_in_total frames, bit for bit, read from a
 * window of that stream: in holds stream frames [in_first, in_first + in_frames) (interleaved float, host or device); out is a
 * device buffer of out_frames frames.  Taps outside [0, n_in_total) read zero and outputs awm_resample zeroes (past its post-roll)
 * are zero, as in awm_resample.  Refused before any work (awm_resample_range_validate, which needs no device): channels <= 0, a
 * ratio outside (1/64, 64) or hlen outside [8, 96], counts or positions above 2^48, outputs that end past
 * awm_resample_stream_frames (n_in_total, ratio, hlen), and a window that misses a frame awm_resample_taps names. */
int awm_resample_range_validate (uint64_t in_first, uint64_t in_frames, uint64_t n_in_total, int channels, double ratio, int hlen,
                                 uint64_t out_first, uint64_t out_frames, char *err, size_t err_cap);
int awm_resample_range (awm_ctx *ctx, const float *in, uint64_t in_first, uint64_t in_frames, uint64_t n_in_total, int channels, double ratio, int hlen,
                        float *out, uint64_t out_first, uint64_t out_frames);
/* device memory on the context's device for callers without a device allocator of their own (bytes = 0: *out = NULL);
 * awm_device_free waits for the work queued on the context stream before it frees */
int awm_device_alloc (awm_ctx *ctx, size_t bytes, void **out);
int awm_device_free (awm_ctx *ctx, void *p);

/* resample_ratio (wav_data, speed, ...) of decode() (src/wmget.cc:916) without leaving the device: the bound PCM is
 * resampled by `ratio` into a context-owned buffer of n_out frames, which becomes the bound PCM; awm_pcm_pop restores
 * the previous binding (the original chunk is not copied again).  One level only; awm_pcm_bind drops a pushed binding. */
int awm_pcm_push_resampled (awm_ctx *ctx, double ratio, int hlen, size_t n_out);
int awm_pcm_pop (awm_ctx *ctx);
/* stream ordered copy device (or host) -> host for callers that keep their PCM in device memory but need a few values on
 * the host (clip selection of detect_speed hashes a sparse subset of the samples, src/wmspeed.cc:533-552) */
int awm_copy_to_host (awm_ctx *ctx, void *dst, const void *src, size_t bytes);
/* copy of `bytes` between any two buffers (host or device, not overlapping) in context stream order: it runs after the work queued
 * before it and the work queued after it sees the result.  Returns at once for a device source; a host source may be reused when it
 * returns (streaming `get`: pieces of a pipe go into the device chunk buffer as they arrive) */
int awm_copy (awm_ctx *ctx, void *dst, const void *src, size_t bytes);
/* dst_host[k] = src[indices[k]] for a device resident src (the sample subset detect_speed hashes) */
int awm_gather (awm_ctx *ctx, const float *src, const uint64_t *indices, size_t n, float *dst_host);
/* 1 if p points to CUDA device / managed memory (such pointers are used in place by the PCM entry points), else 0 */
int awm_is_device_pointer (const void *p);

/* ---- speed detection scan: SpeedSync::prepare_mags + SpeedSync::compare (src/wmspeed.cc:203-375) ------------------
 * clip = the audio SpeedSearch::get_jobs cut out (get_speed_clip, :33-52).  For every centre speed the clip is
 * truncated to seconds / centre, resampled by centre / 2, turned into the MagMatrix (512-point spectra, hop 128), and
 * scored for n_relative relative speeds (relative_speeds[c * n_relative + r] = pow (step, p) * speed / centre, :173).
 * quality_out[c * n_relative + r] = Score::quality of that compare() call (0 if no offset had data).
 * Uses the BLOCK mode sync table of key_slot (awm_set_sync_tables) and frames_per_block of awm_set_mix_tables.
 * Refused before any work: relative speeds that are not finite and > 0, more than 65535 (centre, relative speed) pairs, more
 * distinct centres than the resampler table cache holds (1024), and jobs whose 16.16 start offsets, or the frame offsets of
 * entries that can still land inside the MagMatrix, do not fit in 31 bits (the reference's int arithmetic would overflow; the
 * CLI's scans of at most 50 s never get there).  Entries that land past the last row for every start offset are skipped.
 */
int awm_speed_scan (awm_ctx *ctx, int key_slot, const float *clip, size_t clip_frames, int channels, int sample_rate,
                    double seconds, const double *centers, int n_centers, const double *relative_speeds, int n_relative,
                    double water_delta, double *quality_out);

/* inspection of the last awm_speed_scan: *rows and *n_entries = shape of the MagMatrix of centre `center`; with out, the matrix
 * (float2 (umag, dmag) [n_entries][rows], entries in table order) is copied there (max = capacity in float2) */
int awm_speed_mags (awm_ctx *ctx, int center, float *out, size_t max, int *rows, int *n_entries);

/* resampler filter tables: how many the context holds and how many it keeps before it empties the cache */
int awm_resampler_cache (awm_ctx *ctx, size_t *size, size_t *cap);

/* ---- multi-GPU exchange for the sharded `get` (one process per GPU) ------------------------------------------------------
 * The reference has no counterpart: its thread pool shares one address space.  Here the ranks of a job exchange the small
 * per-chunk lists of the search (peaks, refined scores + soft bits, decoded words) with ncclAllGather on the context stream;
 * no PCM ever crosses NVLink.  awm_dist_unique_id: rank 0 creates the NCCL id, the launcher hands it to every rank (bench.py
 * broadcasts it with torch.distributed); awm_dist_init joins the communicator; awm_dist_allgather: every rank contributes
 * send_bytes (<= slot_bytes - 8) and receives rank r's bytes at recv + r * slot_bytes, its length in recv_bytes[r].  Returns 2
 * when some rank's payload did not fit (recv_bytes then holds all lengths: repeat with a larger slot; every rank sees the same).
 * Without awm_dist_init the "world" is this process alone and the call degenerates to a copy. */
int awm_dist_unique_id (unsigned char id_out[128]);
int awm_dist_init (awm_ctx *ctx, int rank, int world, const unsigned char id[128]);
int awm_dist_world (const awm_ctx *ctx, int *rank, int *world);
int awm_dist_allgather (awm_ctx *ctx, const void *send, size_t send_bytes, size_t slot_bytes, void *recv, size_t *recv_bytes);

#ifdef __cplusplus
}
#endif
#endif /* AWM_B200_H */
