/* b200_stretch.h -- C ABI of the GPU-native (H100) batched Signalsmith-Stretch hot path.
 *
 * One handle = one batch of `batch` independent audio streams that share one configuration
 * and are driven in lock-step (same call sequence), all resident on ONE GPU.  Each stream has its own parameters
 * (b200s_set_*_per_stream) and, through b200s_process_per_stream*, its own input and output length per call.
 * A batch of 1 is exactly one `signalsmith::stretch::SignalsmithStretch<float>` object.
 *
 * Every entry point mirrors one method of the reference class
 *   /root/reference/signalsmith-stretch.h:34-491
 * and follows the precedent of the reference's own extern "C" wrapper
 *   /root/reference/web/emscripten/main.cpp:15-77
 * (scalar arguments, planar float buffers), but handle-based instead of a global singleton
 * (main.cpp:9) and batched.  Buffers are planar: [batch][channels][samples] float32, the
 * batched form of the reference's `buffer[channel][index]` convention (README.md:46).
 *
 * All functions return 0 on success or a negative B200S_E* code; b200s_last_error() gives text.
 * The reference's methods return void and never throw (compile.sh:50 -fno-exceptions); error
 * codes exist here only because a GPU call can fail.  There is NO CPU fallback: without a CUDA
 * device b200s_create() fails with B200S_ENODEVICE.
 *
 * Threading (reference: README.md:93-97): calls on one handle must be serialised by the caller;
 * different handles are independent.  All work is enqueued on the handle's CUDA stream; host
 * buffer variants synchronise before returning, *_device variants do not.
 */
#ifndef B200_STRETCH_H
#define B200_STRETCH_H

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200s_engine b200s_engine;

enum {
	B200S_OK = 0,
	B200S_EINVAL = -1,      /* bad argument / not configured */
	B200S_ENODEVICE = -2,   /* no usable CUDA device: this library has no CPU path */
	B200S_ECUDA = -3,       /* a CUDA runtime call or kernel failed */
	B200S_EUNSUPPORTED = -4 /* feature of the reference not available on the GPU path (see DESIGN.md) */
};

/* ---- lifetime: SignalsmithStretch() / SignalsmithStretch(long seed)  (signalsmith-stretch.h:38-39) ---- */
int b200s_create(int batch, long seed, int device, b200s_engine **out);
void b200s_destroy(b200s_engine *e);
const char *b200s_last_error(const b200s_engine *e); /* e may be NULL: error of the last failed create */
int b200s_version(int *major, int *minor, int *patch); /* reference `version[3]` (:36) = 1.3.2 */

/* Use an existing CUDA stream (a cudaStream_t passed as void*) instead of the handle's own. */
int b200s_set_stream(b200s_engine *e, void *cuda_stream);
int b200s_synchronize(b200s_engine *e);
/* Device-buffer process() can split the batch into sub-batches on prioritised CUDA streams (default 1 = off:
 * the chain kernel is latency-bound, so co-running FFT CTAs only take its issue slots).  The host-buffer calls always pipeline stream groups (key 2 below). */
int b200s_set_sub_batches(b200s_engine *e, int n);
/* Implementation selectors for A/B measurement and cross-checking (results are identical by contract):
 *   key 0: direct chain kernel generation (1..4; 0 = default)   key 1: FFT kernels (1 = scalar Stockham, 0 = default paired)
 *   key 2: stream groups of the host-buffer pipeline in b200s_process (1..16, default 12)
 *   key 3: arithmetic of the stereo direct phase chain: 0 = fast (default: fused multiply-adds, SFU reciprocal / square
 *          root, as an optimising build of the reference), 1 = exact (the reference's unfused IEEE operation order;
 *          bit-identical to the CPU oracle when the FFT is substituted -- used by the tests)
 *   key 0 values: 1..6 (4 = k_chain_direct4, 5 = warp-specialised, 6 = k_chain_direct6)
 *   key 4: mapped / formant calls on the step-major path (1, default) or on the round-1 kernels (0)
 *   key 5: mono plain calls: two streams per warp on the packed wavefront k_chain_direct6 (1) or every stream on its own
 *          warp(s), k_chain_direct2 (0, default) */
int b200s_set_tuning(b200s_engine *e, int key, int value);

/* ---- configuration: presetDefault / presetCheaper / configure / reset  (:49-94) ---- */
int b200s_preset_default(b200s_engine *e, int channels, float sample_rate, int split_computation);
int b200s_preset_cheaper(b200s_engine *e, int channels, float sample_rate, int split_computation);
int b200s_configure(b200s_engine *e, int channels, int block_samples, int interval_samples, int split_computation);
int b200s_reset(b200s_engine *e);
/* Pre-size the per-call scratch so that process() never allocates (the reference asserts
 * "no allocation in process()", cmd/main-dev.cpp:158-163).  Optional: process() grows on demand. */
int b200s_reserve(b200s_engine *e, int max_input_samples, int max_output_samples);

/* ---- queries (:42-47, :96-104, :166-168, :205-207) ---- */
int b200s_batch(const b200s_engine *e);
int b200s_channels(const b200s_engine *e);
int b200s_block_samples(const b200s_engine *e);
int b200s_interval_samples(const b200s_engine *e);
int b200s_input_latency(const b200s_engine *e);
int b200s_output_latency(const b200s_engine *e);
int b200s_split_computation(const b200s_engine *e);
int b200s_seek_length(const b200s_engine *e);
int b200s_output_seek_length(const b200s_engine *e, float playback_rate);
int b200s_fft_samples(const b200s_engine *e);
int b200s_bands(const b200s_engine *e);

/* ---- parameters (:107-135).  Every stream has its own; these setters set every stream of the batch to the same value ---- */
int b200s_set_transpose_factor(b200s_engine *e, float multiplier, float tonality_limit);
int b200s_set_transpose_semitones(b200s_engine *e, float semitones, float tonality_limit);
int b200s_set_formant_factor(b200s_engine *e, float multiplier, int compensate_pitch);
int b200s_set_formant_semitones(b200s_engine *e, float semitones, int compensate_pitch);
int b200s_set_formant_base(b200s_engine *e, float base_freq);
/* The same setters per stream: arrays of `batch` entries, entry s set for stream s with the arithmetic of the setter above
 * (so a stream is bit-identical to a one-stream engine given that stream's values).  tonality_limits / compensate_pitch
 * may be NULL (0 for every stream).  Streams with different parameters run in one call: each stream takes the kernels
 * its own parameters need (a server that transposes every user's stream by that user's amount, or the live wrapper's
 * per-segment parameters, web/web-wrapper.js:233-235; signalsmith_stretch_b200/live.py). */
int b200s_set_transpose_factor_per_stream(b200s_engine *e, const float *multipliers, const float *tonality_limits);
int b200s_set_transpose_semitones_per_stream(b200s_engine *e, const float *semitones, const float *tonality_limits);
int b200s_set_formant_factor_per_stream(b200s_engine *e, const float *multipliers, const int *compensate_pitch);
int b200s_set_formant_semitones_per_stream(b200s_engine *e, const float *semitones, const int *compensate_pitch);
int b200s_set_formant_base_per_stream(b200s_engine *e, const float *base_freqs);
/* setFreqMap(std::function) (:120) cannot cross a C ABI (the reference's own wrapper says
 * "We can't do setFreqMap()", main.cpp:67).  The C++ facade tabulates the callable and passes a
 * monotone piecewise-linear map here: `n` points, freq_in[i] -> freq_out[i] (both as multiples
 * of the sample rate, freq_in ascending); linear extrapolation outside.  n == 0 clears it.
 * The engine's table: it applies to every stream, replacing any table a stream had of its own, until a transpose setter
 * (broadcast or per stream) turns it off for every stream it writes, as setTransposeFactor clears the reference's custom
 * map.  May synchronise the handle's stream. */
int b200s_set_freq_map_table(b200s_engine *e, const float *freq_in, const float *freq_out, int n);
/* Every stream its own map: a server whose users each have their own pitch mapping (a harmoniser that snaps each user to
 * that user's key) runs them in one batch.  Stream streams[i] gets its own table of n_points[i] points; the tables lie one
 * after another in freq_in / freq_out (sum(n_points) floats each), with the same contract as b200s_set_freq_map_table.
 * n_points[i] == 0: the stream has no custom map (the reference's customFreqMap = nullptr).  Streams that are not listed
 * keep what they have; a later b200s_set_freq_map_table replaces every stream's table, and a transpose setter clears the
 * map of every stream it writes.  Stream s is bit-identical to a one-stream engine given its table through
 * b200s_set_freq_map_table.  Tables are kept once per distinct content (1024 streams that share 16 maps hold 16 tables).
 * B200S_EINVAL before anything changes, b200s_last_error() naming the first bad entry: a NULL array with n > 0 (freq_in /
 * freq_out: with sum(n_points) > 0), n < 0, a stream outside [0, batch) or listed twice, n_points[i] < 0.  May
 * synchronise the handle's stream. */
int b200s_set_freq_map_table_per_stream(b200s_engine *e, const int *streams, int n, const int *n_points,
                                        const float *freq_in, const float *freq_out);

/* ---- the hot path (:139-165 seek, :172-204 outputSeek, :209-423 process, :426-464 flush, :467-491 exact) ----
 * Host-buffer variants: `in`/`out` are host pointers, planar [batch][channels][samples]; the call
 * copies host->device, runs, copies device->host and synchronises. */
int b200s_seek(b200s_engine *e, const float *in, int input_samples, double playback_rate);
/* seek() with one playback rate per stream (`playback_rates[batch]`): what a server needs whose streams follow their own
 * time maps (the reference's live wrapper seeks every audio quantum with the current segment's rate,
 * web/web-wrapper.js:314-315); signalsmith_stretch_b200/live.py is that loop for a batch. */
int b200s_seek_rates(b200s_engine *e, const float *in, int input_samples, const double *playback_rates);
/* The live loop without the per-quantum upload: the streams' audio sits in a DEVICE bank [batch][channels][bank_len]
 * (uploaded once); every quantum only the `batch` window positions and rates cross PCIe.  Stream s seeks with the `window`
 * samples that end at bank index window_end[s] (host array; samples outside [0, bank_len) read as zero -- the worklet's zero
 * padding, web-wrapper.js:289-311), at playback_rates[s] (host array).  Asynchronous on the handle's stream. */
int b200s_live_seek(b200s_engine *e, const float *d_bank, long long bank_len, const long long *window_end, int window, const double *playback_rates);
int b200s_output_seek(b200s_engine *e, const float *in, int input_length);
int b200s_process(b200s_engine *e, const float *in, int input_samples, float *out, int output_samples);
/* As b200s_process(), but returns as soon as the copies and kernels are enqueued: consecutive calls pipeline (stream
 * group g of call n+1 starts its host->device copy while other groups still finish call n), which is how a server
 * that streams chunk after chunk keeps both PCIe directions and the GPU busy.  `in` must stay valid and `out` must not
 * be read until b200s_synchronize() (or any synchronous call) returns; pinned host memory is needed for the copies to
 * be asynchronous at all. */
int b200s_process_async(b200s_engine *e, const float *in, int input_samples, float *out, int output_samples);
/* The same call with 16-bit PCM host buffers (what the reference's command-line tool reads and writes, cmd/util/wav.h):
 * sample / 32768 on the way in, round-to-nearest and clamp on the way out, both on the device, so that only two bytes
 * per sample cross PCIe -- the path is PCIe-bound end to end.  wait = 0: asynchronous like b200s_process_async. */
int b200s_process_pcm16(b200s_engine *e, const short *in, int input_samples, short *out, int output_samples, int wait);
int b200s_flush(b200s_engine *e, float *out, int output_samples, float playback_rate);
int b200s_exact(b200s_engine *e, const float *in, int input_samples, float *out, int output_samples, int *ok);
/* Device-buffer variants: pointers are device memory on the handle's GPU, same planar layout;
 * asynchronous on the handle's stream (input/output buffers must not alias, README.md:46). */
int b200s_seek_device(b200s_engine *e, const float *d_in, int input_samples, double playback_rate);
int b200s_process_device(b200s_engine *e, const float *d_in, int input_samples, float *d_out, int output_samples);
int b200s_flush_device(b200s_engine *e, float *d_out, int output_samples, float playback_rate);
/* process() with every stream's own input and output length: a server whose users each pick a tempo, whose slots idle or
 * whose next chunks differ in length runs them in one call.  Buffers are planar [batch][channels][stride]; stream s reads
 * the first input_samples[s] samples of each of its channel rows and writes the first output_samples[s], and the rest of
 * each output row, up to out_stride, is written as zero.  input_samples / output_samples are host arrays of `batch` ints,
 * copied during the call (an asynchronous caller may reuse them once the call returns).  Stream s is bit-identical to a
 * one-stream engine with its parameters that calls process(in_s, input_samples[s], out_s, output_samples[s]) -- (0, n),
 * (n, 0) and (0, 0) included: like the reference's process(), a (0, 0) call counts as silence.  NULL arrays, negative
 * strides or a length outside [0, stride] return B200S_EINVAL before anything is enqueued, and b200s_last_error() names
 * the stream.  b200s_reserve(in_stride, out_stride) sizes these calls as b200s_reserve(n_in, n_out) sizes b200s_process.
 *   b200s_process_per_stream:         host buffers, synchronous, like b200s_process
 *   b200s_process_per_stream_async:   host buffers, like b200s_process_async (consecutive calls whose STRIDES match pipeline
 *                                     without a join, whatever their lengths)
 *   b200s_process_per_stream_device:  device buffers, asynchronous on the handle's stream, like b200s_process_device */
int b200s_process_per_stream(b200s_engine *e, const float *in, int in_stride, const int *input_samples,
                             float *out, int out_stride, const int *output_samples);
int b200s_process_per_stream_async(b200s_engine *e, const float *in, int in_stride, const int *input_samples,
                                   float *out, int out_stride, const int *output_samples);
int b200s_process_per_stream_device(b200s_engine *e, const float *d_in, int in_stride, const int *input_samples,
                                    float *d_out, int out_stride, const int *output_samples);
/* One call in which every stream runs its own operation: a server turns one slot over (flush the track that ended,
 * outputSeek into the next one) while the other slots keep processing.  ops[s] is one of B200S_OP_*; buffers and counts are
 * those of b200s_process_per_stream, and playback_rates[s] (host array, may be NULL when no stream seeks: every FLUSH is
 * then at rate 0, the reference's default) is the rate of a SEEK or FLUSH.  Stream s is bit-identical to a one-stream
 * engine with its parameters that calls the reference method its op names, in the same order, and does nothing for its
 * SKIP calls -- outputs and every piece of state.  Every output sample an op does not produce is written as zero, up to
 * out_stride (the whole row for SEEK, OUTPUT_SEEK, RESET and SKIP).  exact() is OUTPUT_SEEK, PROCESS, FLUSH over three calls.
 * B200S_EINVAL, before anything is enqueued and with b200s_last_error() naming the stream: NULL ops or count arrays, a
 * negative stride, an op out of range, SEEK without rates, a count the op does not use (input for FLUSH / RESET / SKIP,
 * output for SEEK / OUTPUT_SEEK / RESET / SKIP), a count outside [0, stride].  b200s_reserve(in_stride, out_stride) also
 * sizes the flushes (up to in_stride zero samples) and output seeks of these calls; a FLUSH at a rate below 1/2 (rate 0,
 * the default, included) stretches beyond 2x and, like any call beyond 2x, allocates the random path's rows on first use.
 * A call of PROCESS / SKIP ops pipelines like b200s_process_per_stream_async; a call with any other op joins. */
enum {
	B200S_OP_SKIP = 0,        /* the stream sits this call out: state untouched, output row written as zero */
	B200S_OP_PROCESS = 1,     /* process(in, input_samples[s], out, output_samples[s])          :209-423 */
	B200S_OP_SEEK = 2,        /* seek(in, input_samples[s], playback_rates[s])                    :139-165 */
	B200S_OP_OUTPUT_SEEK = 3, /* outputSeek(in, input_samples[s])                                 :172-204 */
	B200S_OP_FLUSH = 4,       /* flush(out, output_samples[s], (float)playback_rates[s])          :426-464 */
	B200S_OP_RESET = 5        /* reset()                                                          :49-60   */
};
int b200s_run_per_stream(b200s_engine *e, const int *ops, const float *in, int in_stride, const int *input_samples,
                         float *out, int out_stride, const int *output_samples, const double *playback_rates);
int b200s_run_per_stream_async(b200s_engine *e, const int *ops, const float *in, int in_stride, const int *input_samples,
                               float *out, int out_stride, const int *output_samples, const double *playback_rates);
int b200s_run_per_stream_device(b200s_engine *e, const int *ops, const float *d_in, int in_stride, const int *input_samples,
                                float *d_out, int out_stride, const int *output_samples, const double *playback_rates);
/* b200s_run_per_stream over a list of streams: a server whose batch has 1024 slots and 100 active sessions moves and
 * processes 100 rows per call, not 1024.  Entry i belongs to stream streams[i], which runs ops[i] with input_samples[i],
 * output_samples[i] and playback_rates[i]; the buffers are packed over the list, [n][channels][stride], row i for stream
 * streams[i], and every array holds n entries.  The slots may be listed in any order.
 *   - A listed stream is bit-identical to what b200s_run_per_stream does with the same op at its slot, outputs and state;
 *     every output sample its op does not produce is written as zero, up to out_stride.
 *   - A stream that is not listed is neither read nor written: its state stays unchanged, byte for byte (SKIP without an
 *     output row).  n == 0 enqueues nothing.
 *   - B200S_EINVAL before anything is enqueued, b200s_last_error() naming the entry: n < 0 or n > batch, NULL streams, ops
 *     or count arrays with n > 0, a slot outside [0, batch) or listed twice, and every rule of b200s_run_per_stream.
 *   - b200s_reserve(in_stride, out_stride) sizes these calls as it sizes b200s_run_per_stream: no allocation afterwards.
 *   - Host buffers: a call of PROCESS / SKIP ops pipelines like b200s_run_per_stream_async when the previous call ran over
 *     the same list (the same slots in the same order) with the same strides; any other call joins.
 *   b200s_run_streams: host buffers, synchronous; _async: host buffers, returns once enqueued; _device: device buffers,
 *   asynchronous on the handle's stream.  The arrays other than the buffers are host arrays, copied during the call. */
int b200s_run_streams(b200s_engine *e, int n, const int *streams, const int *ops, const float *in, int in_stride,
                      const int *input_samples, float *out, int out_stride, const int *output_samples, const double *playback_rates);
int b200s_run_streams_async(b200s_engine *e, int n, const int *streams, const int *ops, const float *in, int in_stride,
                            const int *input_samples, float *out, int out_stride, const int *output_samples,
                            const double *playback_rates);
int b200s_run_streams_device(b200s_engine *e, int n, const int *streams, const int *ops, const float *d_in, int in_stride,
                             const int *input_samples, float *d_out, int out_stride, const int *output_samples,
                             const double *playback_rates);
/* b200s_run_per_stream and b200s_run_streams with 16-bit PCM host buffers, [positions][channels][stride] shorts: half the
 * bytes over PCIe of the float calls.  Per-stream lengths with plain process() are b200s_run_per_stream_pcm16 with every
 * op B200S_OP_PROCESS.
 *   - Every output row, state included, is bit-identical to the float call with the same arguments fed in / 32768, its
 *     output converted as b200s_process_pcm16 converts it: * 32768, round to nearest with halves away from zero, clamp to
 *     [-32768, 32767].  This holds for every op.  Both conversions run on the device.
 *   - Every output sample an op does not produce is 0, up to out_stride.  Slots a listed call leaves out are neither read
 *     nor written.
 *   - B200S_EINVAL, before anything is enqueued and with the same messages: every rule of the float counterpart.
 *   - wait = 0: the call returns once enqueued, like b200s_run_per_stream_async / b200s_run_streams_async.  A call of
 *     PROCESS / SKIP ops pipelines by the float calls' rule (the same list in the same order, the same strides; the sample
 *     format does not matter); any other call joins.  `in` must stay valid and `out` must not be read until
 *     b200s_synchronize(); pinned host memory is needed for the copies to be asynchronous.
 *   - The 16-bit staging of b200s_process_pcm16, [positions][channels][stride] each way, grows on first use after a
 *     synchronisation of the handle's stream; a later call at no larger strides and positions allocates nothing.
 *     b200s_reserve does not size it. */
int b200s_run_per_stream_pcm16(b200s_engine *e, const int *ops, const short *in, int in_stride, const int *input_samples,
                               short *out, int out_stride, const int *output_samples, const double *playback_rates, int wait);
int b200s_run_streams_pcm16(b200s_engine *e, int n, const int *streams, const int *ops, const short *in, int in_stride,
                            const int *input_samples, short *out, int out_stride, const int *output_samples,
                            const double *playback_rates, int wait);

/* ---- moving, duplicating and saving single streams ----
 * A server that rebalances streams over engines or GPUs, forks a session to preview two settings from the same point,
 * or checkpoints a session into another process moves one stream's complete state: history, pending output and its
 * windowProducts, the input / prevInput / output spectra and the prediction energy, the block scheduler, the random
 * engine, the pitch smoother and the stream's parameters.
 *
 * b200s_copy_streams: afterwards stream dst_streams[i] of `dst` is what a reference object is after
 * `*dst_i = *src_i` (member-wise copy); the source is unchanged, byte for byte.  Fed the same calls, the source and the
 * copy then give bit-identical outputs, each equal to a one-stream reference driven through that stream's whole history.
 *   - Every source is read before any destination is written: swaps and rotations within one engine work, and one
 *     source may go to several destinations.  Duplicate destinations are refused.
 *   - src == dst is allowed; src and dst may be different handles on the same or on different devices.  Both must have
 *     the same configuration (channels, block, interval, split); batch, seed and tuning keys may differ (exact math,
 *     key 3, included: the copy continues in the destination's arithmetic).
 *   - Frequency maps.  Within one engine a stream's table is copied as it is, without an upload.  A stream that uses the
 *     engine's table (set by b200s_set_freq_map_table with n > 0 and not cleared since) may only go to another engine whose
 *     table is bit-identical.  A stream with its own table (b200s_set_freq_map_table_per_stream) takes it along to the
 *     other engine: the upload is ordered with the copy on the destination's stream, and only growing the destination's
 *     table storage synchronises it.  A stream without a map arrives without one.
 *   - The parameters copied are the source's current ones (a setter called just before is included).  Whether the next
 *     call may need the random path (stretch beyond 2x, a slow seek) travels with the stream.
 *   - Ordering: the call acts as if it ran at its place in both handles' stream orders.  It enqueues without a host
 *     synchronisation, like the *_device calls (also after chained asynchronous host-buffer calls); later calls on either
 *     handle see the result.  n == 0 enqueues nothing.
 * b200s_export_streams writes n records of b200s_stream_state_bytes(e) bytes to host memory (synchronous);
 * b200s_import_streams reads them into the listed slots (synchronous).  A record starts with a header (magic, format
 * version, configuration, the stream's parameters and a fingerprint of the map table it uses); import checks every
 * header against the engine before anything is enqueued.  Records are in the host's byte order.  A record does not carry
 * the map table itself: a stream that uses the engine's table imports into an engine with the same table, and a stream
 * with its own table only into a slot that already holds a bit-identical table (its own or the engine's), which the
 * caller that checkpointed the stream sets first.
 * b200s_clone: a new handle with the same batch, device, seed, configuration, tuning keys, parameters, map tables and
 * state of every stream (an unconfigured source gives an unconfigured clone).  The copy members of the C++ facade.
 * B200S_EINVAL before anything is enqueued, b200s_last_error() naming the first offending entry (for a copy on both
 * handles): NULL arrays with n > 0, n < 0, an index outside [0, batch), duplicate destinations, an unconfigured engine,
 * a configuration mismatch, a bad record header (unknown flags included), a map-table mismatch.
 * Copies and imports stage through device buffers that grow on first use (b200s_device_allocations counts them); a
 * later call with at most as many streams allocates nothing. */
int b200s_stream_state_bytes(const b200s_engine *e); /* bytes of one stream's record; B200S_EINVAL if not configured */
int b200s_copy_streams(b200s_engine *dst, const int *dst_streams, b200s_engine *src, const int *src_streams, int n);
int b200s_export_streams(b200s_engine *e, const int *streams, int n, void *host_dst);
int b200s_import_streams(b200s_engine *e, const int *streams, int n, const void *host_src);
int b200s_clone(b200s_engine *src, b200s_engine **out);

/* ---- measurement helpers (no reference equivalent; used by bench.py) ---- */
/* CUDA events recorded on the handle's stream around whatever is enqueued in between. */
int b200s_timer_start(b200s_engine *e);
int b200s_timer_stop(b200s_engine *e, float *milliseconds); /* synchronises on the stop event */
/* Kernels launched by this handle since creation (claim for bench.py's "gpu_launches"). */
long long b200s_kernel_launches(const b200s_engine *e);
/* Device allocations (cudaMalloc calls) made by this handle since creation.  The reference asserts "no allocation in
 * process()" (cmd/main-dev.cpp:158-163); the equivalent here: after b200s_reserve() with the largest call sizes (and
 * with the parameters already set), process() leaves this count unchanged (tests/test_gpu_parity.py). */
long long b200s_device_allocations(const b200s_engine *e);
/* Beyond 2x stretch the reference draws a random time factor per bin (:639-640,:749,:769); this library reproduces the
 * draws of std::default_random_engine(seed) exactly (tests/test_host_logic.py).  The kernels of that path are launched
 * whenever the host can tell that a block may need them (input / output ratio of this and the previous call, a seek at a
 * slow rate, flush); the device decides per stream and block.  The one case the host cannot foresee is the first block
 * after a silence that was below the noise floor but not exactly zero: such a block is processed with the deterministic
 * factor (its spectrum is at the 1e-8 level) and counted here.  0 in every other situation.  Synchronises. */
long long b200s_unserved_random_blocks(b200s_engine *e);
/* Per-kernel device time of process(): between begin and end every kernel of the process()
 * launch sequence is bracketed by CUDA events on the handle's stream.  `ms`/`counts` receive, in
 * this order: plan, analyse, prep, chain, synth, commit (n >= 6), then, with n >= 7, the pre and post phases of
 * b200s_run_per_stream (dropped when n == 6). */
int b200s_profile_begin(b200s_engine *e);
int b200s_profile_end(b200s_engine *e, float *ms, int *counts, int n);

/* Device self-test: the branch-free division / square root of the phase chain against the IEEE
 * round-to-nearest intrinsics, bit for bit, on `n` pseudo-random normal-range operand pairs plus `n` pairs from the
 * edge classes (zero, subnormal and huge operands, infinite divisors); returns the mismatch counts. */
int b200s_selftest_divsqrt(b200s_engine *e, long long n, long long seed, long long *div_mismatch, long long *sqrt_mismatch);

/* ---- white-box state for teacher-forced parity tests (SURVEY.md section 8(c)) ----
 * `what`: 0 input spectrum, 1 prevInput, 2 output (complex: 2*bands floats per stream-channel),
 *         4 prediction energy (bands floats per stream-channel),
 *         20 input history (block+interval floats per stream-channel),
 *         21 pending overlap-add buffer, 22 pending windowProducts (per stream-channel).
 * Host buffers, layout [batch][channels][...]. */
int b200s_state_size(const b200s_engine *e, int what); /* floats per stream */
int b200s_get_state(b200s_engine *e, int what, float *dst);
int b200s_set_state(b200s_engine *e, int what, const float *src);

#ifdef __cplusplus
}
#endif
#endif
