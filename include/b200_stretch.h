/* b200_stretch.h -- C ABI of the GPU-native (H100) batched Signalsmith-Stretch hot path.
 *
 * One handle = one batch of `batch` independent audio streams that share one configuration
 * and are driven in lock-step (same call sequence, same buffer sizes), all resident on ONE GPU.
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

/* ---- parameters, broadcast to every stream of the batch (:107-135) ---- */
int b200s_set_transpose_factor(b200s_engine *e, float multiplier, float tonality_limit);
int b200s_set_transpose_semitones(b200s_engine *e, float semitones, float tonality_limit);
int b200s_set_formant_factor(b200s_engine *e, float multiplier, int compensate_pitch);
int b200s_set_formant_semitones(b200s_engine *e, float semitones, int compensate_pitch);
int b200s_set_formant_base(b200s_engine *e, float base_freq);
/* setFreqMap(std::function) (:120) cannot cross a C ABI (the reference's own wrapper says
 * "We can't do setFreqMap()", main.cpp:67).  The C++ facade tabulates the callable and passes a
 * monotone piecewise-linear map here: `n` points, freq_in[i] -> freq_out[i] (both as multiples
 * of the sample rate, freq_in ascending); linear extrapolation outside.  n == 0 clears it. */
int b200s_set_freq_map_table(b200s_engine *e, const float *freq_in, const float *freq_out, int n);

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
 * this order: plan, analyse, prep, chain, synth, commit (n >= 6). */
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
