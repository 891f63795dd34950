// common.cuh -- shared types of the H100 stretch engine (device + host).
//
// Data layout in HBM (all float32 / float2, per engine = per batch of S streams on one GPU):
//   hist     [S][C][B+H]        input history, most recent sample last        (reference: STFT input ring, B+H+1)
//   pend     [S][C][B(+H)]      pending overlap-add accumulator, linearised   (reference: STFT output ring)
//   pendWp   [S][C][B(+H)]      matching windowProducts (one identical copy per channel: single-writer CTAs)
//   stIn/stPrev/stOut [S][C][K] float2   Band::input / prevInput / output of the last block (:538-542)
//   stPredE  [S][C][K]          Prediction::energy of the last block (:593)
// and per process() call scratch, F = blocks in the call:
//   spec     [S][2F][C][K] float2   analysis spectra (slot 2f: block f, slot 2f+1: its re-analysed predecessor)
//   cS, cM   [S][F][K]              smoothed energy / formant envelope of the block (mapped / formant calls only)
//   cE       [S][F][C][K]           Prediction::energy
//   cPI,cFT,cT1,cT2 [S][F][C][K] float2   Prediction::input, freqTwist, short/long vertical twists
//   Y        [S][F][C][K] float2    final Band::output of every block
#pragma once

#ifdef B200S_EMU
#include "cuda_emu.h" // tests/cuda_emu: thread-per-CUDA-thread CPU emulator, TEST BUILDS ONLY
#else
#include <cuda_runtime.h>
#define B200S_SHARED __shared__
#define B200S_DYN_SHARED extern __shared__ float4 dyn_smem[];
#define B200S_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

#include <stdint.h>

namespace b200s {

// ---- constants of the reference ----
#define B200S_NOISE_FLOOR 1e-15f      // signalsmith-stretch.h:508
#define B200S_MAX_CLEAN_STRETCH 2.0f  // :509
#define B200S_ALMOST_ZERO 1e-30f      // dependency's windowProducts floor (SURVEY.md App. B, measured)
#define B200S_NEVER (1ll << 60)       // blockProcess.samplesSinceLast initial value (:496, SIZE_MAX there)

enum FrameFlags {
	FR_NEW_SPECTRUM = 1, // :299
	FR_REANALYSE = 2,    // :303
	FR_MAPPED = 4,       // :300
	FR_FORMANTS = 8,     // :310
	FR_RANDOM = 16       // :639
};

// static configuration of one engine
struct Cfg {
	int S, C;          // streams, channels
	int B, H, N, K;    // block, interval, fftSamples, bands (= N/2 = complex FFT size)
	int L;             // longVerticalStep = round(N/H) (:637)
	int split;         // splitComputation
	int histLen;       // B + H
	int pendLen;       // B (+ H when split)
	int addOff;        // where a block lands in `pend` (H when split, :294-297)
	int o;             // analysis/synthesis offset = B/2
	int nStages;       // Stockham stages of the K-point complex FFT
	int radix[20];
};

// user parameters (:107-135) of one stream in the form map_freq / inv_map_formant take: built by stream_params from the
// stream's entry of Ctx::sprm and its table in the frequency-map pool Ctx::maps
struct Params {
	float freqMultiplier, freqTonalityLimit;
	float formantMultiplier, invFormantMultiplier, formantBaseFreq;
	int formantCompensation;
	int mapN;                 // >0: custom piecewise-linear frequency map (setFreqMap, :120)
	const float *mapIn, *mapOut;
};

// what the setters write for one stream (b200s_set_*_per_stream; the broadcast setters write every entry), and what a
// stream record carries
struct StreamSettings {
	float freqMultiplier, freqTonalityLimit;
	float formantMultiplier, invFormantMultiplier, formantBaseFreq;
	int formantCompensation;
	int customMap; // the stream has a custom frequency map (setFreqMap, :120; cleared by a transpose setter): kMapEngine, kMapOwn
};
enum { kMapNone = 0, kMapEngine = 1, kMapOwn = 2 }; // StreamSettings::customMap: no table, the engine's table, its own table
// the parameters of one stream (Ctx::sprm): its settings and the descriptor of its frequency-map table, which lies at
// mapOff floats into the engine's pool (mapN inputs, then mapN outputs).  mapN is 0 when customMap is kMapNone.
struct StreamParams : StreamSettings {
	int mapOff, mapN;
};
// which path a stream's parameters need: frequency map (:300) and formant processing (:310); neither = pure time-stretch
__host__ __device__ __forceinline__ bool stream_mapped(const StreamParams &p) { return p.mapN > 0 || p.freqMultiplier != 1.0f; }
__host__ __device__ __forceinline__ bool stream_formants(const StreamParams &p, bool mapped) { return p.formantMultiplier != 1.0f || (p.formantCompensation && mapped); }

// per-stream block scheduler state (:494-529)
struct Sched {
	long long samplesSinceLast;
	long long silenceCounter;
	int prevInputOffset;
	int didSeek;
	int silenceFirst;
	float seekTimeFactor;
	long long zeroRun; // input samples, counted back from the newest, known to be exactly 0.0f (>= histLen: the history is all zeros)
};

// one block of the schedule (:281-319)
struct Frame {
	int t;           // output index within the call at which the block triggers
	int inputOffset; // :288
	int flags;
	float timeFactor; // :312, before the clamp of :638
	int inSlot, prevSlot; // spectrum slots: 0 = stIn, 1 = stPrev, 2+2f / 3+2f = this call's analyses
	unsigned rng;         // FR_RANDOM: state of the stream's random engine before this block's 2K-2 draws (:749,:769)
};

// per-stream result of the planner for one process() call
struct Call {
	int bypass;   // silence bypass (:240-271)
	int nFrames;
	int finalIn, finalPrev; // slots that become stIn / stPrev after the call
	int nJobs;              // analyses of this call (entries of the stream's Job list)
	int hasRandom;          // some block of the call stretches beyond 2x (:639): the stream takes the k_prep + k_chain path
	int mapped;             // the stream's parameters need a frequency map or formants: mapped-path kernels, planar spectra
	int autoPitch;          // formants with the automatic pitch estimate (formant base <= 0): k_pitch takes the stream
	int nIn, nOut;          // the stream's input / output samples of this call (Ctx::desc, or the call's uniform counts)
	// the stream's input row, resolved by k_plan: channel c reads in[c*inChan + i].  Every later kernel of the call reads it
	// here.  The output rows stay the call's (Ctx::out): k_synth2 has no register room for a per-stream row pointer.
	const float *in;
	int inChan;
};

// one stream's descriptor of a per-stream call (b200s_run_per_stream; b200s_process_per_stream is every op PROCESS),
// resolved by the host with the reference's arithmetic
struct CallDesc {
	int nIn, nOut; // the stream's counts in the process pass
	int op;        // B200S_OP_*
	int pass;      // 1: the process pass takes the stream (PROCESS, OUTPUT_SEEK, FLUSH with outputBlock > 0); 0: absent
	int seekN;     // SEEK / OUTPUT_SEEK: samples of the seek window (k_seek), at the start of the caller's row
	int at, tail;  // FLUSH: k_flush_tail's output offset and count (:439-455)
	float stf;     // SEEK / OUTPUT_SEEK: the seek time factor (:164)
	// the stream's input row in the process pass (Call::in): PROCESS its caller rows; FLUSH the engine's zero row (inChan
	// 0); OUTPUT_SEEK its caller rows from seekSamples on (:181)
	const float *in;
	int inChan;
	int slot; // b200s_run_streams: the stream this entry belongs to (entries are in list order); unused without Ctx::listed
};
#define B200S_OPBIT(op) (1 << (op))

// one windowed analysis FFT of the call (:333-376): block samples start at stream index `start`
// (history ++ input), the spectrum goes to row `row` = (2*f + w)*C + c of the stream's `spec` scratch
struct Job {
	int start, row, c;
};

// everything a kernel needs, passed by value
struct Ctx {
	Cfg cfg;
	const float *maps;        // the frequency-map pool: every table a stream uses (StreamParams::mapOff / mapN)
	const StreamParams *sprm; // [S] per-stream parameters
	// tables
	const float *window, *winProd, *wpReset;
	const float *wpDiv; // [H] windowProducts of a slot covered by a full H-spaced run of blocks, by phase (k_synth2)
	const float2 *rot, *twiddle, *pretw;
	const float4 *anaTab; // [K] {window[n+o], window[n+o-K], pretw[n].x, pretw[n].y}: one load per element in k_analyse2
	float2 rot0, rotStep; // rot[b+1] = rot[b] * rotStep in float, the reference's own recurrence (:647-655)
	// state
	Sched *sched;
	float *histCur, *histNext;
	float *pend, *pendWp;
	float2 *stIn, *stPrev, *stOut;
	float *stPredE;
	float *stPitch; // [S][2] freqEstimateWeighted, freqEstimateWeight (:927-928): automatic pitch estimate of the formant envelope
	// stereo direct path: spectra are channel-interleaved float4 {re0, re1, im0, im1} per bin (chain_direct3.cuh);
	// stIl [S][2][K] holds such copies of stIn / stPrev, made by k_plan at the start of the call.  Per stream: the
	// streams with Call::mapped keep planar rows (spec_il)
	float4 *stIl;
	int specIl;
	int wsRan; // k_chain_ws ran before k_chain_direct4 in this call: the latter only takes the streams the former left (chain_ws.cuh)
	float one; // 1.0f; unused: padd / psub (chain_direct3.cuh) ignore it since f2 arithmetic is never contracted
	// call scratch
	int maxFrames;
	Frame *frames; // [S][maxFrames]
	Call *call;    // [S]
	Job *jobs;     // [S][2*C*maxFrames], consecutive entries are transformed as one PAIR (fft2.cuh)
	int inAligned; // input / history rows allow 16-byte cp.async (pointer, strides and lengths multiples of 4 floats)
	float2 *spec, *Y, *cPI, *cFT, *cT1, *cT2;
	float *cE;
	// random time factors beyond 2x stretch (:639-640,:749,:769).  The reference draws from std::default_random_engine
	// (libstdc++: minstd_rand0, x <- 16807 x mod 2^31-1) through uniform_real_distribution<float>, 2K-2 draws per block in
	// bin order; draw i of a block is state * 16807^i, so every bin finds its draws by one modular multiplication.
	unsigned *rngState;     // [S] engine state per stream (persists over reset / configure, like the reference's member)
	const unsigned *rngPow; // [2K] 16807^i mod 2^31-1
	unsigned rngJump;       // 16807^(2K-2): one block's worth of draws
	const long long *seekEnd; // k_seek from a device-resident audio bank (b200s_live_seek): per stream, the bank index at which the
	long long bankLen;        // seek window ends; samples outside [0, bankLen) read as zero.  Null: x.in holds the window itself
	const float *seekStf;   // k_seek: per-stream seekTimeFactor (b200s_seek_rates), or null: the launch argument for every stream
	int randomPathOn;       // the kernels of the random path run in this call: the direct chain kernels leave hasRandom streams to them
	unsigned long long *diag; // [1] blocks whose random time factors could not be honoured (random path not launched; see engine.cu)
	int randomOnly;         // k_prep / k_chain launched beside the direct chain kernels: only streams with Call::hasRandom
	float2 *cT1u, *cT2u;    // [S][F][C][K] the "upwards" twists of a random block (:769-781; the downwards ones are cT1 / cT2)
	// step-major path of the mapped / formant configurations (chain_t.cuh): map + formant-ratio rows of k_prep's map-only mode,
	// and the chain's terms transposed by k_products: [S][tGroups][tRows][C][32 lanes]
	int mapOnly, tRows, tGroups;
	float *cMapB, *cMapG, *cRatio; // [S][maxFrames][K]
	float2 *tPI, *tFT, *tT1, *tT2;
	float *tE;
	float *cS, *cM; // [S][maxFrames][K]: smoothed energy (:816-848) and formant envelope (:986-1007) of every block: k_energy / k_passes -> k_prep
	float *cPitch; // [S][maxFrames] freqEstimate of every block when formantBaseFreq <= 0 (k_pitch)
	// sub-batch of streams this launch covers, as positions sBase .. sBase + sCount - 1 (stream_at) (the batch is processed
	// as a few sub-batches on prioritised CUDA streams so that different kernels of the sequence overlap on the SMs)
	int sBase, sCount;
	// I/O of the current call.  nIn / nOut and the rows in / out with their strides are the uniform call's; with `desc` ([S],
	// b200s_run_per_stream) every stream has its own.  In the process pass only k_plan reads either: it resolves them into
	// Call::nIn / nOut / in / out, which every later kernel of the call reads.  A stream whose CallDesc::pass is not `pass` is
	// absent from the process pass.  The phase kernels (k_reset_stft, k_reset_bands, k_seek, k_flush_tail, k_add_output)
	// take, with `desc`, only the streams whose op is in `opMask`, and in / out here are the caller's rows.
	// outTail > 0 (per-stream calls): output samples from Call::nOut up to outTail are written as zero.
	// listed (b200s_run_streams): the launch runs over the positions of a list of streams, not over the batch.  Position i
	// is stream desc[i].slot (stream_at); the caller's I/O rows and desc are indexed by position, state and scratch by stream.
	const float *in;
	float *out;
	int nIn, nOut;
	const CallDesc *desc;
	int pass, opMask;
	int outTail;
	int listed;
	long long inStreamStride, outStreamStride; // floats between streams
	int inChanStride, outChanStride;           // floats between channels
};

// the stream at position i of a launch (sBase + blockIdx, or a persistent kernel's item): the list's entry, or i itself
__device__ __forceinline__ int stream_at(const Ctx &x, int i) { return x.listed ? x.desc[i].slot : i; }

} // namespace b200s
