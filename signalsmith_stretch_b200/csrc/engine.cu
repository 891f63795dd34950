// engine.cu -- host side of the H100 stretch engine + the extern "C" ABI of include/b200_stretch.h.
//
// The host does no DSP: it sizes buffers, builds the constant tables once per configure() and
// enqueues kernels on one CUDA stream.  Even the block scheduler runs on the device (k_plan), so
// a process() call is a fixed, sync-free launch sequence:
//   plain (no frequency map / formants), presets:  k_plan -> k_analyse2 -> k_chain_direct4 (stereo) | k_chain_direct2 (mono)
//                                                  -> k_synth2 || k_commit (side stream)
//   mapped / formants:  k_plan -> k_analyse2 -> [k_pitch] -> k_energy -> k_passes -> k_prep (map-only) -> k_products
//                       -> k_chain_t -> k_synth2 || k_commit                                        (chain_t.cuh)
//   the path is decided per stream from its own parameters (Call::mapped): a call whose streams differ launches both
//   sequences, and each kernel exits at once for the streams of the other path
//   calls that may stretch beyond 2x additionally launch k_prep + k_chain in random-only mode: they take the streams
//   whose blocks draw random time factors (Call::hasRandom, decided per stream by k_plan); every other CTA exits at once
//   generic sizes (not 3072 / 2560 bands): k_analyse / k_synth (fft.cuh), k_chain_direct2 (plain) / k_chain (mapped)
//   selectable for A/B: k_chain_direct6 (stereo presets, tuning key 0 = 6; mono stream pairs, key 5), chain_direct6.cuh
// Reference for every step: /root/reference/signalsmith-stretch.h (cited per kernel in kernels.cuh).
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <climits>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/b200_stretch.h"
#include "kernels.cuh"
#include "chain_direct.cuh"
#include "chain_direct2.cuh"
#include "stft2.cuh"
#include "chain_direct3.cuh"
#include "chain_direct4.cuh"
#include "chain_ws.cuh"
#include "chain_direct6.cuh"
#include "chain_t.cuh"
#include "state_copy.cuh"

using namespace b200s;

static std::string g_createError;

// one frequency-map table (setFreqMap, :120) of the engine's pool: n inputs, then n outputs, at `off` floats into the pool
struct MapTable {
	int off = 0, n = 0;
	uint64_t hash = 0; // FNV-1a over n and the points: the fingerprint a stream record carries
	std::vector<float> pts;
};
static MapTable make_table(int n, const float *in, const float *out) {
	MapTable t;
	t.n = n;
	t.pts.assign(in, in + n);
	t.pts.insert(t.pts.end(), out, out + n);
	uint64_t h = 1469598103934665603ull;
	auto mix = [&](const void *p, size_t bytes) {
		for (size_t i = 0; i < bytes; ++i) h = (h ^ ((const unsigned char *)p)[i]) * 1099511628211ull;
	};
	const int32_t n32 = n;
	mix(&n32, sizeof(n32));
	mix(t.pts.data(), sizeof(float) * t.pts.size());
	t.hash = h;
	return t;
}
// bit for bit (an empty table equals any other empty one)
static bool same_points(const MapTable &a, const MapTable &b) {
	return a.n == b.n && (a.n == 0 || (a.hash == b.hash && !memcmp(a.pts.data(), b.pts.data(), sizeof(float) * a.pts.size())));
}

struct b200s_engine {
	int S = 0, device = 0;
	long seed = 0;
	bool configured = false;
	Cfg cfg;
	// Frequency-map tables (DESIGN.md §3.9): the engine's table (b200s_set_freq_map_table; n = 0: none) and every stream's
	// own table (b200s_set_freq_map_table_per_stream) lie de-duplicated by content in one device pool, dMaps.  `maps` holds
	// the host copies in pool order; a stream finds its table by StreamParams::mapOff / mapN.
	MapTable engMap;
	std::vector<MapTable> maps;
	float *dMaps = 0;
	size_t mapsCap = 0, mapsUsed = 0; // floats
	// per-stream parameters: the host table (what the setters write) and its device copy Ctx::sprm, uploaded by the next
	// process() when dirty; the counts over the table decide which kernels a call launches
	std::vector<StreamParams> hSprm;
	StreamParams *dSprm = 0;
	bool sprmDirty = true;
	// pinned staging of the upload, two copies: an asynchronous call returns once enqueued (from pageable memory the copy
	// could wait for the queued work); a copy is rewritten once the upload issued from it two uploads ago has run
	StreamParams *pinSprm[2] = {0, 0};
	cudaEvent_t evSprm[2] = {0, 0};
	int sprmSlot = 0;
	int nMapped = 0;                              // streams on the mapped / formant path (Call::mapped)
	bool anyFormants = false, anyAutoPitch = false; // some stream processes formants / with the automatic pitch estimate
	cudaStream_t stream = 0;
	bool ownStream = false;
	// sub-batch pipeline: process() splits the batch over these prioritised streams (see process_impl)
	static const int kMaxSub = 16;
	int nSub = 1, maxSub = 1;
	cudaStream_t subStream[kMaxSub] = {};
	cudaEvent_t evBegin = 0, evSubDone[kMaxSub] = {};
	int chainedGroups = 0; // > 0: the last operation was a host-buffer process() over this many stream groups (see process_impl)
	int chainedIn = -1, chainedOut = -1; // its per-channel sample counts (strides): the groups' slabs of the staging buffers sit at sBase*C*n
	bool chainedListed = false;          // it ran over a list of streams (b200s_run_streams), chainedList, in that order
	std::vector<int> chainedList;
	// per-stream call descriptors (b200s_run_per_stream): the device table Ctx::desc [S], allocated at configure, and two
	// pinned staging copies.  In a call of PROCESS / SKIP ops each stream group copies its own slice on its own CUDA stream
	// ahead of its k_plan, so chained calls need no join for it; a call with a pre or post phase copies the whole table on
	// the main stream.  A staging copy is rewritten once every copy issued from it two calls ago has run.
	CallDesc *dDesc = 0;
	CallDesc *pinDesc[2] = {0, 0};
	cudaEvent_t evDesc[2][kMaxSub] = {};
	int descSlot = 0;
	std::vector<int> allProcess; // [S] B200S_OP_PROCESS: b200s_process_per_stream's ops
	int chainV = 0, fftV1 = 0; // b200s_set_tuning overrides (0 = default)
	int exactMath = 0;         // b200s_set_tuning key 3: 1 = the phase chain in the reference's unfused IEEE arithmetic
	// host-buffer API: stream groups whose H2D copy / kernels / D2H copy are pipelined.  H100 SXM, batch 1024 stereo, one run
	// per value, pipelined / blocking ms per step: 4 -> 15.5 / 16.8, 8 -> 18.0 / 18.1, 12 -> 19.7 / 18.5, 16 -> 16.1 / 16.6; the
	// other H100 hosts measured 10.7-14.5 / 13.8-14.6 ms at 12, so the choice is within the host-to-host spread and 12 stays.
	int nHostParts = 12;
	cudaEvent_t evStart = 0, evStop = 0;
	// k_commit (state carry + history append) only needs the chain's output, not the synthesis: it runs on a side stream
	// beside k_synth2 (fork after the chain, join after both)
	cudaStream_t commitStream = 0;
	cudaEvent_t evFork = 0, evJoin = 0;
	long long launches = 0, allocs = 0;
	std::string err;
	// optional per-kernel CUDA-event timing (b200s_profile_begin/end)
	bool profiling = false;
	std::vector<cudaEvent_t> profEv; // pairs
	std::vector<int> profKind;

	// tables
	float *dWindow = 0, *dWinProd = 0, *dWpReset = 0, *dWpDiv = 0;
	float2 *dRot = 0, *dTwiddle = 0, *dPretw = 0;
	float4 *dAnaTab = 0;
	float2 rot0, rotStep;
	// state
	Sched *dSched = 0;
	float *dHist[2] = {0, 0};
	int histCur = 0;
	float *dPend = 0, *dPendWp = 0;
	float2 *dStIn = 0, *dStPrev = 0, *dStOut = 0;
	float *dStPredE = 0;
	float4 *dStIl = 0;
	// call scratch
	int maxFrames = 0, coefFrames = 0; // coefFrames: block capacity of the coefficient rows (mapped / formant calls only)
	Frame *dFrames = 0;
	Call *dCall = 0;
	Job *dJobs = 0;
	int numSMs = 132; // H100 SXM; replaced by the device's own count at configure()
	float2 *dSpec = 0, *dY = 0, *dPI = 0, *dFT = 0, *dT1 = 0, *dT2 = 0;
	float *dE = 0, *dS = 0, *dM = 0;
	// step-major path of the mapped / formant configurations (chain_t.cuh)
	float *dMapB = 0, *dMapG = 0, *dRatio = 0, *dTE = 0;
	float2 *dTPI = 0, *dTFT = 0, *dTT1 = 0, *dTT2 = 0;
	int tFrames = 0;
	int dual = -1;     // b200s_set_tuning key 5: mono plain path, pairs of streams on the packed wavefront (-1: B200S_DUAL or on)
	int stepMajor = 1; // b200s_set_tuning key 4: 0 = the round-1 kernels (k_prep + k_chain) for every stream
	// random time factors beyond 2x stretch (:639-640): engine state per stream (lives as long as the handle, like the
	// reference's randomEngine member), powers of the multiplier, the upwards twists of random blocks
	unsigned *dRng = 0, *dRngPow = 0;
	unsigned long long *dDiag = 0;
	float *dSeekStf = 0; // per-stream seek time factors (b200s_seek_rates)
	std::vector<float> hSeekStf;
	long long *dSeekEnd = 0; // per-stream window ends in the audio bank (b200s_live_seek)
	unsigned rngJump = 1;
	float2 *dT1u = 0, *dT2u = 0;
	int randFrames = 0;
	bool prevCallMayRandom = false, seekMayRandom = false;
	float *dStPitch = 0, *dPitch = 0;
	// staging for the host-buffer API and for flush/outputSeek
	float *dIn = 0, *dOut = 0, *dZero = 0, *dTmp = 0;
	size_t inCap = 0, outCap = 0, zeroCap = 0, tmpCap = 0;
	short *dIn16 = 0, *dOut16 = 0; // 16-bit PCM staging of b200s_process_pcm16 and the _pcm16 per-stream calls (stage_pcm16)
	size_t in16Cap = 0, out16Cap = 0;
	// stream copies, export and import (DESIGN.md §3.12): packed records [xferCap][record bytes], the stream lists of the
	// pack and the unpack (device [2][xferCap]; two pinned staging copies, rewritten once the upload issued from them two
	// uploads ago has run), and the event by which another handle orders its side of a copy after this one's
	char *dXfer = 0;
	int *dXferIdx = 0;
	int xferCap = 0, xferRecCap = 0; // streams the lists / the records have room for
	int *pinIdx[2] = {0, 0};
	cudaEvent_t evIdx[2] = {0, 0};
	int idxSlot = 0;
	cudaEvent_t evXfer = 0;
};

#define CK(call)                                                                                   \
	do {                                                                                           \
		cudaError_t _e = (call);                                                                   \
		if (_e != cudaSuccess) {                                                                   \
			e->err = std::string(#call) + ": " + cudaGetErrorString(_e);                           \
			return B200S_ECUDA;                                                                    \
		}                                                                                          \
	} while (0)
#define CKL()                                                                                      \
	do {                                                                                           \
		++e->launches;                                                                             \
		CK(cudaGetLastError());                                                                    \
	} while (0)
#define NEED_CFG()                                                                                 \
	do {                                                                                           \
		if (!e) return B200S_EINVAL;                                                               \
		if (!e->configured) {                                                                      \
			e->err = "engine not configured";                                                      \
			return B200S_EINVAL;                                                                   \
		}                                                                                          \
	} while (0)

template <typename T>
static int dalloc(b200s_engine *e, T **p, size_t n) {
	if (*p) cudaFree(*p);
	*p = 0;
	++e->allocs;
	CK(cudaMalloc((void **)p, std::max<size_t>(n, 1) * sizeof(T)));
	return 0;
}
template <typename T>
static void dfree(T *&p) {
	if (p) cudaFree(p);
	p = 0;
}

// page-locked host memory (the CPU emulator of the tests has none: plain memory there)
static bool host_alloc(void **p, size_t bytes) {
#ifdef B200S_EMU
	*p = malloc(bytes);
	return *p != 0;
#else
	return cudaMallocHost(p, bytes) == cudaSuccess;
#endif
}
static void host_free(void *p) {
#ifdef B200S_EMU
	free(p);
#else
	if (p) cudaFreeHost(p);
#endif
}

static void free_all(b200s_engine *e) {
	dfree(e->dWindow); dfree(e->dWinProd); dfree(e->dWpReset); dfree(e->dWpDiv); dfree(e->dRot); dfree(e->dTwiddle); dfree(e->dPretw); dfree(e->dAnaTab);
	dfree(e->dSched); dfree(e->dHist[0]); dfree(e->dHist[1]); dfree(e->dPend); dfree(e->dPendWp);
	dfree(e->dStIn); dfree(e->dStPrev); dfree(e->dStOut); dfree(e->dStPredE); dfree(e->dStIl);
	dfree(e->dFrames); dfree(e->dCall); dfree(e->dJobs); dfree(e->dSpec); dfree(e->dY); dfree(e->dPI); dfree(e->dFT); dfree(e->dT1); dfree(e->dT2); dfree(e->dE); dfree(e->dS); dfree(e->dM); dfree(e->dT1u); dfree(e->dT2u); dfree(e->dRngPow); dfree(e->dStPitch);
	dfree(e->dMapB); dfree(e->dMapG); dfree(e->dRatio); dfree(e->dTE); dfree(e->dTPI); dfree(e->dTFT); dfree(e->dTT1); dfree(e->dTT2);
	e->randFrames = e->tFrames = 0; dfree(e->dPitch);
	dfree(e->dIn); dfree(e->dOut); dfree(e->dZero); dfree(e->dTmp); dfree(e->dIn16); dfree(e->dOut16);
	e->in16Cap = e->out16Cap = 0;
	e->maxFrames = e->coefFrames = 0;
	e->inCap = e->outCap = e->zeroCap = e->tmpCap = 0;
}

static Ctx make_ctx(b200s_engine *e) {
	Ctx x;
	memset(&x, 0, sizeof(x));
	x.cfg = e->cfg;
	x.maps = e->dMaps;
	x.sprm = e->dSprm;
	x.window = e->dWindow; x.winProd = e->dWinProd; x.wpReset = e->dWpReset; x.wpDiv = e->dWpDiv;
	x.rot = e->dRot; x.twiddle = e->dTwiddle; x.pretw = e->dPretw; x.anaTab = e->dAnaTab;
	x.rot0 = e->rot0; x.rotStep = e->rotStep;
	x.one = 1.0f;
	x.sched = e->dSched;
	x.histCur = e->dHist[e->histCur]; x.histNext = e->dHist[e->histCur ^ 1];
	x.pend = e->dPend; x.pendWp = e->dPendWp;
	x.stIn = e->dStIn; x.stPrev = e->dStPrev; x.stOut = e->dStOut; x.stPredE = e->dStPredE; x.stIl = e->dStIl;
	x.maxFrames = e->maxFrames;
	x.sBase = 0; x.sCount = e->S;
	x.frames = e->dFrames; x.call = e->dCall; x.jobs = e->dJobs;
	x.spec = e->dSpec; x.Y = e->dY; x.cPI = e->dPI; x.cFT = e->dFT; x.cT1 = e->dT1; x.cT2 = e->dT2; x.cE = e->dE; x.cS = e->dS; x.cM = e->dM; x.cT1u = e->dT1u; x.cT2u = e->dT2u;
	x.cMapB = e->dMapB; x.cMapG = e->dMapG; x.cRatio = e->dRatio; x.tE = e->dTE; x.tPI = e->dTPI; x.tFT = e->dTFT; x.tT1 = e->dTT1; x.tT2 = e->dTT2;
	x.tRows = t_rows(e->cfg); x.tGroups = (e->maxFrames + 31) / 32;
	x.rngState = e->dRng; x.rngPow = e->dRngPow; x.rngJump = e->rngJump; x.diag = e->dDiag; x.stPitch = e->dStPitch; x.cPitch = e->dPitch;
	return x;
}

// complex FFT size the dependency picks for a block: 2^k * {1,3,5} (SURVEY.md App. B, measured)
static int fast_size_above(int n) {
	int p = 1;
	while (p < 16 && p < n) p *= 2;
	while (8 * p < n) p *= 2;
	int m = (n + p - 1) / p;
	if (m == 7) m = 8;
	return m * p;
}
static double bessel0(double x) {
	double sum = 1, term = 1, q = x * x * 0.25;
	for (int k = 1; k < 200; ++k) {
		term *= q / (double(k) * k);
		sum += term;
		if (term < sum * 1e-17) break;
	}
	return sum;
}

static const int kThreads = 256;
static size_t smem_analyse(const Cfg &g) { return sizeof(float2) * 2 * fft_buf_len(g.K) + sizeof(float) * (g.B + 4); }
static size_t smem_prep(const Cfg &g, bool formants = true) { return sizeof(float) * ((formants ? 7 : 6) * (size_t)g.K + 8); }
static size_t smem_synth(const Cfg &g) { return sizeof(float2) * 2 * fft_buf_len(g.K) + sizeof(float) * 2 * g.pendLen; }

// PK_PHASE: the pre and post phases of b200s_run_per_stream (reported when the caller's arrays have room for it)
enum { PK_PLAN = 0, PK_ANALYSE, PK_PREP, PK_CHAIN, PK_SYNTH, PK_COMMIT, PK_PHASE, PK_COUNT };
static int prof_mark(b200s_engine *e, int kind, bool begin) {
	if (!e->profiling) return 0;
	cudaEvent_t ev;
	CK(cudaEventCreate(&ev));
	CK(cudaEventRecord(ev, e->stream));
	e->profEv.push_back(ev);
	if (begin) e->profKind.push_back(kind);
	return 0;
}
#define PROF(kind, stmt)                          \
	do {                                          \
		int _rc;                                  \
		if ((_rc = prof_mark(e, kind, true))) return _rc;  \
		stmt;                                     \
		CKL();                                    \
		if ((_rc = prof_mark(e, kind, false))) return _rc; \
	} while (0)

typedef void (*ChainKernel)(Ctx);
// Superseded kernel generations (first-generation FFT kernels specialised for the preset sizes, chain generations 1, 3 and 5)
// are only instantiated with -DB200S_KEEP_OLD_KERNELS (the emulator test builds: cross-checks between generations); the
// shipped library carries the generic FFT kernels (any size), k_chain (any configuration), k_chain_direct2 / 4 / 6, k_chain_t.
#ifdef B200S_KEEP_OLD_KERNELS
static ChainKernel analyse_kernel(const Cfg &g) { return g.K == 3072 ? k_analyse<3072> : g.K == 2560 ? k_analyse<2560> : k_analyse<0>; }
#else
static ChainKernel analyse_kernel(const Cfg &) { return k_analyse<0>; }
#endif
// paired in-place FFT kernels (stft2.cuh) for the preset sizes
static bool use_pair_fft(const Cfg &g, int forceV1 = 0) {
	static int v1 = -1;
	if (v1 < 0) v1 = getenv("B200S_FFT_V1") ? 1 : 0; // A/B switch for profiling the first-generation kernels
	return !v1 && !forceV1 && (g.K == 3072 || g.K == 2560);
}
#ifdef B200S_ANALYSE_PROBES // profiling builds only: ablations of k_analyse2<3072> (wrong results), B200S_ANALYSE_PROBE=1..4
static int analyse_probe() {
	static int probe = -1;
	if (probe < 0) {
		const char *pv = getenv("B200S_ANALYSE_PROBE");
		probe = pv ? atoi(pv) : 0;
	}
	return probe;
}
#endif
// mixed: a stereo call with interleaved rows for its plain streams and planar rows for its mapped ones (§3.9 of DESIGN.md),
// or a call over a list of streams (§3.13)
static ChainKernel analyse2_kernel(const Cfg &g, bool mixed = false) {
	if (mixed) return g.K == 3072 ? k_analyse2_mixed<3072> : k_analyse2_mixed<2560>;
#ifdef B200S_ANALYSE_PROBES
	if (g.K == 3072) switch (analyse_probe()) {
		case 1: return k_analyse2<3072, 1>;
		case 2: return k_analyse2<3072, 2>;
		case 3: return k_analyse2<3072, 3>;
		case 4: return k_analyse2<3072, 4>;
		default: break;
		}
#endif
	return g.K == 3072 ? k_analyse2<3072> : k_analyse2<2560>;
}
#ifdef B200S_SYNTH_PROBES // profiling builds only: ablations of k_synth2<3072> (wrong results), B200S_SYNTH_PROBE=1..4
static int synth_probe() {
	static int probe = -1;
	if (probe < 0) {
		const char *pv = getenv("B200S_SYNTH_PROBE");
		probe = pv ? atoi(pv) : 0;
	}
	return probe;
}
#endif
static ChainKernel synth2_kernel(const Cfg &g) {
#ifdef B200S_SYNTH_PROBES
	if (g.K == 3072) switch (synth_probe()) {
		case 1: return k_synth2_probe<3072, 1>;
		case 2: return k_synth2_probe<3072, 2>;
		case 3: return k_synth2_probe<3072, 3>;
		case 4: return k_synth2_probe<3072, 4>;
		default: break;
		}
#endif
	return g.K == 3072 ? k_synth2<3072> : k_synth2<2560>;
}
#ifdef B200S_KEEP_OLD_KERNELS
static ChainKernel synth_kernel(const Cfg &g) { return g.K == 3072 ? k_synth<3072> : g.K == 2560 ? k_synth<2560> : k_synth<0>; }
#else
static ChainKernel synth_kernel(const Cfg &) { return k_synth<0>; }
#endif
template <int CT>
static ChainKernel chain_kernel_for(int L, bool direct) {
#ifdef B200S_KEEP_OLD_KERNELS
	if (direct) switch (L) {
		case 1: return k_chain_direct<CT, 1>;
		case 2: return k_chain_direct<CT, 2>;
		case 3: return k_chain_direct<CT, 3>;
		case 4: return k_chain_direct<CT, 4>;
		case 5: return k_chain_direct<CT, 5>;
		case 6: return k_chain_direct<CT, 6>;
		case 7: return k_chain_direct<CT, 7>;
		default: return k_chain_direct<CT, 8>;
		}
#endif
	(void)direct; // (without the old generations chain_version() never asks for the first-generation direct kernel)
	switch (L) {
	case 1: return k_chain<CT, 1, false>;
	case 2: return k_chain<CT, 2, false>;
	case 3: return k_chain<CT, 3, false>;
	case 4: return k_chain<CT, 4, false>;
	case 5: return k_chain<CT, 5, false>;
	case 6: return k_chain<CT, 6, false>;
	case 7: return k_chain<CT, 7, false>;
	default: return k_chain<CT, 8, false>;
	}
}
// second-generation direct chain: lane = (block, channel), several warps per stream (chain_direct2.cuh)
template <int CT, bool FAST>
static ChainKernel chain2_kernel_for(int L) {
	switch (L) {
	case 1: return k_chain_direct2<CT, 1, FAST>;
	case 2: return k_chain_direct2<CT, 2, FAST>;
	case 3: return k_chain_direct2<CT, 3, FAST>;
	case 4: return k_chain_direct2<CT, 4, FAST>;
	case 5: return k_chain_direct2<CT, 5, FAST>;
	case 6: return k_chain_direct2<CT, 6, FAST>;
	case 7: return k_chain_direct2<CT, 7, FAST>;
	default: return k_chain_direct2<CT, 8, FAST>;
	}
}
// fast = the fused arithmetic (mono only: the stereo default is the packed kernel, whose exact cross-check this one is)
static ChainKernel chain2_kernel(const Cfg &g, bool fast = false) {
	return g.C == 1 ? (fast ? chain2_kernel_for<1, true>(g.L) : chain2_kernel_for<1, false>(g.L)) : chain2_kernel_for<2, false>(g.L);
}
// warps per stream for a call of nOut output samples: one per 32/C blocks (blocks trigger every H samples)
static int chain2_warps(const Cfg &g, int nOut) {
	const int blocks = (nOut + g.H - 1) / g.H, bpw = 32 / g.C;
	return std::max(1, std::min(CH2_MAXW, (blocks + bpw - 1) / bpw));
}
// which direct chain kernel: 3 = packed stereo (chain_direct3.cuh, needs the paired analysis kernel),
// 2 = lane-per-(block,channel) multi-warp (chain_direct2.cuh), 1 = first generation; B200S_CHAIN_V overrides (A/B profiling)
static int chain_version(const Cfg &g, int override, int forceFftV1) {
	static int env = -1;
	if (env < 0) {
		const char *v = getenv("B200S_CHAIN_V");
		env = v ? atoi(v) : 0;
	}
	// default 4: the warp-specialised kernel (5) doubles the shared-memory traffic per step with its tile hand-off and its
	// consumer waits for the producer
	int want = override ? override : env ? env : 4;
	// (the packed stereo chains take whole 8-bin chunks of every row: K % CHAIN_CH == 0, true of both paired FFT sizes)
	if (want >= 3 && !(g.C == 2 && use_pair_fft(g, forceFftV1) && g.K % CHAIN_CH == 0)) want = 2;
	if (want == 5 && g.L > 4) want = 4; // k_chain_ws is laid out for L <= 4 (both presets)
#ifndef B200S_KEEP_OLD_KERNELS
	if (want == 1) want = 2;
	if (want == 3 || want == 5) want = 4;
#endif
	return want;
}
// 5 = warp-specialised producer / consumer chain (chain_ws.cuh), followed by k_chain_direct4 for the streams it leaves
#ifdef B200S_KEEP_OLD_KERNELS
template <bool FAST>
static ChainKernel chain_ws_kernel(int L) {
	switch (L) {
	case 1: return k_chain_ws<1, FAST>;
	case 2: return k_chain_ws<2, FAST>;
	case 3: return k_chain_ws<3, FAST>;
	default: return k_chain_ws<4, FAST>;
	}
}
#endif
template <bool FAST>
static ChainKernel chain4_kernel(int L) {
	switch (L) {
	case 1: return k_chain_direct4<1, FAST>;
	case 2: return k_chain_direct4<2, FAST>;
	case 3: return k_chain_direct4<3, FAST>;
	case 4: return k_chain_direct4<4, FAST>;
	case 5: return k_chain_direct4<5, FAST>;
	case 6: return k_chain_direct4<6, FAST>;
	case 7: return k_chain_direct4<7, FAST>;
	default: return k_chain_direct4<8, FAST>;
	}
}
template <bool FAST, bool DUAL>
static ChainKernel chain6_kernel(int L) {
	switch (L) {
	case 1: return k_chain_direct6<1, FAST, DUAL>;
	case 2: return k_chain_direct6<2, FAST, DUAL>;
	case 3: return k_chain_direct6<3, FAST, DUAL>;
	case 4: return k_chain_direct6<4, FAST, DUAL>;
	case 5: return k_chain_direct6<5, FAST, DUAL>;
	case 6: return k_chain_direct6<6, FAST, DUAL>;
	case 7: return k_chain_direct6<7, FAST, DUAL>;
	default: return k_chain_direct6<8, FAST, DUAL>;
	}
}
// mono plain path: pairs of streams on the packed wavefront (k_chain_direct6<.., DUAL>) instead of k_chain_direct2.  Off by
// default: although it issues 40 % fewer instructions per stream, the wavefront kernels are bound by dependent latency, not by
// issue.
// B200S_DUAL=1 / b200s_set_tuning(e, 5, 1) switch it on (cross-check in the tests).
static bool dual_enabled() {
	static int env = -1;
	if (env < 0) {
		const char *v = getenv("B200S_DUAL");
		env = v ? (atoi(v) != 0) : 0;
	}
	return env != 0;
}
static ChainKernel chain3_kernel(const Cfg &g, int v, bool fast) {
#ifdef B200S_CHAIN_PROBES // profiling builds only: ablations of k_chain_direct6 (wrong results), B200S_CHAIN_PROBE=1..7
	if (v >= 6 && fast && g.L == 4) {
		static int probe = -1;
		if (probe < 0) {
			const char *pv = getenv("B200S_CHAIN_PROBE");
			probe = pv ? atoi(pv) : 0;
		}
		switch (probe) {
		case 1: return k_chain_direct6<4, true, false, 1>;
		case 2: return k_chain_direct6<4, true, false, 2>;
		case 3: return k_chain_direct6<4, true, false, 3>;
		case 4: return k_chain_direct6<4, true, false, 4>;
		case 5: return k_chain_direct6<4, true, false, 5>;
		case 6: return k_chain_direct6<4, true, false, 6>;
		case 7: return k_chain_direct6<4, true, false, 7>;
		default: break;
		}
	}
#endif
	if (v >= 6) return fast ? chain6_kernel<true, false>(g.L) : chain6_kernel<false, false>(g.L);
	if (v >= 4) return fast ? chain4_kernel<true>(g.L) : chain4_kernel<false>(g.L);
#ifdef B200S_KEEP_OLD_KERNELS
	switch (g.L) {
	case 1: return k_chain_direct3<1>;
	case 2: return k_chain_direct3<2>;
	case 3: return k_chain_direct3<3>;
	case 4: return k_chain_direct3<4>;
	case 5: return k_chain_direct3<5>;
	case 6: return k_chain_direct3<6>;
	case 7: return k_chain_direct3<7>;
	default: return k_chain_direct3<8>;
	}
#else
	return fast ? chain4_kernel<true>(g.L) : chain4_kernel<false>(g.L);
#endif
}
template <int CT>
static ChainKernel chain_t_kernel_for(int L) {
	switch (L) {
	case 1: return k_chain_t<CT, 1>;
	case 2: return k_chain_t<CT, 2>;
	case 3: return k_chain_t<CT, 3>;
	case 4: return k_chain_t<CT, 4>;
	case 5: return k_chain_t<CT, 5>;
	case 6: return k_chain_t<CT, 6>;
	case 7: return k_chain_t<CT, 7>;
	default: return k_chain_t<CT, 8>;
	}
}
static ChainKernel chain_t_kernel(const Cfg &g) { return g.C == 1 ? chain_t_kernel_for<1>(g.L) : chain_t_kernel_for<2>(g.L); }
static ChainKernel chain_kernel(const Cfg &g, bool direct) {
	return g.C == 1 ? chain_kernel_for<1>(g.L, direct) : chain_kernel_for<2>(g.L, direct);
}
static const int kChainWarps = 1; // one stream per CTA: 1024 streams spread evenly over the SMs
static size_t smem_chain(const Cfg &g, bool direct, bool randTiles = false) {
	size_t per = direct ? (g.C == 1 ? sizeof(DirectTiles2<1>) : sizeof(DirectTiles2<2>)) : (g.C == 1 ? sizeof(ChainTiles<1>) : sizeof(ChainTiles<2>));
	if (!direct && randTiles) per += g.C == 1 ? sizeof(ChainRandTiles<1>) : sizeof(ChainRandTiles<2>);
	return per * kChainWarps;
}

static int reset_impl(b200s_engine *e, bool full) {
	e->chainedGroups = 0;
	Ctx x = make_ctx(e);
	B200S_LAUNCH(k_reset_stft, dim3(e->S), dim3(kThreads), 0, e->stream, x);
	CKL();
	B200S_LAUNCH(k_reset_bands, dim3(e->S), dim3(kThreads), 0, e->stream, x, full ? 15 : 6);
	CKL();
	return 0;
}

static int configure_impl(b200s_engine *e, int channels, int block, int interval, int split) {
	if (!e) return B200S_EINVAL;
	if (channels < 1 || block < 4 || interval < 1 || interval > block) {
		e->err = "configure: need channels >= 1, block >= 4, 1 <= interval <= block";
		return B200S_EINVAL;
	}
	Cfg g;
	memset(&g, 0, sizeof(g));
	g.S = e->S;
	g.C = channels;
	g.B = block;
	g.H = interval;
	g.N = 2 * fast_size_above((block + 1) / 2); // DynamicSTFT::configure (App. B)
	g.K = g.N / 2;
	g.L = (int)std::round(float(g.N) / float(g.H)); // :636-637
	g.split = split ? 1 : 0;
	g.histLen = g.B + g.H;
	g.pendLen = g.B + (g.split ? g.H : 0);
	g.addOff = g.split ? g.H : 0;
	g.o = g.B / 2;
	{ // Stockham plan: power-of-two radices first (16s, then 8/4/2), the radix carrying the odd factor last
		int k = g.K, odd = 1, n = 0;
		if (k % 3 == 0) { odd = 3; k /= 3; }
		else if (k % 5 == 0) { odd = 5; k /= 5; }
		int last = odd;
		if (odd == 3) { int c = 0; while (c < 2 && k % 2 == 0 && k > 1) { last *= 2; k /= 2; ++c; } } // 12, 6 or 3
		if (odd == 5) { if (k % 2 == 0 && k > 1) { last *= 2; k /= 2; } }                            // 10 or 5
		if (k & (k - 1)) { e->err = "unsupported FFT size"; return B200S_EUNSUPPORTED; }
		while (k % 16 == 0 && k > 16) { g.radix[n++] = 16; k /= 16; }
		if (k == 16 && last > 1) { g.radix[n++] = 16; k = 1; }
		else if (k == 16) { g.radix[n++] = 4; last = 4; k = 1; }
		if (k == 8) { g.radix[n++] = 8; k = 1; }
		if (k == 4) { g.radix[n++] = 4; k = 1; }
		if (k == 2) { g.radix[n++] = 2; k = 1; }
		if (last > 1) g.radix[n++] = last;
		g.nStages = n;
		int prod = 1;
		for (int i = 0; i < n; ++i) prod *= g.radix[i];
		if (prod != g.K) { e->err = "internal: FFT plan does not factor the size"; return B200S_EUNSUPPORTED; }
	}
	if (g.L < 1 || g.L > 8 || (channels > 2)) {
		e->err = "GPU path supports 1-2 channels and block/interval ratios with round(fftSamples/interval) in 1..8";
		return B200S_EUNSUPPORTED;
	}
	if (smem_prep(g) > 220 * 1024 || smem_synth(g) > 220 * 1024) {
		e->err = "block too large for the shared-memory FFT (bands must be <= ~6144)";
		return B200S_EUNSUPPORTED;
	}
	CK(cudaSetDevice(e->device));
	CK(cudaStreamSynchronize(e->stream));
	free_all(e);
	e->cfg = g;

	// ---- tables.  Window: Kaiser, the dependency's bandwidth heuristic, forced perfect reconstruction (App. B)
	std::vector<float> window(g.B), winProd(g.B), wpReset(g.pendLen), wpDiv(g.H);
	{
		double bw = double(g.B) / double(g.H);
		bw += 8 / ((bw + 3) * (bw + 3)) + 0.25 * std::max(3 - bw, 0.0);
		bw = std::max(bw, 2.0);
		double beta = M_PI * std::sqrt(bw * bw * 0.25 - 1);
		std::vector<double> w(g.B);
		for (int i = 0; i < g.B; ++i) {
			double r = (2.0 * i + 1) / g.B - 1;
			w[i] = bessel0(beta * std::sqrt(std::max(0.0, 1 - r * r))) / bessel0(beta);
		}
		for (int i = 0; i < g.H && i < g.B; ++i) {
			double s2 = 0;
			for (int k = i; k < g.B; k += g.H) s2 += w[k] * w[k];
			double f = 1 / std::sqrt(s2);
			for (int k = i; k < g.B; k += g.H) w[k] *= f;
		}
		for (int i = 0; i < g.B; ++i) {
			window[i] = float(w[i]);
			winProd[i] = window[i] * window[i] * float(g.N);
		}
		for (int i = 0; i < g.pendLen; ++i) { // DynamicSTFT::reset(0.1) then moveOutput(H)
			int ring = i + g.H;
			if (ring < g.B) {
				float sum = 0;
				for (int k = ring; k < g.B; k += g.H) sum += window[k] * window[k];
				wpReset[i] = 0.1f * float(g.N) * sum + B200S_ALMOST_ZERO;
			} else {
				wpReset[i] = B200S_ALMOST_ZERO;
			}
		}
		// windowProducts of a slot at phase j that every block of a run H apart has reached: the ceil((B - j) / H) blocks
		// that cover it, added to the cleared slot oldest first, as the overlap-add ring does (:397-399)
		for (int j = 0; j < g.H; ++j) {
			float sum = B200S_ALMOST_ZERO;
			for (int k = (g.B - j + g.H - 1) / g.H - 1; k >= 0; --k) sum = sum + winProd[j + k * g.H];
			wpDiv[j] = sum;
		}
	}
	std::vector<float2> rot(g.K), tw(g.K), pre(g.K);
	{ // :647-655, the reference's own float recurrence (its rounding is part of the result)
		auto b2f = [&](float b) { return (b + 0.5f) / float(g.N); };
		std::complex<float> r = std::polar(1.0f, b2f(0) * float(g.H) * float(2 * M_PI));
		float freqStep = b2f(1) - b2f(0);
		std::complex<float> step = std::polar(1.0f, freqStep * float(g.H) * float(2 * M_PI));
		e->rot0 = make_float2(r.real(), r.imag());
		e->rotStep = make_float2(step.real(), step.imag());
		for (int b = 0; b < g.K; ++b) {
			rot[b] = make_float2(r.real(), r.imag());
			r = std::complex<float>(r.real() * step.real() - r.imag() * step.imag(), r.real() * step.imag() + r.imag() * step.real());
		}
		for (int t = 0; t < g.K; ++t) {
			tw[t] = make_float2(float(std::cos(-2.0 * M_PI * t / g.K)), float(std::sin(-2.0 * M_PI * t / g.K)));
			pre[t] = make_float2(float(std::cos(-M_PI * t / g.N)), float(std::sin(-M_PI * t / g.N)));
		}
	}
	int rc;
	if ((rc = dalloc(e, &e->dWindow, g.B))) return rc;
	if ((rc = dalloc(e, &e->dWinProd, g.B))) return rc;
	if ((rc = dalloc(e, &e->dWpReset, g.pendLen))) return rc;
	if ((rc = dalloc(e, &e->dWpDiv, g.H))) return rc;
	if ((rc = dalloc(e, &e->dRot, g.K))) return rc;
	if ((rc = dalloc(e, &e->dTwiddle, g.K))) return rc;
	if ((rc = dalloc(e, &e->dPretw, g.K))) return rc;
	CK(cudaMemcpy(e->dWindow, window.data(), sizeof(float) * g.B, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(e->dWinProd, winProd.data(), sizeof(float) * g.B, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(e->dWpReset, wpReset.data(), sizeof(float) * g.pendLen, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(e->dWpDiv, wpDiv.data(), sizeof(float) * g.H, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(e->dRot, rot.data(), sizeof(float2) * g.K, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(e->dTwiddle, tw.data(), sizeof(float2) * g.K, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(e->dPretw, pre.data(), sizeof(float2) * g.K, cudaMemcpyHostToDevice));
	{ // per-element constants of the analysis load stage, one float4 each
		std::vector<float4> tab(g.K);
		for (int n = 0; n < g.K; ++n) {
			const int i0 = n + g.o, i1 = n + g.o - g.K;
			tab[n] = make_float4(i0 < g.B ? window[i0] : 0.f, i1 >= 0 ? window[i1] : 0.f, pre[n].x, pre[n].y);
		}
		if ((rc = dalloc(e, &e->dAnaTab, g.K))) return rc;
		CK(cudaMemcpy(e->dAnaTab, tab.data(), sizeof(float4) * g.K, cudaMemcpyHostToDevice));
	}

	{ // powers of the random engine's multiplier: draw i of a block is state * 16807^i mod 2^31-1 (kernels.cuh)
		std::vector<unsigned> pw(2 * (size_t)g.K);
		unsigned v = 1;
		for (size_t i = 0; i < pw.size(); ++i) {
			pw[i] = v;
			v = rng_mulmod(v, B200S_RNG_A);
		}
		e->rngJump = pw[2 * (size_t)g.K - 2];
		if ((rc = dalloc(e, &e->dRngPow, pw.size()))) return rc;
		CK(cudaMemcpy(e->dRngPow, pw.data(), sizeof(unsigned) * pw.size(), cudaMemcpyHostToDevice));
		if (!e->dRng) { // std::default_random_engine(seed): state = seed mod (2^31-1), 1 if that is 0; NOT touched by configure / reset
			if ((rc = dalloc(e, &e->dRng, (size_t)g.S))) return rc;
			unsigned x0 = (unsigned)((unsigned long long)e->seed % (unsigned long long)B200S_RNG_M);
			if (x0 == 0) x0 = 1;
			std::vector<unsigned> st((size_t)g.S, x0);
			CK(cudaMemcpy(e->dRng, st.data(), sizeof(unsigned) * st.size(), cudaMemcpyHostToDevice));
			if ((rc = dalloc(e, &e->dDiag, (size_t)1))) return rc;
			CK(cudaMemset(e->dDiag, 0, sizeof(unsigned long long)));
		}
	}

	if (!e->dSprm) { // the per-stream parameter table (kept over configure, like the parameters themselves)
		if ((rc = dalloc(e, &e->dSprm, (size_t)g.S))) return rc;
		e->sprmDirty = true;
	}
	if (!e->dDesc && (rc = dalloc(e, &e->dDesc, (size_t)g.S))) return rc; // per-stream call descriptors (filled by every per-stream call)

	// ---- state
	const size_t SC = (size_t)g.S * g.C;
	if ((rc = dalloc(e, &e->dSched, g.S))) return rc;
	if ((rc = dalloc(e, &e->dHist[0], SC * g.histLen))) return rc;
	if ((rc = dalloc(e, &e->dHist[1], SC * g.histLen))) return rc;
	if ((rc = dalloc(e, &e->dPend, SC * g.pendLen))) return rc;
	if ((rc = dalloc(e, &e->dPendWp, SC * g.pendLen))) return rc;
	if ((rc = dalloc(e, &e->dStIn, SC * g.K))) return rc;
	if ((rc = dalloc(e, &e->dStPrev, SC * g.K))) return rc;
	if ((rc = dalloc(e, &e->dStOut, SC * g.K))) return rc;
	if ((rc = dalloc(e, &e->dStPredE, SC * g.K))) return rc;
	if ((rc = dalloc(e, &e->dStIl, g.C == 2 ? (size_t)g.S * 2 * g.K : 1))) return rc;
	if ((rc = dalloc(e, &e->dCall, g.S))) return rc;
	CK(cudaMemset(e->dStPredE, 0, sizeof(float) * SC * g.K));
	if ((rc = dalloc(e, &e->dStPitch, (size_t)g.S * 2))) return rc;
	CK(cudaMemset(e->dStPitch, 0, sizeof(float) * (size_t)g.S * 2));
	CK(cudaMemset(e->dHist[1], 0, sizeof(float) * SC * g.histLen));
	{
		std::vector<Sched> sc(g.S);
		for (auto &s : sc) {
			s.samplesSinceLast = B200S_NEVER;
			s.silenceCounter = 0;
			s.prevInputOffset = -1;
			s.didSeek = 0;
			s.silenceFirst = 1;
			s.seekTimeFactor = 1;
			s.zeroRun = B200S_NEVER;
		}
		CK(cudaMemcpy(e->dSched, sc.data(), sizeof(Sched) * g.S, cudaMemcpyHostToDevice));
	}
	e->histCur = 0;
#ifndef B200S_EMU
	CK(cudaFuncSetAttribute(analyse_kernel(g), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_analyse(g)));
	CK(cudaFuncSetAttribute(k_prep, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_prep(g)));
	CK(cudaFuncSetAttribute(synth_kernel(g), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_synth(g)));
	CK(cudaFuncSetAttribute(k_flush_tail, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(float) * g.B)));
	CK(cudaFuncSetAttribute(chain_kernel(g, false), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_chain(g, false, true)));
#ifdef B200S_KEEP_OLD_KERNELS // (without the old generations chain_kernel(g, true) is the same function: do not shrink its limit again)
	CK(cudaFuncSetAttribute(chain_kernel(g, true), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_chain(g, true)));
#endif
	CK(cudaFuncSetAttribute(chain2_kernel(g), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_chain2(g.C, CH2_MAXW)));
	CK(cudaFuncSetAttribute(chain2_kernel(g, true), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_chain2(g.C, CH2_MAXW)));
#ifdef B200S_KEEP_OLD_KERNELS
	if (g.L <= 4) { // seven two-warp CTAs of 30.6 KB per SM: ask for the full shared-memory carve-out
		CK(cudaFuncSetAttribute(chain_ws_kernel<true>(g.L), cudaFuncAttributePreferredSharedMemoryCarveout, 100));
		CK(cudaFuncSetAttribute(chain_ws_kernel<false>(g.L), cudaFuncAttributePreferredSharedMemoryCarveout, 100));
	}
#endif
	// k_chain_direct6: seven one-warp CTAs of 31.5 KB per SM need the full shared-memory carve-out
	CK(cudaFuncSetAttribute(g.C == 1 ? chain6_kernel<true, true>(g.L) : chain6_kernel<true, false>(g.L), cudaFuncAttributePreferredSharedMemoryCarveout, 100));
	CK(cudaFuncSetAttribute(g.C == 1 ? chain6_kernel<false, true>(g.L) : chain6_kernel<false, false>(g.L), cudaFuncAttributePreferredSharedMemoryCarveout, 100));
	if (use_pair_fft(g)) {
		CK(cudaFuncSetAttribute(analyse2_kernel(g), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_analyse2(g)));
		CK(cudaFuncSetAttribute(analyse2_kernel(g, true), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_analyse2(g)));
		CK(cudaFuncSetAttribute(synth2_kernel(g), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_synth2(g)));
	}
	{
		int n = 0;
		if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, e->device) == cudaSuccess && n > 0) e->numSMs = n;
	}
#endif
	e->configured = true;
	return reset_impl(e, true);
}

static int frames_bound(const Cfg &g, int nOut) { return nOut <= 0 ? 0 : (nOut + g.H - 1) / g.H + 1; }

static int ensure_scratch(b200s_engine *e, int nOut) {
	const Cfg &g = e->cfg;
	int need = std::max(frames_bound(g, nOut), 1);
	if (need <= e->maxFrames) return 0;
	CK(cudaStreamSynchronize(e->stream));
	const size_t n = (size_t)g.S * need * g.C * g.K;
	int rc;
	if ((rc = dalloc(e, &e->dFrames, (size_t)g.S * need))) return rc;
	if ((rc = dalloc(e, &e->dJobs, (size_t)g.S * need * 2 * g.C))) return rc;
	if ((rc = dalloc(e, &e->dSpec, 2 * n))) return rc;
	if ((rc = dalloc(e, &e->dY, n))) return rc;
	if ((rc = dalloc(e, &e->dE, n))) return rc; // Prediction::energy rows: also the state carry of the generic direct chains
	if ((rc = dalloc(e, &e->dPitch, (size_t)g.S * need))) return rc;
	e->maxFrames = need;
	// the complex coefficient rows follow maxFrames (their row offsets use it) but only exist once a call needed them
	dfree(e->dPI); dfree(e->dFT); dfree(e->dT1); dfree(e->dT2); dfree(e->dS); dfree(e->dM); dfree(e->dT1u); dfree(e->dT2u);
	dfree(e->dMapB); dfree(e->dMapG); dfree(e->dRatio); dfree(e->dTE); dfree(e->dTPI); dfree(e->dTFT); dfree(e->dTT1); dfree(e->dTT2);
	e->coefFrames = e->randFrames = e->tFrames = 0;
	return 0;
}
// The counts over the per-stream table that decide a call's kernels (k_plan decides each stream's path by the same test)
static void count_paths(b200s_engine *e) {
	e->nMapped = 0;
	e->anyFormants = e->anyAutoPitch = false;
	for (const StreamParams &p : e->hSprm) {
		const bool mapped = stream_mapped(p), formants = stream_formants(p, mapped);
		e->nMapped += (mapped || formants) ? 1 : 0;
		e->anyFormants = e->anyFormants || formants;
		e->anyAutoPitch = e->anyAutoPitch || (formants && !(p.formantBaseFreq > 0));
	}
}
static void params_changed(b200s_engine *e) {
	count_paths(e);
	e->sprmDirty = true;
}

// ---- the frequency-map pool ----
// the table a stream's descriptor points at (null: none)
static const MapTable *stream_table(const b200s_engine *e, const StreamParams &p) {
	if (p.mapN == 0) return nullptr;
	return &*std::lower_bound(e->maps.begin(), e->maps.end(), p.mapOff, [](const MapTable &t, int off) { return t.off < off; });
}
// The whole pool from the host copies, grown (to at least twice its capacity) when it has no room.  The caller has
// synchronised the handle's stream: kernels in flight may read the pool.
static int upload_maps(b200s_engine *e) {
	int rc;
	if (e->mapsUsed > e->mapsCap) {
		const size_t cap = std::max(e->mapsUsed, 2 * e->mapsCap);
		if ((rc = dalloc(e, &e->dMaps, cap))) return rc;
		e->mapsCap = cap;
	}
	if (e->mapsUsed == 0) return 0;
	std::vector<float> all(e->mapsUsed);
	for (const MapTable &t : e->maps) std::copy(t.pts.begin(), t.pts.end(), all.begin() + t.off);
	CK(cudaMemcpy(e->dMaps, all.data(), sizeof(float) * all.size(), cudaMemcpyHostToDevice));
	return 0;
}
// Lays the pool out afresh from the tables in use and uploads it: the engine's table, then each stream's (the engine's
// for kMapEngine; for kMapOwn want[s] when given, otherwise the one it has).  Tables nobody uses any more are dropped.
// Synchronises the handle's stream.
static int layout_maps(b200s_engine *e, const std::vector<const MapTable *> &want) {
	CK(cudaStreamSynchronize(e->stream));
	std::vector<MapTable> pool;
	std::unordered_map<uint64_t, std::vector<size_t>> byHash;
	size_t used = 0;
	auto intern = [&](const MapTable &t) {
		for (size_t i : byHash[t.hash])
			if (same_points(pool[i], t)) return pool[i].off;
		byHash[t.hash].push_back(pool.size());
		pool.push_back(t);
		pool.back().off = (int)used;
		used += t.pts.size();
		return pool.back().off;
	};
	if (e->engMap.n > 0) e->engMap.off = intern(e->engMap);
	std::vector<StreamParams> prm = e->hSprm;
	for (int s = 0; s < e->S; ++s) {
		StreamParams &p = prm[s];
		const MapTable *t = p.customMap == kMapEngine ? (e->engMap.n > 0 ? &e->engMap : nullptr)
		                    : p.customMap == kMapOwn  ? (want.empty() || !want[s] ? stream_table(e, p) : want[s])
		                                              : nullptr;
		p.mapOff = t ? intern(*t) : 0;
		p.mapN = t ? t->n : 0;
		if (used > (size_t)INT_MAX) {
			e->err = "frequency-map tables: more than 2^31-1 floats in all";
			return B200S_EINVAL;
		}
	}
	e->maps = std::move(pool);
	e->mapsUsed = used;
	e->hSprm = std::move(prm);
	params_changed(e);
	return upload_maps(e);
}
static cudaError_t copy_peer(void *dst, int dstDevice, const void *src, int srcDevice, size_t bytes, cudaStream_t st);
// The table of a stream that comes from another engine, in dst's pool: found there by content, or appended and copied
// from src's pool on dst's stream (no host synchronisation).  Growing the pool synchronises dst and uploads it whole.
static int carry_table(b200s_engine *dst, const b200s_engine *src, const MapTable &t, int *off) {
	b200s_engine *e = dst;
	for (const MapTable &m : dst->maps)
		if (same_points(m, t)) {
			*off = m.off;
			return 0;
		}
	dst->maps.push_back(t);
	*off = dst->maps.back().off = (int)dst->mapsUsed;
	dst->mapsUsed += t.pts.size();
	if (dst->mapsUsed <= dst->mapsCap) {
		CK(copy_peer(dst->dMaps + *off, dst->device, src->dMaps + t.off, src->device, sizeof(float) * t.pts.size(), dst->stream));
		return 0;
	}
	CK(cudaStreamSynchronize(dst->stream));
	return upload_maps(dst);
}
// Complex coefficient rows of k_prep (32 B per bin-channel and block: 6.6 GB at batch 1024 x 33 blocks stereo): only calls
// with a stream that has a frequency map or formant processing launch k_prep, so only they pay for them (b200s_reserve()
// allocates them when the parameters set at that time need them).
static int ensure_coef(b200s_engine *e) {
	if (e->coefFrames == e->maxFrames && e->dPI) return 0;
	const Cfg &g = e->cfg;
	CK(cudaStreamSynchronize(e->stream));
	const size_t n = (size_t)g.S * e->maxFrames * g.C * g.K;
	int rc;
	if ((rc = dalloc(e, &e->dPI, n))) return rc;
	if ((rc = dalloc(e, &e->dFT, n))) return rc;
	if ((rc = dalloc(e, &e->dT1, n))) return rc;
	if ((rc = dalloc(e, &e->dT2, n))) return rc;
	if ((rc = dalloc(e, &e->dS, n / g.C))) return rc; // smoothed energy / formant envelope rows: one per block (k_passes)
	if ((rc = dalloc(e, &e->dM, n / g.C))) return rc;
	e->coefFrames = e->maxFrames;
	return 0;
}
// rows of the step-major path (mapped / formant calls): map, ratio, smoothed energy, envelope, and the transposed terms
static int ensure_stepmajor(b200s_engine *e) {
	if (e->tFrames == e->maxFrames && e->dTFT) return 0;
	const Cfg &g = e->cfg;
	CK(cudaStreamSynchronize(e->stream));
	const size_t nRow = (size_t)g.S * e->maxFrames * g.K;
	const size_t nT = (size_t)g.S * ((e->maxFrames + 31) / 32) * t_rows(g) * g.C * 32;
	int rc;
	if ((rc = dalloc(e, &e->dMapB, nRow))) return rc;
	if ((rc = dalloc(e, &e->dMapG, nRow))) return rc;
	if ((rc = dalloc(e, &e->dRatio, nRow))) return rc;
	if (!e->dS && (rc = dalloc(e, &e->dS, nRow))) return rc;
	if (!e->dM && (rc = dalloc(e, &e->dM, nRow))) return rc;
	if ((rc = dalloc(e, &e->dTE, nT))) return rc;
	if ((rc = dalloc(e, &e->dTPI, nT))) return rc;
	if ((rc = dalloc(e, &e->dTFT, nT))) return rc;
	if ((rc = dalloc(e, &e->dTT1, nT))) return rc;
	if ((rc = dalloc(e, &e->dTT2, nT))) return rc;
	e->tFrames = e->maxFrames;
	return 0;
}
// the two extra twist rows of blocks with random time factors (calls that may stretch beyond 2x only)
static int ensure_rand(b200s_engine *e) {
	if (e->randFrames == e->maxFrames && e->dT1u) return 0;
	const Cfg &g = e->cfg;
	CK(cudaStreamSynchronize(e->stream));
	const size_t n = (size_t)g.S * e->maxFrames * g.C * g.K;
	int rc;
	if ((rc = dalloc(e, &e->dT1u, n))) return rc;
	if ((rc = dalloc(e, &e->dT2u, n))) return rc;
	e->randFrames = e->maxFrames;
	return 0;
}
static int ensure_buf(b200s_engine *e, float **p, size_t *cap, size_t n, bool zero) {
	if (n <= *cap && *p) return 0;
	CK(cudaStreamSynchronize(e->stream));
	int rc;
	if ((rc = dalloc(e, p, n))) return rc;
	*cap = n;
	if (zero) CK(cudaMemset(*p, 0, sizeof(float) * std::max<size_t>(n, 1)));
	return 0;
}

// process() on device buffers with explicit strides (floats between channels / streams)
// hIn / hOut (host-buffer API only): packed [S][C][n] host arrays mirrored by dIn / dOut; each stream group
// then copies its own slab in, runs its kernels and copies its slab out on its own CUDA stream, so that the
// PCIe transfers of one group overlap the kernels of the others.
// desc (b200s_run_per_stream, resolved by run_impl): the host copy of the call's S descriptors; the streams whose
// CallDesc::pass is `pass` take part, stream s reading desc[s].nIn samples of each row and writing desc[s].nOut, then zeros
// up to outTail; every other stream is absent from the pass (but for zeros up to outTail in its row).  nIn / nOut are then
// the rows' strides.  descSlot >= 0: the stream groups upload their slices of the table from pinDesc[descSlot]; -1: the
// caller has uploaded the whole table on the main stream.  Without desc every stream reads nIn and writes nOut.
// list (b200s_run_streams, with desc): the call runs over the nList streams list[0..nList), in that order: the rows, the
// descriptors, the grids and the stream groups are over list positions, and every stream not listed is absent.
static int process_impl(b200s_engine *e, const float *dIn, int inChanStride, long long inStreamStride, int nIn,
                        float *dOut, int outChanStride, long long outStreamStride, int nOut,
                        const float *hIn = nullptr, float *hOut = nullptr, const short *hIn16 = nullptr, short *hOut16 = nullptr,
                        const CallDesc *desc = nullptr, int pass = 0, int descSlot = -1, int outTail = 0,
                        const int *list = nullptr, int nList = 0) {
	const Cfg &g = e->cfg;
	if (nIn < 0 || nOut < 0) {
		e->err = "process: negative sample count";
		return B200S_EINVAL;
	}
	const bool perStream = desc != nullptr;
	const int P = list ? nList : g.S; // positions of the call
	// the host's decisions over the streams' counts: the longest output sizes the scratch and the grids; a call may need the
	// random path when ANY stream may stretch beyond 2x; bulk-copy staging needs every input length a multiple of 4
	int maxOut = nOut;
	bool lowRatio = nOut > 0 && (long long)nIn * 2 * g.H < (long long)nOut * (g.H + 4), anyIdle = false, lensAligned = nIn % 4 == 0;
	if (perStream) {
		maxOut = 0;
		lowRatio = false;
		anyIdle = P < g.S; // (the streams a list leaves out are absent)
		for (int i = 0; i < P; ++i) {
			const bool in = desc[i].pass == pass;
			const int li = in ? desc[i].nIn : 0, lo = in ? desc[i].nOut : 0;
			maxOut = std::max(maxOut, lo);
			if (lo > 0) lowRatio = lowRatio || (long long)li * 2 * g.H < (long long)lo * (g.H + 4);
			else anyIdle = true;
			// (an output seek's rows start at its seek window's end: bulk copies need it 16-byte aligned too)
			lensAligned = lensAligned && li % 4 == 0 && (!in || ((uintptr_t)desc[i].in % 16 == 0 && desc[i].inChan % 4 == 0));
		}
	}
	int rc;
	if ((rc = ensure_scratch(e, maxOut))) return rc;
	if (e->sprmDirty) {
		// new per-stream parameters, on the main stream ahead of this call's work.  This call then joins (see `chained`
		// below): a chained call's stream groups do not wait for the main stream, so they could read the new table while
		// the previous call's groups are still running.
		const int k = e->sprmSlot ^= 1;
		CK(cudaEventSynchronize(e->evSprm[k]));
		memcpy(e->pinSprm[k], e->hSprm.data(), sizeof(StreamParams) * e->S);
		CK(cudaMemcpyAsync(e->dSprm, e->pinSprm[k], sizeof(StreamParams) * e->S, cudaMemcpyHostToDevice, e->stream));
		CK(cudaEventRecord(e->evSprm[k], e->stream));
		e->sprmDirty = false;
		e->chainedGroups = 0;
	}
	// Can a block of this call stretch beyond 2x (timeFactor = interval / inputInterval > 2, :312,:639)?  Inside a call the
	// input interval is interval * nIn / nOut give or take a sample; the first block's mixes in the previous call's ratio;
	// after a seek it is 1 / playbackRate.  Conservative on purpose: the decision itself is taken per stream on the device
	// (k_plan sets Call::hasRandom); this only says whether the kernels of the random path have to be launched at all.
	// (Per stream: a stream that produces no output keeps its previous ratio or its seek's time factor for its next block,
	// so while one does, the flags carry over.)
	const bool mayRandom = maxOut > 0 && (lowRatio || e->prevCallMayRandom || e->seekMayRandom);
	if (maxOut > 0) {
		e->prevCallMayRandom = lowRatio || (anyIdle && e->prevCallMayRandom);
		e->seekMayRandom = anyIdle && e->seekMayRandom;
	}
	// Each stream takes the path its own parameters need (k_plan sets Call::mapped); a call launches the kernels of the paths
	// some stream takes, and every kernel skips the streams of the other path.  With the same parameters on every stream
	// this is one of the two uniform launch sequences.
	const bool anyMapped = e->nMapped > 0, anyPlain = e->nMapped < e->S;
	const bool useStepMajor = anyMapped && e->stepMajor; // mapped / formant streams on k_products + k_chain_t
	if (((anyMapped && !useStepMajor) || mayRandom) && (rc = ensure_coef(e))) return rc;
	if (useStepMajor && (rc = ensure_stepmajor(e))) return rc;
	if (mayRandom && (rc = ensure_rand(e))) return rc;
	Ctx x = make_ctx(e);
	if (!mayRandom) x.cT1u = x.cT2u = nullptr; // (stale rows of an earlier call are never read)
	x.randomPathOn = (mayRandom || (anyMapped && !useStepMajor)) ? 1 : 0; // the round-1 mapped path runs k_prep + k_chain for every random stream anyway
	x.in = dIn; x.out = dOut; x.nIn = nIn; x.nOut = nOut;
	x.inChanStride = inChanStride; x.inStreamStride = inStreamStride;
	x.outChanStride = outChanStride; x.outStreamStride = outStreamStride;
	x.inAligned = ((uintptr_t)dIn % 16 == 0) && inChanStride % 4 == 0 && inStreamStride % 4 == 0 && lensAligned && g.histLen % 4 == 0;
	const int F = frames_bound(g, maxOut);
	if (perStream) {
		x.desc = e->dDesc;
		x.pass = pass;
		x.outTail = outTail;
		x.listed = list ? 1 : 0;
	}
	// Sub-batch pipeline: the streams of the batch are independent, so the launch sequence is issued
	// per sub-batch on its own CUDA stream (descending priority).  Sub-batch 0's chain then runs while
	// sub-batch 1 is still in its FFT kernel, and so on: the latency-bound wavefront kernel and the
	// throughput-bound FFT kernels share the SMs instead of taking turns.  Per-kernel profiling
	// (b200s_profile_begin) runs unsplit on the main stream so that the event pairs time one kernel each.
	const bool hostIO = hIn || hOut || hIn16 || hOut16;
	const int wantSub = hostIO ? e->nHostParts : e->nSub;
	// (host-buffer pipeline: at least two streams per group; device-resident sub-batches: only for large batches)
	const int nSub = (e->profiling || wantSub <= 1 || P < (hostIO ? 2 * wantSub : 64)) ? 1 : std::min(wantSub, e->maxSub);
	// Consecutive host-buffer calls over the SAME stream groups need no join between them: every group's copies and
	// kernels are ordered on the group's own stream and touch only that group's streams of the state, so group g of
	// call n+1 may start its H2D copy while other groups still finish call n (b200s_process_async pipelines calls this
	// way).  Anything else first joins: the main stream has waited for every group at the end of the previous call.
	// The groups' slabs of the shared staging buffers sit at sBase*C*nIn / sBase*C*nOut, so they only coincide from call to
	// call when the sample counts (the strides of a per-stream call; its streams' own counts may differ) do: a call with
	// different counts must first join (otherwise group g's copy of call n+1
	// could overwrite the slab a neighbouring group still uses for call n); evBegin below is that join, since the main
	// stream has waited for every group's evSubDone at the end of the previous call.  A listed call's groups own the streams
	// at their list positions, so it only chains onto a call over the same list, the same streams in the same order
	// (otherwise a stream could move to another group and run beside itself).
	const bool sameStreams = list ? e->chainedListed && (int)e->chainedList.size() == P && std::equal(list, list + P, e->chainedList.begin())
	                              : !e->chainedListed;
	const bool chained = hostIO && nSub > 1 && e->chainedGroups == nSub && e->chainedIn == nIn && e->chainedOut == nOut && sameStreams;
	e->chainedGroups = (hostIO && nSub > 1) ? nSub : 0;
	e->chainedIn = nIn;
	e->chainedOut = nOut;
	e->chainedListed = list != nullptr;
	if (list) e->chainedList.assign(list, list + P);
	if (nSub > 1 && !chained) CK(cudaEventRecord(e->evBegin, e->stream));
	const int chainV = chain_version(g, e->chainV, e->fftV1);
	const bool pairFft = use_pair_fft(g, e->fftV1);
	x.specIl = (anyPlain && chainV >= 3) ? 1 : 0; // (interleaved rows for the plain streams only, spec_il)
	for (int sub = 0; sub < nSub; ++sub) {
		cudaStream_t st = nSub > 1 ? e->subStream[sub] : e->stream;
		if (nSub > 1 && !chained) CK(cudaStreamWaitEvent(st, e->evBegin, 0));
		x.sBase = (int)((long long)P * sub / nSub);
		x.sCount = (int)((long long)P * (sub + 1) / nSub) - x.sBase;
		if (perStream && descSlot >= 0) { // the group's slice of the table, ordered before its k_plan and after its previous call's kernels
			CK(cudaMemcpyAsync(e->dDesc + x.sBase, e->pinDesc[descSlot] + x.sBase, sizeof(CallDesc) * x.sCount, cudaMemcpyHostToDevice, st));
			CK(cudaEventRecord(e->evDesc[descSlot][sub], st));
		}
		if (hIn && nIn > 0)
			CK(cudaMemcpyAsync((float *)dIn + (size_t)x.sBase * g.C * nIn, hIn + (size_t)x.sBase * g.C * nIn, sizeof(float) * (size_t)x.sCount * g.C * nIn, cudaMemcpyHostToDevice, st));
		if (hIn16 && nIn > 0) { // 16-bit PCM: 2 bytes per sample over PCIe, converted on the device
			const size_t off = (size_t)x.sBase * g.C * nIn, cnt = (size_t)x.sCount * g.C * nIn;
			CK(cudaMemcpyAsync(e->dIn16 + off, hIn16 + off, sizeof(short) * cnt, cudaMemcpyHostToDevice, st));
			B200S_LAUNCH(k_pcm16_in, dim3((unsigned)std::min<size_t>((cnt + 1023) / 1024, 4096)), dim3(256), 0, st, e->dIn16 + off, (float *)dIn + off, cnt);
			CKL();
		}
		{ // (profiling implies nSub == 1, i.e. st == e->stream, which is where PROF() records its events)
			PROF(PK_PLAN, B200S_LAUNCH(k_plan, dim3(x.sCount), dim3(kThreads), 0, st, x));
			if (F > 0) {
				if (pairFft) { // persistent CTAs, two per SM, over the (stream, job pair) items
					const long long items = (long long)x.sCount * g.C * x.maxFrames;
					const int grid = (int)std::min<long long>(items, 2LL * e->numSMs);
					PROF(PK_ANALYSE, B200S_LAUNCH(analyse2_kernel(g, (x.specIl && anyMapped) || x.listed), dim3(grid), dim3(256), smem_analyse2(g), st, x));
				} else {
					ChainKernel ka = analyse_kernel(g);
					PROF(PK_ANALYSE, B200S_LAUNCH(ka, dim3(std::min(2 * F * g.C, ANALYSE_CTAS_PER_STREAM), 1, x.sCount), dim3(kThreads), smem_analyse(g), st, x));
				}
				// Pure time-stretch (no frequency map, no formants): the chain forms its terms directly from
				// the spectra and k_prep is skipped; otherwise k_prep produces the coefficient arrays.
				// formants with setFormantBase(0): the automatic pitch estimate of every block (serial over blocks) first
				if (e->anyAutoPitch) {
					B200S_LAUNCH(k_pitch, dim3(x.sCount), dim3(kThreads), sizeof(float) * g.K, st, x);
					CKL();
				}
				if (anyMapped) {
					int _rc;
					if ((_rc = prof_mark(e, PK_PREP, true))) return _rc;
					// the serial one-pole passes over the bins, one lane per block (kernels.cuh), then the per-bin products
					B200S_LAUNCH(k_energy, dim3(F, x.sCount), dim3(kThreads), 0, st, x);
					CKL();
					B200S_LAUNCH(k_passes, dim3(x.sCount), dim3(32), 0, st, x);
					CKL();
					if (useStepMajor) { // peaks / map / ratio rows, then the per-bin terms in step-major order (chain_t.cuh)
						x.mapOnly = 1;
						B200S_LAUNCH(k_prep, dim3(F, x.sCount), dim3(kThreads), smem_prep(g, e->anyFormants), st, x);
						CKL();
						x.mapOnly = 0;
						B200S_LAUNCH(k_products, dim3(x.tRows / 32, x.tGroups, x.sCount), dim3(256), 0, st, x);
						CKL();
						if (mayRandom) { // streams with a random block (plain or mapped): the full k_prep (random-only mode), consumed by k_chain below
							x.randomOnly = 1;
							B200S_LAUNCH(k_prep, dim3(F, x.sCount), dim3(kThreads), smem_prep(g, e->anyFormants), st, x);
							CKL();
							x.randomOnly = 0;
						}
					} else {
						B200S_LAUNCH(k_prep, dim3(F, x.sCount), dim3(kThreads), smem_prep(g, e->anyFormants), st, x);
						CKL();
					}
					if ((_rc = prof_mark(e, PK_PREP, false))) return _rc;
				}
				// the mapped / formant streams (k_chain_t, or the round-1 k_chain), then the plain streams (a direct chain); in a
				// mixed call each of these kernels exits at once for the other path's streams
				if (useStepMajor) {
					int _rc;
					if ((_rc = prof_mark(e, PK_CHAIN, true))) return _rc;
					ChainKernel kt = chain_t_kernel(g);
					B200S_LAUNCH(kt, dim3(x.sCount), dim3(32), 0, st, x);
					CKL();
					if (mayRandom) { // the streams k_chain_t and the direct chains leave (Call::hasRandom), plain or mapped
						x.randomOnly = 1;
						dim3 grid((x.sCount + kChainWarps - 1) / kChainWarps), block(32 * kChainWarps);
						ChainKernel kc = chain_kernel(g, false);
						B200S_LAUNCH(kc, grid, block, smem_chain(g, false, true), st, x);
						CKL();
						x.randomOnly = 0;
					}
					if ((_rc = prof_mark(e, PK_CHAIN, false))) return _rc;
				} else if (anyMapped) { // round-1 kernels: the mapped streams and every stream with a random block
					dim3 grid((x.sCount + kChainWarps - 1) / kChainWarps), block(32 * kChainWarps);
					ChainKernel kc = chain_kernel(g, false);
					PROF(PK_CHAIN, B200S_LAUNCH(kc, grid, block, smem_chain(g, false, mayRandom), st, x));
				}
				if (!anyPlain) {
#ifdef B200S_KEEP_OLD_KERNELS
				} else if (chainV == 5) {
					int _rc;
					if ((_rc = prof_mark(e, PK_CHAIN, true))) return _rc;
					const bool fast = !e->exactMath;
					ChainKernel kw = fast ? chain_ws_kernel<true>(g.L) : chain_ws_kernel<false>(g.L), k4 = chain3_kernel(g, 4, fast);
					B200S_LAUNCH(kw, dim3(x.sCount), dim3(64), fast ? smem_chain_ws<true>() : smem_chain_ws<false>(), st, x);
					CKL();
					x.wsRan = 1; // streams with a block beyond the 2x stretch limit: k_chain_direct4 (every other CTA exits at once)
					B200S_LAUNCH(k4, dim3(x.sCount), dim3(32), smem_chain4(g.L), st, x);
					CKL();
					x.wsRan = 0;
					if ((_rc = prof_mark(e, PK_CHAIN, false))) return _rc;
#endif
				} else if (chainV >= 3) {
					PROF(PK_CHAIN, B200S_LAUNCH(chain3_kernel(g, chainV, !e->exactMath), dim3(x.sCount), dim3(32), chainV >= 6 ? smem_chain6() : chainV == 4 ? smem_chain4(g.L) : sizeof(Chain3Tiles), st, x));
				} else if (chainV == 2) {
					const int W = chain2_warps(g, maxOut);
					ChainKernel kc = chain2_kernel(g, g.C == 1 && !e->exactMath);
					int _rc;
					if ((_rc = prof_mark(e, PK_CHAIN, true))) return _rc;
					if (g.C == 1 && (e->dual < 0 ? dual_enabled() : e->dual != 0)) { // mono: two streams per warp on the packed wavefront
						ChainKernel kd = e->exactMath ? chain6_kernel<false, true>(g.L) : chain6_kernel<true, true>(g.L);
						B200S_LAUNCH(kd, dim3((x.sCount + 1) / 2), dim3(32), smem_chain6(), st, x);
					} else {
						B200S_LAUNCH(kc, dim3(x.sCount), dim3(32 * W), smem_chain2(g.C, W), st, x);
					}
					CKL();
					if ((_rc = prof_mark(e, PK_CHAIN, false))) return _rc;
				} else { // (first-generation direct chain, -DB200S_KEEP_OLD_KERNELS builds only)
					dim3 grid((x.sCount + kChainWarps - 1) / kChainWarps), block(32 * kChainWarps);
					ChainKernel kc = chain_kernel(g, true);
					PROF(PK_CHAIN, B200S_LAUNCH(kc, grid, block, smem_chain(g, true, mayRandom), st, x));
				}
			}
			if (F > 0 && !anyMapped && mayRandom) {
				// streams with a block beyond 2x stretch (Call::hasRandom): the direct chain kernels above returned at once for
				// them; k_prep forms their coefficient rows with the per-bin random time factors and the generic chain runs
				// them.  Every other CTA of these two launches exits immediately.  (Calls with mapped streams have run these
				// streams on the mapped path's random-only launches above.)
				x.randomOnly = 1;
				B200S_LAUNCH(k_prep, dim3(F, x.sCount), dim3(kThreads), smem_prep(g, false), st, x);
				CKL();
				dim3 grid((x.sCount + kChainWarps - 1) / kChainWarps), block(32 * kChainWarps);
				ChainKernel kc = chain_kernel(g, false);
				B200S_LAUNCH(kc, grid, block, smem_chain(g, false, true), st, x);
				CKL();
				x.randomOnly = 0;
			}
			// fork: the commit of this call runs beside the synthesis (both only read what the chain wrote)
			const bool forkCommit = nSub == 1 && !e->profiling && e->commitStream;
			cudaStream_t cst = forkCommit ? e->commitStream : st;
			if (forkCommit) {
				CK(cudaEventRecord(e->evFork, st));
				CK(cudaStreamWaitEvent(cst, e->evFork, 0));
			}
			if (pairFft) {
				PROF(PK_SYNTH, B200S_LAUNCH(synth2_kernel(g), dim3(g.C, x.sCount), dim3(256), smem_synth2(g), st, x));
			} else {
				ChainKernel ks = synth_kernel(g);
				PROF(PK_SYNTH, B200S_LAUNCH(ks, dim3(g.C, x.sCount), dim3(kThreads), smem_synth(g), st, x));
			}
			PROF(PK_COMMIT, B200S_LAUNCH(k_commit, dim3(g.C, x.sCount), dim3(kThreads), 0, cst, x));
			if (forkCommit) {
				CK(cudaEventRecord(e->evJoin, cst));
				CK(cudaStreamWaitEvent(st, e->evJoin, 0));
			}
		}
		if (hOut && nOut > 0)
			CK(cudaMemcpyAsync(hOut + (size_t)x.sBase * g.C * nOut, dOut + (size_t)x.sBase * g.C * nOut, sizeof(float) * (size_t)x.sCount * g.C * nOut, cudaMemcpyDeviceToHost, st));
		if (hOut16 && nOut > 0) {
			const size_t off = (size_t)x.sBase * g.C * nOut, cnt = (size_t)x.sCount * g.C * nOut;
			B200S_LAUNCH(k_pcm16_out, dim3((unsigned)std::min<size_t>((cnt + 1023) / 1024, 4096)), dim3(256), 0, st, dOut + off, e->dOut16 + off, cnt);
			CKL();
			CK(cudaMemcpyAsync(hOut16 + off, e->dOut16 + off, sizeof(short) * cnt, cudaMemcpyDeviceToHost, st));
		}
		if (nSub > 1) {
			CK(cudaEventRecord(e->evSubDone[sub], st));
			CK(cudaStreamWaitEvent(e->stream, e->evSubDone[sub], 0));
		}
	}
	if (!list) e->histCur ^= 1; // (a listed call's k_commit copies the new history back into histCur)
	return 0;
}

static float seek_time_factor(const Cfg &g, double playbackRate) { return (playbackRate * g.H > 1) ? float(1 / playbackRate) : float(g.H); } // :164
static int seek_impl(b200s_engine *e, const float *dIn, int chanStride, long long streamStride, int n, double playbackRate, const double *rates = nullptr,
                     const long long *bankEnds = nullptr, long long bankLen = 0) {
	const Cfg &g = e->cfg;
	e->chainedGroups = 0;
	Ctx x = make_ctx(e);
	x.in = dIn; x.nIn = n; x.inChanStride = chanStride; x.inStreamStride = streamStride;
	if (bankEnds) { // the windows are cut out of a device-resident audio bank by k_seek itself
		int rc;
		if (!e->dSeekEnd && (rc = dalloc(e, &e->dSeekEnd, (size_t)g.S))) return rc;
		CK(cudaMemcpyAsync(e->dSeekEnd, bankEnds, sizeof(long long) * g.S, cudaMemcpyHostToDevice, e->stream));
		x.seekEnd = e->dSeekEnd;
		x.bankLen = bankLen;
	}
	float stf = seek_time_factor(g, playbackRate);
	e->seekMayRandom = stf > 1.9f; // the next block takes this as its time factor (:312)
	if (rates) { // one playback rate per stream (a server whose streams follow their own time maps)
		int rc;
		if (!e->dSeekStf && (rc = dalloc(e, &e->dSeekStf, (size_t)g.S))) return rc;
		e->hSeekStf.resize(g.S);
		e->seekMayRandom = false;
		for (int s = 0; s < g.S; ++s) {
			e->hSeekStf[s] = seek_time_factor(g, rates[s]);
			if (e->hSeekStf[s] > 1.9f) e->seekMayRandom = true;
		}
		CK(cudaMemcpyAsync(e->dSeekStf, e->hSeekStf.data(), sizeof(float) * g.S, cudaMemcpyHostToDevice, e->stream));
		x.seekStf = e->dSeekStf;
	}
	B200S_LAUNCH(k_seek, dim3(g.S), dim3(kThreads), 0, e->stream, x, stf);
	CKL();
	return 0;
}

static int flush_impl(b200s_engine *e, float *dOut, int outChanStride, long long outStreamStride, int nOut, float playbackRate) {
	const Cfg &g = e->cfg;
	e->chainedGroups = 0;
	int rc;
	int outputBlock = std::max(0, nOut - g.H); // :439
	if (outputBlock > 0) {
		int nIn = int(outputBlock * playbackRate); // :440
		if (nIn < 0) nIn = 0;
		size_t zn = (size_t)g.S * g.C * std::max(nIn, 1);
		if ((rc = ensure_buf(e, &e->dZero, &e->zeroCap, zn, true))) return rc;
		if ((rc = process_impl(e, e->dZero, nIn, (long long)g.C * nIn, nIn, dOut, outChanStride, outStreamStride, outputBlock))) return rc;
	}
	int tail = nOut - outputBlock;
	Ctx x = make_ctx(e);
	x.out = dOut; x.outChanStride = outChanStride; x.outStreamStride = outStreamStride;
	if (tail > 0) {
		B200S_LAUNCH(k_flush_tail, dim3(g.C, g.S), dim3(kThreads), sizeof(float) * g.B, e->stream, x, outputBlock, tail);
		CKL();
	}
	return reset_impl(e, false); // stft.reset(0.1); prevInput = output = 0 (:456-463)
}

static int output_seek_impl(b200s_engine *e, const float *dIn, int chanStride, long long streamStride, int inputLength) {
	const Cfg &g = e->cfg;
	int rc;
	if ((rc = reset_impl(e, true))) return rc; // :175
	const int inLat = g.B - g.B / 2, outLat = g.B / 2 + (g.split ? g.H : 0);
	int surplus = std::max(inputLength - inLat, 0);            // :177
	float playbackRate = surplus / float(outLat);              // :178
	int seekSamples = inputLength - surplus;                   // :181
	if ((rc = seek_impl(e, dIn, chanStride, streamStride, seekSamples, playbackRate))) return rc;
	size_t tn = (size_t)g.S * g.C * outLat;
	if ((rc = ensure_buf(e, &e->dTmp, &e->tmpCap, tn, false))) return rc;
	if ((rc = process_impl(e, dIn + seekSamples, chanStride, streamStride, surplus, e->dTmp, outLat, (long long)g.C * outLat, outLat))) return rc; // :196
	Ctx x = make_ctx(e);
	B200S_LAUNCH(k_add_output, dim3(g.C, g.S), dim3(kThreads), 0, e->stream, x, (const float *)e->dTmp, outLat); // :199-203
	CKL();
	return 0;
}

static int stage_in(b200s_engine *e, const float *in, int n) {
	size_t cnt = (size_t)e->cfg.S * e->cfg.C * std::max(n, 1);
	int rc;
	if ((rc = ensure_buf(e, &e->dIn, &e->inCap, cnt, false))) return rc;
	if (n > 0 && in) CK(cudaMemcpyAsync(e->dIn, in, sizeof(float) * (size_t)e->cfg.S * e->cfg.C * n, cudaMemcpyHostToDevice, e->stream));
	return 0;
}
static int stage_out(b200s_engine *e, int n) {
	size_t cnt = (size_t)e->cfg.S * e->cfg.C * std::max(n, 1);
	return ensure_buf(e, &e->dOut, &e->outCap, cnt, false);
}
// the 16-bit PCM slabs, ci / co samples; growing one first drains the handle's stream (copies may still use the old one)
static int stage_pcm16(b200s_engine *e, size_t ci, size_t co) {
	if (ci <= e->in16Cap && co <= e->out16Cap) return 0;
	CK(cudaStreamSynchronize(e->stream));
	int rc;
	if (ci > e->in16Cap) {
		if ((rc = dalloc(e, &e->dIn16, ci))) return rc;
		e->in16Cap = ci;
	}
	if (co > e->out16Cap) {
		if ((rc = dalloc(e, &e->dOut16, co))) return rc;
		e->out16Cap = co;
	}
	return 0;
}
static int fetch_out(b200s_engine *e, float *out, int n) {
	if (n > 0) CK(cudaMemcpyAsync(out, e->dOut, sizeof(float) * (size_t)e->cfg.S * e->cfg.C * n, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}

// b200s_run_per_stream (arguments validated by check_run): every stream runs its own op, in three phases (DESIGN.md §3.11).
//   pre:     RESET / OUTPUT_SEEK: the full reset (:175), then SEEK / OUTPUT_SEEK: k_seek with the stream's window and factor
//   process: ONE process_impl pass over the PROCESS, OUTPUT_SEEK (:196) and FLUSH (:440-441) streams, each on its own rows
//            (CallDesc::in / out, resolved into Call by k_plan): a FLUSH stream reads the engine's zero row, an OUTPUT_SEEK
//            stream its caller rows after the seek window and writes its pre-roll into dTmp [S][C][outputLatency]
//   post:    FLUSH: k_flush_tail and the flush's reset (:442-463); OUTPUT_SEEK: k_add_output from dTmp (:198-203)
// Every other stream is absent from the pass (k_plan), so its state is untouched and k_commit copies its history
// unchanged into the other buffer.  A phase that no stream needs is not launched.  Host buffers: a call of PROCESS / SKIP
// ops with some PROCESS pipelines its stream groups as b200s_process_async does; any other call copies the input slab in
// on the main stream, runs on the device and copies the output slab back.
// list (b200s_run_streams): the call runs over the n streams list[0..n) instead of the batch.  The arrays, the rows and the
// descriptor table are over list positions i (stream list[i]), and so are the grids of every phase; the streams not listed
// are not part of the call at all.
// in16 / out16 (the _pcm16 calls, host buffers, `in` / `out` NULL): 16-bit PCM rows [positions][C][stride], copied through
// the dIn16 / dOut16 slabs and converted to and from the float rows of dIn / dOut on the device.  A joining call converts
// its input ahead of the pre phase and its output after the post phase and k_copy_rows (the output seeks' pre-roll and the
// flushes' tails are only final then); a chained call converts per stream group in process_impl.
static int run_impl(b200s_engine *e, const int *ops, const float *in, int inStride, const int *nIn, float *out, int outStride,
                    const int *nOut, const double *rates, bool host, bool wait, const int *list = nullptr, int n = 0,
                    const short *in16 = nullptr, short *out16 = nullptr) {
	const Cfg &g = e->cfg;
	const long long C = g.C;
	const int inLat = g.B - g.B / 2, outLat = g.B / 2 + (g.split ? g.H : 0);
	const int P = list ? n : g.S; // positions of the call
	int opsUsed = 0, zeroLen = 0;
	for (int i = 0; i < P; ++i) {
		opsUsed |= B200S_OPBIT(ops[i]);
		if (ops[i] == B200S_OP_FLUSH) {
			const int outputBlock = std::max(0, nOut[i] - g.H); // :439
			zeroLen = std::max(zeroLen, std::max(0, int(outputBlock * (rates ? float(rates[i]) : 0.f)))); // :440
		}
	}
	const int preOps = B200S_OPBIT(B200S_OP_RESET) | B200S_OPBIT(B200S_OP_SEEK) | B200S_OPBIT(B200S_OP_OUTPUT_SEEK);
	const int postOps = B200S_OPBIT(B200S_OP_FLUSH) | B200S_OPBIT(B200S_OP_OUTPUT_SEEK);
	const bool phases = (opsUsed & (preOps | postOps)) != 0;
	int rc;
	// buffers first (growing one synchronises and may move it): the descriptors below hold their addresses
	if (host) {
		if ((size_t)C * g.S * std::max(inStride, 1) > e->inCap || (size_t)C * g.S * std::max(outStride, 1) > e->outCap || !e->dIn || !e->dOut) {
			// growing the staging buffers would invalidate copies still in flight: drain first
			CK(cudaStreamSynchronize(e->stream));
		}
		if ((rc = stage_in(e, nullptr, inStride))) return rc; // capacity only
		if ((rc = stage_out(e, outStride))) return rc;
		if ((in16 || out16) && (rc = stage_pcm16(e, (size_t)P * C * std::max(inStride, 1), (size_t)P * C * std::max(outStride, 1)))) return rc;
	}
	// (sized by b200s_reserve: no allocation then)
	if ((opsUsed & B200S_OPBIT(B200S_OP_FLUSH)) && (rc = ensure_buf(e, &e->dZero, &e->zeroCap, (size_t)std::max(zeroLen, 1), true))) return rc;
	// An output seek writes outputLatency samples of pre-roll into its output rows, which k_add_output reads back and then
	// zeroes.  Rows narrower than that: the pass writes into dTmp [positions][C][outputLatency], copied back to the caller's rows.
	const int W = (opsUsed & B200S_OPBIT(B200S_OP_OUTPUT_SEEK)) ? std::max(outStride, outLat) : outStride;
	if (W > outStride && (rc = ensure_buf(e, &e->dTmp, &e->tmpCap, (size_t)P * C * W, false))) return rc;
	const float *dIn = host ? e->dIn : in;
	float *dOut = host ? e->dOut : out, *pOut = W > outStride ? e->dTmp : dOut;
	const int lk = e->descSlot ^= 1;
	for (int i = 0; i < b200s_engine::kMaxSub; ++i) CK(cudaEventSynchronize(e->evDesc[lk][i]));
	CallDesc *d = e->pinDesc[lk];
	bool anyPass = false, seekSlow = false;
	for (int s = 0; s < P; ++s) { // (s: the position)
		CallDesc c;
		memset(&c, 0, sizeof(c));
		c.op = ops[s];
		c.slot = list ? list[s] : s;
		c.in = dIn + (size_t)s * C * inStride;
		c.inChan = inStride;
		switch (c.op) {
		case B200S_OP_PROCESS:
			c.pass = 1;
			c.nIn = nIn[s];
			c.nOut = nOut[s];
			break;
		case B200S_OP_SEEK:
			c.seekN = nIn[s];
			c.stf = seek_time_factor(g, rates[s]);
			break;
		case B200S_OP_OUTPUT_SEEK: {
			const int surplus = std::max(nIn[s] - inLat, 0); // :177
			const float rate = surplus / float(outLat);      // :178
			c.seekN = nIn[s] - surplus;                      // :181
			c.stf = seek_time_factor(g, rate);
			c.pass = 1;
			c.nIn = surplus;
			c.nOut = outLat;
			c.in += c.seekN;
			break;
		}
		case B200S_OP_FLUSH: {
			const float rate = rates ? float(rates[s]) : 0.f;
			const int outputBlock = std::max(0, nOut[s] - g.H); // :439
			if (outputBlock > 0) {
				c.pass = 1;
				c.nIn = std::max(0, int(outputBlock * rate)); // :440
				c.nOut = outputBlock;
				c.in = e->dZero;
				c.inChan = 0;
			}
			c.at = outputBlock;
			c.tail = nOut[s] - outputBlock;
			break;
		}
		default: break; // RESET, SKIP
		}
		anyPass = anyPass || c.pass;
		seekSlow = seekSlow || c.stf > 1.9f;
		d[s] = c;
	}
	if (host && !phases && anyPass) { // the stream groups copy their own slabs in and out
		if ((rc = process_impl(e, dIn, inStride, C * inStride, inStride, dOut, outStride, C * outStride, outStride, in, out, in16, out16, d, 1, lk, outStride, list, n))) return rc;
		if (wait) CK(cudaStreamSynchronize(e->stream));
		return 0;
	}
	if (host) {
		e->chainedGroups = 0;
		if (in && inStride > 0) CK(cudaMemcpyAsync(e->dIn, in, sizeof(float) * (size_t)P * C * inStride, cudaMemcpyHostToDevice, e->stream));
		if (in16 && inStride > 0) { // (before the pre phase: k_seek reads the seeks' rows)
			const size_t cnt = (size_t)P * C * inStride;
			CK(cudaMemcpyAsync(e->dIn16, in16, sizeof(short) * cnt, cudaMemcpyHostToDevice, e->stream));
			B200S_LAUNCH(k_pcm16_in, dim3((unsigned)std::min<size_t>((cnt + 1023) / 1024, 4096)), dim3(256), 0, e->stream, (const short *)e->dIn16, e->dIn, cnt);
			CKL();
		}
	}
	if (phases) { // the whole table on the main stream, ahead of the pre phase (the call joins)
		e->chainedGroups = 0;
		CK(cudaMemcpyAsync(e->dDesc, d, sizeof(CallDesc) * P, cudaMemcpyHostToDevice, e->stream));
		CK(cudaEventRecord(e->evDesc[lk][0], e->stream));
	}
	Ctx x = make_ctx(e);
	x.desc = e->dDesc;
	x.listed = list ? 1 : 0;
	x.in = dIn; x.inChanStride = inStride; x.inStreamStride = C * inStride;
	if (opsUsed & preOps) {
		if (opsUsed & (B200S_OPBIT(B200S_OP_RESET) | B200S_OPBIT(B200S_OP_OUTPUT_SEEK))) {
			x.opMask = B200S_OPBIT(B200S_OP_RESET) | B200S_OPBIT(B200S_OP_OUTPUT_SEEK);
			PROF(PK_PHASE, B200S_LAUNCH(k_reset_stft, dim3(P), dim3(kThreads), 0, e->stream, x));
			PROF(PK_PHASE, B200S_LAUNCH(k_reset_bands, dim3(P), dim3(kThreads), 0, e->stream, x, 15));
		}
		if (opsUsed & (B200S_OPBIT(B200S_OP_SEEK) | B200S_OPBIT(B200S_OP_OUTPUT_SEEK))) {
			x.opMask = B200S_OPBIT(B200S_OP_SEEK) | B200S_OPBIT(B200S_OP_OUTPUT_SEEK);
			PROF(PK_PHASE, B200S_LAUNCH(k_seek, dim3(P), dim3(kThreads), 0, e->stream, x, 0.f));
			e->seekMayRandom = e->seekMayRandom || seekSlow; // (other streams may still carry an earlier seek's factor)
		}
	}
	if (anyPass) {
		if ((rc = process_impl(e, dIn, inStride, C * inStride, inStride, pOut, W, C * W, W, nullptr, nullptr, nullptr, nullptr, d, 1, phases ? -1 : lk, W, list, n))) return rc;
	} else if (W > 0) { // no process pass: every row is zero but for the flushes' tails (post phase)
		const size_t cnt = (size_t)P * C * W;
		PROF(PK_PHASE, B200S_LAUNCH(k_zero, dim3((unsigned)std::min<size_t>((cnt + 1023) / 1024, 4096)), dim3(256), 0, e->stream, pOut, cnt));
	}
	if (opsUsed & postOps) {
		Ctx y = make_ctx(e); // (after the pass: the history buffer it left current)
		y.desc = e->dDesc;
		y.listed = x.listed;
		y.out = pOut; y.outChanStride = W; y.outStreamStride = C * W;
		y.outTail = W;
		if (opsUsed & B200S_OPBIT(B200S_OP_FLUSH)) {
			y.opMask = B200S_OPBIT(B200S_OP_FLUSH);
			PROF(PK_PHASE, B200S_LAUNCH(k_flush_tail, dim3(g.C, P), dim3(kThreads), sizeof(float) * g.B, e->stream, y, 0, 0));
			PROF(PK_PHASE, B200S_LAUNCH(k_reset_stft, dim3(P), dim3(kThreads), 0, e->stream, y));
			PROF(PK_PHASE, B200S_LAUNCH(k_reset_bands, dim3(P), dim3(kThreads), 0, e->stream, y, 6));
		}
		if (opsUsed & B200S_OPBIT(B200S_OP_OUTPUT_SEEK)) {
			y.opMask = B200S_OPBIT(B200S_OP_OUTPUT_SEEK);
			PROF(PK_PHASE, B200S_LAUNCH(k_add_output, dim3(g.C, P), dim3(kThreads), 0, e->stream, y, (const float *)nullptr, outLat));
		}
	}
	if (pOut != dOut && outStride > 0)
		PROF(PK_PHASE, B200S_LAUNCH(k_copy_rows, dim3((unsigned)std::min<long long>((long long)P * C, 65535)), dim3(256), 0, e->stream, dOut, outStride, (const float *)pOut, W, outStride, (int)(P * C)));
	if (host && out && outStride > 0) CK(cudaMemcpyAsync(out, e->dOut, sizeof(float) * (size_t)P * C * outStride, cudaMemcpyDeviceToHost, e->stream));
	if (host && out16 && outStride > 0) { // (after the post phase and k_copy_rows: the rows are final only now)
		const size_t cnt = (size_t)P * C * outStride;
		B200S_LAUNCH(k_pcm16_out, dim3((unsigned)std::min<size_t>((cnt + 1023) / 1024, 4096)), dim3(256), 0, e->stream, (const float *)e->dOut, e->dOut16, cnt);
		CKL();
		CK(cudaMemcpyAsync(out16, e->dOut16, sizeof(short) * cnt, cudaMemcpyDeviceToHost, e->stream));
	}
	if (wait) CK(cudaStreamSynchronize(e->stream));
	return 0;
}

// =================================================================================================
// Stream state records (b200s_copy_streams / _export_streams / _import_streams / _clone, DESIGN.md §3.12)
// =================================================================================================
// The host-written head of a record: what import checks before anything is enqueued, and the host-held part of the
// stream (its parameters and the engine-wide random-path flags it carries).  Native byte order.
struct StreamRecordHeader {
	char magic[8];     // "B200SREC"
	uint32_t version;  // kRecordVersion
	uint32_t bytes;    // record size
	int32_t C, B, H, split, K;
	uint32_t flags;    // kRecPrevRandom | kRecSeekRandom | (kRecUsesTable or kRecOwnTable)
	int32_t mapN;      // the frequency-map table the stream uses (kRecUsesTable, kRecOwnTable): its points and fingerprint
	uint64_t mapHash;
	StreamSettings params;
};
static_assert(sizeof(StreamRecordHeader) <= B200S_RECORD_HEADER, "record header");
static const uint32_t kRecordVersion = 1;
// kRecUsesTable: the stream uses the engine's table; kRecOwnTable: it has its own
enum { kRecPrevRandom = 1, kRecSeekRandom = 2, kRecUsesTable = 4, kRecOwnTable = 8 };

static StateRegions state_regions(const b200s_engine *e) {
	const Cfg &g = e->cfg;
	const size_t CK = (size_t)g.C * g.K;
	const struct { void *p; size_t bytes; } a[B200S_STATE_REGIONS] = {
		{e->dSched, sizeof(Sched)},
		{e->dRng, sizeof(unsigned)},
		{e->dStPitch, 2 * sizeof(float)},
		{e->dHist[e->histCur], sizeof(float) * g.C * g.histLen},
		{e->dPend, sizeof(float) * g.C * g.pendLen},
		{e->dPendWp, sizeof(float) * g.C * g.pendLen},
		{e->dStIn, sizeof(float2) * CK},
		{e->dStPrev, sizeof(float2) * CK},
		{e->dStOut, sizeof(float2) * CK},
		{e->dStPredE, sizeof(float) * CK},
	};
	StateRegions t;
	unsigned off = B200S_RECORD_HEADER;
	for (int i = 0; i < B200S_STATE_REGIONS; ++i) {
		t.r[i].base = (char *)a[i].p;
		t.r[i].bytes = (unsigned)a[i].bytes;
		t.r[i].off = off;
		off += (unsigned)((a[i].bytes + 15) / 16 * 16);
	}
	t.recBytes = off;
	return t;
}
// the stream uses the engine's table (a stream with its own table is kMapOwn)
static bool uses_table(const b200s_engine *e, const StreamParams &p) { return p.customMap == kMapEngine && e->engMap.n > 0; }
static bool same_table(const b200s_engine *a, const b200s_engine *b) { return same_points(a->engMap, b->engMap); }
static bool same_config(const Cfg &a, const Cfg &b) { return a.C == b.C && a.B == b.B && a.H == b.H && a.split == b.split; }
static std::string cfg_text(const Cfg &g) {
	return std::to_string(g.C) + " channels, block " + std::to_string(g.B) + ", interval " + std::to_string(g.H) + (g.split ? ", split" : "");
}

// a list of n stream indices, checked against [0, S) and (unique) for duplicates; the message names the first bad entry
static bool check_streams(std::string &err, const char *fn, const char *what, const int *streams, int n, int S, bool unique) {
	if (n > 0 && !streams) {
		err = std::string(fn) + ": " + what + " must not be NULL";
		return false;
	}
	std::vector<char> seen(unique ? (size_t)S : 0, 0);
	for (int i = 0; i < n; ++i) {
		const int s = streams[i];
		if (s < 0 || s >= S) {
			err = std::string(fn) + ": " + what + "[" + std::to_string(i) + "] = " + std::to_string(s) + " is outside [0, " + std::to_string(S) + ")";
			return false;
		}
		if (unique && seen[s]++) {
			err = std::string(fn) + ": " + what + "[" + std::to_string(i) + "]: stream " + std::to_string(s) + " is listed twice";
			return false;
		}
	}
	return true;
}

// Staging of copies / export / import for n streams (records only when `records`): grows, never shrinks.  Growing
// synchronises the handle's stream first, which has also waited for every other handle's read of these records.
static int ensure_xfer(b200s_engine *e, int n, bool records) {
	int rc;
	if (n > e->xferCap) {
		CK(cudaStreamSynchronize(e->stream));
		for (int k = 0; k < 2; ++k) {
			host_free(e->pinIdx[k]);
			e->pinIdx[k] = 0;
			if (!host_alloc((void **)&e->pinIdx[k], sizeof(int) * 2 * (size_t)n)) {
				e->err = "pinned host memory allocation failed";
				return B200S_ECUDA;
			}
		}
		if ((rc = dalloc(e, &e->dXferIdx, 2 * (size_t)n))) return rc;
		e->xferCap = n;
	}
	if (records && n > e->xferRecCap) {
		CK(cudaStreamSynchronize(e->stream));
		if ((rc = dalloc(e, &e->dXfer, (size_t)n * state_regions(e).recBytes))) return rc;
		e->xferRecCap = n;
	}
	return 0;
}
// the stream lists of this handle's next pack (first half of dXferIdx) and / or unpack (second half), on its stream
static int upload_lists(b200s_engine *e, const int *pack, const int *unpack, int n) {
	const int k = e->idxSlot ^= 1;
	CK(cudaEventSynchronize(e->evIdx[k]));
	int *h = e->pinIdx[k];
	if (pack) {
		memcpy(h, pack, sizeof(int) * n);
		CK(cudaMemcpyAsync(e->dXferIdx, h, sizeof(int) * n, cudaMemcpyHostToDevice, e->stream));
	}
	if (unpack) {
		memcpy(h + e->xferCap, unpack, sizeof(int) * n);
		CK(cudaMemcpyAsync(e->dXferIdx + e->xferCap, h + e->xferCap, sizeof(int) * n, cudaMemcpyHostToDevice, e->stream));
	}
	CK(cudaEventRecord(e->evIdx[k], e->stream));
	return 0;
}
static dim3 xfer_grid(const StateRegions &t, int n) {
	const unsigned chunks = (t.recBytes - B200S_RECORD_HEADER) / 16;
	return dim3((chunks + 255) / 256, (unsigned)std::min(n, 65535));
}
static int launch_pack(b200s_engine *e, int n) {
	const StateRegions t = state_regions(e);
	B200S_LAUNCH(k_pack_streams, xfer_grid(t, n), dim3(256), 0, e->stream, t, (const int *)e->dXferIdx, n, e->dXfer);
	CKL();
	return 0;
}
static int launch_unpack(b200s_engine *e, int n, const char *records) {
	const StateRegions t = state_regions(e);
	B200S_LAUNCH(k_unpack_streams, xfer_grid(t, n), dim3(256), 0, e->stream, t, (const int *)e->dXferIdx + e->xferCap, n, records);
	CKL();
	return 0;
}
// restores the caller's current device when a call that works on a handle's (or two handles') devices returns (the
// CPU emulator of the tests has one device and no device query: nothing to restore there)
struct DeviceGuard {
	int prev = -1;
	DeviceGuard() {
#ifndef B200S_EMU
		if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
#endif
	}
	~DeviceGuard() {
		if (prev >= 0) cudaSetDevice(prev);
	}
};
// packed records or a frequency-map table from one engine's device to another's (the same or another device), without peer
// access enabled (the emulator has one device)
static cudaError_t copy_peer(void *dst, int dstDevice, const void *src, int srcDevice, size_t bytes, cudaStream_t st) {
#ifdef B200S_EMU
	(void)dstDevice;
	(void)srcDevice;
	return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
#else
	return cudaMemcpyPeerAsync(dst, dstDevice, src, srcDevice, bytes, st);
#endif
}

// Everything b200s_copy_streams refuses, checked before anything is enqueued; the message goes to both handles
static int check_copy(b200s_engine *dst, const int *dstS, b200s_engine *src, const int *srcS, int n) {
	const char *fn = "b200s_copy_streams";
	std::string err;
	if (n < 0) err = std::string(fn) + ": negative stream count";
	else if (!src->configured || !dst->configured) err = std::string(fn) + ": " + (src->configured ? "destination" : "source") + " engine not configured";
	else if (!same_config(src->cfg, dst->cfg))
		err = std::string(fn) + ": configurations differ (source " + cfg_text(src->cfg) + "; destination " + cfg_text(dst->cfg) + ")";
	else if (check_streams(err, fn, "src_streams", srcS, n, src->S, false) && check_streams(err, fn, "dst_streams", dstS, n, dst->S, true) && src != dst) {
		const bool tables = same_table(src, dst);
		for (int i = 0; i < n && !tables; ++i)
			if (uses_table(src, src->hSprm[srcS[i]])) {
				err = std::string(fn) + ": src_streams[" + std::to_string(i) + "]: stream " + std::to_string(srcS[i]) +
				      " uses the source's frequency-map table, and the destination's table differs";
				break;
			}
	}
	if (err.empty()) return 0;
	src->err = dst->err = err;
	return B200S_EINVAL;
}
// b200s_copy_streams, arguments checked: one pack on the source's stream, the records across to the destination's device
// when it is another, one unpack on the destination's stream; then the host-held part
static int copy_impl(b200s_engine *dst, const int *dstS, b200s_engine *src, const int *srcS, int n) {
	if (n == 0) return 0;
	DeviceGuard guard;
	const bool same = src == dst, peer = src->device != dst->device;
	int rc;
	{
		b200s_engine *e = src;
		CK(cudaSetDevice(src->device));
		if ((rc = ensure_xfer(src, n, true))) return rc;
		if ((rc = upload_lists(src, srcS, same ? dstS : nullptr, n))) return rc;
		src->chainedGroups = 0; // (a chained host-buffer call's stream groups would not wait for the pack)
		if ((rc = launch_pack(src, n))) return rc;
		if (!same) CK(cudaEventRecord(src->evXfer, src->stream));
	}
	// parameters through the host table (read before any is written: swaps and forks), uploaded by the next call.  Within
	// one engine a stream keeps its table descriptor; across engines it points into the destination's pool.
	std::vector<StreamParams> p((size_t)n);
	for (int i = 0; i < n; ++i) p[i] = src->hSprm[srcS[i]];
	if (same) {
		if ((rc = launch_unpack(dst, n, dst->dXfer))) return rc;
	} else {
		b200s_engine *e = dst;
		CK(cudaSetDevice(dst->device));
		if ((rc = ensure_xfer(dst, n, peer))) return rc;
		if ((rc = upload_lists(dst, nullptr, dstS, n))) return rc;
		CK(cudaStreamWaitEvent(dst->stream, src->evXfer, 0));
		const size_t bytes = (size_t)n * state_regions(src).recBytes;
		if (peer) CK(copy_peer(dst->dXfer, dst->device, src->dXfer, src->device, bytes, dst->stream));
		if ((rc = launch_unpack(dst, n, peer ? dst->dXfer : src->dXfer))) return rc;
		for (int i = 0; i < n; ++i) {
			if (p[i].customMap == kMapOwn) {
				if ((rc = carry_table(dst, src, *stream_table(src, p[i]), &p[i].mapOff))) return rc;
			} else if (uses_table(src, p[i])) {
				p[i].mapOff = dst->engMap.off; // (check_copy: the same table)
			} else {
				p[i].customMap = kMapNone;
				p[i].mapOff = p[i].mapN = 0;
			}
		}
		// the source's records and tables are free again once the destination has read them
		CK(cudaEventRecord(dst->evXfer, dst->stream));
		e = src;
		CK(cudaSetDevice(src->device));
		CK(cudaStreamWaitEvent(src->stream, dst->evXfer, 0));
	}
	dst->chainedGroups = 0;
	for (int i = 0; i < n; ++i) dst->hSprm[dstS[i]] = p[i];
	params_changed(dst);
	dst->prevCallMayRandom = dst->prevCallMayRandom || src->prevCallMayRandom;
	dst->seekMayRandom = dst->seekMayRandom || src->seekMayRandom;
	return 0;
}

// =================================================================================================
// extern "C" ABI
// =================================================================================================
extern "C" {

int b200s_create(int batch, long seed, int device, b200s_engine **out) {
	if (!out || batch < 1) {
		g_createError = "b200s_create: bad arguments";
		return B200S_EINVAL;
	}
	*out = 0;
	int n = 0;
	cudaError_t ce = cudaGetDeviceCount(&n);
	if (ce != cudaSuccess || n <= 0 || device < 0 || device >= n) {
		g_createError = std::string("no usable CUDA device (this library has no CPU path): ") + (ce != cudaSuccess ? cudaGetErrorString(ce) : "device index out of range");
		return B200S_ENODEVICE;
	}
	b200s_engine *e = new b200s_engine();
	e->S = batch;
	e->allProcess.assign((size_t)batch, B200S_OP_PROCESS);
	e->seed = seed;
	e->device = device;
	memset(&e->cfg, 0, sizeof(e->cfg));
	{
		StreamParams p;
		memset(&p, 0, sizeof(p));
		p.freqMultiplier = 1;
		p.freqTonalityLimit = 0.5f; // :513
		p.formantMultiplier = p.invFormantMultiplier = 1;
		e->hSprm.assign((size_t)batch, p);
		params_changed(e);
	}
	if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess ||
	    cudaEventCreate(&e->evStart) != cudaSuccess || cudaEventCreate(&e->evStop) != cudaSuccess) {
		g_createError = "CUDA stream/event creation failed";
		delete e;
		return B200S_ECUDA;
	}
	e->ownStream = true;
	{
		int lo = 0, hi = 0;
		cudaDeviceGetStreamPriorityRange(&lo, &hi);
		if (cudaStreamCreateWithPriority(&e->commitStream, cudaStreamNonBlocking, hi) != cudaSuccess ||
		    cudaEventCreateWithFlags(&e->evFork, cudaEventDisableTiming) != cudaSuccess ||
		    cudaEventCreateWithFlags(&e->evJoin, cudaEventDisableTiming) != cudaSuccess)
			e->commitStream = 0; // (no fork then: the commit follows the synthesis on the main stream)
	}
	for (int k = 0; k < 2; ++k) {
		bool ok = host_alloc((void **)&e->pinSprm[k], sizeof(StreamParams) * (size_t)batch) &&
		          cudaEventCreateWithFlags(&e->evSprm[k], cudaEventDisableTiming) == cudaSuccess &&
		          cudaEventCreateWithFlags(&e->evIdx[k], cudaEventDisableTiming) == cudaSuccess &&
		          (k || cudaEventCreateWithFlags(&e->evXfer, cudaEventDisableTiming) == cudaSuccess) &&
		          host_alloc((void **)&e->pinDesc[k], sizeof(CallDesc) * (size_t)batch);
		for (int i = 0; i < b200s_engine::kMaxSub && ok; ++i) ok = cudaEventCreateWithFlags(&e->evDesc[k][i], cudaEventDisableTiming) == cudaSuccess;
		if (!ok) {
			g_createError = "pinned host memory / event creation failed";
			b200s_destroy(e);
			return B200S_ECUDA;
		}
	}
	{ // sub-batch streams: highest priority first
		int lo = 0, hi = 0;
		cudaDeviceGetStreamPriorityRange(&lo, &hi);
		bool ok = cudaEventCreateWithFlags(&e->evBegin, cudaEventDisableTiming) == cudaSuccess;
		for (int i = 0; i < b200s_engine::kMaxSub && ok; ++i) {
			int pr = hi + i;
			if (pr > lo) pr = lo;
			ok = cudaStreamCreateWithPriority(&e->subStream[i], cudaStreamNonBlocking, pr) == cudaSuccess &&
			     cudaEventCreateWithFlags(&e->evSubDone[i], cudaEventDisableTiming) == cudaSuccess;
		}
		// Off by default: the wavefront kernel is bound by per-warp latency, not by occupancy, so FFT CTAs
		// co-running with it only steal its issue slots.  Kept (off) for
		// batches large enough to oversubscribe the SMs; b200s_set_sub_batches() turns it on.
		e->nSub = 1;
		e->maxSub = ok ? b200s_engine::kMaxSub : 1;
		if (const char *hp = getenv("B200S_HOST_PARTS")) e->nHostParts = std::max(1, atoi(hp)); // tuning knob of the host-buffer pipeline
	}
	*out = e;
	return 0;
}
void b200s_destroy(b200s_engine *e) {
	if (!e) return;
	cudaSetDevice(e->device);
	cudaStreamSynchronize(e->stream);
	free_all(e);
	dfree(e->dMaps);
	dfree(e->dRng);
	dfree(e->dDiag);
	dfree(e->dSeekStf);
	dfree(e->dSeekEnd);
	dfree(e->dSprm);
	dfree(e->dDesc);
	dfree(e->dXfer);
	dfree(e->dXferIdx);
	if (e->evXfer) cudaEventDestroy(e->evXfer);
	for (int k = 0; k < 2; ++k) {
		host_free(e->pinIdx[k]);
		if (e->evIdx[k]) cudaEventDestroy(e->evIdx[k]);
		host_free(e->pinSprm[k]);
		if (e->evSprm[k]) cudaEventDestroy(e->evSprm[k]);
		host_free(e->pinDesc[k]);
		for (int i = 0; i < b200s_engine::kMaxSub; ++i)
			if (e->evDesc[k][i]) cudaEventDestroy(e->evDesc[k][i]);
	}
	for (int i = 0; i < b200s_engine::kMaxSub; ++i) {
		if (e->subStream[i]) cudaStreamDestroy(e->subStream[i]);
		if (e->evSubDone[i]) cudaEventDestroy(e->evSubDone[i]);
	}
	if (e->evBegin) cudaEventDestroy(e->evBegin);
	if (e->commitStream) cudaStreamDestroy(e->commitStream);
	if (e->evFork) cudaEventDestroy(e->evFork);
	if (e->evJoin) cudaEventDestroy(e->evJoin);
	if (e->evStart) cudaEventDestroy(e->evStart);
	if (e->evStop) cudaEventDestroy(e->evStop);
	if (e->ownStream && e->stream) cudaStreamDestroy(e->stream);
	delete e;
}
const char *b200s_last_error(const b200s_engine *e) { return e ? e->err.c_str() : g_createError.c_str(); }
int b200s_version(int *major, int *minor, int *patch) {
	if (major) *major = 1;
	if (minor) *minor = 3;
	if (patch) *patch = 2;
	return 0;
}
int b200s_set_stream(b200s_engine *e, void *cuda_stream) {
	if (!e) return B200S_EINVAL;
	CK(cudaStreamSynchronize(e->stream));
	if (e->ownStream && e->stream) cudaStreamDestroy(e->stream);
	e->stream = (cudaStream_t)cuda_stream;
	e->ownStream = false;
	return 0;
}
int b200s_set_sub_batches(b200s_engine *e, int n) {
	if (!e || n < 1) return B200S_EINVAL;
	e->nSub = n > e->maxSub ? e->maxSub : n;
	return 0;
}
int b200s_set_tuning(b200s_engine *e, int key, int value) {
	if (!e) return B200S_EINVAL;
	if (key == 0 && value >= 0 && value <= 6) {
#ifndef B200S_KEEP_OLD_KERNELS
		if (value == 1 || value == 3 || value == 5) {
			e->err = "b200s_set_tuning: chain generations 1, 3 and 5 are superseded and not part of this build (-DB200S_KEEP_OLD_KERNELS)";
			return B200S_EUNSUPPORTED;
		}
#endif
		e->chainV = value;
	}
	else if (key == 1 && (value == 0 || value == 1)) e->fftV1 = value;
	else if (key == 2 && value >= 1) e->nHostParts = std::min(value, (int)b200s_engine::kMaxSub);
	else if (key == 3 && (value == 0 || value == 1)) e->exactMath = value;
	else if (key == 4 && (value == 0 || value == 1)) e->stepMajor = value;
	else if (key == 5 && (value == 0 || value == 1)) e->dual = value;
	else {
		e->err = "b200s_set_tuning: unknown key or value";
		return B200S_EINVAL;
	}
	return 0;
}
int b200s_synchronize(b200s_engine *e) {
	if (!e) return B200S_EINVAL;
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}

int b200s_preset_default(b200s_engine *e, int channels, float sr, int split) {
	return configure_impl(e, channels, int(sr * 0.12), int(sr * 0.03), split); // :63-65
}
int b200s_preset_cheaper(b200s_engine *e, int channels, float sr, int split) {
	return configure_impl(e, channels, int(sr * 0.1), int(sr * 0.04), split); // :66-68
}
int b200s_configure(b200s_engine *e, int channels, int block, int interval, int split) { return configure_impl(e, channels, block, interval, split); }
int b200s_reset(b200s_engine *e) {
	NEED_CFG();
	return reset_impl(e, true);
}
int b200s_reserve(b200s_engine *e, int maxIn, int maxOut) {
	NEED_CFG();
	int rc;
	// (an output seek of b200s_run_per_stream writes outputLatency samples of pre-roll in the process pass)
	const int pass2Out = std::max(maxOut, b200s_output_latency(e));
	if ((rc = ensure_scratch(e, pass2Out))) return rc;
	if (e->nMapped > 0 && (rc = e->stepMajor ? ensure_stepmajor(e) : ensure_coef(e))) return rc;
	if ((rc = stage_in(e, 0, 0))) return rc;
	size_t ci = (size_t)e->cfg.S * e->cfg.C * std::max(maxIn, 1), co = (size_t)e->cfg.S * e->cfg.C * std::max(maxOut, 1);
	if ((rc = ensure_buf(e, &e->dIn, &e->inCap, ci, false))) return rc;
	if ((rc = ensure_buf(e, &e->dOut, &e->outCap, co, false))) return rc;
	// b200s_run_per_stream: the zero row of flushes that read up to maxIn zeros; output rows narrower than outputLatency
	// take the output seeks' pre-roll through dTmp
	if ((rc = ensure_buf(e, &e->dZero, &e->zeroCap, (size_t)std::max(maxIn, 1), true))) return rc;
	if (maxOut >= b200s_output_latency(e)) return 0;
	return ensure_buf(e, &e->dTmp, &e->tmpCap, (size_t)e->cfg.S * e->cfg.C * b200s_output_latency(e), false);
}

int b200s_batch(const b200s_engine *e) { return e ? e->S : 0; }
int b200s_channels(const b200s_engine *e) { return e && e->configured ? e->cfg.C : 0; }
int b200s_block_samples(const b200s_engine *e) { return e && e->configured ? e->cfg.B : 0; }
int b200s_interval_samples(const b200s_engine *e) { return e && e->configured ? e->cfg.H : 0; }
int b200s_input_latency(const b200s_engine *e) { return e && e->configured ? e->cfg.B - e->cfg.B / 2 : 0; }                       // :42-44
int b200s_output_latency(const b200s_engine *e) { return e && e->configured ? e->cfg.B / 2 + (e->cfg.split ? e->cfg.H : 0) : 0; } // :45-47
int b200s_split_computation(const b200s_engine *e) { return e && e->configured ? e->cfg.split : 0; }
int b200s_seek_length(const b200s_engine *e) { return e && e->configured ? e->cfg.B + e->cfg.H : 0; } // :166-168
int b200s_output_seek_length(const b200s_engine *e, float rate) {                                       // :205-207
	return e && e->configured ? int(b200s_input_latency(e) + rate * b200s_output_latency(e)) : 0;
}
int b200s_fft_samples(const b200s_engine *e) { return e && e->configured ? e->cfg.N : 0; }
int b200s_bands(const b200s_engine *e) { return e && e->configured ? e->cfg.K : 0; }

// One stream's entry, set by exactly the arithmetic of the reference's setters: the broadcast setters apply these to every
// entry, the per-stream ones entry by entry, so a stream gets the same bits either way (and as a one-stream reference).
static void set_transpose(StreamParams &p, float multiplier, float tonality) { // :107-115
	p.freqMultiplier = multiplier;
	if (tonality > 0) p.freqTonalityLimit = tonality / std::sqrt(multiplier);
	else p.freqTonalityLimit = 1;
	p.customMap = kMapNone; // (setTransposeFactor clears customFreqMap)
	p.mapOff = p.mapN = 0;
}
static float semitones_factor(float semitones) { return std::pow(2, semitones / 12); } // :116-118, :129-131
static void set_formant(StreamParams &p, float multiplier, int comp) { // :124-128
	p.formantMultiplier = multiplier;
	p.invFormantMultiplier = 1 / multiplier;
	p.formantCompensation = comp ? 1 : 0;
}

int b200s_set_transpose_factor(b200s_engine *e, float multiplier, float tonality) {
	if (!e) return B200S_EINVAL;
	for (StreamParams &p : e->hSprm) set_transpose(p, multiplier, tonality);
	params_changed(e);
	return 0;
}
int b200s_set_transpose_semitones(b200s_engine *e, float semitones, float tonality) {
	return b200s_set_transpose_factor(e, semitones_factor(semitones), tonality);
}
int b200s_set_formant_factor(b200s_engine *e, float multiplier, int comp) {
	if (!e) return B200S_EINVAL;
	for (StreamParams &p : e->hSprm) set_formant(p, multiplier, comp);
	params_changed(e);
	return 0;
}
int b200s_set_formant_semitones(b200s_engine *e, float semitones, int comp) {
	return b200s_set_formant_factor(e, semitones_factor(semitones), comp);
}
int b200s_set_formant_base(b200s_engine *e, float f) { // :133-135
	if (!e) return B200S_EINVAL;
	for (StreamParams &p : e->hSprm) p.formantBaseFreq = f;
	params_changed(e);
	return 0;
}
int b200s_set_transpose_factor_per_stream(b200s_engine *e, const float *multipliers, const float *tonality) {
	if (!e || !multipliers) return B200S_EINVAL;
	for (int s = 0; s < e->S; ++s) set_transpose(e->hSprm[s], multipliers[s], tonality ? tonality[s] : 0.f);
	params_changed(e);
	return 0;
}
int b200s_set_transpose_semitones_per_stream(b200s_engine *e, const float *semitones, const float *tonality) {
	if (!e || !semitones) return B200S_EINVAL;
	for (int s = 0; s < e->S; ++s) set_transpose(e->hSprm[s], semitones_factor(semitones[s]), tonality ? tonality[s] : 0.f);
	params_changed(e);
	return 0;
}
int b200s_set_formant_factor_per_stream(b200s_engine *e, const float *multipliers, const int *comp) {
	if (!e || !multipliers) return B200S_EINVAL;
	for (int s = 0; s < e->S; ++s) set_formant(e->hSprm[s], multipliers[s], comp ? comp[s] : 0);
	params_changed(e);
	return 0;
}
int b200s_set_formant_semitones_per_stream(b200s_engine *e, const float *semitones, const int *comp) {
	if (!e || !semitones) return B200S_EINVAL;
	for (int s = 0; s < e->S; ++s) set_formant(e->hSprm[s], semitones_factor(semitones[s]), comp ? comp[s] : 0);
	params_changed(e);
	return 0;
}
int b200s_set_formant_base_per_stream(b200s_engine *e, const float *base) {
	if (!e || !base) return B200S_EINVAL;
	for (int s = 0; s < e->S; ++s) e->hSprm[s].formantBaseFreq = base[s];
	params_changed(e);
	return 0;
}
int b200s_set_freq_map_table(b200s_engine *e, const float *fin, const float *fout, int n) {
	if (!e || n < 0 || (n > 0 && (!fin || !fout))) return B200S_EINVAL;
	e->engMap = make_table(n, fin, fout);
	for (StreamParams &p : e->hSprm) p.customMap = kMapEngine; // every stream, until a transpose setter or its own table
	return layout_maps(e, {});
}
int b200s_set_freq_map_table_per_stream(b200s_engine *e, const int *streams, int n, const int *n_points, const float *fin, const float *fout) {
	if (!e) return B200S_EINVAL;
	std::string why;
	if (n < 0) why = "negative stream count";
	else if (n > 0 && (!streams || !n_points)) why = std::string(streams ? "n_points" : "streams") + " must not be NULL";
	long long total = 0;
	std::vector<char> seen((size_t)e->S, 0);
	for (int i = 0; i < n && why.empty(); ++i) {
		const int s = streams[i];
		const std::string at = "streams[" + std::to_string(i) + "]";
		if (s < 0 || s >= e->S) why = at + " = " + std::to_string(s) + " is outside [0, " + std::to_string(e->S) + ")";
		else if (seen[s]++) why = at + ": stream " + std::to_string(s) + " is listed twice";
		else if (n_points[i] < 0) why = "n_points[" + std::to_string(i) + "] = " + std::to_string(n_points[i]) + " is negative";
		else total += n_points[i];
	}
	if (why.empty() && total > 0 && (!fin || !fout)) why = "freq_in and freq_out must not be NULL";
	if (!why.empty()) {
		e->err = "b200s_set_freq_map_table_per_stream: " + why;
		return B200S_EINVAL;
	}
	if (n == 0) return 0;
	std::vector<MapTable> tabs((size_t)n);
	std::vector<const MapTable *> want((size_t)e->S, nullptr);
	for (long long i = 0, at = 0; i < n; at += n_points[i++]) {
		StreamParams &p = e->hSprm[streams[i]];
		p.customMap = n_points[i] > 0 ? kMapOwn : kMapNone;
		if (n_points[i] == 0) continue;
		tabs[i] = make_table(n_points[i], fin + at, fout + at);
		want[streams[i]] = &tabs[i];
	}
	return layout_maps(e, want);
}

int b200s_seek_device(b200s_engine *e, const float *dIn, int n, double rate) {
	NEED_CFG();
	if (n < 0) return B200S_EINVAL;
	return seek_impl(e, dIn, n, (long long)e->cfg.C * n, n, rate);
}
int b200s_process_device(b200s_engine *e, const float *dIn, int nIn, float *dOut, int nOut) {
	NEED_CFG();
	int rc;
	return process_impl(e, dIn, nIn, (long long)e->cfg.C * nIn, nIn, dOut, nOut, (long long)e->cfg.C * nOut, nOut);
}
int b200s_flush_device(b200s_engine *e, float *dOut, int nOut, float rate) {
	NEED_CFG();
	if (nOut < 0) return B200S_EINVAL;
	return flush_impl(e, dOut, nOut, (long long)e->cfg.C * nOut, nOut, rate);
}
int b200s_seek(b200s_engine *e, const float *in, int n, double rate) {
	NEED_CFG();
	if (n < 0) return B200S_EINVAL;
	int rc;
	if ((rc = stage_in(e, in, n))) return rc;
	if ((rc = seek_impl(e, e->dIn, n, (long long)e->cfg.C * n, n, rate))) return rc;
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}
int b200s_seek_rates(b200s_engine *e, const float *in, int n, const double *rates) {
	NEED_CFG();
	if (n < 0 || !rates) return B200S_EINVAL;
	int rc;
	if ((rc = stage_in(e, in, n))) return rc;
	if ((rc = seek_impl(e, e->dIn, n, (long long)e->cfg.C * n, n, 1.0, rates))) return rc;
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}
int b200s_live_seek(b200s_engine *e, const float *d_bank, long long bank_len, const long long *window_end, int window, const double *rates) {
	NEED_CFG();
	if (window < 0 || bank_len < 0 || !d_bank || !window_end || !rates) return B200S_EINVAL;
	if (bank_len > 0x7fffffffLL) {
		e->err = "b200s_live_seek: bank rows longer than 2^31-1 samples are not supported";
		return B200S_EUNSUPPORTED;
	}
	return seek_impl(e, d_bank, (int)bank_len, (long long)e->cfg.C * bank_len, window, 1.0, rates, window_end, bank_len);
}
int b200s_process(b200s_engine *e, const float *in, int nIn, float *out, int nOut) {
	NEED_CFG();
	int rc;
	if ((rc = stage_in(e, nullptr, nIn))) return rc; // capacity only: the copies are issued per stream group
	if ((rc = stage_out(e, nOut))) return rc;
	if ((rc = process_impl(e, e->dIn, nIn, (long long)e->cfg.C * nIn, nIn, e->dOut, nOut, (long long)e->cfg.C * nOut, nOut, in, out))) return rc;
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}
// 16-bit PCM host buffers (asynchronous like b200s_process_async when `wait` is 0)
int b200s_process_pcm16(b200s_engine *e, const short *in, int nIn, short *out, int nOut, int wait) {
	NEED_CFG();
	int rc;
	const size_t ci = (size_t)e->cfg.S * e->cfg.C * std::max(nIn, 1), co = (size_t)e->cfg.S * e->cfg.C * std::max(nOut, 1);
	if (ci > e->inCap || co > e->outCap || ci > e->in16Cap || co > e->out16Cap || !e->dIn || !e->dOut) CK(cudaStreamSynchronize(e->stream)); // staging grows: drain first
	if ((rc = stage_in(e, nullptr, nIn))) return rc;
	if ((rc = stage_out(e, nOut))) return rc;
	if ((rc = stage_pcm16(e, ci, co))) return rc;
	if ((rc = process_impl(e, e->dIn, nIn, (long long)e->cfg.C * nIn, nIn, e->dOut, nOut, (long long)e->cfg.C * nOut, nOut, nullptr, nullptr, in, out))) return rc;
	if (wait) CK(cudaStreamSynchronize(e->stream));
	return 0;
}
int b200s_process_async(b200s_engine *e, const float *in, int nIn, float *out, int nOut) {
	NEED_CFG();
	int rc;
	if ((size_t)e->cfg.S * e->cfg.C * std::max(nIn, 1) > e->inCap || (size_t)e->cfg.S * e->cfg.C * std::max(nOut, 1) > e->outCap || !e->dIn || !e->dOut) {
		// growing the staging buffers would invalidate copies still in flight: drain first
		CK(cudaStreamSynchronize(e->stream));
	}
	if ((rc = stage_in(e, nullptr, nIn))) return rc;
	if ((rc = stage_out(e, nOut))) return rc;
	return process_impl(e, e->dIn, nIn, (long long)e->cfg.C * nIn, nIn, e->dOut, nOut, (long long)e->cfg.C * nOut, nOut, in, out);
}
// Arguments of the per-stream calls, checked before anything is enqueued: the batch's S entries, or the n entries of a
// list (the message then names the entry and its stream)
static int check_run(b200s_engine *e, const char *fn, const int *ops, int inStride, const int *nIn, int outStride, const int *nOut, const double *rates,
                     const int *list = nullptr, int n = -1) {
	const int P = n >= 0 ? n : e->S;
	if (P > 0 && (!ops || !nIn || !nOut)) {
		e->err = std::string(fn) + ": " + (ops ? "input_samples and output_samples must not be NULL" : "ops must not be NULL");
		return B200S_EINVAL;
	}
	if (inStride < 0 || outStride < 0) {
		e->err = std::string(fn) + ": negative stride";
		return B200S_EINVAL;
	}
	for (int s = 0; s < P; ++s) {
		const int op = ops[s];
		std::string why;
		if (op < B200S_OP_SKIP || op > B200S_OP_RESET) why = "op " + std::to_string(op) + " is not a B200S_OP_*";
		else if (op == B200S_OP_SEEK && !rates) why = "SEEK needs playback_rates";
		else if (nIn[s] != 0 && (op == B200S_OP_FLUSH || op == B200S_OP_RESET || op == B200S_OP_SKIP))
			why = "op " + std::to_string(op) + " reads no input, input_samples is " + std::to_string(nIn[s]);
		else if (nOut[s] != 0 && op != B200S_OP_PROCESS && op != B200S_OP_FLUSH)
			why = "op " + std::to_string(op) + " writes no output, output_samples is " + std::to_string(nOut[s]);
		else if (nIn[s] < 0 || nIn[s] > inStride)
			why = "input_samples " + std::to_string(nIn[s]) + " is outside [0, " + std::to_string(inStride) + "]";
		else if (nOut[s] < 0 || nOut[s] > outStride)
			why = "output_samples " + std::to_string(nOut[s]) + " is outside [0, " + std::to_string(outStride) + "]";
		if (!why.empty()) {
			e->err = std::string(fn) + ": " + (list ? "entry " + std::to_string(s) + " (stream " + std::to_string(list[s]) + ")" : "stream " + std::to_string(s)) + ": " + why;
			return B200S_EINVAL;
		}
	}
	return 0;
}
static int run_entry(b200s_engine *e, const char *fn, const int *ops, const float *in, int inStride, const int *nIn, float *out,
                     int outStride, const int *nOut, const double *rates, bool host, bool wait, const short *in16 = nullptr,
                     short *out16 = nullptr) {
	NEED_CFG();
	int rc;
	if ((rc = check_run(e, fn, ops, inStride, nIn, outStride, nOut, rates))) return rc;
	return run_impl(e, ops, in, inStride, nIn, out, outStride, nOut, rates, host, wait, nullptr, 0, in16, out16);
}
int b200s_run_per_stream(b200s_engine *e, const int *ops, const float *in, int inStride, const int *nIn, float *out, int outStride,
                         const int *nOut, const double *rates) {
	return run_entry(e, "b200s_run_per_stream", ops, in, inStride, nIn, out, outStride, nOut, rates, true, true);
}
int b200s_run_per_stream_async(b200s_engine *e, const int *ops, const float *in, int inStride, const int *nIn, float *out, int outStride,
                               const int *nOut, const double *rates) {
	return run_entry(e, "b200s_run_per_stream_async", ops, in, inStride, nIn, out, outStride, nOut, rates, true, false);
}
int b200s_run_per_stream_device(b200s_engine *e, const int *ops, const float *dIn, int inStride, const int *nIn, float *dOut, int outStride,
                                const int *nOut, const double *rates) {
	return run_entry(e, "b200s_run_per_stream_device", ops, dIn, inStride, nIn, dOut, outStride, nOut, rates, false, false);
}
// b200s_run_per_stream over a list of streams
static int run_streams_entry(b200s_engine *e, const char *fn, int n, const int *streams, const int *ops, const float *in, int inStride,
                             const int *nIn, float *out, int outStride, const int *nOut, const double *rates, bool host, bool wait,
                             const short *in16 = nullptr, short *out16 = nullptr) {
	NEED_CFG();
	if (n < 0 || n > e->S) {
		e->err = std::string(fn) + ": n = " + std::to_string(n) + " is outside [0, " + std::to_string(e->S) + "]";
		return B200S_EINVAL;
	}
	if (!check_streams(e->err, fn, "streams", streams, n, e->S, true)) return B200S_EINVAL;
	int rc;
	if ((rc = check_run(e, fn, ops, inStride, nIn, outStride, nOut, rates, streams, n))) return rc;
	if (n == 0) return 0;
	return run_impl(e, ops, in, inStride, nIn, out, outStride, nOut, rates, host, wait, streams, n, in16, out16);
}
int b200s_run_streams(b200s_engine *e, int n, const int *streams, const int *ops, const float *in, int inStride, const int *nIn,
                      float *out, int outStride, const int *nOut, const double *rates) {
	return run_streams_entry(e, "b200s_run_streams", n, streams, ops, in, inStride, nIn, out, outStride, nOut, rates, true, true);
}
int b200s_run_streams_async(b200s_engine *e, int n, const int *streams, const int *ops, const float *in, int inStride, const int *nIn,
                            float *out, int outStride, const int *nOut, const double *rates) {
	return run_streams_entry(e, "b200s_run_streams_async", n, streams, ops, in, inStride, nIn, out, outStride, nOut, rates, true, false);
}
int b200s_run_streams_device(b200s_engine *e, int n, const int *streams, const int *ops, const float *dIn, int inStride, const int *nIn,
                             float *dOut, int outStride, const int *nOut, const double *rates) {
	return run_streams_entry(e, "b200s_run_streams_device", n, streams, ops, dIn, inStride, nIn, dOut, outStride, nOut, rates, false, false);
}
// 16-bit PCM host buffers (the conversions of b200s_process_pcm16, on the device)
int b200s_run_per_stream_pcm16(b200s_engine *e, const int *ops, const short *in, int inStride, const int *nIn, short *out, int outStride,
                               const int *nOut, const double *rates, int wait) {
	return run_entry(e, "b200s_run_per_stream_pcm16", ops, nullptr, inStride, nIn, nullptr, outStride, nOut, rates, true, wait != 0, in, out);
}
int b200s_run_streams_pcm16(b200s_engine *e, int n, const int *streams, const int *ops, const short *in, int inStride, const int *nIn,
                            short *out, int outStride, const int *nOut, const double *rates, int wait) {
	return run_streams_entry(e, "b200s_run_streams_pcm16", n, streams, ops, nullptr, inStride, nIn, nullptr, outStride, nOut, rates, true,
	                         wait != 0, in, out);
}
// process() with per-stream lengths: b200s_run_per_stream with every op PROCESS
int b200s_process_per_stream(b200s_engine *e, const float *in, int inStride, const int *nIn, float *out, int outStride, const int *nOut) {
	return run_entry(e, "b200s_process_per_stream", e ? e->allProcess.data() : nullptr, in, inStride, nIn, out, outStride, nOut, nullptr, true, true);
}
int b200s_process_per_stream_async(b200s_engine *e, const float *in, int inStride, const int *nIn, float *out, int outStride, const int *nOut) {
	return run_entry(e, "b200s_process_per_stream_async", e ? e->allProcess.data() : nullptr, in, inStride, nIn, out, outStride, nOut, nullptr, true, false);
}
int b200s_process_per_stream_device(b200s_engine *e, const float *dIn, int inStride, const int *nIn, float *dOut, int outStride, const int *nOut) {
	return run_entry(e, "b200s_process_per_stream_device", e ? e->allProcess.data() : nullptr, dIn, inStride, nIn, dOut, outStride, nOut, nullptr, false, false);
}
int b200s_flush(b200s_engine *e, float *out, int nOut, float rate) {
	NEED_CFG();
	if (nOut < 0) return B200S_EINVAL;
	int rc;
	if ((rc = stage_out(e, nOut))) return rc;
	if ((rc = flush_impl(e, e->dOut, nOut, (long long)e->cfg.C * nOut, nOut, rate))) return rc;
	return fetch_out(e, out, nOut);
}
int b200s_output_seek(b200s_engine *e, const float *in, int inputLength) {
	NEED_CFG();
	if (inputLength < 0) return B200S_EINVAL;
	int rc;
	if ((rc = stage_in(e, in, inputLength))) return rc;
	if ((rc = output_seek_impl(e, e->dIn, inputLength, (long long)e->cfg.C * inputLength, inputLength))) return rc;
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}
int b200s_exact(b200s_engine *e, const float *in, int nIn, float *out, int nOut, int *ok) { // :467-491
	NEED_CFG();
	if (nIn < 0 || nOut <= 0) return B200S_EINVAL;
	int rc;
	const Cfg &g = e->cfg;
	float playbackRate = nIn / float(nOut);
	int seekLen = b200s_output_seek_length(e, playbackRate);
	if (ok) *ok = 0;
	if (nIn < seekLen) {
		memset(out, 0, sizeof(float) * (size_t)g.S * g.C * nOut);
		return 0;
	}
	if ((rc = stage_in(e, in, nIn))) return rc;
	if ((rc = stage_out(e, nOut))) return rc;
	const long long inSS = (long long)g.C * nIn, outSS = (long long)g.C * nOut;
	if ((rc = output_seek_impl(e, e->dIn, nIn, inSS, seekLen))) return rc;
	int outputIndex = int(nOut - seekLen / playbackRate); // :484
	if ((rc = process_impl(e, e->dIn + seekLen, nIn, inSS, nIn - seekLen, e->dOut, nOut, outSS, outputIndex))) return rc;
	if ((rc = flush_impl(e, e->dOut + outputIndex, nOut, outSS, nOut - outputIndex, playbackRate))) return rc;
	if (ok) *ok = 1;
	return fetch_out(e, out, nOut);
}

int b200s_timer_start(b200s_engine *e) {
	if (!e) return B200S_EINVAL;
	CK(cudaEventRecord(e->evStart, e->stream));
	return 0;
}
int b200s_timer_stop(b200s_engine *e, float *ms) {
	if (!e || !ms) return B200S_EINVAL;
	CK(cudaEventRecord(e->evStop, e->stream));
	CK(cudaEventSynchronize(e->evStop));
	CK(cudaEventElapsedTime(ms, e->evStart, e->evStop));
	return 0;
}
long long b200s_kernel_launches(const b200s_engine *e) { return e ? e->launches : 0; }
long long b200s_device_allocations(const b200s_engine *e) { return e ? e->allocs : 0; }
long long b200s_unserved_random_blocks(b200s_engine *e) {
	if (!e || !e->dDiag) return 0;
	unsigned long long v = 0;
	if (cudaStreamSynchronize(e->stream) != cudaSuccess || cudaMemcpy(&v, e->dDiag, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
	return (long long)v;
}
int b200s_profile_begin(b200s_engine *e) {
	if (!e) return B200S_EINVAL;
	e->profiling = true;
	return 0;
}
int b200s_profile_end(b200s_engine *e, float *ms, int *counts, int n) {
	if (!e || !ms || !counts || n < PK_PHASE) return B200S_EINVAL;
	e->profiling = false;
	CK(cudaStreamSynchronize(e->stream));
	for (int i = 0; i < n; ++i) {
		ms[i] = 0;
		counts[i] = 0;
	}
	for (size_t i = 0; i < e->profKind.size(); ++i) {
		float t = 0;
		if (e->profKind[i] >= n) continue; // (the phases' kind, when the caller asked for the six kernels only)
		CK(cudaEventElapsedTime(&t, e->profEv[2 * i], e->profEv[2 * i + 1]));
		ms[e->profKind[i]] += t;
		counts[e->profKind[i]] += 1;
	}
	for (cudaEvent_t ev : e->profEv) cudaEventDestroy(ev);
	e->profEv.clear();
	e->profKind.clear();
	return 0;
}

// Device self-test of the branch-free division / square root used by the phase chain.
int b200s_selftest_divsqrt(b200s_engine *e, long long n, long long seed, long long *divMismatch, long long *sqrtMismatch) {
	if (!e || n <= 0) return B200S_EINVAL;
	unsigned long long *d = 0;
	int rc;
	if ((rc = dalloc(e, &d, 2))) return rc;
	CK(cudaMemset(d, 0, 2 * sizeof(unsigned long long)));
	const int threads = 256, blocks = 1184, per = (int)((n + (long long)threads * blocks - 1) / ((long long)threads * blocks));
	B200S_LAUNCH(k_selftest_divsqrt, dim3(blocks), dim3(threads), 0, e->stream, (unsigned long long)seed, per, d);
	CKL();
	unsigned long long h[2] = {0, 0};
	CK(cudaStreamSynchronize(e->stream));
	CK(cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost));
	cudaFree(d);
	if (divMismatch) *divMismatch = (long long)h[0];
	if (sqrtMismatch) *sqrtMismatch = (long long)h[1];
	return 0;
}

// ---- white-box state ----
static int state_desc(const b200s_engine *e, int what, float **ptr, size_t *perStream) {
	const Cfg &g = e->cfg;
	switch (what) {
	case 0: *ptr = (float *)e->dStIn; *perStream = (size_t)2 * g.C * g.K; return 0;
	case 1: *ptr = (float *)e->dStPrev; *perStream = (size_t)2 * g.C * g.K; return 0;
	case 2: *ptr = (float *)e->dStOut; *perStream = (size_t)2 * g.C * g.K; return 0;
	case 4: *ptr = e->dStPredE; *perStream = (size_t)g.C * g.K; return 0;
	case 20: *ptr = e->dHist[e->histCur]; *perStream = (size_t)g.C * g.histLen; return 0;
	case 21: *ptr = e->dPend; *perStream = (size_t)g.C * g.pendLen; return 0;
	case 22: *ptr = e->dPendWp; *perStream = (size_t)g.C * g.pendLen; return 0;
	}
	return B200S_EINVAL;
}
int b200s_state_size(const b200s_engine *e, int what) {
	if (!e || !e->configured) return B200S_EINVAL;
	float *p;
	size_t n;
	if (state_desc(e, what, &p, &n)) return B200S_EINVAL;
	return (int)n;
}
int b200s_get_state(b200s_engine *e, int what, float *dst) {
	NEED_CFG();
	float *p;
	size_t n;
	if (state_desc(e, what, &p, &n)) return B200S_EINVAL;
	CK(cudaStreamSynchronize(e->stream));
	CK(cudaMemcpy(dst, p, sizeof(float) * n * e->S, cudaMemcpyDeviceToHost));
	return 0;
}
int b200s_set_state(b200s_engine *e, int what, const float *src) {
	NEED_CFG();
	float *p;
	size_t n;
	if (state_desc(e, what, &p, &n)) return B200S_EINVAL;
	CK(cudaStreamSynchronize(e->stream));
	CK(cudaMemcpy(p, src, sizeof(float) * n * e->S, cudaMemcpyHostToDevice));
	return 0;
}

// ---- stream state records ----
int b200s_stream_state_bytes(const b200s_engine *e) {
	if (!e || !e->configured) return B200S_EINVAL;
	return (int)state_regions(e).recBytes;
}
int b200s_copy_streams(b200s_engine *dst, const int *dst_streams, b200s_engine *src, const int *src_streams, int n) {
	if (!dst || !src) return B200S_EINVAL;
	int rc;
	if ((rc = check_copy(dst, dst_streams, src, src_streams, n))) return rc;
	return copy_impl(dst, dst_streams, src, src_streams, n);
}
int b200s_export_streams(b200s_engine *e, const int *streams, int n, void *host_dst) {
	NEED_CFG();
	if (n < 0 || (n > 0 && !host_dst)) {
		e->err = std::string("b200s_export_streams: ") + (n < 0 ? "negative stream count" : "host_dst must not be NULL");
		return B200S_EINVAL;
	}
	if (!check_streams(e->err, "b200s_export_streams", "streams", streams, n, e->S, false)) return B200S_EINVAL;
	if (n == 0) return 0;
	DeviceGuard guard;
	CK(cudaSetDevice(e->device));
	int rc;
	if ((rc = ensure_xfer(e, n, true))) return rc;
	if ((rc = upload_lists(e, streams, nullptr, n))) return rc;
	if ((rc = launch_pack(e, n))) return rc;
	const size_t R = state_regions(e).recBytes;
	CK(cudaMemcpyAsync(host_dst, e->dXfer, (size_t)n * R, cudaMemcpyDeviceToHost, e->stream));
	CK(cudaStreamSynchronize(e->stream));
	for (int i = 0; i < n; ++i) {
		StreamRecordHeader h;
		memset(&h, 0, sizeof(h));
		memcpy(h.magic, "B200SREC", 8);
		h.version = kRecordVersion;
		h.bytes = (uint32_t)R;
		h.C = e->cfg.C; h.B = e->cfg.B; h.H = e->cfg.H; h.split = e->cfg.split; h.K = e->cfg.K;
		const StreamParams &p = e->hSprm[streams[i]];
		h.params = p;
		h.flags = (e->prevCallMayRandom ? kRecPrevRandom : 0) | (e->seekMayRandom ? kRecSeekRandom : 0);
		const MapTable *t = uses_table(e, p) ? &e->engMap : p.customMap == kMapOwn ? stream_table(e, p) : nullptr;
		if (t) {
			h.flags |= uses_table(e, p) ? kRecUsesTable : kRecOwnTable;
			h.mapN = t->n;
			h.mapHash = t->hash;
		} else {
			h.params.customMap = kMapNone;
		}
		char *rec = (char *)host_dst + (size_t)i * R;
		memset(rec, 0, B200S_RECORD_HEADER);
		memcpy(rec, &h, sizeof(h));
	}
	return 0;
}
int b200s_import_streams(b200s_engine *e, const int *streams, int n, const void *host_src) {
	NEED_CFG();
	const char *fn = "b200s_import_streams";
	if (n < 0 || (n > 0 && !host_src)) {
		e->err = std::string(fn) + ": " + (n < 0 ? "negative stream count" : "host_src must not be NULL");
		return B200S_EINVAL;
	}
	if (!check_streams(e->err, fn, "streams", streams, n, e->S, true)) return B200S_EINVAL;
	const size_t R = state_regions(e).recBytes;
	std::vector<StreamRecordHeader> hs((size_t)n);
	std::vector<StreamParams> prm((size_t)n); // the streams' parameters after the import, table descriptors included
	for (int i = 0; i < n; ++i) {
		StreamRecordHeader &h = hs[i];
		memcpy(&h, (const char *)host_src + (size_t)i * R, sizeof(h));
		// a stream with its own table goes into a slot that holds the same table already (its own or the engine's)
		const MapTable *slot = stream_table(e, e->hSprm[streams[i]]);
		std::string why;
		if (memcmp(h.magic, "B200SREC", 8)) why = "not a stream record";
		else if (h.version != kRecordVersion) why = "record format " + std::to_string(h.version) + ", this library reads " + std::to_string(kRecordVersion);
		else if (h.C != e->cfg.C || h.B != e->cfg.B || h.H != e->cfg.H || h.split != e->cfg.split || h.K != e->cfg.K || h.bytes != R)
			why = "recorded with another configuration (" + std::to_string(h.C) + " channels, block " + std::to_string(h.B) + ", interval " +
			      std::to_string(h.H) + (h.split ? ", split" : "") + "; this engine: " + cfg_text(e->cfg) + ")";
		else if ((h.flags & ~(uint32_t)(kRecPrevRandom | kRecSeekRandom | kRecUsesTable | kRecOwnTable)) ||
		         ((h.flags & kRecUsesTable) && (h.flags & kRecOwnTable)))
			why = "unknown flags " + std::to_string(h.flags);
		else if ((h.flags & kRecUsesTable) && (h.mapN != e->engMap.n || h.mapHash != e->engMap.hash))
			why = "the stream uses a frequency-map table that differs from this engine's";
		else if ((h.flags & kRecOwnTable) && !(slot && h.mapN == slot->n && h.mapHash == slot->hash))
			why = "the stream has its own frequency-map table, and slot " + std::to_string(streams[i]) + " does not hold the same table";
		StreamParams &p = prm[i];
		static_cast<StreamSettings &>(p) = h.params;
		const MapTable *t = (h.flags & kRecUsesTable) ? &e->engMap : (h.flags & kRecOwnTable) ? slot : nullptr;
		p.customMap = (h.flags & kRecUsesTable) ? kMapEngine : (h.flags & kRecOwnTable) ? kMapOwn : kMapNone;
		p.mapOff = t ? t->off : 0;
		p.mapN = t ? t->n : 0;
		if (!why.empty()) {
			e->err = std::string(fn) + ": record " + std::to_string(i) + ": " + why;
			return B200S_EINVAL;
		}
	}
	if (n == 0) return 0;
	DeviceGuard guard;
	CK(cudaSetDevice(e->device));
	int rc;
	if ((rc = ensure_xfer(e, n, true))) return rc;
	if ((rc = upload_lists(e, nullptr, streams, n))) return rc;
	CK(cudaMemcpyAsync(e->dXfer, host_src, (size_t)n * R, cudaMemcpyHostToDevice, e->stream));
	e->chainedGroups = 0;
	if ((rc = launch_unpack(e, n, e->dXfer))) return rc;
	for (int i = 0; i < n; ++i) {
		e->hSprm[streams[i]] = prm[i];
		e->prevCallMayRandom = e->prevCallMayRandom || (hs[i].flags & kRecPrevRandom);
		e->seekMayRandom = e->seekMayRandom || (hs[i].flags & kRecSeekRandom);
	}
	params_changed(e);
	CK(cudaStreamSynchronize(e->stream));
	return 0;
}
int b200s_clone(b200s_engine *src, b200s_engine **out) {
	if (!src || !out) {
		g_createError = "b200s_clone: bad arguments";
		return B200S_EINVAL;
	}
	*out = 0;
	b200s_engine *e = 0;
	int rc;
	if ((rc = b200s_create(src->S, src->seed, src->device, &e))) {
		src->err = g_createError;
		return rc;
	}
	e->chainV = src->chainV; e->fftV1 = src->fftV1; e->nHostParts = src->nHostParts; e->exactMath = src->exactMath;
	e->stepMajor = src->stepMajor; e->dual = src->dual; e->nSub = src->nSub;
	// the frequency-map pool as the source lays it out, so that every stream's table descriptor holds as it is
	e->engMap = src->engMap;
	e->maps = src->maps;
	e->mapsUsed = src->mapsUsed;
	if ((rc = upload_maps(e))) goto fail;
	e->hSprm = src->hSprm;
	params_changed(e);
	if (src->configured) {
		std::vector<int> all((size_t)src->S);
		for (int s = 0; s < src->S; ++s) all[s] = s;
		if ((rc = configure_impl(e, src->cfg.C, src->cfg.B, src->cfg.H, src->cfg.split)) || (rc = copy_impl(e, all.data(), src, all.data(), src->S))) goto fail;
	}
	*out = e;
	return 0;
fail:
	src->err = g_createError = "b200s_clone: " + e->err;
	b200s_destroy(e);
	return rc;
}

} // extern "C"
