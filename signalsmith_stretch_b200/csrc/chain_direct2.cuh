// chain_direct2.cuh -- k_chain_direct2: the frame-wavefront phase prediction for calls WITHOUT a
// frequency map and WITHOUT formant processing (pure time-stretch, reference :675-686 identity
// map), second generation.  Same algorithm and the same bit-exact arithmetic as k_chain
// (kernels.cuh, see the wavefront comment there); what changed is how the work is spread:
//
//   * ONE LANE = ONE (block, channel).  A warp owns BPW = 32/C consecutive blocks of a stream, the
//     channels of a block sit in adjacent lanes.  The per-channel work (preliminary prediction,
//     twists, the output of the channel) is done once per lane instead of C times per lane; the
//     cross-channel part of :727-799 (max-energy channel, phase locking of the others) is a few
//     __shfl_xor between the lanes of a block.
//   * SEVERAL WARPS PER STREAM.  Warp w of the CTA owns blocks [w*BPW, (w+1)*BPW) and runs
//     D*BPW bins behind warp w-1: the last block of warp w-1 hands its finals (Band::output,
//     Prediction::energy) to the first block of warp w through a small shared-memory ring with
//     chunk-granular progress counters.  The limiter of the first-generation kernel is
//     per-warp latency (MUFU / shuffle / shared-memory round trips on a serial dependency chain,
//     about two warps per scheduler); this doubles the independent warps per stream at the same
//     instruction count.
//   * The chunk body is unrolled by the FIFO period only (renaming), keeping the loop in the
//     instruction cache.
#pragma once
#include <type_traits>

#include "kernels.cuh"

namespace b200s {

#define CH2_RING 32    // rolling window of the input spectrum (bins), per lane
#define CH2_HO 64      // hand-off ring between consecutive warps (bins)
#define CH2_MAXW 4     // warps (= groups of BPW blocks) per CTA
// Tile row stride (float2).  With the lane = (block, channel) layout a step reads
// [k - D*(lane/C)][lane]; stride 36 makes that read AND the chunk fill below (lane -> 4 rows x 8
// bins, 32 B contiguous per quarter-warp) bank-conflict free for every C in {1,2}, L in 1..8
// (scratch/bank_check.py enumerates the half-warp slot sets).
#define CH2_RS 36

template <int CT>
struct Chain2Tiles { // one per warp
	float2 in[CH2_RING][CH2_RS]; // rolling window of each lane's input spectrum row, [bin & 31][lane]
	// previous-input spectrum at the chunk's prelim bins; step i of a lane reads [i][lane] and then
	// stores its final output of that step into the same slot, so after the chunk this tile holds
	// the finals that the write-back streams to Y
	float2 pvy[CHAIN_CH][CH2_RS];
	float2 hoOut[CT][CH2_HO];       // predecessor block of this warp's first block: final outputs ...
	float hoE[CT][CH2_HO];          // ... and Prediction::energy, [channel][bin & 63]
	const float2 *rowIn[32], *rowPv[32];
	float2 *rowY[32];
};
struct Chain2Sync {
	int done[CH2_MAXW]; // chunks completed by warp w in the current round
};

#ifdef B200S_EMU
__device__ __forceinline__ int ld_volatile_shared(const int *p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
__device__ __forceinline__ void st_volatile_shared(int *p, int v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }
__device__ __forceinline__ void fence_block() { __atomic_thread_fence(__ATOMIC_SEQ_CST); }
__device__ __forceinline__ void spin_pause() { emu_yield(); } // the emulator's threads are cooperative fibers
#else
__device__ __forceinline__ int ld_volatile_shared(const int *p) { return *(volatile const int *)p; }
__device__ __forceinline__ void st_volatile_shared(int *p, int v) { *(volatile int *)p = v; }
__device__ __forceinline__ void fence_block() { __threadfence_block(); }
__device__ __forceinline__ void spin_pause() { __nanosleep(64); }
#endif

__device__ __forceinline__ float2 sel2b(bool p, float2 a) { return make_float2(p ? a.x : 0.f, p ? a.y : 0.f); }

// k_chain_direct6<.., DUAL> (chain_direct6.cuh) packs two mono streams into one warp.  It needs both streams of the pair
// at positions i and i + 1 (i - sBase even; streams s = stream_at(x, i) and t = stream_at(x, i + 1), which a listed call
// may take from anywhere in the batch) to be there, free of random blocks, and to walk the same schedule in this call --
// same blocks, flags, time factors and spectrum slots (streams of a batch do, unless one of them was silent or sought
// differently).  Pairs that fail run one stream at a time (the stream in both halves).
__device__ __forceinline__ bool dual_pair_ok(const Ctx &x, int i, int s, int t, int lane) {
	if (i + 1 >= x.sBase + x.sCount) return false;
	const Call a = x.call[s], b = x.call[t];
	if (a.nFrames == 0 || a.nFrames != b.nFrames || a.bypass || b.bypass) return false;
	if ((a.hasRandom || b.hasRandom) && x.randomPathOn) return false;
	if (a.mapped || b.mapped) return false; // a partner on the mapped path: the plain stream runs alone
	bool bad = false;
	for (int f = lane; f < a.nFrames; f += 32) {
		const Frame fa = x.frames[(size_t)s * x.maxFrames + f], fb = x.frames[(size_t)t * x.maxFrames + f];
		bad = bad || fa.flags != fb.flags || fa.timeFactor != fb.timeFactor || fa.inSlot != fb.inSlot || fa.prevSlot != fb.prevSlot;
	}
	return !__any_sync(0xffffffffu, bad);
}

// FAST (round 2; the default of the mono plain path, b200s_set_tuning key 3 = 1 selects the exact form): the fused
// arithmetic of kernels.cuh (fmul_f, make_output_fast, ...), as the packed stereo kernel's fast mode.
template <int CT, int LT, bool FAST = false>
__global__ void __launch_bounds__(32 * CH2_MAXW) k_chain_direct2(Ctx x) {
	const Cfg &g = x.cfg;
	const int K = g.K;
	B200S_DYN_SHARED
	constexpr int BPW = 32 / CT; // blocks per warp
	constexpr int D = LT + 1;    // wavefront skew between consecutive blocks (bins)
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nWarps = blockDim.x >> 5;
	const int j = lane / CT, c = lane % CT; // block within the warp, channel
	const int s = stream_at(x, x.sBase + blockIdx.x);
	const Call cl = x.call[s];
	if (cl.nFrames == 0 || cl.mapped) return; // (streams with a frequency map or formants: the mapped path)
	if (cl.hasRandom && x.randomPathOn) return; // a block beyond 2x stretch draws random time factors: k_prep + k_chain take the stream
	Chain2Sync &SY = *(Chain2Sync *)dyn_smem;
	Chain2Tiles<CT> &U = ((Chain2Tiles<CT> *)((char *)dyn_smem + 64))[warp];
	Chain2Tiles<CT> &UN = ((Chain2Tiles<CT> *)((char *)dyn_smem + 64))[warp + 1 < nWarps ? warp + 1 : warp]; // successor's tiles
	const int fillI = (lane & 3) + 4 * (lane >> 4), fillF = (lane >> 2) & 3; // chunk fill: bin offset, row within a group of 4
	const float2 rot0 = x.rot0, rotStep = x.rotStep;
	const int perRound = BPW * nWarps;

	for (int base = 0; base < cl.nFrames; base += perRound) {
		if (base > 0) __syncthreads(); // previous round complete (its Y / energy rows are this round's predecessor)
		if (threadIdx.x < CH2_MAXW) SY.done[threadIdx.x] = 0;
		__syncthreads();
		const int wBase = base + warp * BPW; // first block of this warp
		if (wBase >= cl.nFrames) continue;   // (uniform per warp; the barriers above are reached by every warp each round)
		const int f = wBase + j;
		const bool active = f < cl.nFrames;
		const Frame fr = x.frames[(size_t)s * x.maxFrames + (active ? f : wBase)];
		const bool rotOn = fr.flags & FR_NEW_SPECTRUM;
		const int nAct = min(BPW, cl.nFrames - wBase);
		const bool hasSucc = warp + 1 < nWarps && wBase + BPW < cl.nFrames; // a later warp consumes this warp's last block
		const bool fromPred = warp > 0;                                       // predecessor block lives in warp-1 (same round)
		// Prediction::energy must reach HBM for the block that the next round / the next call continues from
		const bool carryE = active && (f == cl.nFrames - 1 || (j == BPW - 1 && !hasSucc));
		const float tf = fmaxf(fr.timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH); // :638
		const float longTf = fmul((float)LT, tf);
		const bool farAny = __any_sync(0xffffffffu, active && longTf > (float)(CH2_RING - CHAIN_CH - 3));
		const float2 *prevOut = nullptr;
		const float *prevE = nullptr;
		if (!fromPred) {
			prevOut = base == 0 ? x.stOut + ((size_t)s * CT + c) * K : x.Y + coef_off(x, s, base - 1, c);
			prevE = base == 0 ? x.stPredE + ((size_t)s * CT + c) * K : x.cE + coef_off(x, s, base - 1, c);
		}
		const float2 *myIn = spec_slot(x, s, fr.inSlot, c);
		float *myE = x.cE + coef_off(x, s, active ? f : wBase, c);
		U.rowIn[lane] = myIn;
		U.rowPv[lane] = spec_slot(x, s, fr.prevSlot, c);
		U.rowY[lane] = x.Y + coef_off(x, s, active ? f : wBase, c);
		__syncwarp();
		// register FIFOs; at the start of a step (q = prelim bin, b = q - L = final bin):
		//   pre/eF/t2F/inF[i] <-> prelim output / energy / long twist / input at bin b+i
		//   oh[i] <-> final output at bin b-1-i;   t1P <-> short twist at bin b
		float2 oh[LT], pre[LT], t2F[LT], inF[LT], t1P, lastFinal;
		float eF[LT], lastE;
#pragma unroll
		for (int i = 0; i < LT; ++i) {
			oh[i] = pre[i] = t2F[i] = inF[i] = make_float2(0.f, 0.f);
			eF[i] = 0.f;
		}
		t1P = lastFinal = make_float2(0.f, 0.f);
		lastE = 0.f;
		float2 rotq = rotOn ? rot0 : make_float2(1.f, 0.f); // rot[q] of the reference's float recurrence (:647-655)
		const float2 rotS = rotOn ? rotStep : make_float2(1.f, 0.f);
		const int steps = K + LT + D * (nAct - 1);
		// first chunk start from which every lane (all active) has q - L*tf - 1 >= 0 and b = q - L >= L: q >= D*(BPW-1) + 2L + ceil(max L*tf) + 2
		int interiorFrom = steps;
		if (nAct == BPW) {
			float mx = longTf;
			for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
			interiorFrom = D * (BPW - 1) + 2 * LT + (int)ceilf(mx) + 2;
		}
		int chunk = 0;
		for (int k0 = 0; k0 < steps; k0 += CHAIN_CH, ++chunk) {
			// ---------------- flow control with the neighbouring warps ----------------
			if (fromPred) { // bins k0 .. k0+7 of the predecessor block are final once warp-1 finished its step k0+7 + D*(BPW-1) + LT
				const int need = min((k0 + CHAIN_CH - 1 + D * (BPW - 1) + LT) / CHAIN_CH + 1, (K + LT + D * (BPW - 1) + CHAIN_CH - 1) / CHAIN_CH);
				while (ld_volatile_shared(&SY.done[warp - 1]) < need) spin_pause();
			}
			if (hasSucc) { // do not run more than the hand-off ring ahead of the consumer
				const int over = k0 + CHAIN_CH - 1 - D * (BPW - 1) - LT - CH2_HO; // last bin whose ring slot this chunk overwrites
				if (over >= 0) { // the consumer reads bin q in its step q: its chunk over/8 must be complete
					const int need = min(over / CHAIN_CH + 1, (K + LT + CHAIN_CH - 1) / CHAIN_CH);
					while (ld_volatile_shared(&SY.done[warp + 1]) < need) spin_pause();
				}
			}
			fence_block();
			// ---------------- stage the chunk: 8 new bins per row ----------------
#pragma unroll
			for (int it = 0; it < 8; ++it) {
				const int fl = fillF + 4 * it;
				const int q = k0 + fillI - D * (fl / CT);
				if (wBase + fl / CT < cl.nFrames && (unsigned)q < (unsigned)K) {
					cp_async8(&U.in[q & (CH2_RING - 1)][fl], U.rowIn[fl] + q);
					cp_async8(&U.pvy[fillI][fl], U.rowPv[fl] + q);
				}
			}
			if (!fromPred && lane < CHAIN_CH * CT) { // predecessor from HBM (last call's state / previous round)
				const int qq = k0 + lane / CT;
				if (qq < K) {
					cp_async8(&U.hoOut[c][qq & (CH2_HO - 1)], prevOut + qq);
					cp_async4(&U.hoE[c][qq & (CH2_HO - 1)], prevE + qq);
				}
			}
			cp_async_wait_all();
			__syncwarp();
			// ---------------- CHAIN_CH steps ----------------
			// INTERIOR (about nine chunks in ten of a full warp): every lane is active and all its bins and interpolation points
			// lie inside [L, K) for the whole chunk, so the edge masks below are identities and are compiled out
			auto step = [&](const int i, auto farTag, auto intTag) {
				constexpr bool FAR = decltype(farTag)::value, INTERIOR = decltype(intTag)::value;
				const int q = k0 + i - D * j;
				const int b = q - LT;
				const bool qIn = INTERIOR || (active && (unsigned)q < (unsigned)K);
				const bool bIn = INTERIOR || (active && (unsigned)b < (unsigned)K);
				// the twists need input interpolated at q - L*tf and (b+1) - tf  (:750,:757)
				const float i2 = fsub((float)q, longTf);
				const int l2 = (int)floorf(i2);
				const float f2 = fsub(i2, (float)l2);
				const float i1 = fsub((float)(b + 1), tf);
				const int l1 = (int)floorf(i1);
				const float f1 = fsub(i1, (float)l1);
				// previous block's final output / energy at bin q: finalised by lane-CT in the last step
				float2 ro;
				ro.x = __shfl_up_sync(0xffffffffu, lastFinal.x, CT);
				ro.y = __shfl_up_sync(0xffffffffu, lastFinal.y, CT);
				float re = __shfl_up_sync(0xffffffffu, lastE, CT);
				{
					const int hq = (k0 + i) & (CH2_HO - 1);
					const float2 p0 = U.hoOut[c][hq];
					const float p0e = U.hoE[c][hq];
					ro = make_float2(j == 0 ? p0.x : ro.x, j == 0 ? p0.y : ro.y);
					re = j == 0 ? p0e : re;
				}
				const float2 inq = U.in[q & (CH2_RING - 1)][lane];
				float2 pv = U.pvy[i][lane];
				float2 lo2, hi2, lo1, hi1;
				if constexpr (!FAR) {
					lo2 = sel2b(INTERIOR || l2 >= 0, U.in[l2 & (CH2_RING - 1)][lane]);
					hi2 = sel2b(INTERIOR || l2 >= -1, U.in[(l2 + 1) & (CH2_RING - 1)][lane]);
					lo1 = sel2b(INTERIOR || l1 >= 0, U.in[l1 & (CH2_RING - 1)][lane]);
					hi1 = sel2b(INTERIOR || l1 >= -1, U.in[(l1 + 1) & (CH2_RING - 1)][lane]);
				} else { // extreme stretch (> 2x): gather straight from the spectrum row
					lo2 = spec_at(myIn, l2, K);
					hi2 = spec_at(myIn, l2 + 1, K);
					lo1 = spec_at(myIn, l1, K);
					hi1 = spec_at(myIn, l1 + 1, K);
				}
				pv = FAST ? fmul_f(pv, rotq) : xmul(pv, rotq); // :653-654 rotate Band::output and Band::prevInput by one interval
				ro = FAST ? fmul_f(ro, rotq) : xmul(ro, rotq);
				const float e = FAST ? ffma(inq.x, inq.x, inq.y * inq.y) : xnorm(inq); // :679 (identity map: energy = |input|^2)
				const float2 ph0 = FAST ? fmul_f(ro, fmulc_f(inq, pv)) : xmul(ro, xmulc(inq, pv)); // :714-715
				const float den = fadd(fmaxf(re, e), B200S_NOISE_FLOOR);
				const float rden = FAST ? rcp_fast(den) : 0.f;
				const float2 newPre = sel2b(qIn, FAST ? make_float2(ph0.x * rden, ph0.y * rden) : make_float2(fdivq(ph0.x, den), fdivq(ph0.y, den))); // :716
				const float newE = qIn ? e : 0.f;
				const float2 newIn = sel2b(qIn, inq);
				const float2 newT2 = sel2b(qIn, FAST ? fmulc_f(inq, flerp_f(lo2, hi2, f2)) : xmulc(inq, xlerp2(lo2, hi2, f2))); // long twist at q (:758)
				// short twist at b+1 (:751,:771): Prediction::input[b+1] is inF[1] before the shift
				const float2 in1 = LT > 1 ? inF[LT > 1 ? 1 : 0] : newIn;
				const float2 t1N = FAST ? fmulc_f(in1, flerp_f(lo1, hi1, f1)) : xmulc(in1, xlerp2(lo1, hi1, f1));
				{
					const float2 rn = xmul(rotq, rotS);
					rotq = make_float2((INTERIOR || q >= 0) ? rn.x : rotq.x, (INTERIOR || q >= 0) ? rn.y : rotq.y);
				}
				// ---- FIFO rotation (pure renaming after unrolling): what falls out belongs to bin b
				const float eB = eF[0];
				const float2 t2B = t2F[0], inB = inF[0];
#pragma unroll
				for (int u = 0; u + 1 < LT; ++u) {
					pre[u] = pre[u + 1];
					eF[u] = eF[u + 1];
					t2F[u] = t2F[u + 1];
					inF[u] = inF[u + 1];
				}
				pre[LT - 1] = newPre;
				eF[LT - 1] = newE;
				t2F[LT - 1] = newT2;
				inF[LT - 1] = newIn;
				// ---- main prediction at bin b (:727-800), this lane's channel as if it were the loudest
				float2 phase = make_float2(0.f, 0.f);
				if constexpr (FAST) { // the term that closes the recurrence (the previous bin's final) is added last
					const float2 a = sel2b(INTERIOR || b >= LT, fmul_f(oh[LT - 1], t2B)), bb = sel2b(INTERIOR || b < K - 1, fmulc_f(pre[0], t1N));
					const float2 cc = sel2b(INTERIOR || b < K - LT, fmulc_f(pre[LT - 1], t2F[LT - 1])), dd = sel2b(INTERIOR || b > 0, fmul_f(oh[0], t1P));
					phase = make_float2(((a.x + bb.x) + cc.x) + dd.x, ((a.y + bb.y) + cc.y) + dd.y);
				} else {
					phase = xadd(phase, sel2b(INTERIOR || b > 0, xmul(oh[0], t1P)));               // :754
					phase = xadd(phase, sel2b(INTERIOR || b >= LT, xmul(oh[LT - 1], t2B)));        // :761
					phase = xadd(phase, sel2b(INTERIOR || b < K - 1, xmulc(pre[0], t1N)));         // :774
					phase = xadd(phase, sel2b(INTERIOR || b < K - LT, xmulc(pre[LT - 1], t2F[LT - 1]))); // :784
				}
				const float2 outOwn = FAST ? make_output_fast(phase, eB, inB) : make_output_q(phase, eB, inB); // :788
				float2 oc = outOwn;
				if (CT > 1) { // the loudest channel wins (:729-737, first one on ties); the other is locked to it (:791-799)
					const float eO = __shfl_xor_sync(0xffffffffu, eB, 1);
					const bool isMax = c == 0 ? !(eO > eB) : (eB > eO);
					float2 outM, pinM;
					outM.x = __shfl_xor_sync(0xffffffffu, outOwn.x, 1);
					outM.y = __shfl_xor_sync(0xffffffffu, outOwn.y, 1);
					pinM.x = __shfl_xor_sync(0xffffffffu, inB.x, 1);
					pinM.y = __shfl_xor_sync(0xffffffffu, inB.y, 1);
					const float2 cph = FAST ? fmul_f(outM, fmulc_f(inB, pinM)) : xmul(outM, xmulc(inB, pinM)); // :796-797
					const float2 other = FAST ? make_output_fast(cph, eB, inB) : make_output_q(cph, eB, inB);
					oc = make_float2(isMax ? outOwn.x : other.x, isMax ? outOwn.y : other.y);
				}
				// unconditional: out-of-range steps only produce values that every consumer masks
#pragma unroll
				for (int u = LT - 1; u > 0; --u) oh[u] = oh[u - 1];
				oh[0] = oc;
				lastFinal = oc;
				lastE = eB;
				t1P = t1N;
				if (carryE && bIn) myE[b] = eB;
				U.pvy[i][lane] = oc;
				if (hasSucc && j == BPW - 1 && bIn) { // hand over to the first block of the next warp
					UN.hoOut[c][b & (CH2_HO - 1)] = oc;
					UN.hoE[c][b & (CH2_HO - 1)] = eB;
				}
			};
			if (!farAny && k0 >= interiorFrom && k0 + CHAIN_CH <= K) {
#pragma unroll
				for (int i = 0; i < CHAIN_CH; ++i) step(i, std::false_type{}, std::true_type{});
			} else if (!farAny) {
#pragma unroll
				for (int i = 0; i < CHAIN_CH; ++i) step(i, std::false_type{}, std::false_type{});
			} else {
#pragma unroll 1
				for (int i = 0; i < CHAIN_CH; ++i) step(i, std::true_type{}, std::false_type{});
			}
			__syncwarp();
			// ---------------- write the chunk's finals back, 64 B per row ----------------
#pragma unroll
			for (int it = 0; it < 8; ++it) {
				const int fl = fillF + 4 * it;
				const int b = k0 + fillI - D * (fl / CT) - LT;
				if (wBase + fl / CT < cl.nFrames && (unsigned)b < (unsigned)K) U.rowY[fl][b] = U.pvy[fillI][fl];
			}
			fence_block(); // hand-off ring stores (and Y) before the progress counter
			__syncwarp();
			if (lane == 0) st_volatile_shared(&SY.done[warp], chunk + 1);
		}
	}
}

static inline size_t smem_chain2(int C, int nWarps) {
	return 64 + (size_t)nWarps * (C == 1 ? sizeof(Chain2Tiles<1>) : sizeof(Chain2Tiles<2>));
}

} // namespace b200s
