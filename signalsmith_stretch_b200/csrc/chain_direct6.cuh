// chain_direct6.cuh -- k_chain_direct6: the packed frame wavefront of k_chain_direct4 (reference :722-804) on an
// instruction diet, for stereo streams (DUAL = false) and for PAIRS OF MONO STREAMS (DUAL = true).  Selectable
// (b200s_set_tuning key 0 = 6, key 5 = 1 for the mono pairs); generation 4 / k_chain_direct2 stay the defaults because this
// kernel is no faster -- which is its result: see the end of this comment and DESIGN.md 3.8.
//
// k_chain_direct4 spends 186 SASS instructions per step on its interior path, of which only ~55 % are arithmetic
// (cuobjdump, round 2): 35 MOVs (its five-entry register FIFOs do not rotate by renaming in a loop unrolled by four),
// 6 SHFL + 6 FSEL for the lane-to-lane hand-off (lane 0 takes its predecessor from shared memory instead), 15 shared-
// memory instructions.  Here
//   * every FIFO has at most L entries and every value dies before its slot is rewritten, so for L = 4 (both presets)
//     the loop unrolled by four rotates them by pure renaming: the long vertical twist (:758) is formed ONE BIN BEHIND
//     the preliminary prediction and multiplied into its two products at once (out(b) * T2(b+L), :761, enters a product /
//     accumulator FIFO when out(b) is finalised; pre(b+L) * conj(T2(b+L)), :784, is consumed in the same step), the short
//     twist (:751) TWO bins behind (its :774 product runs one step ahead);
//   * Prediction::input / energy of bin b are re-read from the rolling spectrum window (one LDS.128) instead of
//     travelling through five-entry FIFOs;
//   * the final output of a step goes to the tile slot it is written back from anyway, and the NEXT lane reads it from
//     there ([lane-1], one LDS.128): no shuffles, no selects -- lane 0's predecessor block sits in the padding slot
//     before each tile row, put there by the chunk fill; Prediction::energy travels the same way through a 16-bin ring;
//   * everything a step reads from behind its prelim bin is loaded one step ahead.
// Arithmetic, masks and operation order are those of k_chain_direct4 (exact mode: bit-identical, tested under
// emulation and on the GPU); the fast mode additionally uses energy + noiseFloor for |input|^2 + noiseFloor in
// makeOutput (:599; on this path Prediction::energy IS |input|^2, :679,:708).
//
// DUAL: a mono batch has no second channel to pack -- but it has a second STREAM: lane j runs block j of stream 2p in
// the low halves of its f2 register pairs and block j of stream 2p+1 in the high halves; the halves never meet (no
// loudest-channel choice, no phase lock, each half its own makeOutput :788).  The two streams must walk the same
// schedule in this call (dual_pair_ok, chain_direct2.cuh); pairs that do not, and the odd stream of an odd batch, run
// alone through the same kernel, the stream in both halves.  Spectra stay planar (mono analysis is unchanged): the
// chunk fill copies the two streams' bins into one 16-byte tile slot {A.re, B.re, A.im, B.im}, the layout of the stereo path.
//
// 166-172 instead of 186 instructions per step.  The PROBE template parameter (profiling builds, -DB200S_CHAIN_PROBES)
// removes parts of the step (the SFU instructions, the second makeOutput, the interpolation loads, the lane hand-off, the
// spectrum fetches, the write-back) to measure what the kernel's time goes with.
#pragma once
#include "chain_direct2.cuh"
#include "chain_direct4.cuh"

namespace b200s {

#define CH6_ER 16                // bins of the Prediction::energy ring (>= G + 1 and >= 2 chunks for lane 0's pads)
#define CH6_FAR (CH4_FAR - 1)    // the twists are formed one bin later than in k_chain_direct4: one bin less reach

struct Chain6Tiles {
	float4 in[CH3_RING][CH3_RS];     // rolling window of each block's input spectrum, [bin & 31][lane]
	float4 lead[2];                  // lead[1] is the "lane -1" slot of pvy[0][0]
	float4 pvy[2][CHAIN_CH][CH3_RS]; // previous-input spectrum at the chunk's bins, overwritten by the finals of the same step;
	                                 // slot [..][i][-1] (= the padding of the row before): lane 0's predecessor for the NEXT step
	float2 eLead[2];                 // eLead[1] is the "lane -1" slot of eR[0]
	float2 eR[CH6_ER][CH3_RS];       // Prediction::energy at bin q of each block, [bin & 15][lane]; [..][-1]: lane 0's predecessor
	const void *rowIn[2][32], *rowPv[2][32];
};

template <bool DUAL>
__device__ __forceinline__ c2 ld_t(const float4 *p) { return ld_c2s(p); } // tile slot {re0, re1, im0, im1} (halves: channels, or streams A / B)
template <bool DUAL>
__device__ __forceinline__ float4 pack_t(c2 v) { return make_float4(f2_lo(v.re), f2_hi(v.re), f2_lo(v.im), f2_hi(v.im)); }
__device__ __forceinline__ f2 ld_f2s(const float2 *p) {
	const float2 v = *p;
	return f2_make(v.x, v.y);
}
// Prediction::makeOutput (:596-603) where Prediction::energy is |input|^2 (plain path): the weak branch's norm is energy + noiseFloor
// (sqrtE = sqrt(energy), taken one step ahead of its use: only the rsqrt of the phase's norm sits on the recurrence)
template <int PROBE = 0>
__device__ __forceinline__ float2 make_output_fast_e(float2 phase, float energy, float sqrtE, float2 input) {
	const float pn = ffma(phase.x, phase.x, phase.y * phase.y);
	const bool weak = pn <= B200S_NOISE_FLOOR;
	const float g = PROBE == 1 ? ffma(energy, 0.5f, weak ? energy + B200S_NOISE_FLOOR : pn) : sqrtE * rsqrt_fast(weak ? energy + B200S_NOISE_FLOOR : pn);
	return make_float2((weak ? input.x : phase.x) * g, (weak ? input.y : phase.y) * g);
}

// PROBE (profiling builds only, results are WRONG): ablations that time what a part of the step costs --
//   1: no SFU (rcp / rsqrt / sqrt replaced by one FMA)   2: the locked channel copies the leader (no second makeOutput)
//   3: no interpolation loads (the twists use the prelim bin's input)   4: no lane-to-lane hand-off (every lane re-reads its own slots)
//   5: the previous-input spectrum is not fetched (half the reads)   6: the finals are not written back   7: 5 + 6 + no input fetch either
template <int LT, bool FAST, bool DUAL, int PROBE = 0>
__global__ void __launch_bounds__(32) k_chain_direct6(Ctx x) {
	const Cfg &g = x.cfg;
	const int K = g.K;
	B200S_DYN_SHARED
	const int lane = threadIdx.x & 31;
	// DUAL: CTA p owns the streams s0, s1 at positions i0 = sBase + 2p and i0 + 1 (stream_at: a listed call pairs its list
	// entries, wherever their streams are).  When they share their schedule (dual_pair_ok) they run packed, stream s0 in the
	// low halves and s1 in the high halves; otherwise (and for the odd stream of an odd batch) each runs alone with itself in
	// both halves, one after the other -- every mono stream goes through the same arithmetic.
	const int i0 = x.sBase + (DUAL ? 2 : 1) * blockIdx.x;
	const bool hasPartner = DUAL && i0 + 1 < x.sBase + x.sCount;
	const int s0 = stream_at(x, i0), s1 = hasPartner ? stream_at(x, i0 + 1) : s0;
	const bool pairOk = DUAL && dual_pair_ok(x, i0, s0, s1, lane);
	const int nPass = (hasPartner && !pairOk) ? 2 : 1;
	constexpr int G = LT + 2; // lane skew in bins
	static_assert(G + 1 <= CH6_ER && 2 * CHAIN_CH <= CH6_ER, "energy ring too short");
	Chain6Tiles &U = *(Chain6Tiles *)dyn_smem;
	// chunk fill: lane -> (bin offset, row within a group of 4); a quarter-warp covers 4 bins (64 B) of 2 rows
	const int fillI = (lane & 3) | (((lane >> 3) & 1) << 2), fillF = ((lane >> 2) & 1) | (((lane >> 4) & 1) << 1);
	const float2 rot0 = x.rot0, rotStep = x.rotStep;
	const float one = x.one; // unused by the f2 arithmetic (see padd / psub)
	const f2 z2 = f2_make(0.f, 0.f);
	const c2 zc = c2{z2, z2};

	for (int pass = 0; pass < nPass; ++pass) {
	const int s = pass ? s1 : s0;
	const Call cl = x.call[s];
	if (cl.nFrames == 0 || cl.mapped) continue; // (streams with a frequency map or formants: the mapped path)
	if (cl.hasRandom && x.randomPathOn) continue; // a block beyond 2x stretch draws random time factors: k_prep + k_chain take the stream
	const int sH[2] = {s, pairOk ? s1 : s};
	for (int base = 0; base < cl.nFrames; base += 32) {
		__syncwarp();
		const int f = base + lane;
		const bool active = f < cl.nFrames;
		const Frame fr = x.frames[(size_t)s * x.maxFrames + (active ? f : base)];
		const bool rotOn = fr.flags & FR_NEW_SPECTRUM;
		const int nAct = min(32, cl.nFrames - base);
		const float tf = fmaxf(fr.timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH); // :638
		const float longTf = fmul((float)LT, tf);
		const bool farAny = __any_sync(0xffffffffu, active && longTf > (float)CH6_FAR);
		// lane 0's predecessor block: the state rows (first group of the call) or the last block of the previous group.
		// half h = channel h (stereo) or stream sH[h] (DUAL); rows are planar float2.  Pointer of half 0 + distance to half 1
		// (not arrays: indexed by a run-time half they would live in local memory)
		const float2 *prevOut0;
		const float *prevE0; // base == 0 only; later groups recompute the energy from the predecessor's input row, see the fill
		ptrdiff_t prevOutD, prevED;
		if constexpr (DUAL) {
			prevOut0 = base == 0 ? x.stOut + (size_t)sH[0] * K : x.Y + coef_off(x, sH[0], base - 1, 0);
			prevOutD = (base == 0 ? x.stOut + (size_t)sH[1] * K : x.Y + coef_off(x, sH[1], base - 1, 0)) - prevOut0;
			prevE0 = x.stPredE + (size_t)sH[0] * K;
			prevED = (ptrdiff_t)(sH[1] - sH[0]) * K;
		} else {
			prevOut0 = base == 0 ? x.stOut + (size_t)s * 2 * K : x.Y + coef_off(x, s, base - 1, 0);
			prevOutD = K; // the channel rows of a block are adjacent (state rows and Y rows alike)
			prevE0 = x.stPredE + (size_t)s * 2 * K;
			prevED = K;
		}
		// Prediction::energy of a block on this path is |input|^2 of its own spectrum (:679,:708): the chain never stores
		// it -- the next group recomputes it from the predecessor's input row, k_commit from the final input spectrum
		// (DUAL: k_commit of the mono path reads the last block's row of cE, written below)
		const int prevSlotIn = base == 0 ? 0 : x.frames[(size_t)s * x.maxFrames + base - 1].inSlot;
		const float4 *prevInIl = nullptr, *myInIl = nullptr;
		const float2 *prevInD0 = nullptr, *myInD[2] = {nullptr, nullptr};
		ptrdiff_t prevInDD = 0;
		float2 *yBaseA = nullptr, *yBaseB = nullptr; // Band::output rows of block base (+ r: r rows on), the two halves (channels, or streams A / B)
		float *eRowD[2] = {nullptr, nullptr};
		if constexpr (DUAL) {
			if (base > 0) {
				prevInD0 = spec_slot(x, sH[0], prevSlotIn, 0);
				prevInDD = spec_slot(x, sH[1], prevSlotIn, 0) - prevInD0;
			}
#pragma unroll
			for (int h = 0; h < 2; ++h) {
				myInD[h] = spec_slot(x, sH[h], fr.inSlot, 0);
				U.rowIn[h][lane] = myInD[h];
				U.rowPv[h][lane] = spec_slot(x, sH[h], fr.prevSlot, 0);
				eRowD[h] = x.cE + coef_off(x, sH[h], active ? f : base, 0);
			}
			yBaseA = x.Y + coef_off(x, sH[0], base, 0); // mono: one row per block
			yBaseB = x.Y + coef_off(x, sH[1], base, 0);
		} else {
			prevInIl = base == 0 ? nullptr : il_row(x, s, prevSlotIn);
			myInIl = il_row(x, s, fr.inSlot);
			U.rowIn[0][lane] = myInIl;
			U.rowPv[0][lane] = il_row(x, s, fr.prevSlot);
			yBaseA = x.Y + coef_off(x, s, base, 0); // stereo: two rows per block, channel 1 after channel 0
			yBaseB = yBaseA + K;
		}
		const bool lastFrame = DUAL && active && f == cl.nFrames - 1; // its Prediction::energy is the state the next call continues from
		__syncwarp();
		// Register FIFOs (pairs {channel 0, channel 1} or {stream A, stream B}).  Every value lives FEWER than L steps (or its
		// successor in the same slot depends on its last use), so for L = 4 the loop unrolled by four rotates them by pure
		// renaming.  At the start of a step (q = prelim bin, b = q - L - 1 = final bin):
		//   PR[j] <-> prelim output at bin q-j           T1[j] <-> short twist (:751) at bin q-D1-j      (j >= 1; entry 0: this step's)
		//   RF[j] <-> out(b+j-L) * longTwist(b+j) (:761), formed when out(b+j-L) was finalised       (exact mode)
		//   AC[j] <-> the part of the phase sum of bin b+j that does not depend on out(b+j-1)          (fast mode)
		//   P3c   <-> prelim(b+1) * conj(shortTwist(b+1)) (:774), formed one step ahead (A = 1)        (exact mode)
		//   oc1   <-> final output at bin b-1
		constexpr int D1 = LT >= 3 ? 2 : 1; // the short twist is formed at bin q-D1, the long twist (:758) at bin q-1
		constexpr int A = LT >= 3 ? 1 : 0;  // steps by which the :774 term runs ahead
		constexpr int NPR = (LT - A > 1 ? LT - A : 1) + 1, NT1 = LT + 2 - D1;
		c2 PR[NPR], T1[NT1], RF[LT], P3c = zc, oc1 = zc;
#pragma unroll
		for (int i = 0; i < NPR; ++i) PR[i] = zc;
#pragma unroll
		for (int i = 0; i < NT1; ++i) T1[i] = zc;
#pragma unroll
		for (int i = 0; i < LT; ++i) RF[i] = zc;
		c2 inP = zc, inP2 = zc; // Prediction::input at bins q-1, q-2 (masked)
		float2 rotq = rotOn ? rot0 : make_float2(1.f, 0.f); // rot[q] by the reference's float recurrence (:647-655)
		const float2 rotS = rotOn ? rotStep : make_float2(1.f, 0.f);
		const int steps = K + LT + 1 + G * (nAct - 1);
		// first chunk start from which every ACTIVE lane has (q-1) - L*tf - 1 >= 0, (q-1) - tf - 1 >= 0 and b = q - L - 1 >= L
		// (inactive lanes only produce values nobody consumes)
		int interiorFrom;
		{
			float mx = active ? longTf : 0.f;
			for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
			interiorFrom = G * (nAct - 1) + 2 * LT + (int)ceilf(mx) + 4;
		}
		// asynchronous fill of the chunk starting at kf into buffer `buf`: 8 new bins per block, both halves per tile slot.
		// The ring slots it writes (the 8 bins after the chunk's own 8, per lane) are disjoint from what the chunk in
		// progress reads (at most CH6_FAR + 3 bins behind its own 8: 8 + 8 + CH6_FAR + 3 <= CH3_RING).
		// Lane 0's predecessor: finals of bins kf+1 .. kf+8 into the padding slots before rows [buf][0..7] of pvy (step i
		// reads, for step i+1, the slot before its own row), energies of the same bins into the padding before rows
		// [bin & 15] of eR (every step reads the energy of the NEXT step's bin).  None of these slots is read by the chunk in
		// progress (other buffer / other half of the ring).
		auto fill = [&](int kf, int buf) {
			if constexpr (DUAL) {
				const float2 *rIn[2][8], *rPv[2][8];
#pragma unroll
				for (int it = 0; it < 8; ++it) {
#pragma unroll
					for (int h = 0; h < 2; ++h) {
						rIn[h][it] = (const float2 *)U.rowIn[h][fillF + 4 * it];
						rPv[h][it] = (const float2 *)U.rowPv[h][fillF + 4 * it];
					}
				}
#pragma unroll
				for (int it = 0; it < 8; ++it) {
					const int fl = fillF + 4 * it;
					const int q = kf + fillI - G * fl;
					if (fl < nAct && (unsigned)q < (unsigned)K) {
						// slot = {A.re, B.re, A.im, B.im}: the layout the packed arithmetic wants (as the interleaved stereo spectra),
						// so the two 8-byte bins go in as four 4-byte copies
#pragma unroll
						for (int h = 0; h < 2; ++h) {
							float *dIn = (float *)&U.in[q & (CH3_RING - 1)][fl] + h, *dPv = (float *)&U.pvy[buf][fillI][fl] + h;
							const float *sIn = (const float *)(rIn[h][it] + q), *sPv = (const float *)(rPv[h][it] + q);
							cp_async4(dIn, sIn);
							cp_async4(dIn + 2, sIn + 1);
							cp_async4(dPv, sPv);
							cp_async4(dPv + 2, sPv + 1);
						}
					}
				}
			} else {
				const float4 *rIn[8], *rPv[8];
#pragma unroll
				for (int it = 0; it < 8; ++it) {
					rIn[it] = (const float4 *)U.rowIn[0][fillF + 4 * it];
					rPv[it] = (const float4 *)U.rowPv[0][fillF + 4 * it];
				}
#pragma unroll
				for (int it = 0; it < 8; ++it) {
					const int fl = fillF + 4 * it;
					const int q = kf + fillI - G * fl;
					if (fl < nAct && (unsigned)q < (unsigned)K) {
						if (PROBE != 7) cp_async16(&U.in[q & (CH3_RING - 1)][fl], rIn[it] + q);
						if (PROBE != 5 && PROBE != 7) cp_async16(&U.pvy[buf][fillI][fl], rPv[it] + q);
					}
				}
			}
			{ // lane 0's predecessor finals: 4 floats per bin, one 4-byte copy per lane
				const int i = lane >> 2, comp = lane & 3, qq = kf + 1 + i;
				const int h = comp & 1, part = comp >> 1; // tile slot component {re0, re1, im0, im1} -> (half, re / im)
				if (qq < K) cp_async4((float *)(&U.pvy[buf][i][0] - 1) + comp, (const float *)(prevOut0 + h * prevOutD + qq) + part);
			}
			if (lane < 2 * CHAIN_CH) { // ... and its Prediction::energy {half 0, half 1}, bins kf+1 .. kf+8 (read one step ahead, too)
				const int qq = kf + 1 + (lane >> 1), h = lane & 1;
				float *pad = (float *)(&U.eR[qq & (CH6_ER - 1)][0] - 1) + h;
				if (qq < K) {
					if (base == 0) {
						cp_async4(pad, prevE0 + h * prevED + qq);
					} else if constexpr (DUAL) {
						*pad = xnorm((prevInD0 + h * prevInDD)[qq]);
					} else {
						const float4 v = prevInIl[qq];
						*pad = h ? xnorm(make_float2(v.y, v.w)) : xnorm(make_float2(v.x, v.z));
					}
				}
			}
		};
		fill(0, 0);
		// final output of the previous block at the prelim bin of the NEXT step (read from the tile at the end of each step);
		// for the first step: lane 0's predecessor at bin 0, nothing for the others (their q is negative)
		c2 roN = zc;
		f2 cRe = z2; // ... and its Prediction::energy at that bin
		if (lane == 0) {
			const float2 a = prevOut0[0], bb = prevOut0[prevOutD];
			roN = c2{f2_make(a.x, bb.x), f2_make(a.y, bb.y)};
			if (base == 0) {
				cRe = f2_make(prevE0[0], prevE0[prevED]);
			} else if constexpr (DUAL) {
				cRe = f2_make(xnorm(prevInD0[0]), xnorm(prevInD0[prevInDD]));
			} else {
				const float4 v = prevInIl[0];
				cRe = f2_make(xnorm(make_float2(v.x, v.z)), xnorm(make_float2(v.y, v.w)));
			}
		}
		// Everything a step reads from BEHIND its prelim bin -- the interpolation points of the two twists, Prediction::input of
		// the final bin, the predecessor's energy -- is loaded ONE STEP AHEAD into these registers, so that the shared-memory
		// latency (and the float -> int conversions in front of the addresses) overlaps the previous step's arithmetic instead
		// of stalling this one.
		c2 cLo2 = zc, cHi2 = zc, cLo1 = zc, cHi1 = zc, cInB = zc;
		f2 cEB = z2, cSqB = z2; // Prediction::energy at bin b (= |input|^2 on this path, :679,:708) and, fast mode, its square root
		float cF2s = 0.f, cF1s = 0.f;
		auto preload = [&](const int qn, auto farTag, auto intTag, bool withRe) {
			constexpr bool FAR = decltype(farTag)::value, INTERIOR = decltype(intTag)::value;
			const int bn = qn - LT - 1, p2 = qn - 1, p1 = qn - D1;
			// the long twist of bin p2 needs input interpolated at p2 - L*tf, the short twist of bin p1 at p1 - tf  (:750,:757)
			const float pf2 = (float)p2;
			const float pf1 = D1 == 1 ? pf2 : (float)p1;
			const float i2 = fsub(pf2, longTf);
			const int l2 = (int)floorf(i2);
			cF2s = fsub(i2, (float)l2);
			const float i1 = fsub(pf1, tf);
			const int l1 = (int)floorf(i1);
			cF1s = fsub(i1, (float)l1);
			if (withRe) cRe = ld_f2s(&U.eR[qn & (CH6_ER - 1)][0] + lane - (PROBE == 4 ? 0 : 1));
			cInB = sel_c2(INTERIOR || (active && (unsigned)bn < (unsigned)K), ld_t<DUAL>(&U.in[bn & (CH3_RING - 1)][lane])); // Prediction::input at bin bn
			if constexpr (FAST) {
				cEB = fnorm2(cInB);
				cSqB = PROBE == 1 ? cEB : f2_make(sqrt_fast(f2_lo(cEB)), sqrt_fast(f2_hi(cEB)));
			} else {
				cEB = xnorm2(cInB, one);
			}
			if constexpr (PROBE == 3) {
				cLo2 = cHi2 = cLo1 = cHi1 = cInB;
			} else if constexpr (!FAR) {
				cLo2 = sel_c2(INTERIOR || l2 >= 0, ld_t<DUAL>(&U.in[l2 & (CH3_RING - 1)][lane]));
				cHi2 = sel_c2(INTERIOR || l2 >= -1, ld_t<DUAL>(&U.in[(l2 + 1) & (CH3_RING - 1)][lane]));
				cLo1 = sel_c2(INTERIOR || l1 >= 0, ld_t<DUAL>(&U.in[l1 & (CH3_RING - 1)][lane]));
				cHi1 = sel_c2(INTERIOR || l1 >= -1, ld_t<DUAL>(&U.in[(l1 + 1) & (CH3_RING - 1)][lane]));
			} else { // extreme stretch (> 2x): gather straight from the spectrum row(s)
				auto gather = [&](int bb) -> c2 {
					if (bb < 0 || bb >= K) return zc;
					if constexpr (DUAL) {
						const float2 a = myInD[0][bb], c = myInD[1][bb];
						return c2{f2_make(a.x, c.x), f2_make(a.y, c.y)};
					} else {
						return ld_c2s(myInIl + bb);
					}
				};
				cLo2 = gather(l2);
				cHi2 = gather(l2 + 1);
				cLo1 = gather(l1);
				cHi1 = gather(l1 + 1);
			}
		};
		// first step (every q <= 0: nothing behind it is inside the spectrum, but the masks need their indices)
		if (farAny) preload(-G * lane, std::true_type{}, std::false_type{}, false);
		else preload(-G * lane, std::false_type{}, std::false_type{}, false);
		int cb = 0; // buffer of the chunk being computed
		for (int k0 = 0; k0 < steps; k0 += CHAIN_CH, cb ^= 1) {
			cp_async_wait_all(); // this chunk's tiles (issued one chunk ago)
			__syncwarp();
			if (k0 + CHAIN_CH < steps) fill(k0 + CHAIN_CH, cb ^ 1); // next chunk: in flight during the 8 steps below
			// ---------------- CHAIN_CH steps ----------------
			// INTERIOR: every lane's q, b and interpolation points are inside [0, K) for the whole chunk, so all the
			// edge masks below are identities and are compiled out (about nine chunks in ten)
			auto step = [&](const int i, auto farTag, auto intTag) {
				constexpr bool FAR = decltype(farTag)::value, INTERIOR = decltype(intTag)::value;
				const int q = k0 + i - G * lane;
				const int b = q - LT - 1, p2 = q - 1, p1 = q - D1;
				const bool qIn = INTERIOR || (active && (unsigned)q < (unsigned)K);
				const bool p2In = INTERIOR || (active && (unsigned)p2 < (unsigned)K);
				const bool p1In = INTERIOR || (active && (unsigned)p1 < (unsigned)K);
				// loaded one step ahead: interpolation points / fractions of the twists of bins p2 and p1, Prediction::input at bin b,
				// the previous block's final output / energy at bin q
				const c2 lo2 = cLo2, hi2 = cHi2, lo1 = cLo1, hi1 = cHi1, inB = cInB;
				const float f2s = cF2s, f1s = cF1s;
				const f2 re = cRe, eB = cEB, sqB = cSqB;
				c2 ro = roN;
				const c2 inq = ld_t<DUAL>(&U.in[q & (CH3_RING - 1)][lane]);
				c2 pv = ld_t<DUAL>(&U.pvy[cb][i][lane]);
				preload(q + 1, farTag, intTag, true); // ... and the same for the next step
				const c2 in1 = D1 == 1 ? inP : inP2; // Prediction::input at bin p1
				c2 newPre, T2, t1n;
				f2 newE;
				if constexpr (FAST) {
					pv = fmul_s(pv, rotq); // :653-654 rotate Band::output and Band::prevInput by one interval
					ro = fmul_s(ro, rotq);
					const f2 e = fnorm2(inq);                    // :679 (identity map: energy = |input|^2)
					const c2 ph0 = fmul_c(ro, fmulc_c(inq, pv)); // :714-715
					const f2 den = f2_make(fmaxf(f2_lo(re), f2_lo(e)), fmaxf(f2_hi(re), f2_hi(e))) + f2_make(B200S_NOISE_FLOOR, B200S_NOISE_FLOOR);
					const f2 rden = PROBE == 1 ? fma2(den, f2_make(0.5f, 0.5f), den) : f2_make(rcp_fast(f2_lo(den)), rcp_fast(f2_hi(den)));
					newPre = sel_c2(qIn, c2{mul2(ph0.re, rden), mul2(ph0.im, rden)}); // :716
					newE = sel_f2(qIn, e);
					T2 = sel_c2(p2In, fmulc_c(inP, flerp2(lo2, hi2, f2s)));  // long twist at p2 (:758)
					t1n = sel_c2(p1In, fmulc_c(in1, flerp2(lo1, hi1, f1s))); // short twist at p1 (:751,:771)
				} else {
					pv = xmul2s(pv, rotq, one);
					ro = xmul2s(ro, rotq, one);
					const f2 e = xnorm2(inq, one);
					const c2 ph0 = xmul2(ro, xmulc2(inq, pv, one), one);
					const f2 den = f2_make(fmaxf(f2_lo(re), f2_lo(e)), fmaxf(f2_hi(re), f2_hi(e))) + f2_make(B200S_NOISE_FLOOR, B200S_NOISE_FLOOR);
					newPre = sel_c2(qIn, c2{fdivq2(ph0.re, den), fdivq2(ph0.im, den)});
					newE = sel_f2(qIn, e);
					T2 = sel_c2(p2In, xmulc2(inP, xlerp2p(lo2, hi2, f2s, one), one));
					t1n = sel_c2(p1In, xmulc2(in1, xlerp2p(lo1, hi1, f1s, one), one));
				}
				{
					const float2 st = make_float2(f2_lo(newE), f2_hi(newE));
					U.eR[q & (CH6_ER - 1)][lane] = st;
				}
				inP2 = inP;
				inP = sel_c2(qIn, inq);
				{
					const float2 rn = xmul(rotq, rotS); // the table recurrence stays in the reference's own arithmetic
					rotq = make_float2((INTERIOR || q >= 0) ? rn.x : rotq.x, (INTERIOR || q >= 0) ? rn.y : rotq.y);
				}
				// ---- FIFO taps; entry 0 is this step's new value
				PR[0] = newPre;
				T1[0] = t1n;
				const c2 pre1 = PR[1];           // prelim output at b+L = q-1
				const c2 preA = PR[LT - A];      // prelim output at b+A+1
				const c2 t1b = T1[LT + 1 - D1];  // short twist at b
				const c2 t1A = T1[LT - A - D1];  // short twist at b+A+1
#pragma unroll
				for (int u = NPR - 1; u > 0; --u) PR[u] = PR[u - 1];
#pragma unroll
				for (int u = NT1 - 1; u > 0; --u) T1[u] = T1[u - 1];
				// ---- main prediction at bin b (:727-800)
				c2 oc, ph2;
				if constexpr (FAST) {
					// RF is the running phase sum here: :761 went in when out(b-L) was finalised, :774 one step ago (A = 1);
					// the term that closes the recurrence (:754) comes last
					c2 acc = RF[0];
					if constexpr (INTERIOR) {
						if constexpr (A == 0) acc = fmulc_acc(acc, preA, t1A); // :774
						acc = fmulc_acc(acc, pre1, T2);                         // :784
						ph2 = fmul_acc(acc, oc1, t1b);                          // :754
						if constexpr (A == 1) RF[1] = fmulc_acc(RF[1], preA, t1A); // :774 of bin b+1
					} else {
						if constexpr (A == 0) acc = acc + sel_c2(b < K - 1, fmulc_c(preA, t1A));
						acc = acc + sel_c2(b < K - LT, fmulc_c(pre1, T2));
						ph2 = acc + sel_c2(b > 0, fmul_c(oc1, t1b));
						if constexpr (A == 1) RF[1] = RF[1] + sel_c2(b + 1 < K - 1, fmulc_c(preA, t1A));
					}
					if constexpr (DUAL) { // :788, each half its own (mono) stream
						const float2 oA = make_output_fast_e<PROBE>(pick(false, ph2), f2_lo(eB), f2_lo(sqB), pick(false, inB));
						const float2 oB = make_output_fast_e<PROBE>(pick(true, ph2), f2_hi(eB), f2_hi(sqB), pick(true, inB));
						oc = c2{f2_make(oA.x, oB.x), f2_make(oA.y, oB.y)};
					} else { // the louder channel (first on ties, :733) leads, the other is locked in phase (:791-799)
						const bool m = f2_hi(eB) > f2_lo(eB);
						const float maxE = m ? f2_hi(eB) : f2_lo(eB);
						const float2 phase = pick(m, ph2), pinM = pick(m, inB);
						const float sqM = m ? f2_hi(sqB) : f2_lo(sqB), sqO = m ? f2_lo(sqB) : f2_hi(sqB);
						const float2 outM = make_output_fast_e<PROBE>(phase, maxE, sqM, pinM); // :788
						const float2 inO = pick(!m, inB);
						const float eO = m ? f2_lo(eB) : f2_hi(eB);
						const float2 outO = PROBE == 2 ? outM : make_output_fast_e<PROBE>(fmul_f(outM, fmulc_f(inO, pinM)), eO, sqO, inO);
						oc = c2{f2_make(m ? outO.x : outM.x, m ? outM.x : outO.x), f2_make(m ? outO.y : outM.y, m ? outM.y : outO.y)};
					}
				} else {
					// the phase sum of :754-784 is formed for both halves at once, each from its own registers, in the
					// reference's order; the products were formed when their factors became available
					const c2 p3x = xmulc2(preA, t1A, one); // :774 of bin b+A
					const c2 P3b = A == 1 ? P3c : p3x;
					if constexpr (A == 1) P3c = p3x;
					const c2 P4b = xmulc2(pre1, T2, one);  // :784
					ph2 = zc;
					ph2 = ph2 + sel_c2(INTERIOR || b > 0, xmul2(oc1, t1b, one)); // :754
					ph2 = ph2 + sel_c2(INTERIOR || b >= LT, RF[0]);              // :761
					ph2 = ph2 + sel_c2(INTERIOR || b < K - 1, P3b);              // :774
					ph2 = ph2 + sel_c2(INTERIOR || b < K - LT, P4b);             // :784
					if constexpr (DUAL) {
						oc = make_output_q2(ph2, eB, inB, one); // :788
					} else {
						const bool m = f2_hi(eB) > f2_lo(eB);
						const float maxE = m ? f2_hi(eB) : f2_lo(eB);
						const float2 phase = pick(m, ph2), pinM = pick(m, inB);
						const float2 outM = make_output_q(phase, maxE, pinM); // :788
						// the other channel is locked in phase (:791-799); computed for both, the leader keeps outM
						const c2 tw = c2{padd(muls(inB.re, pinM.x), muls(inB.im, pinM.y), one), psub(muls(inB.im, pinM.x), muls(inB.re, pinM.y), one)};
						const c2 cph = c2{psub(muls(tw.re, outM.x), muls(tw.im, outM.y), one), padd(muls(tw.im, outM.x), muls(tw.re, outM.y), one)};
						const c2 other = make_output_q2(cph, eB, inB, one);
						oc = c2{f2_make(m ? f2_lo(other.re) : outM.x, m ? outM.x : f2_hi(other.re)),
						        f2_make(m ? f2_lo(other.im) : outM.y, m ? outM.y : f2_hi(other.im))};
					}
				}
				// unconditional: out-of-range steps only produce values that every consumer masks
				oc1 = oc;
				// :761 of bin b+L: out(b) * longTwist(b+L); bins below L have no such term (b < 0: masked here)
				c2 rNew;
				if constexpr (FAST) rNew = sel_c2(INTERIOR || b >= 0, fmul_c(oc, T2));
				else rNew = xmul2(oc, T2, one);
#pragma unroll
				for (int u = 0; u + 1 < LT; ++u) RF[u] = RF[u + 1];
				RF[LT - 1] = rNew;
				U.pvy[cb][i][lane] = pack_t<DUAL>(oc); // for the next lane (its prelim bin of the next step) and for the write-back
				if constexpr (DUAL) {
					if (lastFrame && (unsigned)b < (unsigned)K) {
						eRowD[0][b] = f2_lo(eB);
						eRowD[1][b] = f2_hi(eB);
					}
				}
				__syncwarp();
				roN = ld_t<DUAL>(&U.pvy[cb][i][0] + lane - (PROBE == 4 ? 0 : 1)); // the next step's prelim bin of this lane is the bin lane-1 just finalised
			};
			// unrolled by 4 (for L = 4 the register FIFOs rotate by pure renaming) so that the hot loop stays in the
			// instruction cache; branch-free inside
			auto run_chunk = [&](auto farTag, auto intTag) {
#pragma unroll 1
				for (int h = 0; h < CHAIN_CH; h += 4) {
#pragma unroll
					for (int u = 0; u < 4; ++u) step(h + u, farTag, intTag);
				}
			};
			if (farAny) run_chunk(std::true_type{}, std::false_type{});
			else if (k0 >= interiorFrom && k0 + CHAIN_CH <= K) run_chunk(std::false_type{}, std::true_type{});
			else run_chunk(std::false_type{}, std::false_type{});
			// ---------------- write the chunk's finals back: planar Band::output rows, 32 B per row and quarter-warp;
			//                  all tile reads first, then the stores (row addresses are arithmetic).
			// (Every lane storing its own final straight to its row in every step would be 64 partial-sector writes per warp
			//  and step instead of 16 full-sector stores per chunk.)
			{
				float4 v[8];
#pragma unroll
				for (int it = 0; it < 8; ++it) v[it] = U.pvy[cb][fillI][fillF + 4 * it];
				const int rowMul = DUAL ? 1 : 2; // rows per block in Y
#pragma unroll
				for (int it = 0; it < 8; ++it) {
					const int fl = fillF + 4 * it;
					const int b = k0 + fillI - G * fl - LT - 1;
					if (PROBE != 6 && PROBE != 7 && fl < nAct && (unsigned)b < (unsigned)K) {
						const size_t o = (size_t)(rowMul * fl) * K + b;
						yBaseA[o] = make_float2(v[it].x, v[it].z);
						yBaseB[o] = make_float2(v[it].y, v[it].w);
					}
				}
			}
			__syncwarp();
		}
	}
	__syncwarp();
	} // pass
}

static inline size_t smem_chain6() { return sizeof(Chain6Tiles); }

} // namespace b200s
