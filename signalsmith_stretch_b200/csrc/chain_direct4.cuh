// chain_direct4.cuh -- k_chain_direct4: k_chain_direct3 (packed stereo frame wavefront, reference :722-804)
// with the cross-lane dependency taken OFF the per-step critical path.
//
// In k_chain_direct3 block t+1 runs the minimum L+1 bins behind block t, so within one step the chain is
//   lane-1's final of the previous step -> shuffle -> rotate -> preliminary prediction (:714-716, one exact
//   division) -> fourth term of the phase sum (:784) -> makeOutput of the leader -> makeOutput of the locked
//   channel -> next step,
// a long chain of dependent latency per step, and nothing of step k+1 can start before step k ends.
// Here the lanes are skewed by G = L+2 bins and every lane computes its preliminary prediction ONE BIN AHEAD
// of what the phase sum consumes (FIFOs of L+1 entries): the preliminary part of a step depends only on
// values finalised in the previous step and is independent of the step's own serial recurrence, so the
// scheduler overlaps the two; the per-step critical path is the in-lane recurrence alone (:754 -> :788 ->
// :791-799).  Cost: F-1 extra steps per call (1 %).  Results are bit-identical to the other generations.
#pragma once
#include "chain_direct3.cuh"

namespace b200s {

// largest L*timeFactor served from the shared-memory ring: the chunk in progress reads at most CH4_FAR + 2 bins
// behind its own 8 while the next 8 are in flight (8 + 8 + CH4_FAR + 2 <= CH3_RING); beyond it: global gathers
#define CH4_FAR (CH3_RING - 2 * CHAIN_CH - 3)

// ---- FAST arithmetic (default on the GPU; b200s_set_tuning key 3 selects the exact mode) ------------------------
// The exact mode reproduces the reference compiled WITHOUT floating-point contraction, operation by operation
// (separate multiplies and adds, IEEE division and square root): about 40 % of the instructions of a step and most of
// its dependent latency exist only for that.  The fast mode computes the same expressions the way an optimising build
// of the reference does -- the reference's own shipped binary is built with -O3 -ffast-math
// (web/emscripten/compile.sh:50): multiply-adds fused, the phase sum re-associated so that the term that closes the
// recurrence is added last, a / b as a * rcp(b), phase * sqrt(energy / |phase|^2) as phase * (sqrt(energy) *
// rsqrt(|phase|^2)) on the SFU approximations (1-2 ulp).  Results agree with the exact mode to float rounding per
// operation; both are tested against the oracle to the north-star tolerance (tests/test_gpu_parity.py).
__device__ __forceinline__ f2 neg2(f2 a) { return f2_make(-f2_lo(a), -f2_hi(a)); } // folded into operand modifiers by ptxas
// (the scalar fast helpers -- rcp_fast, rsqrt_fast, sqrt_fast, ffma, fmul_f, fmulc_f, make_output_fast -- live in kernels.cuh:
//  the mono direct chain uses them too)
// a * b and a * conj(b), fused
__device__ __forceinline__ c2 fmul_c(c2 a, c2 b) {
	return c2{fma2(a.re, b.re, neg2(mul2(a.im, b.im))), fma2(a.re, b.im, mul2(a.im, b.re))};
}
__device__ __forceinline__ c2 fmulc_c(c2 a, c2 b) {
	return c2{fma2(a.re, b.re, mul2(a.im, b.im)), fma2(a.im, b.re, neg2(mul2(a.re, b.im)))};
}
// acc + a * b, acc + a * conj(b)
__device__ __forceinline__ c2 fmul_acc(c2 acc, c2 a, c2 b) {
	return c2{fma2(neg2(a.im), b.im, fma2(a.re, b.re, acc.re)), fma2(a.im, b.re, fma2(a.re, b.im, acc.im))};
}
__device__ __forceinline__ c2 fmulc_acc(c2 acc, c2 a, c2 b) {
	return c2{fma2(a.im, b.im, fma2(a.re, b.re, acc.re)), fma2(neg2(a.re), b.im, fma2(a.im, b.re, acc.im))};
}
// a * (r.x + i r.y), r common to both channels
__device__ __forceinline__ c2 fmul_s(c2 a, float2 r) {
	return c2{fmas(a.im, -r.y, muls(a.re, r.x)), fmas(a.im, r.x, muls(a.re, r.y))};
}
__device__ __forceinline__ f2 fnorm2(c2 a) { return fma2(a.re, a.re, mul2(a.im, a.im)); }
__device__ __forceinline__ c2 flerp2(c2 lo, c2 hi, float fr) { return c2{fmas(hi.re - lo.re, fr, lo.re), fmas(hi.im - lo.im, fr, lo.im)}; }
// Tiles of k_chain_direct4: as Chain3Tiles ([bin][lane] tiles, conflict-free for the per-step reads and for the
// quarter-warp fill), without the output-row table (Band::output rows of consecutive blocks are equidistant).
// (Lane-private rows filled with cp.async.bulk are no alternative: bulk copies take uniform operands, so per-lane copies
// are serialised lane by lane.)
struct Chain4Tiles {
	float4 in[CH3_RING][CH3_RS]; // rolling window of each block's interleaved input spectrum, [bin & 31][lane]
	float4 pvy[2][CHAIN_CH][CH3_RS]; // previous-input spectrum at the chunk's bins, overwritten by the finals of the same step
	float4 p0Out[2][CHAIN_CH];    // lane 0's predecessor block: {c0.re, c0.im, c1.re, c1.im}
	float2 p0E[2][CHAIN_CH];      // its Prediction::energy {c0, c1}
	const float4 *rowIn[32], *rowPv[32];
};

// true when k_chain_ws (chain_ws.cuh) takes this stream: every block's time factor is within the reach of its 16-bin
// spectrum ring (timeFactor <= 2, the clean-stretch limit of :509).  Evaluated identically by both kernels.
__device__ __forceinline__ bool ws_stream_ok(const Ctx &x, int s, int nFrames, int lane) {
	bool bad = false;
	for (int f = lane; f < nFrames; f += 32)
		bad = bad || !(fmaxf(x.frames[(size_t)s * x.maxFrames + f].timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH) <= B200S_MAX_CLEAN_STRETCH);
	return !__any_sync(0xffffffffu, bad);
}

template <int LT, bool FAST>
__global__ void __launch_bounds__(32) k_chain_direct4(Ctx x) {
	const Cfg &g = x.cfg;
	const int K = g.K;
	B200S_DYN_SHARED
	const int lane = threadIdx.x & 31;
	const int s = x.sBase + blockIdx.x;
	const Call cl = x.call[s];
	if (cl.nFrames == 0) return;
	if (cl.hasRandom && x.randomPathOn) return; // a block beyond 2x stretch draws random time factors: k_prep + k_chain take the stream
	if (x.wsRan && ws_stream_ok(x, s, cl.nFrames, lane)) return; // k_chain_ws has done this stream
	constexpr int G = LT + 2; // lane skew in bins
	constexpr int NF = LT + 1; // FIFO entries: bins b .. b+L of the lane's block
	Chain4Tiles &U = *(Chain4Tiles *)dyn_smem;
	// chunk fill: lane -> (bin offset, row within a group of 4); a quarter-warp covers 4 bins (64 B) of 2 rows
	const int fillI = (lane & 3) | (((lane >> 3) & 1) << 2), fillF = ((lane >> 2) & 1) | (((lane >> 4) & 1) << 1);
	const float2 rot0 = x.rot0, rotStep = x.rotStep;
	const float one = x.one; // unused by the f2 arithmetic (see padd / psub)

	for (int base = 0; base < cl.nFrames; base += 32) {
		__syncwarp();
		const int f = base + lane;
		const bool active = f < cl.nFrames;
		const Frame fr = x.frames[(size_t)s * x.maxFrames + (active ? f : base)];
		const bool rotOn = fr.flags & FR_NEW_SPECTRUM;
		const int nAct = min(32, cl.nFrames - base);
		const float tf = fmaxf(fr.timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH); // :638
		const float longTf = fmul((float)LT, tf);
		const bool farAny = __any_sync(0xffffffffu, active && longTf > (float)CH4_FAR);
		const float2 *prevOut[2];
		const float *prevE[2];
#pragma unroll
		for (int c = 0; c < 2; ++c) {
			prevOut[c] = base == 0 ? x.stOut + ((size_t)s * 2 + c) * K : x.Y + coef_off(x, s, base - 1, c);
			prevE[c] = x.stPredE + ((size_t)s * 2 + c) * K; // base == 0 only; later groups recompute it, see the fill
		}
		// Prediction::energy of a block on this path is |input|^2 of its own spectrum (:679,:708): the chain never stores
		// it -- the next group recomputes it from the predecessor's input row, k_commit from the final input spectrum
		const float4 *prevIn = base == 0 ? nullptr : il_row(x, s, x.frames[(size_t)s * x.maxFrames + base - 1].inSlot);
		const float4 *myIn = il_row(x, s, fr.inSlot);
		U.rowIn[lane] = myIn;
		U.rowPv[lane] = il_row(x, s, fr.prevSlot);
		float2 *const yBase = x.Y + coef_off(x, s, base, 0); // Band::output row of block base + r, channel c: yBase + (2r + c) * K
		__syncwarp();
		// register FIFOs (channel pairs); at the start of a step (q = prelim bin, b = q - L - 1 = final bin):
		//   pre/eF/t2F/inF[i] <-> prelim output / energy / long twist / input at bin b+i, i = 0..L (b+L = q-1)
		//   oh[i] <-> final output at bin b-1-i;   t1P <-> short twist at bin b
		const f2 z2 = f2_make(0.f, 0.f);
		const c2 zc = c2{z2, z2};
		c2 oh[LT], pre[NF], t2F[NF], inF[NF], t1P = zc, lastFinal = zc;
		f2 eF[NF], lastE = z2;
#pragma unroll
		for (int i = 0; i < LT; ++i) oh[i] = zc;
#pragma unroll
		for (int i = 0; i < NF; ++i) {
			pre[i] = t2F[i] = inF[i] = zc;
			eF[i] = z2;
		}
		float2 rotq = rotOn ? rot0 : make_float2(1.f, 0.f); // rot[q] by the reference's float recurrence (:647-655)
		const float2 rotS = rotOn ? rotStep : make_float2(1.f, 0.f);
		const int steps = K + LT + 1 + G * (nAct - 1);
		// first chunk start from which every ACTIVE lane has q - L*tf - 1 >= 0, (b+1) - tf - 1 >= 0 and b = q - L - 1 >= L
		// (inactive lanes only produce values nobody consumes): q >= G*(nAct-1) + 2L + ceil(max L*tf) + 2
		int interiorFrom;
		{
			float mx = active ? longTf : 0.f;
			for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
			interiorFrom = G * (nAct - 1) + 2 * LT + (int)ceilf(mx) + 3;
		}
		// asynchronous fill of the chunk starting at kf into buffer `buf`: 8 new bins per block, both channels per
		// 16-byte copy.  The ring slots it writes (the 8 bins after the chunk's own 8, per lane) are disjoint from what
		// the chunk in progress reads (at most CH4_FAR + 2 bins behind its own 8: 8 + 8 + CH4_FAR + 2 <= CH3_RING).
		// The row pointers are read first, all at once: the copies are asm volatile and would otherwise serialise the
		// shared-memory latency of every pointer load.
		auto fill = [&](int kf, int buf) {
			const float4 *rIn[8], *rPv[8];
#pragma unroll
			for (int it = 0; it < 8; ++it) {
				rIn[it] = U.rowIn[fillF + 4 * it];
				rPv[it] = U.rowPv[fillF + 4 * it];
			}
#pragma unroll
			for (int it = 0; it < 8; ++it) {
				const int fl = fillF + 4 * it;
				const int q = kf + fillI - G * fl;
				if (fl < nAct && (unsigned)q < (unsigned)K) {
					cp_async16(&U.in[q & (CH3_RING - 1)][fl], rIn[it] + q);
					cp_async16(&U.pvy[buf][fillI][fl], rPv[it] + q);
				}
			}
			if (lane < 2 * CHAIN_CH) { // lane 0's predecessor: planar state / previous group rows -> {c0, c1} slots
				const int qq = kf + (lane >> 1), c = lane & 1;
				if (qq < K) {
					cp_async8((float2 *)&U.p0Out[buf][lane >> 1] + c, (c ? prevOut[1] : prevOut[0]) + qq);
					if (base == 0) {
						cp_async4((float *)&U.p0E[buf][lane >> 1] + c, (c ? prevE[1] : prevE[0]) + qq);
					} else {
						const float4 v = prevIn[qq];
						((float *)&U.p0E[buf][lane >> 1])[c] = c ? xnorm(make_float2(v.y, v.w)) : xnorm(make_float2(v.x, v.z));
					}
				}
			}
		};
		fill(0, 0);
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
				const int b = q - LT - 1;
				const bool qIn = INTERIOR || (active && (unsigned)q < (unsigned)K);
				// the twists need input interpolated at q - L*tf and (b+1) - tf  (:750,:757)
				const float i2 = fsub((float)q, longTf);
				const int l2 = (int)floorf(i2);
				const float f2s = fsub(i2, (float)l2);
				const float i1 = fsub((float)(b + 1), tf);
				const int l1 = (int)floorf(i1);
				const float f1s = fsub(i1, (float)l1);
				// previous block's final output / energy at bin q: finalised by lane-1 in the last step
				c2 ro;
				f2 re;
				{
					const float a0 = __shfl_up_sync(0xffffffffu, f2_lo(lastFinal.re), 1), a1 = __shfl_up_sync(0xffffffffu, f2_hi(lastFinal.re), 1);
					const float b0 = __shfl_up_sync(0xffffffffu, f2_lo(lastFinal.im), 1), b1 = __shfl_up_sync(0xffffffffu, f2_hi(lastFinal.im), 1);
					const float e0 = __shfl_up_sync(0xffffffffu, f2_lo(lastE), 1), e1 = __shfl_up_sync(0xffffffffu, f2_hi(lastE), 1);
					const float4 p0 = U.p0Out[cb][i];
					const float2 p0e = U.p0E[cb][i];
					const bool first = lane == 0;
					ro = c2{f2_make(first ? p0.x : a0, first ? p0.z : a1), f2_make(first ? p0.y : b0, first ? p0.w : b1)};
					re = f2_make(first ? p0e.x : e0, first ? p0e.y : e1);
				}
				const c2 inq = ld_c2s(&U.in[q & (CH3_RING - 1)][lane]);
				c2 pv = ld_c2s(&U.pvy[cb][i][lane]);
				c2 lo2, hi2, lo1, hi1;
				if constexpr (!FAR) {
					lo2 = sel_c2(INTERIOR || l2 >= 0, ld_c2s(&U.in[l2 & (CH3_RING - 1)][lane]));
					hi2 = sel_c2(INTERIOR || l2 >= -1, ld_c2s(&U.in[(l2 + 1) & (CH3_RING - 1)][lane]));
					lo1 = sel_c2(INTERIOR || l1 >= 0, ld_c2s(&U.in[l1 & (CH3_RING - 1)][lane]));
					hi1 = sel_c2(INTERIOR || l1 >= -1, ld_c2s(&U.in[(l1 + 1) & (CH3_RING - 1)][lane]));
				} else { // extreme stretch (> 2x): gather straight from the spectrum row
					lo2 = (l2 < 0 || l2 >= K) ? zc : ld_c2s(myIn + l2);
					hi2 = (l2 + 1 < 0 || l2 + 1 >= K) ? zc : ld_c2s(myIn + l2 + 1);
					lo1 = (l1 < 0 || l1 >= K) ? zc : ld_c2s(myIn + l1);
					hi1 = (l1 + 1 < 0 || l1 + 1 >= K) ? zc : ld_c2s(myIn + l1 + 1);
				}
				pv = xmul2s(pv, rotq, one); // :653-654 rotate Band::output and Band::prevInput by one interval
				ro = xmul2s(ro, rotq, one);
				const f2 e = xnorm2(inq, one);                       // :679 (identity map: energy = |input|^2)
				const c2 ph0 = xmul2(ro, xmulc2(inq, pv, one), one);      // :714-715
				const f2 den = f2_make(fmaxf(f2_lo(re), f2_lo(e)), fmaxf(f2_hi(re), f2_hi(e))) + f2_make(B200S_NOISE_FLOOR, B200S_NOISE_FLOOR);
				const c2 newPre = sel_c2(qIn, c2{fdivq2(ph0.re, den), fdivq2(ph0.im, den)}); // :716
				const f2 newE = sel_f2(qIn, e);
				const c2 newIn = sel_c2(qIn, inq);
				const c2 newT2 = sel_c2(qIn, xmulc2(inq, xlerp2p(lo2, hi2, f2s, one), one)); // long twist at q (:758)
				// short twist at b+1 (:751,:771): Prediction::input[b+1] is inF[1]
				const c2 t1N = xmulc2(inF[1], xlerp2p(lo1, hi1, f1s, one), one);
				{
					const float2 rn = xmul(rotq, rotS);
					rotq = make_float2((INTERIOR || q >= 0) ? rn.x : rotq.x, (INTERIOR || q >= 0) ? rn.y : rotq.y);
				}
				// ---- the FIFO heads belong to bin b; the new preliminary values (bin q = b+L+1) enter after the main
				//      prediction below, which only reads entries computed in EARLIER steps
				const f2 eB = eF[0];
				const c2 t2B = t2F[0], inB = inF[0];
				const c2 preN = pre[1], preL = pre[LT], t2L = t2F[LT]; // prelim output at b+1, b+L; long twist at b+L
#pragma unroll
				for (int u = 0; u + 1 < NF; ++u) {
					pre[u] = pre[u + 1];
					eF[u] = eF[u + 1];
					t2F[u] = t2F[u + 1];
					inF[u] = inF[u + 1];
				}
				pre[NF - 1] = newPre;
				eF[NF - 1] = newE;
				t2F[NF - 1] = newT2;
				inF[NF - 1] = newIn;
				// ---- main prediction at bin b (:727-800): the louder channel (first on ties, :733) leads
				const bool m = f2_hi(eB) > f2_lo(eB);
				const float maxE = m ? f2_hi(eB) : f2_lo(eB);
				// the phase sum of :754-784 is formed for both channels at once (packed, each channel from its own
				// registers, exactly as if it were the leader) and the leader's is picked afterwards
				c2 ph2 = zc;
				ph2 = ph2 + sel_c2(INTERIOR || b > 0, xmul2(oh[0], t1P, one));                      // :754
				ph2 = ph2 + sel_c2(INTERIOR || b >= LT, xmul2(oh[LT - 1], t2B, one));               // :761
				ph2 = ph2 + sel_c2(INTERIOR || b < K - 1, xmulc2(preN, t1N, one));                  // :774
				ph2 = ph2 + sel_c2(INTERIOR || b < K - LT, xmulc2(preL, t2L, one));                // :784
				const float2 phase = pick(m, ph2), pinM = pick(m, inB);
				const float2 outM = make_output_q(phase, maxE, pinM);     // :788
				// the other channel is locked in phase (:791-799); computed for both, the leader keeps outM
				//   cph = xmul(outM, xmulc(inB_c, pinM)), operand order of the scalar helpers
				const c2 tw = c2{padd(muls(inB.re, pinM.x), muls(inB.im, pinM.y), one), psub(muls(inB.im, pinM.x), muls(inB.re, pinM.y), one)};
				const c2 cph = c2{psub(muls(tw.re, outM.x), muls(tw.im, outM.y), one), padd(muls(tw.im, outM.x), muls(tw.re, outM.y), one)};
				const c2 other = make_output_q2(cph, eB, inB, one);
				const c2 oc = c2{f2_make(m ? f2_lo(other.re) : outM.x, m ? outM.x : f2_hi(other.re)),
				                 f2_make(m ? f2_lo(other.im) : outM.y, m ? outM.y : f2_hi(other.im))};
				// unconditional: out-of-range steps only produce values that every consumer masks
#pragma unroll
				for (int u = LT - 1; u > 0; --u) oh[u] = oh[u - 1];
				oh[0] = oc;
				lastFinal = oc;
				lastE = eB;
				t1P = t1N;
				U.pvy[cb][i][lane] = make_float4(f2_lo(oc.re), f2_hi(oc.re), f2_lo(oc.im), f2_hi(oc.im));
			};
			// FAST arithmetic (see the top of the file): same data flow, fused operations, re-associated phase sum
			auto step_fast = [&](const int i, auto farTag, auto intTag) {
				constexpr bool FAR = decltype(farTag)::value, INTERIOR = decltype(intTag)::value;
				const int q = k0 + i - G * lane;
				const int b = q - LT - 1;
				const bool qIn = INTERIOR || (active && (unsigned)q < (unsigned)K);
				const float i2 = fsub((float)q, longTf);
				const int l2 = (int)floorf(i2);
				const float f2s = fsub(i2, (float)l2);
				const float i1 = fsub((float)(b + 1), tf);
				const int l1 = (int)floorf(i1);
				const float f1s = fsub(i1, (float)l1);
				c2 ro;
				f2 re;
				{
					const float a0 = __shfl_up_sync(0xffffffffu, f2_lo(lastFinal.re), 1), a1 = __shfl_up_sync(0xffffffffu, f2_hi(lastFinal.re), 1);
					const float b0 = __shfl_up_sync(0xffffffffu, f2_lo(lastFinal.im), 1), b1 = __shfl_up_sync(0xffffffffu, f2_hi(lastFinal.im), 1);
					const float e0 = __shfl_up_sync(0xffffffffu, f2_lo(lastE), 1), e1 = __shfl_up_sync(0xffffffffu, f2_hi(lastE), 1);
					const float4 p0 = U.p0Out[cb][i];
					const float2 p0e = U.p0E[cb][i];
					const bool first = lane == 0;
					ro = c2{f2_make(first ? p0.x : a0, first ? p0.z : a1), f2_make(first ? p0.y : b0, first ? p0.w : b1)};
					re = f2_make(first ? p0e.x : e0, first ? p0e.y : e1);
				}
				const c2 inq = ld_c2s(&U.in[q & (CH3_RING - 1)][lane]);
				c2 pv = ld_c2s(&U.pvy[cb][i][lane]);
				c2 lo2, hi2, lo1, hi1;
				if constexpr (!FAR) {
					lo2 = sel_c2(INTERIOR || l2 >= 0, ld_c2s(&U.in[l2 & (CH3_RING - 1)][lane]));
					hi2 = sel_c2(INTERIOR || l2 >= -1, ld_c2s(&U.in[(l2 + 1) & (CH3_RING - 1)][lane]));
					lo1 = sel_c2(INTERIOR || l1 >= 0, ld_c2s(&U.in[l1 & (CH3_RING - 1)][lane]));
					hi1 = sel_c2(INTERIOR || l1 >= -1, ld_c2s(&U.in[(l1 + 1) & (CH3_RING - 1)][lane]));
				} else {
					lo2 = (l2 < 0 || l2 >= K) ? zc : ld_c2s(myIn + l2);
					hi2 = (l2 + 1 < 0 || l2 + 1 >= K) ? zc : ld_c2s(myIn + l2 + 1);
					lo1 = (l1 < 0 || l1 >= K) ? zc : ld_c2s(myIn + l1);
					hi1 = (l1 + 1 < 0 || l1 + 1 >= K) ? zc : ld_c2s(myIn + l1 + 1);
				}
				pv = fmul_s(pv, rotq); // :653-654
				ro = fmul_s(ro, rotq);
				const f2 e = fnorm2(inq);                      // :679
				const c2 ph0 = fmul_c(ro, fmulc_c(inq, pv));     // :714-715
				const f2 den = f2_make(fmaxf(f2_lo(re), f2_lo(e)), fmaxf(f2_hi(re), f2_hi(e))) + f2_make(B200S_NOISE_FLOOR, B200S_NOISE_FLOOR);
				const f2 rden = f2_make(rcp_fast(f2_lo(den)), rcp_fast(f2_hi(den)));
				const c2 newPre = sel_c2(qIn, c2{mul2(ph0.re, rden), mul2(ph0.im, rden)}); // :716
				const f2 newE = sel_f2(qIn, e);
				const c2 newIn = sel_c2(qIn, inq);
				const c2 newT2 = sel_c2(qIn, fmulc_c(inq, flerp2(lo2, hi2, f2s))); // long twist at q (:758)
				const c2 t1N = fmulc_c(inF[1], flerp2(lo1, hi1, f1s));             // short twist at b+1 (:751,:771)
				{
					const float2 rn = xmul(rotq, rotS); // the table recurrence stays in the reference's own arithmetic
					rotq = make_float2((INTERIOR || q >= 0) ? rn.x : rotq.x, (INTERIOR || q >= 0) ? rn.y : rotq.y);
				}
				const f2 eB = eF[0];
				const c2 t2B = t2F[0], inB = inF[0];
				const c2 preN = pre[1], preL = pre[LT], t2L = t2F[LT];
#pragma unroll
				for (int u = 0; u + 1 < NF; ++u) {
					pre[u] = pre[u + 1];
					eF[u] = eF[u + 1];
					t2F[u] = t2F[u + 1];
					inF[u] = inF[u + 1];
				}
				pre[NF - 1] = newPre;
				eF[NF - 1] = newE;
				t2F[NF - 1] = newT2;
				inF[NF - 1] = newIn;
				// ---- main prediction at bin b (:727-800); the terms that do not depend on the previous bin first
				const bool m = f2_hi(eB) > f2_lo(eB);
				const float maxE = m ? f2_hi(eB) : f2_lo(eB);
				c2 ph2;
				if constexpr (INTERIOR) {
					ph2 = fmul_c(oh[LT - 1], t2B);        // :761
					ph2 = fmulc_acc(ph2, preN, t1N);      // :774
					ph2 = fmulc_acc(ph2, preL, t2L);      // :784
					ph2 = fmul_acc(ph2, oh[0], t1P);      // :754
				} else {
					ph2 = sel_c2(b >= LT, fmul_c(oh[LT - 1], t2B));
					ph2 = ph2 + sel_c2(b < K - 1, fmulc_c(preN, t1N));
					ph2 = ph2 + sel_c2(b < K - LT, fmulc_c(preL, t2L));
					ph2 = ph2 + sel_c2(b > 0, fmul_c(oh[0], t1P));
				}
				const float2 phase = pick(m, ph2), pinM = pick(m, inB);
				const float2 outM = make_output_fast(phase, maxE, pinM); // :788
				// the other channel is locked in phase (:791-799)
				const float2 inO = pick(!m, inB);
				const float eO = m ? f2_lo(eB) : f2_hi(eB);
				const float2 outO = make_output_fast(fmul_f(outM, fmulc_f(inO, pinM)), eO, inO);
				const c2 oc = c2{f2_make(m ? outO.x : outM.x, m ? outM.x : outO.x), f2_make(m ? outO.y : outM.y, m ? outM.y : outO.y)};
#pragma unroll
				for (int u = LT - 1; u > 0; --u) oh[u] = oh[u - 1];
				oh[0] = oc;
				lastFinal = oc;
				lastE = eB;
				t1P = t1N;
				U.pvy[cb][i][lane] = make_float4(f2_lo(oc.re), f2_hi(oc.re), f2_lo(oc.im), f2_hi(oc.im));
			};
			// unrolled by 4 (for L = 4 the register FIFOs rotate by pure renaming) so that the hot loop stays in the
			// instruction cache; branch-free inside
			auto run_chunk = [&](auto farTag, auto intTag) {
#pragma unroll 1
				for (int h = 0; h < CHAIN_CH; h += 4) {
#pragma unroll
					for (int u = 0; u < 4; ++u) {
						if constexpr (FAST) step_fast(h + u, farTag, intTag);
						else step(h + u, farTag, intTag);
					}
				}
			};
			if (farAny) run_chunk(std::true_type{}, std::false_type{});
			else if (k0 >= interiorFrom && k0 + CHAIN_CH <= K) run_chunk(std::false_type{}, std::true_type{});
			else run_chunk(std::false_type{}, std::false_type{});
			__syncwarp();
			// ---------------- write the chunk's finals back: planar Band::output rows, 32 B per row and quarter-warp;
			//                  all tile reads first, then the stores (row addresses are arithmetic) ----------------
			{
				float4 v[8];
#pragma unroll
				for (int it = 0; it < 8; ++it) v[it] = U.pvy[cb][fillI][fillF + 4 * it];
#pragma unroll
				for (int it = 0; it < 8; ++it) {
					const int fl = fillF + 4 * it;
					const int b = k0 + fillI - G * fl - LT - 1;
					if (fl < nAct && (unsigned)b < (unsigned)K) {
						float2 *row = yBase + (size_t)(2 * fl) * K + b;
						row[0] = make_float2(v[it].x, v[it].z);
						row[K] = make_float2(v[it].y, v[it].w);
					}
				}
			}
			__syncwarp();
		}
	}
}

static inline size_t smem_chain4(int) { return sizeof(Chain4Tiles); }

} // namespace b200s
