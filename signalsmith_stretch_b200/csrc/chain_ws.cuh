// chain_ws.cuh -- k_chain_ws: the frame-wavefront phase prediction (reference :696-719 preliminary prediction,
// :722-804 main prediction) of k_chain_direct4, WARP-SPECIALISED: one CTA of two warps per stream.
//
// Why (DESIGN.md section 3.2): k_chain_direct4 is one warp per stream -- 1024 warps, about two per scheduler -- and every
// warp issues its ~245 instructions per step strictly in order; the serial recurrence itself is only ~25 of them.  Everything else in a step depends only on the
// analysis spectra (twists, energies, rotation, the factor that turns the previous block's final output into the
// preliminary prediction), so it does not have to sit in the serial warp's instruction stream at all:
//
//   * warp 1, the PRODUCER (lane = block, one chunk of WS_CH steps ahead), stages the spectra (cp.async, as before),
//     forms per (block, bin)   A  = rot * input * conj(prevInput * rot) / (max(prevEnergy, energy) + noiseFloor)   (:653-654,:708-716)
//                              T1 = short vertical twist (:750-751)      T2 = long vertical twist (:757-758)
//                              P  = Prediction::input (:710)
//     with every edge / inactive-lane mask already applied (masked entries are exact zeros), writes them to
//     step-indexed shared-memory tiles, and writes the finished chunk's finals back to the Band::output rows;
//   * warp 0, the CONSUMER (lane = block), runs the recurrence alone: preliminary output = previous block's final
//     (one shuffle) * A, the four-term phase sum, makeOutput for the leading channel, the phase lock of the other
//     channel (:727-800).  No index arithmetic, no edge conditions, no global memory: ~90 instructions per step.
//
// The two warps meet at one CTA barrier per chunk (double-buffered tiles).  Twice the warps per stream also means
// twice the latency hiding per scheduler.  FAST = false keeps the reference's unfused IEEE arithmetic operation for
// operation (the producer then hands over freqTwist, the denominator and the rotation separately), bit-identical to
// the exact mode of k_chain_direct4 -- that is how tests/test_host_logic.py checks this kernel against the oracle.
//
// Geometry: the preliminary prediction runs WS_D = 6 bins ahead of the final bin and lanes are skewed by WS_G = 7 bins,
// for every L <= 4: the register FIFOs of the consumer then have six entries whatever L is, and 12 steps (three
// chunks) bring every FIFO back to its starting rotation, so the steps are unrolled with compile-time register
// renaming only.  The spectrum ring holds 16 bins per block: 4 being filled for the chunk after next, 4 the producer
// is working on, and 8 behind them, which is the reach of the long twist at the 2x stretch limit (L * timeFactor <= 8).
// Streams with a block beyond that (timeFactor > 2) are left to k_chain_direct4, which is launched right after this
// kernel and skips every stream this kernel took (ws_stream_ok).
#pragma once
#include "chain_direct4.cuh"

namespace b200s {

#define WS_CH 4
#define WS_RING 16
#define WS_RS 34
#define WS_D 6
#define WS_G 7

template <bool FAST>
struct WsTiles {
	float4 in[WS_RING][WS_RS];    // rolling window of each block's interleaved input spectrum, [bin & 15][lane]
	float4 pv[2][WS_CH][WS_RS];   // previous-input spectrum at the bins of the chunk the producer works on / the one in flight
	float4 A[2][WS_CH][WS_RS];    // FAST: prelim factor, exact: freqTwist (:714); the consumer overwrites it with the finals
	float4 T1[2][WS_CH][WS_RS];   // short twist at bin b+1
	float4 T2[2][WS_CH][WS_RS];   // long twist at bin q
	float4 P[2][WS_CH][WS_RS];    // Prediction::input at bin b
	float4 X[FAST ? 1 : 2][FAST ? 1 : WS_CH][FAST ? 1 : WS_RS]; // exact mode only: {den c0, den c1, rot.x, rot.y}
	float4 p0Out[4][WS_CH];       // lane 0's predecessor block: {c0.re, c0.im, c1.re, c1.im}
	float2 p0E[4][WS_CH];         // its Prediction::energy {c0, c1}
	const float4 *rowIn[32], *rowPv[32];
};

__device__ __forceinline__ float4 pack_c2(c2 v) { return make_float4(f2_lo(v.re), f2_hi(v.re), f2_lo(v.im), f2_hi(v.im)); }

template <int LT, bool FAST>
__global__ void __launch_bounds__(64, 7) k_chain_ws(Ctx x) {
	static_assert(LT >= 1 && LT <= 4, "ring reach and FIFO geometry are laid out for L <= 4");
	const Cfg &g = x.cfg;
	const int K = g.K;
	B200S_DYN_SHARED
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int s = stream_at(x, x.sBase + blockIdx.x);
	const Call cl = x.call[s];
	if (cl.nFrames == 0) return;
	if (cl.mapped || (cl.hasRandom && x.randomPathOn)) return; // a block beyond 2x stretch draws random time factors: k_prep + k_chain take the stream
	if (!ws_stream_ok(x, s, cl.nFrames, lane)) return; // k_chain_direct4 takes this stream
	WsTiles<FAST> &U = *(WsTiles<FAST> *)dyn_smem;
	const float one = x.one; // unused by the f2 arithmetic (see padd / psub)
	const f2 z2 = f2_make(0.f, 0.f);
	const c2 zc = c2{z2, z2};
	if (threadIdx.x < 4 * WS_CH) { // slots that are never loaded must hold finite values (0 * stale NaN would get past the zero masks)
		U.p0Out[threadIdx.x / WS_CH][threadIdx.x % WS_CH] = make_float4(0.f, 0.f, 0.f, 0.f);
		U.p0E[threadIdx.x / WS_CH][threadIdx.x % WS_CH] = make_float2(0.f, 0.f);
	}

	for (int base = 0; base < cl.nFrames; base += 32) {
		__syncthreads(); // the previous group's finals are in their Band::output rows, its tiles are free
		const int nAct = min(32, cl.nFrames - base);
		const int steps = K + WS_D + WS_G * (nAct - 1);
		const int nChunks = (steps + WS_CH - 1) / WS_CH;
		if (warp == 1) {
			// =============================== PRODUCER ===============================
			const int f = base + lane;
			const bool active = f < cl.nFrames;
			const Frame fr = x.frames[(size_t)s * x.maxFrames + (active ? f : base)];
			const bool rotOn = fr.flags & FR_NEW_SPECTRUM;
			const float tf = fmaxf(fr.timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH); // :638
			const float longTf = fmul((float)LT, tf);
			const float2 *prevOut[2];
			const float *prevE[2];
#pragma unroll
			for (int c = 0; c < 2; ++c) {
				prevOut[c] = base == 0 ? x.stOut + ((size_t)s * 2 + c) * K : x.Y + coef_off(x, s, base - 1, c);
				prevE[c] = x.stPredE + ((size_t)s * 2 + c) * K; // base == 0 only; later groups recompute it from the predecessor's input row
			}
			const float4 *prevIn = base == 0 ? nullptr : il_row(x, s, x.frames[(size_t)s * x.maxFrames + base - 1].inSlot);
			U.rowIn[lane] = il_row(x, s, fr.inSlot);
			U.rowPv[lane] = il_row(x, s, fr.prevSlot);
			float2 *const yBase = x.Y + coef_off(x, s, base, 0); // Band::output row of block base + r, channel c: yBase + (2r + c) * K
			float2 rotq = rotOn ? x.rot0 : make_float2(1.f, 0.f); // rot[q] by the reference's float recurrence (:647-655)
			const float2 rotS = rotOn ? x.rotStep : make_float2(1.f, 0.f);
			const int fI = lane & 3, fF = lane >> 2; // fill / write-back: lane -> (bin offset, row within a group of 8): a quarter-warp covers 64 B of two rows
			__syncwarp();
			const float4 *rIn[4], *rPv[4]; // the four rows this lane copies from, for the whole group
#pragma unroll
			for (int it = 0; it < 4; ++it) {
				rIn[it] = U.rowIn[fF + 8 * it];
				rPv[it] = U.rowPv[fF + 8 * it];
			}
			// asynchronous fill of chunk n: 4 new bins per block, both channels per 16-byte copy
			auto fill = [&](int n) {
				const int kf = n * WS_CH, buf = n & 1;
#pragma unroll
				for (int it = 0; it < 4; ++it) {
					const int fl = fF + 8 * it;
					const int q = kf + fI - WS_G * fl;
					if (fl < nAct && (unsigned)q < (unsigned)K) {
						cp_async16(&U.in[q & (WS_RING - 1)][fl], rIn[it] + q);
						cp_async16(&U.pv[buf][fI][fl], rPv[it] + q);
					}
				}
				if (lane < 2 * WS_CH) { // lane 0's predecessor: planar state / previous group rows -> {c0, c1} slots
					const int qq = kf + (lane >> 1), c = lane & 1;
					if (qq < K) {
						cp_async8((float2 *)&U.p0Out[n & 3][lane >> 1] + c, (c ? prevOut[1] : prevOut[0]) + qq);
						if (base == 0) {
							cp_async4((float *)&U.p0E[n & 3][lane >> 1] + c, (c ? prevE[1] : prevE[0]) + qq);
						} else {
							const float4 v = prevIn[qq];
							((float *)&U.p0E[n & 3][lane >> 1])[c] = c ? xnorm(make_float2(v.y, v.w)) : xnorm(make_float2(v.x, v.z));
						}
					}
				}
			};
			// the tiles of chunk n (its raw spectra are complete and visible)
			// INTERIOR (about nine chunks in ten of a full group): every lane is active and all its bins and interpolation
			// points lie inside [L, K) for the whole chunk, so every mask below is an identity and is compiled out
			auto produce = [&](int n, auto intTag) {
				constexpr bool INTERIOR = decltype(intTag)::value;
				const int nb = n & 1;
#pragma unroll
				for (int i = 0; i < WS_CH; ++i) {
					const int q = n * WS_CH + i - WS_G * lane; // bin of the preliminary prediction
					const int b = q - WS_D, q1 = b + 1;        // final bin of the same step; bin of the short twist
					const bool qIn = INTERIOR || (active && (unsigned)q < (unsigned)K);
					const bool q1In = INTERIOR || (active && q1 > 0 && q1 < K); // the short twist of bin 0 is never used (b > 0, :748)
					const bool bIn = INTERIOR || (active && (unsigned)b < (unsigned)K);
					const float i2 = fsub((float)q, longTf); // :757
					const int l2 = (int)floorf(i2);
					const float f2s = fsub(i2, (float)l2);
					const float i1 = fsub((float)q1, tf); // :750
					const int l1 = (int)floorf(i1);
					const float f1s = fsub(i1, (float)l1);
					const c2 inq = ld_c2s(&U.in[q & (WS_RING - 1)][lane]);
					const c2 pv = ld_c2s(&U.pv[nb][i][lane]);
					const c2 in1 = ld_c2s(&U.in[q1 & (WS_RING - 1)][lane]);
					const c2 lo2 = sel_c2(INTERIOR || l2 >= 0, ld_c2s(&U.in[l2 & (WS_RING - 1)][lane]));
					const c2 hi2 = sel_c2(INTERIOR || l2 >= -1, ld_c2s(&U.in[(l2 + 1) & (WS_RING - 1)][lane]));
					const c2 lo1 = sel_c2(INTERIOR || l1 >= 0, ld_c2s(&U.in[l1 & (WS_RING - 1)][lane]));
					const c2 hi1 = sel_c2(INTERIOR || l1 >= -1, ld_c2s(&U.in[(l1 + 1) & (WS_RING - 1)][lane]));
					// the previous block's Prediction::energy at bin q (:707): |its input|^2 on this path; lane 0: state / predecessor row
					f2 re;
					{
						const c2 pin = ld_c2s(&U.in[q & (WS_RING - 1)][lane > 0 ? lane - 1 : 0]);
						const f2 en = FAST ? fnorm2(pin) : xnorm2(pin, one);
						const float2 e0 = U.p0E[n & 3][i];
						re = f2_make(lane == 0 ? e0.x : f2_lo(en), lane == 0 ? e0.y : f2_hi(en));
					}
					const float2 rot = rotq;
					{
						const float2 rn = xmul(rotq, rotS); // the table recurrence stays in the reference's own arithmetic
						rotq = make_float2((INTERIOR || q >= 0) ? rn.x : rotq.x, (INTERIOR || q >= 0) ? rn.y : rotq.y);
					}
					c2 a, t1, t2;
					if constexpr (FAST) {
						const c2 fT = fmulc_c(inq, fmul_s(pv, rot));   // :653-654,:714
						const f2 e = fnorm2(inq);                        // :679
						const f2 den = f2_make(fmaxf(f2_lo(re), f2_lo(e)), fmaxf(f2_hi(re), f2_hi(e))) + f2_make(B200S_NOISE_FLOOR, B200S_NOISE_FLOOR);
						const f2 rden = f2_make(rcp_fast(f2_lo(den)), rcp_fast(f2_hi(den)));
						const c2 fr2 = fmul_s(fT, rot); // the rotation of Band::output (:653), folded into the factor
						a = c2{mul2(fr2.re, rden), mul2(fr2.im, rden)};
						t2 = fmulc_c(inq, flerp2(lo2, hi2, f2s));        // :758
						t1 = fmulc_c(in1, flerp2(lo1, hi1, f1s));        // :751,:771
					} else {
						const c2 pvr = xmul2s(pv, rot, one);             // :654
						a = xmulc2(inq, pvr, one);                       // :714
						const f2 e = xnorm2(inq, one);                   // :679
						const f2 den = f2_make(fmaxf(f2_lo(re), f2_lo(e)), fmaxf(f2_hi(re), f2_hi(e))) + f2_make(B200S_NOISE_FLOOR, B200S_NOISE_FLOOR);
						U.X[nb][i][lane] = make_float4(qIn ? f2_lo(den) : 1.f, qIn ? f2_hi(den) : 1.f, rot.x, rot.y); // (masked: a finite divisor for 0 / den)
						t2 = xmulc2(inq, xlerp2p(lo2, hi2, f2s, one), one);
						t1 = xmulc2(in1, xlerp2p(lo1, hi1, f1s, one), one);
					}
					// timeFactor <= 2: floor(b + 1 - timeFactor) is b or b - 1, so Prediction::input at bin b is one of the two
					// interpolation points of the short twist
					const c2 pB = sel_c2(bIn, c2{f2_make(l1 == b ? f2_lo(lo1.re) : f2_lo(hi1.re), l1 == b ? f2_hi(lo1.re) : f2_hi(hi1.re)),
					                              f2_make(l1 == b ? f2_lo(lo1.im) : f2_lo(hi1.im), l1 == b ? f2_hi(lo1.im) : f2_hi(hi1.im))});
					U.A[nb][i][lane] = pack_c2(sel_c2(qIn, a));
					U.T2[nb][i][lane] = pack_c2(sel_c2(INTERIOR || (qIn && q >= LT), t2)); // used at b = q (b >= L, :755) and at b = q - L (b < K - L, :776)
					U.T1[nb][i][lane] = pack_c2(sel_c2(q1In, t1));           // used at b = q1 (b > 0) and at b = q1 - 1 (b < K - 1, :766)
					U.P[nb][i][lane] = pack_c2(pB);
				}
			};
			// finals of chunk n -> planar Band::output rows, 32 B per row and quarter-warp; all tile reads first
			auto writeback = [&](int n) {
				const int buf = n & 1;
				float4 v[4];
#pragma unroll
				for (int it = 0; it < 4; ++it) v[it] = U.A[buf][fI][fF + 8 * it];
#pragma unroll
				for (int it = 0; it < 4; ++it) {
					const int fl = fF + 8 * it;
					const int b = n * WS_CH + fI - WS_G * fl - WS_D;
					if (fl < nAct && (unsigned)b < (unsigned)K) {
						float2 *row = yBase + (size_t)(2 * fl) * K + b;
						row[0] = make_float2(v[it].x, v[it].z);
						row[K] = make_float2(v[it].y, v[it].w);
					}
				}
			};
			// chunks [intFrom, intTo): lane 31's interpolation points (down to q - 8 - 1) and final bin are >= L, lane 0's q < K
			const int intFrom = nAct == 32 ? (WS_G * 31 + 16 + WS_CH - 1) / WS_CH : nChunks, intTo = (K - WS_CH + 1) / WS_CH;
			auto produce_any = [&](int n) {
				if (n >= intFrom && n < intTo) produce(n, std::true_type{});
				else produce(n, std::false_type{});
			};
			fill(0);
			if (nChunks > 1) fill(1);
			cp_async_wait_all();
			__syncwarp();
			produce_any(0);
			for (int n = 0; n < nChunks; ++n) {
				__syncthreads(); // tiles of chunk n complete; the consumer is done with chunk n-1
				cp_async_wait_all(); // raw spectra of chunk n+1 (issued one iteration ago)
				__syncwarp();
				if (n + 2 < nChunks) fill(n + 2); // in flight while chunk n+1 is produced: touches ring slots / buffers nobody reads now
				if (n >= 1) writeback(n - 1);
				__syncwarp();
				if (n + 1 < nChunks) produce_any(n + 1);
			}
			__syncthreads();
			writeback(nChunks - 1);
		} else {
			// =============================== CONSUMER ===============================
			// register FIFOs with compile-time rotation; at step t of a 12-step round (final bin b, prelim bin q = b + 6):
			//   pre / t2F [(t + u) % 6]  <-> preliminary output / long twist at bin b + u, u = 0..5
			//   oh [(t - 1 - u) & 3]     <-> final output at bin b - 1 - u;   t1P <-> short twist at bin b
			c2 pre[6], t2F[6], oh[4], t1P = zc, lastFinal = zc;
#pragma unroll
			for (int u = 0; u < 6; ++u) pre[u] = t2F[u] = zc;
#pragma unroll
			for (int u = 0; u < 4; ++u) oh[u] = zc;
			auto chunk = [&](int n, auto phTag) {
				constexpr int PH = decltype(phTag)::value;
				const int cb = n & 1;
				static_for<WS_CH>([&](auto ic) {
					constexpr int i = decltype(ic)::value, t = PH * WS_CH + i, h = t % 6;
					const c2 a = ld_c2s(&U.A[cb][i][lane]);
					const c2 t1N = ld_c2s(&U.T1[cb][i][lane]);
					const c2 t2N = ld_c2s(&U.T2[cb][i][lane]);
					const c2 inB = ld_c2s(&U.P[cb][i][lane]);
					// the previous block's final output at bin q: finalised by lane-1 in the last step (lane 0: its predecessor's row)
					c2 ro;
					{
						const float a0 = __shfl_up_sync(0xffffffffu, f2_lo(lastFinal.re), 1), a1 = __shfl_up_sync(0xffffffffu, f2_hi(lastFinal.re), 1);
						const float b0 = __shfl_up_sync(0xffffffffu, f2_lo(lastFinal.im), 1), b1 = __shfl_up_sync(0xffffffffu, f2_hi(lastFinal.im), 1);
						const float4 p0 = U.p0Out[n & 3][i];
						const bool first = lane == 0;
						ro = c2{f2_make(first ? p0.x : a0, first ? p0.z : a1), f2_make(first ? p0.y : b0, first ? p0.w : b1)};
					}
					c2 newPre;
					f2 eB;
					if constexpr (FAST) {
						newPre = fmul_c(ro, a); // :653,:714-716 with the bin's rotation, twist and denominator folded into `a`
						eB = fnorm2(inB);       // :679,:708 (identity map: Prediction::energy = |input|^2)
					} else {
						const float4 xv = U.X[cb][i][lane];
						const c2 ror = xmul2s(ro, make_float2(xv.z, xv.w), one);      // :653
						const c2 ph0 = xmul2(ror, a, one);                             // :715
						const f2 den = f2_make(xv.x, xv.y);
						newPre = c2{fdivq2(ph0.re, den), fdivq2(ph0.im, den)};         // :716
						eB = xnorm2(inB, one);
					}
					const c2 t2B = t2F[h], preN = pre[(h + 1) % 6], preL = pre[(h + LT) % 6], t2L = t2F[(h + LT) % 6];
					const c2 oh0 = oh[(t + 3) & 3], ohL = oh[(t + 4 - LT) & 3];
					pre[h] = newPre; // bin q = b + 6 takes the slot of bin b
					t2F[h] = t2N;
					// ---- main prediction at bin b (:727-800): the louder channel (first on ties, :733) leads
					const bool m = f2_hi(eB) > f2_lo(eB);
					const float maxE = m ? f2_hi(eB) : f2_lo(eB);
					c2 oc;
					if constexpr (FAST) {
						c2 ph2 = fmul_c(ohL, t2B);           // :761
						ph2 = fmulc_acc(ph2, preN, t1N);     // :774
						ph2 = fmulc_acc(ph2, preL, t2L);     // :784
						ph2 = fmul_acc(ph2, oh0, t1P);       // :754 (the term that closes the recurrence, last)
						const float2 phase = pick(m, ph2), pinM = pick(m, inB);
						const float2 outM = make_output_fast(phase, maxE, pinM); // :788
						const float2 inO = pick(!m, inB);
						const float eO = m ? f2_lo(eB) : f2_hi(eB);
						const float2 outO = make_output_fast(fmul_f(outM, fmulc_f(inO, pinM)), eO, inO); // :791-799
						oc = c2{f2_make(m ? outO.x : outM.x, m ? outM.x : outO.x), f2_make(m ? outO.y : outM.y, m ? outM.y : outO.y)};
					} else {
						// masked terms arrive as exact zeros (a twist of +-0 adds +-0 to the sum, which leaves it unchanged)
						c2 ph2 = zc;
						ph2 = ph2 + xmul2(oh0, t1P, one);    // :754
						ph2 = ph2 + xmul2(ohL, t2B, one);    // :761
						ph2 = ph2 + xmulc2(preN, t1N, one);  // :774
						ph2 = ph2 + xmulc2(preL, t2L, one);  // :784
						const float2 phase = pick(m, ph2), pinM = pick(m, inB);
						const float2 outM = make_output_q(phase, maxE, pinM); // :788
						const c2 tw = c2{padd(muls(inB.re, pinM.x), muls(inB.im, pinM.y), one), psub(muls(inB.im, pinM.x), muls(inB.re, pinM.y), one)};
						const c2 cph = c2{psub(muls(tw.re, outM.x), muls(tw.im, outM.y), one), padd(muls(tw.im, outM.x), muls(tw.re, outM.y), one)};
						const c2 other = make_output_q2(cph, eB, inB, one);
						oc = c2{f2_make(m ? f2_lo(other.re) : outM.x, m ? outM.x : f2_hi(other.re)),
						        f2_make(m ? f2_lo(other.im) : outM.y, m ? outM.y : f2_hi(other.im))};
					}
					oh[t & 3] = oc; // replaces the final of bin b - 4
					lastFinal = oc;
					t1P = t1N;
					U.A[cb][i][lane] = pack_c2(oc);
				});
			};
			for (int n = 0; n < nChunks;) {
				__syncthreads();
				chunk(n, std::integral_constant<int, 0>{});
				if (++n >= nChunks) break;
				__syncthreads();
				chunk(n, std::integral_constant<int, 1>{});
				if (++n >= nChunks) break;
				__syncthreads();
				chunk(n, std::integral_constant<int, 2>{});
				++n;
			}
			__syncthreads(); // the producer writes the last chunk back after this one
		}
	}
}

template <bool FAST>
static inline size_t smem_chain_ws() { return sizeof(WsTiles<FAST>); }

} // namespace b200s
