// chain_direct.cuh -- k_chain_direct: the frame-wavefront phase prediction for calls WITHOUT a
// frequency map and WITHOUT formant processing (pure time-stretch, reference :675-686 identity
// map).  Same algorithm and same bit-exact arithmetic as k_chain (kernels.cuh) -- see the comment
// there for the wavefront -- but specialised and instruction-lean, because this is the kernel the
// BASELINE benchmark configuration spends its time in:
//   * Prediction::energy/input (:708-710), freqTwist (:714) and the short/long vertical twists
//     (:750-758,:770-781) are formed on the fly from the analysis spectra, staged through a rolling
//     32-bin shared-memory window per lane (16 B per bin-channel from HBM, k_prep not launched);
//   * the CHAIN_CH steps of a chunk are fully unrolled, so the register FIFOs rotate by renaming;
//   * edge conditions are selects, not branches; the per-bin rotation (:647-655) is the
//     reference's own float recurrence carried in registers instead of a table lookup;
//   * row pointers of the 32 blocks live in shared memory, so the cp.async fill and the write-back
//     of a chunk are a handful of predicated instructions per lane.
#pragma once
#include <type_traits>

#include "kernels.cuh"

namespace b200s {

template <int CT>
struct DirectTiles2 { // one per warp
	float2 in[CT][CHAIN_RING][CHAIN_RS2]; // rolling window of each block's input spectrum, row = bin & 31
	float2 pv[CT][CHAIN_CH][CHAIN_RS2];   // previous-input spectrum at the chunk's prelim bins
	float2 y[CT][CHAIN_CH][CHAIN_RS2];    // finals of the chunk
	float2 p0Out[CT][CHAIN_CH];           // lane 0's predecessor block (state or previous group)
	float p0E[CT][CHAIN_CH];
	const float2 *rowIn[CT][32], *rowPv[CT][32];
	float2 *rowY[CT][32];
};

__device__ __forceinline__ float2 sel2(bool p, float2 a) { return make_float2(p ? a.x : 0.f, p ? a.y : 0.f); }

template <int CT, int LT>
__global__ void __launch_bounds__(32) k_chain_direct(Ctx x) {
	const Cfg &g = x.cfg;
	const int K = g.K;
	B200S_DYN_SHARED
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int pos = x.sBase + blockIdx.x * (blockDim.x >> 5) + warp;
	if (pos >= x.sBase + x.sCount) return;
	const int s = stream_at(x, pos);
	const Call cl = x.call[s];
	if (cl.nFrames == 0) return;
	if (cl.mapped || (cl.hasRandom && x.randomPathOn)) return; // a block beyond 2x stretch draws random time factors: k_prep + k_chain take the stream
	constexpr int D = LT + 1;
	DirectTiles2<CT> &U = ((DirectTiles2<CT> *)dyn_smem)[warp];
	const int fillI = lane & 7, fillF = lane >> 3;
	const float2 rot0 = x.rot0, rotStep = x.rotStep;

	for (int base = 0; base < cl.nFrames; base += 32) {
		__syncwarp();
		const int f = base + lane;
		const bool active = f < cl.nFrames;
		const Frame fr = x.frames[(size_t)s * x.maxFrames + (active ? f : base)];
		const bool rotOn = fr.flags & FR_NEW_SPECTRUM;
		const int nAct = min(32, cl.nFrames - base);
		const bool carryE = active && (lane == 31 || f == cl.nFrames - 1); // Prediction::energy needed later
		const float tf = fmaxf(fr.timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH); // :638
		const float longTf = fmul((float)LT, tf);
		// stretch beyond 2x: the interpolation points fall outside the staged window; the whole warp then
		// takes the slow variant of the step (gathers from HBM)
		const bool farAny = __any_sync(0xffffffffu, active && longTf > (float)(CHAIN_RING - CHAIN_CH - 3));
		const float2 *prevOut[CT];
		const float *prevE[CT];
		const float2 *myIn[CT];
		float *myE[CT];
#pragma unroll
		for (int c = 0; c < CT; ++c) {
			prevOut[c] = base == 0 ? x.stOut + ((size_t)s * CT + c) * K : x.Y + coef_off(x, s, base - 1, c);
			prevE[c] = base == 0 ? x.stPredE + ((size_t)s * CT + c) * K : x.cE + coef_off(x, s, base - 1, c);
			myIn[c] = spec_slot(x, s, fr.inSlot, c);
			myE[c] = x.cE + coef_off(x, s, active ? f : base, c);
			U.rowIn[c][lane] = myIn[c];
			U.rowPv[c][lane] = spec_slot(x, s, fr.prevSlot, c);
			U.rowY[c][lane] = x.Y + coef_off(x, s, active ? f : base, c);
		}
		__syncwarp();
		// register FIFOs; at the start of a step (q = prelim bin, b = q - L = final bin):
		//   pre/eF/t2F/inF[c][i] <-> prelim output / energy / long twist / input at bin b+i
		//   oh[c][i] <-> final output at bin b-1-i;   t1P[c] <-> short twist at bin b
		float2 oh[CT][LT], pre[CT][LT], t2F[CT][LT], inF[CT][LT], t1P[CT], lastFinal[CT];
		float eF[CT][LT], lastE[CT];
#pragma unroll
		for (int c = 0; c < CT; ++c) {
#pragma unroll
			for (int i = 0; i < LT; ++i) {
				oh[c][i] = pre[c][i] = t2F[c][i] = inF[c][i] = make_float2(0.f, 0.f);
				eF[c][i] = 0.f;
			}
			t1P[c] = lastFinal[c] = make_float2(0.f, 0.f);
			lastE[c] = 0.f;
		}
		// rot[q] for this lane's current q (valid once q >= 0); blocks without a new spectrum are not
		// rotated (:642): multiplying by 1+0i is exact, so they just carry the identity
		float2 rotq = rotOn ? rot0 : make_float2(1.f, 0.f);
		const float2 rotS = rotOn ? rotStep : make_float2(1.f, 0.f);
		const int steps = K + LT + D * (nAct - 1);
		for (int k0 = 0; k0 < steps; k0 += CHAIN_CH) {
			// ---------------- stage the chunk: 8 new bins per block ----------------
#pragma unroll
			for (int it = 0; it < 8; ++it) {
				const int fl = fillF + 4 * it;
				const int q = k0 + fillI - D * fl;
				if (base + fl < cl.nFrames && (unsigned)q < (unsigned)K) {
#pragma unroll
					for (int c = 0; c < CT; ++c) {
						cp_async8(&U.in[c][q & (CHAIN_RING - 1)][fl], U.rowIn[c][fl] + q);
						cp_async8(&U.pv[c][fillI][fl], U.rowPv[c][fl] + q);
					}
				}
			}
			if (lane < CHAIN_CH && k0 + lane < K) {
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					cp_async8(&U.p0Out[c][lane], prevOut[c] + k0 + lane);
					cp_async4(&U.p0E[c][lane], prevE[c] + k0 + lane);
				}
			}
			cp_async_wait_all();
			__syncwarp();
			// ---------------- CHAIN_CH steps ----------------
			auto step = [&](const int i, auto farTag) {
				constexpr bool FAR = decltype(farTag)::value;
				const int q = k0 + i - D * lane;
				const int b = q - LT;
				const bool qIn = active && (unsigned)q < (unsigned)K;
				const bool bIn = active && (unsigned)b < (unsigned)K;
				// the twists need input interpolated at q - L*tf and (b+1) - tf  (:750,:757)
				const float i2 = fsub((float)q, longTf);
				const int l2 = (int)floorf(i2);
				const float f2 = fsub(i2, (float)l2);
				const float i1 = fsub((float)(b + 1), tf);
				const int l1 = (int)floorf(i1);
				const float f1 = fsub(i1, (float)l1);
				float2 newPre[CT], newT2[CT], newIn[CT], t1N[CT];
				float newE[CT];
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					// previous block's final output / energy at bin q: finalised by lane-1 last step
					float2 ro;
					ro.x = __shfl_up_sync(0xffffffffu, lastFinal[c].x, 1);
					ro.y = __shfl_up_sync(0xffffffffu, lastFinal[c].y, 1);
					float re = __shfl_up_sync(0xffffffffu, lastE[c], 1);
					{
						const float2 p0 = U.p0Out[c][i];
						const float p0e = U.p0E[c][i];
						ro = make_float2(lane == 0 ? p0.x : ro.x, lane == 0 ? p0.y : ro.y);
						re = lane == 0 ? p0e : re;
					}
					const float2 inq = U.in[c][q & (CHAIN_RING - 1)][lane];
					float2 pv = U.pv[c][i][lane];
					float2 lo2, hi2, lo1, hi1;
					if constexpr (!FAR) {
						lo2 = sel2(l2 >= 0, U.in[c][l2 & (CHAIN_RING - 1)][lane]);
						hi2 = sel2(l2 >= -1, U.in[c][(l2 + 1) & (CHAIN_RING - 1)][lane]);
						lo1 = sel2(l1 >= 0, U.in[c][l1 & (CHAIN_RING - 1)][lane]);
						hi1 = sel2(l1 >= -1, U.in[c][(l1 + 1) & (CHAIN_RING - 1)][lane]);
					} else { // extreme stretch (> 2x): gather straight from the spectrum row
						lo2 = spec_at(myIn[c], l2, K);
						hi2 = spec_at(myIn[c], l2 + 1, K);
						lo1 = spec_at(myIn[c], l1, K);
						hi1 = spec_at(myIn[c], l1 + 1, K);
					}
					pv = xmul(pv, rotq); // :653-654 rotate Band::output and Band::prevInput by one interval
					ro = xmul(ro, rotq);
					const float e = xnorm(inq);                           // :679 (identity map: energy = |input|^2)
					const float2 phase = xmul(ro, xmulc(inq, pv));         // :714-715
					const float den = fadd(fmaxf(re, e), B200S_NOISE_FLOOR);
					newPre[c] = sel2(qIn, make_float2(fdivq(phase.x, den), fdivq(phase.y, den))); // :716
					newE[c] = qIn ? e : 0.f;
					newIn[c] = sel2(qIn, inq);
					newT2[c] = sel2(qIn, xmulc(inq, xlerp2(lo2, hi2, f2))); // long twist at q (:758)
					// short twist at b+1 (:751,:771): Prediction::input[b+1] is inF[c][1] before the shift
					t1N[c] = xmulc(LT > 1 ? inF[c][LT > 1 ? 1 : 0] : newIn[c], xlerp2(lo1, hi1, f1));
				}
				{
					const float2 rn = xmul(rotq, rotS);
					rotq = make_float2(q >= 0 ? rn.x : rotq.x, q >= 0 ? rn.y : rotq.y);
				}
				// ---- FIFO rotation (pure renaming after unrolling): what falls out belongs to bin b
				float eB[CT];
				float2 t2B[CT], inB[CT];
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					eB[c] = eF[c][0];
					t2B[c] = t2F[c][0];
					inB[c] = inF[c][0];
#pragma unroll
					for (int u = 0; u + 1 < LT; ++u) {
						pre[c][u] = pre[c][u + 1];
						eF[c][u] = eF[c][u + 1];
						t2F[c][u] = t2F[c][u + 1];
						inF[c][u] = inF[c][u + 1];
					}
					pre[c][LT - 1] = newPre[c];
					eF[c][LT - 1] = newE[c];
					t2F[c][LT - 1] = newT2[c];
					inF[c][LT - 1] = newIn[c];
				}
				// ---- main prediction at bin b (:727-800)
				int m = 0;
				float maxE = eB[0];
#pragma unroll
				for (int c = 1; c < CT; ++c) {
					if (eB[c] > maxE) { // :733
						m = c;
						maxE = eB[c];
					}
				}
				float2 oh1 = oh[0][0], ohL = oh[0][LT - 1], pr1 = pre[0][0], prL = pre[0][LT - 1];
				float2 t1b = t1P[0], t2b = t2B[0], t1n = t1N[0], t2n = t2F[0][LT - 1], pinM = inB[0];
#pragma unroll
				for (int c = 1; c < CT; ++c) {
					if (m == c) {
						oh1 = oh[c][0]; ohL = oh[c][LT - 1]; pr1 = pre[c][0]; prL = pre[c][LT - 1];
						t1b = t1P[c]; t2b = t2B[c]; t1n = t1N[c]; t2n = t2F[c][LT - 1]; pinM = inB[c];
					}
				}
				float2 phase = make_float2(0.f, 0.f);
				phase = xadd(phase, sel2(b > 0, xmul(oh1, t1b)));         // :754
				phase = xadd(phase, sel2(b >= LT, xmul(ohL, t2b)));       // :761
				phase = xadd(phase, sel2(b < K - 1, xmulc(pr1, t1n)));    // :774
				phase = xadd(phase, sel2(b < K - LT, xmulc(prL, t2n)));   // :784
				const float2 outM = make_output_q(phase, maxE, pinM);     // :788
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					float2 oc = outM;
					if (CT > 1) {
						const float2 cph = xmul(outM, xmulc(inB[c], pinM)); // :796-797
						const float2 other = make_output_q(cph, eB[c], inB[c]);
						if (c != m) oc = other;
					}
					// unconditional: out-of-range steps only produce values that every consumer masks
#pragma unroll
					for (int u = LT - 1; u > 0; --u) oh[c][u] = oh[c][u - 1];
					oh[c][0] = oc;
					lastFinal[c] = oc;
					lastE[c] = eB[c];
					t1P[c] = t1N[c];
					if (carryE && bIn) myE[c][b] = eB[c];
					U.y[c][i][lane] = oc;
				}
			};
			if (!farAny) { // fully unrolled, branch-free: one basic block the scheduler can interleave
#pragma unroll
				for (int i = 0; i < CHAIN_CH; ++i) step(i, std::false_type{});
			} else {
#pragma unroll 1
				for (int i = 0; i < CHAIN_CH; ++i) step(i, std::true_type{});
			}
			__syncwarp();
			// ---------------- write the chunk's finals back, 64 B per block ----------------
#pragma unroll
			for (int it = 0; it < 8; ++it) {
				const int fl = fillF + 4 * it;
				const int b = k0 + fillI - D * fl - LT;
				if (base + fl < cl.nFrames && (unsigned)b < (unsigned)K) {
#pragma unroll
					for (int c = 0; c < CT; ++c) U.rowY[c][fl][b] = U.y[c][fillI][fl];
				}
			}
			__syncwarp();
		}
	}
}

} // namespace b200s
