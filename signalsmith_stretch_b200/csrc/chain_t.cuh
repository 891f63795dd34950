// chain_t.cuh -- k_products + k_chain_t: the frequency-mapped / formant configurations with the chain-independent terms
// handed to the chain in STEP-MAJOR order (round 2).
//
// The generic path of round 1 (k_prep -> coefficient rows [block][bin] -> k_chain) made the chain warp turn rows into
// columns: per chunk of 8 steps every lane needs 8 bins of ITS OWN block's five coefficient rows, i.e. 40-80 small
// cp.async per lane, staged through [step][lane] shared-memory tiles, waited for before the chunk could start.
// Here the transposition happens once, in a throughput kernel:
//   * k_prep (map-only mode) stops after the serial-free part that needs a whole block in shared memory -- peaks,
//     output map, formant ratio -- and writes 12 B per bin: mapBin, mapGrad, ratio rows.
//   * k_products (grid: 32-step chunks x 32-block groups x streams) evaluates, per (block j, bin q), exactly what
//     k_prep's last stage evaluates -- Prediction::energy / input, freqTwist, the short and long vertical twists
//     (:696-719,:750-758) -- with lanes along the BINS of one block (the gathers at the mapped positions are then
//     nearly contiguous), collects a [32 steps][32 blocks] tile per quantity in shared memory and writes it out as rows
//     of 32 lanes: element (j, q) of every quantity lands at row k = (the step at which lane j consumes it), so
//     FT / T2 / E at k = q + D j, T1 at k = q + L - 1 + D j, PI at k = q + L + D j   (D = L + 1, the lane skew).
//   * k_chain_t (one warp per stream, lane = block, as k_chain) reads ROW k of every array at step k: five coalesced
//     128 / 256-byte loads per channel, next step's already in flight, no shared-memory staging, no index arithmetic.
// Arithmetic is the exact (unfused IEEE) arithmetic of k_prep / k_chain, operation for operation: the emulator tests
// compare it with the oracle bit for bit.  Streams with a random block (beyond 2x stretch) keep the round-1 kernels.
#pragma once
#include "kernels.cuh"

namespace b200s {

__host__ __device__ __forceinline__ int t_rows(const Cfg &g) { return ((g.K + g.L + (g.L + 1) * 31 + 1) + 31) & ~31; } // steps of a group, padded to 32
__device__ __forceinline__ size_t t_idx(const Ctx &x, int s, int grp, int k, int c, int lane) {
	return ((((size_t)s * x.tGroups + grp) * x.tRows + k) * x.cfg.C + c) * 32 + lane;
}

__global__ void __launch_bounds__(256) k_products(Ctx x) {
	const Cfg &g = x.cfg;
	const int K = g.K, LT = g.L, D = LT + 1;
	const int k0 = blockIdx.x * 32, grp = blockIdx.y, s = stream_at(x, x.sBase + blockIdx.z);
	const int i = threadIdx.x & 31, w = threadIdx.x >> 5;
	const Call cl = x.call[s];
	const int base = 32 * grp, nAct = min(32, cl.nFrames - base);
	// (plain streams of a mixed call: the direct chain writes their Y rows)
	if (cl.bypass || nAct <= 0 || !cl.mapped || (cl.hasRandom && x.randomPathOn)) return;
	B200S_SHARED float2 tFT[32][33], tT2[32][33], tT1[32][33], tPI[32][33];
	B200S_SHARED float tE[32][33];
	for (int c = 0; c < g.C; ++c) {
		for (int j = w; j < 32; j += 8) {
			float2 ft = make_float2(0.f, 0.f), t1 = ft, t2 = ft, pin = ft;
			float e = 0.f;
			const int q = k0 + i - D * j;
			// everything that depends on the block only: once per warp iteration (the lanes of a warp share j)
			const int f = base + min(j, nAct - 1);
			const Frame fr = x.frames[(size_t)s * x.maxFrames + f];
			const bool mapped = fr.flags & FR_MAPPED, formants = fr.flags & FR_FORMANTS, rotOn = fr.flags & FR_NEW_SPECTRUM;
			const float2 *inRow = spec_slot(x, s, fr.inSlot, c), *pvRow = spec_slot(x, s, fr.prevSlot, c); // (mapped calls: planar spectra)
			const size_t row = ((size_t)s * x.maxFrames + f) * K;
			const float *mapB = x.cMapB + row, *mapG = x.cMapG + row, *ratio = x.cRatio + row;
			float *eRow = x.cE + coef_off(x, s, f, c);
			const float tf = fmaxf(fr.timeFactor, 1.0f / B200S_MAX_CLEAN_STRETCH); // :638
			const float longTf = fmul((float)LT, tf);
			if (j < nAct && q >= 0 && q < K) {
				// gathers without branches: clamped address, value selected afterwards (zero outside the spectrum, :564-568)
				auto gin = [&](int b) {
					const float2 v = inRow[min(max(b, 0), K - 1)];
					const bool in = (unsigned)b < (unsigned)K;
					return make_float2(in ? v.x : 0.f, in ? v.y : 0.f);
				};
				auto gpv = [&](int b) { // prevInput is rotated in place before being interpolated (:654)
					const int bc = min(max(b, 0), K - 1);
					const float2 v = pvRow[bc], vr = xmul(v, __ldg(x.rot + bc));
					const bool in = (unsigned)b < (unsigned)K;
					return make_float2(in ? (rotOn ? vr.x : v.x) : 0.f, in ? (rotOn ? vr.y : v.y) : 0.f);
				};
				const float mb = mapped ? mapB[q] : (float)q;
				const float mg = mapped ? mapG[q] : 1.f;
				const int lo = (int)floorf(mb);
				const float frac = fsub(mb, (float)lo);
				const float2 inLo = gin(lo), inHi = gin(lo + 1);
				float eLo = xnorm(inLo), eHi = xnorm(inHi); // Band::inputEnergy (:679,:826)
				if (formants) {
					const float rLo = ratio[min(max(lo, 0), K - 1)], rHi = ratio[min(max(lo + 1, 0), K - 1)];
					eLo = (unsigned)lo < (unsigned)K ? fmul(eLo, rLo) : eLo;
					eHi = (unsigned)(lo + 1) < (unsigned)K ? fmul(eHi, rHi) : eHi;
				}
				e = fmul(xlerp(eLo, eHi, frac), fmaxf(0.f, mg)); // :708-709
				pin = xlerp2(inLo, inHi, frac);                  // :710
				const float2 pprev = xlerp2(gpv(lo), gpv(lo + 1), frac); // :713
				ft = xmulc(pin, pprev);                          // :714
				const float i1 = fsub(mb, tf); // :750-751
				const int l1 = (int)floorf(i1);
				t1 = xmulc(pin, xlerp2(gin(l1), gin(l1 + 1), fsub(i1, (float)l1)));
				const float i2 = fsub(mb, longTf); // :757-758
				const int l2 = (int)floorf(i2);
				t2 = xmulc(pin, xlerp2(gin(l2), gin(l2 + 1), fsub(i2, (float)l2)));
				eRow[q] = e; // row layout too: the state carry (k_commit, next group's first lane) reads it
			}
			tFT[i][j] = ft;
			tT2[i][j] = t2;
			tT1[i][j] = t1;
			tPI[i][j] = pin;
			tE[i][j] = e;
		}
		__syncthreads();
		const size_t a0 = t_idx(x, s, grp, k0, c, i), st = (size_t)g.C * 32; // element of row k0; elements per row
		for (int r = w; r < 32; r += 8) { // rows of 32 lanes; T1 / PI are consumed L-1 / L steps after the step of their bin
			const int k = k0 + r;
			const size_t a = a0 + (size_t)r * st;
			if (k < x.tRows) {
				x.tFT[a] = tFT[r][i];
				x.tT2[a] = tT2[r][i];
				x.tE[a] = tE[r][i];
			}
			if (k + LT - 1 < x.tRows) x.tT1[a + (size_t)(LT - 1) * st] = tT1[r][i];
			if (k + LT < x.tRows) x.tPI[a + (size_t)LT * st] = tPI[r][i];
		}
		__syncthreads();
	}
}

#define CT_CH 12 // steps per chunk: rows rotate through 3 register sets and the FIFOs through L slots, so 12 steps (L in
                 // {1,2,3,4,6}) bring every rotation back to its start and the steps are unrolled with compile-time renaming only
struct ChainTY { // finals of a chunk, [step][lane]
	float2 y[2][CT_CH][CHAIN_RS2];
};

template <int CT, int LT>
__global__ void __launch_bounds__(32) k_chain_t(Ctx x) {
	const Cfg &g = x.cfg;
	const int K = g.K;
	const int lane = threadIdx.x & 31;
	const int s = stream_at(x, x.sBase + blockIdx.x);
	// plain streams of a mixed call: the direct chain.  (A separate read-only load: testing the field of `cl` below costs the
	// L = 8 stereo instantiation 60 more bytes of spills.)
	if (!__ldg(&x.call[s].mapped)) return;
	const Call cl = x.call[s];
	if (cl.nFrames == 0) return;
	if (cl.hasRandom && x.randomPathOn) return; // random time factors: k_prep + k_chain take the stream
	constexpr int D = LT + 1;
	constexpr bool ROT = (CT_CH % LT) == 0; // FIFO slots by compile-time rotation; otherwise (L = 5, 7, 8) they are shifted
	B200S_SHARED ChainTY T;

	for (int base = 0, grp = 0; base < cl.nFrames; base += 32, ++grp) {
		__syncwarp(); // lane 31's Y of the previous group must be visible to lane 0's loads
		const int f = base + lane;
		const bool active = f < cl.nFrames;
		const Frame fr = x.frames[(size_t)s * x.maxFrames + (active ? f : base)];
		const bool rotOn = fr.flags & FR_NEW_SPECTRUM;
		const int nAct = min(32, cl.nFrames - base);
		const float2 *prevOut[CT];
		const float *prevE[CT];
#pragma unroll
		for (int c = 0; c < CT; ++c) {
			prevOut[c] = base == 0 ? x.stOut + ((size_t)s * CT + c) * K : x.Y + coef_off(x, s, base - 1, c);
			prevE[c] = base == 0 ? x.stPredE + ((size_t)s * CT + c) * K : x.cE + coef_off(x, s, base - 1, c);
		}
		// per-lane register FIFOs.  Rotating form (ROT), at step t: slot t % L holds the values of bin b (pushed L steps ago) and
		// takes those of bin q = b + L; the final of bin b - 1 - u sits in slot (t - 1 - u) % L.  Shifted form: as k_chain.
		float2 outHist[CT][LT], pre[CT][LT], t2Fifo[CT][LT], t1Prev[CT], lastFinal[CT];
		float eFifo[CT][LT], lastE[CT];
#pragma unroll
		for (int c = 0; c < CT; ++c) {
#pragma unroll
			for (int u = 0; u < LT; ++u) {
				outHist[c][u] = pre[c][u] = t2Fifo[c][u] = make_float2(0.f, 0.f);
				eFifo[c][u] = 0.f;
			}
			t1Prev[c] = lastFinal[c] = make_float2(0.f, 0.f);
			lastE[c] = 0.f;
		}
		const int steps = K + LT + D * (nAct - 1);
		// row k of the step-major arrays: this lane's terms of step k (k_products), fetched two steps ahead
		struct Row {
			float2 ft[CT], t2[CT], t1[CT], pi[CT], p0[CT];
			float e[CT], p0e[CT];
			float2 rot; // rot[q] of the step (:647-655 table), fetched with the row so that nothing waits for it
		};
		const size_t a00 = t_idx(x, s, grp, 0, 0, lane);
		const float2 *pFT = x.tFT + a00, *pT2 = x.tT2 + a00, *pT1 = x.tT1 + a00, *pPI = x.tPI + a00;
		const float *pE = x.tE + a00;
		auto load_row = [&](int k, Row &r) {
			const int q = k - D * lane;
			r.rot = __ldg(x.rot + min(max(q, 0), K - 1));
#pragma unroll
			for (int c = 0; c < CT; ++c) {
				const size_t a = ((size_t)k * CT + c) * 32;
				r.ft[c] = pFT[a];
				r.t2[c] = pT2[a];
				r.t1[c] = pT1[a];
				r.pi[c] = pPI[a];
				r.e[c] = pE[a];
				// lane 0's predecessor block: last call's state or the previous group's rows, at bin q = k
				const bool p = lane == 0 && q < K;
				r.p0[c] = p ? prevOut[c][q] : make_float2(0.f, 0.f);
				r.p0e[c] = p ? prevE[c][q] : 0.f;
			}
		};
		Row rows[3]; // rows[t % 3]: the row of step t; the one of step t + 2 is loaded while step t is computed
		load_row(0, rows[0]);
		load_row(1, rows[1]);
		for (int k0 = 0; k0 < steps; k0 += CT_CH) {
			static_for<CT_CH>([&](auto tc) {
				constexpr int t = decltype(tc)::value;
				const Row &cur = rows[t % 3];
				const int k = k0 + t;
				const int q = k - D * lane;
				const int b = q - LT;
				if (k + 2 < x.tRows) load_row(k + 2, rows[(t + 2) % 3]);
				// previous block's final output / energy at bin q: finalised by lane-1 last step
				float2 recvOut[CT];
				float recvE[CT];
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					recvOut[c].x = __shfl_up_sync(0xffffffffu, lastFinal[c].x, 1);
					recvOut[c].y = __shfl_up_sync(0xffffffffu, lastFinal[c].y, 1);
					recvE[c] = __shfl_up_sync(0xffffffffu, lastE[c], 1);
				}
				const bool qIn = active && q >= 0 && q < K;
				if (lane == 0 && qIn) {
#pragma unroll
					for (int c = 0; c < CT; ++c) {
						recvOut[c] = cur.p0[c];
						recvE[c] = cur.p0e[c];
					}
				}
				// preliminary prediction at bin q (:712-716)
				float2 newPre[CT], newT2[CT];
				float newE[CT];
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					newPre[c] = make_float2(0.f, 0.f);
					newT2[c] = make_float2(0.f, 0.f);
					newE[c] = 0.f;
					if (qIn) {
						const float e = cur.e[c];
						newT2[c] = cur.t2[c];
						float2 o = recvOut[c];
						if (rotOn) o = xmul(o, cur.rot); // :653
						const float2 phase = xmul(o, cur.ft[c]);  // :715
						const float den = fadd(fmaxf(recvE[c], e), B200S_NOISE_FLOOR);
						newPre[c] = make_float2(fdivq(phase.x, den), fdivq(phase.y, den)); // :716 (branch-free, correctly rounded: kernels.cuh)
						newE[c] = e;
					}
				}
				// what belongs to bin b leaves the FIFOs, the values of bin q enter
				constexpr int S0 = ROT ? t % LT : 0;                    // slot of bin b (and, afterwards, of bin q)
				constexpr int S1 = ROT ? (t + 1) % LT : 0;              // bin b + 1 (after the push)
				constexpr int SQ = ROT ? t % LT : LT - 1;               // bin q (after the push)
				constexpr int H1 = ROT ? (t + LT - 1) % LT : 0;         // final of bin b - 1
				constexpr int HL = ROT ? t % LT : LT - 1;               // final of bin b - L
				float eAtB[CT];
				float2 t2AtB[CT];
#pragma unroll
				for (int c = 0; c < CT; ++c) {
					eAtB[c] = eFifo[c][S0];
					t2AtB[c] = t2Fifo[c][S0];
					if constexpr (!ROT) {
#pragma unroll
						for (int u = 0; u + 1 < LT; ++u) {
							pre[c][u] = pre[c][u + 1];
							eFifo[c][u] = eFifo[c][u + 1];
							t2Fifo[c][u] = t2Fifo[c][u + 1];
						}
					}
					pre[c][SQ] = newPre[c];
					eFifo[c][SQ] = newE[c];
					t2Fifo[c][SQ] = newT2[c];
				}
				// main prediction at bin b (:727-800)
				if (active && b >= 0 && b < K) {
					int m = 0;
					float maxE = eAtB[0];
#pragma unroll
					for (int c = 1; c < CT; ++c) {
						if (eAtB[c] > maxE) { // :733
							m = c;
							maxE = eAtB[c];
						}
					}
					float2 t1Next[CT], pin[CT];
#pragma unroll
					for (int c = 0; c < CT; ++c) {
						t1Next[c] = (b < K - 1) ? cur.t1[c] : make_float2(0.f, 0.f);
						pin[c] = cur.pi[c];
					}
					// (L = 1: bin b + 1 IS bin q, i.e. slot SQ)
					float2 oh1 = outHist[0][H1], ohL = outHist[0][HL], pr1 = pre[0][LT == 1 ? SQ : S1], prL = pre[0][SQ];
					float2 t1b = t1Prev[0], t2b = t2AtB[0], t1n = t1Next[0], t2n = t2Fifo[0][SQ], pinM = pin[0];
#pragma unroll
					for (int c = 1; c < CT; ++c) {
						if (m == c) {
							oh1 = outHist[c][H1];
							ohL = outHist[c][HL];
							pr1 = pre[c][LT == 1 ? SQ : S1];
							prL = pre[c][SQ];
							t1b = t1Prev[c];
							t2b = t2AtB[c];
							t1n = t1Next[c];
							t2n = t2Fifo[c][SQ];
							pinM = pin[c];
						}
					}
					float2 phase = make_float2(0.f, 0.f);
					if (b > 0) {
						phase = xadd(phase, xmul(oh1, t1b));              // :754
						if (b >= LT) phase = xadd(phase, xmul(ohL, t2b)); // :761
					}
					if (b < K - 1) {
						phase = xadd(phase, xmulc(pr1, t1n));                  // :774
						if (b < K - LT) phase = xadd(phase, xmulc(prL, t2n)); // :784
					}
					const float2 outM = make_output_q(phase, maxE, pinM); // :788
#pragma unroll
					for (int c = 0; c < CT; ++c) {
						float2 oc = outM;
						if (c != m) { // all other channels are locked in phase (:791-799)
							const float2 cph = xmul(outM, xmulc(pin[c], pinM));
							oc = make_output_q(cph, eAtB[c], pin[c]);
						}
						if constexpr (!ROT) {
#pragma unroll
							for (int u = LT - 1; u > 0; --u) outHist[c][u] = outHist[c][u - 1];
						}
						outHist[c][ROT ? t % LT : 0] = oc; // (rotating: replaces the final of bin b - L, read above)
						lastFinal[c] = oc;
						lastE[c] = eAtB[c];
						t1Prev[c] = t1Next[c];
						T.y[c][t][lane] = oc;
					}
				}
			});
			__syncwarp();
			// ---------------- write the chunk's finals back: 32 B (4 bins) per frame and quarter-warp ----------------
#pragma unroll
			for (int m4 = 0; m4 < CT_CH / 4; ++m4) {
#pragma unroll
				for (int it = 0; it < 4; ++it) {
					const int t = 4 * m4 + (lane & 3), fl = (lane >> 2) + 8 * it, ff = base + fl;
					const int b = k0 + t - D * fl - LT;
					if (ff < cl.nFrames && b >= 0 && b < K) {
#pragma unroll
						for (int c = 0; c < CT; ++c) x.Y[coef_off(x, s, ff, c) + b] = T.y[c][t][fl];
					}
				}
			}
			__syncwarp();
		}
	}
}

} // namespace b200s
