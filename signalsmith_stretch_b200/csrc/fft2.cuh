// fft2.cuh -- PAIRED in-place shared-memory FFT for the preset sizes (K = 3072 = 16*16*12 and
// K = 2560 = 16*16*10 complex points; reference call sites signalsmith-stretch.h:337,359,398 via
// the dependency's modified real FFT, SURVEY.md App. F).
//
// Design:
//   * TWO independent transforms (two channels, or the block and its re-analysed predecessor, or two
//     consecutive blocks) run in one CTA, element-wise interleaved as float4 {re_a, re_b, im_a, im_b}.
//     Every butterfly operation acts on the pair (f2 below), every shared-memory access is one LDS.128 /
//     STS.128, and the twiddle / address arithmetic is shared by the two transforms: fewer issue slots
//     per transform than a scalar FFT, whose kernels are issue-bound.
//   * IN-PLACE: a pass reads R elements into registers, does the radix-R butterfly and writes the
//     results to the SAME R slots, so one buffer (K float4 + padding) suffices and no pass needs a
//     barrier between its loads and stores.  Three passes 16 x 16 x R3 (R3 = 12 or 10).
//   * The first and the last pass are FUSED with the caller's data movement, which removes two of the
//     six shared-memory sweeps (the kernels were bound by shared-memory wavefronts and issue slots):
//       - analysis: decimation in time.  The thread that windows and pre-twiddles its R3 input samples
//         does the first (radix R3) butterfly on them in registers; the last radix-16 pass leaves the
//         spectrum in registers in natural order and the caller stores it (k_analyse2: back into the
//         buffer in bin order, from where bulk copies take whole rows to HBM).
//       - synthesis: decimation in frequency.  The first radix-16 pass takes its inputs from the caller
//         (k_synth2 reads them from the spectra staged in the buffer); the last pass leaves the time samples
//         in registers.
//   * Inter-pass twiddles: w, w^2, w^4, w^8 of the thread's (fixed) item are loaded once (analysis: for the
//     lifetime of the CTA; synthesis: before each pass), the other powers are products of at most three of them.
// No cuFFT, no tensor cores.  Generic sizes use the scalar Stockham FFT of fft.cuh.
#pragma once
#include "common.cuh"
#include "fft.cuh"

namespace b200s {

// ---- f2: two floats operated on element-wise ----
// sm_90 has no packed FP32 instructions, so each operation is two scalar ones.  The explicit .rn intrinsics are never
// contracted into multiply-adds by the compiler, so every element is rounded exactly like the scalar kernels.
struct f2 { float a, b; };
__device__ __forceinline__ f2 f2_make(float a, float b) { return f2{a, b}; }
__device__ __forceinline__ float f2_lo(f2 v) { return v.a; }
__device__ __forceinline__ float f2_hi(f2 v) { return v.b; }
__device__ __forceinline__ f2 operator+(f2 x, f2 y) { return f2{__fadd_rn(x.a, y.a), __fadd_rn(x.b, y.b)}; }
__device__ __forceinline__ f2 operator-(f2 x, f2 y) { return f2{__fsub_rn(x.a, y.a), __fsub_rn(x.b, y.b)}; }
__device__ __forceinline__ f2 muls(f2 x, float s) { return f2{__fmul_rn(x.a, s), __fmul_rn(x.b, s)}; } // x * s
__device__ __forceinline__ f2 fmas(f2 x, float s, f2 z) { return f2{__fmaf_rn(x.a, s, z.a), __fmaf_rn(x.b, s, z.b)}; } // x * s + z
__device__ __forceinline__ f2 mul2(f2 x, f2 y) { return f2{__fmul_rn(x.a, y.a), __fmul_rn(x.b, y.b)}; }

// two complex numbers (one per transform of the pair)
struct c2 {
	f2 re, im;
};
__device__ __forceinline__ c2 operator+(c2 a, c2 b) { return c2{a.re + b.re, a.im + b.im}; }
__device__ __forceinline__ c2 operator-(c2 a, c2 b) { return c2{a.re - b.re, a.im - b.im}; }
// a * (c + i*s)
__device__ __forceinline__ c2 cmulw(c2 a, float c, float s) {
	return c2{fmas(a.im, -s, muls(a.re, c)), fmas(a.re, s, muls(a.im, c))};
}
// a + (-i)*b and a - (-i)*b (forward); INV swaps the two
template <bool INV>
__device__ __forceinline__ c2 add_mi(c2 a, c2 b) { // a + w*b, w = -i (forward) / +i (inverse)
	return INV ? c2{a.re - b.im, a.im + b.re} : c2{a.re + b.im, a.im - b.re};
}
template <bool INV>
__device__ __forceinline__ c2 sub_mi(c2 a, c2 b) { // a - w*b
	return INV ? c2{a.re + b.im, a.im - b.re} : c2{a.re - b.im, a.im + b.re};
}
template <bool INV>
__device__ __forceinline__ c2 rot90p(c2 a) { // w*a, w = -i (forward) / +i (inverse): pure renaming + one negation folded by ptxas
	const f2 z = f2_make(0.f, 0.f);
	return INV ? c2{z - a.im, a.re} : c2{a.im, z - a.re};
}

// a * exp(-+2*pi*i*M/R), M and R compile-time
template <int R, int M, bool INV>
__device__ __forceinline__ c2 twmul2(c2 a) {
	constexpr int m = ((M % R) + R) % R;
	if constexpr (m == 0) {
		return a;
	} else if constexpr (2 * m == R) {
		const f2 z = f2_make(0.f, 0.f);
		return c2{z - a.re, z - a.im};
	} else if constexpr (4 * m == R) {
		return rot90p<INV>(a);
	} else if constexpr (4 * m == 3 * R) {
		return rot90p<!INV>(a);
	} else {
		constexpr float c = float(ct::cosq(m, R));
		constexpr float s = INV ? float(ct::sinq(m, R)) : -float(ct::sinq(m, R));
		return cmulw(a, c, s);
	}
}

template <int R, bool INV>
struct PairDFT;
template <bool INV>
struct PairDFT<2, INV> {
	static __device__ __forceinline__ void run(c2 (&v)[2]) {
		const c2 a = v[0], b = v[1];
		v[0] = a + b;
		v[1] = a - b;
	}
};
template <bool INV>
struct PairDFT<3, INV> {
	static __device__ __forceinline__ void run(c2 (&v)[3]) {
		constexpr float s60 = 0.86602540378443864676f;
		const c2 t1 = v[1] + v[2], d = v[1] - v[2];
		const c2 m1 = c2{fmas(t1.re, -0.5f, v[0].re), fmas(t1.im, -0.5f, v[0].im)};
		v[0] = v[0] + t1;
		// m1 +- w*(s60*d), w = -i (forward) / +i (inverse)
		constexpr float sg = INV ? -s60 : s60;
		v[1] = c2{fmas(d.im, sg, m1.re), fmas(d.re, -sg, m1.im)};
		v[2] = c2{fmas(d.im, -sg, m1.re), fmas(d.re, sg, m1.im)};
	}
};
template <bool INV>
struct PairDFT<4, INV> {
	static __device__ __forceinline__ void run(c2 (&v)[4]) {
		const c2 a = v[0] + v[2], b = v[0] - v[2], c = v[1] + v[3], d = v[1] - v[3];
		v[0] = a + c;
		v[2] = a - c;
		v[1] = add_mi<INV>(b, d);
		v[3] = sub_mi<INV>(b, d);
	}
};
template <bool INV>
struct PairDFT<5, INV> {
	static __device__ __forceinline__ void run(c2 (&v)[5]) {
		constexpr float c1 = 0.30901699437494742410f, c2c = -0.80901699437494742410f;
		constexpr float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
		const c2 a1 = v[1] + v[4], a2 = v[2] + v[3], b1 = v[1] - v[4], b2 = v[2] - v[3];
		const c2 r1 = c2{fmas(a2.re, c2c, fmas(a1.re, c1, v[0].re)), fmas(a2.im, c2c, fmas(a1.im, c1, v[0].im))};
		const c2 r2 = c2{fmas(a2.re, c1, fmas(a1.re, c2c, v[0].re)), fmas(a2.im, c1, fmas(a1.im, c2c, v[0].im))};
		// q1 = s1*b1 + s2*b2, q2 = s2*b1 - s1*b2; outputs r1 +- w*q1, r2 +- w*q2
		const c2 q1 = c2{fmas(b2.re, s2, muls(b1.re, s1)), fmas(b2.im, s2, muls(b1.im, s1))};
		const c2 q2 = c2{fmas(b2.re, -s1, muls(b1.re, s2)), fmas(b2.im, -s1, muls(b1.im, s2))};
		v[0] = v[0] + a1 + a2;
		v[1] = add_mi<INV>(r1, q1);
		v[4] = sub_mi<INV>(r1, q1);
		v[2] = add_mi<INV>(r2, q2);
		v[3] = sub_mi<INV>(r2, q2);
	}
};
// Cooley-Tukey R = R1*R2 in registers: input index n = R2*n1 + n2, output k = k1 + R1*k2
template <int R1, int R2, bool INV>
struct PairComposite {
	static __device__ __forceinline__ void run(c2 (&v)[R1 * R2]) {
		constexpr int R = R1 * R2;
		c2 t[R2][R1];
		static_for<R2>([&](auto n2c) {
			constexpr int n2 = decltype(n2c)::value;
			c2 a[R1];
			static_for<R1>([&](auto n1c) { a[decltype(n1c)::value] = v[R2 * decltype(n1c)::value + n2]; });
			PairDFT<R1, INV>::run(a);
			static_for<R1>([&](auto k1c) {
				constexpr int k1 = decltype(k1c)::value;
				t[n2][k1] = twmul2<R, n2 * k1, INV>(a[k1]);
			});
		});
		static_for<R1>([&](auto k1c) {
			constexpr int k1 = decltype(k1c)::value;
			c2 b[R2];
			static_for<R2>([&](auto n2c) { b[decltype(n2c)::value] = t[decltype(n2c)::value][k1]; });
			PairDFT<R2, INV>::run(b);
			static_for<R2>([&](auto k2c) { v[k1 + R1 * decltype(k2c)::value] = b[decltype(k2c)::value]; });
		});
	}
};
template <bool INV> struct PairDFT<10, INV> : PairComposite<2, 5, INV> {};
template <bool INV> struct PairDFT<12, INV> : PairComposite<4, 3, INV> {};
template <bool INV> struct PairDFT<16, INV> : PairComposite<4, 4, INV> {};

// ---- geometry of the paired in-place FFT ----
// K = 16 * 16 * R3 points in one buffer of LEN float4 slots; a slot address is d1*P1 + d2*P2 + d3 for digits
// (d1, d2 in [0,16), d3 in [0,R3)).  P2 = R3 (dense), P1 = 16*R3 + 1 (odd): in every pass the lanes of a warp
// either walk d1 (odd stride) or consecutive slots, so the 128-bit accesses are bank-conflict free.
template <int KT>
struct PairGeo {
	static constexpr int K = KT;
	static constexpr int R3 = KT / 256; // 12 or 10
	static constexpr int M1 = 16 * R3;  // items of the radix-16 passes
	static constexpr int P2 = R3;
	static constexpr int P1 = M1 + 1;
	static constexpr int LEN = 16 * P1; // float4 slots
	static_assert(KT == 3072 || KT == 2560, "paired FFT is specialised for the preset sizes");
	// "slow-digit-first" index  i = d1*M1 + d2*R3 + d3  ->  slot (natural order up to the padding)
	static __device__ __forceinline__ int slot_nat(int i) { return i + i / M1; }
	// "fast-digit-first" index  i = d1 + 16*d2 + 256*d3  ->  slot (digit-reversed placement)
	static __device__ __forceinline__ int slot_rev(int i) { return (i & 15) * P1 + ((i >> 4) & 15) * P2 + (i >> 8); }
};

__device__ __forceinline__ c2 ld_c2(const float4 *p) {
	const float4 v = *p;
	return c2{f2_make(v.x, v.y), f2_make(v.z, v.w)};
}
__device__ __forceinline__ void st_c2(float4 *p, c2 v) {
	*p = make_float4(f2_lo(v.re), f2_hi(v.re), f2_lo(v.im), f2_hi(v.im));
}

// per-thread twiddle bases, loaded once per CTA: w^(2^i), i = 0..3, of the thread's two radix-16 passes
// (w = W_K^ia for the first, W_K^ib for the second); the other powers are products of at most three of them
struct PairTw {
	float2 a[4], b[4];
};
template <int KT>
__device__ __forceinline__ PairTw pair_tw_load(const float2 *__restrict__ tw, int ia, int ib) {
	PairTw t;
#pragma unroll
	for (int i = 0; i < 4; ++i) {
		t.a[i] = __ldg(tw + ((ia << i) % KT));
		t.b[i] = __ldg(tw + ((ib << i) % KT));
	}
	return t;
}
// v[q] *= w^q for q = 1..15, w^(2^i) = base[i] (conjugated for the inverse transform)
template <bool INV>
__device__ __forceinline__ void apply_tw16(c2 (&v)[16], const float2 (&base)[4]) {
	float2 wp[4];
#pragma unroll
	for (int i = 0; i < 4; ++i) wp[i] = make_float2(base[i].x, INV ? -base[i].y : base[i].y);
	static_for<16>([&](auto qc) {
		constexpr int q = decltype(qc)::value;
		if constexpr (q > 0) {
			constexpr int lowBit = (q & 1) ? 0 : (q & 2) ? 1 : (q & 4) ? 2 : 3;
			float2 w = wp[lowBit];
			constexpr int rest = q & ~(1 << lowBit);
			if constexpr (rest & 2) w = cmulf(w, wp[1]);
			if constexpr (rest & 4) w = cmulf(w, wp[2]);
			if constexpr (rest & 8) w = cmulf(w, wp[3]);
			v[q] = cmulw(v[q], w.x, w.y);
		}
	});
}

// =====================  FORWARD transform, decimation in TIME (analysis)  =====================
// Input x[n], n = n1 + 16*n2 + 256*n3, is placed at slot_rev(n); the result X[k], k = j3 + R3*j2 + M1*k1,
// ends at slot_nat(k) -- and the last pass hands it to the caller in registers instead of storing it.
//   stage A (caller): radix R3 over n3 for the thread's (n1, n2) = (tid & 15, tid >> 4): 12 contiguous slots,
//                     no twiddle; fused with the windowing / pre-twiddle of the input (k_analyse2)
//   stage B: item (n1, j3) = (tid & 15, tid >> 4), inputs n2 = 0..15 (stride P2) times W_M1^(n2*j3), radix 16 -> j2
//   stage C: item m = j3 + R3*j2 = tid, inputs n1 = 0..15 (stride P1) times W_K^(n1*m), radix 16 -> k1;
//            output q of the item is X[m + M1*q]
template <int KT>
__device__ __forceinline__ PairTw pair_tw_dit(const float2 *__restrict__ tw, int tid) {
	using G = PairGeo<KT>;
	const int t = tid < G::M1 ? tid : 0;
	return pair_tw_load<KT>(tw, 16 * (t >> 4), t); // stage B: W_M1^j3 = W_K^(16*j3); stage C: W_K^m
}
template <int KT>
__device__ __forceinline__ void pair_dit_stage_b(float4 *buf, const PairTw &tw, int tid) {
	using G = PairGeo<KT>;
	if (tid < G::M1) {
		float4 *p = buf + (tid & 15) * G::P1 + (tid >> 4);
		c2 v[16];
		static_for<16>([&](auto qc) { v[decltype(qc)::value] = ld_c2(p + decltype(qc)::value * G::P2); });
		apply_tw16<false>(v, tw.a);
		PairDFT<16, false>::run(v);
		static_for<16>([&](auto qc) { st_c2(p + decltype(qc)::value * G::P2, v[decltype(qc)::value]); });
	}
}
// stage C for thread tid < M1: v[q] = X[tid + M1*q] on return (nothing is stored)
template <int KT>
__device__ __forceinline__ void pair_dit_stage_c(const float4 *buf, const PairTw &tw, int tid, c2 (&v)[16]) {
	using G = PairGeo<KT>;
	const float4 *p = buf + tid; // slot of (n1 = 0, j2, j3) is j2*P2 + j3 = m
	static_for<16>([&](auto qc) { v[decltype(qc)::value] = ld_c2(p + decltype(qc)::value * G::P1); });
	apply_tw16<false>(v, tw.b);
	PairDFT<16, false>::run(v);
}

// =====================  INVERSE transform, decimation in FREQUENCY (synthesis)  =====================
// Input Z[k], k = k1*M1 + k', enters pass 1 from registers (the caller loads it from the staged spectra);
// the result z[n], n = n1 + 16*n2 + 256*n3, ends at slot_rev(n).
//   pass 1: item k' = tid (< M1), radix 16 over k1, times conj W_K^(k'*q), stored at slots q*P1 + k'
//   pass 2: item (q1, r) = (tid & 15, tid >> 4) (< M1): radix 16 over the R3-strided digit, times conj W_M1^(r*q)
//   pass 3: item (q1, q2) = (tid & 15, tid >> 4): radix R3 over the contiguous digit, no twiddle
template <int KT>
__device__ __forceinline__ PairTw pair_tw_dif(const float2 *__restrict__ tw, int tid) {
	using G = PairGeo<KT>;
	const int t = tid < G::M1 ? tid : 0;
	return pair_tw_load<KT>(tw, t, 16 * (t >> 4));
}
// pass 1 for thread tid < M1: v[q] = Z[q*M1 + tid] on entry
template <int KT>
__device__ __forceinline__ void pair_dif_pass1(float4 *buf, const PairTw &tw, int tid, c2 (&v)[16]) {
	using G = PairGeo<KT>;
	PairDFT<16, true>::run(v);
	apply_tw16<true>(v, tw.a);
	float4 *p = buf + tid;
	static_for<16>([&](auto qc) { st_c2(p + decltype(qc)::value * G::P1, v[decltype(qc)::value]); });
}
// pass 2 (in place; the buffer must be complete on entry) and pass 3, which leaves its outputs in registers:
// for thread (q1, q2) = (tid & 15, tid >> 4), v[q3] = z[q1 + 16*q2 + 256*q3] on return.  Contains the barrier
// between the two passes; the caller decides where the results go.
template <int KT>
__device__ __forceinline__ void pair_dif_pass23(float4 *buf, const PairTw &tw, int tid, c2 (&out)[PairGeo<KT>::R3]) {
	using G = PairGeo<KT>;
	if (tid < G::M1) {
		float4 *p = buf + (tid & 15) * G::P1 + (tid >> 4);
		c2 v[16];
		static_for<16>([&](auto qc) { v[decltype(qc)::value] = ld_c2(p + decltype(qc)::value * G::P2); });
		PairDFT<16, true>::run(v);
		apply_tw16<true>(v, tw.b);
		static_for<16>([&](auto qc) { st_c2(p + decltype(qc)::value * G::P2, v[decltype(qc)::value]); });
	}
	__syncthreads();
	{
		const float4 *p = buf + (tid & 15) * G::P1 + (tid >> 4) * G::P2;
		static_for<G::R3>([&](auto qc) { out[decltype(qc)::value] = ld_c2(p + decltype(qc)::value); });
		PairDFT<G::R3, true>::run(out);
	}
}

} // namespace b200s
