// stft2.cuh -- analysis and synthesis kernels for the preset FFT sizes on the PAIRED in-place FFT
// (fft2.cuh).  Same results as k_analyse / k_synth (kernels.cuh), which stay for generic sizes.
//
//   k_analyse2  windowed modified real FFT of TWO analyses at a time (dependency analyseStep,
//               reference call sites signalsmith-stretch.h:337,359).  Persistent CTAs walk the
//               (stream, job pair) items of the call; the raw samples of the NEXT pair are bulk-copied to
//               shared memory while the current FFT runs, and the spectrum rows leave the FFT buffer by
//               bulk copies.
//   k_synth2    inverse FFT of TWO consecutive blocks of one stream-channel at a time, synthesis
//               window and overlap-add (synthesiseStep / readOutput / moveOutput, :397-414).  The two
//               spectra of the NEXT pair are bulk-copied into the FFT buffer while the ring is updated;
//               the time samples go from registers into the pending ring, per ring slot in the
//               reference's order: block A's contribution, the emission of the samples between the two
//               blocks, block B's contribution.
#pragma once
#include "fft2.cuh"
#include "kernels.cuh"

namespace b200s {


__host__ __device__ __forceinline__ int stage_len(int B) { return (B + 8 + 3) & ~3; }

// streaming accesses (read once / written once): keep them out of L1, which -- next to two 95 KB CTAs -- is only
// large enough for the window / twiddle tables that every item re-reads
#ifdef B200S_EMU
__device__ __forceinline__ void st_stream(float *p, float v) { *p = v; }
__device__ __forceinline__ void st_stream4(float *p, float4 v) { *(float4 *)p = v; }
#else
__device__ __forceinline__ void st_stream4(float *p, float4 v) { __stcs((float4 *)p, v); }
__device__ __forceinline__ void st_stream(float *p, float v) { __stcs(p, v); }
#endif

// ---------------------------------------------------------------------------------------------
// k_analyse2: grid = persistent CTAs (a multiple of the SM count), 256 threads.
// dyn smem: PairGeo::LEN float4 (FFT pair; after the last pass it holds the pair's spectrum rows, stored by a bulk copy)
// + 2 * stage_len(B) floats (raw samples of the next pair).
// PROBE (profiling builds, -DB200S_ANALYSE_PROBES; wrong results on purpose) removes one part of the item to measure what
// the kernel's time goes with: 1 the spectrum store, 2 the window / pre-twiddle table loads (a constant instead),
// 3 the wait for the staged input (moved to just before the next copies are issued), 4 the FFT's stages B and C.
// ---------------------------------------------------------------------------------------------
// MIXED (k_analyse2_mixed): a stereo call whose streams take both paths -- the store form is chosen per item, planar
// rows for the streams on the mapped path (spec_il) -- and every call over a list of streams (Ctx::listed: the item's
// stream is looked up in the list; k_analyse2 keeps the whole batch's item fetch, which is on its critical path).  Otherwise (k_analyse2) the form is the call's, x.specIl, and the
// per-item test is not in the code at all.
template <int KT, int PROBE, bool MIXED>
__device__ __forceinline__ void analyse2_body(const Ctx &x) {
	using G = PairGeo<KT>;
	static_assert(2 * KT * sizeof(float2) <= G::LEN * sizeof(float4), "the spectrum rows of a pair fit the FFT buffer");
	const Cfg &g = x.cfg;
	B200S_DYN_SHARED
	float4 *buf = (float4 *)dyn_smem;
	const int B = g.B, o = g.o, tid = threadIdx.x;
	float *stA = (float *)(buf + G::LEN), *stB = stA + stage_len(B);
	const PairTw tw = pair_tw_dit<KT>(x.twiddle, tid);
	const int PJ = g.C * x.maxFrames;         // pair slots per stream (2*C*maxFrames jobs)
	const long long total = (long long)x.sCount * PJ;

	struct Item {
		int s, hasB, nIn; // nIn, in, inChan: the stream's Call (loaded with the descriptors, off the staging path)
		const float *in;
		int inChan;
		Job a, b;
	};
	// item -> jobs; false when the stream has fewer pairs than slots
	// (the four loads are independent of each other: the job slots exist even when the stream has fewer jobs)
	// fetch_raw only issues the loads (m.hasB temporarily holds the stream's job count); fetch_done turns them into
	// an item.  Keeping the two apart lets the loads of the item after next fly for a whole iteration.
	auto fetch_raw = [&](long long it, Item &m) {
		const Job *jb;
		if constexpr (MIXED) { // (one 64-bit division, not two: with the list look-up the kernel fits 128 registers)
			const int q = (int)(it / PJ);
			m.s = stream_at(x, x.sBase + q);
			jb = x.jobs + (size_t)m.s * 2 * g.C * x.maxFrames + 2 * (int)(it - (long long)q * PJ);
		} else {
			m.s = x.sBase + (int)(it / PJ);
			jb = x.jobs + (size_t)m.s * 2 * g.C * x.maxFrames + 2 * (int)(it % PJ);
		}
		m.hasB = x.call[m.s].nJobs;
		m.nIn = x.call[m.s].nIn;
		m.in = x.call[m.s].in;
		m.inChan = x.call[m.s].inChan;
		m.a = jb[0];
		m.b = jb[1];
	};
	auto fetch_done = [&](long long it, Item &m) -> bool {
		const int p = (int)(it % PJ), nJ = m.hasB;
		m.hasB = 2 * p + 1 < nJ;
		if (!m.hasB) m.b = m.a;
		return 2 * p < nJ;
	};
	auto fetch = [&](long long it, Item &m) -> bool {
		fetch_raw(it, m);
		return fetch_done(it, m);
	};
	auto next_valid = [&](long long it, Item &m) -> long long {
		while (it < total && !fetch(it, m)) it += gridDim.x;
		return it;
	};
	// asynchronously copy the B samples (history ++ input) of one job into a staging buffer.
	// Aligned mode copies the enclosing 4-aligned range (sample i lands at st[i + (start & 3)]) with at most two BULK
	// copies issued by one thread -- the part that lies in the history and the part that lies in this call's input --
	// which complete on the CTA's mbarrier (two arrivals per item: one per job); whatever lies outside both (before the
	// history, after the input) is zero-filled by all threads.  (This replaces a per-16-byte cp.async loop and its
	// instructions.)
	B200S_SHARED unsigned long long stageBar;
	if (tid == 0) mbar_init(&stageBar, 2);
	fence_async_proxy();
	__syncthreads();
	unsigned stagePar = 0u;
	auto stage_job = [&](float *st, const Item &m, const Job &j, int t0, int nT) {
		const int s = m.s, nIn = m.nIn;
		const float *ib = m.in + (size_t)j.c * m.inChan;
		const float *he = x.histCur + ((size_t)s * g.C + j.c) * g.histLen + g.histLen;
		if (x.inAligned) {
			const int sh = j.start & 3, a00 = j.start - sh, nCh = (B + sh + 3) >> 2;
			// chunk q holds samples a00 + 4q ..: [qh0, z) comes from the history, [z, qi1) from the input
			const int z = min(max((-a00) >> 2, 0), nCh);
			const int qh0 = min(max((-g.histLen - a00) >> 2, 0), z), qi1 = min(max((nIn - a00) >> 2, z), nCh);
			if (tid == t0) {
				fence_async_proxy(); // the staging buffer was last read through the generic proxy
				mbar_expect(&stageBar, 16u * (unsigned)(qi1 - qh0));
				if (z > qh0) bulk_g2s(st + 4 * qh0, he + a00 + 4 * qh0, 16u * (unsigned)(z - qh0), &stageBar);
				if (qi1 > z) bulk_g2s(st + 4 * z, ib + a00 + 4 * z, 16u * (unsigned)(qi1 - z), &stageBar);
			}
			for (int q = tid; q < qh0; q += 256) *(float4 *)(st + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
			for (int q = qi1 + tid; q < nCh; q += 256) *(float4 *)(st + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
		} else {
			for (int i = tid; i < B; i += nT) {
				const int a = j.start + i;
				if (a < nIn && a >= -g.histLen) cp_async4(st + i, a >= 0 ? ib + a : he + a);
				else st[i] = 0.f;
			}
		}
	};
	// Items are looked up TWO iterations ahead: the descriptor loads of the item after next are issued while the
	// current pair is transformed and are only consumed at the end of the iteration, so that the copies of the next
	// item's input can start the moment the staging buffers are free.  (Letting the two warps that idle during the
	// radix-16 passes do the look-up and the copies instead makes the other six wait for them at the next barrier.)
	Item cur, nxt;
	long long item = next_valid(blockIdx.x, cur);
	if (item < total) {
		stage_job(stA, cur, cur.a, 0, 256);
		stage_job(stB, cur, cur.b, 32, 256);
	}
	long long nitem = item < total ? next_valid(item + gridDim.x, nxt) : total;
	while (item < total) {
		float2 *dstA = x.spec + ((size_t)cur.s * 2 * x.maxFrames * g.C + cur.a.row) * g.K;
		float2 *dstB = x.spec + ((size_t)cur.s * 2 * x.maxFrames * g.C + cur.b.row) * g.K;
		// window samples and pre-twiddles of this thread's R3 elements: issued before the wait so that their latency overlaps it.
		// (The values are the same for every pair; `wofs` is opaque to the compiler so that they are re-loaded,
		// L1/L2 hits, instead of being hoisted into 2*R3 permanently live registers.)
		float4 tabr[G::R3]; // {window[n+o], window[n+o-K], pre-twiddle exp(-i*pi*n/N)} of element n = tid + 256*it
		{
			int wofs = 0;
#ifndef B200S_EMU
			asm volatile("" : "+r"(wofs));
#endif
			static_for<G::R3>([&](auto itc) {
				constexpr int it = decltype(itc)::value;
				if constexpr (PROBE == 2) tabr[it] = make_float4(1.f, 1.f, 1.f, 0.f);
				else tabr[it] = __ldg(x.anaTab + tid + 256 * it + wofs);
			});
		}
		cp_async_wait_all();
		if (x.inAligned && PROBE != 3) {
			mbar_wait(&stageBar, stagePar);
			stagePar ^= 1u;
		}
		if (tid == 0) bulk_wait_read(); // the previous pair's spectrum has left buf
		__syncthreads(); // staging complete and visible; buf free
#ifdef B200S_EMU_EXACT_FFT // test builds only: swap in the oracle's double FFT to isolate the non-FFT logic
		{
			const int shA = x.inAligned ? (cur.a.start & 3) : 0, shB = x.inAligned ? (cur.b.start & 3) : 0;
			if (tid == 0) {
				float *xw = (float *)buf;
				const bool il = MIXED ? spec_il(x, x.call[cur.s]) : x.specIl != 0;
				// interleaved mode: transform into scratch rows (the Y rows of block 0: the chain writes them only later), then interleave
				float2 *tA = il ? x.Y + coef_off(x, cur.s, 0, 0) : dstA, *tB = il ? tA + KT : dstB;
				for (int i = 0; i < B; ++i) xw[i] = fmul(stA[i + shA], x.window[i]);
				emu_exact_forward(xw, B, o, 2 * KT, tA);
				if (cur.hasB) {
					for (int i = 0; i < B; ++i) xw[i] = fmul(stB[i + shB], x.window[i]);
					emu_exact_forward(xw, B, o, 2 * KT, tB);
				}
				if (il) {
					float4 *d4 = (float4 *)x.spec + ((size_t)cur.s * 2 * x.maxFrames + (cur.a.row >> 1)) * g.K;
					for (int b = 0; b < KT; ++b) d4[b] = make_float4(tA[b].x, tB[b].x, tA[b].y, tB[b].y);
				}
			}
			__syncthreads();
			item = nitem;
			cur = nxt;
			if (item < total) {
				stage_job(stA, cur, cur.a, 0, 256);
				stage_job(stB, cur, cur.b, 32, 256);
				nitem = next_valid(item + gridDim.x, nxt);
			}
			continue;
		}
#endif
		{ // ---- load stage fused with the first FFT pass: window, wrap-sign fold (SURVEY.md App. F), half-bin
		  //      pre-twiddle of the thread's R3 samples n = tid + 256*n3, radix-R3 butterfly over n3 in registers
			const int shA = x.inAligned ? (cur.a.start & 3) : 0, shB = x.inAligned ? (cur.b.start & 3) : 0;
			c2 v[G::R3];
			static_for<G::R3>([&](auto itc) {
				constexpr int it = decltype(itc)::value;
				const int n = tid + 256 * it, i0 = n + o, i1 = n + o - KT;
				const bool in0 = i0 < B, in1 = i1 >= 0;
				const float w0 = tabr[it].x, w1 = tabr[it].y;
				const float a0 = in0 ? stA[i0 + shA] : 0.f, a1 = in1 ? stA[i1 + shA] : 0.f;
				const float b0 = in0 ? stB[i0 + shB] : 0.f, b1 = in1 ? stB[i1 + shB] : 0.f;
				const float2 pw = make_float2(tabr[it].z, tabr[it].w); // exp(-i*pi*n/N), exactly rounded table entry
				const c2 t = c2{muls(f2_make(a0, b0), w0), muls(f2_make(a1, b1), w1)}; // (x0*w0) + i*(x1*w1)
				v[it] = cmulw(t, pw.x, pw.y);
			});
			PairDFT<G::R3, false>::run(v);
			float4 *p = buf + (tid & 15) * G::P1 + (tid >> 4) * G::P2;
			static_for<G::R3>([&](auto qc) { st_c2(p + decltype(qc)::value, v[decltype(qc)::value]); });
		}
		__syncthreads(); // staging consumed, buf complete
		Item n2;
		long long cand = nitem + gridDim.x;
		bool ok2 = false;
		if constexpr (PROBE == 3) {
			if (x.inAligned) {
				mbar_wait(&stageBar, stagePar);
				stagePar ^= 1u;
			}
		}
		if (nitem < total) { // start the next pair's input on its way while this FFT runs
			stage_job(stA, nxt, nxt.a, 0, 256);
			stage_job(stB, nxt, nxt.b, 32, 256);
			if (cand < total) fetch_raw(cand, n2); // descriptor of the item after next: loads in flight until the end of the iteration
		}
		if constexpr (PROBE != 4) pair_dit_stage_b<KT>(buf, tw, tid);
		__syncthreads();
		// ---- last pass: thread tid < M1 holds X[tid + M1*q], q = 0..15, in registers.
		//      bin b = Z[b/2] (b even) or conj(Z[K-1-b/2]) (b odd): Z[k] with k < K/2 (q < 8) is bin 2k, the rest bin 2(K-1-k)+1.
		//      The bins go back into buf in bin order and leave it as whole rows by bulk copies: stored from registers, each
		//      warp instruction would write every other 16-byte half of its sectors (the other halves come from the mirror
		//      warp), and two warps would sit idle through 96 store instructions per pair.
		c2 v[16];
		if (tid < G::M1) {
			if constexpr (PROBE == 4) {
				static_for<16>([&](auto qc) { v[decltype(qc)::value] = c2{f2_make((float)tid, 0.f), f2_make(0.f, (float)decltype(qc)::value)}; });
			} else {
				pair_dit_stage_c<KT>(buf, tw, tid, v);
			}
		} else {
			// defined on the idle threads too: ptxas would otherwise keep all 64 registers live around the whole loop
			static_for<16>([&](auto qc) { v[decltype(qc)::value] = c2{f2_make(0.f, 0.f), f2_make(0.f, 0.f)}; });
		}
		// (MIXED: per item, the streams on the mapped path keep planar rows; the job pairing is the same in both forms)
		const bool hasB = cur.hasB, il = MIXED ? spec_il(x, x.call[cur.s]) : x.specIl != 0;
		if constexpr (PROBE == 1) {
#ifndef B200S_EMU
			if (tid < G::M1) static_for<16>([&](auto qc) {
				const c2 w = v[decltype(qc)::value];
				asm volatile("" ::"f"(w.re.a), "f"(w.re.b), "f"(w.im.a), "f"(w.im.b));
			});
#endif
		} else {
			__syncthreads(); // every read of buf has ended
			if (tid < G::M1) {
				// stereo direct path: the pair is (channel 0, channel 1) of one analysis, one row of float4 {re0, re1, im0, im1};
				// otherwise row A at buf's first K float2, row B behind it
				float2 *rowA = (float2 *)buf, *rowB = rowA + KT;
				static_for<16>([&](auto qc) {
					constexpr int q = decltype(qc)::value;
					const int k = tid + G::M1 * q;
					const int b = q < 8 ? 2 * k : 2 * (KT - 1 - k) + 1;
					const float sg = q < 8 ? 1.f : -1.f;
					const float ra = f2_lo(v[q].re), rb = f2_hi(v[q].re), ia = sg * f2_lo(v[q].im), ib = sg * f2_hi(v[q].im);
					if (il) {
						buf[b] = make_float4(ra, rb, ia, ib);
					} else {
						rowA[b] = make_float2(ra, ia);
						rowB[b] = make_float2(rb, ib);
					}
				});
			}
			fence_async_proxy(); // the rows were written through the generic proxy; the bulk copies read them through the async one
			__syncthreads();
			if (tid == 0) {
				constexpr unsigned row = (unsigned)sizeof(float2) * KT;
				if (il) {
					bulk_s2g((float4 *)x.spec + ((size_t)cur.s * 2 * x.maxFrames + (cur.a.row >> 1)) * g.K, buf, 2 * row);
				} else {
					bulk_s2g(dstA, buf, row);
					if (hasB) bulk_s2g(dstB, (float2 *)buf + KT, row);
				}
				bulk_commit(); // waited for (source read) before the next pair's first pass writes buf
			}
		}
		item = nitem;
		cur = nxt;
		if (nitem < total) {
			if (cand < total) ok2 = fetch_done(cand, n2);
			if (cand < total && !ok2) cand = next_valid(cand + gridDim.x, n2); // rare: a stream with fewer pairs than slots
			nitem = cand < total ? cand : total;
			nxt = n2;
		}
	}
	if (tid == 0) bulk_wait_read(); // the shared memory of the last pair's rows stays allocated until they are read
}
template <int KT, int PROBE = 0>
__global__ void __launch_bounds__(256, 2) k_analyse2(Ctx x) { analyse2_body<KT, PROBE, false>(x); }
template <int KT>
__global__ void __launch_bounds__(256, 2) k_analyse2_mixed(Ctx x) { analyse2_body<KT, 0, true>(x); }

// ---------------------------------------------------------------------------------------------
// k_synth2: grid (C, S), 256 threads, one CTA per stream-channel; blocks of the call two at a time.
// dyn smem: PairGeo::LEN float4 (FFT pair; between two FFTs it holds the next pair's two spectra, staged by a bulk
// copy) + pendLen floats (pending ring).  The windowProducts divisor is not carried in a ring: it depends on the block
// schedule only, and each emitted sample computes its own (wp_at).
// PROBE (profiling builds, -DB200S_SYNTH_PROBES; wrong results on purpose) removes one part of the kernel to measure what
// its time goes with: 1 the windowProducts divisor (the samples are emitted undivided), 2 every ring update of the overlap-add,
// 3 the wait for the staged spectra (moved to just before the next copies are issued), 4 the inverse FFT's passes 2-3.
// ---------------------------------------------------------------------------------------------
template <int KT, int PROBE>
__device__ __forceinline__ void synth2_body(const Ctx &x) {
	using G = PairGeo<KT>;
	static_assert(2 * KT * sizeof(float2) <= G::LEN * sizeof(float4), "the two spectra of a pair fit the FFT buffer");
	const Cfg &g = x.cfg;
	B200S_DYN_SHARED
	float4 *buf = (float4 *)dyn_smem;
	float *pend = (float *)(buf + G::LEN);
	const int c = blockIdx.x, pos = x.sBase + blockIdx.y, s = stream_at(x, pos), tid = threadIdx.x;
	const Call cl = x.call[s];
	float *out = x.out + (size_t)pos * x.outStreamStride + (size_t)c * x.outChanStride; // (the caller's row: by position)
	if (cl.bypass) { // :252-267
		const float *in = cl.in + (size_t)c * cl.inChan;
		for (int i = tid; i < cl.nOut; i += 256) out[i] = cl.nIn > 0 ? in[i % cl.nIn] : 0.f;
		for (int i = cl.nOut + tid; i < x.outTail; i += 256) out[i] = 0.f;
		return;
	}
	const int P = g.pendLen, B = g.B, o = g.o, addOff = g.addOff;
	float *gp = x.pend + ((size_t)s * g.C + c) * P, *gw = x.pendWp + ((size_t)s * g.C + c) * P;
	const Frame *frames = x.frames + (size_t)s * x.maxFrames;
	// the spectra of a pair of blocks are staged in the FFT buffer: block f's row at stY, block f+1's at stY + K.
	// One thread issues the bulk copies of the NEXT pair as soon as the current FFT has its outputs in registers; they
	// complete on stageBar while the ring is updated and emitted.
	float2 *const stY = (float2 *)buf;
	B200S_SHARED unsigned long long stageBar;
	if (tid == 0) mbar_init(&stageBar, 1);
	fence_async_proxy();
	__syncthreads();
	unsigned stagePar = 0u;
	auto stage_pair = [&](int f) { // callers: every generic-proxy access to buf has ended (a barrier lies between)
		if (tid == 0) {
			const unsigned row = (unsigned)sizeof(float2) * KT;
			const bool two = f + 1 < cl.nFrames;
			fence_async_proxy();
			mbar_expect(&stageBar, two ? 2 * row : row);
			bulk_g2s(stY, x.Y + coef_off(x, s, f, c), row, &stageBar);
			if (two) bulk_g2s(stY + KT, x.Y + coef_off(x, s, f + 1, c), row, &stageBar);
		}
	};
	if (cl.nFrames > 0) stage_pair(0);
	for (int i = tid; i < P; i += 256) pend[i] = gp[i];
	__syncthreads();
	int head = 0, emitted = 0;
	// windowProducts (:397-399, :408-414) of output sample T of the call (T = emitted + ring offset): the carried value
	// gw[T] (T < P; slots beyond were cleared to ALMOST_ZERO when emitted), plus winProd[u - f*H] of every block f of the call
	// that covers it, in block order, u = T - addOff - t0.  k_plan triggers the blocks of a call exactly H apart from t0
	// (samplesSinceLast restarts at 0 on a trigger, :281-286), so wherever T >= P and the covering blocks are the full
	// H-spaced run (B - H <= u < nFrames*H), the sum is the table entry wpDiv[u mod H], accumulated in the same order.
	// The other samples -- the first ones of a call and the ring's tail at its end -- add the terms one by one.
	const int uOff = addOff + (cl.nFrames > 0 ? frames[0].t : 0);
	auto wp_at = [&](int T) -> float {
		const int u = T - uOff, H = g.H, nF = __ldg(&x.call[s].nFrames);
		if (T >= P && u >= B - H && u < nF * H) return __ldg(x.wpDiv + u % H);
		float w = T < P ? gw[T] : B200S_ALMOST_ZERO;
		if (u >= 0)
			for (int f = (u >= B ? (u - B) / H + 1 : 0), fHi = min(u / H, nF - 1); f <= fHi; ++f) w = fadd(w, __ldg(x.winProd + u - f * H));
		return w;
	};
	// samples T .. T+3: one index computation for the four table entries when all four are in the full run
	auto wp_at4 = [&](int T) -> float4 {
		const int u = T - uOff, H = g.H, nF = __ldg(&x.call[s].nFrames);
		if (T >= P && u >= B - H && u + 3 < nF * H) {
			int j = u % H;
			float4 w;
			w.x = __ldg(x.wpDiv + j);
			if (++j == H) j = 0;
			w.y = __ldg(x.wpDiv + j);
			if (++j == H) j = 0;
			w.z = __ldg(x.wpDiv + j);
			if (++j == H) j = 0;
			w.w = __ldg(x.wpDiv + j);
			return w;
		}
		return make_float4(wp_at(T), wp_at(T + 1), wp_at(T + 2), wp_at(T + 3));
	};
	// emit n samples from the ring head, zero them behind (:408-414)
	// VECTOR form of the ring loops: when the ring head, the counts and the output row are multiples of four floats
	// (the presets at 48 kHz with chunks that are multiples of four), four consecutive ring slots are one 16-byte
	// shared-memory access each and never straddle the wrap; element for element the same operations in the same order.
	const bool ioVec = ((uintptr_t)out & 15) == 0 && ((P | B | addOff) & 3) == 0;
	auto emit = [&](int n) {
		if (ioVec && ((head | n | emitted) & 3) == 0 && n <= P) {
			for (int i = 4 * tid; i < n; i += 1024) {
				int p = head + i;
				if (p >= P) p -= P;
				const float4 a = *(float4 *)(pend + p);
				if constexpr (PROBE == 1) {
					st_stream4(out + emitted + i, a);
				} else {
					const float4 w = wp_at4(emitted + i);
					st_stream4(out + emitted + i, make_float4(fdiv(a.x, w.x), fdiv(a.y, w.y), fdiv(a.z, w.z), fdiv(a.w, w.w)));
				}
				*(float4 *)(pend + p) = make_float4(0.f, 0.f, 0.f, 0.f);
			}
			head = (head + n) % P;
			emitted += n;
			return;
		}
		for (int i = tid; i < n; i += 256) {
			float v = 0.f;
			if (i < P) {
				int p = head + i;
				if (p >= P) p -= P;
				v = PROBE == 1 ? pend[p] : fdiv(pend[p], wp_at(emitted + i));
				pend[p] = 0.f;
			}
			st_stream(out + emitted + i, v);
		}
		head = (head + (n < P ? n : P)) % P; // n >= P leaves an all-clear ring; any head is fine
		emitted += n;
	};
	// time samples of this thread's R3 elements n2 = tid + 256*q3, {block A, block B} each, synthesis window applied:
	// yRe[q3] is sample n2 + o (if < B), yIm[q3] is sample n2 + o - K (if >= 0).  Every sample of the block has exactly
	// one owner, so the overlap-add goes from registers straight into the ring, one writing thread per slot.
	// block A (hi = false) or B (hi = true) into the ring (:397-399): sample i lands in slot head + addOff + i
	auto add_block = [&](const f2 (&yRe)[G::R3], const f2 (&yIm)[G::R3], bool hi) {
		auto add = [&](int i, f2 y) {
			int p = head + addOff + i;
			if (p >= P) p -= P;
			if constexpr (PROBE == 2) {
#ifndef B200S_EMU
				asm volatile("" ::"f"(hi ? f2_hi(y) : f2_lo(y)), "r"(p));
#endif
				return;
			}
			pend[p] = fadd(pend[p], hi ? f2_hi(y) : f2_lo(y));
		};
		static_for<G::R3>([&](auto qc) {
			constexpr int q3 = decltype(qc)::value;
			const int iRe = tid + 256 * q3 + o, iIm = iRe - KT;
			if (iRe < B) add(iRe, yRe[q3]);
			if (iIm >= 0) add(iIm, yIm[q3]);
			// a warp sync every eight samples bounds how many ring loads the compiler keeps in flight at once: with
			// all 24 in flight, the kernel no longer fits the 128 registers of two CTAs per SM
			if constexpr (q3 % 4 == 3) __syncwarp();
		});
	};
	// the twiddle bases of the two radix-16 passes, re-read (L1 hits) right before the pass that needs them: an offset
	// that is opaque to the compiler keeps them from being hoisted into 32 registers live for the whole kernel
	auto tw_bases = [&]() {
		int wofs = 0;
#ifndef B200S_EMU
		asm volatile("" : "+r"(wofs));
#endif
		return pair_tw_dif<KT>(x.twiddle + wofs, tid);
	};
	for (int f = 0; f < cl.nFrames; f += 2) {
		f2 yRe[G::R3], yIm[G::R3];
		const bool hasB = f + 1 < cl.nFrames;
		const int tA = frames[f].t;
		// samples emitted between the two blocks; without a second block nothing is emitted between them
		const int gap = hasB ? frames[f + 1].t - tA : 0;
		emit(tA - emitted); // while the spectra are on their way
		if constexpr (PROBE != 3) {
			mbar_wait(&stageBar, stagePar);
			stagePar ^= 1u;
		}
		const float2 *sA = stY, *sB = hasB ? stY + KT : stY;
#ifdef B200S_EMU_EXACT_FFT // test builds only: the oracle's double FFT, results handed over in the registers of the real path
		{
			float *yt = (float *)buf;
			if (tid == 0) {
				std::vector<float> ta(B), tb(B);
				emu_exact_inverse(sA, B, o, g.N, ta.data());
				if (hasB) emu_exact_inverse(sB, B, o, g.N, tb.data());
				for (int i = 0; i < B; ++i) { // the synthesis window, as in the register path
					yt[i] = fmul(ta[i], x.window[i]);
					yt[B + i] = hasB ? fmul(tb[i], x.window[i]) : 0.f;
				}
			}
			__syncthreads();
			static_for<G::R3>([&](auto qc) {
				constexpr int q3 = decltype(qc)::value;
				const int iRe = tid + 256 * q3 + o, iIm = iRe - KT;
				yRe[q3] = iRe < B ? f2_make(yt[iRe], yt[B + iRe]) : f2_make(0.f, 0.f);
				yIm[q3] = iIm >= 0 ? f2_make(yt[iIm], yt[B + iIm]) : f2_make(0.f, 0.f);
			});
		}
#else
		{
			// ---- first inverse-FFT pass takes its inputs from the staged spectra:
			//      Z'[k] = Y[2k] for k < K/2, conj(Y[2(K-1-k)+1]) otherwise; thread tid < M1 needs k = q*M1 + tid, q = 0..15
			c2 v[16];
			if (tid < G::M1) {
				static_for<16>([&](auto qc) {
					constexpr int q = decltype(qc)::value;
					const int k = q * G::M1 + tid;
					const int b = q < 8 ? 2 * k : 2 * (KT - 1 - k) + 1;
					const float sg = q < 8 ? 1.f : -1.f;
					const float2 a = sA[b], bb = sB[b];
					v[q] = c2{f2_make(a.x, bb.x), f2_make(sg * a.y, sg * bb.y)};
				});
			} else {
				// defined on the idle threads too: ptxas would otherwise keep all 64 registers live around the whole loop
				static_for<16>([&](auto qc) { v[decltype(qc)::value] = c2{f2_make(0.f, 0.f), f2_make(0.f, 0.f)}; });
			}
			const PairTw tw = tw_bases();
			__syncthreads(); // every staged spectrum is read: pass 1 writes over them
			if (tid < G::M1) pair_dif_pass1<KT>(buf, tw, tid, v); // (uses tw.a only)
		}
		__syncthreads(); // buf complete
		{
			// last pass in registers, then the half-bin post-twiddle: time sample i of the block is
			// 2*Re(z[i-o] * conj(pre[i-o])) for i >= o and 2*Im(z[i-o+K] * conj(pre[i-o+K])) for i < o,
			// so z[n2] yields sample n2+o (if < B) from its real part and sample n2+o-K (if >= 0) from its imaginary part
			c2 z[G::R3];
			if constexpr (PROBE == 4) {
				static_for<G::R3>([&](auto qc) { z[decltype(qc)::value] = c2{f2_make((float)tid, 0.f), f2_make(0.f, (float)decltype(qc)::value)}; });
			} else {
				pair_dif_pass23<KT>(buf, tw_bases(), tid, z); // (uses tw.b only)
			}
			static_for<G::R3>([&](auto qc) {
				constexpr int q3 = decltype(qc)::value;
				const int n2 = (tid & 15) + 16 * (tid >> 4) + 256 * q3;
				// one 16-byte table entry per element: {window[n2+o], window[n2+o-K], pre-twiddle}; the synthesis window
				// (:397-399, y * window) is applied here, where the index is fixed per thread
				const float4 tb = __ldg(x.anaTab + n2);
				yRe[q3] = muls(muls(fmas(z[q3].im, tb.w, muls(z[q3].re, tb.z)), 2.f), tb.x);
				yIm[q3] = muls(muls(fmas(z[q3].re, -tb.w, muls(z[q3].im, tb.z)), 2.f), tb.y);
			});
		}
#endif
		__syncthreads(); // every read of buf has ended: the next pair's spectra may land there
		if constexpr (PROBE == 3) {
			mbar_wait(&stageBar, stagePar);
			stagePar ^= 1u;
		}
		if (f + 2 < cl.nFrames) stage_pair(f + 2);
		// ---- overlap-add, per ring slot in the reference's order: block A's sample, the emission of the samples
		//      between the two blocks, then block B's sample (relative to the head after the emission)
		add_block(yRe, yIm, false);
		if (hasB) {
			// gap <= P: inside a call k_plan triggers block f+1 exactly H output samples after block f (samplesSinceLast
			// restarts at 0 on a trigger and a block fires the moment it reaches H, :281-286), and H <= B <= P (configure)
			__syncthreads();
			emit(gap);
			__syncthreads();
			add_block(yRe, yIm, true);
		}
		__syncthreads();
	}
	{
		// (re-read here: a register that holds the count through the block loop costs the kernel spills)
		const int nOut = __ldg(&x.call[s].nOut);
		emit(nOut - emitted);
		for (int i = nOut + tid; i < x.outTail; i += 256) st_stream(out + i, 0.f); // (per-stream calls: the row's zero tail)
	}
	__syncthreads();
	// the windowProducts the ring would carry into the next call, slot i for output sample emitted + i: gathered in the
	// (now idle) FFT buffer before any is stored, since in a short call they read the carried values they replace
	// (P <= B + H <= 2B < 2N floats: the buffer holds 4K)
	float *wpNext = (float *)buf;
	for (int i = tid; i < P; i += 256) wpNext[i] = wp_at(emitted + i);
	__syncthreads();
	for (int i = tid; i < P; i += 256) {
		int p = head + i;
		if (p >= P) p -= P;
		gp[i] = pend[p];
		gw[i] = wpNext[i];
	}
}
template <int KT>
__global__ void __launch_bounds__(256, 2) k_synth2(Ctx x) { synth2_body<KT, 0>(x); }
#ifdef B200S_SYNTH_PROBES
template <int KT, int PROBE>
__global__ void __launch_bounds__(256, 2) k_synth2_probe(Ctx x) { synth2_body<KT, PROBE>(x); }
#endif

static inline size_t smem_analyse2(const Cfg &g) {
	const int len = g.K == 3072 ? PairGeo<3072>::LEN : PairGeo<2560>::LEN;
	return sizeof(float4) * len + sizeof(float) * 2 * stage_len(g.B);
}
static inline size_t smem_synth2(const Cfg &g) {
	const int len = g.K == 3072 ? PairGeo<3072>::LEN : PairGeo<2560>::LEN;
	return sizeof(float4) * len + sizeof(float) * g.pendLen;
}

} // namespace b200s
