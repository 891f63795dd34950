// state_copy.cuh -- one stream's complete state as a packed record: k_pack_streams gathers the listed streams' state into
// consecutive records, k_unpack_streams scatters records into the listed slots (b200s_copy_streams / _export_streams /
// _import_streams, DESIGN.md §3.12).
//
// A record is [header | region 0 | region 1 | ...]: the header (B200S_RECORD_HEADER bytes) is written and checked by the
// host and never touched here; every region is one per-stream state array (its bytes of the stream, padded with zeros
// to a multiple of 16).  One thread moves one 16-byte chunk of one record: a single 16-byte load / store on the state
// side when the region's bytes per stream are a multiple of 16 (every row then starts 16-byte aligned), four 4-byte
// accesses otherwise (the scheduler entry, the random engine, the pitch smoother, and the history at 44.1 kHz, whose
// length B+H is odd).  Plain bandwidth-bound copies: nothing is staged in shared memory.
#pragma once
#include "common.cuh"

namespace b200s {

#define B200S_STATE_REGIONS 10
#define B200S_RECORD_HEADER 128

struct StateRegion {
	char *base;     // stream s's bytes start at base + s * bytes
	unsigned bytes; // per stream, a multiple of 4
	unsigned off;   // where the region starts in the record, a multiple of 16
};
// passed by value: the engine's state arrays (with the history buffer that is current when the launch is enqueued)
struct StateRegions {
	StateRegion r[B200S_STATE_REGIONS]; // ascending `off`, r[0].off = B200S_RECORD_HEADER
	unsigned recBytes;                  // bytes of one record, a multiple of 16
};

// the region that holds record byte `pos` (static indices only: the table stays in the parameter space)
__device__ __forceinline__ StateRegion state_region(const StateRegions &t, unsigned pos) {
	StateRegion g = t.r[0];
#pragma unroll
	for (int j = 1; j < B200S_STATE_REGIONS; ++j)
		if (pos >= t.r[j].off) g = t.r[j];
	return g;
}

// (float4 is only the 16-byte container of the wide accesses: loads and stores move its bits unchanged, whatever the
// region holds)
// grid (chunk blocks, min(n, 65535)), 256 threads: record k of `rec` <- stream streams[k]
__global__ void __launch_bounds__(256) k_pack_streams(StateRegions t, const int *streams, int n, char *rec) {
	const unsigned pos = B200S_RECORD_HEADER + 16u * (blockIdx.x * blockDim.x + threadIdx.x);
	if (pos >= t.recBytes) return;
	const StateRegion g = state_region(t, pos);
	const unsigned o = pos - g.off;
	const bool wide = o < g.bytes && g.bytes % 16 == 0;
	const unsigned m = o < g.bytes ? (g.bytes - o) / 4 : 0; // words of the region left from here (narrow regions)
	for (int k = blockIdx.y; k < n; k += gridDim.y) {
		const char *src = g.base + (size_t)streams[k] * g.bytes + o;
		char *dst = rec + (size_t)k * t.recBytes + pos;
		if (wide) {
			*(float4 *)dst = *(const float4 *)src;
		} else {
			const unsigned *w = (const unsigned *)src;
			unsigned *q = (unsigned *)dst;
			q[0] = m > 0 ? w[0] : 0u;
			q[1] = m > 1 ? w[1] : 0u;
			q[2] = m > 2 ? w[2] : 0u;
			q[3] = m > 3 ? w[3] : 0u;
		}
	}
}

// grid (chunk blocks, min(n, 65535)), 256 threads: stream streams[k] <- record k of `rec` (padding is not written)
__global__ void __launch_bounds__(256) k_unpack_streams(StateRegions t, const int *streams, int n, const char *rec) {
	const unsigned pos = B200S_RECORD_HEADER + 16u * (blockIdx.x * blockDim.x + threadIdx.x);
	if (pos >= t.recBytes) return;
	const StateRegion g = state_region(t, pos);
	const unsigned o = pos - g.off;
	if (o >= g.bytes) return;
	const unsigned m = (g.bytes - o) / 4;
	for (int k = blockIdx.y; k < n; k += gridDim.y) {
		char *dst = g.base + (size_t)streams[k] * g.bytes + o;
		const char *src = rec + (size_t)k * t.recBytes + pos;
		if (g.bytes % 16 == 0) {
			*(float4 *)dst = *(const float4 *)src;
		} else {
			const unsigned *q = (const unsigned *)src;
			unsigned *w = (unsigned *)dst;
			w[0] = q[0];
			if (m > 1) w[1] = q[1];
			if (m > 2) w[2] = q[2];
			if (m > 3) w[3] = q[3];
		}
	}
}

} // namespace b200s
