// IVF range batch (rxgpu_ivf_search_range_batch): the key pass of the any-k select (ivf_select.cuh) writes every probed (query, row) key
// ord(dist) << 32 | row; these kernels then keep, per query, the keys whose distance is below its radius.
//
//   ivf_range_count_kernel  -- one CTA per tile of up to kIvfRangeTile keys of one query (a host plan of (query, tile) pairs, so a
//                              query with 10^6 probed rows is spread over many CTAs): matches per query
//   ivf_range_emit_kernel   -- the same tiles, for the queries of one survivor sub-chunk: each match's (ordered distance word, label)
//                              at its query's survivor offset, in no particular order (the segmented sorts order them)
//   ivf_range_gather_kernel -- after the sorts: the best min(matches, max_out) survivors of each query, packed, distances decoded
// The test is the range-mode scan's own: ord_float(key word) < radius as floats (the key holds -0 as +0, which compares equal), so a
// NaN radius matches nothing, -inf nothing and +inf every probed row.
#pragma once
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace rxgpu {

constexpr int kIvfRangeThreads = 256;
constexpr int kIvfRangeItems = 8;
constexpr uint32_t kIvfRangeTile = kIvfRangeThreads * kIvfRangeItems;

__device__ __forceinline__ bool range_hit(uint64_t key, float radius) { return ord_float(uint32_t(key >> 32)) < radius; }

// tile t = (query qi of the chunk, tile index j): keys [j * kIvfRangeTile, + kIvfRangeTile) of the query's keys[qoff[qi] - origin, + nkeys[qi])
__global__ void __launch_bounds__(kIvfRangeThreads) ivf_range_count_kernel(const uint64_t* keys, const uint64_t* qoff, const uint64_t* nkeys,
																			uint64_t origin, const float* radius, const uint2* tiles,
																			uint32_t* count) {
	using Reduce = cub::BlockReduce<uint32_t, kIvfRangeThreads>;
	__shared__ Reduce::TempStorage tmp;
	const uint2 t = tiles[blockIdx.x];
	const uint64_t* kq = keys + (qoff[t.x] - origin);
	const uint64_t i0 = uint64_t(t.y) * kIvfRangeTile, i1 = min(nkeys[t.x], i0 + kIvfRangeTile);
	const float r = radius[t.x];
	uint32_t c = 0;
	for (uint64_t i = i0 + threadIdx.x; i < i1; i += kIvfRangeThreads) {
		c += range_hit(kq[i], r);
	}
	c = Reduce(tmp).Sum(c);
	if (threadIdx.x == 0 && c) {
		atomicAdd(&count[t.x], c);
	}
}

// the tiles of the sub-chunk's queries [s0, s0 + ns): query qi's matches go to out_*[seg[qi - s0], + its matches); cursor (zero on entry)
// hands out the places
__global__ void __launch_bounds__(kIvfRangeThreads) ivf_range_emit_kernel(const uint64_t* keys, const uint64_t* qoff, const uint64_t* nkeys,
																		   uint64_t origin, const float* radius, const uint2* tiles, uint32_t s0,
																		   const int* seg, const uint64_t* labels, uint32_t* cursor,
																		   uint32_t* out_ord, uint64_t* out_label) {
	using Scan = cub::BlockScan<uint32_t, kIvfRangeThreads>;
	__shared__ Scan::TempStorage tmp;
	__shared__ uint32_t base;
	const uint2 t = tiles[blockIdx.x];
	const uint64_t* kq = keys + (qoff[t.x] - origin);
	const uint64_t i0 = uint64_t(t.y) * kIvfRangeTile, n = nkeys[t.x];
	const float r = radius[t.x];
	uint64_t key[kIvfRangeItems];
	uint32_t hits = 0, c = 0;
#pragma unroll
	for (int j = 0; j < kIvfRangeItems; ++j) {
		const uint64_t i = i0 + uint64_t(j) * kIvfRangeThreads + threadIdx.x;
		key[j] = i < n ? kq[i] : kKeyNone;
		if (i < n && range_hit(key[j], r)) {
			hits |= 1u << j;
			++c;
		}
	}
	uint32_t before, total;
	Scan(tmp).ExclusiveSum(c, before, total);
	if (threadIdx.x == 0) {
		base = total ? atomicAdd(&cursor[t.x], total) : 0u;
	}
	__syncthreads();
	uint32_t pos = uint32_t(seg[t.x - s0]) + base + before;
#pragma unroll
	for (int j = 0; j < kIvfRangeItems; ++j) {
		if (hits >> j & 1u) {
			out_ord[pos] = uint32_t(key[j] >> 32);
			out_label[pos] = labels[uint32_t(key[j])];
			++pos;
		}
	}
}

// query qi of the sub-chunk: its sorted survivors ord / label[seg[qi], ...) -> out_*[pack[qi], pack[qi + 1]), the distance decoded as the
// single-query range call decodes it (ord_float: a zero distance is +0)
__global__ void ivf_range_gather_kernel(const uint32_t* ord, const uint64_t* label, const int* seg, const int* pack, float* out_dist,
										uint64_t* out_label) {
	const uint32_t qi = blockIdx.x;
	const int from = seg[qi], to = pack[qi], len = pack[qi + 1] - to;
	for (int j = blockIdx.y * blockDim.x + threadIdx.x; j < len; j += gridDim.y * blockDim.x) {
		out_dist[to + j] = ord_float(ord[from + j]);
		out_label[to + j] = label[from + j];
	}
}

}  // namespace rxgpu
