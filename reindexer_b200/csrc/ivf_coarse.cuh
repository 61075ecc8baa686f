// IVF coarse quantiser (faiss::IndexIVF::search -> quantizer->search(nprobe), IndexIVF.cpp) at any nlist: the nprobe nearest centroids
// of every query under (distance, centroid id), emitted as the work items of the list scans, probe-major:
// work[p * nq + q] = (q, list_begin[c], list_end[c] or list_begin[c + 1], c), p-th nearest centroid c.
//
// Per chunk of queries (at most kIvfKeyCap keys, query-major, 8 bytes per (query, centroid)):
//   ivf_coarse_dist_kernel   -- grid (query tile, centroid slice): QT queries staged in shared memory, each warp takes kCoarseRows
//                               centroids at a time against the whole tile through row_dists_warp (the exact scan's per-row
//                               arithmetic, so every centroid distance has the same bits on every path) and writes make_key(d, c)
//   ivf_coarse_select_kernel -- one CTA per query: the radix select of ivf_select.cuh (2048-bin passes over the distance word, then the
//                               centroid word) finds the nprobe-th smallest key; the keys <= it are compacted (in no order) with the
//                               query's segment bounds for the sort
//   cub::DeviceSegmentedSort -- the survivors of each query in ascending key order
//   ivf_coarse_emit_kernel   -- the work items
// Keys of one query are unique (one per centroid), so exactly nprobe keys survive.
#pragma once
#include "ivf_select.cuh"
#include "knn_scan.cuh"

namespace rxgpu {

constexpr int kCoarseRows = 4;          // centroids per warp step: each staged query float4 feeds 4 rows
constexpr int kCoarseTile = 16;         // queries per tile of a batch
constexpr size_t kCoarseSmemMax = 200 * 1024;

// shared memory of a query tile of qt queries, zero padded to whole 128-float chunks
__host__ __device__ inline size_t coarse_smem_bytes(int qt, uint32_t dim) { return size_t(qt) * ((dim + 127u) / 128u) * 512u; }

// kArgmin (k-means assignment, rxgpu_ivf_train / rxgpu_ivf_assign): instead of every key, the query's smallest key goes to keys[query]
// through a 64-bit atomicMin over the CTAs of its centroid slices (order-independent, so deterministic; keys preset to kKeyNone)
template <bool kIsL2, int QT, bool kArgmin = false>
__global__ void __launch_bounds__(kScanThreads, 2) ivf_coarse_dist_kernel(const float* centroids, uint32_t pitch, uint32_t dim, uint32_t nlist,
																		   const float* queries, uint32_t cq, const float* centroid_norm_coefs,
																		   uint64_t* keys) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t nch = (dim + 127u) / 128u, dp4 = nch * 32u, pitch4 = pitch >> 2;
	const uint32_t t0 = blockIdx.x * QT;  // first query of the tile in the chunk
	float4* sq4 = reinterpret_cast<float4*>(smem_raw);
	{
		float* sq = reinterpret_cast<float*>(sq4);
		const uint32_t dp = dp4 * 4;
		for (uint32_t i = threadIdx.x; i < QT * dp; i += blockDim.x) {
			const uint32_t qi = i / dp, c = i - qi * dp;
			sq[i] = (t0 + qi < cq && c < dim) ? queries[size_t(t0 + qi) * dim + c] : 0.f;
		}
	}
	__syncthreads();
	const float4* q4[kCoarseRows][QT];
#pragma unroll
	for (int r = 0; r < kCoarseRows; ++r) {
#pragma unroll
		for (int j = 0; j < QT; ++j) {
			q4[r][j] = sq4 + j * dp4;
		}
	}
	const float4* rows4 = reinterpret_cast<const float4*>(centroids);
	const uint32_t ngroups = (nlist + kCoarseRows - 1) / kCoarseRows;
	uint64_t best = kKeyNone;  // kArgmin: lane j < QT keeps the best key of query j over this warp's centroids
	for (uint32_t g = blockIdx.y * kScanWarps + warp; g < ngroups; g += gridDim.y * kScanWarps) {
		uint32_t row[kCoarseRows];
#pragma unroll
		for (int r = 0; r < kCoarseRows; ++r) {
			row[r] = min(g * kCoarseRows + r, nlist - 1);  // past the end: a valid row, its distance is not written
		}
		float d[kCoarseRows][QT];
		// IndexFlatCosine: knn_cosine = IP * norm coefficient of the centroid
		row_dists_warp<kIsL2, kCoarseRows, QT>(rows4, pitch4, nch, row, q4, centroid_norm_coefs, lane, d);
		if constexpr (kArgmin) {
#pragma unroll
			for (int j = 0; j < QT; ++j) {
#pragma unroll
				for (int r = 0; r < kCoarseRows; ++r) {
					const uint32_t c = g * kCoarseRows + r;
					if (j == lane && c < nlist) {
						best = min(best, make_key(d[r][j], c));
					}
				}
			}
		} else {
			// every lane holds every distance: lane l writes slots l, l + 32, ... of the (query, row) pairs, rows fastest
#pragma unroll
			for (int j = 0; j < QT; ++j) {
#pragma unroll
				for (int r = 0; r < kCoarseRows; ++r) {
					const uint32_t c = g * kCoarseRows + r;
					if (((j * kCoarseRows + r) & 31) == lane && c < nlist && t0 + j < cq) {
						keys[size_t(t0 + j) * nlist + c] = make_key(d[r][j], c);
					}
				}
			}
		}
	}
	if constexpr (kArgmin) {
		static_assert(QT <= 32, "one lane per query of the tile");
		if (lane < QT && t0 + lane < cq && best != kKeyNone) {
			atomicMin(reinterpret_cast<unsigned long long*>(keys) + t0 + lane, static_cast<unsigned long long>(best));
		}
	}
}

// One CTA per query of a chunk (its keys at keys[qi * nlist, + nlist)): the nprobe smallest keys to out[qi * nprobe, + nprobe) in no
// particular order, and the query's segment [seg_begin[qi], seg_end[qi]) of out for the sort
__global__ void __launch_bounds__(kIvfSelThreads) ivf_coarse_select_kernel(const uint64_t* keys, uint32_t nlist, uint32_t nprobe, uint64_t* out,
																		   int* seg_begin, int* seg_end) {
	__shared__ uint32_t hist[kIvfSelBins];
	__shared__ SelState s;
	__shared__ SelScan::TempStorage tmp;
	__shared__ uint32_t cnt;
	const uint32_t qi = blockIdx.x;
	const uint64_t* kq = keys + size_t(qi) * nlist;
	if (threadIdx.x == 0) {
		s = SelState{0ull, kKeyNone, nprobe, nlist <= nprobe ? 1u : 0u};
		cnt = 0;
	}
	for (int pass = 0; pass < kIvfSelPasses; ++pass) {
		__syncthreads();
		if (s.done) {
			break;
		}
		for (uint32_t b = threadIdx.x; b < kIvfSelBins; b += kIvfSelThreads) {
			hist[b] = 0;
		}
		__syncthreads();
		sel_histogram(kq, threadIdx.x, nlist, kIvfSelThreads, s.prefix, pass, hist);
		__syncthreads();
		sel_pick(hist, &s, pass, tmp);
	}
	__syncthreads();
	const uint64_t cut = s.cut;
	uint64_t* oq = out + size_t(qi) * nprobe;
	for (uint32_t i = threadIdx.x; i < nlist; i += kIvfSelThreads) {
		const uint64_t key = kq[i];
		if (key <= cut) {
			oq[atomicAdd(&cnt, 1u)] = key;
		}
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		seg_begin[qi] = int(qi * nprobe);
		seg_end[qi] = int(qi * nprobe + cnt);
	}
}

// work items of the chunk [q0, q0 + cq) from its sorted survivors (sorted[qi * nprobe + p] = the p-th nearest centroid's key)
__global__ void ivf_coarse_emit_kernel(const uint64_t* sorted, uint32_t nq, uint32_t nprobe, uint32_t q0, uint32_t cq, const uint32_t* list_begin,
									   const uint32_t* list_end, uint4* work) {
	const uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
	if (i >= uint64_t(cq) * nprobe) {
		return;
	}
	const uint32_t qi = uint32_t(i / nprobe), p = uint32_t(i - uint64_t(qi) * nprobe);
	const uint32_t c = uint32_t(sorted[i]);
	work[size_t(p) * nq + q0 + qi] = make_uint4(q0 + qi, list_begin[c], list_end ? list_end[c] : list_begin[c + 1], c);
}

}  // namespace rxgpu
