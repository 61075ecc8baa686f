// IVF KNN at any k (rxgpu_ivf_search_knn_large_k): one distance pass over the probed lists writes every probed (query, row) key
// ord(dist) << 32 | row to a workspace at a fixed position; an exact MSB radix select then keeps the k smallest keys per query.
//
//   ivf_probe_rows_kernel    -- probed rows per query (sum of its probed lists' sizes)
//   ivf_key_plan_kernel      -- per query chunk: its work items query-major, each with the workspace slot of its first key
//                               (query offset, from a device scan of the totals, + prefix of the query's earlier lists)
//   knn_scan_warp<kKeysOut>  -- the keys (knn_scan.cuh: the exact scan's own per-row arithmetic, so the same bits as the fused path)
//   ivf_select_cta_kernel    -- one CTA per query: radix histograms of the keys in shared memory, 11 / 11 / 10 bits of the distance
//                               word, then of the row word (only reached when a group of bit-equal distances straddles the k-th
//                               place), then the keys <= the k-th key are compacted with their labels
//   ivf_select_hist / _pick / _compact_kernel -- the same select for one query with more than kIvfSelCtaKeys keys, spread over many CTAs
//                               (global histogram, one picking CTA per digit)
// Keys of one query are unique (a row sits in one list), so the k-th smallest key is well defined and exactly k keys are <= it.
#pragma once
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace rxgpu {

constexpr int kIvfSelThreads = 1024;
constexpr uint32_t kIvfSelBins = 2048;      // 11-bit digits
constexpr int kIvfSelPasses = 6;            // 64 key bits: 11 + 11 + 10 (distance word), 11 + 11 + 10 (row word)
constexpr uint64_t kIvfSelCtaKeys = 1u << 16;  // up to this many keys a query is selected by one CTA
constexpr uint32_t kMaxLargeK = 65535;   // rxgpu_ivf_search_knn_large_k: k in [1, 65535], as rxgpu_search_knn
// workspace of one query chunk: keys (8 bytes each; 512 MiB at the cap) and survivor slots (k per query, 24 bytes each with the sort
// buffers; 384 MiB at the cap).  A batch above either cap runs in query chunks; one query above the key cap is a chunk of its own.
constexpr uint64_t kIvfKeyCap = 1ull << 26;
constexpr uint64_t kIvfSlotCap = 1ull << 24;

// bits [sel_lo(p), sel_hi(p)) of the key are the digit of pass p
__host__ __device__ constexpr int sel_hi(int pass) { return pass == 0 ? 64 : pass == 1 ? 53 : pass == 2 ? 42 : pass == 3 ? 32 : pass == 4 ? 21 : 10; }
__host__ __device__ constexpr int sel_lo(int pass) { return pass == 5 ? 0 : sel_hi(pass + 1); }

// select state of one query: the keys matching `prefix` above the current digit hold the k-th key at position `rank` (1-based) among
// them; once `done`, the survivors are exactly the keys <= cut
struct SelState {
	unsigned long long prefix;
	unsigned long long cut;
	uint32_t rank;
	uint32_t done;
};
using SelScan = cub::BlockScan<uint32_t, kIvfSelThreads>;

__device__ __forceinline__ bool sel_match(uint64_t key, uint64_t prefix, int pass) {
	const int hi = sel_hi(pass);
	return hi == 64 || (key >> hi) == (prefix >> hi);
}
__device__ __forceinline__ uint32_t sel_digit(uint64_t key, int pass) {
	return uint32_t(key >> sel_lo(pass)) & ((1u << (sel_hi(pass) - sel_lo(pass))) - 1u);
}

// histogram of the digit of pass `pass` over the keys [i0, n) step `step` that match the prefix (shared-memory atomics)
__device__ __forceinline__ void sel_histogram(const uint64_t* keys, uint64_t i0, uint64_t n, uint64_t step, uint64_t prefix, int pass,
											  uint32_t* hist) {
	for (uint64_t i = i0; i < n; i += step) {
		const uint64_t key = keys[i];
		if (sel_match(key, prefix, pass)) {
			atomicAdd(&hist[sel_digit(key, pass)], 1u);
		}
	}
}

// block of kIvfSelThreads: find the bin of the rank-th matching key in hist; either every key of that bin is in (done, cut = the bin's
// largest key) or the select narrows to the bin for the next pass.  The caller synchronises before s is read again.
__device__ __forceinline__ void sel_pick(const uint32_t* hist, SelState* s, int pass, SelScan::TempStorage& tmp) {
	const uint32_t h0 = hist[2 * threadIdx.x], h1 = hist[2 * threadIdx.x + 1];
	const uint32_t rank = s->rank;  // read before the scan's barriers, written after them
	uint32_t before;
	SelScan(tmp).ExclusiveSum(h0 + h1, before);
	if (before < rank && rank <= before + h0 + h1) {  // exactly one thread
		uint32_t b = 2 * threadIdx.x, cb = before, hb = h0;
		if (rank > before + h0) {
			b += 1, cb += h0, hb = h1;
		}
		const int lo = sel_lo(pass);
		const unsigned long long p = s->prefix | (uint64_t(b) << lo);
		if (cb + hb == rank) {
			s->cut = p | ((1ull << lo) - 1ull);
			s->done = 1;
		} else {
			s->prefix = p;
			s->rank = rank - cb;
		}
	}
}

// a survivor: its distance word, and its label -- or, with no labels (the local part of a sharded search), its row
__device__ __forceinline__ void sel_emit(uint64_t key, const uint64_t* labels, uint32_t pos, uint32_t* out_ord, uint64_t* out_label) {
	out_ord[pos] = uint32_t(key >> 32);
	out_label[pos] = labels ? labels[uint32_t(key)] : uint64_t(uint32_t(key));
}

// the survivors of the query chunk [q0, q0 + cq) -- ordered by (distance word, row) -- into a sharded KNN's payload at row q0:
// one thread per slot, rows of `stride` entries
__global__ void ivf_shard_emit_kernel(const uint32_t* ord, const uint64_t* row, const uint32_t* count, uint32_t k, uint32_t cq,
									  const uint64_t* labels, uint32_t stride, float* out_dist, uint32_t* out_idx, uint64_t* out_label,
									  uint32_t* out_count) {
	const uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
	const uint32_t qi = uint32_t(i / k), j = uint32_t(i % k);
	if (qi >= cq) {
		return;
	}
	if (j == 0) {
		out_count[qi] = count[qi];
	}
	if (j < count[qi]) {
		const size_t at = size_t(qi) * stride + j;
		const uint32_t r = uint32_t(row[i]);
		out_dist[at] = key_dist(ord[i], false);  // as the fused path decodes it: a zero distance is +0
		out_idx[at] = r;
		out_label[at] = labels[r];
	}
}

// one warp per query: rows[q] = sum of the sizes of its probed lists (work items probe-major, work[p * nq + q])
__global__ void ivf_probe_rows_kernel(const uint4* work, uint32_t nq, uint32_t nprobe, uint64_t* rows) {
	const uint32_t q = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
	const int lane = threadIdx.x & 31;
	if (q >= nq) {
		return;
	}
	uint64_t s = 0;
	for (uint32_t p = lane; p < nprobe; p += 32) {
		const uint4 w = work[size_t(p) * nq + q];
		s += w.z - w.y;
	}
#pragma unroll
	for (int off = 16; off > 0; off >>= 1) {
		s += __shfl_xor_sync(0xffffffffu, s, off);
	}
	if (lane == 0) {
		rows[q] = s;
	}
}

// one warp per query of the chunk [q0, q0 + cq): its work items query-major, work_chunk[(q - q0) * nprobe + p] = work[p * nq + q] with .w
// (the centroid, unused by the scan) replaced by the slot of the item's first key in the chunk's workspace: the query's key offset in
// the chunk + the rows of the lists probed before p.  A chunk holds at most 2^26 keys or one query (fewer than 2^32 rows): 32 bits.
__global__ void ivf_key_plan_kernel(const uint4* work, uint32_t nq, uint32_t nprobe, uint32_t q0, uint32_t cq, const uint64_t* qoff,
									uint4* work_chunk) {
	const uint32_t qi = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
	const int lane = threadIdx.x & 31;
	if (qi >= cq) {
		return;
	}
	const uint32_t q = q0 + qi;
	uint64_t run = qoff[q] - qoff[q0];
	for (uint32_t p0 = 0; p0 < nprobe; p0 += 32) {
		const uint32_t p = p0 + lane;
		const uint4 w = p < nprobe ? work[size_t(p) * nq + q] : make_uint4(0, 0, 0, 0);
		const uint64_t len = w.z - w.y;
		uint64_t incl = len;
#pragma unroll
		for (int off = 1; off < 32; off <<= 1) {
			const uint64_t o = __shfl_up_sync(0xffffffffu, incl, off);
			incl += lane >= off ? o : 0;
		}
		if (p < nprobe) {
			work_chunk[size_t(qi) * nprobe + p] = make_uint4(w.x, w.y, w.z, uint32_t(run + incl - len));
		}
		run += __shfl_sync(0xffffffffu, incl, 31);
	}
}

// One CTA per query of a chunk (query qi's keys at keys[qoff[qi] - origin, + nkeys[qi])): the k keys <= the k-th key go to
// out_*[qi * k, + out_count[qi]) in no particular order.  Queries with more than kIvfSelCtaKeys keys are left to the multi-CTA kernels.
__global__ void __launch_bounds__(kIvfSelThreads) ivf_select_cta_kernel(const uint64_t* keys, const uint64_t* qoff, const uint64_t* nkeys,
																	 uint64_t origin, uint32_t k, const uint64_t* labels, uint32_t* out_ord,
																	 uint64_t* out_label, uint32_t* out_count) {
	__shared__ uint32_t hist[kIvfSelBins];
	__shared__ SelState s;
	__shared__ SelScan::TempStorage tmp;
	__shared__ uint32_t cnt;
	const uint32_t qi = blockIdx.x;
	const uint64_t n = nkeys[qi];
	if (n > kIvfSelCtaKeys) {
		return;
	}
	const uint64_t* kq = keys + (qoff[qi] - origin);
	if (threadIdx.x == 0) {
		s = SelState{0ull, kKeyNone, k, n <= k ? 1u : 0u};
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
		sel_histogram(kq, threadIdx.x, n, kIvfSelThreads, s.prefix, pass, hist);
		__syncthreads();
		sel_pick(hist, &s, pass, tmp);
	}
	__syncthreads();
	const uint64_t cut = s.cut;
	for (uint64_t i = threadIdx.x; i < n; i += kIvfSelThreads) {
		const uint64_t key = kq[i];
		if (key <= cut) {
			sel_emit(key, labels, qi * k + atomicAdd(&cnt, 1u), out_ord, out_label);
		}
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		out_count[qi] = cnt;
	}
}

// the select of one query with many keys: per pass, every CTA histograms a slice into ghist (zero on entry), then one CTA picks the bin
// and zeroes ghist again; passes after the select is done return at once
__global__ void __launch_bounds__(kIvfSelThreads) ivf_select_hist_kernel(const uint64_t* keys, uint64_t n, const SelState* s, int pass,
																	  uint32_t* ghist) {
	__shared__ uint32_t hist[kIvfSelBins];
	if (s->done) {
		return;
	}
	for (uint32_t b = threadIdx.x; b < kIvfSelBins; b += kIvfSelThreads) {
		hist[b] = 0;
	}
	__syncthreads();
	sel_histogram(keys, blockIdx.x * uint64_t(kIvfSelThreads) + threadIdx.x, n, uint64_t(gridDim.x) * kIvfSelThreads, s->prefix, pass, hist);
	__syncthreads();
	for (uint32_t b = threadIdx.x; b < kIvfSelBins; b += kIvfSelThreads) {
		if (hist[b]) {
			atomicAdd(&ghist[b], hist[b]);
		}
	}
}
__global__ void __launch_bounds__(kIvfSelThreads) ivf_select_pick_kernel(SelState* s, int pass, uint32_t* ghist) {
	__shared__ uint32_t hist[kIvfSelBins];
	__shared__ SelScan::TempStorage tmp;
	if (s->done) {
		return;
	}
	for (uint32_t b = threadIdx.x; b < kIvfSelBins; b += kIvfSelThreads) {
		hist[b] = ghist[b];
		ghist[b] = 0;
	}
	__syncthreads();
	sel_pick(hist, s, pass, tmp);
}
__global__ void __launch_bounds__(kIvfSelThreads) ivf_select_compact_kernel(const uint64_t* keys, uint64_t n, const SelState* s,
																		 const uint64_t* labels, uint32_t* out_ord, uint64_t* out_label,
																		 uint32_t* out_count) {
	const uint64_t cut = s->cut;
	for (uint64_t i = blockIdx.x * uint64_t(kIvfSelThreads) + threadIdx.x; i < n; i += uint64_t(gridDim.x) * kIvfSelThreads) {
		const uint64_t key = keys[i];
		if (key <= cut) {
			sel_emit(key, labels, atomicAdd(out_count, 1u), out_ord, out_label);
		}
	}
}

// segment bounds of the survivors for the segmented sorts: query i owns [i * k, i * k + count[i])
__global__ void ivf_sort_bounds_kernel(const uint32_t* count, uint32_t k, uint32_t nseg, int* begin, int* end) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < nseg) {
		begin[i] = int(i * k);
		end[i] = int(i * k + count[i]);
	}
}

}  // namespace rxgpu
