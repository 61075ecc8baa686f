// HNSW search on the device over a graph built by the reference's CPU code.
//
// Replaces hnswlib::HierarchicalNSWImpl<float>::SearchKnn (cpp_src/core/index/float_vector/hnswlib/hnswalg.h:1988-2012):
//   getLayer0EntryPoint  (:799-827)  greedy descent through levels maxlevel..1
//   searchBaseLayerST<bare_bone=true> (:829-975: initLayer0SearchState, layer0ShouldStopBeforePop, runLayer0Step)
//   trim to k, internal id -> label
// One warp per query ("the HNSW neighbour-expansion step becomes a batched gather + distance kernel"): the neighbour list
// of the expanded node is fetched with one coalesced load, the visited test is a batched atomicOr on a per-warp bitmap in
// HBM, the rows of all unvisited neighbours are gathered with 128-bit coalesced loads (4 rows in flight per lane) and
// reduced with the same per-row arithmetic as knn_scan_warp (so a row's distance is bit-identical on both paths), and then
// the reference's sequential accept logic is replayed over the batch in neighbour order.
//
// The reference's two heaps (top_candidates: max-heap of <= ef; candidate_set: min-heap, both ordered by distance only,
// hnswalg.h:581-585) are represented by ONE list of the <= ef best visited nodes, sorted by distance, each with an "expanded"
// flag: the next node to expand is the first unexpanded entry, the search stops when none is left.  This is equivalent:
// a candidate worse than the current ef-th best (lowerBound) can never be expanded (the loop stops at the first such pop and
// lowerBound only decreases), and every candidate at or below lowerBound is in top_candidates.  Requires a graph without
// deleted nodes (num_deleted_ == 0, the bare-bone branch of hnswalg.h:1982); distances tie only on duplicate vectors.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "internal.h"
#include "hnsw_graph.cuh"
#include "sq8.cuh"
#include "../host/knn_select.h"

using namespace rxgpu;

namespace {

template <bool kIsL2>
__global__ void __launch_bounds__(kHnswThreads, 8) hnsw_search_kernel(const HnswArgs a) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int lane = threadIdx.x & 31;
	const int warp = threadIdx.x >> 5;
	const uint32_t dp4 = hnsw_query_words(a.dim);
	// per-warp shared memory: query | list dist[ef] | list id[ef] | neighbour ids[64] | neighbour dists[64]
	const uint32_t efp = (a.ef + 3u) & ~3u;  // keeps every warp's region 16-byte aligned
	const size_t per_warp = size_t(dp4) * 16 + size_t(efp) * 8 + kMaxNeighbours * 8;
	unsigned char* base = smem_raw + per_warp * warp;
	float4* sq4 = reinterpret_cast<float4*>(base);
	float* l_dist = reinterpret_cast<float*>(base + size_t(dp4) * 16);
	uint32_t* l_id = reinterpret_cast<uint32_t*>(l_dist + efp);
	uint32_t* s_ids = l_id + efp;
	float* s_d = reinterpret_cast<float*>(s_ids + kMaxNeighbours);

	const uint32_t slot = blockIdx.x * kHnswWarps + warp;
	uint32_t* visited = a.visited + size_t(slot) * a.words;
	uint32_t* vlog = a.vlog + size_t(slot) * kVlogCap;
	// deleted candidates (in candidate_set, never in top_candidates): a sorted list per slot in HBM, touched only when the graph
	// holds tombstones
	float* x_dist = a.x_dist ? a.x_dist + size_t(slot) * kHnswXCap : nullptr;
	uint32_t* x_id = a.x_id ? a.x_id + size_t(slot) * kHnswXCap : nullptr;

	for (;;) {
		uint32_t qi = 0;
		if (lane == 0) {
			qi = atomicAdd(a.next_query, 1u);
		}
		qi = __shfl_sync(0xffffffffu, qi, 0);
		if (qi >= a.nq) {
			break;
		}
		float qcorr = 0.f, qcoef = 1.f;
		if (a.codes != nullptr) {  // SQ8: the query's codes (already zero padded to code_pitch) + its corrective offset and coefficient
			uint4* squ = reinterpret_cast<uint4*>(sq4);
			const uint4* q = reinterpret_cast<const uint4*>(a.qcodes + size_t(qi) * a.code_pitch);
			for (uint32_t c = lane; c < a.code_pitch / 16; c += 32) {
				squ[c] = q[c];
			}
			qcorr = a.qcorr[qi];
			qcoef = a.qcoef[qi];
		} else {  // stage_query's loop written out: through the helper, ptxas allocates this kernel's 64 registers differently
			float* sq = reinterpret_cast<float*>(sq4);
			const float* q = a.queries + size_t(qi) * a.dim;
			for (uint32_t c = lane; c < dp4 * 4; c += 32) {
				sq[c] = c < a.dim ? q[c] : 0.f;
			}
		}
		__syncwarp();
		uint32_t n_dist = 0, n_hops = 0;

		// ---- getLayer0EntryPoint (hnswalg.h:799-827): the entry point's distance is not counted
		uint32_t cur = a.enterpoint;
		if (lane == 0) {
			s_ids[0] = cur;
		}
		__syncwarp();
		warp_dists<kIsL2>(a, sq4, s_ids, 1, s_d, lane, qcorr, qcoef);
		float curdist = s_d[0];
		__syncwarp();
		greedy_descent<kIsL2>(a, sq4, cur, curdist, a.maxlevel, 0, s_ids, s_d, lane, n_dist, n_hops, qcorr, qcoef);

		// ---- searchBaseLayerST (hnswalg.h:829-975), unified sorted list
		// With deleted nodes (a.deleted != nullptr, the reference's non-bare-bone branch) the two heaps differ: a deleted node is a
		// candidate (it is expanded) but never a result.  Deleted candidates wait in a second small sorted list X; the next node to
		// expand is the closer of (first unexpanded entry of the result list, head of X); the stop rule becomes "closest candidate
		// worse than the ef-th result AND the result list is full" (layer0ShouldStopBeforePop :860-869).
		const bool has_deleted = a.deleted != nullptr;
		auto is_deleted = [&](uint32_t id) { return has_deleted && ((a.deleted[id >> 5] >> (id & 31)) & 1u); };
		uint32_t size = 0, xsize = 0;
		uint32_t vcount = 0;
		bool x_overflow = false;
		if (lane == 0) {
			if (!is_deleted(cur)) {  // initLayer0SearchState :844-855
				l_dist[0] = curdist;
				l_id[0] = cur;
			} else {
				x_dist[0] = 3.402823466e+38f;
				x_id[0] = cur;
			}
			atomicOr(&visited[cur >> 5], 1u << (cur & 31));
			vlog[0] = cur;
		}
		if (!is_deleted(cur)) {
			size = 1;
		} else {
			xsize = 1;
		}
		vcount = 1;
		__syncwarp();
		for (;;) {
			const int pos = first_unexpanded(l_id, size, lane);
			uint32_t node;
			if (xsize && (pos < 0 || x_dist[0] < l_dist[pos])) {
				// a deleted candidate is the closest one: expanded unless it is worse than a full result list
				if (size >= a.ef && x_dist[0] > l_dist[size - 1]) {
					break;
				}
				node = x_id[0];
				__syncwarp();
				for (uint32_t b = 0; b + 1 < xsize; b += 32) {  // pop the head
					const uint32_t i = b + lane;
					float td = 0.f;
					uint32_t ti = 0;
					if (i + 1 < xsize) {
						td = x_dist[i + 1];
						ti = x_id[i + 1];
					}
					__syncwarp();
					if (i + 1 < xsize) {
						x_dist[i] = td;
						x_id[i] = ti;
					}
					__syncwarp();
				}
				--xsize;
			} else {
				if (pos < 0) {
					break;  // candidate_set exhausted / next candidate worse than lowerBound (layer0ShouldStopBeforePop :860-869)
				}
				node = l_id[pos];
				__syncwarp();
				if (lane == 0) {
					l_id[pos] = node | kExpanded;
				}
			}
			const uint32_t* ll = a.level0 + size_t(node) * a.l0_stride;
			const uint32_t cnt = min(ll[0], uint32_t(kMaxNeighbours));
			n_hops++;
			n_dist += cnt;
			const uint32_t ucnt = gather_fresh(ll, cnt, visited, vlog, vcount, s_ids, lane);
			if (ucnt == 0) {
				continue;
			}
			warp_dists<kIsL2>(a, sq4, s_ids, ucnt, s_d, lane, qcorr, qcoef);
			// sequential accept logic of runLayer0Step (:931-957) over the batch, in neighbour order
			for (uint32_t j = 0; j < ucnt; ++j) {
				const float d = s_d[j];
				const uint32_t nid = s_ids[j];
				const bool consider = size < a.ef || l_dist[size - 1] > d;  // flag_consider_candidate
				if (!consider) {
					continue;
				}
				if (is_deleted(nid)) {  // candidate_set only (:943-953): sorted insert into X
					if (xsize == kHnswXCap) {
						x_overflow = true;
						continue;
					}
					const uint32_t p = warp_count(xsize, lane, [&](uint32_t i) { return x_dist[i] <= d; });
					// list_insert(x_dist, x_id, p, xsize + 1, ...) written out: its `i < xsize + 1` changes the register allocation of
					// the whole kernel
					for (int b = int(xsize / 32) * 32; b >= 0; b -= 32) {
						const uint32_t i = uint32_t(b) + lane;
						const bool mv = i > p && i <= xsize;
						float td = 0.f;
						uint32_t ti = 0;
						if (mv) {
							td = x_dist[i - 1];
							ti = x_id[i - 1];
						}
						__syncwarp();
						if (mv) {
							x_dist[i] = td;
							x_id[i] = ti;
						}
						__syncwarp();
					}
					if (lane == 0) {
						x_dist[p] = d;
						x_id[p] = nid;
					}
					__syncwarp();
					++xsize;
					continue;
				}
				const uint32_t p = warp_count(size, lane, [&](uint32_t i) { return l_dist[i] <= d; });  // insert after every entry <= d
				const uint32_t newsize = min(size + 1, a.ef);
				if (p < newsize) {
					list_insert(l_dist, l_id, p, newsize, d, nid, lane);
				}
				size = newsize;
			}
		}
		if (lane == 0 && a.overflow) {
			a.overflow[qi] = x_overflow ? 1u : 0u;
		}

		// ---- results: the k best of the list (SearchKnn :1998-2011), then clean the visited bitmap for the next query
		const uint32_t outn = min(a.k, size);
		for (uint32_t j = lane; j < outn; j += 32) {
			a.out_dist[size_t(qi) * a.out_stride + j] = l_dist[j];
			a.out_idx[size_t(qi) * a.out_stride + j] = l_id[j] & ~kExpanded;
		}
		if (lane == 0) {
			a.out_count[qi] = outn;
			if (a.stats) {
				a.stats[size_t(qi) * 2] = n_dist;
				a.stats[size_t(qi) * 2 + 1] = n_hops;
			}
		}
		__syncwarp();
		if (vcount <= kVlogCap) {
			for (uint32_t j = lane; j < vcount; j += 32) {
				visited[vlog[j] >> 5] = 0;
			}
		} else {
			for (uint32_t j = lane; j < a.words; j += 32) {
				visited[j] = 0;
			}
		}
		__syncwarp();
	}
}


// ---- SearchRange (hnswalg.h:2015-2070) for a chunk of queries: the ef-search result seeds a breadth-first expansion over level-0
// neighbours with dist < radius.  The closure is independent of the traversal order, so the reference's FIFO queue becomes a
// level-synchronous frontier: each query's result region IS its queue (every accepted node is appended exactly once, guarded by the
// query's own visited bitmap), one warp expands one frontier node, and one launch expands the frontiers of every query of the chunk.
// Slot s of the chunk answers query qmap[s] of the batch with bitmap s of the search kernel's [slots][words] (zero on entry and exit).
struct RangeArgs {
	const float* rows;
	const float* norm_coefs;
	const uint32_t* level0;
	const float* queries;     // [batch][dim]
	const float* radius;      // [batch]
	const uint32_t* qmap;     // [nq] slot -> query of the batch
	uint32_t* visited;        // [nq][words]
	const uint32_t* deleted;  // MarkDelete bitmap or null: deleted neighbours are skipped without being marked (:2053-2055)
	float* reg_dist;          // [nq][cap]
	uint32_t* reg_idx;        // [nq][cap]
	RangeQuery* rq;           // [nq]
	unsigned int* units;      // CTAs of this level's expansion
	const float* seed_dist;   // [batch][kseed] the ef-search's results (:2034-2041)
	const uint32_t* seed_idx;
	const uint32_t* seed_count;
	uint32_t pitch, dim, l0_stride, words, nq, cap, kseed;
};
// one CTA per query: every seed is marked visited, the ones with dist < radius start the queue
__global__ void hnsw_range_seed(const RangeArgs a) {
	const uint32_t s = blockIdx.x, qi = a.qmap[s];
	uint32_t* visited = a.visited + size_t(s) * a.words;
	const float radius = a.radius[qi];
	for (uint32_t j = threadIdx.x; j < a.seed_count[qi]; j += blockDim.x) {
		const uint32_t id = a.seed_idx[size_t(qi) * a.kseed + j];
		const float d = a.seed_dist[size_t(qi) * a.kseed + j];
		atomicOr(&visited[id >> 5], 1u << (id & 31));
		if (d < radius) {
			const unsigned pos = atomicAdd(&a.rq[s].tail, 1u);
			if (pos < a.cap) {
				a.reg_dist[size_t(s) * a.cap + pos] = d;
				a.reg_idx[size_t(s) * a.cap + pos] = id;
			}
		}
	}
}
// one CTA: the next level's frontier of every query is what the last level appended; an overflowed query stops.  Each query gets
// ceil(frontier / kHnswWarps) CTAs of the expansion (one node per warp); *units = their sum, the only value the host reads per level.
__global__ void __launch_bounds__(1024) hnsw_range_advance(const RangeArgs a) {
	__shared__ unsigned int s_warp[32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned int carry = 0;
	for (uint32_t b = 0; b < a.nq; b += 1024) {
		const uint32_t s = b + threadIdx.x;
		unsigned int u = 0;
		if (s < a.nq) {
			RangeQuery& r = a.rq[s];
			r.begin = r.end;
			r.end = r.tail > a.cap ? r.begin : r.tail;
			u = (r.end - r.begin + kHnswWarps - 1) / kHnswWarps;
		}
		unsigned int x = u;  // inclusive scan: warp, then the warp totals
#pragma unroll
		for (int off = 1; off < 32; off <<= 1) {
			const unsigned int y = __shfl_up_sync(0xffffffffu, x, off);
			x += lane >= off ? y : 0u;
		}
		if (lane == 31) {
			s_warp[warp] = x;
		}
		__syncthreads();
		if (warp == 0) {
			unsigned int w = s_warp[lane];
#pragma unroll
			for (int off = 1; off < 32; off <<= 1) {
				const unsigned int y = __shfl_up_sync(0xffffffffu, w, off);
				w += lane >= off ? y : 0u;
			}
			s_warp[lane] = w;
		}
		__syncthreads();
		if (s < a.nq) {
			a.rq[s].unit0 = carry + (warp ? s_warp[warp - 1] : 0u) + x - u;
		}
		carry += s_warp[31];
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		*a.units = carry;
	}
}
// CTA u expands frontier nodes [4j, 4j + 4) of the query whose CTAs hold u (j = u - its unit0), the query staged in shared memory
template <bool kIsL2>
__global__ void __launch_bounds__(kHnswThreads) hnsw_range_expand(const RangeArgs a) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	__shared__ uint32_t s_slot;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t dp4 = hnsw_query_words(a.dim);
	float4* sq4 = reinterpret_cast<float4*>(smem_raw);
	uint32_t* s_ids = reinterpret_cast<uint32_t*>(smem_raw + size_t(dp4) * 16) + warp * 2 * kMaxNeighbours;
	float* s_d = reinterpret_cast<float*>(s_ids + kMaxNeighbours);
	const uint32_t u = blockIdx.x;
	if (threadIdx.x == 0) {  // the last slot whose unit0 <= u (a query without CTAs shares its unit0 with the next one)
		uint32_t lo = 0, hi = a.nq - 1;
		while (lo < hi) {
			const uint32_t mid = (lo + hi + 1) / 2;
			if (a.rq[mid].unit0 <= u) {
				lo = mid;
			} else {
				hi = mid - 1;
			}
		}
		s_slot = lo;
	}
	__syncthreads();
	const uint32_t s = s_slot, qi = a.qmap[s];
	stage_query(sq4, a.queries + size_t(qi) * a.dim, a.dim, dp4, threadIdx.x, blockDim.x);
	__syncthreads();
	const uint32_t f = a.rq[s].begin + (u - a.rq[s].unit0) * kHnswWarps + warp;
	if (f >= a.rq[s].end) {
		return;
	}
	HnswArgs h{};  // warp_dists reads rows / pitch / dim / norm_coefs only
	h.rows = a.rows;
	h.norm_coefs = a.norm_coefs;
	h.pitch = a.pitch;
	h.dim = a.dim;
	const float radius = a.radius[qi];
	uint32_t* visited = a.visited + size_t(s) * a.words;
	float* reg_dist = a.reg_dist + size_t(s) * a.cap;
	uint32_t* reg_idx = a.reg_idx + size_t(s) * a.cap;
	const uint32_t node = reg_idx[f];
	const uint32_t* ll = a.level0 + size_t(node) * a.l0_stride;
	const uint32_t cnt = min(ll[0], uint32_t(kMaxNeighbours));
	uint32_t ucnt = 0;
	for (uint32_t b = 0; b < cnt; b += 32) {
		const uint32_t j = b + lane;
		uint32_t nid = 0;
		bool fresh = false;
		if (j < cnt) {
			nid = ll[1 + j];
			const uint32_t bit = 1u << (nid & 31);
			const bool gone = a.deleted != nullptr && (a.deleted[nid >> 5] & bit);
			fresh = !gone && !(atomicOr(&visited[nid >> 5], bit) & bit);  // exactly one warp of the grid wins a node
		}
		const unsigned fm = __ballot_sync(0xffffffffu, fresh);
		if (fresh) {
			s_ids[ucnt + __popc(fm & ((1u << lane) - 1u))] = nid;
		}
		ucnt += __popc(fm);
	}
	__syncwarp();
	if (ucnt == 0) {
		return;
	}
	warp_dists<kIsL2>(h, sq4, s_ids, ucnt, s_d, lane);
	for (uint32_t b = 0; b < ucnt; b += 32) {
		const uint32_t j = b + lane;
		const bool hit = j < ucnt && s_d[j] < radius;  // strict, :2060
		const unsigned hm = __ballot_sync(0xffffffffu, hit);
		if (hm) {
			unsigned base = 0;
			if (lane == 0) {
				base = atomicAdd(&a.rq[s].tail, unsigned(__popc(hm)));
			}
			base = __shfl_sync(0xffffffffu, base, 0);
			const unsigned pos = base + __popc(hm & ((1u << lane) - 1u));
			if (hit && pos < a.cap) {
				reg_dist[pos] = s_d[j];
				reg_idx[pos] = s_ids[j];
			}
		}
	}
}
// one CTA per query: zero the bitmap again.  Every visited node is a seed or a level-0 neighbour of a match, so the words of those
// suffice -- unless the region lost matches (overflow) or the matches' lists reach more entries than the bitmap has words.
__global__ void __launch_bounds__(kHnswThreads) hnsw_range_clear(const RangeArgs a) {
	const uint32_t s = blockIdx.x, qi = a.qmap[s];
	uint32_t* visited = a.visited + size_t(s) * a.words;
	const unsigned int tail = a.rq[s].tail;
	if (tail > a.cap || uint64_t(tail) * (a.l0_stride - 1) + a.kseed > a.words) {
		for (uint32_t j = threadIdx.x; j < a.words; j += blockDim.x) {
			visited[j] = 0;
		}
		return;
	}
	for (uint32_t j = threadIdx.x; j < a.seed_count[qi]; j += blockDim.x) {
		visited[a.seed_idx[size_t(qi) * a.kseed + j] >> 5] = 0;
	}
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t* reg_idx = a.reg_idx + size_t(s) * a.cap;
	for (uint32_t i = warp; i < tail; i += kHnswWarps) {
		const uint32_t* ll = a.level0 + size_t(reg_idx[i]) * a.l0_stride;
		const uint32_t cnt = min(ll[0], uint32_t(kMaxNeighbours));
		for (uint32_t j = lane; j < cnt; j += 32) {
			visited[ll[1 + j] >> 5] = 0;
		}
	}
}

// ---- streaming (resumable) search: HierarchicalNSWImpl::Begin/ContinueStreamingSearch (hnswalg.h:1864-1975) ------------------------------
// A session keeps, in HBM between calls: the visited bitmap, candidate_set (every visited, not yet expanded node), top_candidates (the
// <= ef closest EXPANDED nodes), top_candidates_extras (expanded nodes pushed out of top_candidates) and lowerBound.  One warp runs a
// ContinueStreamingSearch call: the closest candidates (<= kStreamList keys) and top_candidates live sorted in shared memory for the
// duration of the call; candidates that do not fit wait in an unsorted HBM spill array that is only ever worse than the shared list
// (spill_min guards the invariant; the list is refilled from it when it runs dry), so nodes are expanded in exact (distance, id) order.
constexpr uint32_t kStreamList = 1024;
struct StreamHeader {
	uint32_t initialized, n_top, n_cand, n_spill, n_extra, exhausted, overflow, pad;
	float lower_bound, spill_min;
};
struct StreamArgs {
	HnswArgs h;             // graph / rows (queries, nq, k, out_* unused)
	StreamHeader* hdr;
	uint64_t* top;          // [kMaxEf]
	uint64_t* cand;         // [kStreamList]
	uint64_t* spill;        // [cap]
	uint64_t* extras;       // [cap]
	uint32_t* visited;      // [words]
	uint32_t cap, ef, batch;
	float* out_dist;        // [batch]
	uint32_t* out_idx;
	uint32_t* out_count;    // [0] results, [1] exhausted
};
__device__ __forceinline__ uint64_t stream_key(float d, uint32_t id) { return (uint64_t(float_ord(d)) << 32) | id; }
__device__ __forceinline__ float stream_dist(uint64_t k) { return ord_float(uint32_t(k >> 32)); }
// sorted insert into list[0, n) (ascending); returns the new size.  When the list is full (n == cap) the largest key falls out and
// is returned through *evicted (kKeyNone otherwise); a key larger than every entry of a full list is itself the one that falls out.
__device__ __forceinline__ uint32_t stream_insert(uint64_t* list, uint32_t n, uint32_t cap, uint64_t key, uint64_t* evicted, int lane) {
	*evicted = kKeyNone;
	if (n == cap) {
		if (key >= list[n - 1]) {
			*evicted = key;
			return n;
		}
		*evicted = list[n - 1];
		n -= 1;
	}
	const uint32_t pos = warp_count(n, lane, [&](uint32_t i) { return list[i] < key; });  // entries smaller than key
	for (int b = int((n - pos + 31) / 32) - 1; b >= 0; --b) {  // shift [pos, n) up by one, highest block first
		const uint32_t i = pos + uint32_t(b) * 32 + lane;
		const uint64_t v = i < n ? list[i] : 0;
		__syncwarp();
		if (i < n) {
			list[i + 1] = v;
		}
		__syncwarp();
	}
	if (lane == 0) {
		list[pos] = key;
	}
	__syncwarp();
	return n + 1;
}
// index of the smallest key of arr[0, n) (n > 0), warp-wide
__device__ __forceinline__ uint32_t stream_argmin(const uint64_t* arr, uint32_t n, uint64_t* best_out, int lane) {
	uint64_t best = kKeyNone;
	uint32_t bpos = 0;
	for (uint32_t i = lane; i < n; i += 32) {
		const uint64_t k = arr[i];
		if (k < best) {
			best = k;
			bpos = i;
		}
	}
#pragma unroll
	for (int off = 16; off > 0; off >>= 1) {
		const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
		const uint32_t op = __shfl_xor_sync(0xffffffffu, bpos, off);
		if (ok < best) {
			best = ok;
			bpos = op;
		}
	}
	*best_out = best;
	return bpos;
}

template <bool kIsL2>
__global__ void __launch_bounds__(32) hnsw_stream_kernel(const StreamArgs s) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const HnswArgs& a = s.h;
	const int lane = threadIdx.x;
	const uint32_t dp4 = hnsw_query_words(a.dim);
	float4* sq4 = reinterpret_cast<float4*>(smem_raw);
	uint64_t* l_top = reinterpret_cast<uint64_t*>(smem_raw + size_t(dp4) * 16);
	uint64_t* l_cand = l_top + kMaxEf;
	uint32_t* s_ids = reinterpret_cast<uint32_t*>(l_cand + kStreamList);
	float* s_d = reinterpret_cast<float*>(s_ids + kMaxNeighbours);
	StreamHeader hd = *s.hdr;
	stage_query(sq4, a.queries, a.dim, dp4, lane, 32);
	for (uint32_t i = lane; i < hd.n_top; i += 32) {
		l_top[i] = s.top[i];
	}
	for (uint32_t i = lane; i < hd.n_cand; i += 32) {
		l_cand[i] = s.cand[i];
	}
	__syncwarp();
	const bool has_deleted = a.deleted != nullptr;
	auto is_deleted = [&](uint32_t id) { return has_deleted && ((a.deleted[id >> 5] >> (id & 31)) & 1u); };
	uint32_t n_top = hd.n_top, n_cand = hd.n_cand, n_spill = hd.n_spill, n_extra = hd.n_extra;
	float lower = hd.lower_bound, spill_min = hd.spill_min;
	bool overflow = hd.overflow != 0;
	uint64_t ev;
	if (!hd.initialized) {
		// getLayer0EntryPoint (hnswalg.h:799-827) + initLayer0SearchState in streaming mode (:829-858): the entry point is a candidate only
		uint32_t cur = a.enterpoint;
		if (lane == 0) {
			s_ids[0] = cur;
		}
		__syncwarp();
		warp_dists<kIsL2>(a, sq4, s_ids, 1, s_d, lane);
		float curdist = s_d[0];
		__syncwarp();
		uint32_t n_dist = 0, n_hops = 0;  // not reported by the streaming search
		greedy_descent<kIsL2>(a, sq4, cur, curdist, a.maxlevel, 0, s_ids, s_d, lane, n_dist, n_hops);
		const bool epDeleted = is_deleted(cur);
		lower = epDeleted ? 3.402823466e+38f : curdist;
		if (lane == 0) {
			l_cand[0] = stream_key(lower, cur);
			atomicOr(&s.visited[cur >> 5], 1u << (cur & 31));
		}
		n_cand = 1;
		spill_min = INFINITY;
		__syncwarp();
	}
	const uint32_t ef = max(s.ef, s.batch);  // ContinueStreamingSearch: state.ef = max(state.ef, batchSize)
	// mergeExtrasIntoTopCandidates (:1894-1925): the best extras refill top_candidates up to ef
	while (n_top < ef && n_extra > 0) {
		uint64_t best;
		const uint32_t pos = stream_argmin(s.extras, n_extra, &best, lane);
		if (lane == 0) {
			s.extras[pos] = s.extras[n_extra - 1];
		}
		n_extra -= 1;
		__syncwarp();
		n_top = stream_insert(l_top, n_top, kMaxEf, best, &ev, lane);
		lower = stream_dist(l_top[n_top - 1]);
	}
	for (;;) {
		if (n_cand == 0 && n_spill > 0) {  // refill the shared list with the closest spilled candidates
			while (n_cand < kStreamList / 2 && n_spill > 0) {
				uint64_t best;
				const uint32_t pos = stream_argmin(s.spill, n_spill, &best, lane);
				if (lane == 0) {
					s.spill[pos] = s.spill[n_spill - 1];
				}
				n_spill -= 1;
				__syncwarp();
				n_cand = stream_insert(l_cand, n_cand, kStreamList, best, &ev, lane);
			}
			spill_min = INFINITY;
			if (n_spill) {
				uint64_t best;
				stream_argmin(s.spill, n_spill, &best, lane);
				spill_min = stream_dist(best);
			}
		}
		if (n_cand == 0) {
			break;  // candidate_set.empty() (layer0ShouldStopBeforePop :861-863)
		}
		const uint64_t ck = l_cand[0];
		const float cdist = stream_dist(ck);
		const uint32_t cid = uint32_t(ck);
		if (cdist > lower && n_top >= ef) {
			break;  // :868
		}
		// pop the closest candidate
		for (uint32_t b = 0; b + 1 < n_cand; b += 32) {
			const uint32_t i = b + lane;
			const uint64_t v = i + 1 < n_cand ? l_cand[i + 1] : 0;
			__syncwarp();
			if (i + 1 < n_cand) {
				l_cand[i] = v;
			}
			__syncwarp();
		}
		n_cand -= 1;
		// runLayer0Step, streaming branch (:880-893): an expanded live node enters top_candidates (or pushes its worst entry to extras)
		if (!is_deleted(cid)) {
			if (n_top < ef) {
				n_top = stream_insert(l_top, n_top, kMaxEf, ck, &ev, lane);
			} else if (lower > cdist) {
				const uint64_t worst = l_top[n_top - 1];
				__syncwarp();
				n_top = stream_insert(l_top, n_top - 1, kMaxEf, ck, &ev, lane);
				if (n_extra < s.cap) {
					if (lane == 0) {
						s.extras[n_extra] = worst;
					}
					n_extra += 1;
				} else {
					overflow = true;
				}
			}
			lower = stream_dist(l_top[n_top - 1]);
		}
		// expand: every unvisited neighbour becomes a candidate (:931-938)
		const uint32_t* ll = a.level0 + size_t(cid) * a.l0_stride;
		const uint32_t cnt = min(ll[0], uint32_t(kMaxNeighbours));
		uint32_t ucnt = 0;
		for (uint32_t b = 0; b < cnt; b += 32) {
			const uint32_t j = b + lane;
			uint32_t nid = 0;
			bool fresh = false;
			if (j < cnt) {
				nid = ll[1 + j];
				const uint32_t bit = 1u << (nid & 31);
				fresh = !(s.visited[nid >> 5] & bit);
			}
			// two neighbours may share a bitmap word: set the bits after the ballot, one lane per word is not needed for correctness of
			// `fresh` because a list holds every neighbour once
			if (fresh) {
				atomicOr(&s.visited[nid >> 5], 1u << (nid & 31));
			}
			const unsigned fm = __ballot_sync(0xffffffffu, fresh);
			if (fresh) {
				s_ids[ucnt + __popc(fm & ((1u << lane) - 1u))] = nid;
			}
			ucnt += __popc(fm);
		}
		__syncwarp();
		if (ucnt) {
			warp_dists<kIsL2>(a, sq4, s_ids, ucnt, s_d, lane);
			for (uint32_t j = 0; j < ucnt; ++j) {
				const float d = s_d[j];
				const uint64_t key = stream_key(d, s_ids[j]);
				if (d < spill_min) {
					n_cand = stream_insert(l_cand, n_cand, kStreamList, key, &ev, lane);
				} else {
					ev = key;
				}
				if (ev != kKeyNone) {  // does not fit the shared list: it is worse than everything in it
					if (n_spill < s.cap) {
						if (lane == 0) {
							s.spill[n_spill] = ev;
						}
						n_spill += 1;
						spill_min = fminf(spill_min, stream_dist(ev));
					} else {
						overflow = true;
					}
				}
			}
		}
		__syncwarp();
	}
	// emitStreamingBatch (:1927-1945): the `batch` closest entries of top_candidates leave it
	const uint32_t nout = min(s.batch, n_top);
	for (uint32_t i = lane; i < nout; i += 32) {
		s.out_dist[i] = stream_dist(l_top[i]);
		s.out_idx[i] = uint32_t(l_top[i]);
	}
	__syncwarp();
	for (uint32_t b = 0; b < n_top - nout; b += 32) {
		const uint32_t i = b + lane;
		const uint64_t v = i < n_top - nout ? l_top[i + nout] : 0;
		__syncwarp();
		if (i < n_top - nout) {
			l_top[i] = v;
		}
		__syncwarp();
	}
	n_top -= nout;
	for (uint32_t i = lane; i < n_top; i += 32) {
		s.top[i] = l_top[i];
	}
	for (uint32_t i = lane; i < n_cand; i += 32) {
		s.cand[i] = l_cand[i];
	}
	if (lane == 0) {
		StreamHeader o{};
		o.initialized = 1;
		o.n_top = n_top;
		o.n_cand = n_cand;
		o.n_spill = n_spill;
		o.n_extra = n_extra;
		o.exhausted = (n_cand == 0 && n_spill == 0 && n_top == 0 && n_extra == 0) ? 1u : 0u;  // :1972
		o.overflow = overflow ? 1u : 0u;
		o.lower_bound = lower;
		o.spill_min = spill_min;
		*s.hdr = o;
		s.out_count[0] = nout;
		s.out_count[1] = o.exhausted;
		s.out_count[2] = o.overflow;
	}
}

__global__ void gather_labels_kernel(const uint64_t* labels, uint64_t size, uint64_t n, const uint32_t* idx, uint64_t* out) {
	const uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
	if (i < n) {
		out[i] = idx[i] < size ? labels[idx[i]] : ~0ull;
	}
}

}  // namespace

namespace rxgpu {
void hnswRelease(rxgpu_hnsw_device* h) { delete h; }

int checkGraph(const rxgpu_index* ix) {
	const rxgpu_hnsw_device* h = ix->hnsw;
	if (!h) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no HNSW graph imported into this index");
	}
	if (h->n != ix->size || h->index_version != ix->version) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the index changed after the HNSW graph was imported");
	}
	return 0;
}

int allocGraph(const rxgpu_index* ix, rxgpu_hnsw_device* h, size_t capNodes, size_t upperEntries) {
	const size_t s0 = 1 + size_t(h->maxM0), s1 = 1 + size_t(h->M);
	RX_CUDA(h->level0.ensure(capNodes * s0));
	RX_CUDA(h->levels.ensure(capNodes));
	RX_CUDA(h->upper_off.ensure(capNodes + 1));
	RX_CUDA(h->upper.ensure(upperEntries + (capNodes - ix->size) / 8 * s1 + 64 * s1));
	h->cap_nodes = capNodes;
	h->slots = hnswSlots(ix);
	h->words = uint32_t((capNodes + 31) / 32);
	RX_CUDA(h->visited.ensure(size_t(h->slots) * h->words));
	RX_CUDA(h->vlog.ensure(size_t(h->slots) * kVlogCap));
	RX_CUDA(h->counter.ensure(1));
	RX_CUDA(h->deleted.ensure(h->words));
	RX_CUDA(cudaMemsetAsync(h->visited.p, 0, size_t(h->slots) * h->words * 4, ix->stream));
	RX_CUDA(cudaMemsetAsync(h->deleted.p, 0, size_t(h->words) * 4, ix->stream));
	h->h_deleted.assign(h->words, 0u);
	return 0;
}
}  // namespace rxgpu

extern "C" {

int rxgpu_hnsw_import(rxgpu_index* ix, const rxgpu_hnsw_graph* g) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!g || !g->level0 || !g->levels || !g->upper_offsets) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null graph");
	}
	if (g->n != ix->size) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: HNSW graph size differs from the number of rows in the index");
	}
	if (g->maxM0 > uint32_t(kMaxNeighbours) || g->M > uint32_t(kMaxNeighbours) || g->n == 0 || g->enterpoint >= g->n) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: unsupported HNSW graph (M and maxM0 must be <= 64, graph must be non-empty)");
	}
	if (g->upper_slots && !g->upper) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null graph");
	}
	{  // one host pass over the lists: the search kernel indexes rows, the visited bitmap and the upper-level slab with these values
		const size_t s0 = size_t(1) + g->maxM0;
		for (uint32_t i = 0; i < g->n; ++i) {
			const uint32_t* l = g->level0 + size_t(i) * s0;
			if (l[0] > g->maxM0) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: level-0 neighbour count of node " + std::to_string(i) + " exceeds maxM0");
			}
			for (uint32_t j = 1; j <= l[0]; ++j) {
				if (l[j] >= g->n) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: level-0 neighbour id of node " + std::to_string(i) + " is out of range");
				}
			}
		}
		if (g->upper_offsets[0] < 0 || uint64_t(g->upper_offsets[g->n]) > g->upper_slots) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: upper_offsets do not fit upper_slots");
		}
		for (uint32_t i = 0; i < g->n; ++i) {
			const int64_t span = g->upper_offsets[i + 1] - g->upper_offsets[i];
			if (g->levels[i] < 0 || g->levels[i] > g->maxlevel || span < 0 || span < int64_t(g->levels[i])) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: levels / upper_offsets of node " + std::to_string(i) + " are inconsistent");
			}
		}
		if (g->levels[g->enterpoint] != g->maxlevel) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: the enter point is not on the top level");
		}
		const size_t s1 = size_t(1) + g->M;
		for (uint64_t sl = 0; sl < g->upper_slots; ++sl) {
			const uint32_t* l = g->upper + sl * s1;
			if (l[0] > g->M) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: an upper-level neighbour count exceeds M");
			}
			for (uint32_t j = 1; j <= l[0]; ++j) {
				if (l[j] >= g->n) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW graph: an upper-level neighbour id is out of range");
				}
			}
		}
	}
	auto h = std::make_unique<rxgpu_hnsw_device>();
	h->n = g->n;
	h->M = g->M;
	h->maxM0 = g->maxM0;
	h->maxlevel = g->maxlevel;
	h->enterpoint = g->enterpoint;
	// sized for the index's capacity so that rxgpu_hnsw_update can append nodes without reallocating
	const size_t capNodes = std::max<size_t>(ix->capacity, g->n);
	if (int rc = allocGraph(ix, h.get(), capNodes, std::max<size_t>(1, size_t(g->upper_slots) * (1 + g->M)))) {
		return rc;
	}
	h->upper_slots = g->upper_slots;
	h->h_upper_off.assign(g->upper_offsets, g->upper_offsets + g->n);
	h->h_levels.assign(g->levels, g->levels + g->n);
	// every upload goes through the index's stream, which is non-blocking: a plain cudaMemcpy runs on the legacy stream, is not
	// ordered before the search kernels and may return before a pageable copy has landed
	cudaStream_t st = ix->stream;
	RX_CUDA(cudaMemcpyAsync(h->level0.p, g->level0, size_t(g->n) * (1 + g->maxM0) * 4, cudaMemcpyHostToDevice, st));
	RX_CUDA(cudaMemcpyAsync(h->levels.p, g->levels, size_t(g->n) * 4, cudaMemcpyHostToDevice, st));
	RX_CUDA(cudaMemcpyAsync(h->upper_off.p, g->upper_offsets, (size_t(g->n) + 1) * 8, cudaMemcpyHostToDevice, st));
	if (g->upper_slots) {
		RX_CUDA(cudaMemcpyAsync(h->upper.p, g->upper, size_t(g->upper_slots) * (1 + g->M) * 4, cudaMemcpyHostToDevice, st));
	}
	RX_CUDA(cudaStreamSynchronize(st));  // the caller's graph arrays may go away after the return
	h->index_version = ix->version;
	if (ix->hnsw) {
		hnswRelease(ix->hnsw);
	}
	ix->hnsw = h.release();
	ix->rows_touched_from = ~0ull;
	return 0;
}

}  // extern "C"

namespace {
struct Sq8Query {  // device pointers of the quantised query batch (rxgpu_hnsw_search_knn_sq8)
	const uint8_t* qcodes;
	const float* qcorr;
	const float* qcoef;
};
int hnswSearchDevice(const rxgpu_index* ix, uint32_t nq, const float* d_queries, uint32_t k, uint32_t ef, float* d_out_dist, uint32_t* d_out_idx,
					 uint32_t* d_out_count, uint32_t* d_stats, void* stream, const Sq8Query* sq) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (int rc = checkGraph(ix)) {
		return rc;
	}
	rxgpu_hnsw_device* h = ix->hnsw;
	if (nq == 0) {
		return 0;
	}
	const uint32_t outStride = k;  // the caller's buffers are [nq][k]; only the number of entries written is clamped
	k = uint32_t(std::min<uint64_t>(k, ix->size));  // hnswalg.h:1993
	if (k == 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be positive");
	}
	ef = ef ? ef : k * 3 / 2;  // hnswalg.h:1995
	ef = std::max(ef, 1u);
	if (ef > kMaxEf) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: ef must be <= 1024 on the device path");
	}
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
	std::lock_guard<std::mutex> lck(h->mtx);
	HnswArgs a = graphArgs(ix, h);
	a.queries = d_queries;
	a.visited = h->visited.p;
	a.vlog = h->vlog.p;
	a.next_query = h->counter.p;
	a.out_dist = d_out_dist;
	a.out_idx = d_out_idx;
	a.out_count = d_out_count;
	a.stats = d_stats;
	if (h->num_deleted) {
		RX_CUDA(h->overflow.ensure(nq));
		RX_CUDA(h->x_dist.ensure(size_t(h->slots) * kHnswXCap));
		RX_CUDA(h->x_id.ensure(size_t(h->slots) * kHnswXCap));
		a.overflow = h->overflow.p;
		a.x_dist = h->x_dist.p;
		a.x_id = h->x_id.p;
	}
	a.nq = nq;
	a.k = k;
	a.out_stride = outStride;
	a.ef = ef;
	if (sq) {
		const rxgpu_sq8_device* s8 = ix->sq8;
		if (!s8 || s8->index_version != ix->version || s8->n != h->n) {
			return fail(RXGPU_ERR_LOGIC, "rxgpu: no SQ8 codes attached to this index (or the index changed since)");
		}
		a.codes = s8->codes.p;
		a.corr = s8->corr.p;
		a.code_pitch = s8->code_pitch;
		a.alpha2 = s8->params.alpha_2;
		a.qcodes = sq->qcodes;
		a.qcorr = sq->qcorr;
		a.qcoef = sq->qcoef;
	}
	const size_t smem = (size_t(hnsw_query_words(ix->dim)) * 16 + size_t((ef + 3u) & ~3u) * 8 + kMaxNeighbours * 8) * kHnswWarps;
	if (smem > 200 * 1024) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: dimension/ef combination exceeds the shared-memory budget of the HNSW kernel");
	}
	const unsigned grid = std::min<unsigned>(h->slots / kHnswWarps, (nq + kHnswWarps - 1) / kHnswWarps);
	RX_CUDA(cudaMemsetAsync(h->counter.p, 0, sizeof(unsigned int), st));
	if (ix->metric == RXGPU_L2) {
		RX_CUDA(raiseSmemCeilingOnce(hnsw_search_kernel<true>, ix->device, 200 * 1024));
		hnsw_search_kernel<true><<<grid, kHnswThreads, smem, st>>>(a);
	} else {
		RX_CUDA(raiseSmemCeilingOnce(hnsw_search_kernel<false>, ix->device, 200 * 1024));
		hnsw_search_kernel<false><<<grid, kHnswThreads, smem, st>>>(a);
	}
	RX_CUDA(cudaGetLastError());
	RX_CUDA(cudaStreamSynchronize(st));
	g_stats = rxgpu_search_stats{};
	g_stats.launches = 1;
	if (h->num_deleted) {  // a query that met more deleted nodes than the device keeps track of cannot be trusted
		std::vector<uint32_t> flags(nq);
		RX_CUDA(cudaMemcpy(flags.data(), h->overflow.p, size_t(nq) * 4, cudaMemcpyDeviceToHost));
		for (uint32_t q = 0; q < nq; ++q) {
			if (flags[q]) {
				return fail(RXGPU_ERR_LOGIC, "rxgpu: too many deleted nodes around query " + std::to_string(q) +
												 " for the device search (more than 4096 waiting at once); rebuild the graph or search on the CPU map");
			}
		}
	}
	return 0;
}

// the host-pointer entry points' read-back: a finished device search's [nq][kEff] results d_dist / d_idx / d_count / d_stats to
// out_* as [nq][k], labels for rows
int readKnnResults(const rxgpu_index* ix, uint32_t nq, uint32_t k, uint32_t kEff, const float* d_dist, const uint32_t* d_idx,
				   const uint32_t* d_count, const uint32_t* d_stats, float* out_dist, uint64_t* out_label, uint32_t* out_count, uint32_t* stats) {
	std::vector<float> hd(size_t(nq) * kEff);
	std::vector<uint32_t> hi(size_t(nq) * kEff), hc(nq);
	RX_CUDA(cudaMemcpy(hd.data(), d_dist, hd.size() * 4, cudaMemcpyDeviceToHost));
	RX_CUDA(cudaMemcpy(hi.data(), d_idx, hi.size() * 4, cudaMemcpyDeviceToHost));
	RX_CUDA(cudaMemcpy(hc.data(), d_count, hc.size() * 4, cudaMemcpyDeviceToHost));
	if (stats) {
		RX_CUDA(cudaMemcpy(stats, d_stats, size_t(nq) * 2 * 4, cudaMemcpyDeviceToHost));
	}
	std::vector<Hit> hits;
	for (uint32_t q = 0; q < nq; ++q) {
		hits.clear();
		for (uint32_t j = 0; j < hc[q]; ++j) {
			const uint32_t row = hi[size_t(q) * kEff + j];
			hits.push_back(Hit{hd[size_t(q) * kEff + j], row, ix->h_labels[row]});
		}
		orderTiesByLabel(hits);  // the final SearchResultQueue uses std::less<pair> (hnswalg.h:2003-2010)
		for (size_t j = 0; j < hits.size(); ++j) {
			out_dist[size_t(q) * k + j] = hits[j].dist;
			out_label[size_t(q) * k + j] = hits[j].label;
		}
		out_count[q] = uint32_t(hits.size());
	}
	return 0;
}
}  // namespace

extern "C" {

int rxgpu_hnsw_search_knn_device(const rxgpu_index* ix, uint32_t nq, const float* d_queries, uint32_t k, uint32_t ef, float* d_out_dist,
								 uint32_t* d_out_idx, uint32_t* d_out_count, uint32_t* d_stats, void* stream) {
	return hnswSearchDevice(ix, nq, d_queries, k, ef, d_out_dist, d_out_idx, d_out_count, d_stats, stream, nullptr);
}

// HierarchicalNSWImpl<uint8_t>::SearchKnn: the queries are quantised on the host exactly like prepareData does (hnswalg.h:510-535),
// the kernel gathers codes + corrective offsets instead of fp32 rows
int rxgpu_hnsw_search_knn_sq8(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* query_norms, uint32_t k, uint32_t ef,
							  float* out_dist, uint64_t* out_label, uint32_t* out_count, uint32_t* stats) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (nq == 0) {
		return 0;
	}
	if (!queries || !out_dist || !out_label || !out_count) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	rxgpu_sq8_device* s8 = ix->sq8;
	if (!ix->hnsw || !s8) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the quantised HNSW search needs an imported graph and attached SQ8 codes");
	}
	if (ix->metric == RXGPU_COS && !query_norms) {
		return fail(RXGPU_ERR_PARAMS, "Norm is required for Cosine-metric during corrective offsets calculation in quantized graph");  // hnswalg.h:1857
	}
	if (ix->size == 0) {
		std::memset(out_count, 0, nq * sizeof(uint32_t));
		return 0;
	}
	const uint32_t kEff = uint32_t(std::min<uint64_t>(k, ix->size));
	if (kEff == 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be positive");
	}
	try {
		const uint32_t cp = s8->code_pitch;
		std::vector<uint8_t> hq(size_t(nq) * cp, 0);
		std::vector<float> hcorr(nq), hcoef(nq, 1.f);
		for (uint32_t q = 0; q < nq; ++q) {
			const float coef = ix->metric == RXGPU_COS ? 1.f / query_norms[q] : 1.f;  // queryNormCoef, hnswalg.h:1854-1863
			hcoef[q] = coef;
			hcorr[q] = sq8QuantizeHost(s8, ix->metric, ix->dim, queries + size_t(q) * ix->dim, ix->metric == RXGPU_COS ? 1.f / coef : 1.f,
									   hq.data() + size_t(q) * cp);
		}
		std::lock_guard<std::mutex> hostLock(ix->hnsw->host_mtx);
		std::lock_guard<std::mutex> sqLock(s8->mtx);
		DevBuf<float>& dd = ix->hnsw->h_d;
		DevBuf<uint32_t>&di = ix->hnsw->h_i, &dc = ix->hnsw->h_c, &ds = ix->hnsw->h_s;
		RX_CUDA(s8->d_q.ensure(hq.size()));
		RX_CUDA(s8->d_qcorr.ensure(nq));
		RX_CUDA(s8->d_qcoef.ensure(nq));
		RX_CUDA(dd.ensure(size_t(nq) * kEff));
		RX_CUDA(di.ensure(size_t(nq) * kEff));
		RX_CUDA(dc.ensure(nq));
		RX_CUDA(ds.ensure(size_t(nq) * 2));
		// on the stream the search runs on (hnswSearchDevice synchronises it before returning, so the host vectors outlive the copies)
		RX_CUDA(cudaMemcpyAsync(s8->d_q.p, hq.data(), hq.size(), cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaMemcpyAsync(s8->d_qcorr.p, hcorr.data(), size_t(nq) * 4, cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaMemcpyAsync(s8->d_qcoef.p, hcoef.data(), size_t(nq) * 4, cudaMemcpyHostToDevice, ix->stream));
		const Sq8Query sq{s8->d_q.p, s8->d_qcorr.p, s8->d_qcoef.p};
		if (int rc = hnswSearchDevice(ix, nq, nullptr, kEff, ef, dd.p, di.p, dc.p, ds.p, nullptr, &sq)) {
			return rc;
		}
		return readKnnResults(ix, nq, k, kEff, dd.p, di.p, dc.p, ds.p, out_dist, out_label, out_count, stats);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_hnsw_search_knn(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, uint32_t ef, float* out_dist,
						  uint64_t* out_label, uint32_t* out_count, uint32_t* stats) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (nq == 0) {
		return 0;
	}
	if (!queries || !out_dist || !out_label || !out_count) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (ix->size == 0) {  // hnswalg.h:1989-1991
		std::memset(out_count, 0, nq * sizeof(uint32_t));
		return 0;
	}
	const uint32_t kEff = uint32_t(std::min<uint64_t>(k, ix->size));
	if (kEff == 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be positive");
	}
	if (!ix->hnsw) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no HNSW graph imported into this index");
	}
	std::lock_guard<std::mutex> hostLock(ix->hnsw->host_mtx);
	DevBuf<float>&dq = ix->hnsw->h_q, &dd = ix->hnsw->h_d;
	DevBuf<uint32_t>&di = ix->hnsw->h_i, &dc = ix->hnsw->h_c, &ds = ix->hnsw->h_s;
	RX_CUDA(dq.ensure(size_t(nq) * ix->dim));
	RX_CUDA(dd.ensure(size_t(nq) * kEff));
	RX_CUDA(di.ensure(size_t(nq) * kEff));
	RX_CUDA(dc.ensure(nq));
	RX_CUDA(ds.ensure(size_t(nq) * 2));
	RX_CUDA(cudaMemcpyAsync(dq.p, queries, size_t(nq) * ix->dim * 4, cudaMemcpyHostToDevice, ix->stream));  // ordered before the search
	if (int rc = rxgpu_hnsw_search_knn_device(ix, nq, dq.p, kEff, ef, dd.p, di.p, dc.p, ds.p, nullptr)) {
		return rc;
	}
	return readKnnResults(ix, nq, k, kEff, dd.p, di.p, dc.p, ds.p, out_dist, out_label, out_count, stats);
}

}  // extern "C"

namespace {
constexpr uint64_t kRangeChunkEntries = uint64_t(1) << 27;  // region entries of one chunk: 1 GiB of (dist, idx)

// SearchRange for nq host queries: one ef-search for the whole batch, then the closures of at most h->slots queries at a time, all
// under h->mtx.  bounded: regions of min(n, max(4096, 2 * min(max_out, 2^17))) entries, and a query that finds more matches is
// answered again with a region of n entries (tc_fallbacks); otherwise every region holds n entries and nothing overflows.  Either
// way a query's answer is its closure, so the two give the same bits.  Row q of out_* gets query q's best min(out_n[q], max_out)
// matches; a non-empty index with an imported graph.
int hnswRangeBatch(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint32_t ef, uint64_t max_out, bool bounded,
				   float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	rxgpu_hnsw_device* h = ix->hnsw;
	ef = std::max(ef, 1u);
	const uint32_t kSeed = uint32_t(std::min<uint64_t>(ef, ix->size));
	std::lock_guard<std::mutex> hostLock(h->host_mtx);
	DevBuf<float>&dq = h->h_q, &dd = h->h_d;
	DevBuf<uint32_t>&di = h->h_i, &dc = h->h_c;
	RX_CUDA(dq.ensure(size_t(nq) * ix->dim));
	RX_CUDA(dd.ensure(size_t(nq) * kSeed));
	RX_CUDA(di.ensure(size_t(nq) * kSeed));
	RX_CUDA(dc.ensure(nq));
	RX_CUDA(cudaMemcpyAsync(dq.p, queries, size_t(nq) * ix->dim * 4, cudaMemcpyHostToDevice, ix->stream));  // ordered before the search
	// search(): the whole top_candidates heap of the ef-search = its ef best nodes (SearchKnn with k = ef on the same routine)
	if (int rc = rxgpu_hnsw_search_knn_device(ix, nq, dq.p, kSeed, ef, dd.p, di.p, dc.p, nullptr, nullptr)) {
		return rc;
	}
	cudaStream_t st = ix->stream;
	std::lock_guard<std::mutex> lck(h->mtx);
	rxgpu_search_stats stats{};
	stats.launches = 1;
	RX_CUDA(h->rg_radius.ensure(nq));
	RX_CUDA(h->rg_units.ensure(1));
	RX_CUDA(cudaMemcpyAsync(h->rg_radius.p, radius, size_t(nq) * 4, cudaMemcpyHostToDevice, st));
	RangeArgs a{};
	a.rows = ix->d_rows;
	a.norm_coefs = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	a.level0 = h->level0.p;
	a.queries = dq.p;
	a.radius = h->rg_radius.p;
	a.visited = h->visited.p;
	a.deleted = h->num_deleted ? h->deleted.p : nullptr;
	a.units = h->rg_units.p;
	a.seed_dist = dd.p;
	a.seed_idx = di.p;
	a.seed_count = dc.p;
	a.pitch = ix->pitch;
	a.dim = ix->dim;
	a.l0_stride = 1 + h->maxM0;
	a.words = h->words;
	a.kseed = kSeed;
	const size_t smem = size_t(hnsw_query_words(ix->dim)) * 16 + size_t(kHnswWarps) * kMaxNeighbours * 8;
	if (ix->metric == RXGPU_L2) {
		RX_CUDA(raiseSmemCeilingOnce(hnsw_range_expand<true>, ix->device, 100 * 1024));
	} else {
		RX_CUDA(raiseSmemCeilingOnce(hnsw_range_expand<false>, ix->device, 100 * 1024));
	}
	uint32_t cap = bounded ? uint32_t(std::min<uint64_t>(h->n, std::max<uint64_t>(4096u, 2 * std::min<uint64_t>(max_out, 1u << 17)))) : h->n;
	std::vector<uint32_t> pending(nq), overflowed;
	for (uint32_t q = 0; q < nq; ++q) {
		pending[q] = q;
	}
	std::vector<RangeQuery> state;
	std::vector<float> hd;
	std::vector<uint32_t> hi;
	std::vector<Hit> hits;
	while (!pending.empty()) {
		const uint32_t chunk = uint32_t(std::min<uint64_t>(h->slots, std::max<uint64_t>(1, kRangeChunkEntries / cap)));
		for (size_t c0 = 0; c0 < pending.size(); c0 += chunk) {
			const uint32_t m = uint32_t(std::min<size_t>(chunk, pending.size() - c0));
			RX_CUDA(h->rg_qmap.ensure(m));
			RX_CUDA(h->rg_state.ensure(m));
			RX_CUDA(h->rg_dist.ensure(size_t(m) * cap));
			RX_CUDA(h->rg_idx.ensure(size_t(m) * cap));
			RX_CUDA(cudaMemcpyAsync(h->rg_qmap.p, pending.data() + c0, size_t(m) * 4, cudaMemcpyHostToDevice, st));
			RX_CUDA(cudaMemsetAsync(h->rg_state.p, 0, size_t(m) * sizeof(RangeQuery), st));
			a.qmap = h->rg_qmap.p;
			a.rq = h->rg_state.p;
			a.reg_dist = h->rg_dist.p;
			a.reg_idx = h->rg_idx.p;
			a.nq = m;
			a.cap = cap;
			hnsw_range_seed<<<m, 256, 0, st>>>(a);
			RX_CUDA(cudaGetLastError());
			stats.launches += 1;
			for (;;) {  // one expansion per BFS level for the whole chunk; the host reads one word per level
				hnsw_range_advance<<<1, 1024, 0, st>>>(a);
				RX_CUDA(cudaGetLastError());
				stats.launches += 1;
				unsigned int units = 0;
				RX_CUDA(cudaMemcpyAsync(&units, h->rg_units.p, 4, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaStreamSynchronize(st));
				if (units == 0) {
					break;
				}
				if (ix->metric == RXGPU_L2) {
					hnsw_range_expand<true><<<units, kHnswThreads, smem, st>>>(a);
				} else {
					hnsw_range_expand<false><<<units, kHnswThreads, smem, st>>>(a);
				}
				RX_CUDA(cudaGetLastError());
				stats.launches += 1;
				stats.passes += 1;
			}
			hnsw_range_clear<<<m, kHnswThreads, 0, st>>>(a);
			RX_CUDA(cudaGetLastError());
			stats.launches += 1;
			state.resize(m);
			RX_CUDA(cudaMemcpyAsync(state.data(), h->rg_state.p, size_t(m) * sizeof(RangeQuery), cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			// one 2-D copy of the first `width` entries of every region: as many as the largest answer that fit
			uint32_t width = 0;
			for (uint32_t s = 0; s < m; ++s) {
				if (state[s].tail <= cap) {
					width = std::max(width, state[s].tail);
				}
			}
			if (width) {
				hd.resize(size_t(m) * width);
				hi.resize(size_t(m) * width);
				RX_CUDA(cudaMemcpy2DAsync(hd.data(), size_t(width) * 4, h->rg_dist.p, size_t(cap) * 4, size_t(width) * 4, m, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaMemcpy2DAsync(hi.data(), size_t(width) * 4, h->rg_idx.p, size_t(cap) * 4, size_t(width) * 4, m, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaStreamSynchronize(st));
			}
			for (uint32_t s = 0; s < m; ++s) {
				const uint32_t q = pending[c0 + s], tail = state[s].tail;
				if (tail > cap) {
					overflowed.push_back(q);
					stats.tc_fallbacks += 1;
					continue;
				}
				hits.resize(tail);
				for (uint32_t j = 0; j < tail; ++j) {
					const uint32_t row = hi[size_t(s) * width + j];
					hits[j] = Hit{hd[size_t(s) * width + j], row, ix->h_labels[row]};
				}
				std::sort(hits.begin(), hits.end(), [](const Hit& l, const Hit& r) { return l.dist < r.dist || (l.dist == r.dist && l.label < r.label); });
				const uint64_t nout = std::min<uint64_t>(tail, max_out);  // best-first = the drain order of the reference's max-heap (std::less<pair>)
				for (uint64_t j = 0; j < nout; ++j) {
					out_dist[size_t(q) * max_out + j] = hits[j].dist;
					out_label[size_t(q) * max_out + j] = hits[j].label;
				}
				out_n[q] = tail;
			}
		}
		pending.swap(overflowed);
		overflowed.clear();
		cap = h->n;  // the overflowed queries once more, with regions that hold the whole graph
	}
	g_stats = stats;
	return 0;
}
}  // namespace

extern "C" {

int rxgpu_hnsw_search_range(const rxgpu_index* ix, const float* query, float radius, uint32_t ef, uint64_t max_out, float* out_dist,
							uint64_t* out_label, uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!query || !out_n || (max_out && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	*out_n = 0;
	if (ix->size == 0) {  // hnswalg.h:2017-2019
		return 0;
	}
	if (!ix->hnsw) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no HNSW graph imported into this index");
	}
	try {
		return hnswRangeBatch(ix, 1, query, &radius, ef, max_out, false, out_dist, out_label, out_n);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_hnsw_search_range_batch(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint32_t ef, uint64_t max_out,
								  float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (nq && (!queries || !radius || !out_n || (max_out && (!out_dist || !out_label)))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (nq == 0) {
		return 0;
	}
	std::fill(out_n, out_n + nq, uint64_t(0));
	if (ix->size == 0) {  // hnswalg.h:2017-2019
		return 0;
	}
	if (!ix->hnsw) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no HNSW graph imported into this index");
	}
	try {
		return hnswRangeBatch(ix, nq, queries, radius, ef, max_out, true, out_dist, out_label, out_n);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

}  // extern "C"

struct rxgpu_hnsw_stream {
	const rxgpu_index* ix = nullptr;
	uint64_t index_version = 0;
	uint32_t ef = 0, cap = 0;
	bool finished = false;
	DevBuf<float> query, out_dist;
	DevBuf<StreamHeader> hdr;
	DevBuf<uint64_t> top, cand, spill, extras;
	DevBuf<uint32_t> visited, out_idx, out_count;
};

extern "C" {

// BeginStreamingSearch (hnswalg.h:1864-1892): nothing is searched yet -- the first ContinueStreamingSearch descends to the entry point
int rxgpu_hnsw_stream_begin(const rxgpu_index* ix, const float* query, uint32_t ef, rxgpu_hnsw_stream** out) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!query || !out) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	*out = nullptr;
	if (int rc = checkGraph(ix)) {
		return rc;
	}
	const rxgpu_hnsw_device* h = ix->hnsw;
	ef = ef ? ef : 100u;  // kDefaultStreamingEf (hnswalg.h:1866)
	if (ef > kMaxEf) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: ef must be <= 1024 on the device path");
	}
	try {
		auto s = std::make_unique<rxgpu_hnsw_stream>();
		s->ix = ix;
		s->index_version = ix->version;
		s->ef = ef;
		s->cap = uint32_t(std::min<uint64_t>(std::max<uint64_t>(h->n, 1), 1u << 20));  // spill / extras never hold more than the visited nodes
		RX_CUDA(s->query.ensure(ix->dim));
		RX_CUDA(s->hdr.ensure(1));
		RX_CUDA(s->top.ensure(kMaxEf));
		RX_CUDA(s->cand.ensure(kStreamList));
		RX_CUDA(s->spill.ensure(s->cap));
		RX_CUDA(s->extras.ensure(s->cap));
		RX_CUDA(s->visited.ensure(h->words));
		RX_CUDA(s->out_dist.ensure(kMaxEf));
		RX_CUDA(s->out_idx.ensure(kMaxEf));
		RX_CUDA(s->out_count.ensure(4));
		RX_CUDA(cudaMemcpyAsync(s->query.p, query, size_t(ix->dim) * 4, cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaMemsetAsync(s->hdr.p, 0, sizeof(StreamHeader), ix->stream));
		RX_CUDA(cudaMemsetAsync(s->visited.p, 0, size_t(h->words) * 4, ix->stream));
		RX_CUDA(cudaStreamSynchronize(ix->stream));
		*out = s.release();
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

// ContinueStreamingSearch (hnswalg.h:1947-1975): the next `batch_size` closest expanded nodes, best first (ties by label);
// *exhausted != 0 when the whole reachable graph has been returned
int rxgpu_hnsw_stream_next(rxgpu_hnsw_stream* s, uint32_t batch_size, float* out_dist, uint64_t* out_label, uint32_t* out_count, int* exhausted) {
	if (!s || !out_count || !exhausted || (batch_size && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	const rxgpu_index* ix = s->ix;
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	*out_count = 0;
	*exhausted = s->finished ? 1 : 0;
	if (batch_size == 0 || s->finished) {
		return 0;  // hnswalg.h:1960-1962
	}
	rxgpu_hnsw_device* h = ix->hnsw;
	if (!h || s->index_version != ix->version || h->index_version != ix->version) {
		*exhausted = 1;  // the session's graph is gone (the reference answers "exhausted" for a foreign graph, :1956-1959)
		return 0;
	}
	if (batch_size > kMaxEf) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: batch size must be <= 1024 on the device path");
	}
	StreamArgs a{};
	a.h = graphArgs(ix, h);
	a.h.queries = s->query.p;
	a.hdr = s->hdr.p;
	a.top = s->top.p;
	a.cand = s->cand.p;
	a.spill = s->spill.p;
	a.extras = s->extras.p;
	a.visited = s->visited.p;
	a.cap = s->cap;
	a.ef = s->ef;
	a.batch = batch_size;
	a.out_dist = s->out_dist.p;
	a.out_idx = s->out_idx.p;
	a.out_count = s->out_count.p;
	const size_t smem = size_t(hnsw_query_words(ix->dim)) * 16 + size_t(kMaxEf) * 8 + size_t(kStreamList) * 8 + kMaxNeighbours * 8;
	if (smem > 200 * 1024) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: dimension exceeds the shared-memory budget of the streaming HNSW kernel");
	}
	// Sessions and the searches under h->mtx share the maintenance stream without a lock.  That is safe: the kernel reads only the
	// graph and rows, which no search writes, and writes only this session's own buffers, and the stream synchronise below completes
	// it before any of them is read.  Other calls' work on the stream can only delay that synchronise, never reach these buffers.
	cudaStream_t st = ix->stream;
	if (ix->metric == RXGPU_L2) {
		RX_CUDA(raiseSmemCeilingOnce(hnsw_stream_kernel<true>, ix->device, 200 * 1024));
		hnsw_stream_kernel<true><<<1, 32, smem, st>>>(a);
	} else {
		RX_CUDA(raiseSmemCeilingOnce(hnsw_stream_kernel<false>, ix->device, 200 * 1024));
		hnsw_stream_kernel<false><<<1, 32, smem, st>>>(a);
	}
	RX_CUDA(cudaGetLastError());
	uint32_t cnt[4] = {0, 0, 0, 0};
	RX_CUDA(cudaMemcpyAsync(cnt, s->out_count.p, 16, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	if (cnt[2]) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the streaming session outgrew its device buffers (more than 2^20 waiting nodes)");
	}
	const uint32_t n = std::min(cnt[0], batch_size);
	try {
		std::vector<float> hd(n);
		std::vector<uint32_t> hi(n);
		if (n) {
			RX_CUDA(cudaMemcpy(hd.data(), s->out_dist.p, size_t(n) * 4, cudaMemcpyDeviceToHost));
			RX_CUDA(cudaMemcpy(hi.data(), s->out_idx.p, size_t(n) * 4, cudaMemcpyDeviceToHost));
		}
		std::vector<Hit> hits(n);
		for (uint32_t j = 0; j < n; ++j) {
			hits[j] = Hit{hd[j], hi[j], ix->h_labels[hi[j]]};
		}
		orderTiesByLabel(hits);  // the batch is a SearchResultQueue under std::less<pair<float, label>> (:1928-1944)
		for (uint32_t j = 0; j < n; ++j) {
			out_dist[j] = hits[j].dist;
			out_label[j] = hits[j].label;
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	*out_count = n;
	s->finished = cnt[1] != 0;
	*exhausted = s->finished ? 1 : 0;
	g_stats = rxgpu_search_stats{};
	g_stats.launches = 1;
	return 0;
}

void rxgpu_hnsw_stream_end(rxgpu_hnsw_stream* s) {
	if (s) {
		cudaSetDevice(s->ix->device);
		delete s;
	}
}

int rxgpu_gather_labels_device(const rxgpu_index* ix, uint64_t n, const uint32_t* d_idx, uint64_t* d_out_label, void* stream) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (n == 0) {
		return 0;
	}
	if (!d_idx || !d_out_label) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
	gather_labels_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(ix->d_labels, ix->size, n, d_idx, d_out_label);
	RX_CUDA(cudaGetLastError());
	if (!stream) {
		RX_CUDA(cudaStreamSynchronize(st));
	}
	return 0;
}

// Restores a graph straight from the reference's index cache (what HierarchicalNSWImpl::SaveIndex writes, hnswalg.h:1213-1263, and its
// loader constructor reads, :297-403; the token stream is hnswlib::IReader's, hnswlib.h -- hnsw_index.cc:455-483 implements it over the
// storage blob and the namespace's primary keys): no host-side graph is built, rows and lists go to the device as they are decoded.
int rxgpu_hnsw_load_index_cache(rxgpu_index* ix, const rxgpu_hnsw_cache_reader* r, rxgpu_hnsw_cache_info* info) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!r || !r->get_var_uint || !r->get_var_int || !r->get_vstring || !r->read_pk_encoded_data) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (ix->size != 0) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the index cache is loaded into an empty index");
	}
	try {
		void* c = r->ctx;
		const uint64_t maxElements = r->get_var_uint(c);
		const uint64_t count = r->get_var_uint(c);
		if (count > maxElements) {
			return fail(RXGPU_ERR_PARAMS, "Current elements count is larger than max elements count");  // hnswalg.h:303
		}
		const int64_t maxlevel = r->get_var_int(c);
		const uint64_t enterpoint = r->get_var_uint(c);
		if (count ? enterpoint >= count : enterpoint != 0xFFFFFFFFull) {
			return fail(RXGPU_ERR_PARAMS, count ? "Incorrect entrypoint node ID" : "Unexpected entrypoint node ID for empty HNSW");  // :325-330
		}
		const uint64_t M = r->get_var_uint(c);
		const uint64_t efConstruction = r->get_var_uint(c);
		if (M == 0 || M > 4096 || count > 0xFFFFFFF0ull || count > ix->capacity) {
			return fail(RXGPU_ERR_PARAMS, count > ix->capacity ? "rxgpu: the index cache holds more elements than the index's capacity"
																: "rxgpu: malformed HNSW index cache header");
		}
		if (info) {
			*info = rxgpu_hnsw_cache_info{maxElements, count, int32_t(maxlevel), uint32_t(enterpoint), uint32_t(M), uint32_t(efConstruction), 0};
		}
		if (count == 0) {
			return 0;
		}
		const uint32_t n = uint32_t(count), m0 = uint32_t(2 * M);
		std::vector<uint32_t> level0(size_t(n) * (1 + m0), 0u);
		std::vector<uint64_t> labels(n);
		std::vector<uint32_t> deleted;
		const size_t slice = std::max<size_t>(1, (size_t(64) << 20) / (size_t(ix->dim) * 4));
		std::vector<float> rows(std::min<size_t>(slice, n) * ix->dim);
		size_t sliceBase = 0;
		for (uint32_t i = 0; i < n; ++i) {
			const uint32_t marked = uint32_t(r->get_var_uint(c));  // [u16 count | u8 flags | pad] (hnswalg.h:221-228)
			const uint32_t cnt = marked & 0xFFFFu;
			if (cnt > m0) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW index cache: a level-0 neighbour count exceeds 2*M");
			}
			uint32_t* l0 = level0.data() + size_t(i) * (1 + m0);
			l0[0] = cnt;
			for (uint32_t j = 0; j < cnt; ++j) {
				l0[1 + j] = uint32_t(r->get_var_uint(c));
			}
			float* dst = rows.data() + (i - sliceBase) * ix->dim;
			if ((marked >> 16) & 0x01u) {  // DELETE_MARK: the vector itself is stored, the label is gone (:372-375)
				const char* data = nullptr;
				uint64_t len = 0;
				if (r->get_vstring(c, &data, &len) || len != size_t(ix->dim) * 4) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW index cache: a deleted element's vector has the wrong size");
				}
				std::memcpy(dst, data, len);
				labels[i] = (uint64_t(1) << 63) | uint64_t(i);  // a tombstone's slot keeps a label of its own
				deleted.push_back(i);
			} else {
				labels[i] = r->read_pk_encoded_data(c, dst);  // the namespace resolves the primary key and copies the row's vector
			}
			if (i + 1 - sliceBase == slice || i + 1 == n) {
				if (int rc = rxgpu_index_upsert_batch(ix, i + 1 - sliceBase, labels.data() + sliceBase, rows.data())) {
					return rc;
				}
				sliceBase = i + 1;
			}
		}
		const size_t s1 = 1 + size_t(M);
		std::vector<int32_t> levels(n);
		std::vector<int64_t> upperOff(size_t(n) + 1, 0);
		std::vector<uint32_t> upper;
		for (uint32_t i = 0; i < n; ++i) {
			const char* data = nullptr;
			uint64_t len = 0;
			if (r->get_vstring(c, &data, &len) || len % (s1 * 4) != 0) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW index cache: an upper-level list blob has the wrong size");
			}
			levels[i] = int32_t(len / (s1 * 4));  // element_levels_[i] = size / size_links_per_element_ (:1278)
			upperOff[i + 1] = upperOff[i] + levels[i];
			const size_t at = upper.size();
			upper.resize(at + len / 4);
			std::memcpy(upper.data() + at, data, len);
			for (int32_t lv = 0; lv < levels[i]; ++lv) {
				upper[at + size_t(lv) * s1] &= 0xFFFFu;  // the count word carries flag bits
			}
		}
		rxgpu_hnsw_graph g{};
		g.n = n;
		g.M = uint32_t(M);
		g.maxM0 = m0;
		g.maxlevel = int32_t(maxlevel);
		g.enterpoint = uint32_t(enterpoint);
		g.upper_slots = uint64_t(upperOff[n]);
		g.level0 = level0.data();
		g.levels = levels.data();
		g.upper_offsets = upperOff.data();
		g.upper = upper.empty() ? nullptr : upper.data();
		if (int rc = rxgpu_hnsw_import(ix, &g)) {
			return rc;
		}
		for (const uint32_t i : deleted) {
			if (int rc = rxgpu_hnsw_mark_deleted(ix, labels[i])) {
				return rc;
			}
		}
		if (info) {
			info->deleted = uint32_t(deleted.size());
		}
		return 0;
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	} catch (const std::exception& e) {  // the reader's callbacks may throw (corrupted blob, missing row)
		return fail(RXGPU_ERR_PARAMS, std::string("rxgpu: HNSW index cache: ") + e.what());
	}
}

// Incremental maintenance after the reference's inserter changed the host graph: HierarchicalNSWImpl::addPoint (hnswalg.h:1695-1852)
// touches the new node's lists and the lists of the neighbours it was linked to (mutuallyConnectNewElement, :1070-1180); the adapter
// hands over exactly those nodes.  Nothing else of the device copy moves: an upsert costs O(M) small copies, not a re-import.
int rxgpu_hnsw_update(rxgpu_index* ix, int32_t maxlevel, uint32_t enterpoint, uint32_t nupdates, const rxgpu_hnsw_node_update* upd) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	rxgpu_hnsw_device* h = ix->hnsw;
	if (!h) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no HNSW graph imported into this index");
	}
	if (nupdates && !upd) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	std::lock_guard<std::mutex> lck(h->mtx);
	const size_t s0 = size_t(1) + h->maxM0, s1 = size_t(1) + h->M;
	// validate first: nothing is applied when any update is malformed
	uint64_t newRows = 0, newSlots = 0;
	for (uint32_t i = 0; i < nupdates; ++i) {
		const rxgpu_hnsw_node_update& u = upd[i];
		if (!u.level0 || u.level < 0 || (u.level > 0 && !u.upper) || u.level0[0] > h->maxM0) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW update: malformed node");
		}
		const bool appended = u.node >= ix->size;
		if (appended) {
			if (!u.vec || u.node != ix->size + newRows) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW update: new nodes carry their vector and arrive in internal-id order");
			}
			newRows += 1;
			newSlots += uint64_t(u.level);
		} else if (u.level != h->h_levels[u.node]) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW update: the level of an existing node cannot change");
		}
	}
	const uint64_t nAfter = ix->size + newRows;
	if (nAfter > ix->capacity || nAfter > h->cap_nodes || h->upper_slots + newSlots > h->upper.n / s1) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: HNSW update exceeds the device copy's capacity (re-import the graph)");
	}
	for (uint32_t i = 0; i < nupdates; ++i) {
		const rxgpu_hnsw_node_update& u = upd[i];
		for (uint32_t j = 1; j <= u.level0[0]; ++j) {
			if (u.level0[j] >= nAfter) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW update: neighbour id out of range");
			}
		}
		for (int32_t lv = 0; lv < u.level; ++lv) {
			const uint32_t* l = u.upper + size_t(lv) * s1;
			if (l[0] > h->M) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW update: malformed upper list");
			}
			for (uint32_t j = 1; j <= l[0]; ++j) {
				if (l[j] >= nAfter) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW update: neighbour id out of range");
				}
			}
		}
	}
	cudaStream_t st = ix->stream;
	for (uint32_t i = 0; i < nupdates; ++i) {
		const rxgpu_hnsw_node_update& u = upd[i];
		if (u.vec) {  // a new node, or a slot whose vector was replaced (updatePoint; a reused tombstone, hnswalg.h:1445-1451): row + label
			const bool appended = u.node >= ix->size;
			const uint32_t other = ix->dict.find(u.label);
			if (other != LabelMap::kNotFound && other != u.node && ((h->h_deleted[other >> 5] >> (other & 31)) & 1u)) {
				// the label lives again in another slot: its tombstone takes a label of its own
				const uint64_t tomb = (uint64_t(1) << 63) | uint64_t(other);
				ix->dict.erase(u.label);
				ix->dict.put(tomb, other);
				ix->h_labels[other] = tomb;
				RX_CUDA(cudaMemcpyAsync(ix->d_labels + other, &ix->h_labels[other], 8, cudaMemcpyHostToDevice, st));
			}
			if (int rc = setRowAt(ix, u.node, u.label, u.vec)) {
				return rc;
			}
			if (appended) {
				const long long off = (long long)h->upper_slots;  // its upper-level lists take fresh slots at the end of the slab
				h->upper_slots += uint64_t(u.level);
				h->h_upper_off.push_back(off);
				h->h_levels.push_back(u.level);
				RX_CUDA(cudaMemcpyAsync(h->upper_off.p + u.node, &h->h_upper_off[u.node], 8, cudaMemcpyHostToDevice, st));
				RX_CUDA(cudaMemcpyAsync(h->levels.p + u.node, &h->h_levels[u.node], 4, cudaMemcpyHostToDevice, st));
				RX_CUDA(cudaStreamSynchronize(st));  // the vectors above may reallocate on the next push_back
			}
		}
		RX_CUDA(cudaMemcpyAsync(h->level0.p + size_t(u.node) * s0, u.level0, s0 * 4, cudaMemcpyHostToDevice, st));
		if (u.level > 0) {
			RX_CUDA(cudaMemcpyAsync(h->upper.p + size_t(h->h_upper_off[u.node]) * s1, u.upper, size_t(u.level) * s1 * 4, cudaMemcpyHostToDevice, st));
		}
		// tombstone bit follows the host graph (a reused slot is alive again)
		const uint32_t bit = 1u << (u.node & 31);
		const bool was = (h->h_deleted[u.node >> 5] & bit) != 0;
		if (was != (u.deleted != 0)) {
			h->h_deleted[u.node >> 5] ^= bit;
			h->num_deleted += u.deleted ? 1 : -1;
			RX_CUDA(cudaMemcpyAsync(h->deleted.p + (u.node >> 5), &h->h_deleted[u.node >> 5], 4, cudaMemcpyHostToDevice, st));
		}
	}
	RX_CUDA(cudaStreamSynchronize(st));
	h->maxlevel = maxlevel;
	h->enterpoint = enterpoint;
	h->n = uint32_t(ix->size);
	h->index_version = ix->version;
	h->updates += nupdates;
	ix->rows_touched_from = ~0ull;
	return 0;
}
uint64_t rxgpu_hnsw_update_count(const rxgpu_index* ix) { return ix && ix->hnsw ? ix->hnsw->updates : 0; }

int rxgpu_hnsw_mark_deleted(rxgpu_index* ix, uint64_t label) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (int rc = checkGraph(ix)) {
		return rc;
	}
	rxgpu_hnsw_device* h = ix->hnsw;
	const uint32_t idx = ix->dict.find(label);
	if (idx == LabelMap::kNotFound) {
		return fail(RXGPU_ERR_NOT_FOUND, "markDelete: Label not found: " + std::to_string(label));  // hnswalg.h:1307
	}
	std::lock_guard<std::mutex> lck(h->mtx);
	const uint32_t bit = 1u << (idx & 31);
	if (h->h_deleted[idx >> 5] & bit) {
		return fail(RXGPU_ERR_LOGIC, "The requested to delete element is already deleted");  // hnswalg.h:1335
	}
	h->h_deleted[idx >> 5] |= bit;
	RX_CUDA(cudaMemcpyAsync(h->deleted.p + (idx >> 5), &h->h_deleted[idx >> 5], 4, cudaMemcpyHostToDevice, ix->stream));
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	h->num_deleted += 1;
	return 0;
}
uint64_t rxgpu_hnsw_deleted_count(const rxgpu_index* ix) { return ix && ix->hnsw ? ix->hnsw->num_deleted : 0; }

}  // extern "C"
