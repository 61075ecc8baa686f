// HNSW graph construction on the device: a deterministic batched insertion (DESIGN.md §3.8).
//
// Rows [first, n) of the index are inserted in row order, in batches that the host plans from the levels alone
// (rxgpu_hnsw_build_plan).  Every row of a batch is inserted against the graph as it stood when the batch began:
//   search + select (one warp per row, the persistent slots of the search kernel): the greedy descent of addPoint
//     (hnswalg.h:1781-1811), searchBaseLayer with ef = efConstruction at each of the row's levels (:644-975), and
//     getNeighborsByHeuristic2 with M (:976-1030) in-warp; the row's lists are written farthest first (:1059-1062) and every
//     selected neighbour v at level l gets a reverse-link key (l, v, row);
//   reverse links (one kernel boundary later): the keys are radix sorted, one warp takes each (l, v) segment: the old list plus the
//     incoming rows in ascending order are appended when they fit in Mcurmax, otherwise the union is pruned once with the heuristic
//     against v (:1128-1162) -- one prune per batch where the reference prunes once per insert.
// Equal distances are ordered by row id everywhere (the reference's heaps leave that order undefined).  d(a, b) is the search path's
// distance with row a as the query: warp_dists over the row staged in shared memory (for Cosine normalised as NormalizeCopyVector
// normalises a query, times b's norm coefficient).  tests/hnsw_build_model.py replays these rules and must give the same graph.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "common.cuh"
#include "internal.h"
#include "hnsw_graph.cuh"

using namespace rxgpu;

namespace {

// The batch rules.  A batch starting at graph size s holds at most max(1, s >> kBuildBatchShift) rows (a fraction rho = 1/64 of the
// graph, the order of ParlayANN's deterministic batch insertion, which bounds how many of a row's near neighbours are still invisible to
// it) and never more than kBuildBatchMax: the row's offset in its batch is the low 16 bits of a reverse-link key, and the batch's keys,
// sorted copy and segment list (about 20 bytes per link) stay a few tens of MB at M = 32.
constexpr uint32_t kBuildBatchShift = 6;
constexpr uint32_t kBuildBatchMax = 1u << 16;
constexpr int32_t kBuildMaxLevel = 0xFFFF;  // the level takes the top 16 bits of a reverse-link key
constexpr int kBuildSelMax = 32;            // M <= 32: the selected list of a row fits one warp

struct BuildArgs {
	HnswArgs g;                // rows, graph, visited bitmaps + clear logs, the row counter; ef = efConstruction; maxlevel / enterpoint
							   // as the batch began
	const float* qk;           // Cosine: the factor NormalizeCopyVector applies to a row staged as the query; else null
	uint32_t b0, nb, M;        // the batch: rows [b0, b0 + nb)
	uint64_t* keys;            // reverse-link keys level << 48 | v << 16 | (u - b0), appended; unused entries stay kKeyNone.  After the
							   // sort a pruned segment keeps the distance keys of its incoming rows in its own range here
	unsigned int* nkeys;
	unsigned long long* ndist;  // distance evaluations
	// reverse links
	uint64_t* sorted;          // the keys in ascending order; read-only once sorted (every warp scans past its own run)
	uint64_t* alt;             // a pruned segment's incoming rows in ascending (distance, id) order, in its own range
	uint32_t key_cap;          // entries of keys / sorted / alt this batch
	uint32_t* seg;             // first key of every (level, v) segment
	unsigned int* nseg;
	unsigned int* next_seg;
	unsigned long long* npruned;
};

__device__ __forceinline__ uint32_t* list_of_mut(const HnswArgs& a, uint32_t node, int level) {
	return const_cast<uint32_t*>(list_of(a, node, level));
}

// row `row` as the query, zero padded: for Cosine multiplied by its normalisation factor (out[i] = x[i] * k, tools/normalize.h:16-20)
__device__ __forceinline__ void stage_row(const BuildArgs& b, float4* sq4, uint32_t row, uint32_t dp4, int lane) {
	__syncwarp();
	float* sq = reinterpret_cast<float*>(sq4);
	const float* r = b.g.rows + size_t(row) * b.g.pitch;
	const float k = b.qk ? b.qk[row] : 1.f;
	for (uint32_t c = lane; c < dp4 * 4; c += 32) {
		sq[c] = c < b.g.dim ? (b.qk ? __fmul_rn(r[c], k) : r[c]) : 0.f;
	}
	__syncwarp();
}

// (d, id) before (e, jd): distance first, equal distances by row id
__device__ __forceinline__ bool key_less(float d, uint32_t id, float e, uint32_t jd) { return d < e || (d == e && id < jd); }

// searchBaseLayer (hnswalg.h:644-975) at `level` from `ep`: the <= ef closest visited nodes, ascending by (distance, id), in
// l_dist / l_id (kExpanded set on the expanded ones) -- the unified list of the search kernel with ties ordered by id.  Returns the size.
template <bool kIsL2>
__device__ uint32_t search_layer(const BuildArgs& b, const float4* sq4, uint32_t ep, int level, float* l_dist, uint32_t* l_id, uint32_t* s_ids,
								 float* s_d, uint32_t* visited, uint32_t* vlog, int lane, uint32_t& n_dist) {
	const HnswArgs& a = b.g;
	if (lane == 0) {
		s_ids[0] = ep;
	}
	__syncwarp();
	warp_dists<kIsL2>(a, sq4, s_ids, 1, s_d, lane);
	n_dist += 1;
	if (lane == 0) {
		l_dist[0] = s_d[0];
		l_id[0] = ep;
		atomicOr(&visited[ep >> 5], 1u << (ep & 31));
		vlog[0] = ep;
	}
	__syncwarp();
	uint32_t size = 1, vcount = 1;
	for (;;) {
		const int pos = first_unexpanded(l_id, size, lane);
		if (pos < 0) {
			break;  // every candidate at or below lowerBound is expanded (:681)
		}
		const uint32_t node = l_id[pos];
		__syncwarp();
		if (lane == 0) {
			l_id[pos] = node | kExpanded;
		}
		const uint32_t* ll = list_of(a, node, level);
		const uint32_t ucnt = gather_fresh(ll, min(ll[0], uint32_t(kMaxNeighbours)), visited, vlog, vcount, s_ids, lane);
		if (ucnt == 0) {
			continue;
		}
		warp_dists<kIsL2>(a, sq4, s_ids, ucnt, s_d, lane);
		n_dist += ucnt;
		for (uint32_t j = 0; j < ucnt; ++j) {  // the accept rule of :931-957, in list order
			const float d = s_d[j];
			const uint32_t nid = s_ids[j];
			if (size >= a.ef && !key_less(d, nid, l_dist[size - 1], l_id[size - 1] & ~kExpanded)) {
				continue;
			}
			const uint32_t p = warp_count(size, lane, [&](uint32_t i) { return key_less(l_dist[i], l_id[i] & ~kExpanded, d, nid); });
			const uint32_t newsize = min(size + 1, a.ef);
			list_insert(l_dist, l_id, p, newsize, d, nid, lane);
			size = newsize;
		}
	}
	// the visited bitmap cleared from its log, as the search kernel does: as a helper shared with that kernel, ptxas allocated
	// hnsw_build_insert<true> differently and its insert phase ran 5 % slower
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
	return size;
}

// true when no selected row s has d(x, s) < dx, x staged as the query (the test of getNeighborsByHeuristic2, :1009-1011)
template <bool kIsL2>
__device__ __forceinline__ bool heuristic_keeps(const BuildArgs& b, float4* sq4, uint32_t x, float dx, const uint32_t* sel, uint32_t nsel,
												uint32_t* s_ids, float* s_d, uint32_t dp4, int lane, uint32_t& n_dist) {
	if (nsel == 0) {
		return true;
	}
	stage_row(b, sq4, x, dp4, lane);
	for (uint32_t t = lane; t < nsel; t += 32) {
		s_ids[t] = sel[t];
	}
	__syncwarp();
	warp_dists<kIsL2>(b.g, sq4, s_ids, nsel, s_d, lane);
	n_dist += nsel;
	bool closer = false;
	for (uint32_t t = lane; t < nsel; t += 32) {
		closer |= s_d[t] < dx;
	}
	const bool keep = !__any_sync(0xffffffffu, closer);
	__syncwarp();
	return keep;
}

// search + select: one warp inserts one row of the batch at a time
template <bool kIsL2>
__global__ void __launch_bounds__(kHnswThreads) hnsw_build_insert(const BuildArgs b) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const HnswArgs& a = b.g;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t dp4 = hnsw_query_words(a.dim);
	// per warp: query | list dist[ef] | list id[ef] | gather ids[64] | gather dists[64] | selected[32]
	const uint32_t efp = (a.ef + 3u) & ~3u;
	const size_t per_warp = size_t(dp4) * 16 + size_t(efp) * 8 + kMaxNeighbours * 8 + kBuildSelMax * 4;
	unsigned char* base = smem_raw + per_warp * warp;
	float4* sq4 = reinterpret_cast<float4*>(base);
	float* l_dist = reinterpret_cast<float*>(base + size_t(dp4) * 16);
	uint32_t* l_id = reinterpret_cast<uint32_t*>(l_dist + efp);
	uint32_t* s_ids = l_id + efp;
	float* s_d = reinterpret_cast<float*>(s_ids + kMaxNeighbours);
	uint32_t* sel = reinterpret_cast<uint32_t*>(s_d + kMaxNeighbours);
	const uint32_t slot = blockIdx.x * kHnswWarps + warp;
	uint32_t* visited = a.visited + size_t(slot) * a.words;
	uint32_t* vlog = a.vlog + size_t(slot) * kVlogCap;
	uint32_t n_dist = 0;
	for (;;) {
		uint32_t qi = 0;
		if (lane == 0) {
			qi = atomicAdd(a.next_query, 1u);
		}
		qi = __shfl_sync(0xffffffffu, qi, 0);
		if (qi >= b.nb) {
			break;
		}
		const uint32_t u = b.b0 + qi;
		stage_row(b, sq4, u, dp4, lane);
		const int lvl = a.levels[u];
		// greedy descent through maxlevel .. lvl + 1 (:1781-1811), the entry point's distance counted: greedy_descent's rule, written
		// out with list_of because through the helper ptxas gives the Cosine instantiation 64 registers instead of 56
		uint32_t cur = a.enterpoint;
		if (lvl < a.maxlevel) {
			if (lane == 0) {
				s_ids[0] = cur;
			}
			__syncwarp();
			warp_dists<kIsL2>(a, sq4, s_ids, 1, s_d, lane);
			n_dist += 1;
			float curdist = s_d[0];
			__syncwarp();
			for (int level = a.maxlevel; level > lvl; --level) {
				bool changed = true;
				while (changed) {
					changed = false;
					const uint32_t* ll = list_of(a, cur, level);
					const uint32_t cnt = min(ll[0], uint32_t(kMaxNeighbours));
					for (uint32_t j = lane; j < cnt; j += 32) {
						s_ids[j] = ll[1 + j];
					}
					__syncwarp();
					if (cnt) {
						warp_dists<kIsL2>(a, sq4, s_ids, cnt, s_d, lane);
						n_dist += cnt;
					}
					for (uint32_t j = 0; j < cnt; ++j) {
						if (s_d[j] < curdist) {
							curdist = s_d[j];
							cur = s_ids[j];
							changed = true;
						}
					}
					__syncwarp();
				}
			}
		}
		for (int l = min(lvl, a.maxlevel); l >= 0; --l) {
			const uint32_t size = search_layer<kIsL2>(b, sq4, cur, l, l_dist, l_id, s_ids, s_d, visited, vlog, lane, n_dist);
			// getNeighborsByHeuristic2 with M (:976-1030): fewer than M candidates are all kept
			uint32_t nsel = 0;
			bool staged_other = false;
			if (size < b.M) {
				for (uint32_t i = lane; i < size; i += 32) {
					sel[i] = l_id[i] & ~kExpanded;
				}
				nsel = size;
			} else {
				for (uint32_t i = 0; i < size && nsel < b.M; ++i) {
					const uint32_t x = l_id[i] & ~kExpanded;
					staged_other |= nsel > 0;
					if (heuristic_keeps<kIsL2>(b, sq4, x, l_dist[i], sel, nsel, s_ids, s_d, dp4, lane, n_dist)) {
						if (lane == 0) {
							sel[nsel] = x;
						}
						__syncwarp();
						++nsel;
					}
				}
			}
			__syncwarp();
			// the row's list, farthest first (:1059-1062), and a reverse-link key per selected neighbour
			uint32_t* ll = list_of_mut(a, u, l);
			unsigned int kbase = 0;
			if (lane == 0) {
				ll[0] = nsel;
				kbase = atomicAdd(b.nkeys, nsel);
			}
			kbase = __shfl_sync(0xffffffffu, kbase, 0);
			for (uint32_t j = lane; j < nsel; j += 32) {
				const uint32_t v = sel[nsel - 1 - j];
				ll[1 + j] = v;
				if (kbase + j < b.key_cap) {
					b.keys[kbase + j] = (uint64_t(l) << 48) | (uint64_t(v) << 16) | uint64_t(qi);
				}
			}
			__syncwarp();
			cur = sel[0];  // the next level starts from the closest selected node (:1064)
			__syncwarp();
			if (staged_other && l > 0) {
				stage_row(b, sq4, u, dp4, lane);
			}
		}
	}
	if (lane == 0 && n_dist) {
		atomicAdd(b.ndist, (unsigned long long)n_dist);
	}
}

// the first key of every (level, v) run of the sorted keys
__global__ void hnsw_build_heads(const BuildArgs b) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= b.key_cap) {
		return;
	}
	const uint64_t k = b.sorted[i];
	if (k != kKeyNone && (i == 0 || (b.sorted[i - 1] >> 16) != (k >> 16))) {
		b.seg[atomicAdd(b.nseg, 1u)] = i;
	}
}

// reverse links: one warp per (level, v) segment
template <bool kIsL2>
__global__ void __launch_bounds__(kHnswThreads) hnsw_build_link(const BuildArgs b) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const HnswArgs& a = b.g;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t dp4 = hnsw_query_words(a.dim);
	// per warp: query | gather ids[64] | gather dists[64] | old list keys[64] | old list sorted[64] | selected[64]
	const size_t per_warp = size_t(dp4) * 16 + kMaxNeighbours * (4 + 4 + 8 + 8 + 4);
	unsigned char* base = smem_raw + per_warp * warp;
	float4* sq4 = reinterpret_cast<float4*>(base);
	uint64_t* o_key = reinterpret_cast<uint64_t*>(base + size_t(dp4) * 16);
	uint64_t* o_sorted = o_key + kMaxNeighbours;
	uint32_t* s_ids = reinterpret_cast<uint32_t*>(o_sorted + kMaxNeighbours);
	float* s_d = reinterpret_cast<float*>(s_ids + kMaxNeighbours);
	uint32_t* sel = reinterpret_cast<uint32_t*>(s_d + kMaxNeighbours);
	uint32_t n_dist = 0;
	for (;;) {
		uint32_t si = 0;
		if (lane == 0) {
			si = atomicAdd(b.next_seg, 1u);
		}
		si = __shfl_sync(0xffffffffu, si, 0);
		if (si >= *b.nseg) {
			break;
		}
		const uint32_t h = b.seg[si];
		const uint64_t prefix = b.sorted[h] >> 16;
		const int l = int(prefix >> 32);
		const uint32_t v = uint32_t(prefix);
		uint32_t k = 0;  // incoming rows: the run [h, h + k)
		for (uint32_t c = h;; c += 32) {
			const uint32_t i = c + lane;
			const unsigned m = __ballot_sync(0xffffffffu, i < b.key_cap && (b.sorted[i] >> 16) == prefix);
			if (m != 0xffffffffu) {  // the run is contiguous: it ends at the first lane outside it
				k += uint32_t(__ffs(~m) - 1);
				break;
			}
			k += 32;
		}
		uint32_t* ll = list_of_mut(a, v, l);
		const uint32_t c = ll[0];
		const uint32_t mc = l ? b.M : 2 * b.M;  // Mcurmax
		if (c + k <= mc) {  // append in ascending row order
			for (uint32_t j = lane; j < k; j += 32) {
				ll[1 + c + j] = b.b0 + uint32_t(b.sorted[h + j] & 0xFFFFu);
			}
			__syncwarp();
			if (lane == 0) {
				ll[0] = c + k;
			}
			__syncwarp();
			continue;
		}
		// prune the union once: d(v, x) for the old list and the incoming rows, both in ascending (distance, id) order
		stage_row(b, sq4, v, dp4, lane);
		for (uint32_t j = lane; j < c; j += 32) {
			s_ids[j] = ll[1 + j];
		}
		__syncwarp();
		warp_dists<kIsL2>(a, sq4, s_ids, c, s_d, lane);
		n_dist += c;
		for (uint32_t j = lane; j < c; j += 32) {
			o_key[j] = make_key(s_d[j], s_ids[j]);
		}
		__syncwarp();
		for (uint32_t j = lane; j < c; j += 32) {
			uint32_t r = 0;
			for (uint32_t t = 0; t < c; ++t) {
				r += o_key[t] < o_key[j];
			}
			o_sorted[r] = o_key[j];
		}
		for (uint32_t off = 0; off < k; off += kMaxNeighbours) {
			const uint32_t m = min(k - off, uint32_t(kMaxNeighbours));
			__syncwarp();
			for (uint32_t j = lane; j < m; j += 32) {
				s_ids[j] = b.b0 + uint32_t(b.sorted[h + off + j] & 0xFFFFu);
			}
			__syncwarp();
			warp_dists<kIsL2>(a, sq4, s_ids, m, s_d, lane);
			n_dist += m;
			for (uint32_t j = lane; j < m; j += 32) {
				b.keys[h + off + j] = make_key(s_d[j], s_ids[j]);
			}
		}
		__syncwarp();
		for (uint32_t j = lane; j < k; j += 32) {  // the run reordered by rank; a hub's run may be far longer than Mcurmax
			const uint64_t key = b.keys[h + j];
			uint32_t r = 0;
			for (uint32_t t = 0; t < k; ++t) {
				r += b.keys[h + t] < key;
			}
			b.alt[h + r] = key;
		}
		__syncwarp();
		// getNeighborsByHeuristic2 with Mcurmax over the merged order
		uint32_t nsel = 0, io = 0, in = 0;
		while (nsel < mc && (io < c || in < k)) {
			const uint64_t ko = io < c ? o_sorted[io] : kKeyNone;
			const uint64_t kn = in < k ? b.alt[h + in] : kKeyNone;
			const uint64_t key = ko < kn ? ko : kn;
			if (ko < kn) {
				++io;
			} else {
				++in;
			}
			const uint32_t x = uint32_t(key);
			if (heuristic_keeps<kIsL2>(b, sq4, x, ord_float(uint32_t(key >> 32)), sel, nsel, s_ids, s_d, dp4, lane, n_dist)) {
				if (lane == 0) {
					sel[nsel] = x;
				}
				__syncwarp();
				++nsel;
			}
		}
		for (uint32_t j = lane; j < nsel; j += 32) {  // farthest first, as the reference drains its heap
			ll[1 + j] = sel[nsel - 1 - j];
		}
		__syncwarp();
		if (lane == 0) {
			ll[0] = nsel;
			atomicAdd(b.npruned, 1ull);
		}
		__syncwarp();
	}
	if (lane == 0 && n_dist) {
		atomicAdd(b.ndist, (unsigned long long)n_dist);
	}
}

// the factor NormalizeCopyVector applies to a query (tools/normalize.cc:10-23): sequential sum of squares, one thread per row
__global__ void hnsw_build_query_coefs(const float* rows, uint32_t pitch, uint32_t dim, uint32_t n, float* qk) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) {
		return;
	}
	const float* p = rows + size_t(i) * pitch;
	float s = 0.f;
	for (uint32_t c = 0; c < dim; ++c) {
		s = __fadd_rn(s, __fmul_rn(p[c], p[c]));
	}
	float k = 1.f;
	if (s > 0.f && fabsf(1.0f - s) > 0.00001f) {
		k = float(1.0 / double(__fsqrt_rn(s)));
	}
	qk[i] = k;
}

// rows idx[i] of a [*][width] u32 array to out[i][width]
__global__ void hnsw_gather_lists(const uint32_t* src, uint32_t width, const uint64_t* idx, uint64_t n, uint32_t* out) {
	const uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x;
	if (i < n * width) {
		const uint64_t r = i / width;
		out[i] = src[idx[r] * width + (i - r * width)];
	}
}

size_t insertSmem(uint32_t dim, uint32_t ef) {
	return (size_t(hnsw_query_words(dim)) * 16 + size_t((ef + 3u) & ~3u) * 8 + kMaxNeighbours * 8 + kBuildSelMax * 4) * kHnswWarps;
}
size_t linkSmem(uint32_t dim) { return (size_t(hnsw_query_words(dim)) * 16 + kMaxNeighbours * (4 + 4 + 8 + 8 + 4)) * kHnswWarps; }
constexpr size_t kBuildSmemBudget = 200 * 1024;

// getRandomLevel (hnswalg.h:625-635) for `count` rows: std::default_random_engine seeded like level_generator_ (:293), one draw each
void drawLevels(uint32_t M, uint64_t seed, uint64_t count, int32_t* out) {
	std::default_random_engine gen;
	gen.seed(seed);
	const double mult = 1.0 / log(1.0 * M);
	for (uint64_t i = 0; i < count; ++i) {
		std::uniform_real_distribution<double> distribution(0.0, 1.0);
		const double r = -log(distribution(gen)) * mult;
		out[i] = int(r);
	}
}

// the batch ends of rows [first, n) with levels lv[0, n - first), the graph's top level being maxlevel (-1: no graph)
void planBatches(uint64_t first, uint64_t n, int32_t maxlevel, const int32_t* lv, std::vector<uint64_t>& ends) {
	uint64_t s = first;
	int32_t ml = maxlevel;
	if (first == 0 && n > 0) {  // the first row is inserted alone
		ends.push_back(1);
		s = 1;
		ml = lv[0];
	}
	while (s < n) {
		const uint64_t cap = std::min<uint64_t>(kBuildBatchMax, std::max<uint64_t>(1, s >> kBuildBatchShift));
		uint64_t e = s;
		while (e < n && e - s < cap) {
			const int32_t l = lv[e - first];
			++e;
			if (l > ml) {  // a new top level: the row becomes the enter point of the next batch
				ml = l;
				break;
			}
		}
		ends.push_back(e);
		s = e;
	}
}

int checkPlanArgs(uint32_t M, uint64_t first, uint64_t n, int32_t maxlevel, const int32_t* levels) {
	if (M < 2 || M > 32) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: M must be in [2, 32]");
	}
	if (first > n || n >= (uint64_t(1) << 31)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: rows must satisfy first <= n < 2^31");
	}
	if ((first == 0) != (maxlevel < 0) || maxlevel > kBuildMaxLevel) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: maxlevel must be -1 exactly when there is no graph");
	}
	if (levels) {
		for (uint64_t i = 0; i < n - first; ++i) {
			if (levels[i] < 0 || levels[i] > kBuildMaxLevel) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: levels must be in [0, 65535]");
			}
		}
	}
	return 0;
}

// rows [first, ix->size) with levels lv inserted into a copy of `old` (null: no graph yet); the result goes to `out`
int buildGraph(rxgpu_index* ix, const rxgpu_hnsw_device* old, uint32_t M, uint32_t ef_construction, const std::vector<int32_t>& lv,
			   std::unique_ptr<rxgpu_hnsw_device>& out, rxgpu_hnsw_build_stats& st) {
	const uint64_t n = ix->size, first = old ? old->n : 0;
	const uint32_t nNew = uint32_t(n - first);
	std::vector<uint64_t> ends;
	planBatches(first, n, old ? old->maxlevel : -1, lv.data(), ends);
	// the new graph: the old one copied, every new row's upper-level slots assigned from its level before the first batch
	out = std::make_unique<rxgpu_hnsw_device>();
	rxgpu_hnsw_device* h = out.get();
	h->M = M;
	h->maxM0 = 2 * M;
	const uint32_t s0 = 1 + 2 * M, s1 = 1 + M;
	const size_t capNodes = std::max<size_t>({size_t(ix->capacity), size_t(n), old ? old->cap_nodes : 0});
	h->h_levels = old ? old->h_levels : std::vector<int32_t>();
	h->h_upper_off = old ? old->h_upper_off : std::vector<long long>();
	uint64_t slots = old ? old->upper_slots : 0;
	for (uint32_t i = 0; i < nNew; ++i) {
		h->h_levels.push_back(lv[i]);
		h->h_upper_off.push_back((long long)slots);
		slots += uint64_t(lv[i]);
	}
	h->h_upper_off.push_back((long long)slots);
	h->upper_slots = slots;
	// keys of a batch: at most M per selected level of each row
	uint64_t keyCap = 1;
	{
		int32_t ml = old ? old->maxlevel : -1;
		uint64_t b0 = first;
		for (const uint64_t e : ends) {
			uint64_t cnt = 0;
			for (uint64_t r = b0; r < e; ++r) {
				cnt += ml < 0 ? 0 : uint64_t(std::min(lv[r - first], ml) + 1) * M;
			}
			keyCap = std::max(keyCap, cnt);
			ml = std::max(ml, lv[e - 1 - first]);
			b0 = e;
		}
	}
	cudaStream_t s = ix->stream;
	if (int rc = allocGraph(ix, h, capNodes, std::max<size_t>(1, slots) * s1)) {
		return rc;
	}
	DevBuf<uint64_t> keys, sorted, alt;
	DevBuf<uint32_t> seg;
	DevBuf<unsigned int> cnt32;         // next row, keys, segments, next segment
	DevBuf<unsigned long long> cnt64;   // distances, lists pruned
	DevBuf<float> qk;
	DevBuf<unsigned char> cubTmp;
	size_t cubBytes = 0;
	RX_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, cubBytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, int(keyCap), 0, 64, s));
	RX_CUDA(keys.ensure(keyCap));
	RX_CUDA(sorted.ensure(keyCap));
	RX_CUDA(alt.ensure(keyCap));
	RX_CUDA(seg.ensure(keyCap));
	RX_CUDA(cnt32.ensure(4));
	RX_CUDA(cnt64.ensure(2));
	RX_CUDA(cubTmp.ensure(std::max<size_t>(cubBytes, 1)));
	if (ix->metric == RXGPU_COS) {
		RX_CUDA(qk.ensure(n));
	}
	// the old graph, then empty lists and the levels / slots of the new rows
	if (old) {
		RX_CUDA(cudaMemcpyAsync(h->level0.p, old->level0.p, size_t(first) * s0 * 4, cudaMemcpyDeviceToDevice, s));
		if (old->upper_slots) {
			RX_CUDA(cudaMemcpyAsync(h->upper.p, old->upper.p, size_t(old->upper_slots) * s1 * 4, cudaMemcpyDeviceToDevice, s));
		}
	}
	RX_CUDA(cudaMemsetAsync(h->level0.p + size_t(first) * s0, 0, size_t(nNew) * s0 * 4, s));
	if (slots > (old ? old->upper_slots : 0)) {
		const uint64_t o = old ? old->upper_slots : 0;
		RX_CUDA(cudaMemsetAsync(h->upper.p + o * s1, 0, size_t(slots - o) * s1 * 4, s));
	}
	RX_CUDA(cudaMemcpyAsync(h->levels.p, h->h_levels.data(), size_t(n) * 4, cudaMemcpyHostToDevice, s));
	RX_CUDA(cudaMemcpyAsync(h->upper_off.p, h->h_upper_off.data(), (size_t(n) + 1) * 8, cudaMemcpyHostToDevice, s));
	RX_CUDA(cudaMemsetAsync(cnt64.p, 0, 16, s));
	if (ix->metric == RXGPU_COS) {
		hnsw_build_query_coefs<<<unsigned((n + 255) / 256), 256, 0, s>>>(ix->d_rows, ix->pitch, ix->dim, uint32_t(n), qk.p);
		RX_CUDA(cudaGetLastError());
	}
	h->h_upper_off.pop_back();  // the host copy keeps one offset per node
	const bool l2 = ix->metric == RXGPU_L2;
	const size_t smemI = insertSmem(ix->dim, ef_construction), smemL = linkSmem(ix->dim);
	void (*insertK)(BuildArgs) = l2 ? hnsw_build_insert<true> : hnsw_build_insert<false>;
	void (*linkK)(BuildArgs) = l2 ? hnsw_build_link<true> : hnsw_build_link<false>;
	RX_CUDA(raiseSmemCeilingOnce(insertK, ix->device, int(kBuildSmemBudget)));
	RX_CUDA(raiseSmemCeilingOnce(linkK, ix->device, int(kBuildSmemBudget)));
	cudaEvent_t ev[4];
	for (auto& e : ev) {
		RX_CUDA(cudaEventCreate(&e));
	}
	struct EventsGuard {
		cudaEvent_t* e;
		~EventsGuard() {
			for (int i = 0; i < 4; ++i) {
				cudaEventDestroy(e[i]);
			}
		}
	} evGuard{ev};
	BuildArgs b{};
	b.g = graphArgs(ix, h);
	b.g.visited = h->visited.p;
	b.g.vlog = h->vlog.p;
	b.g.next_query = cnt32.p;
	b.g.ef = ef_construction;
	b.qk = ix->metric == RXGPU_COS ? qk.p : nullptr;
	b.M = M;
	b.keys = keys.p;
	b.nkeys = cnt32.p + 1;
	b.nseg = cnt32.p + 2;
	b.next_seg = cnt32.p + 3;
	b.ndist = cnt64.p;
	b.npruned = cnt64.p + 1;
	b.sorted = sorted.p;
	b.alt = alt.p;
	b.seg = seg.p;
	int32_t ml = old ? old->maxlevel : -1;
	uint32_t ep = old ? old->enterpoint : 0;
	uint64_t b0 = first;
	for (const uint64_t e : ends) {
		uint64_t kc = 0;
		for (uint64_t r = b0; r < e; ++r) {
			kc += ml < 0 ? 0 : uint64_t(std::min(lv[r - first], ml) + 1) * M;
		}
		if (ml >= 0) {  // a batch on an empty graph is its first row alone: it has no neighbours yet
			b.g.maxlevel = ml;
			b.g.enterpoint = ep;
			b.b0 = uint32_t(b0);
			b.nb = uint32_t(e - b0);
			b.key_cap = uint32_t(kc);
			RX_CUDA(cudaMemsetAsync(cnt32.p, 0, 16, s));
			RX_CUDA(cudaMemsetAsync(keys.p, 0xFF, kc * 8, s));
			RX_CUDA(cudaEventRecord(ev[0], s));
			const unsigned gridI = unsigned(std::min<uint64_t>(h->slots / kHnswWarps, (b.nb + kHnswWarps - 1) / kHnswWarps));
			insertK<<<gridI, kHnswThreads, smemI, s>>>(b);
			RX_CUDA(cudaGetLastError());
			RX_CUDA(cudaEventRecord(ev[1], s));
			size_t tmpBytes = cubTmp.n;
			RX_CUDA(cub::DeviceRadixSort::SortKeys(cubTmp.p, tmpBytes, keys.p, sorted.p, int(kc), 0, 64, s));
			RX_CUDA(cudaEventRecord(ev[2], s));
			hnsw_build_heads<<<unsigned((kc + 255) / 256), 256, 0, s>>>(b);
			RX_CUDA(cudaGetLastError());
			const unsigned gridL = unsigned(std::min<uint64_t>(h->slots / kHnswWarps, (kc + kHnswWarps - 1) / kHnswWarps));
			linkK<<<gridL, kHnswThreads, smemL, s>>>(b);
			RX_CUDA(cudaGetLastError());
			RX_CUDA(cudaEventRecord(ev[3], s));
			RX_CUDA(cudaEventSynchronize(ev[3]));
			float ms[3] = {0.f, 0.f, 0.f};
			for (int i = 0; i < 3; ++i) {
				RX_CUDA(cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]));
			}
			st.search_select_ms += ms[0];
			st.sort_ms += ms[1];
			st.link_ms += ms[2];
			unsigned int nk = 0;
			RX_CUDA(cudaMemcpy(&nk, cnt32.p + 1, 4, cudaMemcpyDeviceToHost));
			st.reverse_links += nk;
		}
		if (ml < 0 || lv[e - 1 - first] > ml) {
			ml = lv[e - 1 - first];
			ep = uint32_t(e - 1);
		}
		st.batches += 1;
		b0 = e;
	}
	unsigned long long c64[2] = {0, 0};
	RX_CUDA(cudaMemcpyAsync(c64, cnt64.p, 16, cudaMemcpyDeviceToHost, s));
	RX_CUDA(cudaStreamSynchronize(s));
	st.rows = nNew;
	st.distances = c64[0];
	st.lists_pruned = c64[1];
	h->n = uint32_t(n);
	h->maxlevel = ml;
	h->enterpoint = ep;
	h->index_version = ix->version;
	if (old) {
		h->updates = old->updates;
	}
	return 0;
}

}  // namespace

extern "C" {

int rxgpu_hnsw_build_plan(uint32_t M, uint64_t first, uint64_t n, int32_t maxlevel, const int32_t* levels, uint64_t seed, int32_t* out_levels,
						  uint64_t* out_ends, uint64_t* out_nbatches) {
	if (int rc = checkPlanArgs(M, first, n, maxlevel, levels)) {
		return rc;
	}
	if (!out_nbatches) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		std::vector<int32_t> drawn;
		if (!levels) {
			drawn.resize(n - first);
			drawLevels(M, seed, n - first, drawn.data());
			levels = drawn.data();
		}
		std::vector<uint64_t> ends;
		planBatches(first, n, maxlevel, levels, ends);
		if (out_levels) {
			std::copy(levels, levels + (n - first), out_levels);
		}
		if (out_ends) {
			std::copy(ends.begin(), ends.end(), out_ends);
		}
		*out_nbatches = ends.size();
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_hnsw_build(rxgpu_index* ix, uint32_t M, uint32_t ef_construction, uint64_t first, const int32_t* levels, uint64_t seed,
					 rxgpu_hnsw_build_stats* stats) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	rxgpu_hnsw_device* old = ix->hnsw;
	const uint64_t n = ix->size;
	if (ef_construction < 4 || ef_construction > kMaxEf) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: efConstruction must be in [4, 1024]");
	}
	if (first != (old ? old->n : 0)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: first must equal the graph's node count");
	}
	if (old && (old->M != M || old->maxM0 != 2 * M)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: M differs from the graph's");
	}
	if (int rc = checkPlanArgs(M, first, n, old ? old->maxlevel : -1, levels)) {
		return rc;
	}
	if (old && ix->rows_touched_from < first) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: HNSW build: rows the graph covers were rewritten or moved since it was made (rows may only be appended)");
	}
	if (old && old->num_deleted) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: HNSW build: the graph has deleted nodes (their slots are reused by replace_deleted; the builder only appends)");
	}
	if (insertSmem(ix->dim, ef_construction) > kBuildSmemBudget || linkSmem(ix->dim) > kBuildSmemBudget) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW build: dimension/efConstruction combination exceeds the shared-memory budget");
	}
	rxgpu_hnsw_build_stats st{};
	if (n == first) {
		if (stats) {
			*stats = st;
		}
		return 0;
	}
	try {
		std::vector<int32_t> lv(levels ? std::vector<int32_t>(levels, levels + (n - first)) : std::vector<int32_t>(n - first));
		if (!levels) {
			drawLevels(M, seed, n - first, lv.data());
		}
		std::unique_ptr<rxgpu_hnsw_device> h;
		{
			std::unique_lock<std::mutex> lck;
			if (old) {
				lck = std::unique_lock<std::mutex>(old->mtx);
			}
			if (int rc = buildGraph(ix, old, M, ef_construction, lv, h, st)) {
				cudaGetLastError();  // a failed allocation stays the thread's last error: later calls must not see it
				return rc;
			}
		}
		if (old) {
			hnswRelease(old);
		}
		ix->hnsw = h.release();
		ix->rows_touched_from = ~0ull;
		if (stats) {
			*stats = st;
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_hnsw_export(const rxgpu_index* ix, uint64_t nnodes, const uint32_t* nodes, uint32_t* level0, int32_t* levels, int64_t* upper_offsets,
					  uint32_t* upper, rxgpu_hnsw_graph* info) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (int rc = checkGraph(ix)) {
		return rc;
	}
	const rxgpu_hnsw_device* h = ix->hnsw;
	if (info) {
		*info = rxgpu_hnsw_graph{h->n, h->M, h->maxM0, h->maxlevel, h->enterpoint, h->upper_slots, nullptr, nullptr, nullptr, nullptr};
	}
	if (!nodes && nnodes > h->n) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW export: more nodes than the graph holds");
	}
	if (nnodes == 0) {
		if (upper_offsets) {
			upper_offsets[0] = 0;
		}
		return 0;
	}
	try {
		const uint32_t s0 = 1 + h->maxM0, s1 = 1 + h->M;
		std::vector<uint64_t> idx(nnodes), slot;
		for (uint64_t i = 0; i < nnodes; ++i) {
			idx[i] = nodes ? nodes[i] : i;
			if (idx[i] >= h->n) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: HNSW export: node id out of range");
			}
		}
		int64_t off = 0;
		for (uint64_t i = 0; i < nnodes; ++i) {
			const int32_t l = h->h_levels[idx[i]];
			if (levels) {
				levels[i] = l;
			}
			if (upper_offsets) {
				upper_offsets[i] = off;
			}
			off += l;
			if (upper) {
				for (int32_t j = 0; j < l; ++j) {
					slot.push_back(uint64_t(h->h_upper_off[idx[i]]) + uint64_t(j));
				}
			}
		}
		if (upper_offsets) {
			upper_offsets[nnodes] = off;
		}
		cudaStream_t st = ix->stream;
		DevBuf<uint64_t> d_idx;
		DevBuf<uint32_t> d_out;
		auto gather = [&](const uint32_t* src, uint32_t width, const std::vector<uint64_t>& rows, uint32_t* dst) -> int {
			if (rows.empty()) {
				return 0;
			}
			RX_CUDA(d_idx.ensure(rows.size()));
			RX_CUDA(d_out.ensure(rows.size() * width));
			RX_CUDA(cudaMemcpyAsync(d_idx.p, rows.data(), rows.size() * 8, cudaMemcpyHostToDevice, st));
			const uint64_t total = rows.size() * width;
			hnsw_gather_lists<<<unsigned((total + 255) / 256), 256, 0, st>>>(src, width, d_idx.p, rows.size(), d_out.p);
			RX_CUDA(cudaGetLastError());
			RX_CUDA(cudaMemcpyAsync(dst, d_out.p, total * 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			return 0;
		};
		if (level0) {
			if (int rc = gather(h->level0.p, s0, idx, level0)) {
				return rc;
			}
		}
		if (upper) {
			if (int rc = gather(h->upper.p, s1, slot, upper)) {
				return rc;
			}
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

}  // extern "C"
