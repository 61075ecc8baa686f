// The device HNSW graph, the distance gather and the warp-level traversal steps shared by the search kernels (hnsw.cu) and the graph
// builder (hnsw_build.cu), and the host set-up of a graph both entry points use.
#pragma once
#include <algorithm>
#include <cstdlib>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "internal.h"

using namespace rxgpu;

namespace {

constexpr int kHnswWarps = 4;
constexpr int kHnswThreads = kHnswWarps * 32;
constexpr uint32_t kExpanded = 0x80000000u;
constexpr uint32_t kMaxEf = 1024;
constexpr uint32_t kVlogCap = 1u << 15;
constexpr int kMaxNeighbours = 64;  // maxM0 = 2*M; M <= 32 on the device path
constexpr uint32_t kHnswXCap = 4096;  // deleted nodes waiting for expansion (per query, in HBM), see the search kernel

struct HnswArgs {
	const float* rows;
	const float* norm_coefs;
	const uint32_t* level0;
	const int32_t* levels;
	const long long* upper_off;
	const uint32_t* upper;
	const float* queries;
	uint32_t* visited;  // [slots][words]
	uint32_t* vlog;     // [slots][kVlogCap]
	unsigned int* next_query;
	float* out_dist;    // [nq][k]
	uint32_t* out_idx;  // [nq][k]
	uint32_t* out_count;
	uint32_t* stats;    // [nq][2] or null
	const uint32_t* deleted;  // bitmap by internal id (MarkDelete, hnswalg.h:1303-1335) or null: the bare-bone search
	uint32_t* overflow;       // [nq] set when more than kHnswXCap deleted nodes were waiting at once (result not trustworthy)
	float* x_dist;            // [slots][kHnswXCap] deleted candidates of the slot's current query, ascending (only with `deleted`)
	uint32_t* x_id;
	uint32_t pitch, dim, n, l0_stride, up_stride;
	int maxlevel;
	uint32_t enterpoint;
	uint32_t nq, k, ef, words;
	uint32_t out_stride;  // entries per query in out_dist / out_idx: the caller's k (a.k may be clamped to the row count)
	// SQ8 (HierarchicalNSWImpl<uint8_t>): codes != null -> distances from the codes and corrective offsets, queries = qcodes
	const uint8_t* codes;
	const float* corr;
	const uint8_t* qcodes;  // [nq][code_pitch]
	const float* qcorr;     // [nq]
	const float* qcoef;     // [nq] query norm coefficient (1 unless Cosine)
	uint32_t code_pitch;
	float alpha2;
};

__device__ __forceinline__ float4 ldg4(const float4* p) {
	float4 v;
	asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
	return v;
}

// distances of `cnt` rows (ids in s_ids) to the query in sq4; results to s_d.  Per-row arithmetic == knn_scan_warp.
// SQ8: two rows per step (16 lanes each, 16 codes per load); dist = qcoef * (+-(alpha2 * int_dist + qcorr + corr[row]) * norm_coef[row])
// in the reference's operation order (hnswlib.h:147-165,192-197; hnswalg.h:801,935)
template <bool kIsL2>
__device__ __forceinline__ void warp_dists_sq8(const HnswArgs& a, const uint4* squ, const uint32_t* s_ids, uint32_t cnt, float* s_d, int lane,
											   float qcorr, float qcoef) {
	const uint32_t nch = a.code_pitch / 16;
	const int half = lane >> 4, hl = lane & 15;
	for (uint32_t g = 0; g < cnt; g += 2) {
		const uint32_t id = s_ids[min(g + half, cnt - 1)];
		const uint4* rp = reinterpret_cast<const uint4*>(a.codes + size_t(id) * a.code_pitch);
		unsigned acc = 0;
		for (uint32_t c = hl; c < nch; c += 16) {
			uint4 v;
			asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(rp + c));
			const uint4 q = squ[c];
			if constexpr (kIsL2) {
				unsigned d;
				d = __vabsdiffu4(v.x, q.x);
				acc = __dp4a(d, d, acc);
				d = __vabsdiffu4(v.y, q.y);
				acc = __dp4a(d, d, acc);
				d = __vabsdiffu4(v.z, q.z);
				acc = __dp4a(d, d, acc);
				d = __vabsdiffu4(v.w, q.w);
				acc = __dp4a(d, d, acc);
			} else {
				acc = __dp4a(v.x, q.x, acc);
				acc = __dp4a(v.y, q.y, acc);
				acc = __dp4a(v.z, q.z, acc);
				acc = __dp4a(v.w, q.w, acc);
			}
		}
#pragma unroll
		for (int off = 8; off > 0; off >>= 1) {
			acc += __shfl_xor_sync(0xffffffffu, acc, off);
		}
		if (hl == 0 && g + half < cnt) {
			float dist = __fadd_rn(__fadd_rn(__fmul_rn(a.alpha2, __uint2float_rn(acc)), qcorr), a.corr[id]);
			if (!kIsL2) {
				dist = -dist;
				if (a.norm_coefs != nullptr) {
					dist = __fmul_rn(dist, a.norm_coefs[id]);
				}
			}
			s_d[g + half] = __fmul_rn(qcoef, dist);
		}
	}
	__syncwarp();
}

template <bool kIsL2>
__device__ __forceinline__ void warp_dists(const HnswArgs& a, const float4* sq4, const uint32_t* s_ids, uint32_t cnt, float* s_d,
										   int lane, float qcorr = 0.f, float qcoef = 1.f) {
	if (a.codes != nullptr) {  // warp-uniform
		warp_dists_sq8<kIsL2>(a, reinterpret_cast<const uint4*>(sq4), s_ids, cnt, s_d, lane, qcorr, qcoef);
		return;
	}
	const float4* rows4 = reinterpret_cast<const float4*>(a.rows);
	const uint32_t pitch4 = a.pitch >> 2;
	const uint32_t nch = (a.dim + 127u) / 128u;
	for (uint32_t g = 0; g < cnt; g += 4) {
		uint32_t id[4];
		float acc[4];
#pragma unroll
		for (int r = 0; r < 4; ++r) {
			id[r] = s_ids[min(g + r, cnt - 1)];
			acc[r] = 0.f;
		}
#pragma unroll 2
		for (uint32_t c = 0; c < nch; ++c) {
			const uint32_t f4 = c * 32u + lane;
			float4 db[4];
#pragma unroll
			for (int r = 0; r < 4; ++r) {
				db[r] = f4 < pitch4 ? ldg4(rows4 + size_t(id[r]) * pitch4 + f4) : make_float4(0.f, 0.f, 0.f, 0.f);
			}
			const float4 q = sq4[f4];
#pragma unroll
			for (int r = 0; r < 4; ++r) {
				float s = acc[r];
				if constexpr (kIsL2) {
					float d;
					d = q.x - db[r].x;
					s = fmaf(d, d, s);
					d = q.y - db[r].y;
					s = fmaf(d, d, s);
					d = q.z - db[r].z;
					s = fmaf(d, d, s);
					d = q.w - db[r].w;
					s = fmaf(d, d, s);
				} else {
					s = fmaf(q.x, db[r].x, s);
					s = fmaf(q.y, db[r].y, s);
					s = fmaf(q.z, db[r].z, s);
					s = fmaf(q.w, db[r].w, s);
				}
				acc[r] = s;
			}
		}
#pragma unroll
		for (int r = 0; r < 4; ++r) {
			float v = acc[r];
#pragma unroll
			for (int off = 16; off > 0; off >>= 1) {
				v += __shfl_xor_sync(0xffffffffu, v, off);
			}
			float dist = kIsL2 ? v : -v;
			if (!kIsL2 && a.norm_coefs != nullptr) {
				dist *= a.norm_coefs[id[r]];
			}
			if (lane == 0 && g + r < cnt) {
				s_d[g + r] = dist;
			}
		}
	}
	__syncwarp();
}

// float4 slots of a query staged in shared memory: the dimension rounded up to whole 128-float chunks of warp_dists
__host__ __device__ __forceinline__ uint32_t hnsw_query_words(uint32_t dim) { return ((dim + 127u) / 128u) * 32u; }

// the neighbour list of `node` at `level`: [count, ids...]; upper_list_of for level >= 1
__device__ __forceinline__ const uint32_t* upper_list_of(const HnswArgs& a, uint32_t node, int level) {
	return a.upper + (size_t(a.upper_off[node]) + size_t(level - 1)) * a.up_stride;
}
__device__ __forceinline__ const uint32_t* list_of(const HnswArgs& a, uint32_t node, int level) {
	return level ? upper_list_of(a, node, level) : a.level0 + size_t(node) * a.l0_stride;
}

// the query q[0, dim) zero padded to dp4 float4 slots, thread t of nt
__device__ __forceinline__ void stage_query(float4* sq4, const float* q, uint32_t dim, uint32_t dp4, uint32_t t, uint32_t nt) {
	float* sq = reinterpret_cast<float*>(sq4);
	for (uint32_t c = t; c < dp4 * 4; c += nt) {
		sq[c] = c < dim ? q[c] : 0.f;
	}
}

// greedy descent through levels top .. stop + 1 (stop >= 0) from cur at distance curdist (hnswalg.h:799-827, :1781-1811): strict <,
// the first minimum wins
template <bool kIsL2>
__device__ __forceinline__ void greedy_descent(const HnswArgs& a, const float4* sq4, uint32_t& cur, float& curdist, int top, int stop, uint32_t* s_ids,
											   float* s_d, int lane, uint32_t& n_dist, uint32_t& n_hops, float qcorr = 0.f, float qcoef = 1.f) {
	for (int level = top; level > stop; --level) {
		bool changed = true;
		while (changed) {
			changed = false;
			const uint32_t* ll = upper_list_of(a, cur, level);
			const uint32_t cnt = min(ll[0], uint32_t(kMaxNeighbours));
			for (uint32_t j = lane; j < cnt; j += 32) {
				s_ids[j] = ll[1 + j];
			}
			__syncwarp();
			n_hops++;
			n_dist += cnt;
			if (cnt) {
				warp_dists<kIsL2>(a, sq4, s_ids, cnt, s_d, lane, qcorr, qcoef);
			}
			for (uint32_t j = 0; j < cnt; ++j) {
				const float d = s_d[j];
				if (d < curdist) {
					curdist = d;
					cur = s_ids[j];
					changed = true;
				}
			}
			__syncwarp();
		}
	}
}

// the batched visited test of list ll's first cnt neighbours: atomicOr on the warp's bitmap, the fresh ones to s_ids in neighbour order
// and to the visited log (entries past kVlogCap are counted, not kept).  Returns the number of fresh neighbours.
__device__ __forceinline__ uint32_t gather_fresh(const uint32_t* ll, uint32_t cnt, uint32_t* visited, uint32_t* vlog, uint32_t& vcount,
												 uint32_t* s_ids, int lane) {
	uint32_t ucnt = 0;
	for (uint32_t b = 0; b < cnt; b += 32) {
		const uint32_t j = b + lane;
		uint32_t nid = 0;
		bool fresh = false;
		if (j < cnt) {
			nid = ll[1 + j];
			const uint32_t bit = 1u << (nid & 31);
			fresh = !(atomicOr(&visited[nid >> 5], bit) & bit);
		}
		const unsigned fm = __ballot_sync(0xffffffffu, fresh);
		if (fresh) {
			const uint32_t o = ucnt + __popc(fm & ((1u << lane) - 1u));
			s_ids[o] = nid;
			if (vcount + o - ucnt < kVlogCap) {
				vlog[vcount + o - ucnt] = nid;
			}
		}
		ucnt += __popc(fm);
		vcount += __popc(fm);
	}
	__syncwarp();
	return ucnt;
}

// position of the first entry of l_id[0, size) without kExpanded, -1 when every entry is expanded
__device__ __forceinline__ int first_unexpanded(const uint32_t* l_id, uint32_t size, int lane) {
	int pos = -1;
	for (uint32_t b = 0; b < size && pos < 0; b += 32) {
		const uint32_t i = b + lane;
		const unsigned m = __ballot_sync(0xffffffffu, i < size && !(l_id[i] & kExpanded));
		if (m) {
			pos = int(b) + __ffs(m) - 1;
		}
	}
	return pos;
}

// how many i in [0, n) satisfy pred(i), warp-wide
template <class Pred>
__device__ __forceinline__ uint32_t warp_count(uint32_t n, int lane, Pred pred) {
	uint32_t c = 0;
	for (uint32_t b = 0; b < n; b += 32) {
		const uint32_t i = b + lane;
		c += __popc(__ballot_sync(0xffffffffu, i < n && pred(i)));
	}
	return c;
}

// (d, nid) into the sorted list dist / id at p < newsize, the entries from p on shifted right (highest chunk first) within
// [0, newsize): the last entry falls out when the list does not grow
__device__ __forceinline__ void list_insert(float* dist, uint32_t* id, uint32_t p, uint32_t newsize, float d, uint32_t nid, int lane) {
	for (int b = int((newsize - 1) / 32) * 32; b >= 0; b -= 32) {
		const uint32_t i = uint32_t(b) + lane;
		const bool mv = i > p && i < newsize;
		float td = 0.f;
		uint32_t ti = 0;
		if (mv) {
			td = dist[i - 1];
			ti = id[i - 1];
		}
		__syncwarp();
		if (mv) {
			dist[i] = td;
			id[i] = ti;
		}
		__syncwarp();
	}
	if (lane == 0) {
		dist[p] = d;
		id[p] = nid;
	}
	__syncwarp();
}

}  // namespace

// per-query state of a batched range search (hnsw.cu)
struct RangeQuery {
	unsigned int tail;        // matches found; past `cap` the region keeps the first cap and the query is answered again without a bound
	unsigned int begin, end;  // this level's frontier: region entries [begin, end)
	unsigned int unit0;       // the query's first CTA of this level's expansion (exclusive prefix over the chunk)
};

struct rxgpu_hnsw_device {
	uint32_t n = 0, M = 0, maxM0 = 0;
	int32_t maxlevel = -1;
	uint32_t enterpoint = 0;
	uint64_t index_version = 0;
	size_t cap_nodes = 0;      // nodes the arrays below are sized for
	uint64_t upper_slots = 0;  // used slots of `upper`
	uint64_t updates = 0;      // nodes rewritten in place by rxgpu_hnsw_update since the import
	std::vector<long long> h_upper_off;  // first upper-level slot of every node (host copy)
	std::vector<int32_t> h_levels;       // element_levels_ (host copy)
	DevBuf<uint32_t> level0;
	DevBuf<int32_t> levels;
	DevBuf<long long> upper_off;
	DevBuf<uint32_t> upper;
	// search scratch (guarded by mtx: one HNSW batch at a time per index; batches are internally parallel)
	std::mutex mtx;
	DevBuf<uint32_t> visited;
	DevBuf<uint32_t> vlog;
	DevBuf<unsigned int> counter;
	DevBuf<uint32_t> deleted;        // bitmap by internal id (MarkDelete)
	std::vector<uint32_t> h_deleted;
	uint32_t num_deleted = 0;
	DevBuf<uint32_t> overflow;       // [nq] per-query flag of the deleted-candidate list
	DevBuf<float> x_dist;            // [slots][kHnswXCap], allocated with the first tombstone
	DevBuf<uint32_t> x_id;
	// SearchRange scratch (the visited bitmaps are the search kernel's): per-query radius, chunk slot -> query, result/queue regions
	DevBuf<float> rg_radius, rg_dist;
	DevBuf<uint32_t> rg_qmap, rg_idx;
	DevBuf<RangeQuery> rg_state;
	DevBuf<unsigned int> rg_units;
	// staging of the host-pointer entry points (guarded by host_mtx; cudaMalloc per call would cost more than a small batch)
	std::mutex host_mtx;
	DevBuf<float> h_q, h_d;
	DevBuf<uint32_t> h_i, h_c, h_s;
	uint32_t slots = 0, words = 0;
};

// resident warps of the search kernels, one visited bitmap each: the search is a chain of dependent gathers, so occupancy hides its
// latency; 64 registers per thread allow 8 CTAs (32 warps) per SM.  RXGPU_HNSW_CTAS_PER_SM is a tuning aid.
inline uint32_t hnswSlots(const rxgpu_index* ix) {
	const char* e = std::getenv("RXGPU_HNSW_CTAS_PER_SM");
	const uint32_t perSm = e ? std::max(1, std::min(16, std::atoi(e))) : 8u;
	return uint32_t(ix->sm_count) * perSm * kHnswWarps;
}

namespace rxgpu {
// errLogic unless ix holds a graph made at its current version (hnsw.cu)
int checkGraph(const rxgpu_index* ix);
// sizes h's graph arrays for capNodes nodes, the upper slab for upperEntries words plus room for appended nodes, and sizes and zeroes
// the search scratch (hnsw.cu); h->M and h->maxM0 are set
int allocGraph(const rxgpu_index* ix, rxgpu_hnsw_device* h, size_t capNodes, size_t upperEntries);
}  // namespace rxgpu

namespace {
// the rows and graph h of ix, as the search, streaming and build kernels read them
inline HnswArgs graphArgs(const rxgpu_index* ix, const rxgpu_hnsw_device* h) {
	HnswArgs a{};
	a.rows = ix->d_rows;
	a.norm_coefs = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	a.level0 = h->level0.p;
	a.levels = h->levels.p;
	a.upper_off = h->upper_off.p;
	a.upper = h->upper.p;
	a.deleted = h->num_deleted ? h->deleted.p : nullptr;  // num_deleted_ == 0 -> the bare-bone search (hnswalg.h:1982)
	a.pitch = ix->pitch;
	a.dim = ix->dim;
	a.n = h->n;
	a.l0_stride = 1 + h->maxM0;
	a.up_stride = 1 + h->M;
	a.maxlevel = h->maxlevel;
	a.enterpoint = h->enterpoint;
	a.words = h->words;
	return a;
}
}  // namespace
