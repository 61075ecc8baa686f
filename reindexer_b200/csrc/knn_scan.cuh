// Brute-force float_vector scan kernels for sm_90a: distance (L2 / inner product / cosine) fused with top-k selection.
//
// Replaces the hot loop of hnswlib::BruteforceSearch::SearchKnn / SearchRange
// (cpp_src/core/index/float_vector/hnswlib/bruteforce.cc:103-127, :129-143) and the distance functors it calls
// (cpp_src/tools/distances/l2_dist.cc, ip_dist.cc; DistCalculator hnswlib/hnswlib.h:147-165).
//
// knn_scan_warp -- the HBM-bound exact fp32 kernel (QT <= 4 queries share one pass over the rows):
//   * rows are row-major in HBM with a 16-byte aligned pitch; one warp owns RW consecutive rows per step and streams them
//     with 128-bit coalesced, L1-bypassing loads (lane l reads float4 #l of every 128-float chunk), RW*CG loads in flight
//     per lane before the first use;
//   * the QT query vectors sit in shared memory, zero padded to a multiple of 128 floats, read as conflict-free float4;
//   * per-lane partial sums are combined with an xor-butterfly of warp shuffles (every lane ends with the full sum);
//     the per-row arithmetic sequence is identical for every row and every template variant, so bit-equal rows give
//     bit-equal distances (required by the tie rule);
//   * top-k is fused: each warp keeps, per query, its best k1 keys plus a 32-entry candidate buffer in shared memory and
//     a threshold; a row is looked at again only if it beats the threshold (expected k*ln(rows/k) times per warp), so no
//     distance ever goes back to HBM.  A CTA merges its warps' lists at the end and writes one list per query.
//   Algorithmic HBM bytes per launch: n*dim*4 (+ n*4 for cosine) + QT*dim*4 + lists.
// knn_merge_lists -- merges the per-CTA lists of one query into the final sorted top-k1 and gathers the labels.
// The kernels that are not templates (knn_merge_lists and the maintenance kernels) are defined in index.cu only: nvcc links device
// code per translation unit, so a non-template kernel defined in a header that two .cu files include is a multiple definition.
#pragma once
#include "common.cuh"

namespace rxgpu {

constexpr int kScanThreads = 256;
constexpr int kScanWarps = kScanThreads / 32;
constexpr int kCandBuf = 32;  // candidate buffer entries per (warp, query)
constexpr uint32_t kMaxFusedK1 = 256;   // results per scan round (k + 1 <= 256 is answered by a single pass)
constexpr uint32_t kMaxSearchK1 = 65536;  // larger k: ceil(k1 / 256) rounds

struct ScanArgs {
	const float* rows;        // [n][pitch] fp32
	const float* norm_coefs;  // [n] 1/||row|| (cosine) or nullptr
	const float* queries;     // [nq][dim] fp32 (device)
	uint64_t* lists;          // out: [gridDim.x][QT][k1] keys
	uint64_t* range_out;      // range mode: [range_cap] keys
	unsigned long long* range_count;
	uint64_t range_cap;
	uint32_t pitch;           // floats, multiple of 4
	uint32_t dim;
	uint32_t row_begin;       // scan rows [row_begin, row_end)
	uint32_t row_end;
	uint32_t nq;              // valid queries in this pass (<= QT)
	uint32_t k1;              // keys kept per list
	int mode;                 // ScanMode or kModeRange
	float bound;              // tie mode: dstar (dist <= bound); range mode: radius (dist < bound)
	const uint64_t* floor_keys;  // [nq] only keys ABOVE the floor compete (rounds of a k > 255 search), or nullptr
	// work-item mode (IVF list scans, QT = 1): CTA b scans rows [work[b].y, work[b].z) for query work[b].x with its own 8 warps and
	// writes list b; row_begin / row_end / nq are ignored (nq = 1)
	// key mode (knn_scan_warp<..., kKeysOut = true>, work-item mode only): no top-k; the key make_key(dist, row) of every scanned row goes
	// to lists[work[b].w + (row - work[b].y)] -- one fixed slot per (work item, row), no atomics
	const uint4* work;
	uint32_t nwork;
};
enum : int { kModeRange = 2 };

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
	float4 v;
	asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
	return v;
}

__host__ __device__ inline size_t scan_smem_bytes(int qt, uint32_t dim, uint32_t k1) {
	const size_t dp = size_t((dim + 127) / 128) * 128;
	const size_t m = size_t(k1) + kCandBuf;
	return qt * dp * 4 + size_t(kScanWarps) * qt * m * 8 + size_t(kScanWarps) * qt * 8 + size_t(kScanWarps) * qt * 4;
}

// in-place selection of the best `want` keys of arr[0, total) into arr[0, want) (ascending); one warp
__device__ __forceinline__ void warp_select(uint64_t* arr, uint32_t total, uint32_t want, int lane) {
	for (uint32_t r = 0; r < want; ++r) {
		uint64_t best = kKeyNone;
		uint32_t bpos = r;
		for (uint32_t i = r + lane; i < total; i += 32) {
			const uint64_t kx = arr[i];
			if (kx < best) {
				best = kx;
				bpos = i;
			}
		}
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) {
			const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
			const uint32_t op = __shfl_xor_sync(0xffffffffu, bpos, off);
			if (ok < best || (ok == best && op < bpos)) {
				best = ok;
				bpos = op;
			}
		}
		if (lane == 0 && bpos != r) {
			const uint64_t tmp = arr[r];
			arr[r] = best;
			arr[bpos] = tmp;
		}
		__syncwarp();
	}
}

template <int QT, int RW, int CG, bool kIsL2, bool kKeysOut = false>
__global__ void __launch_bounds__(kScanThreads, 2) knn_scan_warp(const ScanArgs a) {
	static_assert(RW * QT <= 32, "one lane per (row, query) result");
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const float* qsrc = a.queries;
	uint32_t row_begin = a.row_begin, row_end = a.row_end;
	uint32_t gfirst = blockIdx.x * kScanWarps + (threadIdx.x >> 5), gstride = gridDim.x * kScanWarps;
	uint32_t key_base = 0;  // key mode: slot of the work item's first row
	if (a.work != nullptr) {
		const uint4 w = a.work[blockIdx.x];
		qsrc += size_t(w.x) * a.dim;
		row_begin = w.y;
		row_end = w.z;
		gfirst = threadIdx.x >> 5;
		gstride = kScanWarps;
		if constexpr (kKeysOut) {
			key_base = w.w;
		}
	}
	const int lane = threadIdx.x & 31;
	const int warp = threadIdx.x >> 5;
	const uint32_t nch = (a.dim + 127u) / 128u;
	const uint32_t dp4 = nch * 32u;  // float4 per padded query
	const uint32_t pitch4 = a.pitch >> 2;
	const uint32_t m = a.k1 + kCandBuf;

	float4* sq4 = reinterpret_cast<float4*>(smem_raw);
	uint64_t* skeys = reinterpret_cast<uint64_t*>(smem_raw + size_t(QT) * dp4 * 16);
	uint64_t* sthr = skeys + size_t(kScanWarps) * QT * m;
	uint32_t* scnt = reinterpret_cast<uint32_t*>(sthr + kScanWarps * QT);

	{  // stage the queries, zero padded
		float* sq = reinterpret_cast<float*>(sq4);
		const uint32_t dp = dp4 * 4;
		for (uint32_t i = threadIdx.x; i < QT * dp; i += blockDim.x) {
			const uint32_t qi = i / dp, c = i - qi * dp;
			sq[i] = (qi < a.nq && c < a.dim) ? qsrc[size_t(qi) * a.dim + c] : 0.f;
		}
		for (uint32_t i = threadIdx.x; i < kScanWarps * QT * m; i += blockDim.x) {
			skeys[i] = kKeyNone;
		}
		if (threadIdx.x < kScanWarps * QT) {
			sthr[threadIdx.x] = kKeyNone;
			scnt[threadIdx.x] = 0;
		}
	}
	__syncthreads();

	uint64_t* wkeys = skeys + size_t(warp) * QT * m;
	uint64_t* wthr = sthr + warp * QT;
	uint32_t* wcnt = scnt + warp * QT;

	const float4* rows4 = reinterpret_cast<const float4*>(a.rows);
	const uint32_t nrows = row_end - row_begin;
	const uint32_t ngroups = (nrows + RW - 1) / RW;

	// lanes {r*QT + qi} hold the result of (row r, query qi)
	unsigned qpattern = 0;
#pragma unroll
	for (int r = 0; r < RW; ++r) {
		qpattern |= 1u << (r * QT);
	}
	const int my_r = lane / QT, my_q = lane % QT;
	const bool has_floor = a.floor_keys != nullptr;
	const uint64_t my_floor = has_floor && uint32_t(my_q) < a.nq ? a.floor_keys[my_q] : 0;

	for (uint32_t g = gfirst; g < ngroups; g += gstride) {
		float acc[RW][QT];
#pragma unroll
		for (int r = 0; r < RW; ++r) {
#pragma unroll
			for (int qi = 0; qi < QT; ++qi) {
				acc[r][qi] = 0.f;
			}
		}
		const uint32_t row0 = row_begin + g * RW;
		for (uint32_t c0 = 0; c0 < nch; c0 += CG) {
			float4 db[RW][CG];
#pragma unroll
			for (int r = 0; r < RW; ++r) {
#pragma unroll
				for (int j = 0; j < CG; ++j) {
					const uint32_t f4 = (c0 + j) * 32u + lane;
					const uint32_t row = row0 + r;
					if (row < row_end && f4 < pitch4) {
						db[r][j] = ldg_stream(rows4 + size_t(row) * pitch4 + f4);
					} else {
						db[r][j] = make_float4(0.f, 0.f, 0.f, 0.f);
					}
				}
			}
#pragma unroll
			for (int j = 0; j < CG; ++j) {
#pragma unroll
				for (int qi = 0; qi < QT; ++qi) {
					const float4 q = sq4[qi * dp4 + (c0 + j) * 32u + lane];
#pragma unroll
					for (int r = 0; r < RW; ++r) {
						float s = acc[r][qi];
						if constexpr (kIsL2) {
							float d;
							d = q.x - db[r][j].x;
							s = fmaf(d, d, s);
							d = q.y - db[r][j].y;
							s = fmaf(d, d, s);
							d = q.z - db[r][j].z;
							s = fmaf(d, d, s);
							d = q.w - db[r][j].w;
							s = fmaf(d, d, s);
						} else {
							s = fmaf(q.x, db[r][j].x, s);
							s = fmaf(q.y, db[r][j].y, s);
							s = fmaf(q.z, db[r][j].z, s);
							s = fmaf(q.w, db[r][j].w, s);
						}
						acc[r][qi] = s;
					}
				}
			}
		}
		// xor butterfly: every lane ends with the full sums, in a fixed order
		float mine = 0.f;
#pragma unroll
		for (int r = 0; r < RW; ++r) {
#pragma unroll
			for (int qi = 0; qi < QT; ++qi) {
				float v = acc[r][qi];
#pragma unroll
				for (int off = 16; off > 0; off >>= 1) {
					v += __shfl_xor_sync(0xffffffffu, v, off);
				}
				if (lane == r * QT + qi) {
					mine = v;
				}
			}
		}
		// epilogue: lane (r, qi) owns one distance
		const uint32_t row = row0 + my_r;
		const bool valid = lane < RW * QT && row < row_end && uint32_t(my_q) < a.nq;
		float dist = kIsL2 ? mine : -mine;  // DistCalculator::l2 / ::ip (hnswlib.h:192-197), alpha2 = 1, offsets 0
		if (!kIsL2 && a.norm_coefs != nullptr && valid) {
			dist *= a.norm_coefs[row];  // Cosine: hnswlib.h:160-161
		}
		if constexpr (kKeysOut) {
			if (valid) {
				a.lists[size_t(key_base) + (row - row_begin)] = make_key(dist, row);
			}
			continue;
		}
		if (a.mode == kModeRange) {
			const bool hit = valid && dist < a.bound;  // strict, bruteforce.cc:137
			const unsigned hm = __ballot_sync(0xffffffffu, hit);
			if (hm) {
				unsigned long long base = 0;
				if (lane == 0) {
					base = atomicAdd(a.range_count, (unsigned long long)__popc(hm));
				}
				base = __shfl_sync(0xffffffffu, base, 0);
				const unsigned long long pos = base + __popc(hm & ((1u << lane) - 1u));
				if (hit && pos < a.range_cap) {
					a.range_out[pos] = make_key(dist, row);
				}
			}
			continue;
		}
		uint64_t key;
		bool cand;
		if (a.mode == kModeTieRows) {
			key = (uint64_t(row) << 32) | float_ord(dist);
			cand = valid && dist <= a.bound;
		} else {
			key = make_key(dist, row);
			cand = valid;
		}
		cand = cand && key < wthr[my_q] && (!has_floor || key > my_floor);
		const unsigned cm = __ballot_sync(0xffffffffu, cand);
		if (cm) {
			const unsigned mineq = cm & (qpattern << my_q);
			if (cand) {
				const uint32_t pos = wcnt[my_q] + __popc(mineq & ((1u << lane) - 1u));
				wkeys[my_q * m + a.k1 + pos] = key;
			}
			__syncwarp();
			if (lane < QT) {
				wcnt[lane] += __popc(cm & (qpattern << lane));
			}
			__syncwarp();
#pragma unroll
			for (int qi = 0; qi < QT; ++qi) {
				const uint32_t c = wcnt[qi];
				if (c > uint32_t(kCandBuf - RW)) {  // the next step may add up to RW more
					warp_select(wkeys + qi * m, a.k1 + c, a.k1, lane);
					if (lane == 0) {
						wthr[qi] = wkeys[qi * m + a.k1 - 1];
						wcnt[qi] = 0;
					}
					__syncwarp();
				}
			}
		}
	}
	if (a.mode == kModeRange) {
		return;
	}
	if constexpr (!kKeysOut) {  // key mode wrote every key in the loop: no lists
		// flush the candidate buffers
#pragma unroll
		for (int qi = 0; qi < QT; ++qi) {
			const uint32_t c = wcnt[qi];
			if (c) {
				warp_select(wkeys + qi * m, a.k1 + c, a.k1, lane);
			}
		}
		__syncthreads();
		// CTA merge: warp w merges query w, w+8, ... over the 8 warp lists into warp 0's list region, then writes it out
		for (int qi = warp; qi < QT; qi += kScanWarps) {
			if (uint32_t(qi) >= a.nq) {
				continue;
			}
			// gather the 8 x k1 best keys behind warp 0's list of this query (its buffer region is free now) -- may not fit:
			// do a k1-round selection over the strided sources instead.
			uint64_t* out = a.lists + (size_t(blockIdx.x) * QT + qi) * a.k1;
			uint64_t last = 0;  // keys are unique except kKeyNone: select strictly increasing keys
			bool first = true;
			for (uint32_t r = 0; r < a.k1; ++r) {
				uint64_t best = kKeyNone;
				for (uint32_t i = lane; i < kScanWarps * a.k1; i += 32) {
					const uint32_t w = i / a.k1, j = i - w * a.k1;
					const uint64_t kx = skeys[(size_t(w) * QT + qi) * m + j];
					if ((first || kx > last) && kx < best) {
						best = kx;
					}
				}
#pragma unroll
				for (int off = 16; off > 0; off >>= 1) {
					const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
					best = ok < best ? ok : best;
				}
				if (lane == 0) {
					out[r] = best;
				}
				last = best;
				first = false;
				if (best == kKeyNone) {
					for (uint32_t rr = r + 1 + lane; rr < a.k1; rr += 32) {
						out[rr] = kKeyNone;
					}
					break;
				}
			}
		}
	}
}

// One CTA per query: k-way merge of nlists ASCENDING lists of k1 unique keys (kKeyNone padded) into the ascending top-k1, then decode
// and gather labels.  Thread t owns the heads of lists t, t+256, ...; a round is one block-wide min over the heads and the owner of
// the winner advances -- O(k1) rounds of O(1) work per thread.  Rounds of a k > 255 search write at out_offset and hand the last key
// to the next round as its floor.
constexpr int kMergeOwn = 4;  // lists per thread => nlists <= 1024
struct MergeArgs {
	const uint64_t* lists;  // [nlists][qt][k1]
	const uint64_t* labels;
	float* out_dist;       // [nq][out_stride]
	uint32_t* out_idx;     // [nq][out_stride]
	uint64_t* out_label;   // [nq][out_stride] (may be null)
	uint32_t* out_count;   // [nq]
	uint64_t* floor_out;   // [qt] last key written per query of this pass (kKeyNone when the lists ran dry), or null
	uint32_t nlists;
	uint32_t qt;           // list stride in queries
	uint32_t k1;           // keys per list = results of this round
	uint32_t q_offset;     // first output query of this pass
	uint32_t out_stride;   // result slots per query
	uint32_t out_offset;   // first slot of this round
	int mode;
	bool neg_zero;         // key_dist: zero distances come out as -0 (inner product, cosine)
};

// ---- one exact distance outside the scan ------------------------------------------------------------------------------------
// The per-row arithmetic of knn_scan_warp for every other exact fp32 distance (knn_rerank, the IVF coarse pass, the int8
// filter's seed and its bookkeepers): lane l accumulates float4 #l of every 128-float chunk, chunk after chunk, with sequential FMAs
// (x, y, z, w); an xor butterfly adds the lanes; then the sign (inner product, cosine) and the row's Cosine norm coefficient
// (norm_coefs != nullptr).  So a row's distance has the same bits on every path: the tie rule needs that, and the filter's bound list
// holds the exact scan's own distances.  R rows x Q queries at once: row r against the queries q4[r][0, Q) (zero padded to nch * 128
// floats), the R rows' loads of a chunk in flight together and each row read once for its Q queries.  Every lane returns every distance.
template <bool kIsL2, int R, int Q>
__device__ __forceinline__ void row_dists_warp(const float4* rows4, uint32_t pitch4, uint32_t nch, const uint32_t (&row)[R],
											   const float4* const (&q4)[R][Q], const float* norm_coefs, int lane, float (&dist)[R][Q]) {
	float s[R][Q];
#pragma unroll
	for (int r = 0; r < R; ++r) {
#pragma unroll
		for (int j = 0; j < Q; ++j) {
			s[r][j] = 0.f;
		}
	}
	for (uint32_t c = 0; c < nch; ++c) {
		const uint32_t f4 = c * 32u + lane;
		float4 v[R];
#pragma unroll
		for (int r = 0; r < R; ++r) {
			v[r] = f4 < pitch4 ? ldg_stream(rows4 + size_t(row[r]) * pitch4 + f4) : make_float4(0.f, 0.f, 0.f, 0.f);
		}
#pragma unroll
		for (int r = 0; r < R; ++r) {
#pragma unroll
			for (int j = 0; j < Q; ++j) {
				const float4 q = q4[r][j][f4];
				if constexpr (kIsL2) {
					float d;
					d = q.x - v[r].x;
					s[r][j] = fmaf(d, d, s[r][j]);
					d = q.y - v[r].y;
					s[r][j] = fmaf(d, d, s[r][j]);
					d = q.z - v[r].z;
					s[r][j] = fmaf(d, d, s[r][j]);
					d = q.w - v[r].w;
					s[r][j] = fmaf(d, d, s[r][j]);
				} else {
					s[r][j] = fmaf(q.x, v[r].x, s[r][j]);
					s[r][j] = fmaf(q.y, v[r].y, s[r][j]);
					s[r][j] = fmaf(q.z, v[r].z, s[r][j]);
					s[r][j] = fmaf(q.w, v[r].w, s[r][j]);
				}
			}
		}
	}
#pragma unroll
	for (int r = 0; r < R; ++r) {
		const float coef = !kIsL2 && norm_coefs != nullptr ? norm_coefs[row[r]] : 1.f;
#pragma unroll
		for (int j = 0; j < Q; ++j) {
			float t = s[r][j];
#pragma unroll
			for (int off = 16; off > 0; off >>= 1) {
				t += __shfl_xor_sync(0xffffffffu, t, off);
			}
			t = kIsL2 ? t : -t;
			if (!kIsL2 && norm_coefs != nullptr) {
				t *= coef;  // Cosine: hnswlib.h:160-161
			}
			dist[r][j] = t;
		}
	}
}
// one row against the query staged in sq4
template <bool kIsL2>
__device__ __forceinline__ float row_dist_warp(const float4* rows4, uint32_t pitch4, uint32_t nch, uint32_t row, const float4* sq4,
											   const float* norm_coefs, int lane) {
	const uint32_t r[1] = {row};
	const float4* const q[1][1] = {{sq4}};
	float d[1][1];
	row_dists_warp<kIsL2, 1, 1>(rows4, pitch4, nch, r, q, norm_coefs, lane, d);
	return d[0][0];
}

}  // namespace rxgpu
