// librxgpu: C ABI (include/rxgpu.h) over the sm_90a brute-force float_vector kernels.
// Host logic mirrors hnswlib::BruteforceSearch (cpp_src/core/index/float_vector/hnswlib/bruteforce.{h,cc}) and the
// search/select wrappers of HnswIndexBase<Map> (cpp_src/core/index/float_vector/hnsw_index.cc:160-288).
// There is no CPU fallback anywhere in this file: without a usable CUDA device every compute entry point fails.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/rxgpu.h"
#include "internal.h"
#include "../host/knn_select.h"
#include "knn_scan.cuh"
#include "knn_tc.cuh"

using namespace rxgpu;

namespace rxgpu {
thread_local std::string g_err;
thread_local rxgpu_search_stats g_stats{};
thread_local std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;
std::atomic<int> g_profile{0};

// ---------------------------------------------------------------------------------------------------------------- kernels
// knn_scan.cuh's kernels that are not templates: defined in this translation unit only, the IVF index (ivf.cu) launches them
// through the host functions declared in internal.h
__global__ void __launch_bounds__(256) knn_merge_lists(const MergeArgs a) {
	__shared__ uint64_t s_best[2][8];
	__shared__ uint64_t s_res[kMaxFusedK1];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t qi = blockIdx.x;
	uint32_t head[kMergeOwn];
	uint64_t hk[kMergeOwn];
#pragma unroll
	for (int j = 0; j < kMergeOwn; ++j) {
		const uint32_t l = threadIdx.x + j * 256u;
		head[j] = 0;
		hk[j] = l < a.nlists ? a.lists[(size_t(l) * a.qt + qi) * a.k1] : kKeyNone;
	}
	uint32_t count = 0;
	for (uint32_t r = 0; r < a.k1; ++r) {
		uint64_t best = hk[0];
#pragma unroll
		for (int j = 1; j < kMergeOwn; ++j) {
			best = hk[j] < best ? hk[j] : best;
		}
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) {
			const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
			best = ok < best ? ok : best;
		}
		if (lane == 0) {
			s_best[r & 1][warp] = best;
		}
		__syncthreads();
		uint64_t b = s_best[r & 1][0];
#pragma unroll
		for (int w = 1; w < 8; ++w) {
			const uint64_t o = s_best[r & 1][w];
			b = o < b ? o : b;
		}
		if (b == kKeyNone) {
			break;
		}
#pragma unroll
		for (int j = 0; j < kMergeOwn; ++j) {
			if (hk[j] == b) {  // keys are unique: exactly one owner
				const uint32_t l = threadIdx.x + j * 256u;
				++head[j];
				hk[j] = head[j] < a.k1 ? a.lists[(size_t(l) * a.qt + qi) * a.k1 + head[j]] : kKeyNone;
				s_res[r] = b;
			}
		}
		++count;
	}
	__syncthreads();
	const size_t ob = size_t(a.q_offset + qi) * a.out_stride + a.out_offset;
	for (uint32_t r = threadIdx.x; r < count; r += blockDim.x) {
		const uint64_t b = s_res[r];
		float dist;
		uint32_t idx;
		if (a.mode == kModeTieRows) {
			idx = uint32_t(b >> 32);
			dist = key_dist(uint32_t(b), a.neg_zero);
		} else {
			idx = uint32_t(b);
			dist = key_dist(uint32_t(b >> 32), a.neg_zero);
		}
		a.out_dist[ob + r] = dist;
		a.out_idx[ob + r] = idx;
		if (a.out_label) {
			a.out_label[ob + r] = a.labels[idx];
		}
	}
	if (threadIdx.x == 0) {
		a.out_count[a.q_offset + qi] = (a.out_offset ? a.out_count[a.q_offset + qi] : 0u) + count;
		if (a.floor_out) {
			a.floor_out[qi] = count == a.k1 ? s_res[count - 1] : kKeyNone;
		}
	}
}

// ---- maintenance kernels ------------------------------------------------------------------------------------------------
// 1/||row|| with the reference's shortcut (cpp_src/tools/normalize.cc:10-23); one warp per row, fixed summation order
__global__ void norm_coef_kernel(const float* rows, uint32_t pitch, uint32_t dim, uint32_t row_begin, uint32_t row_end, float* coefs) {
	const uint32_t row = row_begin + (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (row >= row_end) {
		return;
	}
	const float* p = rows + size_t(row) * pitch;
	float s = 0.f;
	for (uint32_t c = lane; c < dim; c += 32) {
		s = fmaf(p[c], p[c], s);
	}
#pragma unroll
	for (int off = 16; off > 0; off >>= 1) {
		s += __shfl_xor_sync(0xffffffffu, s, off);
	}
	if (lane == 0) {
		float k = 1.f;
		if (s > 0.f && fabsf(1.0f - s) > 0.00001f) {
			k = float(1.0 / double(__fsqrt_rn(s)));
		}
		coefs[row] = k;
	}
}

__global__ void synth_rows_kernel(float* rows, uint64_t* labels, uint32_t pitch, uint32_t dim, uint32_t dst_row, uint64_t seed,
								  uint64_t first_row, uint64_t n) {
	const uint64_t total = n * pitch;
	for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < total; i += uint64_t(gridDim.x) * blockDim.x) {
		const uint64_t r = i / pitch;
		const uint32_t c = uint32_t(i - r * pitch);
		rows[(dst_row + r) * pitch + c] = c < dim ? synth_value(seed, (first_row + r) * dim + c) : 0.f;
		if (c == 0) {
			labels[dst_row + r] = (first_row + r) << 32;
		}
	}
}

__global__ void synth_fill_kernel(float* out, uint64_t seed, uint64_t first_index, uint64_t count) {
	for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < count; i += uint64_t(gridDim.x) * blockDim.x) {
		out[i] = synth_value(seed, first_index + i);
	}
}

// norm coefficients of scattered rows (one warp per entry of dst), same arithmetic as norm_coef_kernel
__global__ void norm_coef_at_kernel(const float* rows, uint32_t pitch, uint32_t dim, const uint32_t* dst, uint32_t n, float* coefs) {
	const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (i >= n) {
		return;
	}
	const uint32_t row = dst[i];
	const float* p = rows + size_t(row) * pitch;
	float s = 0.f;
	for (uint32_t c = lane; c < dim; c += 32) {
		s = fmaf(p[c], p[c], s);
	}
#pragma unroll
	for (int off = 16; off > 0; off >>= 1) {
		s += __shfl_xor_sync(0xffffffffu, s, off);
	}
	if (lane == 0) {
		float k = 1.f;
		if (s > 0.f && fabsf(1.0f - s) > 0.00001f) {
			k = float(1.0 / double(__fsqrt_rn(s)));
		}
		coefs[row] = k;
	}
}

// staged rows [n][dim] -> rows[dst[i]][pitch] (zero padded) + labels
__global__ void scatter_rows_kernel(const float* staged, const uint32_t* dst, const uint64_t* staged_labels, uint32_t n, uint32_t dim,
									uint32_t pitch, float* rows, uint64_t* labels) {
	const uint32_t i = blockIdx.x;
	if (i >= n) {
		return;
	}
	const uint32_t d = dst[i];
	for (uint32_t c = threadIdx.x; c < pitch; c += blockDim.x) {
		rows[size_t(d) * pitch + c] = c < dim ? staged[size_t(i) * dim + c] : 0.f;
	}
	if (threadIdx.x == 0) {
		labels[d] = staged_labels[i];
	}
}
}  // namespace rxgpu

namespace {

thread_local std::vector<float> g_row_scratch;
thread_local std::vector<Hit> g_range_result;  // the last range search of this thread, retained for rxgpu_last_range_results()

int allocDevice(rxgpu_index* ix, uint64_t capacity, float** rows, uint64_t** labels, float** norms) {
	const size_t cap = capacity ? capacity : 1;
	RX_CUDA(cudaMalloc(reinterpret_cast<void**>(rows), cap * ix->pitch * sizeof(float)));
	RX_CUDA(cudaMalloc(reinterpret_cast<void**>(labels), cap * sizeof(uint64_t)));
	*norms = nullptr;
	if (ix->metric == RXGPU_COS) {
		RX_CUDA(cudaMalloc(reinterpret_cast<void**>(norms), cap * sizeof(float)));
	}
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------- launches
template <int QT, int RW, int CG, bool kKeysOut>
cudaError_t launchScanT(const rxgpu_index* ix, const ScanArgs& a, unsigned grid, size_t smem, cudaStream_t st) {
	if (smem > size_t(kScanSmemBudget)) {
		return cudaErrorInvalidValue;
	}
	if (ix->metric == RXGPU_L2) {
		auto kfn = knn_scan_warp<QT, RW, CG, true, kKeysOut>;
		if (const cudaError_t e = raiseSmemCeilingOnce(kfn, ix->device, kScanSmemBudget); e != cudaSuccess) {
			return e;
		}
		kfn<<<grid, kScanThreads, smem, st>>>(a);
	} else {
		auto kfn = knn_scan_warp<QT, RW, CG, false, kKeysOut>;
		if (const cudaError_t e = raiseSmemCeilingOnce(kfn, ix->device, kScanSmemBudget); e != cudaSuccess) {
			return e;
		}
		kfn<<<grid, kScanThreads, smem, st>>>(a);
	}
	return cudaGetLastError();
}

// kKeysOut: the key mode of the work-item scan (every scanned row's key to ScanArgs::lists), QT = 1 only
template <int QT, bool kKeysOut = false>
cudaError_t launchScanQ(const rxgpu_index* ix, const ScanArgs& a, uint32_t nch, unsigned* gridOut, cudaStream_t st, bool dryRun) {
	// chunk group CG divides nch; RW*CG float4 loads in flight per lane
	int cg, rw;
	if (nch % 6 == 0) {
		cg = 6, rw = 2;
	} else if (nch % 4 == 0) {
		cg = 4, rw = 2;
	} else if (nch % 3 == 0) {
		cg = 3, rw = 4;
	} else if (nch % 2 == 0) {
		cg = 2, rw = 4;
	} else {
		cg = 1, rw = 8;
	}
	const uint32_t nrows = a.row_end - a.row_begin;
	const uint32_t ngroups = (nrows + rw - 1) / rw;
	unsigned grid = std::min<unsigned>(unsigned(ix->sm_count) * 2u, std::max<unsigned>(1u, (ngroups + kScanWarps - 1) / kScanWarps));
	if (a.work != nullptr) {
		grid = a.nwork;  // one CTA per (query, inverted list)
	}
	*gridOut = grid;
	if (dryRun) {
		return cudaSuccess;
	}
	const size_t smem = scan_smem_bytes(QT, a.dim, a.k1);
	switch (cg) {
		case 6:
			return launchScanT<QT, 2, 6, kKeysOut>(ix, a, grid, smem, st);
		case 4:
			return launchScanT<QT, 2, 4, kKeysOut>(ix, a, grid, smem, st);
		case 3:
			return launchScanT<QT, 4, 3, kKeysOut>(ix, a, grid, smem, st);
		case 2:
			return launchScanT<QT, 4, 2, kKeysOut>(ix, a, grid, smem, st);
		default:
			return launchScanT<QT, 8, 1, kKeysOut>(ix, a, grid, smem, st);
	}
}

}  // namespace

namespace rxgpu {
cudaError_t launchScan(const rxgpu_index* ix, int qt, const ScanArgs& a, unsigned* gridOut, cudaStream_t st, bool dryRun, bool keysOut) {
	const uint32_t nch = (a.dim + 127u) / 128u;
	if (keysOut) {
		return launchScanQ<1, true>(ix, a, nch, gridOut, st, dryRun);
	}
	switch (qt) {
		case 4:
			return launchScanQ<4>(ix, a, nch, gridOut, st, dryRun);
		case 2:
			return launchScanQ<2>(ix, a, nch, gridOut, st, dryRun);
		default:
			return launchScanQ<1>(ix, a, nch, gridOut, st, dryRun);
	}
}

cudaError_t launchMergeLists(const MergeArgs& m, uint32_t nq, cudaStream_t st) {
	knn_merge_lists<<<nq, 256, 0, st>>>(m);
	return cudaGetLastError();
}

cudaError_t launchNormCoefs(const float* rows, uint32_t pitch, uint32_t dim, uint32_t row_begin, uint32_t row_end, float* coefs, cudaStream_t st) {
	const uint64_t n = row_end - row_begin;
	norm_coef_kernel<<<unsigned((n * 32 + 255) / 256), 256, 0, st>>>(rows, pitch, dim, row_begin, row_end, coefs);
	return cudaGetLastError();
}

cudaError_t scatterRows(const float* staged, const uint32_t* dst, const uint64_t* staged_labels, uint32_t n, uint32_t dim, uint32_t pitch,
						float* rows, uint64_t* labels, float* norms, cudaStream_t st) {
	scatter_rows_kernel<<<n, 128, 0, st>>>(staged, dst, staged_labels, n, dim, pitch, rows, labels);
	if (norms) {
		norm_coef_at_kernel<<<unsigned((uint64_t(n) * 32 + 255) / 256), 256, 0, st>>>(rows, pitch, dim, dst, n, norms);
	}
	return cudaGetLastError();
}
}  // namespace rxgpu

namespace {
int pickQueryTile(const rxgpu_index* ix, uint32_t nq) {
	uint32_t qt = ix->qt_override ? ix->qt_override : (nq >= 4 ? 4u : (nq >= 2 ? 2u : 1u));
	return qt >= 4 ? 4 : (qt >= 2 ? 2 : 1);
}

// Top-k1 rows per query under the total order (dist, internal index) -- or, in tie mode, the first k1 rows in internal
// order with dist <= bound.  Everything stays on the device; results land in d_out_* ([nq][k1]).  rowEnd < size: only the rows
// [0, rowEnd) (the seed of the staged thresholds).
int scanTopKExact(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t k1, int mode,
				  float bound, float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count,
				  uint32_t rowEnd = UINT32_MAX) {
	const uint32_t nrows = uint32_t(std::min<uint64_t>(rowEnd, ix->size));
	// k1 > kMaxFusedK1: rounds of <= kMaxFusedK1 results; a round only admits keys above the previous round's last key, so the
	// rounds concatenate to the top-k1 under the same total order (one pass over the rows per round)
	const uint32_t kr = std::min<uint32_t>(k1, kMaxFusedK1);
	const uint32_t rounds = (k1 + kr - 1) / kr;
	int qt = mode == kModeTieRows ? 1 : pickQueryTile(ix, nq);
	while (qt > 1 && scan_smem_bytes(qt, ix->dim, kr) > 100 * 1024) {
		qt /= 2;
	}
	if (scan_smem_bytes(qt, ix->dim, kr) > 100 * 1024) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: dimension/k combination exceeds the fused top-k shared-memory budget");
	}
	ScanArgs a{};
	a.rows = ix->d_rows;
	a.norm_coefs = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	a.pitch = ix->pitch;
	a.dim = ix->dim;
	a.row_begin = 0;
	a.row_end = nrows;
	a.k1 = kr;
	a.mode = mode;
	a.bound = bound;
	unsigned grid = 0;
	RX_CUDA(launchScan(ix, qt, a, &grid, st, true));
	if (grid > 256u * kMergeOwn) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: scan grid exceeds the merge fan-in");
	}
	RX_CUDA(ws.d_lists.ensure(size_t(grid) * qt * kr));
	a.lists = ws.d_lists.p;
	if (rounds > 1) {
		RX_CUDA(ws.d_floor.ensure(size_t(qt)));
	}
	for (uint32_t q0 = 0; q0 < nq; q0 += qt) {
		a.queries = d_queries + size_t(q0) * ix->dim;
		a.nq = std::min<uint32_t>(qt, nq - q0);
		for (uint32_t round = 0; round < rounds; ++round) {
			a.k1 = std::min(kr, k1 - round * kr);
			a.floor_keys = round ? ws.d_floor.p : nullptr;
			cudaEvent_t e0 = nullptr, e1 = nullptr;
			if (g_profile.load(std::memory_order_relaxed)) {
				RX_CUDA(cudaEventCreate(&e0));
				RX_CUDA(cudaEventCreate(&e1));
				RX_CUDA(cudaEventRecord(e0, st));
			}
			RX_CUDA(launchScan(ix, qt, a, &grid, st));
			if (e0) {
				RX_CUDA(cudaEventRecord(e1, st));
				g_prof_events.emplace_back(e0, e1);
			}
			MergeArgs m{};
			m.lists = ws.d_lists.p;
			m.labels = ix->d_labels;
			m.out_dist = d_out_dist;
			m.out_idx = d_out_idx;
			m.out_label = d_out_label;
			m.out_count = d_out_count;
			m.floor_out = rounds > 1 ? ws.d_floor.p : nullptr;
			m.nlists = grid;
			m.qt = qt;
			m.k1 = a.k1;
			m.q_offset = q0;
			m.out_stride = k1;
			m.out_offset = round * kr;
			m.mode = mode;
			m.neg_zero = ix->metric != RXGPU_L2;
			knn_merge_lists<<<a.nq, 256, 0, st>>>(m);
			RX_CUDA(cudaGetLastError());
			g_stats.launches += 2;
			g_stats.passes += 1;
		}
	}
	g_stats.query_tile = uint32_t(qt);
	const uint64_t perPass = uint64_t(nrows) * ix->dim * 4 + (ix->metric == RXGPU_COS ? uint64_t(nrows) * 4 : 0) +
							 uint64_t(qt) * ix->dim * 4 + uint64_t(qt) * kr * 12;
	g_stats.algorithmic_bytes += perPass * ((nq + qt - 1) / qt) * rounds;
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------- tensor-core filter
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
								   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
								   CUtensorMapFloatOOBfill);
EncodeTiledFn encodeTiled() {  // libcuda is never linked: resolve the one driver entry point we need at run time
	static EncodeTiledFn fn = [] {
		void* p = nullptr;
		cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
			cudaGetLastError();
			return EncodeTiledFn(nullptr);
		}
		return reinterpret_cast<EncodeTiledFn>(p);
	}();
	return fn;
}
// int8 query codes [rows][pitchBytes]: boxes of 128 bytes x boxRows, written to shared memory in the SWIZZLE_128B pattern
int makeCodeMap(CUtensorMap* m, void* base, uint64_t pitchBytes, uint64_t rows, uint32_t boxRows) {
	const cuuint64_t gdim[2] = {pitchBytes, rows};
	const cuuint64_t gstr[1] = {pitchBytes};
	const cuuint32_t box[2] = {uint32_t(kTcChunkK), boxRows};
	const cuuint32_t estr[2] = {1, 1};
	const CUresult r = encodeTiled()(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
									  CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: cuTensorMapEncodeTiled failed (" + std::to_string(int(r)) + ")");
	}
	return 0;
}

constexpr size_t kTcSmemLimit = 227 * 1024;  // the per-block opt-in maximum of sm_90
// per-query candidate list entries: the rows within the bound's window of the k1-th distance grow about in proportion to k1
// (config 1, int8 filter, candidates per query: k = 10: 1 620, k = 30: 3 820, k = 63: 6 880, k = 127: 12 000); 4096 is also the floor, so masses of near-duplicates still overflow to the
// exact scan instead of being re-ranked one list entry at a time
uint32_t tcCandCap(uint32_t k1) { return std::max<uint32_t>(4096u, 256u * k1); }
// per-query candidate list entries of a range batch: twice the matches the caller asked for (the bound's window of candidates that
// do not match), the KNN floor of 4096, and at most 2^18 (1 GiB of candidate rows for 1024 queries); a query with more candidates
// is answered by the exact range scan
uint32_t tcRangeCap(uint64_t max_out) { return uint32_t(std::max<uint64_t>(4096u, 2 * std::min<uint64_t>(max_out, 1u << 17))); }
// Staged thresholds (k1 > kTcMaxK1, DESIGN 3.2): the seed is the exact top-k1 of the first kStageSeedPerK1 * k1 rows, each stage's
// prefix is kStageRatio times the previous one, and a stage re-ranks about kStageRatio * k1 * (the bound's window factor) candidates
// per query.  Lists of kStageCapPerK1 * k1 entries, at most 2^18.  Chosen at config 1 on an H100 (DESIGN 3.2): r = 4 against 8 and
// 16, a seed of 2 k1 rows against 8 k1.
constexpr uint32_t kStageRatio = 4;
constexpr uint32_t kStageSeedPerK1 = 2;
constexpr uint32_t kStageCapPerK1 = 64;
uint32_t stageSeedRows(uint32_t k1) { return kStageSeedPerK1 * k1; }
uint32_t stageCandCap(uint32_t k1) { return std::min<uint32_t>(1u << 18, std::max<uint32_t>(4096u, kStageCapPerK1 * k1)); }

// knn_tc_filter<query block, cluster size>: one instantiation per wgmma N and per cluster shape (C = 1, 2, 4)
using TcKernel = void (*)(const CUtensorMap, const TcArgs);
int tcClusterIndex(uint32_t cluster) { return cluster == 4 ? 2 : cluster == 2 ? 1 : 0; }
TcKernel tcKernel(uint32_t nqb, uint32_t cluster) {
	static const TcKernel table[4][3] = {{knn_tc_filter<32, 1>, knn_tc_filter<32, 2>, knn_tc_filter<32, 4>},
										 {knn_tc_filter<64, 1>, knn_tc_filter<64, 2>, knn_tc_filter<64, 4>},
										 {knn_tc_filter<96, 1>, knn_tc_filter<96, 2>, knn_tc_filter<96, 4>},
										 {knn_tc_filter<128, 1>, knn_tc_filter<128, 2>, knn_tc_filter<128, 4>}};
	return table[nqb / 32 - 1][tcClusterIndex(cluster)];
}
// rxgpu_tc_diag: the diagnostic instantiation every filter launch of this process takes instead (0 = none), and its counters
std::atomic<int> g_tc_diag{0};
unsigned long long* g_tc_diag_buf = nullptr;
template <int kCluster>
TcKernel tcDiagKernelC(int mode) {
	static const TcKernel table[4] = {knn_tc_filter<128, kCluster, kTcDiagStamps>, knn_tc_filter<128, kCluster, kTcDiagNoRare>,
									  knn_tc_filter<128, kCluster, kTcDiagNoFetch>, knn_tc_filter<128, kCluster, kTcDiagNoTest>};
	return table[mode - 1];
}
TcKernel tcDiagKernel(int mode, uint32_t cluster) {
	return cluster == 4 ? tcDiagKernelC<4>(mode) : cluster == 2 ? tcDiagKernelC<2>(mode) : tcDiagKernelC<1>(mode);
}

uint32_t tcQueryBlock(uint32_t nq, uint32_t kchunks) {
	uint32_t nqb = std::min<uint32_t>(kTcMaxNq, (nq + 31u) & ~31u);
	while (nqb >= 32 && tc_smem_bytes(nqb, kchunks) > kTcSmemLimit) {
		nqb -= 32;
	}
	if (nqb < 32) {
		return 0;
	}
	const uint32_t blocks = (nq + nqb - 1) / nqb;
	return std::min(nqb, (((nq + blocks - 1) / blocks) + 31u) & ~31u);  // even out the blocks
}

// whether the filter serves a batch of nq queries at all (KNN and range search alike)
bool tcServes(const rxgpu_index* ix, uint32_t nq) {
	if (ix->tc_mode == 2 || !encodeTiled()) {
		return false;
	}
	if (tcQueryBlock(nq, (ix->dim + kTcChunkK - 1) / kTcChunkK) == 0) {
		return false;
	}
	// the s32 accumulator holds the exact code dot product while dim * 127^2 < 2^31; beyond 2048 dims the exact scan answers
	if (ix->dim > 2048) {
		return false;
	}
	return ix->tc_mode == 1 || (nq >= 64 && ix->size >= 100000);
}
bool tcEligible(const rxgpu_index* ix, uint32_t nq, uint32_t k1, int mode) {
	return mode == kModeTopK && k1 <= kTcStagedMaxK1 && tcServes(ix, nq);
}

// The shadow is rebuilt whole, sorted, once its dead and unsorted slots pass 1 / kShadowResortDiv of the slots; the slot capacity
// leaves that much room for appended rows beyond the row capacity.
constexpr uint32_t kShadowResortDiv = 8;

void releaseShadow(const rxgpu_index* ix) {
	cudaFree(ix->d_shadow);
	cudaFree(ix->d_rowc);
	cudaFree(ix->d_slot_row);
	cudaFree(ix->d_row_slot);
	cudaFree(ix->d_blockc);
	ix->d_shadow = nullptr;
	ix->d_rowc = nullptr;
	ix->d_slot_row = nullptr;
	ix->d_row_slot = nullptr;
	ix->d_blockc = nullptr;
}

// The slot order of a full build: the rows sorted by tc_sort_keys (stable, so ties keep the row order), slot s = the s-th row of it
int sortShadowSlots(const rxgpu_index* ix, cudaStream_t st, uint32_t n) {
	uint64_t *keys = nullptr, *keys_sorted = nullptr;
	uint32_t* vals = nullptr;
	void* temp = nullptr;
	size_t temp_bytes = 0;
	const int end_bit = ix->metric == RXGPU_L2 ? 64 : 32;  // IP and Cosine keys have no bucket
	cudaError_t e = cudaMalloc(&keys, size_t(n) * 8);
	if (e == cudaSuccess) e = cudaMalloc(&keys_sorted, size_t(n) * 8);
	if (e == cudaSuccess) e = cudaMalloc(&vals, size_t(n) * 4);
	if (e == cudaSuccess) {
		tc_sort_keys<<<unsigned((uint64_t(n) * 32 + 255) / 256), 256, 0, st>>>(ix->d_rows, ix->pitch, ix->dim, n,
																				 ix->metric == RXGPU_COS ? ix->d_norms : nullptr, ix->metric, keys, vals);
		e = cub::DeviceRadixSort::SortPairs(nullptr, temp_bytes, keys, keys_sorted, vals, ix->d_slot_row, n, 0, end_bit, st);
	}
	if (e == cudaSuccess) e = cudaMalloc(&temp, temp_bytes);
	if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys, keys_sorted, vals, ix->d_slot_row, n, 0, end_bit, st);
	if (e == cudaSuccess) {
		tc_invert_slots<<<(n + 255) / 256, 256, 0, st>>>(ix->d_slot_row, n, ix->d_row_slot);
		e = cudaGetLastError();
	}
	if (e == cudaSuccess) e = cudaStreamSynchronize(st);
	cudaFree(keys);
	cudaFree(keys_sorted);
	cudaFree(vals);
	cudaFree(temp);
	RX_CUDA(e);
	g_stats.launches += 3;
	return 0;
}

// int8 shadow + per-slot and per-block constants, brought up to date when the rows changed since the last large-batch search.  A full
// build sorts the rows into slots (knn_tc.cuh: tc_block_threshold); otherwise only what the mutations since then touched: rows
// rewritten in place are reconverted in their own slots, appended rows take new slots at the end, the slots of rows past the new size
// die.  The block constants are then recomputed over all slots.
int ensureShadow(const rxgpu_index* ix, cudaStream_t st) {
	std::lock_guard<std::mutex> lck(ix->tc_mtx);
	const uint32_t pitchQ = (ix->dim + kTcChunkK - 1) / kTcChunkK * kTcChunkK;
	if (!ix->d_shadow) {
		const size_t cap = (size_t(ix->capacity ? ix->capacity : 1) + kTcTileRows - 1) / kTcTileRows * kTcTileRows;  // whole tiles
		const size_t slotCap = (cap + cap / kShadowResortDiv + kTcTileRows - 1) / kTcTileRows * kTcTileRows;
		RX_CUDA(cudaMalloc(&ix->d_shadow, slotCap * pitchQ));
		RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ix->d_rowc), slotCap * sizeof(float4)));
		RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ix->d_slot_row), slotCap * sizeof(uint32_t)));
		RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ix->d_row_slot), cap * sizeof(uint32_t)));
		RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&ix->d_blockc), slotCap / 64 * 2 * sizeof(float4)));
		ix->pitch_q = pitchQ;
		ix->shadow_slot_cap = slotCap;
		ix->shadow_version = ~0ull;
		ix->shadow_dirty_all = true;
		ix->shadow_dirty.clear();
	}
	if (ix->shadow_version != ix->version) {
		const uint32_t size = uint32_t(ix->size), old = ix->shadow_rows;
		auto convert = [&](uint32_t b, uint32_t e) {
			const unsigned blocks = unsigned((uint64_t(e - b) * 32 + 255) / 256);
			tc_convert_rows<<<blocks, 256, 0, st>>>(ix->d_rows, ix->pitch, ix->dim, b, e, ix->d_row_slot, static_cast<unsigned char*>(ix->d_shadow),
													pitchQ / kTcChunkK, ix->metric == RXGPU_COS ? ix->d_norms : nullptr, ix->d_rowc);
			g_stats.launches += 1;
		};
		bool full = ix->shadow_dirty_all;
		if (!full) {
			const uint32_t kept = std::min(old, size), added = size - kept, gone = old - kept;
			uint64_t rewritten = 0;
			for (const auto& r : ix->shadow_dirty) {
				rewritten += r.first < kept ? std::min(r.second, kept) - r.first : 0u;
			}
			const uint64_t slots = uint64_t(ix->shadow_slots) + added;
			full = slots > ix->shadow_slot_cap ||
				   (uint64_t(ix->shadow_dead) + gone + ix->shadow_unsorted + added + rewritten) * kShadowResortDiv > slots;
			if (!full) {
				if (gone) {
					tc_kill_rows<<<(gone + 255) / 256, 256, 0, st>>>(kept, old, ix->d_row_slot, ix->d_slot_row, ix->d_rowc);
					g_stats.launches += 1;
				}
				for (const auto& r : ix->shadow_dirty) {
					if (r.first < kept) {
						convert(r.first, std::min(r.second, kept));
					}
				}
				if (added) {
					tc_assign_slots<<<(added + 255) / 256, 256, 0, st>>>(kept, size, ix->shadow_slots, ix->d_slot_row, ix->d_row_slot);
					g_stats.launches += 1;
					convert(kept, size);
				}
				ix->shadow_slots = uint32_t(slots);
				ix->shadow_dead += gone;
				ix->shadow_unsorted += uint32_t(added + rewritten);
			}
		}
		if (full) {
			if (size) {
				if (int rc = sortShadowSlots(ix, st, size)) {
					return rc;
				}
				convert(0, size);
			}
			ix->shadow_slots = size;
			ix->shadow_dead = 0;
			ix->shadow_unsorted = 0;
		}
		ix->shadow_rows = size;
		ix->shadow_dirty_all = false;
		ix->shadow_dirty.clear();
		// slots past the end, up to whole tiles, have all-zero constants (their codes are never tested: the kernel masks slots >= n)
		const uint32_t slots = ix->shadow_slots;
		const uint64_t padded = (uint64_t(slots) + kTcTileRows - 1) / kTcTileRows * kTcTileRows;
		RX_CUDA(cudaMemsetAsync(ix->d_rowc + slots, 0, size_t(padded - slots) * sizeof(float4), st));
		const uint32_t nblocks = uint32_t(padded / 64);
		if (nblocks) {
			tc_block_consts<<<(nblocks * 32 + 255) / 256, 256, 0, st>>>(ix->d_rowc, ix->d_slot_row, slots, nblocks,
																		   1.f - tc_l2eps(ix->dim), ix->metric, ix->d_blockc);
			g_stats.launches += 1;
		}
		RX_CUDA(cudaGetLastError());
		RX_CUDA(cudaStreamSynchronize(st));
		ix->shadow_version = ix->version;
	}
	return 0;
}

// Cluster shape by default (rxgpu_set_tensor_core_filter modes 0 and 1), measured on an H100 80GB HBM3 (700 W limit) at config 1
// (DESIGN 3.2): clusters of up to two, 69.0-69.5 k queries/s against 65.9-66.1 k with single CTAs and 65.5-66.1 k with clusters of
// four (30 clusters of four are resident: 120 CTAs instead of 128).  Multicast halves the row bytes the SMs read from L2, but a
// cluster waits for its slowest CTA; that pays only on long walks: at 2^22 rows the launch took 5.76 ms in clusters of two against
// 5.67 ms in single CTAs, so indexes below kTcClusterMinRows rows keep single CTAs.
constexpr uint32_t kTcClusterDefault = 2;
constexpr uint64_t kTcClusterMinRows = 1u << 23;
// The cluster size of a batch of nblocks query blocks: a cluster owns C consecutive blocks, and a block count that is not a multiple
// of C is padded with blocks of no valid queries, which walk every row for nothing.  The largest C <= cmax whose padding is at most
// one block, and fewer blocks than the batch has (one block is never paired with a padding block).
uint32_t tcClusterSize(uint32_t nblocks, uint32_t ntiles, uint32_t cmax) {
	for (uint32_t c = cmax; c > 1; c /= 2) {
		const uint32_t pad = (c - nblocks % c) % c;
		if (ntiles >= 2 && pad <= 1 && pad < nblocks) {
			return c;
		}
	}
	return 1;
}

// One batch of queries on the candidate filter: the int8 query codes and their tensor map, prepared once, and the launch shape.
struct TcBatch {
	uint32_t nq, nqb, cluster, ngroups, nqPad, kchunks, stages, queueSlots;
	int diag;     // the diagnostic instantiation taken (rxgpu_tc_diag), 0 = the production kernel
	size_t smem;  // tc_smem_bytes + the candidate queues
	int resident;
	TcKernel kfn;
	CUtensorMap mapQ;
};

int tcPrepare(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t candCap, TcBatch& b) {
	if (int rc = ensureShadow(ix, st)) {
		return rc;
	}
	const uint32_t pitchQ = ix->pitch_q, kchunks = pitchQ / kTcChunkK;
	const uint32_t nqb = tcQueryBlock(nq, kchunks);
	const uint32_t ntiles = uint32_t((ix->size + kTcTileRows - 1) / kTcTileRows);
	const uint32_t nblocks = (nq + nqb - 1) / nqb;
	const uint32_t cmax = ix->tc_cluster_max ? ix->tc_cluster_max : ix->size >= kTcClusterMinRows ? kTcClusterDefault : 1u;
	const uint32_t cluster = tcClusterSize(nblocks, ntiles, cmax);
	const uint32_t ngroups = (nblocks + cluster - 1) / cluster;
	const uint32_t nqPad = ngroups * cluster * nqb;
	RX_CUDA(ws.d_qcodes.ensure(size_t(nqPad) * pitchQ));
	RX_CUDA(ws.d_qc.ensure(nqPad));
	RX_CUDA(ws.d_qf.ensure(size_t(nqPad) * pitchQ));
	RX_CUDA(ws.d_tau.ensure(nqPad));
	RX_CUDA(ws.d_cand_count.ensure(nqPad));
	RX_CUDA(ws.d_cand_rows.ensure(size_t(nqPad) * candCap));
	RX_CUDA(ws.h_cand_count.ensure(nqPad));
	tc_prepare_queries<<<(nqPad * 32 + 255) / 256, 256, 0, st>>>(d_queries, nq, nqPad, ix->dim, pitchQ, ws.d_qcodes.p, ws.d_qc.p,
																 ws.d_qf.p);
	g_stats.launches += 1;
	RX_CUDA(cudaGetLastError());
	if (int rc = makeCodeMap(&b.mapQ, ws.d_qcodes.p, pitchQ, nqPad, nqb)) {
		return rc;
	}
	b.kfn = tcKernel(nqb, cluster);
	b.stages = tc_ring_stages(nqb, kchunks, kTcSmemLimit);
	b.queueSlots = tc_queue_slots(nqb, kchunks, b.stages, kTcSmemLimit);
	b.smem = tc_smem_bytes(nqb, kchunks, b.stages) + tc_queue_bytes(b.queueSlots);
	if (b.stages == 0 || b.queueSlots == 0) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: no room for the tensor-core filter's candidate queues");
	}
	b.diag = g_tc_diag.load();
	if (const int diag = b.diag) {
		if (nqb != 128) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: the diagnostic filter instantiations take query blocks of 128");
		}
		b.kfn = tcDiagKernel(diag, cluster);
	}
	RX_CUDA(raiseSmemCeilingOnce(b.kfn, ix->device, int(kTcSmemLimit)));
	cudaLaunchConfig_t cfg{};
	cfg.gridDim = dim3(unsigned(ix->sm_count) / cluster * cluster);
	cfg.blockDim = dim3(kTcThreads);
	cfg.dynamicSmemBytes = b.smem;
	cudaLaunchAttribute attr[1];
	attr[0].id = cudaLaunchAttributeClusterDimension;
	attr[0].val.clusterDim.x = cluster;
	attr[0].val.clusterDim.y = 1;
	attr[0].val.clusterDim.z = 1;
	cfg.attrs = attr;
	cfg.numAttrs = 1;
	b.resident = 0;  // GPC boundaries can strand SMs for clusters: ask how many fit at once
	RX_CUDA(cudaOccupancyMaxActiveClusters(&b.resident, b.kfn, &cfg));
	if (b.resident < 1) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: tensor-core filter kernel cannot be made resident");
	}
	b.nq = nq;
	b.nqb = nqb;
	b.cluster = cluster;
	b.ngroups = ngroups;
	b.nqPad = nqPad;
	b.kchunks = kchunks;
	return 0;
}

// The filter launches of a prepared batch over the shadow's slots [0, nrows), with the thresholds already in ws.d_tau: the rows whose certified
// lower bound is at or below the query's threshold tau go to ws.d_cand_rows[q][candCap], and ws.d_cand_count[q] counts them all (also
// past candCap: an overflowed list).  fixedTau: init_rows = UINT32_MAX keeps every row out of the bound list, so tau never moves
// (knn_tc.cuh header comment) and k1 is not used; otherwise tau tightens to the k1-th best exact distance of the bound list that
// the seed (tc_seed_slices, tc_seed_merge) filled.
int tcLaunch(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const TcBatch& b, uint32_t k1, uint32_t candCap, uint32_t nrows, bool fixedTau) {
	const uint32_t nq = b.nq, nqb = b.nqb, cluster = b.cluster, ngroups = b.ngroups, kchunks = b.kchunks, pitchQ = ix->pitch_q;
	const uint32_t ntiles = (nrows + kTcTileRows - 1) / kTcTileRows;
	const int resident = b.resident;
	const TcKernel kfn = b.kfn;
	const CUtensorMap mapQ = b.mapQ;
	RX_CUDA(cudaMemsetAsync(ws.d_cand_count.p, 0, size_t(b.nqPad) * 4, st));
	RX_CUDA(cudaGetLastError());
	cudaLaunchConfig_t cfg{};
	cfg.blockDim = dim3(kTcThreads);
	cfg.dynamicSmemBytes = b.smem;
	cfg.stream = st;
	cudaLaunchAttribute attr[1];
	attr[0].id = cudaLaunchAttributeClusterDimension;
	attr[0].val.clusterDim.x = cluster;
	attr[0].val.clusterDim.y = 1;
	attr[0].val.clusterDim.z = 1;
	cfg.attrs = attr;
	cfg.numAttrs = 1;
	TcArgs a{};
	a.shadow = static_cast<const unsigned char*>(ix->d_shadow);
	a.rowc = ix->d_rowc;
	a.slot_row = ix->d_slot_row;
	a.blockc = ix->d_blockc;
	a.qc = ws.d_qc.p;
	a.tau = ws.d_tau.p;
	a.ub_list = fixedTau ? nullptr : ws.d_ub_list.p;
	a.ub_lock = fixedTau ? nullptr : ws.d_ub_lock.p;
	a.init_rows = fixedTau ? UINT32_MAX : uint32_t(std::min<uint64_t>(ix->size, kTcInitRows));
	a.rows = ix->d_rows;
	a.norm_coefs = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	a.qf = ws.d_qf.p;
	a.pitch = ix->pitch;
	a.cand_rows = ws.d_cand_rows.p;
	a.cand_lb = fixedTau ? nullptr : ws.d_cand_lb.p;
	a.cand_count = ws.d_cand_count.p;
	a.cand_cap = candCap;
	a.n = nrows;
	a.dim = ix->dim;
	a.kchunks = kchunks;
	a.nq_total = nq;
	a.k1 = k1;
	a.metric = ix->metric;
	a.queue_slots = b.queueSlots;
	a.stages = b.stages;
	a.diag = g_tc_diag_buf;
	// One launch serves G = min(groups left, resident) query groups with W = resident / G tile walkers each, so the G clusters of a
	// walker read every row tile from HBM about once and from L2 otherwise (config 1: 8 blocks x 16 walkers = 128 CTAs, the shadow
	// streamed once per batch instead of once per block).  The grid never exceeds what is resident at once: a second wave would put
	// the clusters of one walker far apart in time and lose the L2 reuse.  Larger batches take several such launches.
	for (uint32_t g0 = 0; g0 < ngroups;) {
		const uint32_t groups = std::min<uint32_t>(ngroups - g0, uint32_t(resident));
		const uint32_t walkers = uint32_t(std::min<uint64_t>(uint32_t(resident) / groups, ntiles));
		cfg.gridDim = dim3(groups * walkers * cluster);
		a.q0 = g0 * cluster * nqb;
		a.groups = groups;
		cudaEvent_t e0 = nullptr, e1 = nullptr;
		if (g_profile.load(std::memory_order_relaxed)) {
			RX_CUDA(cudaEventCreate(&e0));
			RX_CUDA(cudaEventCreate(&e1));
			RX_CUDA(cudaEventRecord(e0, st));
		}
		RX_CUDA(cudaLaunchKernelEx(&cfg, kfn, mapQ, a));
		RX_CUDA(cudaGetLastError());
		if (e0) {
			RX_CUDA(cudaEventRecord(e1, st));
			g_prof_events.emplace_back(e0, e1);
		}
		g_stats.launches += 1;
		g_stats.passes += 1;
		const uint32_t served = std::min(groups * cluster * nqb, nq - a.q0);  // queries of this launch, padding excluded
		g_stats.algorithmic_bytes += uint64_t(nrows) * pitchQ + uint64_t(nrows) * sizeof(float4) + uint64_t(served) * pitchQ;
		g0 += groups;
	}
	g_stats.tc_cluster = cluster;
	g_stats.tc_kernel = 1 + uint32_t(b.diag);  // > 1: a diagnostic instantiation answered, the results are not to be used
	g_stats.query_tile = nqb * cluster;
	return 0;
}

// The candidate filter over a whole batch and all rows.  KNN (h_tau == nullptr): tau starts from the seed and tightens to the k1-th
// best exact distance of the bound list.  Range search: h_tau[q] = float_ord(radius) fixes tau.
int tcFilter(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t k1, uint32_t candCap,
			 const unsigned int* h_tau) {
	TcBatch b;
	if (int rc = tcPrepare(ix, ws, st, d_queries, nq, candCap, b)) {
		return rc;
	}
	if (h_tau) {
		RX_CUDA(cudaMemcpyAsync(ws.d_tau.p, h_tau, size_t(nq) * 4, cudaMemcpyHostToDevice, st));
	} else {
		RX_CUDA(ws.d_ub_list.ensure(size_t(b.nqPad) * kTcMaxK1));
		RX_CUDA(ws.d_ub_lock.ensure(b.nqPad));
		RX_CUDA(ws.d_cand_lb.ensure(size_t(b.nqPad) * candCap));
		RX_CUDA(ws.d_seed_part.ensure(size_t(nq) * kTcSeedSlices * kTcMaxK1));
		const size_t smem = tc_seed_smem_bytes(b.kchunks);
		RX_CUDA(raiseSmemCeilingOnce(tc_seed_slices, ix->device, int(tc_seed_smem_bytes(2048 / kTcChunkK))));
		tc_seed_slices<<<dim3((nq + kTcSeedQ - 1) / kTcSeedQ, kTcSeedSlices), 256, smem, st>>>(
			ix->d_rows, ix->pitch, b.kchunks, ix->metric == RXGPU_COS ? ix->d_norms : nullptr, uint32_t(std::min<uint64_t>(ix->size, kTcInitRows)),
			ws.d_qf.p, nq, k1, ix->metric, ws.d_seed_part.p);
		tc_seed_merge<<<(nq + 7) / 8, 256, 0, st>>>(ws.d_seed_part.p, nq, k1, ws.d_tau.p, ws.d_ub_list.p, ws.d_ub_lock.p);
		RX_CUDA(cudaGetLastError());
		g_stats.launches += 2;
	}
	return tcLaunch(ix, ws, st, b, k1, candCap, ix->shadow_slots, h_tau != nullptr);
}

// knn_rerank's range mode over the candidate lists: CTA b keeps the candidates of query q = qsel[b] (b without qsel) with
// dist < radius[q] as make_key(dist, row) in keys[q][cap], counted in nkeys[q] (zeroed here)
int rerankRange(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t nctas, const uint32_t* d_qsel,
				uint32_t cap, const float* d_radius, uint64_t* d_keys, unsigned int* d_nkeys) {
	RX_CUDA(cudaMemsetAsync(d_nkeys, 0, size_t(nq) * 4, st));
	const size_t rsmem = size_t((ix->dim + 127) / 128) * 512 + size_t(kScanWarps) * (1 + kCandBuf) * 8;
	const float* norms = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	if (ix->metric == RXGPU_L2) {
		RX_CUDA(raiseSmemCeilingOnce(knn_rerank<true>, ix->device, kScanSmemBudget));
		knn_rerank<true><<<nctas, kScanThreads, rsmem, st>>>(ix->d_rows, ix->pitch, ix->dim, norms, d_queries, ws.d_cand_rows.p, ws.d_cand_count.p,
															  cap, 1, nullptr, d_qsel, nullptr, d_radius, d_keys, d_nkeys);
	} else {
		RX_CUDA(raiseSmemCeilingOnce(knn_rerank<false>, ix->device, kScanSmemBudget));
		knn_rerank<false><<<nctas, kScanThreads, rsmem, st>>>(ix->d_rows, ix->pitch, ix->dim, norms, d_queries, ws.d_cand_rows.p, ws.d_cand_count.p,
															   cap, 1, nullptr, d_qsel, nullptr, d_radius, d_keys, d_nkeys);
	}
	RX_CUDA(cudaGetLastError());
	g_stats.launches += 1;
	return 0;
}

// KNN with k1 in (kTcMaxK1, kTcStagedMaxK1] on the filter, by staged exact thresholds (knn_tc.cuh, DESIGN 3.2).  Output = the same
// top-k1 under (dist, internal index) as scanTopKExact, bit for bit.  The thresholds stay on the device between the stages; the batch
// synchronises with the host once, at the end.
int scanTopKStaged(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t k1,
				   float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count) {
	const uint32_t cap = stageCandCap(k1);
	const uint32_t size = uint32_t(ix->size);
	TcBatch b;
	if (int rc = tcPrepare(ix, ws, st, d_queries, nq, cap, b)) {
		return rc;
	}
	RX_CUDA(ws.d_radius.ensure(nq));
	RX_CUDA(ws.d_range_n.ensure(nq));
	RX_CUDA(ws.d_range.ensure(size_t(nq) * cap));
	RX_CUDA(ws.d_stage_status.ensure(nq));
	RX_CUDA(ws.h_stage_status.ensure(nq));
	RX_CUDA(ws.d_reranked.ensure(1));
	RX_CUDA(ws.h_reranked.ensure(1));
	RX_CUDA(cudaMemsetAsync(ws.d_reranked.p, 0, sizeof(unsigned long long), st));
	// the seed: the exact top-k1 of a prefix, in the output arrays (the last stage or the exact scan overwrites every query's)
	uint32_t rows = std::min(size, stageSeedRows(k1));
	if (int rc = scanTopKExact(ix, ws, st, d_queries, nq, k1, kModeTopK, 0.f, d_out_dist, d_out_idx, d_out_label, d_out_count, rows)) {
		return rc;
	}
	knn_seed_tau<<<(nq + 255) / 256, 256, 0, st>>>(d_out_dist, d_out_count, k1, nq, ws.d_tau.p, ws.d_radius.p, ws.d_stage_status.p);
	RX_CUDA(cudaGetLastError());
	g_stats.launches += 1;
	SelectArgs s{};
	s.keys = ws.d_range.p;
	s.nkeys = ws.d_range_n.p;
	s.cand_count = ws.d_cand_count.p;
	s.labels = ix->d_labels;
	s.cap = cap;
	s.k1 = k1;
	s.mode = kModeTopK;
	s.tau = ws.d_tau.p;
	s.radius = ws.d_radius.p;
	s.status = ws.d_stage_status.p;
	s.reranked = ws.d_reranked.p;
	s.out_dist = d_out_dist;
	s.out_idx = d_out_idx;
	s.out_label = d_out_label;
	s.out_count = d_out_count;
	s.neg_zero = ix->metric != RXGPU_L2;
	// the stages filter growing prefixes of the shadow's slots (sorted, so not the seed's rows); the last one covers every slot
	const uint32_t slots = ix->shadow_slots;
	uint32_t prefix = rows;
	do {
		prefix = uint32_t(std::min<uint64_t>(slots, uint64_t(prefix) * kStageRatio));
		if (int rc = tcLaunch(ix, ws, st, b, k1, cap, prefix, true)) {
			return rc;
		}
		if (int rc = rerankRange(ix, ws, st, d_queries, nq, nq, nullptr, cap, ws.d_radius.p, ws.d_range.p, ws.d_range_n.p)) {
			return rc;
		}
		s.last = prefix == slots;
		knn_select_topk<<<nq, kSelThreads, 0, st>>>(s);
		RX_CUDA(cudaGetLastError());
		g_stats.launches += 1;
	} while (prefix < slots);
	RX_CUDA(cudaMemcpyAsync(ws.h_cand_count.p, ws.d_cand_count.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(ws.h_stage_status.p, ws.d_stage_status.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(ws.h_reranked.p, ws.d_reranked.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	for (uint32_t q = 0; q < nq; ++q) {
		if (ws.h_stage_status.p[q]) {  // an overflowed last list, a non-finite threshold or too few survivors: the exact scan answers
			g_stats.tc_fallbacks += 1;
			ws.h_cand_count.p[q] = UINT32_MAX;  // and no tie replay reads its list
			if (int rc = scanTopKExact(ix, ws, st, d_queries + size_t(q) * ix->dim, 1, k1, kModeTopK, 0.f, d_out_dist + size_t(q) * k1,
									   d_out_idx + size_t(q) * k1, d_out_label ? d_out_label + size_t(q) * k1 : nullptr, d_out_count + q)) {
				return rc;
			}
		}
	}
	ws.tc_lists_valid = true;
	ws.tc_lists_nq = nq;
	ws.tc_lists_cap = cap;
	ws.tc_lists_version = ix->version;
	g_stats.tc_used = 1;
	g_stats.tc_candidates = *ws.h_reranked.p;
	g_stats.algorithmic_bytes += *ws.h_reranked.p * (uint64_t(ix->dim) * 4 + 4);
	return 0;
}

// Large batches: approximate int8 tensor-core scores with a certified error bound select the candidates, the exact fp32 routine
// re-ranks them.  Output = the same top-k1 under (dist, internal index) as scanTopKExact, bit for bit.
int scanTopKTensorCore(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t k1,
					   float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count) {
	const uint32_t candCap = tcCandCap(k1);
	if (int rc = tcFilter(ix, ws, st, d_queries, nq, k1, candCap, nullptr)) {
		return rc;
	}
	RX_CUDA(ws.d_lists.ensure(size_t(nq) * k1));
	// exact re-rank of the candidates under the final thresholds with the arithmetic of knn_scan_warp, then decode + labels
	const size_t rsmem = size_t((ix->dim + 127) / 128) * 512 + size_t(kScanWarps) * (k1 + kCandBuf) * 8;
	const float* norms = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	unsigned long long* gathered = g_tc_diag.load() ? g_tc_diag_buf + kTcDgGathered : nullptr;
	if (ix->metric == RXGPU_L2) {
		RX_CUDA(raiseSmemCeilingOnce(knn_rerank<true>, ix->device, kScanSmemBudget));
		knn_rerank<true><<<nq, kScanThreads, rsmem, st>>>(ix->d_rows, ix->pitch, ix->dim, norms, d_queries, ws.d_cand_rows.p,
														   ws.d_cand_count.p, candCap, k1, ws.d_lists.p, nullptr, nullptr, nullptr,
														   nullptr, nullptr, ws.d_cand_lb.p, ws.d_tau.p, gathered);
	} else {
		RX_CUDA(raiseSmemCeilingOnce(knn_rerank<false>, ix->device, kScanSmemBudget));
		knn_rerank<false><<<nq, kScanThreads, rsmem, st>>>(ix->d_rows, ix->pitch, ix->dim, norms, d_queries, ws.d_cand_rows.p,
															ws.d_cand_count.p, candCap, k1, ws.d_lists.p, nullptr, nullptr, nullptr,
															nullptr, nullptr, ws.d_cand_lb.p, ws.d_tau.p, gathered);
	}
	MergeArgs m{};
	m.lists = ws.d_lists.p;
	m.labels = ix->d_labels;
	m.out_dist = d_out_dist;
	m.out_idx = d_out_idx;
	m.out_label = d_out_label;
	m.out_count = d_out_count;
	m.nlists = 1;
	m.qt = nq;
	m.k1 = k1;
	m.q_offset = 0;
	m.out_stride = k1;
	m.out_offset = 0;
	m.mode = kModeTopK;
	m.neg_zero = ix->metric != RXGPU_L2;
	knn_merge_lists<<<nq, 256, 0, st>>>(m);
	RX_CUDA(cudaGetLastError());
	g_stats.launches += 2;
	// a query whose candidate list overflowed (pathological data, e.g. masses of near-duplicates) is answered by the exact scan
	RX_CUDA(cudaMemcpyAsync(ws.h_cand_count.p, ws.d_cand_count.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	uint64_t cands = 0;
	for (uint32_t q = 0; q < nq; ++q) {
		cands += std::min<unsigned>(ws.h_cand_count.p[q], candCap);
		if (ws.h_cand_count.p[q] > candCap) {
			g_stats.tc_fallbacks += 1;
			if (int rc = scanTopKExact(ix, ws, st, d_queries + size_t(q) * ix->dim, 1, k1, kModeTopK, 0.f, d_out_dist + size_t(q) * k1,
									   d_out_idx + size_t(q) * k1, d_out_label ? d_out_label + size_t(q) * k1 : nullptr, d_out_count + q)) {
				return rc;
			}
		}
	}
	ws.tc_lists_valid = true;
	ws.tc_lists_nq = nq;
	ws.tc_lists_cap = candCap;
	ws.tc_lists_version = ix->version;
	g_stats.tc_used = 1;
	g_stats.tc_candidates = cands;
	g_stats.algorithmic_bytes += cands * (uint64_t(ix->dim) * 4 + 4);
	return 0;
}

}  // namespace

namespace rxgpu {
int scanTopK(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t k1, int mode, float bound,
			 float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count) {
	if (tcEligible(ix, nq, k1, mode) && k1 > kTcMaxK1) {
		return scanTopKStaged(ix, ws, st, d_queries, nq, k1, d_out_dist, d_out_idx, d_out_label, d_out_count);
	}
	if (tcEligible(ix, nq, k1, mode)) {
		return scanTopKTensorCore(ix, ws, st, d_queries, nq, k1, d_out_dist, d_out_idx, d_out_label, d_out_count);
	}
	if (mode == kModeTopK) {
		ws.tc_lists_valid = false;
	}
	return scanTopKExact(ix, ws, st, d_queries, nq, k1, mode, bound, d_out_dist, d_out_idx, d_out_label, d_out_count);
}

int setRowAt(rxgpu_index* ix, uint32_t idx, uint64_t label, const float* vec) {
	if (idx > ix->size || (idx == ix->size && ix->size >= ix->capacity)) {
		return fail(RXGPU_ERR_LOGIC, "The number of elements exceeds the specified limit\n");
	}
	const uint32_t other = ix->dict.find(label);
	if (other != LabelMap::kNotFound && other != idx) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: label already belongs to another row");
	}
	RX_CUDA(ix->st_rows.ensure(ix->pitch));
	RX_CUDA(cudaMemsetAsync(ix->st_rows.p, 0, size_t(ix->pitch) * 4, ix->stream));
	RX_CUDA(cudaMemcpyAsync(ix->st_rows.p, vec, size_t(ix->dim) * 4, cudaMemcpyHostToDevice, ix->stream));
	RX_CUDA(cudaMemcpyAsync(ix->d_rows + size_t(idx) * ix->pitch, ix->st_rows.p, size_t(ix->pitch) * 4, cudaMemcpyDeviceToDevice, ix->stream));
	RX_CUDA(cudaMemcpyAsync(ix->d_labels + idx, &label, 8, cudaMemcpyHostToDevice, ix->stream));
	if (ix->metric == RXGPU_COS) {
		norm_coef_kernel<<<1, 32, 0, ix->stream>>>(ix->d_rows, ix->pitch, ix->dim, idx, idx + 1, ix->d_norms);
		RX_CUDA(cudaGetLastError());
	}
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	if (idx < ix->size) {
		if (ix->h_labels[idx] != label) {
			ix->dict.erase(ix->h_labels[idx]);
		}
		ix->h_labels[idx] = label;
	} else {
		ix->h_labels.push_back(label);
		ix->size += 1;
	}
	ix->dict.put(label, idx);
	if (ix->flags & RXGPU_FLAG_HOST_MIRROR) {
		std::memcpy(ix->h_rows.data() + size_t(idx) * ix->dim, vec, ix->dim * sizeof(float));
	}
	ix->touchRows(idx, uint64_t(idx) + 1);
	ix->version++;
	return 0;
}

int tieRowsAfterScan(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nsel, const uint32_t* sel,
					 const float* dstar, uint32_t k, float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count) {
	if (nsel == 0) {
		return 0;
	}
	bool fromLists = ws.tc_lists_valid && ws.tc_lists_version == ix->version && k < kTcStagedMaxK1;
	for (uint32_t i = 0; fromLists && i < nsel; ++i) {  // a query whose list overflowed was answered by the exact scan: no list
		fromLists = sel[i] < ws.tc_lists_nq && ws.h_cand_count.p[sel[i]] <= ws.tc_lists_cap;
	}
	if (!fromLists) {
		for (uint32_t i = 0; i < nsel; ++i) {
			if (int rc = scanTopKExact(ix, ws, st, d_queries + size_t(sel[i]) * ix->dim, 1, k, kModeTieRows, dstar[i], d_out_dist + size_t(i) * k,
									   d_out_idx + size_t(i) * k, d_out_label ? d_out_label + size_t(i) * k : nullptr, d_out_count + i)) {
				return rc;
			}
		}
		g_stats.tie_replays += nsel;
		return 0;
	}
	RX_CUDA(ws.d_sel.ensure(nsel));
	RX_CUDA(cudaMemcpyAsync(ws.d_sel.p, sel, size_t(nsel) * 4, cudaMemcpyHostToDevice, st));
	if (k > kTcMaxK1) {
		// the lists of staged thresholds: the candidates with dist <= d* (range mode, radius = the next float above d*), then the first k
		// of them in internal order (knn_select_topk on row-major keys)
		const uint32_t nq = ws.tc_lists_nq, cap = ws.tc_lists_cap;
		std::vector<float> rad(nq, -INFINITY);
		for (uint32_t i = 0; i < nsel; ++i) {
			rad[sel[i]] = nextafterf(dstar[i], INFINITY);
		}
		RX_CUDA(ws.d_radius.ensure(nq));
		RX_CUDA(ws.d_range_n.ensure(nq));
		RX_CUDA(ws.d_range.ensure(size_t(nq) * cap));
		RX_CUDA(cudaMemcpyAsync(ws.d_radius.p, rad.data(), size_t(nq) * 4, cudaMemcpyHostToDevice, st));
		if (int rc = rerankRange(ix, ws, st, d_queries, nq, nsel, ws.d_sel.p, cap, ws.d_radius.p, ws.d_range.p, ws.d_range_n.p)) {
			return rc;
		}
		SelectArgs s{};
		s.keys = ws.d_range.p;
		s.nkeys = ws.d_range_n.p;
		s.cand_count = ws.d_cand_count.p;
		s.qsel = ws.d_sel.p;
		s.labels = ix->d_labels;
		s.cap = cap;
		s.k1 = k;
		s.mode = kModeTieRows;
		s.out_dist = d_out_dist;
		s.out_idx = d_out_idx;
		s.out_label = d_out_label;
		s.out_count = d_out_count;
		s.neg_zero = ix->metric != RXGPU_L2;
		knn_select_topk<<<nsel, kSelThreads, 0, st>>>(s);
		RX_CUDA(cudaGetLastError());
		g_stats.launches += 1;
		g_stats.tie_replays += nsel;
		g_stats.tie_from_lists += nsel;
		return 0;
	}
	RX_CUDA(ws.d_selbound.ensure(nsel));
	RX_CUDA(ws.d_lists.ensure(size_t(nsel) * k));
	RX_CUDA(cudaMemcpyAsync(ws.d_selbound.p, dstar, size_t(nsel) * 4, cudaMemcpyHostToDevice, st));
	const size_t rsmem = size_t((ix->dim + 127) / 128) * 512 + size_t(kScanWarps) * (k + kCandBuf) * 8;
	const float* norms = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	if (ix->metric == RXGPU_L2) {
		RX_CUDA(raiseSmemCeilingOnce(knn_rerank<true>, ix->device, kScanSmemBudget));
		knn_rerank<true><<<nsel, kScanThreads, rsmem, st>>>(ix->d_rows, ix->pitch, ix->dim, norms, d_queries, ws.d_cand_rows.p, ws.d_cand_count.p,
															 ws.tc_lists_cap, k, ws.d_lists.p, ws.d_sel.p, ws.d_selbound.p);
	} else {
		RX_CUDA(raiseSmemCeilingOnce(knn_rerank<false>, ix->device, kScanSmemBudget));
		knn_rerank<false><<<nsel, kScanThreads, rsmem, st>>>(ix->d_rows, ix->pitch, ix->dim, norms, d_queries, ws.d_cand_rows.p, ws.d_cand_count.p,
															  ws.tc_lists_cap, k, ws.d_lists.p, ws.d_sel.p, ws.d_selbound.p);
	}
	MergeArgs m{};
	m.lists = ws.d_lists.p;
	m.labels = ix->d_labels;
	m.out_dist = d_out_dist;
	m.out_idx = d_out_idx;
	m.out_label = d_out_label;
	m.out_count = d_out_count;
	m.nlists = 1;
	m.qt = nsel;
	m.k1 = k;
	m.q_offset = 0;
	m.out_stride = k;
	m.out_offset = 0;
	m.mode = kModeTieRows;
	m.neg_zero = ix->metric != RXGPU_L2;
	knn_merge_lists<<<nsel, 256, 0, st>>>(m);
	RX_CUDA(cudaGetLastError());
	g_stats.launches += 2;
	g_stats.tie_replays += nsel;
	g_stats.tie_from_lists += nsel;
	return 0;
}
}  // namespace rxgpu

namespace {

int normsForRange(rxgpu_index* ix, uint64_t begin, uint64_t end) {
	if (ix->metric != RXGPU_COS || begin >= end) {
		return 0;
	}
	RX_CUDA(launchNormCoefs(ix->d_rows, ix->pitch, ix->dim, uint32_t(begin), uint32_t(end), ix->d_norms, ix->stream));
	return 0;
}

}  // namespace

extern "C" {

const char* rxgpu_last_error(void) { return g_err.c_str(); }
int rxgpu_abi_version(void) { return RXGPU_ABI_VERSION; }
int rxgpu_device_count(void) {
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) {
		cudaGetLastError();
		return 0;
	}
	return n;
}

int rxgpu_index_create(rxgpu_index** out, rxgpu_metric metric, uint32_t dim, uint64_t capacity, int device, uint32_t flags) {
	if (!out) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null output handle");
	}
	*out = nullptr;
	if (dim == 0 || dim > 65536) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: vector dimension must be in [1, 65536]");
	}
	if (int(metric) < 0 || int(metric) > 2) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: unknown vector metric");
	}
	if (capacity >= (1ull << 31)) {  // the reference scans with an `int` index (bruteforce.cc:116)
		return fail(RXGPU_ERR_PARAMS, "rxgpu: capacity must be below 2^31 rows per shard");
	}
	if (rxgpu_device_count() <= device || device < 0) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: no usable CUDA device (this library has no CPU fallback)");
	}
	RX_CUDA(cudaSetDevice(device));
	std::unique_ptr<rxgpu_index> ix;
	try {
		ix = std::make_unique<rxgpu_index>();
		ix->metric = int(metric);
		ix->dim = dim;
		ix->pitch = (dim + 3u) & ~3u;
		ix->capacity = capacity;
		ix->device = device;
		ix->flags = flags;
		ix->h_labels.reserve(capacity);
		ix->dict.reserve(capacity);
		if (flags & RXGPU_FLAG_HOST_MIRROR) {
			ix->h_rows.resize(size_t(capacity) * dim);
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "Not enough memory: BruteforceSearch failed to allocate data");
	}
	cudaDeviceProp prop{};
	RX_CUDA(cudaGetDeviceProperties(&prop, device));
	ix->sm_count = prop.multiProcessorCount;
	RX_CUDA(cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking));
	if (int rc = allocDevice(ix.get(), capacity, &ix->d_rows, &ix->d_labels, &ix->d_norms)) {
		return rc;
	}
	*out = ix.release();
	return 0;
}

int rxgpu_index_clone(rxgpu_index** out, const rxgpu_index* src, uint64_t new_capacity) {
	if (!out || !src) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null handle");
	}
	const uint64_t cap = std::max(src->capacity, new_capacity);  // bruteforce.cc:22
	rxgpu_index* ix = nullptr;
	if (int rc = rxgpu_index_create(&ix, rxgpu_metric(src->metric), src->dim, cap, src->device, src->flags)) {
		return rc;
	}
	std::unique_ptr<rxgpu_index> guard(ix);
	try {
		ix->h_labels = src->h_labels;
		ix->dict = src->dict;
		if (src->flags & RXGPU_FLAG_HOST_MIRROR) {
			std::memcpy(ix->h_rows.data(), src->h_rows.data(), size_t(src->size) * src->dim * sizeof(float));
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "Not enough memory: BruteforceSearch failed to allocate data");
	}
	ix->size = src->size;
	ix->qt_override = src->qt_override;
	ix->tc_mode = src->tc_mode;
	ix->tc_cluster_max = src->tc_cluster_max;
	RX_CUDA(cudaMemcpyAsync(ix->d_rows, src->d_rows, size_t(src->size) * src->pitch * sizeof(float), cudaMemcpyDeviceToDevice, ix->stream));
	RX_CUDA(cudaMemcpyAsync(ix->d_labels, src->d_labels, size_t(src->size) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, ix->stream));
	if (src->d_norms) {
		RX_CUDA(cudaMemcpyAsync(ix->d_norms, src->d_norms, size_t(src->size) * sizeof(float), cudaMemcpyDeviceToDevice, ix->stream));
	}
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	*out = guard.release();
	return 0;
}

void rxgpu_index_destroy(rxgpu_index* ix) { delete ix; }

int rxgpu_index_resize(rxgpu_index* ix, uint64_t new_capacity) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (new_capacity < ix->size) {
		return fail(RXGPU_ERR_LOGIC, "Cannot resize, max element is less than the current number of elements");
	}
	if (new_capacity >= (1ull << 31)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: capacity must be below 2^31 rows per shard");
	}
	if (new_capacity == ix->capacity) {
		return 0;
	}
	float *rows = nullptr, *norms = nullptr;
	uint64_t* labels = nullptr;
	if (int rc = allocDevice(ix, new_capacity, &rows, &labels, &norms)) {
		cudaFree(rows);
		cudaFree(labels);
		cudaFree(norms);
		return fail(RXGPU_ERR_SYSTEM, "Not enough memory: resizeIndex failed to allocate data");
	}
	RX_CUDA(cudaMemcpyAsync(rows, ix->d_rows, size_t(ix->size) * ix->pitch * sizeof(float), cudaMemcpyDeviceToDevice, ix->stream));
	RX_CUDA(cudaMemcpyAsync(labels, ix->d_labels, size_t(ix->size) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, ix->stream));
	if (norms) {
		RX_CUDA(cudaMemcpyAsync(norms, ix->d_norms, size_t(ix->size) * sizeof(float), cudaMemcpyDeviceToDevice, ix->stream));
	}
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	cudaFree(ix->d_rows);
	cudaFree(ix->d_labels);
	cudaFree(ix->d_norms);
	ix->d_rows = rows;
	ix->d_labels = labels;
	ix->d_norms = norms;
	ix->capacity = new_capacity;
	if (ix->d_shadow) {  // rebuilt lazily at the new capacity
		std::lock_guard<std::mutex> lck(ix->tc_mtx);
		releaseShadow(ix);
	}
	try {
		if (ix->flags & RXGPU_FLAG_HOST_MIRROR) {
			ix->h_rows.resize(size_t(new_capacity) * ix->dim);
		}
		ix->h_labels.reserve(new_capacity);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "Not enough memory: resizeIndex failed to allocate data");
	}
	return 0;
}

int rxgpu_index_upsert_batch(rxgpu_index* ix, uint64_t n, const uint64_t* labels, const float* vecs) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (n == 0) {
		return 0;
	}
	if (!labels || !vecs) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null labels / vectors");
	}
	// Resolve destinations sequentially, exactly like n AddPointNoLock calls (bruteforce.cc:44-64) -- into temporaries: the
	// dictionary, h_labels, the host mirror and size are committed only after every device operation of the batch succeeded, so a
	// failed call (staging allocation, copy or launch error) leaves the index exactly as it was.
	try {
		std::vector<uint32_t> dst(n);
		std::vector<uint64_t> fresh;  // new labels in arrival order; fresh[i] goes to row size + i
		std::unordered_map<uint64_t, uint32_t> pending;  // new label -> row, for repeats of a new label inside the batch
		uint64_t newSize = ix->size;
		bool pureAppend = true;
		uint64_t accepted = n;
		for (uint64_t i = 0; i < n; ++i) {
			uint32_t idx = ix->dict.find(labels[i]);
			if (idx == LabelMap::kNotFound) {
				const auto it = pending.find(labels[i]);
				if (it != pending.end()) {
					idx = it->second;
					pureAppend = false;
				} else {
					if (newSize >= ix->capacity) {
						accepted = i;  // rows before i are applied, like the reference's sequential calls
						break;
					}
					idx = uint32_t(newSize++);
					pending.emplace(labels[i], idx);
					fresh.push_back(labels[i]);
				}
			} else {
				pureAppend = false;
			}
			dst[i] = idx;
		}
		const uint64_t m = accepted;
		if (m) {
			if (pureAppend && ix->pitch == ix->dim) {
				RX_CUDA(cudaMemcpyAsync(ix->d_rows + size_t(ix->size) * ix->pitch, vecs, size_t(m) * ix->dim * sizeof(float),
										cudaMemcpyHostToDevice, ix->stream));
				RX_CUDA(cudaMemcpyAsync(ix->d_labels + ix->size, labels, size_t(m) * sizeof(uint64_t), cudaMemcpyHostToDevice, ix->stream));
				if (int rc = normsForRange(ix, ix->size, ix->size + m)) {
					return rc;
				}
			} else {
				// stage + scatter in bounded slices; the staging buffers live in the index (no cudaMalloc / cudaFree per call)
				const uint64_t slice = std::max<uint64_t>(1, (64ull << 20) / (ix->dim * sizeof(float)));
				RX_CUDA(ix->st_rows.ensure(size_t(std::min(slice, m)) * ix->dim));
				RX_CUDA(ix->st_dst.ensure(size_t(std::min(slice, m))));
				RX_CUDA(ix->st_labels.ensure(size_t(std::min(slice, m))));
				for (uint64_t off = 0; off < m; off += slice) {
					const uint64_t cnt = std::min(slice, m - off);
					RX_CUDA(cudaMemcpyAsync(ix->st_rows.p, vecs + off * ix->dim, size_t(cnt) * ix->dim * sizeof(float), cudaMemcpyHostToDevice,
											ix->stream));
					RX_CUDA(cudaMemcpyAsync(ix->st_dst.p, dst.data() + off, size_t(cnt) * sizeof(uint32_t), cudaMemcpyHostToDevice, ix->stream));
					RX_CUDA(cudaMemcpyAsync(ix->st_labels.p, labels + off, size_t(cnt) * sizeof(uint64_t), cudaMemcpyHostToDevice, ix->stream));
					// duplicates of one label inside a slice must apply in order: one launch per row when present
					bool dup = false;
					if (cnt > 1) {
						std::vector<uint32_t> sorted(dst.begin() + off, dst.begin() + off + cnt);
						std::sort(sorted.begin(), sorted.end());
						dup = std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end();
					}
					if (!dup) {
						scatter_rows_kernel<<<unsigned(cnt), 128, 0, ix->stream>>>(ix->st_rows.p, ix->st_dst.p, ix->st_labels.p, uint32_t(cnt), ix->dim,
																				   ix->pitch, ix->d_rows, ix->d_labels);
						RX_CUDA(cudaGetLastError());
					} else {
						for (uint64_t i = 0; i < cnt; ++i) {
							scatter_rows_kernel<<<1, 128, 0, ix->stream>>>(ix->st_rows.p + i * ix->dim, ix->st_dst.p + i, ix->st_labels.p + i, 1, ix->dim,
																		   ix->pitch, ix->d_rows, ix->d_labels);
						}
						RX_CUDA(cudaGetLastError());
					}
					if (ix->metric == RXGPU_COS) {
						for (uint64_t i = 0; i < cnt;) {  // norms for maximal runs of consecutive destinations
							uint64_t j = i + 1;
							while (j < cnt && dst[off + j] == dst[off + j - 1] + 1) {
								++j;
							}
							if (int rc = normsForRange(ix, dst[off + i], uint64_t(dst[off + j - 1]) + 1)) {
								return rc;
							}
							i = j;
						}
					}
					if (off + slice < m) {
						RX_CUDA(cudaStreamSynchronize(ix->stream));  // the staging buffers are reused by the next slice
					}
				}
			}
			RX_CUDA(cudaStreamSynchronize(ix->stream));
			// ---- commit (host state only; nothing below can fail except by std::bad_alloc, which reserve() at create/resize precludes)
			for (size_t i = 0; i < fresh.size(); ++i) {
				ix->dict.put(fresh[i], uint32_t(ix->size + i));
				ix->h_labels.push_back(fresh[i]);
			}
			if (ix->flags & RXGPU_FLAG_HOST_MIRROR) {
				for (uint64_t i = 0; i < m; ++i) {
					std::memcpy(ix->h_rows.data() + size_t(dst[i]) * ix->dim, vecs + i * ix->dim, ix->dim * sizeof(float));
				}
			}
			for (uint64_t i = 0; i < m;) {  // maximal runs of consecutive destinations (an appended batch is one range)
				uint64_t j = i + 1;
				while (j < m && dst[j] == dst[j - 1] + 1) {
					++j;
				}
				ix->touchRows(dst[i], uint64_t(dst[j - 1]) + 1);
				i = j;
			}
			ix->size = newSize;
			ix->version++;
		}
		if (accepted < n) {
			return fail(RXGPU_ERR_LOGIC, "The number of elements exceeds the specified limit\n");
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_index_upsert(rxgpu_index* ix, uint64_t label, const float* vec) { return rxgpu_index_upsert_batch(ix, 1, &label, vec); }

int rxgpu_index_remove(rxgpu_index* ix, uint64_t label) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	const uint32_t cur = ix->dict.find(label);
	if (cur == LabelMap::kNotFound) {
		return 0;  // bruteforce.cc:72-74
	}
	ix->dict.erase(label);
	ix->version++;
	const uint64_t last = ix->size - 1;
	if (cur != last) {  // move the last row into the hole (bruteforce.cc:78-82)
		ix->touchRows(cur, uint64_t(cur) + 1);
		const uint64_t lastLabel = ix->h_labels[last];
		ix->dict.put(lastLabel, cur);
		ix->h_labels[cur] = lastLabel;
		RX_CUDA(cudaMemcpyAsync(ix->d_rows + size_t(cur) * ix->pitch, ix->d_rows + size_t(last) * ix->pitch, ix->pitch * sizeof(float),
								cudaMemcpyDeviceToDevice, ix->stream));
		RX_CUDA(cudaMemcpyAsync(ix->d_labels + cur, ix->d_labels + last, sizeof(uint64_t), cudaMemcpyDeviceToDevice, ix->stream));
		if (ix->d_norms) {
			RX_CUDA(cudaMemcpyAsync(ix->d_norms + cur, ix->d_norms + last, sizeof(float), cudaMemcpyDeviceToDevice, ix->stream));
		}
		if (ix->flags & RXGPU_FLAG_HOST_MIRROR) {
			std::memcpy(ix->h_rows.data() + size_t(cur) * ix->dim, ix->h_rows.data() + size_t(last) * ix->dim, ix->dim * sizeof(float));
		}
		RX_CUDA(cudaStreamSynchronize(ix->stream));
	}
	ix->h_labels.pop_back();
	ix->size--;
	return 0;
}

int rxgpu_index_get(const rxgpu_index* ix, uint64_t label, const float** host_row) {
	if (!ix || !host_row) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null handle");
	}
	const uint32_t idx = ix->dict.find(label);
	if (idx == LabelMap::kNotFound) {
		return fail(RXGPU_ERR_NOT_FOUND, "Label not found");
	}
	if (ix->flags & RXGPU_FLAG_HOST_MIRROR) {
		*host_row = ix->h_rows.data() + size_t(idx) * ix->dim;
		return 0;
	}
	RX_CUDA(cudaSetDevice(ix->device));
	g_row_scratch.resize(ix->dim);
	RX_CUDA(cudaMemcpy(g_row_scratch.data(), ix->d_rows + size_t(idx) * ix->pitch, ix->dim * sizeof(float), cudaMemcpyDeviceToHost));
	*host_row = g_row_scratch.data();
	return 0;
}

uint64_t rxgpu_index_size(const rxgpu_index* ix) { return ix ? ix->size : 0; }
uint64_t rxgpu_index_capacity(const rxgpu_index* ix) { return ix ? ix->capacity : 0; }
uint64_t rxgpu_index_element_size(const rxgpu_index* ix) { return ix ? uint64_t(ix->dim) * 4 + 8 : 0; }
uint64_t rxgpu_index_device_bytes(const rxgpu_index* ix) {
	if (!ix) {
		return 0;
	}
	const uint64_t cap = ix->capacity ? ix->capacity : 1;
	return cap * ix->pitch * 4 + cap * 8 + (ix->d_norms ? cap * 4 : 0);
}
uint32_t rxgpu_index_dim(const rxgpu_index* ix) { return ix ? ix->dim : 0; }
int rxgpu_index_metric(const rxgpu_index* ix) { return ix ? ix->metric : -1; }
int rxgpu_index_device(const rxgpu_index* ix) { return ix ? ix->device : -1; }

int rxgpu_set_query_tile(rxgpu_index* ix, uint32_t qt) {
	if (!ix) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null handle");
	}
	ix->qt_override = qt;
	return 0;
}
int rxgpu_set_tensor_core_filter(rxgpu_index* ix, int mode) {
	if (!ix || mode < 0 || mode > 5) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: tensor-core filter mode must be 0..5");
	}
	ix->tc_mode = uint32_t(mode >= 3 ? 1 : mode);
	ix->tc_cluster_max = mode == 3 ? 1u : mode == 4 ? 2u : mode == 5 ? 4u : 0u;
	return 0;
}
int rxgpu_tc_diag(int mode, void* d_counters) {
	if (mode < 0 || mode > kTcDiagNoTest || (mode && !d_counters)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: diagnostic filter mode must be 0..4, with a counter buffer");
	}
	const char* env = std::getenv("RXGPU_TC_DIAG");
	if (mode && !(env && std::strcmp(env, "1") == 0)) {  // a stray call must not turn every search of the process into a diagnostic
		return fail(RXGPU_ERR_LOGIC, "rxgpu: diagnostic filter instantiations are enabled only with RXGPU_TC_DIAG=1 in the environment");
	}
	g_tc_diag_buf = static_cast<unsigned long long*>(d_counters);
	g_tc_diag.store(mode);
	return 0;
}
int rxgpu_tc_audit(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* tau, uint32_t query_block, uint32_t* out_shape,
				   uint32_t* slot_row, float* rowc, float* blockc, signed char* row_codes, signed char* query_codes, float* qc, float* kab,
				   int32_t* block_thr, float* row_bound) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!out_shape || (nq && (!queries || !tau)) || query_block == 0 || query_block > kTcMaxNq || query_block % 32) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: audit needs the shape output, queries with their thresholds and a query block of 32..128");
	}
	RX_CUDA(cudaSetDevice(ix->device));
	cudaStream_t st = ix->stream;
	if (int rc = ensureShadow(ix, st)) {
		return rc;
	}
	const uint32_t pitch = ix->pitch_q, kchunks = pitch / kTcChunkK, dim = ix->dim, slots = ix->shadow_slots;
	const uint32_t nblocks = uint32_t((uint64_t(slots) + kTcTileRows - 1) / kTcTileRows * kTcTileRows / 64);  // as the filter walks them
	const uint32_t nqblocks = (nq + query_block - 1) / query_block;
	out_shape[0] = slots;
	out_shape[1] = nblocks;
	auto fetch = [&](void* dst, const void* src, size_t bytes) -> cudaError_t {
		return dst && bytes ? cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) : cudaSuccess;
	};
	RX_CUDA(fetch(slot_row, ix->d_slot_row, size_t(slots) * 4));
	RX_CUDA(fetch(rowc, ix->d_rowc, size_t(slots) * sizeof(float4)));
	RX_CUDA(fetch(blockc, ix->d_blockc, size_t(nblocks) * 2 * sizeof(float4)));
	// the row codes by slot, un-swizzled (tc_convert_rows' layout): [64-slot block][K chunk][64 slots x 128 B]
	std::vector<signed char> sh(size_t(nblocks) * 64 * pitch), codes(size_t(nblocks) * 64 * pitch);
	RX_CUDA(fetch(sh.data(), ix->d_shadow, sh.size()));
	for (uint32_t s = 0; s < nblocks * 64; ++s) {
		const uint32_t blk = s / 64, r = s % 64;
		for (uint32_t c = 0; c < pitch; c += 16) {
			const uint32_t kc = c / kTcChunkK, unit = ((c % kTcChunkK) >> 4) ^ (r & 7u);
			std::memcpy(&codes[size_t(s) * pitch + c], &sh[(size_t(blk) * kchunks + kc) * kTcBlockBytes + r * 128u + unit * 16u], 16);
		}
	}
	if (row_codes) {
		for (uint32_t s = 0; s < slots; ++s) {
			std::memcpy(row_codes + size_t(s) * dim, &codes[size_t(s) * pitch], dim);
		}
	}
	if (nq == 0) {
		return 0;
	}
	DevBuf<float> d_q, d_qf, d_tau;
	DevBuf<unsigned char> d_qcodes;
	DevBuf<signed char> d_rcodes;
	DevBuf<float4> d_qc;
	DevBuf<float2> d_kab, d_bound;
	DevBuf<int> d_thr;
	RX_CUDA(d_q.ensure(size_t(nq) * dim));
	RX_CUDA(d_qf.ensure(size_t(nq) * pitch));
	RX_CUDA(d_tau.ensure(nq));
	RX_CUDA(d_qcodes.ensure(size_t(nq) * pitch));
	RX_CUDA(d_qc.ensure(nq));
	RX_CUDA(d_kab.ensure(nqblocks));
	RX_CUDA(d_thr.ensure(std::max<size_t>(size_t(nq) * nblocks, 1)));
	RX_CUDA(cudaMemcpyAsync(d_q.p, queries, size_t(nq) * dim * 4, cudaMemcpyHostToDevice, st));
	RX_CUDA(cudaMemcpyAsync(d_tau.p, tau, size_t(nq) * 4, cudaMemcpyHostToDevice, st));
	tc_prepare_queries<<<(nq * 32 + 255) / 256, 256, 0, st>>>(d_q.p, nq, nq, dim, pitch, d_qcodes.p, d_qc.p, d_qf.p);
	tc_audit_thresholds<<<nqblocks, 256, 0, st>>>(d_qc.p, d_tau.p, nq, query_block, dim, ix->metric, ix->d_blockc, nblocks, d_kab.p, d_thr.p);
	if (row_bound && slots) {
		RX_CUDA(d_rcodes.ensure(size_t(slots) * pitch));
		RX_CUDA(d_bound.ensure(size_t(nq) * slots));
		RX_CUDA(cudaMemcpyAsync(d_rcodes.p, codes.data(), size_t(slots) * pitch, cudaMemcpyHostToDevice, st));
		tc_audit_bounds<<<dim3((slots + 255) / 256, nq), 256, 0, st>>>(reinterpret_cast<const signed char*>(d_qcodes.p), d_qc.p, d_rcodes.p,
																		ix->d_rowc, pitch, slots, dim, ix->metric, d_bound.p);
	}
	RX_CUDA(cudaGetLastError());
	RX_CUDA(cudaStreamSynchronize(st));
	if (query_codes) {
		std::vector<signed char> qcodes(size_t(nq) * pitch);
		RX_CUDA(fetch(qcodes.data(), d_qcodes.p, qcodes.size()));
		for (uint32_t q = 0; q < nq; ++q) {
			std::memcpy(query_codes + size_t(q) * dim, &qcodes[size_t(q) * pitch], dim);
		}
	}
	RX_CUDA(fetch(qc, d_qc.p, size_t(nq) * sizeof(float4)));
	RX_CUDA(fetch(kab, d_kab.p, size_t(nqblocks) * sizeof(float2)));
	RX_CUDA(fetch(block_thr, d_thr.p, size_t(nq) * nblocks * 4));
	if (row_bound && slots) {
		RX_CUDA(fetch(row_bound, d_bound.p, size_t(nq) * slots * sizeof(float2)));
	}
	return 0;
}
int rxgpu_set_profile(int on) {
	g_profile.store(on ? 1 : 0);
	return 0;
}
void rxgpu_last_search_stats(rxgpu_search_stats* out) {
	if (out) {
		*out = g_stats;
	}
}

// ---------------------------------------------------------------------------------------------------------------- search
int rxgpu_search_knn_device(const rxgpu_index* ix, uint32_t nq, const float* d_queries, uint32_t k1, float* d_out_dist,
							uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count, void* stream) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (k1 == 0 || k1 > kMaxSearchK1) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be in [1, 65535]");
	}
	WsLease lease(ix);
	Workspace& ws = *lease.ws;
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
	lease.st = st;
	if (ix->size == 0) {
		RX_CUDA(cudaMemsetAsync(d_out_count, 0, nq * sizeof(uint32_t), st));
		RX_CUDA(cudaStreamSynchronize(st));
		return 0;
	}
	if (int rc = scanTopK(ix, ws, st, d_queries, nq, k1, kModeTopK, 0.f, d_out_dist, d_out_idx, d_out_label, d_out_count)) {
		return rc;
	}
	RX_CUDA(cudaStreamSynchronize(st));  // the workspace goes back to the pool: nothing of this call may still be running
	collectProfile();
	return 0;
}

int rxgpu_search_tie_rows_device(const rxgpu_index* ix, const float* d_query, float dstar, uint32_t k, float* d_out_dist,
								 uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count, void* stream) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (k == 0 || k > kMaxSearchK1) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be in [1, 65535]");
	}
	WsLease lease(ix);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ix->stream;
	lease.st = st;
	if (ix->size == 0) {
		RX_CUDA(cudaMemsetAsync(d_out_count, 0, sizeof(uint32_t), st));
		RX_CUDA(cudaStreamSynchronize(st));
		return 0;
	}
	if (int rc = scanTopK(ix, *lease.ws, st, d_query, 1, k, kModeTieRows, dstar, d_out_dist, d_out_idx, d_out_label, d_out_count)) {
		return rc;
	}
	RX_CUDA(cudaStreamSynchronize(st));
	g_stats.tie_replays += 1;
	return 0;
}

int rxgpu_merge_shards(uint32_t nshards, uint32_t nq, uint32_t k, uint32_t k1, const float* dist, const uint32_t* idx,
					   const uint64_t* label, const uint32_t* count, const uint64_t* shard_base, float* out_dist, uint64_t* out_gidx,
					   uint64_t* out_label, uint32_t* out_count, uint8_t* need_tie) {
	if (!dist || !idx || !label || !count || !shard_base || !out_dist || !out_gidx || !out_label || !out_count || !need_tie) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		std::vector<Hit> all;
		for (uint32_t q = 0; q < nq; ++q) {
			all.clear();
			for (uint32_t s = 0; s < nshards; ++s) {
				const size_t b = (size_t(s) * nq + q) * k1;
				const uint32_t c = std::min(count[size_t(s) * nq + q], k1);
				for (uint32_t j = 0; j < c; ++j) {
					all.push_back(Hit{dist[b + j], shard_base[s] + idx[b + j], label[b + j]});
				}
			}
			std::sort(all.begin(), all.end(), hitLessByIndex);
			const uint32_t n = uint32_t(std::min<size_t>(all.size(), k));
			// a tie straddling the k-th place: the reference's survivors depend on arrival order and labels
			need_tie[q] = all.size() > k && k > 0 && !(all[k - 1].dist < all[k].dist) ? 1 : 0;
			std::vector<Hit> top(all.begin(), all.begin() + n);
			orderTiesByLabel(top);
			for (uint32_t j = 0; j < n; ++j) {
				out_dist[size_t(q) * k + j] = top[j].dist;
				out_gidx[size_t(q) * k + j] = top[j].gidx;
				out_label[size_t(q) * k + j] = top[j].label;
			}
			out_count[q] = n;
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_tie_replay(uint32_t k, float dstar, uint32_t n_lower, const float* lower_dist, const uint64_t* lower_gidx,
					 const uint64_t* lower_label, uint32_t n_first, const float* first_dist, const uint64_t* first_gidx,
					 const uint64_t* first_label, float* out_dist, uint64_t* out_label, uint32_t* out_count) {
	try {
		std::vector<Hit> lower(n_lower), first(n_first);
		for (uint32_t i = 0; i < n_lower; ++i) {
			lower[i] = Hit{lower_dist[i], lower_gidx[i], lower_label[i]};
		}
		for (uint32_t i = 0; i < n_first; ++i) {
			first[i] = Hit{first_dist[i], first_gidx[i], first_label[i]};
		}
		const auto res = tieReplay(k, dstar, lower, first);
		for (size_t i = 0; i < res.size(); ++i) {
			out_dist[i] = res[i].dist;
			out_label[i] = res[i].label;
		}
		*out_count = uint32_t(res.size());
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

static int searchKnnHost(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, std::vector<std::vector<Hit>>& results) {
	results.assign(nq, {});
	g_stats = rxgpu_search_stats{};
	if (nq == 0 || k == 0 || ix->size == 0) {
		return 0;  // bruteforce.cc:106-108
	}
	const uint32_t kEff = uint32_t(std::min<uint64_t>(k, ix->size));           // bruteforce.cc:111
	const uint32_t k1 = uint32_t(std::min<uint64_t>(uint64_t(kEff) + 1, ix->size));  // one extra row exposes a tie at the k-th place
	if (k1 > kMaxSearchK1) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be in [1, 65535]");
	}
	WsLease lease(ix);
	Workspace& ws = *lease.ws;
	if (!ws.stream) {
		RX_CUDA(cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking));
	}
	cudaStream_t st = ws.stream;
	lease.st = st;
	const size_t qn = size_t(nq) * ix->dim, on = size_t(nq) * k1;
	RX_CUDA(ws.d_queries.ensure(qn));
	RX_CUDA(ws.h_queries.ensure(qn));
	RX_CUDA(ws.d_out_dist.ensure(on));
	RX_CUDA(ws.d_out_idx.ensure(on));
	RX_CUDA(ws.d_out_label.ensure(on));
	RX_CUDA(ws.d_out_count.ensure(nq));
	RX_CUDA(ws.h_out_dist.ensure(on));
	RX_CUDA(ws.h_out_idx.ensure(on));
	RX_CUDA(ws.h_out_label.ensure(on));
	RX_CUDA(ws.h_out_count.ensure(nq));
	std::memcpy(ws.h_queries.p, queries, qn * sizeof(float));
	RX_CUDA(cudaMemcpyAsync(ws.d_queries.p, ws.h_queries.p, qn * sizeof(float), cudaMemcpyHostToDevice, st));
	if (int rc = scanTopK(ix, ws, st, ws.d_queries.p, nq, k1, kModeTopK, 0.f, ws.d_out_dist.p, ws.d_out_idx.p, ws.d_out_label.p,
						  ws.d_out_count.p)) {
		return rc;
	}
	RX_CUDA(cudaMemcpyAsync(ws.h_out_dist.p, ws.d_out_dist.p, on * sizeof(float), cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(ws.h_out_idx.p, ws.d_out_idx.p, on * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(ws.h_out_label.p, ws.d_out_label.p, on * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(ws.h_out_count.p, ws.d_out_count.p, nq * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	collectProfile();

	for (uint32_t q = 0; q < nq; ++q) {
		const uint32_t cnt = std::min(ws.h_out_count.p[q], k1);
		const float* d = ws.h_out_dist.p + size_t(q) * k1;
		const uint32_t* ii = ws.h_out_idx.p + size_t(q) * k1;
		const uint64_t* ll = ws.h_out_label.p + size_t(q) * k1;
		std::vector<Hit>& res = results[q];
		const uint32_t n = std::min(cnt, kEff);
		const bool tie = cnt > kEff && !(d[kEff - 1] < d[kEff]);
		if (!tie) {
			res.reserve(n);
			for (uint32_t j = 0; j < n; ++j) {
				res.push_back(Hit{d[j], ii[j], ll[j]});
			}
			orderTiesByLabel(res);
			continue;
		}
		// replay the reference's heap tie rule: fetch the first kEff rows (internal order) with dist <= dstar -- from the filter's
		// candidate lists when this batch went through the tensor-core path (no second pass over the rows)
		const float dstar = d[kEff - 1];
		std::vector<Hit> lower;
		for (uint32_t j = 0; j < kEff && d[j] < dstar; ++j) {
			lower.push_back(Hit{d[j], ii[j], ll[j]});
		}
		RX_CUDA(ws.d_tie_dist.ensure(kEff));
		RX_CUDA(ws.d_tie_idx.ensure(kEff));
		RX_CUDA(ws.d_tie_label.ensure(kEff));
		RX_CUDA(ws.d_tie_count.ensure(1));
		if (int rc = tieRowsAfterScan(ix, ws, st, ws.d_queries.p, 1, &q, &dstar, kEff, ws.d_tie_dist.p, ws.d_tie_idx.p, ws.d_tie_label.p,
									  ws.d_tie_count.p)) {
			return rc;
		}
		std::vector<float> td(kEff);
		std::vector<uint32_t> ti(kEff);
		std::vector<uint64_t> tl(kEff);
		uint32_t tc = 0;
		RX_CUDA(cudaMemcpyAsync(td.data(), ws.d_tie_dist.p, kEff * sizeof(float), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(ti.data(), ws.d_tie_idx.p, kEff * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(tl.data(), ws.d_tie_label.p, kEff * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(&tc, ws.d_tie_count.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		std::vector<Hit> first;
		for (uint32_t j = 0; j < std::min(tc, kEff); ++j) {
			first.push_back(Hit{td[j], ti[j], tl[j]});
		}
		res = tieReplay(kEff, dstar, lower, first);
	}
	return 0;
}

int rxgpu_search_knn(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, float* out_dist, uint64_t* out_label,
					 uint32_t* out_count) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (nq && (!queries || !out_count || (k && (!out_dist || !out_label)))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		std::vector<std::vector<Hit>> results;
		if (int rc = searchKnnHost(ix, nq, queries, k, results)) {
			return rc;
		}
		for (uint32_t q = 0; q < nq; ++q) {
			const auto& r = results[q];
			for (size_t j = 0; j < r.size(); ++j) {
				out_dist[size_t(q) * k + j] = r[j].dist;
				out_label[size_t(q) * k + j] = r[j].label;
			}
			out_count[q] = uint32_t(r.size());
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

}  // extern "C"

namespace rxgpu {
int scanRangeHits(const rxgpu_index* ix, cudaStream_t st, ScanArgs a, DevBuf<uint64_t>& d_keys, DevBuf<unsigned long long>& d_count,
				  PinBuf<uint64_t>& h_keys, const uint64_t* h_labels, std::vector<Hit>& res, uint32_t& scans) {
	res.clear();
	scans = 0;
	RX_CUDA(d_count.ensure(1));
	for (;;) {
		RX_CUDA(d_keys.ensure(a.range_cap));
		RX_CUDA(cudaMemsetAsync(d_count.p, 0, sizeof(unsigned long long), st));
		a.range_out = d_keys.p;
		a.range_count = d_count.p;
		unsigned grid = 0;
		RX_CUDA(launchScan(ix, 1, a, &grid, st));
		++scans;
		unsigned long long total = 0;
		RX_CUDA(cudaMemcpyAsync(&total, d_count.p, sizeof(total), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		if (total > a.range_cap) {  // buffer too small: grow and rescan (results are a set, the scan is deterministic)
			a.range_cap = total;
			continue;
		}
		RX_CUDA(h_keys.ensure(std::max<uint64_t>(total, 1)));
		RX_CUDA(cudaMemcpyAsync(h_keys.p, d_keys.p, total * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		res.reserve(total);
		for (unsigned long long i = 0; i < total; ++i) {
			const uint64_t key = h_keys.p[i];
			const uint32_t row = uint32_t(key);
			res.push_back(Hit{ord_float(uint32_t(key >> 32)), row, h_labels[row]});
		}
		break;
	}
	std::sort(res.begin(), res.end(), hitLessByLabel);  // the order in which the reference's heap drains backwards
	return 0;
}
}  // namespace rxgpu

extern "C" {

// The exact range scan of one device-resident query: every row with dist < radius, in the order of hitLessByLabel.  Uses ws.d_range.
static int scanRangeExact(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_query, float radius, std::vector<Hit>& res) {
	ScanArgs a{};
	a.rows = ix->d_rows;
	a.norm_coefs = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
	a.queries = d_query;
	a.pitch = ix->pitch;
	a.dim = ix->dim;
	a.row_begin = 0;
	a.row_end = uint32_t(ix->size);
	a.nq = 1;
	a.k1 = 1;
	a.mode = kModeRange;
	a.bound = radius;
	// result buffer: up to 4M matches (32 MB) without a rescan; a larger result grows the buffer and scans once more
	a.range_cap = std::max<uint64_t>(ws.d_range.n, std::min<uint64_t>(std::max<uint64_t>(ix->size, 1), 1u << 22));
	uint32_t scans = 0;
	const int rc = scanRangeHits(ix, st, a, ws.d_range, ws.d_range_count, ws.h_range, ix->h_labels.data(), res, scans);
	g_stats.launches += scans;
	g_stats.passes += scans;
	if (rc) {
		return rc;
	}
	g_stats.algorithmic_bytes += uint64_t(ix->size) * ix->dim * 4 + (ix->metric == RXGPU_COS ? uint64_t(ix->size) * 4 : 0) + ix->dim * 4 +
								 res.size() * 8;
	return 0;
}

static int searchRangeHost(const rxgpu_index* ix, const float* query, float radius, std::vector<Hit>& res) {
	res.clear();
	g_stats = rxgpu_search_stats{};
	if (ix->size == 0) {
		return 0;
	}
	WsLease lease(ix);
	Workspace& ws = *lease.ws;
	if (!ws.stream) {
		RX_CUDA(cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking));
	}
	cudaStream_t st = ws.stream;
	lease.st = st;
	RX_CUDA(ws.d_queries.ensure(ix->dim));
	RX_CUDA(cudaMemcpyAsync(ws.d_queries.p, query, ix->dim * sizeof(float), cudaMemcpyHostToDevice, st));
	if (int rc = scanRangeExact(ix, ws, st, ws.d_queries.p, radius, res)) {
		return rc;
	}
	g_stats.query_tile = 1;
	return 0;
}

}  // extern "C"

namespace rxgpu {
// Range search for a batch of device-resident queries on a non-empty index, enqueued on `st`.  A batch the filter serves (tcServes)
// runs one filter pass with tau = radius, then the range mode of knn_rerank keeps the candidates with dist < radius -- the same set and
// distance bits as the exact range scan, which answers every other query.  Adds to g_stats.
int rangeBatch(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, const float* radius,
			   uint64_t max_out, const RangeEmit& emit) {
	std::vector<Hit> res;
	// dist < radius never holds for a NaN or -inf radius: no matches, no scan.  A +inf radius matches every row: the exact scan.
	auto filtered = [&](uint32_t q) { return radius[q] > -INFINITY && radius[q] < INFINITY; };
	std::vector<uint32_t> exact;  // queries the exact range scan answers
	if (tcServes(ix, nq)) {
		const uint32_t cap = tcRangeCap(max_out);
		// the queries outside the filter get a radius of -inf: no candidate passes, and none would match
		std::vector<float> rad(nq);
		std::vector<unsigned int> tau(nq);
		for (uint32_t q = 0; q < nq; ++q) {
			rad[q] = filtered(q) ? radius[q] : -INFINITY;
			tau[q] = float_ord(rad[q]);
		}
		if (int rc = tcFilter(ix, ws, st, d_queries, nq, 0, cap, tau.data())) {
			return rc;
		}
		ws.tc_lists_valid = false;  // the candidate lists now hold this batch's range candidates: no tie replay may read them
		RX_CUDA(ws.d_radius.ensure(nq));
		RX_CUDA(ws.d_range_n.ensure(nq));
		RX_CUDA(ws.h_range_n.ensure(nq));
		RX_CUDA(ws.d_range.ensure(size_t(nq) * cap));
		RX_CUDA(cudaMemcpyAsync(ws.d_radius.p, rad.data(), size_t(nq) * 4, cudaMemcpyHostToDevice, st));
		if (int rc = rerankRange(ix, ws, st, d_queries, nq, nq, nullptr, cap, ws.d_radius.p, ws.d_range.p, ws.d_range_n.p)) {
			return rc;
		}
		RX_CUDA(cudaMemcpyAsync(ws.h_cand_count.p, ws.d_cand_count.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(ws.h_range_n.p, ws.d_range_n.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		// copy back the first `width` keys of every query's region: as many as the largest answer the filter decided
		uint64_t cands = 0;
		uint32_t width = 0;
		for (uint32_t q = 0; q < nq; ++q) {
			if (!filtered(q)) {
				continue;
			}
			cands += std::min(ws.h_cand_count.p[q], cap);
			if (ws.h_cand_count.p[q] > cap) {  // an overflowed list (masses of rows near the radius): the exact scan answers it
				g_stats.tc_fallbacks += 1;
			} else {
				width = std::max(width, ws.h_range_n.p[q]);
			}
		}
		if (width) {
			RX_CUDA(ws.h_range.ensure(size_t(nq) * width));
			RX_CUDA(cudaMemcpy2DAsync(ws.h_range.p, size_t(width) * 8, ws.d_range.p, size_t(cap) * 8, size_t(width) * 8, nq,
									  cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
		}
		for (uint32_t q = 0; q < nq; ++q) {
			if (!filtered(q) || ws.h_cand_count.p[q] > cap) {
				exact.push_back(q);
				continue;
			}
			res.clear();
			const uint64_t* keys = ws.h_range.p + size_t(q) * width;
			for (uint32_t i = 0; i < ws.h_range_n.p[q]; ++i) {
				const uint32_t row = uint32_t(keys[i]);
				res.push_back(Hit{ord_float(uint32_t(keys[i] >> 32)), row, ix->h_labels[row]});
			}
			std::sort(res.begin(), res.end(), hitLessByLabel);  // the order of the exact range scan
			emit(q, res);
		}
		g_stats.tc_used = 1;
		g_stats.tc_candidates = cands;
		g_stats.algorithmic_bytes += cands * (uint64_t(ix->dim) * 4 + 4);
	} else {
		for (uint32_t q = 0; q < nq; ++q) {
			exact.push_back(q);
		}
		g_stats.query_tile = 1;
	}
	for (const uint32_t q : exact) {
		if (radius[q] == INFINITY || filtered(q)) {
			if (int rc = scanRangeExact(ix, ws, st, d_queries + size_t(q) * ix->dim, radius[q], res)) {
				return rc;
			}
		} else {
			res.clear();
		}
		emit(q, res);
	}
	return 0;
}
}  // namespace rxgpu

extern "C" {

// rxgpu_search_range_batch: the host queries go to the device, rangeBatch answers them, row q of the output gets query q's answer
static int searchRangeBatchHost(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint64_t max_out,
								float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	g_stats = rxgpu_search_stats{};
	auto emit = [&](uint32_t q, const std::vector<Hit>& hits) {  // hits in the order of hitLessByLabel
		const uint64_t n = std::min<uint64_t>(hits.size(), max_out);
		for (uint64_t i = 0; i < n; ++i) {
			out_dist[q * max_out + i] = hits[i].dist;
			out_label[q * max_out + i] = hits[i].label;
		}
		out_n[q] = hits.size();
	};
	if (ix->size == 0) {
		const std::vector<Hit> none;
		for (uint32_t q = 0; q < nq; ++q) {
			emit(q, none);
		}
		return 0;
	}
	WsLease lease(ix);
	Workspace& ws = *lease.ws;
	if (!ws.stream) {
		RX_CUDA(cudaStreamCreateWithFlags(&ws.stream, cudaStreamNonBlocking));
	}
	cudaStream_t st = ws.stream;
	lease.st = st;
	const size_t qn = size_t(nq) * ix->dim;
	RX_CUDA(ws.d_queries.ensure(qn));
	RX_CUDA(ws.h_queries.ensure(qn));
	std::memcpy(ws.h_queries.p, queries, qn * sizeof(float));
	RX_CUDA(cudaMemcpyAsync(ws.d_queries.p, ws.h_queries.p, qn * sizeof(float), cudaMemcpyHostToDevice, st));
	return rangeBatch(ix, ws, st, ws.d_queries.p, nq, radius, max_out, emit);
}

int rxgpu_search_range(const rxgpu_index* ix, const float* query, float radius, uint64_t max_out, float* out_dist, uint64_t* out_label,
					   uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!query || !out_n) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		std::vector<Hit>& res = g_range_result;
		if (int rc = searchRangeHost(ix, query, radius, res)) {
			return rc;
		}
		const uint64_t n = std::min<uint64_t>(res.size(), max_out);
		for (uint64_t i = 0; i < n; ++i) {
			out_dist[i] = res[i].dist;
			out_label[i] = res[i].label;
		}
		*out_n = res.size();
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_search_range_batch(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint64_t max_out,
							 float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (nq && (!queries || !radius || !out_n || (max_out && (!out_dist || !out_label)))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		return searchRangeBatchHost(ix, nq, queries, radius, max_out, out_dist, out_label, out_n);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_last_range_results(uint64_t offset, uint64_t n, float* out_dist, uint64_t* out_label) {
	if (offset > g_range_result.size() || n > g_range_result.size() - offset || (n && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: range outside the retained result of this thread's last rxgpu_search_range");
	}
	for (uint64_t i = 0; i < n; ++i) {
		out_dist[i] = g_range_result[offset + i].dist;
		out_label[i] = g_range_result[offset + i].label;
	}
	return 0;
}

int rxgpu_select_postprocess(int metric, const rxgpu_select_params* p, uint64_t n, const float* dist, const uint64_t* label, int32_t* out_row_ids,
							 float* out_ranks, uint64_t* out_n) {
	if (!p || !out_n || (n && (!dist || !label || !out_row_ids || !out_ranks)) || metric < 0 || metric > 2) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: bad argument");
	}
	try {
		std::vector<Hit> res(n);
		for (uint64_t i = 0; i < n; ++i) {
			res[i] = Hit{dist[i], 0, label[i]};
		}
		SelectParams sp;
		sp.metric = metric;
		sp.needSort = p->need_sort != 0;
		sp.isArray = p->is_array != 0;
		sp.raw = p->raw != 0;
		sp.hasK = p->k != 0;
		sp.k = p->k;
		sp.hasRadius = p->has_radius != 0;
		std::vector<int32_t> ids;
		std::vector<float> ranks;
		selectPostprocess(sp, res, ids, ranks);
		for (size_t i = 0; i < ids.size(); ++i) {
			out_row_ids[i] = ids[i];
			out_ranks[i] = ranks[i];
		}
		*out_n = ids.size();
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_select_knn(const rxgpu_index* ix, const float* query, const rxgpu_select_params* p, uint64_t max_out, int32_t* out_row_ids,
					 float* out_ranks, uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!query || !p || !out_n) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (p->k == 0 && !p->has_radius) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: KNN query needs k or radius");
	}
	try {
		// HnswIndexBase::search, hnsw_index.cc:160-191
		std::vector<float> normalized;
		const float* keyData = query;
		if (ix->metric == RXGPU_COS) {
			normalized.resize(ix->dim);
			normalizeCopyVector(query, int32_t(ix->dim), normalized.data());
			keyData = normalized.data();
		}
		std::vector<Hit> res;
		if (p->has_radius) {
			if (int rc = searchRangeHost(ix, keyData, ix->metric == RXGPU_L2 ? p->radius : -p->radius, res)) {
				return rc;
			}
		} else {
			std::vector<std::vector<Hit>> results;
			if (int rc = searchKnnHost(ix, 1, keyData, p->k, results)) {
				return rc;
			}
			res = std::move(results[0]);
		}
		SelectParams sp;
		sp.metric = ix->metric;
		sp.needSort = p->need_sort != 0;
		sp.isArray = p->is_array != 0;
		sp.raw = p->raw != 0;
		sp.hasK = p->k != 0;
		sp.k = p->k;
		sp.hasRadius = p->has_radius != 0;
		std::vector<int32_t> ids;
		std::vector<float> ranks;
		selectPostprocess(sp, res, ids, ranks);
		const uint64_t n = std::min<uint64_t>(ids.size(), max_out);
		for (uint64_t i = 0; i < n; ++i) {
			out_row_ids[i] = ids[i];
			out_ranks[i] = ranks[i];
		}
		*out_n = ids.size();
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

// ---------------------------------------------------------------------------------------------------------------- bench support
int rxgpu_index_append_synth(rxgpu_index* ix, uint64_t seed, uint64_t first_row, uint64_t n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->flags & RXGPU_FLAG_HOST_MIRROR) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: device-side synthetic fill is not available with a host mirror");
	}
	if (ix->size + n > ix->capacity) {
		return fail(RXGPU_ERR_LOGIC, "The number of elements exceeds the specified limit\n");
	}
	if (n == 0) {
		return 0;
	}
	// refuse before touching the dictionary: a refused call leaves the index exactly as it was
	for (uint64_t r = 0; r < n; ++r) {
		if (ix->dict.find((first_row + r) << 32) != LabelMap::kNotFound) {
			return fail(RXGPU_ERR_LOGIC, "rxgpu: synthetic rows must have fresh labels");
		}
	}
	try {
		ix->h_labels.reserve(ix->size + n);
		ix->dict.reserve(ix->size + n);
		for (uint64_t r = 0; r < n; ++r) {
			const uint64_t label = (first_row + r) << 32;
			ix->dict.put(label, uint32_t(ix->size + r));
			ix->h_labels.push_back(label);
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	synth_rows_kernel<<<unsigned(ix->sm_count) * 8, 256, 0, ix->stream>>>(ix->d_rows, ix->d_labels, ix->pitch, ix->dim, uint32_t(ix->size),
																		 seed, first_row, n);
	RX_CUDA(cudaGetLastError());
	if (int rc = normsForRange(ix, ix->size, ix->size + n)) {
		return rc;
	}
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	ix->touchRows(ix->size, ix->size + n);
	ix->size += n;
	ix->version++;
	return 0;
}

int rxgpu_synth_fill_device(float* d_out, uint64_t seed, uint64_t first_index, uint64_t count, int device, void* stream) {
	if (rxgpu_device_count() <= device || device < 0) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: no usable CUDA device (this library has no CPU fallback)");
	}
	RX_CUDA(cudaSetDevice(device));
	cudaStream_t st = static_cast<cudaStream_t>(stream);
	synth_fill_kernel<<<1184, 256, 0, st>>>(d_out, seed, first_index, count);
	RX_CUDA(cudaGetLastError());
	RX_CUDA(cudaStreamSynchronize(st));
	return 0;
}

}  // extern "C"
