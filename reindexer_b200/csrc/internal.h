// Internal declarations shared by the translation units of librxgpu (index.cu, ivf.cu, hnsw.cu, ft_bm25.cu, ...).  Not part of the ABI.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rxgpu.h"
#include "../host/flat_map.h"

namespace rxgpu {

extern thread_local std::string g_err;
extern thread_local rxgpu_search_stats g_stats;
extern thread_local std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_events;
extern std::atomic<int> g_profile;

// sum the event pairs recorded by this thread's launches; call after the stream has been synchronised
inline void collectProfile() {
	for (auto& ev : g_prof_events) {
		float ms = 0.f;
		if (cudaEventElapsedTime(&ms, ev.first, ev.second) == cudaSuccess) {
			g_stats.scan_kernel_ms += ms;
			g_stats.scan_launches += 1;
		}
		cudaEventDestroy(ev.first);
		cudaEventDestroy(ev.second);
	}
	g_prof_events.clear();
}

inline int fail(int code, std::string msg) {
	g_err = std::move(msg);
	return code;
}

#define RX_CUDA(expr)                                                                                        \
	do {                                                                                                     \
		cudaError_t e_ = (expr);                                                                             \
		if (e_ != cudaSuccess) {                                                                             \
			return fail(RXGPU_ERR_SYSTEM, std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " #expr); \
		}                                                                                                    \
	} while (0)

template <typename T>
struct DevBuf {
	T* p = nullptr;
	size_t n = 0;
	~DevBuf() { release(); }
	void release() {
		if (p) {
			cudaFree(p);
			p = nullptr;
			n = 0;
		}
	}
	cudaError_t ensure(size_t want) {
		if (want <= n) {
			return cudaSuccess;
		}
		release();
		cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T));
		if (e == cudaSuccess) {
			n = want;
		}
		return e;
	}
};
template <typename T>
struct PinBuf {
	T* p = nullptr;
	size_t n = 0;
	~PinBuf() {
		if (p) {
			cudaFreeHost(p);
		}
	}
	cudaError_t ensure(size_t want) {
		if (want <= n) {
			return cudaSuccess;
		}
		if (p) {
			cudaFreeHost(p);
			p = nullptr;
			n = 0;
		}
		cudaError_t e = cudaMallocHost(reinterpret_cast<void**>(&p), want * sizeof(T));
		if (e == cudaSuccess) {
			n = want;
		}
		return e;
	}
};

// The dynamic shared-memory ceiling of a kernel is a per-device FUNCTION attribute: searches run concurrently from many threads
// (the reference's read-side concurrency), so it is raised once per (kernel, device) to the budget every caller stays within --
// never per launch, where a thread asking for less would lower it under another thread's launch (cudaErrorInvalidValue).
constexpr int kScanSmemBudget = 100 * 1024;
inline cudaError_t raiseSmemCeilingOnceImpl(const void* fn, int device, int bytes) {
	static std::mutex mtx;
	static std::vector<std::pair<const void*, int>> done;  // (kernel entry point, device); a handful of entries
	std::lock_guard<std::mutex> lck(mtx);
	for (const auto& d : done) {
		if (d.first == fn && d.second == device) {
			return cudaSuccess;
		}
	}
	const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
	if (e == cudaSuccess) {
		done.emplace_back(fn, device);
	}
	return e;
}
template <typename Kernel>
inline cudaError_t raiseSmemCeilingOnce(Kernel kfn, int device, int bytes) {  // keyed by the entry point, not by its type
	return raiseSmemCeilingOnceImpl(reinterpret_cast<const void*>(kfn), device, bytes);
}

// per-call scratch: searches are re-entrant, each takes one workspace from the pool
struct Workspace {
	cudaStream_t stream = nullptr;
	DevBuf<float> d_queries;
	DevBuf<uint64_t> d_lists;
	DevBuf<uint64_t> d_floor;  // per-query floor keys between the rounds of a k > 255 search
	DevBuf<float> d_out_dist;
	DevBuf<uint32_t> d_out_idx;
	DevBuf<uint64_t> d_out_label;
	DevBuf<uint32_t> d_out_count;
	DevBuf<uint64_t> d_range;  // single-query range scan: its matches; range batch on the filter: [nq][cand cap] matches per query
	DevBuf<unsigned long long> d_range_count;
	DevBuf<float> d_radius;          // range batch on the filter: per-query radius, and its per-query match counts
	DevBuf<unsigned int> d_range_n;
	PinBuf<unsigned int> h_range_n;
	DevBuf<unsigned char> d_qcodes;  // int8 query codes for the tensor-core filter
	DevBuf<float4> d_qc;             // their per-query constants (s_q, r_q, ||q||, 1 / k_q)
	DevBuf<float> d_qf;              // the fp32 queries zero padded to the codes' pitch (exact distances of the bound list)
	DevBuf<unsigned int> d_tau, d_cand_count, d_ub_lock;
	DevBuf<float> d_ub_list;
	DevBuf<float> d_seed_part;  // the seed's per-slice lists [nq][kTcSeedSlices][kTcMaxK1] (tc_seed_slices -> tc_seed_merge)
	DevBuf<uint32_t> d_cand_rows;
	DevBuf<float> d_cand_lb;  // KNN on the filter: the lower bound of every listed row (knn_rerank gathers those under the final tau)
	PinBuf<unsigned int> h_cand_count;
	DevBuf<unsigned int> d_stage_status;  // KNN with staged thresholds: per-query fallback status, and the candidates re-ranked
	PinBuf<unsigned int> h_stage_status;
	DevBuf<unsigned long long> d_reranked;
	PinBuf<unsigned long long> h_reranked;
	PinBuf<float> h_queries;
	PinBuf<float> h_out_dist;
	PinBuf<uint32_t> h_out_idx;
	PinBuf<uint64_t> h_out_label;
	PinBuf<uint32_t> h_out_count;
	PinBuf<uint64_t> h_range;
	// state of the last scanTopK on this workspace: when the tensor-core filter answered it, the per-query candidate lists
	// (d_cand_rows / h_cand_count; the last stage's with staged thresholds) hold every row at or below each query's k1-th distance --
	// tieRowsAfterScan reads them
	bool tc_lists_valid = false;
	uint32_t tc_lists_nq = 0;
	uint32_t tc_lists_cap = 0;  // entries per query list of that call
	uint64_t tc_lists_version = 0;
	DevBuf<uint32_t> d_sel;
	DevBuf<float> d_selbound;
	DevBuf<float> d_tie_dist;
	DevBuf<uint32_t> d_tie_idx, d_tie_count;
	DevBuf<uint64_t> d_tie_label;
	~Workspace() {
		if (stream) {
			cudaStreamDestroy(stream);
		}
	}
};

}  // namespace rxgpu

struct rxgpu_hnsw_device;  // hnsw.cu
struct rxgpu_ivf_device;   // ivf.cu
struct rxgpu_sq8_device;   // sq8.cu
namespace rxgpu {
void hnswRelease(rxgpu_hnsw_device*);
void ivfRelease(rxgpu_ivf_device*);
void sq8Release(rxgpu_sq8_device*);
}

struct rxgpu_index {
	int metric = 0;
	uint32_t dim = 0;
	uint32_t pitch = 0;  // floats, multiple of 4
	uint64_t capacity = 0;
	uint64_t size = 0;
	int device = 0;
	uint32_t flags = 0;
	int sm_count = 132;
	uint32_t qt_override = 0;
	uint64_t version = 0;  // bumped by every mutation of rows/labels (staleness check of attached structures)

	float* d_rows = nullptr;
	uint64_t* d_labels = nullptr;
	float* d_norms = nullptr;  // Cosine only (DistCalculator::normCoefs_, hnswlib.h:33-35)

	std::vector<uint64_t> h_labels;  // by internal index
	rxgpu::LabelMap dict;
	std::vector<float> h_rows;  // optional host mirror [capacity][dim]

	cudaStream_t stream = nullptr;  // maintenance stream
	rxgpu::DevBuf<float> st_rows;   // staging of scattered upserts (mutators run one at a time under the namespace write lock)
	rxgpu::DevBuf<uint32_t> st_dst;
	rxgpu::DevBuf<uint64_t> st_labels;
	mutable std::mutex ws_mtx;
	mutable std::vector<std::unique_ptr<rxgpu::Workspace>> ws_free;
	rxgpu_hnsw_device* hnsw = nullptr;  // graph attached by rxgpu_hnsw_import (hnsw.cu)
	rxgpu_ivf_device* ivf = nullptr;    // centroids + list boundaries attached by rxgpu_ivf_import
	rxgpu_sq8_device* sq8 = nullptr;    // SQ8 codes + corrective offsets attached by rxgpu_sq8_attach (sq8.cu)

	// tensor-core filter state, built lazily by the first large-batch search: int8 shadow of the rows + per-row constants
	mutable std::mutex tc_mtx;
	// The shadow holds the rows in SLOT order: sorted by the block test's row factors at a full build (ensureShadow), rows appended
	// since then in new slots at the end, the slots of vanished rows dead (knn_tc.cuh: kTcDeadSlot).
	mutable void* d_shadow = nullptr;  // int8 codes, [slot capacity / 64 blocks][pitch_q / 128 chunks][64 x 128 B], knn_tc.cuh
	mutable float4* d_rowc = nullptr;  // [slot capacity] (scale, residual norm, norm, Cosine coefficient) of every slot's row
	mutable uint32_t* d_slot_row = nullptr;  // [slot capacity] the row of a slot, kTcDeadSlot for none
	mutable uint32_t* d_row_slot = nullptr;  // [capacity] the slot of a row
	mutable float4* d_blockc = nullptr;      // [slot capacity / 64][2] tc_block_consts
	mutable uint32_t pitch_q = 0;      // bytes of codes per row, dim rounded up to 128
	mutable uint64_t shadow_slot_cap = 0;    // slots allocated (whole tiles)
	mutable uint32_t shadow_slots = 0;       // slots in use, dead ones included
	mutable uint32_t shadow_rows = 0;        // rows the shadow holds (the index size when it was last brought up to date)
	mutable uint32_t shadow_unsorted = 0;    // slots appended or rewritten since the last full build
	mutable uint32_t shadow_dead = 0;        // dead slots
	mutable uint64_t shadow_version = ~0ull;
	// rows rewritten since the shadow was last brought up to date (the mutations log them beside `version`): ensureShadow converts
	// only these; the log gives up (full rebuild) beyond kShadowLogMax ranges
	static constexpr size_t kShadowLogMax = 4096;
	mutable std::vector<std::pair<uint32_t, uint32_t>> shadow_dirty;
	mutable bool shadow_dirty_all = true;
	// lowest row written since the attached HNSW graph was imported, built or patched (~0: none): an append onto the graph needs
	// its rows unchanged
	uint64_t rows_touched_from = ~0ull;
	void touchRows(uint64_t begin, uint64_t end) {
		std::lock_guard<std::mutex> lck(tc_mtx);
		if (begin < end) {
			rows_touched_from = std::min(rows_touched_from, begin);
		}
		if (!d_shadow || shadow_dirty_all || begin >= end) {
			return;
		}
		if (!shadow_dirty.empty() && shadow_dirty.back().second == begin) {
			shadow_dirty.back().second = uint32_t(end);
		} else if (shadow_dirty.size() < kShadowLogMax) {
			shadow_dirty.emplace_back(uint32_t(begin), uint32_t(end));
		} else {
			shadow_dirty_all = true;
			shadow_dirty.clear();
		}
	}
	uint32_t tc_mode = 0;  // 0 auto, 1 force on, 2 off
	uint32_t tc_cluster_max = 0;  // most CTAs per cluster (1, 2 or 4); 0 = the default shape (index.cu: kTcClusterDefault)

	~rxgpu_index() {
		cudaSetDevice(device);
		ws_free.clear();
		if (hnsw) {
			rxgpu::hnswRelease(hnsw);
		}
		if (ivf) {
			rxgpu::ivfRelease(ivf);
		}
		if (sq8) {
			rxgpu::sq8Release(sq8);
		}
		if (d_rows) {
			cudaFree(d_rows);
		}
		if (d_labels) {
			cudaFree(d_labels);
		}
		if (d_norms) {
			cudaFree(d_norms);
		}
		if (d_shadow) {
			cudaFree(d_shadow);
		}
		cudaFree(d_rowc);
		cudaFree(d_slot_row);
		cudaFree(d_row_slot);
		cudaFree(d_blockc);
		if (stream) {
			cudaStreamDestroy(stream);
		}
	}
};

namespace rxgpu {

// The workspace's buffers are used on whichever stream the call enqueues on (ws.stream, the caller's stream, ix->stream or a
// communicator's), so stream order alone does not keep the next lease-holder off them.  A call that returns early after a launch (an
// allocation or launch error) would hand back buffers a kernel may still be writing: the lease synchronises the call's stream `st`
// before the workspace goes back to the pool.  On success the call has synchronised it already, so this waits for nothing.
struct WsLease {
	const rxgpu_index* idx;
	std::unique_ptr<Workspace> ws;
	cudaStream_t st = nullptr;  // set by the call once it has picked its stream
	explicit WsLease(const rxgpu_index* i) : idx(i) {
		{
			std::lock_guard<std::mutex> lck(idx->ws_mtx);
			if (!idx->ws_free.empty()) {
				ws = std::move(idx->ws_free.back());
				idx->ws_free.pop_back();
			}
		}
		if (!ws) {
			ws = std::make_unique<Workspace>();
		}
	}
	~WsLease() {
		if (st) {
			cudaStreamSynchronize(st);
		}
		std::lock_guard<std::mutex> lck(idx->ws_mtx);
		idx->ws_free.emplace_back(std::move(ws));
	}
};

// index.cu -- shared with shard.cu
// Top-k1 rows per query under (dist, internal row) [kModeTopK], or the first k1 rows in internal order with dist <= bound
// [kModeTieRows, one query]; large batches go through the tensor-core filter + exact re-rank (same bits).  Device in / out.
int scanTopK(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, uint32_t k1, int mode, float bound,
			 float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count);
// After a scanTopK(kModeTopK) of `d_queries` on the SAME workspace: for the selected queries sel[i] the first k rows in internal order
// with dist <= dstar[i] (what the reference's tie rule needs, SURVEY.md 8a rule 2), [nsel][k] device outputs.  Served from the
// filter's candidate lists when they exist (no second pass over the rows), else by one kModeTieRows scan per selected query.
int tieRowsAfterScan(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nsel, const uint32_t* sel,
					 const float* dstar, uint32_t k, float* d_out_dist, uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count);

// Range search of nq device-resident queries on a non-empty index (the core of rxgpu_search_range_batch, and each shard's part of
// rxgpu_sharded_search_range_batch).  emit(q, hits) is called once per query with ALL its matches (dist < radius[q], radius on the host)
// in the order of hitLessByLabel; only the first min(hits, max_out) are ever returned, which sizes the filter's candidate lists.
struct Hit;  // host/knn_select.h
using RangeEmit = std::function<void(uint32_t q, const std::vector<Hit>& hits)>;
int rangeBatch(const rxgpu_index* ix, Workspace& ws, cudaStream_t st, const float* d_queries, uint32_t nq, const float* radius,
			   uint64_t max_out, const RangeEmit& emit);

// index.cu -- the kernels of knn_scan.cuh, which are compiled there only; the IVF index (ivf.cu) launches them through these
struct ScanArgs;
struct MergeArgs;
// the exact scan (knn_scan_warp) with a qt-query tile, its grid to *gridOut (dryRun: nothing launched); keysOut: the key mode of the
// work-item scan (qt = 1)
cudaError_t launchScan(const rxgpu_index* ix, int qt, const ScanArgs& a, unsigned* gridOut, cudaStream_t st, bool dryRun = false,
					   bool keysOut = false);
cudaError_t launchMergeLists(const MergeArgs& m, uint32_t nq, cudaStream_t st);  // knn_merge_lists, one CTA per query
// 1/||row|| of the rows [row_begin, row_end) (norm_coef_kernel)
cudaError_t launchNormCoefs(const float* rows, uint32_t pitch, uint32_t dim, uint32_t row_begin, uint32_t row_end, float* coefs, cudaStream_t st);
// staged rows [n][dim] to rows[dst[i]] (zero padded to pitch) with their labels, and with `norms` their 1/||row|| too
cudaError_t scatterRows(const float* staged, const uint32_t* dst, const uint64_t* staged_labels, uint32_t n, uint32_t dim, uint32_t pitch,
						float* rows, uint64_t* labels, float* norms, cudaStream_t st);
// The range-mode scan `a` until its key buffer held every match: zeroes the counter, scans, reads the count, and when the buffer
// (a.range_cap keys) was too small grows it and scans again.  The matches with their labels (h_labels, by row), in the order of
// hitLessByLabel; `scans` counts the launches.
int scanRangeHits(const rxgpu_index* ix, cudaStream_t st, ScanArgs a, DevBuf<uint64_t>& d_keys, DevBuf<unsigned long long>& d_count,
				  PinBuf<uint64_t>& h_keys, const uint64_t* h_labels, std::vector<Hit>& res, uint32_t& scans);

// ivf.cu -- the coarse quantiser of the attached IVF lists, for the k-means assignment (ivf_train.cu): errLogic as the searches report it
// when no lists are attached or the index changed since
struct IvfCentroids {
	const float* centroids;  // [nlist][pitch]
	const float* cnorm;      // Cosine: 1/||centroid||, else nullptr
	uint32_t nlist;
	bool own;                // lists made by rxgpu_ivf_create
};
int ivfCentroids(const rxgpu_index* ix, IvfCentroids& out);
// errParams when the coarse pass cannot stage one query of `dim` floats in shared memory
int ivfCheckCoarseDim(uint32_t dim);
// keys[i] = make_key(distance, centroid) of the nearest of the nlist centroids [nlist][ix->pitch] to the device row x[i] ([n][ix->dim],
// Cosine rows normalised) under (distance, centroid id): the coarse pass's distance kernel in argmin mode, same tile and grid
cudaError_t ivfAssignRows(const rxgpu_index* ix, const float* centroids, const float* cnorm, uint32_t nlist, const float* x, uint32_t n,
						  uint64_t* keys, cudaStream_t st);
constexpr uint32_t kIvfMaxCentroids = 1u << 17;  // the reference's centroids_count bound (kIvfNCentroidsMax, indexopts.cc)
// the local parts of the sharded IVF searches (shard.cu), each after rxgpu_ivf_search_*'s own checks.  `view` receives what the ranks
// must agree on: a fingerprint of the centroids, nlist, nprobe as clamped, and the rows the lists address (the shard's size in the merge)
struct IvfShardView {
	uint64_t fingerprint;
	uint32_t nlist, nprobe;
	uint64_t rows;
};
// the best min(k, probed rows) rows of every query under (distance, local internal row), in that order, into the device rows
// d_*[q * stride, + d_count[q]): the coarse pass, then the fused top-k or the key pass and exact select, as
// rxgpu_ivf_search_knn_large_k chooses.  Done (synchronised) on return.
int ivfShardKnn(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, uint32_t nprobe, uint32_t stride, float* d_dist,
				uint32_t* d_idx, uint64_t* d_label, uint32_t* d_count, IvfShardView& view);
// rxgpu_ivf_search_range_batch without its output step: emit(q, n, dist, label, m) once per query with its n matches and the best
// m = min(n, max_out) of them, in the order of hitLessByLabel (host arrays, valid during the call)
using IvfRangeEmit = std::function<void(uint32_t q, uint64_t n, const float* dist, const uint64_t* label, uint64_t m)>;
int ivfShardRange(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint32_t nprobe, uint64_t max_out,
				  const IvfRangeEmit& emit, IvfShardView& view);

// writes row `idx` (== size: appends) with a new vector and label, keeping the label dictionary consistent (index.cu)
int setRowAt(rxgpu_index* ix, uint32_t idx, uint64_t label, const float* vec);

inline int checkIndex(const rxgpu_index* ix) {
	if (!ix) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null index handle");
	}
	RX_CUDA(cudaSetDevice(ix->device));
	return 0;
}

// ---- collectives over an rxgpu_comm (shard.cu): NCCL between processes, a host rendezvous between the threads of one process -------
enum class CommOp { SumU64, SumU32, MaxU32 };
int commRank(const rxgpu_comm*);
int commSize(const rxgpu_comm*);
int commDevice(const rxgpu_comm*);
std::mutex& commMutex(rxgpu_comm*);
int commAllReduce(rxgpu_comm*, void* d_buf, size_t count, CommOp op, cudaStream_t st);        // in place
int commAllGather(rxgpu_comm*, const void* d_send, void* d_recv, size_t bytes, cudaStream_t st);  // d_recv: nranks x bytes

}  // namespace rxgpu
