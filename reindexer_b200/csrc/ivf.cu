// librxgpu: the IVF index (rxgpu_ivf_*) -- faiss::IndexIVFFlat over the rows of a brute-force index (rxgpu_ivf_import) or over lists
// that own their rows (rxgpu_ivf_create / _add / _remove).  The coarse quantiser and the any-k select are this file's kernels
// (ivf_coarse.cuh, ivf_select.cuh, ivf_range.cuh); the list scans and their merge are the brute-force index's exact scan, launched
// through internal.h (index.cu).
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>
#include <functional>
#include <limits>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

#include "../../include/rxgpu.h"
#include "internal.h"
#include "../host/knn_select.h"
#include "knn_scan.cuh"
#include "ivf_select.cuh"
#include "ivf_range.cuh"
#include "ivf_coarse.cuh"

using namespace rxgpu;

struct rxgpu_ivf_device {
	uint32_t nlist = 0;
	uint64_t index_version = 0;
	DevBuf<float> centroids;       // [nlist][pitch]
	DevBuf<float> cnorm;           // Cosine: 1/||centroid|| (IndexFlatCosine's norm coefficients)
	DevBuf<uint32_t> list_begin;   // [nlist + 1] rows of list l = [list_begin[l], list_begin[l + 1])
	std::mutex mtx;                // one IVF batch at a time per index (scratch below)
	DevBuf<float> d_q, d_dist;
	DevBuf<uint4> d_work;
	DevBuf<uint64_t> d_lists, d_label;
	DevBuf<uint32_t> d_idx, d_count;
	DevBuf<uint64_t> d_range;
	DevBuf<unsigned long long> d_range_count;
	PinBuf<uint64_t> h_range;
	// any-k select path (rxgpu_ivf_search_knn_large_k): probed rows and key offsets per query, a query chunk's work items (query-major,
	// with the slot of their first key) and key workspace, the survivors (ordered distance word + label, double-buffered for the sorts)
	DevBuf<uint64_t> d_qrows, d_qoff, d_keys;
	DevBuf<uint4> d_work_chunk;
	DevBuf<uint32_t> d_sel_ord, d_sel_ord2, d_sel_count, d_sel_hist;
	DevBuf<uint64_t> d_sel_label, d_sel_label2;
	DevBuf<int> d_seg_begin, d_seg_end;
	DevBuf<SelState> d_sel_state;
	DevBuf<unsigned char> d_cub;
	// range batch (rxgpu_ivf_search_range_batch), beside the key workspace and survivors above: radius per query, a chunk's key tiles
	// (query, tile), its matches per query, a sub-chunk's survivor and output offsets
	DevBuf<float> d_radius;
	DevBuf<uint2> d_tiles;
	DevBuf<uint32_t> d_range_n;
	DevBuf<int> d_range_seg;
	// mutable lists (rxgpu_ivf_create / _add / _remove): every list owns a region [begin, begin + cap) of a row slab; size <= cap
	struct Slab {
		float* rows = nullptr;           // [slab_rows][pitch]
		uint64_t* labels = nullptr;      // [slab_rows]
		float* norms = nullptr;          // [slab_rows] (Cosine)
		std::vector<uint64_t> h_labels;  // host mirror of `labels`
		Slab() = default;
		Slab(const Slab&) = delete;
		Slab& operator=(const Slab&) = delete;
		~Slab() {
			cudaFree(rows);
			cudaFree(labels);
			cudaFree(norms);
		}
		void swap(Slab& o) {
			std::swap(rows, o.rows);
			std::swap(labels, o.labels);
			std::swap(norms, o.norms);
			h_labels.swap(o.h_labels);
		}
	};
	bool own = false;
	Slab slab;
	uint64_t slab_rows = 0, high_water = 0, live = 0, dead = 0;
	std::vector<uint32_t> begin, size, cap;
	DevBuf<uint32_t> list_end;   // begin + size (list_begin holds begin)
	std::unordered_map<uint64_t, std::pair<uint32_t, uint32_t>> where;     // id -> (list, offset), faiss::DirectMap::Hashtable
	DevBuf<float> st_rows;
	DevBuf<uint32_t> st_dst;
	DevBuf<uint64_t> st_labels;
	uint64_t relocations = 0, compactions = 0;
	uint64_t fingerprint = 0;  // of the centroids, made by the first sharded search (ivfShardView); 0: not yet
};
namespace rxgpu {
void ivfRelease(rxgpu_ivf_device* p) { delete p; }
int ivfCentroids(const rxgpu_index* ix, IvfCentroids& out) {
	const rxgpu_ivf_device* h = ix->ivf;
	if (!h) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no IVF lists imported into this index");
	}
	if (h->index_version != ix->version) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the index changed after the IVF lists were imported");
	}
	out = IvfCentroids{h->centroids.p, ix->metric == RXGPU_COS ? h->cnorm.p : nullptr, h->nlist, h->own};
	return 0;
}
int ivfCheckCoarseDim(uint32_t dim) {
	if (coarse_smem_bytes(1, dim) > kCoarseSmemMax) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: dimension exceeds the coarse quantiser's shared memory");
	}
	return 0;
}
}  // namespace rxgpu

namespace {
// The checks every IVF search makes after its own argument checks, in this order: lists imported and the index unchanged since;
// k in [1, kmax] (kmax 0: no k); nprobe clamped to [1, nlist] as faiss::IndexIVF::search does, and at most probeMax; the coarse pass
// stages one query (at least) in shared memory: dim <= 51 200.
int ivfSearchChecks(const rxgpu_index* ix, uint32_t k, uint32_t kmax, uint32_t probeMax, uint32_t& nprobe) {
	const rxgpu_ivf_device* h = ix->ivf;
	if (!h) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no IVF lists imported into this index");
	}
	if (h->index_version != ix->version) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the index changed after the IVF lists were imported");
	}
	if (kmax && (k == 0 || k > kmax)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF search needs k in [1, " + std::to_string(kmax) + "]");
	}
	nprobe = std::max(1u, std::min(nprobe, h->nlist));
	if (nprobe > probeMax) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: nprobe exceeds the merge fan-in (1024)");
	}
	return ivfCheckCoarseDim(ix->dim);
}

// where the lists' rows live: in the index (rxgpu_ivf_import) or in the lists' own slab (rxgpu_ivf_create)
struct IvfRows {
	const float* rows;
	const float* norms;  // Cosine norm coefficients, nullptr for the other metrics
	const uint64_t* labels;
	const uint64_t* h_labels;
};
IvfRows ivfRows(const rxgpu_index* ix, const rxgpu_ivf_device* h) {
	const bool cos = ix->metric == RXGPU_COS;
	if (h->own) {
		return {h->slab.rows, cos ? h->slab.norms : nullptr, h->slab.labels, h->slab.h_labels.data()};
	}
	return {ix->d_rows, cos ? ix->d_norms : nullptr, ix->d_labels, ix->h_labels.data()};
}

// the exact scan over probed lists in work-item mode: CTA b scans the rows of work[b] for its query in h->d_q
ScanArgs ivfScanArgs(const rxgpu_index* ix, const rxgpu_ivf_device* h, const IvfRows& r, const uint4* work, uint32_t nwork, uint32_t k1, int mode) {
	ScanArgs a{};
	a.rows = r.rows;
	a.norm_coefs = r.norms;
	a.queries = h->d_q.p;
	a.pitch = ix->pitch;
	a.dim = ix->dim;
	a.nq = 1;
	a.k1 = k1;
	a.mode = mode;
	a.work = work;
	a.nwork = nwork;
	return a;
}

template <bool kIsL2, int QT, bool kArgmin = false>
cudaError_t launchCoarseDist(const rxgpu_index* ix, const float* centroids, uint32_t nlist, dim3 grid, size_t smem, const float* queries,
							 uint32_t cq, const float* cnorm, uint64_t* keys, cudaStream_t st) {
	if (cudaError_t e = raiseSmemCeilingOnce(ivf_coarse_dist_kernel<kIsL2, QT, kArgmin>, ix->device, int(kCoarseSmemMax))) {
		return e;
	}
	ivf_coarse_dist_kernel<kIsL2, QT, kArgmin><<<grid, kScanThreads, smem, st>>>(centroids, ix->pitch, ix->dim, nlist, queries, cq, cnorm, keys);
	return cudaGetLastError();
}
// the coarse pass's query tile for a batch of nq, and its grid over tiles x centroid slices: query tiles fastest, so the CTAs in flight
// share centroid slices through L2; about 4 CTAs per SM over the whole grid
int coarseTile(const rxgpu_index* ix, uint32_t nq) { return nq > 1 && coarse_smem_bytes(kCoarseTile, ix->dim) <= kCoarseSmemMax ? kCoarseTile : 1; }
dim3 coarseGrid(const rxgpu_index* ix, uint32_t nlist, uint32_t cq, int qt) {
	const uint32_t groups = (nlist + kCoarseRows - 1) / kCoarseRows;
	const uint32_t tiles = (cq + qt - 1) / qt;
	const uint32_t slices = std::max(1u, std::min((groups + kScanWarps - 1) / kScanWarps, (uint32_t(ix->sm_count) * 4 + tiles - 1) / tiles));
	return dim3(tiles, slices);
}
// the coarse quantiser (ivf_coarse.cuh) over nq queries (host, or device on the index's GPU), staged in h->d_q: work items of the list scans in h->d_work, probe-major.
// Per query chunk of at most kIvfKeyCap keys: distances, select, sort, emit (4 launches, counted in g_stats with the centroid bytes, read
// once per query tile).  The chunk's keys go to h->d_keys, its survivors to h->d_sel_label: the key pass and the selects that follow
// reuse them.  A batch stages kCoarseTile queries per tile (dim <= 3 200), one query stages itself alone.
int ivfLaunchCoarse(const rxgpu_index* ix, rxgpu_ivf_device* h, uint32_t nq, const float* queries, uint32_t nprobe, cudaStream_t st) {
	const uint32_t nlist = h->nlist;
	RX_CUDA(h->d_q.ensure(size_t(nq) * ix->dim));
	RX_CUDA(h->d_work.ensure(size_t(nq) * nprobe));
	RX_CUDA(cudaMemcpyAsync(h->d_q.p, queries, size_t(nq) * ix->dim * 4, cudaMemcpyDefault, st));  // host or device queries
	const int qt = coarseTile(ix, nq);
	const size_t smem = coarse_smem_bytes(qt, ix->dim);
	const uint32_t chunk = uint32_t(std::max<uint64_t>(1, kIvfKeyCap / nlist));
	const uint32_t cqMax = std::min(nq, chunk);
	RX_CUDA(h->d_keys.ensure(size_t(cqMax) * nlist));
	RX_CUDA(h->d_sel_label.ensure(size_t(cqMax) * nprobe));
	RX_CUDA(h->d_seg_begin.ensure(cqMax));
	RX_CUDA(h->d_seg_end.ensure(cqMax));
	const float* cnorm = ix->metric == RXGPU_COS ? h->cnorm.p : nullptr;
	for (uint32_t q0 = 0; q0 < nq; q0 += chunk) {
		const uint32_t cq = std::min(chunk, nq - q0);
		const dim3 grid = coarseGrid(ix, nlist, cq, qt);
		const uint32_t tiles = grid.x;
		const float* qs = h->d_q.p + size_t(q0) * ix->dim;
		const float* cp = h->centroids.p;
		uint64_t* keys = h->d_keys.p;
		if (ix->metric == RXGPU_L2) {
			RX_CUDA(qt == 1 ? (launchCoarseDist<true, 1>(ix, cp, nlist, grid, smem, qs, cq, cnorm, keys, st))
							: (launchCoarseDist<true, kCoarseTile>(ix, cp, nlist, grid, smem, qs, cq, cnorm, keys, st)));
		} else {
			RX_CUDA(qt == 1 ? (launchCoarseDist<false, 1>(ix, cp, nlist, grid, smem, qs, cq, cnorm, keys, st))
							: (launchCoarseDist<false, kCoarseTile>(ix, cp, nlist, grid, smem, qs, cq, cnorm, keys, st)));
		}
		ivf_coarse_select_kernel<<<cq, kIvfSelThreads, 0, st>>>(h->d_keys.p, nlist, nprobe, h->d_sel_label.p, h->d_seg_begin.p, h->d_seg_end.p);
		RX_CUDA(cudaGetLastError());
		// the keys are spent once the survivors are out: they are the sort's second buffer
		cub::DoubleBuffer<uint64_t> sorted(h->d_sel_label.p, h->d_keys.p);
		const int n = int(size_t(cq) * nprobe);
		size_t sortBytes = 0;
		RX_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, sortBytes, sorted, n, int(cq), h->d_seg_begin.p, h->d_seg_end.p, st));
		RX_CUDA(h->d_cub.ensure(sortBytes));
		RX_CUDA(cub::DeviceSegmentedSort::SortKeys(h->d_cub.p, sortBytes, sorted, n, int(cq), h->d_seg_begin.p, h->d_seg_end.p, st));
		ivf_coarse_emit_kernel<<<unsigned((size_t(n) + 255) / 256), 256, 0, st>>>(sorted.Current(), nq, nprobe, q0, cq, h->list_begin.p,
																				  h->own ? h->list_end.p : nullptr, h->d_work.p);
		RX_CUDA(cudaGetLastError());
		g_stats.launches += 4;
		g_stats.algorithmic_bytes += uint64_t(tiles) * nlist * ix->dim * 4;
	}
	return 0;
}

// the prologue of the key pass (rxgpu_ivf_search_knn_large_k, rxgpu_ivf_search_range_batch), under h->mtx: the coarse quantiser over
// the nq queries, probed rows per query (h->d_qrows, and rows on the host) and their exclusive scan, each query's first key
// (h->d_qoff; off[q] on the host, off[nq] = all probed rows).  2 launches after the coarse pass's.
int ivfProbedRows(const rxgpu_index* ix, rxgpu_ivf_device* h, uint32_t nq, const float* queries, uint32_t nprobe, cudaStream_t st,
				  std::vector<uint64_t>& rows, std::vector<uint64_t>& off) {
	RX_CUDA(h->d_qrows.ensure(nq));
	RX_CUDA(h->d_qoff.ensure(nq));
	if (int rc = ivfLaunchCoarse(ix, h, nq, queries, nprobe, st)) {
		return rc;
	}
	ivf_probe_rows_kernel<<<(nq + 7u) / 8u, 256, 0, st>>>(h->d_work.p, nq, nprobe, h->d_qrows.p);
	RX_CUDA(cudaGetLastError());
	size_t cubBytes = 0;
	RX_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, cubBytes, h->d_qrows.p, h->d_qoff.p, int(nq), st));
	RX_CUDA(h->d_cub.ensure(cubBytes));
	RX_CUDA(cub::DeviceScan::ExclusiveSum(h->d_cub.p, cubBytes, h->d_qrows.p, h->d_qoff.p, int(nq), st));
	rows.assign(nq, 0);
	off.assign(size_t(nq) + 1, 0);
	RX_CUDA(cudaMemcpyAsync(rows.data(), h->d_qrows.p, size_t(nq) * 8, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	for (uint32_t q = 0; q < nq; ++q) {
		off[q + 1] = off[q] + rows[q];
	}
	return 0;
}

// the query chunk [q0, return value): at most kIvfKeyCap keys and slotsPerQuery * queries <= kIvfSlotCap; a query above the key cap is a
// chunk of its own
uint32_t ivfChunkEnd(const std::vector<uint64_t>& off, uint32_t q0, uint64_t slotsPerQuery) {
	const uint32_t nq = uint32_t(off.size() - 1);
	uint32_t q1 = q0 + 1;
	while (q1 < nq && off[q1 + 1] - off[q0] <= kIvfKeyCap && uint64_t(q1 + 1 - q0) * slotsPerQuery <= kIvfSlotCap) {
		++q1;
	}
	return q1;
}

// the key pass of the chunk [q0, q0 + cq) (nkeys > 0): the exact scan in work-item key mode, one CTA per (query, probed list), every
// probed row's key to h->d_keys at the chunk's slot.  2 launches.
int ivfKeyPass(const rxgpu_index* ix, rxgpu_ivf_device* h, const IvfRows& r, uint32_t nq, uint32_t nprobe, uint32_t q0, uint32_t cq,
			   uint64_t nkeys, cudaStream_t st) {
	RX_CUDA(h->d_keys.ensure(std::max<uint64_t>(nkeys, 1)));
	RX_CUDA(h->d_work_chunk.ensure(size_t(cq) * nprobe));
	ivf_key_plan_kernel<<<(cq + 7u) / 8u, 256, 0, st>>>(h->d_work.p, nq, nprobe, q0, cq, h->d_qoff.p, h->d_work_chunk.p);
	RX_CUDA(cudaGetLastError());
	ScanArgs a = ivfScanArgs(ix, h, r, h->d_work_chunk.p, cq * nprobe, 1, kModeTopK);
	a.lists = h->d_keys.p;
	unsigned grid = 0;
	RX_CUDA(launchScan(ix, 1, a, &grid, st, false, true));
	return 0;
}

// survivors h->d_sel_ord / d_sel_label [n items, nseg segments [begin[i], end[i])) into (distance, label) order, in place: stable radix
// sorts by label, then by the ordered distance word (through d_sel_ord2 / d_sel_label2).  2 launches.
int ivfSortSurvivors(rxgpu_ivf_device* h, int n, int nseg, int* begin, int* end, cudaStream_t st) {
	size_t sortBytes = 0, sortBytes2 = 0;
	RX_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, sortBytes, h->d_sel_label.p, h->d_sel_label2.p, h->d_sel_ord.p,
													 h->d_sel_ord2.p, n, nseg, begin, end, 0, 64, st));
	RX_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(nullptr, sortBytes2, h->d_sel_ord2.p, h->d_sel_ord.p, h->d_sel_label2.p,
													 h->d_sel_label.p, n, nseg, begin, end, 0, 32, st));
	RX_CUDA(h->d_cub.ensure(std::max(sortBytes, sortBytes2)));
	RX_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(h->d_cub.p, sortBytes, h->d_sel_label.p, h->d_sel_label2.p, h->d_sel_ord.p,
													 h->d_sel_ord2.p, n, nseg, begin, end, 0, 64, st));
	RX_CUDA(cub::DeviceSegmentedRadixSort::SortPairs(h->d_cub.p, sortBytes2, h->d_sel_ord2.p, h->d_sel_ord.p, h->d_sel_label2.p,
													 h->d_sel_label.p, n, nseg, begin, end, 0, 32, st));
	return 0;
}

// The fused path of rxgpu_ivf_search_knn (k <= kMaxFusedK1, nprobe <= 256 * kMergeOwn), under h->mtx: the coarse pass, the list scans
// with a fused top-k per (query, probed list), and one merge into out_* (rows of `stride` entries) under (distance, internal row),
// bit-equal distances not yet ordered by label.  Device outputs, enqueued on st.
int ivfFusedKnn(const rxgpu_index* ix, rxgpu_ivf_device* h, const IvfRows& r, uint32_t nq, const float* queries, uint32_t k, uint32_t nprobe,
				uint32_t stride, float* out_dist, uint32_t* out_idx, uint64_t* out_label, uint32_t* out_count, cudaStream_t st) {
	const size_t nwork = size_t(nq) * nprobe;
	RX_CUDA(h->d_lists.ensure(nwork * k));
	if (int rc = ivfLaunchCoarse(ix, h, nq, queries, nprobe, st)) {
		return rc;
	}
	// list scans: the exact scan kernel in work-item mode, one CTA per (query, probed list), fused top-k per CTA
	ScanArgs a = ivfScanArgs(ix, h, r, h->d_work.p, uint32_t(nwork), k, kModeTopK);
	a.lists = h->d_lists.p;
	if (scan_smem_bytes(1, ix->dim, k) > 100 * 1024) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: dimension/k combination exceeds the fused top-k shared-memory budget");
	}
	unsigned grid = 0;
	RX_CUDA(launchScan(ix, 1, a, &grid, st));
	MergeArgs m{};
	m.lists = h->d_lists.p;
	m.labels = r.labels;
	m.out_dist = out_dist;
	m.out_idx = out_idx;
	m.out_label = out_label;
	m.out_count = out_count;
	m.nlists = nprobe;
	m.qt = nq;  // lists are probe-major: list of (probe p, query q) = p * nq + q
	m.k1 = k;
	m.q_offset = 0;
	m.out_stride = stride;
	m.out_offset = 0;
	m.mode = kModeTopK;
	RX_CUDA(launchMergeLists(m, nq, st));
	g_stats.launches += 2;  // list scans, merge (the coarse pass counts its own)
	g_stats.passes = 1;
	return 0;
}

// called once per query chunk [q0, q0 + cq) with its nkeys probed rows: the chunk's survivors are in h->d_sel_ord / d_sel_label
// ([cq][k]), h->d_sel_count holds how many each query kept
using IvfChunkDone = std::function<int(uint32_t q0, uint32_t cq, uint64_t nkeys)>;

// The any-k select of rxgpu_ivf_search_knn_large_k, under h->mtx: the coarse pass over the nq queries, then per query chunk the key pass
// and the exact select of the k smallest keys ((distance, internal row)), their survivors ordered by (distance word, selLabels' word)
// -- selLabels = the rows' labels, or nullptr for the rows themselves -- and handed to `done`.  Adds launches and bytes to g_stats.
int ivfSelectChunks(const rxgpu_index* ix, rxgpu_ivf_device* h, const IvfRows& r, uint32_t nq, const float* queries, uint32_t k, uint32_t nprobe,
					const uint64_t* selLabels, const IvfChunkDone& done, cudaStream_t st) {
	uint32_t launches = 2;  // probed rows, their scan (one CUB call); the coarse pass counts its own
	std::vector<uint64_t> rows, off;
	if (int rc = ivfProbedRows(ix, h, nq, queries, nprobe, st, rows, off)) {
		return rc;
	}
	// query chunks: at most kIvfKeyCap keys and kIvfSlotCap survivor slots each; a query above the key cap is a chunk of its own
	for (uint32_t q0 = 0, q1 = 0; q0 < nq; q0 = q1) {
		q1 = ivfChunkEnd(off, q0, k);
		const uint32_t cq = q1 - q0;
		const uint64_t nkeys = off[q1] - off[q0];
		const size_t slots = size_t(cq) * k;
		RX_CUDA(h->d_sel_ord.ensure(slots));
		RX_CUDA(h->d_sel_ord2.ensure(slots));
		RX_CUDA(h->d_sel_label.ensure(slots));
		RX_CUDA(h->d_sel_label2.ensure(slots));
		RX_CUDA(h->d_sel_count.ensure(cq));
		RX_CUDA(h->d_seg_begin.ensure(cq));
		RX_CUDA(h->d_seg_end.ensure(cq));
		RX_CUDA(cudaMemsetAsync(h->d_sel_count.p, 0, size_t(cq) * 4, st));
		if (nkeys) {
			if (int rc = ivfKeyPass(ix, h, r, nq, nprobe, q0, cq, nkeys, st)) {
				return rc;
			}
			ivf_select_cta_kernel<<<cq, kIvfSelThreads, 0, st>>>(h->d_keys.p, h->d_qoff.p + q0, h->d_qrows.p + q0, off[q0], k, selLabels,
															  h->d_sel_ord.p, h->d_sel_label.p, h->d_sel_count.p);
			RX_CUDA(cudaGetLastError());
			launches += 3;
			for (uint32_t qi = 0; qi < cq; ++qi) {  // queries with many keys: the same select over many CTAs
				const uint64_t n = rows[q0 + qi];
				if (n <= kIvfSelCtaKeys) {
					continue;
				}
				RX_CUDA(h->d_sel_state.ensure(1));
				RX_CUDA(h->d_sel_hist.ensure(kIvfSelBins));
				const SelState init{0ull, kKeyNone, k, 0u};
				RX_CUDA(cudaMemcpyAsync(h->d_sel_state.p, &init, sizeof(init), cudaMemcpyHostToDevice, st));
				RX_CUDA(cudaMemsetAsync(h->d_sel_hist.p, 0, kIvfSelBins * 4, st));
				const uint64_t* kq = h->d_keys.p + (off[q0 + qi] - off[q0]);
				const unsigned g = unsigned(std::min<uint64_t>((n + 16 * kIvfSelThreads - 1) / (16 * kIvfSelThreads), uint64_t(ix->sm_count) * 2));
				for (int pass = 0; pass < kIvfSelPasses; ++pass) {
					ivf_select_hist_kernel<<<g, kIvfSelThreads, 0, st>>>(kq, n, h->d_sel_state.p, pass, h->d_sel_hist.p);
					ivf_select_pick_kernel<<<1, kIvfSelThreads, 0, st>>>(h->d_sel_state.p, pass, h->d_sel_hist.p);
				}
				ivf_select_compact_kernel<<<g, kIvfSelThreads, 0, st>>>(kq, n, h->d_sel_state.p, selLabels, h->d_sel_ord.p + size_t(qi) * k,
																	 h->d_sel_label.p + size_t(qi) * k, h->d_sel_count.p + qi);
				RX_CUDA(cudaGetLastError());
				launches += 2 * kIvfSelPasses + 1;
			}
			// order the survivors by (distance, label): stable radix sorts by label, then by the ordered distance word
			ivf_sort_bounds_kernel<<<(cq + 255u) / 256u, 256, 0, st>>>(h->d_sel_count.p, k, cq, h->d_seg_begin.p, h->d_seg_end.p);
			RX_CUDA(cudaGetLastError());
			if (int rc = ivfSortSurvivors(h, int(slots), int(cq), h->d_seg_begin.p, h->d_seg_end.p, st)) {
				return rc;
			}
			launches += 3;
		}
		if (int rc = done(q0, cq, nkeys)) {
			return rc;
		}
	}
	const uint64_t probed = off[nq];
	g_stats.launches += launches;
	g_stats.passes = 1;
	// rows read once; each key written once and read once by the select
	g_stats.algorithmic_bytes += probed * ix->dim * 4 + (ix->metric == RXGPU_COS ? probed * 4 : 0) + probed * 16;
	return 0;
}

// The range batch of rxgpu_ivf_search_range_batch, under h->mtx (arguments checked): one coarse pass and one key pass per key chunk; each
// query's matches counted, kept, sorted by (distance, label) and gathered on the device.  emit(q, n, dist, label, m) once per query with
// its n matches in total and the best m = min(n, max_out) of them, best first (host arrays, valid during the call).
int ivfRangeBatch(const rxgpu_index* ix, rxgpu_ivf_device* h, uint32_t nq, const float* queries, const float* radius, uint32_t nprobe,
				  uint64_t max_out, const IvfRangeEmit& emit) {
	cudaStream_t st = ix->stream;
	const IvfRows r = ivfRows(ix, h);
	uint32_t launches = 2;  // probed rows, their scan; the coarse pass counts its own
	std::vector<uint64_t> rows, off;
	if (int rc = ivfProbedRows(ix, h, nq, queries, nprobe, st, rows, off)) {
		return rc;
	}
	RX_CUDA(h->d_radius.ensure(nq));
	RX_CUDA(cudaMemcpyAsync(h->d_radius.p, radius, size_t(nq) * 4, cudaMemcpyHostToDevice, st));
	std::vector<uint2> tiles;
	std::vector<size_t> tileAt;
	std::vector<uint32_t> cnt;
	std::vector<int> plan;
	std::vector<float> dist;
	std::vector<uint64_t> lab;
	// the key chunks of the any-k select (no survivor slots to bound yet: a query's matches are counted before they are kept)
	for (uint32_t q0 = 0, q1 = 0; q0 < nq; q0 = q1) {
		q1 = ivfChunkEnd(off, q0, 0);
		const uint32_t cq = q1 - q0;
		const uint64_t nkeys = off[q1] - off[q0];
		if (nkeys == 0) {
			for (uint32_t q = q0; q < q1; ++q) {
				emit(q, 0, nullptr, nullptr, 0);
			}
			continue;
		}
		if (int rc = ivfKeyPass(ix, h, r, nq, nprobe, q0, cq, nkeys, st)) {
			return rc;
		}
		tiles.clear();
		tileAt.assign(size_t(cq) + 1, 0);
		for (uint32_t qi = 0; qi < cq; ++qi) {
			for (uint64_t j = 0; j * kIvfRangeTile < rows[q0 + qi]; ++j) {
				tiles.push_back(make_uint2(qi, uint32_t(j)));
			}
			tileAt[qi + 1] = tiles.size();
		}
		RX_CUDA(h->d_tiles.ensure(tiles.size()));
		RX_CUDA(h->d_range_n.ensure(cq));
		RX_CUDA(h->d_sel_count.ensure(cq));
		RX_CUDA(cudaMemcpyAsync(h->d_tiles.p, tiles.data(), tiles.size() * sizeof(uint2), cudaMemcpyHostToDevice, st));
		RX_CUDA(cudaMemsetAsync(h->d_range_n.p, 0, size_t(cq) * 4, st));
		RX_CUDA(cudaMemsetAsync(h->d_sel_count.p, 0, size_t(cq) * 4, st));
		ivf_range_count_kernel<<<unsigned(tiles.size()), kIvfRangeThreads, 0, st>>>(
			h->d_keys.p, h->d_qoff.p + q0, h->d_qrows.p + q0, off[q0], h->d_radius.p + q0, h->d_tiles.p, h->d_range_n.p);
		RX_CUDA(cudaGetLastError());
		launches += 3;  // key plan, key scan, count
		cnt.resize(cq);
		RX_CUDA(cudaMemcpyAsync(cnt.data(), h->d_range_n.p, size_t(cq) * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		// survivor sub-chunks of at most kIvfSlotCap matches; a query with more is a sub-chunk of its own.  Without max_out nothing is kept.
		for (uint32_t s0 = 0, s1 = 0; s0 < cq; s0 = s1) {
			uint64_t total = cnt[s0];
			for (s1 = s0 + 1; s1 < cq && total + cnt[s1] <= kIvfSlotCap; ++s1) {
				total += cnt[s1];
			}
			if (total == 0 || max_out == 0) {
				for (uint32_t i = s0; i < s1; ++i) {
					emit(q0 + i, cnt[i], nullptr, nullptr, 0);
				}
				continue;
			}
			if (total > uint64_t(std::numeric_limits<int>::max())) {  // the segmented sorts count items in an int
				return fail(RXGPU_ERR_PARAMS, "rxgpu: more than 2^31 - 1 range matches for one IVF query");
			}
			const uint32_t ns = s1 - s0;
			plan.assign(2 * (size_t(ns) + 1), 0);
			int* seg = plan.data();     // survivors of query s0 + i: [seg[i], seg[i + 1])
			int* pack = seg + ns + 1;   // its best min(matches, max_out) in the packed output: [pack[i], pack[i + 1])
			int longest = 0;
			for (uint32_t i = 0; i < ns; ++i) {
				const int m = int(std::min<uint64_t>(cnt[s0 + i], max_out));
				seg[i + 1] = seg[i] + int(cnt[s0 + i]);
				pack[i + 1] = pack[i] + m;
				longest = std::max(longest, m);
			}
			RX_CUDA(h->d_range_seg.ensure(plan.size()));
			RX_CUDA(h->d_sel_ord.ensure(total));
			RX_CUDA(h->d_sel_ord2.ensure(total));
			RX_CUDA(h->d_sel_label.ensure(total));
			RX_CUDA(h->d_sel_label2.ensure(total));
			RX_CUDA(cudaMemcpyAsync(h->d_range_seg.p, plan.data(), plan.size() * sizeof(int), cudaMemcpyHostToDevice, st));
			int* dseg = h->d_range_seg.p;
			const int* dpack = dseg + ns + 1;
			ivf_range_emit_kernel<<<unsigned(tileAt[s1] - tileAt[s0]), kIvfRangeThreads, 0, st>>>(
				h->d_keys.p, h->d_qoff.p + q0, h->d_qrows.p + q0, off[q0], h->d_radius.p + q0, h->d_tiles.p + tileAt[s0], s0, dseg, r.labels,
				h->d_sel_count.p, h->d_sel_ord.p, h->d_sel_label.p);
			RX_CUDA(cudaGetLastError());
			if (int rc = ivfSortSurvivors(h, int(total), int(ns), dseg, dseg + 1, st)) {
				return rc;
			}
			// the packed output goes to the sorts' second buffers, free again once the sorts are done
			float* pdist = reinterpret_cast<float*>(h->d_sel_ord2.p);
			const dim3 gg(ns, unsigned(std::min(1024, (longest + 255) / 256)));
			ivf_range_gather_kernel<<<gg, 256, 0, st>>>(h->d_sel_ord.p, h->d_sel_label.p, dseg, dpack, pdist, h->d_sel_label2.p);
			RX_CUDA(cudaGetLastError());
			launches += 4;  // emit, two sorts, gather
			dist.resize(size_t(pack[ns]));
			lab.resize(size_t(pack[ns]));
			RX_CUDA(cudaMemcpyAsync(dist.data(), pdist, dist.size() * 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaMemcpyAsync(lab.data(), h->d_sel_label2.p, lab.size() * 8, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			for (uint32_t i = 0; i < ns; ++i) {
				emit(q0 + s0 + i, cnt[s0 + i], dist.data() + pack[i], lab.data() + pack[i], uint64_t(pack[i + 1] - pack[i]));
			}
		}
	}
	const uint64_t probed = off[nq];
	g_stats.launches += launches;
	g_stats.passes = 1;
	// as rxgpu_ivf_search_knn_large_k: rows read once; each key written once and read once
	g_stats.algorithmic_bytes += probed * ix->dim * 4 + (ix->metric == RXGPU_COS ? probed * 4 : 0) + probed * 16;
	return 0;
}
}  // namespace

namespace rxgpu {
cudaError_t ivfAssignRows(const rxgpu_index* ix, const float* centroids, const float* cnorm, uint32_t nlist, const float* x, uint32_t n,
						  uint64_t* keys, cudaStream_t st) {
	if (cudaError_t e = cudaMemsetAsync(keys, 0xFF, size_t(n) * 8, st)) {
		return e;
	}
	const int qt = coarseTile(ix, n);
	const size_t smem = coarse_smem_bytes(qt, ix->dim);
	const dim3 grid = coarseGrid(ix, nlist, n, qt);
	if (ix->metric == RXGPU_L2) {
		return qt == 1 ? launchCoarseDist<true, 1, true>(ix, centroids, nlist, grid, smem, x, n, cnorm, keys, st)
					   : launchCoarseDist<true, kCoarseTile, true>(ix, centroids, nlist, grid, smem, x, n, cnorm, keys, st);
	}
	return qt == 1 ? launchCoarseDist<false, 1, true>(ix, centroids, nlist, grid, smem, x, n, cnorm, keys, st)
				   : launchCoarseDist<false, kCoarseTile, true>(ix, centroids, nlist, grid, smem, x, n, cnorm, keys, st);
}
}  // namespace rxgpu

namespace {
// the view a sharded search compares across ranks, after ivfSearchChecks: a 64-bit FNV-1a of the centroids' bits (made once: the
// centroids never change while the lists exist), nlist, the clamped nprobe, and the rows the lists address (the shard's size in the
// (rank, local row) order the merge cuts ties by)
int ivfShardView(const rxgpu_index* ix, rxgpu_ivf_device* h, uint32_t nprobe, IvfShardView& v) {
	if (!h->fingerprint) {
		std::vector<uint32_t> hc(size_t(h->nlist) * ix->dim);
		RX_CUDA(cudaMemcpy2DAsync(hc.data(), size_t(ix->dim) * 4, h->centroids.p, size_t(ix->pitch) * 4, size_t(ix->dim) * 4, h->nlist,
								  cudaMemcpyDeviceToHost, ix->stream));
		RX_CUDA(cudaStreamSynchronize(ix->stream));
		uint64_t f = 0xcbf29ce484222325ull;
		for (const uint32_t w : hc) {
			f = (f ^ w) * 0x100000001b3ull;
		}
		h->fingerprint = f ? f : 1;
	}
	v = IvfShardView{h->fingerprint, h->nlist, nprobe, h->own ? h->high_water : ix->size};
	return 0;
}
}  // namespace

namespace rxgpu {
int ivfShardKnn(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, uint32_t nprobe, uint32_t stride, float* d_dist,
				uint32_t* d_idx, uint64_t* d_label, uint32_t* d_count, IvfShardView& view) {
	if (int rc = ivfSearchChecks(ix, k, kMaxLargeK, UINT32_MAX, nprobe)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	std::lock_guard<std::mutex> lck(h->mtx);
	cudaStream_t st = ix->stream;
	const IvfRows r = ivfRows(ix, h);
	if (int rc = ivfShardView(ix, h, nprobe, view)) {
		return rc;
	}
	if (k <= kMaxFusedK1 && nprobe <= 256u * kMergeOwn) {  // the path rxgpu_ivf_search_knn_large_k takes here
		if (int rc = ivfFusedKnn(ix, h, r, nq, queries, k, nprobe, stride, d_dist, d_idx, d_label, d_count, st)) {
			return rc;
		}
	} else {
		// the survivors by (distance word, row): the select keeps rows instead of labels, the emit looks the labels up
		const IvfChunkDone done = [&](uint32_t q0, uint32_t cq, uint64_t) -> int {
			const uint64_t slots = uint64_t(cq) * k;
			ivf_shard_emit_kernel<<<unsigned((slots + 255) / 256), 256, 0, st>>>(h->d_sel_ord.p, h->d_sel_label.p, h->d_sel_count.p, k, cq, r.labels,
																			   stride, d_dist + size_t(q0) * stride, d_idx + size_t(q0) * stride,
																			   d_label + size_t(q0) * stride, d_count + q0);
			RX_CUDA(cudaGetLastError());
			g_stats.launches += 1;
			return 0;
		};
		if (int rc = ivfSelectChunks(ix, h, r, nq, queries, k, nprobe, nullptr, done, st)) {
			return rc;
		}
	}
	RX_CUDA(cudaStreamSynchronize(st));
	return 0;
}

int ivfShardRange(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint32_t nprobe, uint64_t max_out,
				  const IvfRangeEmit& emit, IvfShardView& view) {
	if (int rc = ivfSearchChecks(ix, 0, 0, UINT32_MAX, nprobe)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	std::lock_guard<std::mutex> lck(h->mtx);
	if (int rc = ivfShardView(ix, h, nprobe, view)) {
		return rc;
	}
	return ivfRangeBatch(ix, h, nq, queries, radius, nprobe, max_out, emit);
}
}  // namespace rxgpu

extern "C" {

int rxgpu_ivf_import(rxgpu_index* ix, uint32_t nlist, const float* centroids, const uint64_t* list_sizes) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!centroids || !list_sizes || nlist == 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (nlist > kIvfMaxCentroids) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: at most 131072 IVF centroids (the reference's centroids_count bound)");
	}
	try {
		std::vector<uint32_t> begin(size_t(nlist) + 1, 0u);
		uint64_t total = 0;
		for (uint32_t l = 0; l < nlist; ++l) {
			total += list_sizes[l];
			if (total > ix->size) {
				break;
			}
			begin[l + 1] = uint32_t(total);
		}
		if (total != ix->size) {
			return fail(RXGPU_ERR_LOGIC, "rxgpu: IVF list sizes do not add up to the number of rows in the index");
		}
		auto h = std::make_unique<rxgpu_ivf_device>();
		h->nlist = nlist;
		RX_CUDA(h->centroids.ensure(size_t(nlist) * ix->pitch));
		RX_CUDA(h->list_begin.ensure(size_t(nlist) + 1));
		// on the index's stream, which the IVF kernels use: a legacy-stream copy would not be ordered before them
		RX_CUDA(cudaMemsetAsync(h->centroids.p, 0, size_t(nlist) * ix->pitch * sizeof(float), ix->stream));
		RX_CUDA(cudaMemcpy2DAsync(h->centroids.p, size_t(ix->pitch) * 4, centroids, size_t(ix->dim) * 4, size_t(ix->dim) * 4, nlist,
								  cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaMemcpyAsync(h->list_begin.p, begin.data(), begin.size() * 4, cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaStreamSynchronize(ix->stream));
		if (ix->metric == RXGPU_COS) {
			RX_CUDA(h->cnorm.ensure(nlist));
			RX_CUDA(launchNormCoefs(h->centroids.p, ix->pitch, ix->dim, 0, nlist, h->cnorm.p, ix->stream));
			RX_CUDA(cudaStreamSynchronize(ix->stream));
		}
		h->index_version = ix->version;
		if (ix->ivf) {
			ivfRelease(ix->ivf);
		}
		ix->ivf = h.release();
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_ivf_search_knn(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, uint32_t nprobe, float* out_dist,
						 uint64_t* out_label, uint32_t* out_count) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (!queries || !out_count || (k && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (int rc = ivfSearchChecks(ix, k, kMaxFusedK1, 256u * kMergeOwn, nprobe)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	std::lock_guard<std::mutex> lck(h->mtx);
	cudaStream_t st = ix->stream;
	const IvfRows r = ivfRows(ix, h);
	RX_CUDA(h->d_dist.ensure(size_t(nq) * k));
	RX_CUDA(h->d_idx.ensure(size_t(nq) * k));
	RX_CUDA(h->d_label.ensure(size_t(nq) * k));
	RX_CUDA(h->d_count.ensure(nq));
	if (int rc = ivfFusedKnn(ix, h, r, nq, queries, k, nprobe, k, h->d_dist.p, h->d_idx.p, h->d_label.p, h->d_count.p, st)) {
		return rc;
	}
	try {
		std::vector<float> hd(size_t(nq) * k);
		std::vector<uint64_t> hl(size_t(nq) * k);
		std::vector<uint32_t> hi(size_t(nq) * k), hc(nq);
		RX_CUDA(cudaMemcpyAsync(hd.data(), h->d_dist.p, hd.size() * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(hl.data(), h->d_label.p, hl.size() * 8, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(hi.data(), h->d_idx.p, hi.size() * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(hc.data(), h->d_count.p, hc.size() * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		std::vector<Hit> hits;
		for (uint32_t q = 0; q < nq; ++q) {
			hits.clear();
			for (uint32_t j = 0; j < std::min(hc[q], k); ++j) {
				hits.push_back(Hit{hd[size_t(q) * k + j], hi[size_t(q) * k + j], hl[size_t(q) * k + j]});
			}
			orderTiesByLabel(hits);  // FAISS' heap leaves bit-equal distances in no particular order: (distance, label) here
			for (size_t j = 0; j < hits.size(); ++j) {
				out_dist[size_t(q) * k + j] = hits[j].dist;
				out_label[size_t(q) * k + j] = hits[j].label;
			}
			out_count[q] = uint32_t(hits.size());
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_ivf_search_knn_large_k(const rxgpu_index* ix, uint32_t nq, const float* queries, uint32_t k, uint32_t nprobe, float* out_dist,
								 uint64_t* out_label, uint32_t* out_count) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (!queries || !out_count || (k && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (int rc = ivfSearchChecks(ix, k, kMaxLargeK, UINT32_MAX, nprobe)) {
		return rc;
	}
	if (k <= kMaxFusedK1 && nprobe <= 256u * kMergeOwn) {  // what the fused per-list top-k serves: that path, same bits
		return rxgpu_ivf_search_knn(ix, nq, queries, k, nprobe, out_dist, out_label, out_count);
	}
	rxgpu_ivf_device* h = ix->ivf;
	std::lock_guard<std::mutex> lck(h->mtx);
	cudaStream_t st = ix->stream;
	const IvfRows r = ivfRows(ix, h);
	try {
		std::vector<uint32_t> ord, cnt;
		std::vector<uint64_t> lab;
		const IvfChunkDone done = [&](uint32_t q0, uint32_t cq, uint64_t nkeys) -> int {
			const size_t slots = size_t(cq) * k;
			ord.resize(slots);
			lab.resize(slots);
			cnt.resize(cq);
			RX_CUDA(cudaMemcpyAsync(cnt.data(), h->d_sel_count.p, size_t(cq) * 4, cudaMemcpyDeviceToHost, st));
			if (nkeys) {
				RX_CUDA(cudaMemcpyAsync(ord.data(), h->d_sel_ord.p, slots * 4, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaMemcpyAsync(lab.data(), h->d_sel_label.p, slots * 8, cudaMemcpyDeviceToHost, st));
			}
			RX_CUDA(cudaStreamSynchronize(st));
			for (uint32_t qi = 0; qi < cq; ++qi) {
				const size_t at = size_t(q0 + qi) * k, from = size_t(qi) * k;
				for (uint32_t j = 0; j < cnt[qi]; ++j) {
					out_dist[at + j] = key_dist(ord[from + j], false);  // as the fused path decodes it: a zero distance is +0
					out_label[at + j] = lab[from + j];
				}
				out_count[q0 + qi] = cnt[qi];
			}
			return 0;
		};
		return ivfSelectChunks(ix, h, r, nq, queries, k, nprobe, r.labels, done, st);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_ivf_search_range(const rxgpu_index* ix, const float* query, float radius, uint32_t nprobe, uint64_t max_out, float* out_dist,
						   uint64_t* out_label, uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!query || !out_n || (max_out && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	*out_n = 0;
	g_stats = rxgpu_search_stats{};
	if (int rc = ivfSearchChecks(ix, 0, 0, UINT32_MAX, nprobe)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	std::lock_guard<std::mutex> lck(h->mtx);
	cudaStream_t st = ix->stream;
	const IvfRows r = ivfRows(ix, h);
	if (int rc = ivfLaunchCoarse(ix, h, 1, query, nprobe, st)) {
		return rc;
	}
	// like the brute-force range search: grow the result buffer and rescan when it was too small
	ScanArgs a = ivfScanArgs(ix, h, r, h->d_work.p, nprobe, 1, kModeRange);
	a.bound = radius;
	a.range_cap = std::max<uint64_t>(h->d_range.n, 1u << 14);
	try {
		std::vector<Hit> res;
		uint32_t scans = 0;
		const int rc = scanRangeHits(ix, st, a, h->d_range, h->d_range_count, h->h_range, r.h_labels, res, scans);
		g_stats.launches += scans;
		if (rc) {
			return rc;
		}
		*out_n = res.size();  // IvfIndex sorts the range result by distance (ivf_index.cc:220-224); ties by label here
		const uint64_t nout = std::min<uint64_t>(res.size(), max_out);
		for (uint64_t j = 0; j < nout; ++j) {
			out_dist[j] = res[j].dist;
			out_label[j] = res[j].label;
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_ivf_search_range_batch(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* radius, uint32_t nprobe,
								 uint64_t max_out, float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (!queries || !radius || !out_n || (max_out && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (int rc = ivfSearchChecks(ix, 0, 0, UINT32_MAX, nprobe)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	std::lock_guard<std::mutex> lck(h->mtx);
	try {
		const IvfRangeEmit emit = [&](uint32_t q, uint64_t n, const float* dist, const uint64_t* label, uint64_t m) {
			out_n[q] = n;
			std::copy(dist, dist + m, out_dist + size_t(q) * max_out);
			std::copy(label, label + m, out_label + size_t(q) * max_out);
		};
		return ivfRangeBatch(ix, h, nq, queries, radius, nprobe, max_out, emit);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

}  // extern "C"

// ---- mutable IVF lists -----------------------------------------------------------------------------------------------------------
namespace {
using Slab = rxgpu_ivf_device::Slab;

// rows [src, src + n) of slab `from` to [dst, dst + n) of slab `to` (the same slab or its rewrite): the rows, their labels, Cosine norms
// and host label mirror, enqueued on the index's stream
cudaError_t ivfCopyRows(const rxgpu_index* ix, const Slab& from, Slab& to, uint64_t src, uint64_t dst, uint64_t n) {
	if (n == 0) {
		return cudaSuccess;
	}
	cudaStream_t st = ix->stream;
	cudaError_t e = cudaMemcpyAsync(to.rows + dst * ix->pitch, from.rows + src * ix->pitch, n * ix->pitch * sizeof(float), cudaMemcpyDeviceToDevice, st);
	if (e == cudaSuccess) {
		e = cudaMemcpyAsync(to.labels + dst, from.labels + src, n * sizeof(uint64_t), cudaMemcpyDeviceToDevice, st);
	}
	if (e == cudaSuccess && from.norms) {
		e = cudaMemcpyAsync(to.norms + dst, from.norms + src, n * sizeof(float), cudaMemcpyDeviceToDevice, st);
	}
	std::copy_n(from.h_labels.begin() + src, n, to.h_labels.begin() + dst);
	return e;
}

struct IvfMove {
	uint64_t src, dst, n;  // rows [src, src + n) of the old slab go to [dst, dst + n) of the new one
};
// rewrites the slab at `rows` rows with the old slab's regions `moves` copied over, then frees the old slab; the caller updates the lists'
// regions.  On failure the slab is unchanged.
int ivfRewriteSlab(rxgpu_index* ix, rxgpu_ivf_device* h, uint64_t rows, const std::vector<IvfMove>& moves) {
	Slab s;  // frees whatever it holds when it goes: the new rows on failure, the old ones on success
	s.h_labels.resize(rows);
	cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&s.rows), rows * ix->pitch * sizeof(float));
	if (e == cudaSuccess) {
		e = cudaMalloc(reinterpret_cast<void**>(&s.labels), rows * sizeof(uint64_t));
	}
	if (e == cudaSuccess && ix->metric == RXGPU_COS) {
		e = cudaMalloc(reinterpret_cast<void**>(&s.norms), rows * sizeof(float));
	}
	for (size_t i = 0; e == cudaSuccess && i < moves.size(); ++i) {
		e = ivfCopyRows(ix, h->slab, s, moves[i].src, moves[i].dst, moves[i].n);
	}
	if (e == cudaSuccess) {
		e = cudaStreamSynchronize(ix->stream);
	}
	if (e != cudaSuccess) {
		return fail(RXGPU_ERR_SYSTEM, std::string("CUDA error: ") + cudaGetErrorString(e) + " at the IVF slab rewrite");
	}
	h->slab.swap(s);
	h->slab_rows = rows;
	return 0;
}
// moves list l to the end of the slab with room for `need` rows (amortised x1.5 growth); the old region becomes dead space
int ivfRelocate(rxgpu_index* ix, rxgpu_ivf_device* h, uint32_t l, uint32_t need) {
	const uint32_t newCap = std::max<uint32_t>(32u, (need + need / 2 + 31u) & ~31u);
	const uint64_t want = h->high_water + newCap;
	if (want > h->slab_rows) {  // grow the slab, keeping its contents where they are
		if (want > 0xFFFFFFF0ull) {
			return fail(RXGPU_ERR_LOGIC, "rxgpu: IVF row slab exceeds 2^32 rows");
		}
		const uint64_t rows = std::min<uint64_t>(std::max<uint64_t>(want, h->slab_rows + h->slab_rows / 2), 0xFFFFFFF0ull);
		if (int rc = ivfRewriteSlab(ix, h, rows, {IvfMove{0, 0, h->high_water}})) {
			return rc;
		}
	}
	const uint64_t dst = h->high_water;
	RX_CUDA(ivfCopyRows(ix, h->slab, h->slab, h->begin[l], dst, h->size[l]));
	h->dead += h->cap[l];
	h->begin[l] = uint32_t(dst);
	h->cap[l] = newCap;
	h->high_water += newCap;
	h->relocations++;
	return 0;
}
// rewrites the slab without the dead regions (every list keeps 25 % slack)
int ivfCompact(rxgpu_index* ix, rxgpu_ivf_device* h) {
	uint64_t total = 0;
	std::vector<uint32_t> newBegin(h->nlist), newCap(h->nlist);
	std::vector<IvfMove> moves(h->nlist);
	for (uint32_t l = 0; l < h->nlist; ++l) {
		newBegin[l] = uint32_t(total);
		newCap[l] = std::max<uint32_t>(32u, (h->size[l] + h->size[l] / 4 + 31u) & ~31u);
		moves[l] = IvfMove{h->begin[l], total, h->size[l]};
		total += newCap[l];
	}
	if (int rc = ivfRewriteSlab(ix, h, total, moves)) {
		return rc;
	}
	h->begin.swap(newBegin);
	h->cap.swap(newCap);
	h->high_water = total;
	h->dead = 0;
	h->compactions++;
	return 0;
}
int ivfPushBounds(rxgpu_index* ix, rxgpu_ivf_device* h) {
	std::vector<uint32_t> end(h->nlist);
	for (uint32_t l = 0; l < h->nlist; ++l) {
		end[l] = h->begin[l] + h->size[l];
	}
	RX_CUDA(cudaMemcpyAsync(h->list_begin.p, h->begin.data(), size_t(h->nlist) * 4, cudaMemcpyHostToDevice, ix->stream));
	RX_CUDA(cudaMemcpyAsync(h->list_end.p, end.data(), size_t(h->nlist) * 4, cudaMemcpyHostToDevice, ix->stream));
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	return 0;
}
}  // namespace

extern "C" {

int rxgpu_ivf_create(rxgpu_index* ix, uint32_t nlist, const float* centroids) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->size != 0) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: rxgpu_ivf_create needs an empty index (the rows live in the lists)");
	}
	const std::vector<uint64_t> zeros(nlist ? nlist : 1, 0);
	if (int rc = rxgpu_ivf_import(ix, nlist, centroids, zeros.data())) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	try {
		h->own = true;
		h->begin.assign(nlist, 0u);
		h->size.assign(nlist, 0u);
		h->cap.assign(nlist, 0u);
		RX_CUDA(h->list_end.ensure(nlist));
		return ivfPushBounds(ix, h);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_ivf_add(rxgpu_index* ix, uint64_t n, const uint32_t* list_nos, const uint64_t* labels, const float* vecs) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	if (!h || !h->own) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: rxgpu_ivf_add needs lists made by rxgpu_ivf_create");
	}
	if (n == 0) {
		return 0;
	}
	if (!list_nos || !labels || !vecs) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	std::lock_guard<std::mutex> lck(h->mtx);
	try {
		std::unordered_set<uint64_t> seen;
		std::vector<uint32_t> adds(h->nlist, 0u);
		for (uint64_t i = 0; i < n; ++i) {
			if (list_nos[i] >= h->nlist) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF list number out of range");
			}
			if (h->where.count(labels[i]) || !seen.insert(labels[i]).second) {
				return fail(RXGPU_ERR_LOGIC, "rxgpu: the id is already in the IVF lists");
			}
			adds[list_nos[i]]++;
		}
		if (h->dead > h->live + n + 4096) {  // more dead space than rows: rewrite the slab before growing it further
			if (int rc = ivfCompact(ix, h)) {
				return rc;
			}
		}
		for (uint32_t l = 0; l < h->nlist; ++l) {
			if (adds[l] && h->size[l] + adds[l] > h->cap[l]) {
				if (int rc = ivfRelocate(ix, h, l, h->size[l] + adds[l])) {
					return rc;
				}
			}
		}
		cudaStream_t st = ix->stream;
		const uint64_t slice = std::max<uint64_t>(1, (uint64_t(64) << 20) / (size_t(ix->dim) * 4));
		std::vector<uint32_t> dst;
		for (uint64_t off = 0; off < n; off += slice) {
			const uint64_t cnt = std::min(slice, n - off);
			dst.resize(cnt);
			for (uint64_t i = 0; i < cnt; ++i) {
				const uint32_t l = list_nos[off + i];
				const uint32_t row = h->begin[l] + h->size[l];
				dst[i] = row;
				h->where.emplace(labels[off + i], std::make_pair(l, h->size[l]));
				h->slab.h_labels[row] = labels[off + i];
				h->size[l]++;
			}
			RX_CUDA(h->st_rows.ensure(cnt * ix->dim));
			RX_CUDA(h->st_dst.ensure(cnt));
			RX_CUDA(h->st_labels.ensure(cnt));
			RX_CUDA(cudaMemcpyAsync(h->st_rows.p, vecs + off * ix->dim, cnt * ix->dim * sizeof(float), cudaMemcpyHostToDevice, st));
			RX_CUDA(cudaMemcpyAsync(h->st_dst.p, dst.data(), cnt * 4, cudaMemcpyHostToDevice, st));
			RX_CUDA(cudaMemcpyAsync(h->st_labels.p, labels + off, cnt * 8, cudaMemcpyHostToDevice, st));
			RX_CUDA(scatterRows(h->st_rows.p, h->st_dst.p, h->st_labels.p, uint32_t(cnt), ix->dim, ix->pitch, h->slab.rows, h->slab.labels,
								h->slab.norms, st));
			RX_CUDA(cudaStreamSynchronize(st));  // `dst` is reused by the next slice
		}
		h->live += n;
		return ivfPushBounds(ix, h);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_ivf_remove(rxgpu_index* ix, uint64_t label) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	rxgpu_ivf_device* h = ix->ivf;
	if (!h || !h->own) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: rxgpu_ivf_remove needs lists made by rxgpu_ivf_create");
	}
	std::lock_guard<std::mutex> lck(h->mtx);
	const auto it = h->where.find(label);
	if (it == h->where.end()) {
		return fail(RXGPU_ERR_NOT_FOUND, "rxgpu: the id is not in the IVF lists");
	}
	// InvertedLists swap-remove (faiss DirectMap::remove_ids, Hashtable flavour): the list's last entry fills the hole
	const uint32_t l = it->second.first, pos = it->second.second, last = h->size[l] - 1;
	if (pos != last) {
		const uint64_t at = uint64_t(h->begin[l]) + pos;
		RX_CUDA(ivfCopyRows(ix, h->slab, h->slab, uint64_t(h->begin[l]) + last, at, 1));
		h->where[h->slab.h_labels[at]].second = pos;
	}
	h->where.erase(it);
	h->size[l] = last;
	h->live--;
	const uint32_t end = h->begin[l] + last;
	RX_CUDA(cudaMemcpyAsync(h->list_end.p + l, &end, 4, cudaMemcpyHostToDevice, ix->stream));
	RX_CUDA(cudaStreamSynchronize(ix->stream));
	return 0;
}

uint64_t rxgpu_ivf_size(const rxgpu_index* ix) { return ix && ix->ivf ? (ix->ivf->own ? ix->ivf->live : ix->size) : 0; }
int rxgpu_ivf_list_stats(const rxgpu_index* ix, uint64_t* slab_rows, uint64_t* dead_rows, uint64_t* relocations, uint64_t* compactions) {
	if (!ix || !ix->ivf) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no IVF lists in this index");
	}
	const rxgpu_ivf_device* h = ix->ivf;
	if (slab_rows) *slab_rows = h->slab_rows;
	if (dead_rows) *dead_rows = h->dead;
	if (relocations) *relocations = h->relocations;
	if (compactions) *compactions = h->compactions;
	return 0;
}

}  // extern "C"
