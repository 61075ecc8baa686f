// librxgpu: IVF training and list assignment on the device (rxgpu_ivf_train, rxgpu_ivf_assign, rxgpu_ivf_add_assign, rxgpu_kmeans_plan)
// -- faiss::Clustering::train as IndexIVFFlat::train reaches it, and quantizer->assign as IndexIVF::add_with_ids calls it.  The
// assignment is the coarse pass's distance kernel in argmin mode (ivf_coarse.cuh), launched by ivf.cu (ivfAssignRows); the update,
// split and renormalisation kernels are ivf_train.cuh's.  The host keeps what FAISS decides with its RNG: the sample, the initial centroids and which cluster an empty one
// splits.  rxgpu_sharded_ivf_train runs the same iterations over ranks: each assigns a slice of the sample, the keys are all-gathered.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <functional>
#include <limits>
#include <new>
#include <random>
#include <string>
#include <vector>

#include "../../include/rxgpu.h"
#include "internal.h"
#include "../host/knn_select.h"
#include "ivf_train.cuh"

using namespace rxgpu;

namespace {

// faiss::rand_perm (utils/random.cpp): Fisher-Yates with RandomGenerator(seed), i.e. std::mt19937((unsigned)seed), rand_int(max) = mt() % max
std::vector<int32_t> randPerm(size_t n, int64_t seed) {
	std::vector<int32_t> perm(n);
	for (size_t i = 0; i < n; ++i) {
		perm[i] = int32_t(i);
	}
	std::mt19937 mt(static_cast<unsigned int>(seed));
	for (size_t i = 0; i + 1 < n; ++i) {
		const int max = int(n - i);
		const size_t i2 = i + size_t(mt() % static_cast<unsigned long>(max));
		std::swap(perm[i], perm[i2]);
	}
	return perm;
}

// Clustering::train_encoded's sample (subsample_training_set with rand_perm, Clustering.cpp:88-138, 342-356) and the input rows of the
// initial centroids (rand_perm(nx, seed + 1), :440-451; the corner case nx == k copies the first k input rows, :358-383)
struct KmeansPlan {
	std::vector<int32_t> sample;   // empty: no subsampling, the sample is the input
	std::vector<int32_t> init;     // [nlist] input rows
	std::vector<int32_t> initPos;  // [nlist] their positions among the training rows (gatheredRow)
	uint64_t nx = 0;
	bool copy = false;             // nx == nlist: the centroids are the first nlist input rows, no iterations
};
KmeansPlan kmeansPlan(uint64_t n, uint32_t nlist, int32_t seed, int32_t maxPpc) {
	KmeansPlan p;
	p.nx = n;
	if (n > uint64_t(nlist) * uint64_t(maxPpc)) {
		std::vector<int32_t> perm = randPerm(n, seed);
		p.nx = uint64_t(nlist) * uint64_t(maxPpc);
		perm.resize(p.nx);
		p.sample = std::move(perm);
	}
	p.init.resize(nlist);
	p.initPos.resize(nlist);
	if (p.nx == nlist) {
		p.copy = true;
		for (uint32_t c = 0; c < nlist; ++c) {
			p.init[c] = p.initPos[c] = int32_t(c);
		}
		return p;
	}
	const std::vector<int32_t> perm = randPerm(p.nx, int64_t(seed) + 1);
	for (uint32_t c = 0; c < nlist; ++c) {
		p.initPos[c] = perm[c];
		p.init[c] = p.sample.empty() ? perm[c] : p.sample[perm[c]];
	}
	return p;
}

// the input row at position pos of what the training reads: the sample, or in the copy case the first nlist input rows (FAISS copies
// x_in, Clustering.cpp:358-383, even when the sample was drawn from more rows)
uint64_t gatheredRow(const KmeansPlan& p, uint64_t pos) { return p.copy || p.sample.empty() ? pos : uint64_t(p.sample[pos]); }

int checkPlanArgs(uint64_t n, uint32_t nlist, int32_t seed, int32_t maxPpc) {
	if (nlist == 0 || nlist > kIvfMaxCentroids) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF training needs nlist in [1, 131072]");
	}
	if (n < nlist) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF training needs at least as many points as centroids");
	}
	if (n > uint64_t(std::numeric_limits<int32_t>::max())) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF training takes at most 2^31 - 1 points (FAISS's permutation is int)");
	}
	if (seed < 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF training needs a seed >= 0 (a negative seed would be clock-based)");
	}
	if (maxPpc < 1) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: max_points_per_centroid must be >= 1");
	}
	return 0;
}

// The rows rows[0, cnt) of vecs (or vecs' rows first, first + cnt when rows is null) as the coarse quantiser sees them, dense [cnt][dim]:
// Cosine normalised (times norm_coefs[row] when given, else as rxgpu_select_knn normalises a query), the other metrics as they are
void prepareRows(const rxgpu_index* ix, const float* vecs, const float* normCoefs, const int32_t* rows, uint64_t first, uint64_t cnt,
				 float* out) {
	const uint32_t dim = ix->dim;
	for (uint64_t i = 0; i < cnt; ++i) {
		const uint64_t r = rows ? uint64_t(rows[first + i]) : first + i;
		const float* src = vecs + r * dim;
		float* dst = out + i * dim;
		if (ix->metric != RXGPU_COS) {
			std::copy_n(src, dim, dst);
		} else if (normCoefs) {
			const float k = normCoefs[r];
			for (uint32_t j = 0; j < dim; ++j) {
				dst[j] = src[j] * k;
			}
		} else {
			normalizeCopyVector(src, int32_t(dim), dst);
		}
	}
}

// uploads the prepared rows (see prepareRows) to d_out [cnt][dim] through a pinned staging buffer of about 64 MB
int uploadRows(const rxgpu_index* ix, const float* vecs, const float* normCoefs, const int32_t* rows, uint64_t first, uint64_t cnt,
			   float* d_out, PinBuf<float>& stage, cudaStream_t st) {
	const uint64_t slice = std::max<uint64_t>(1, (uint64_t(64) << 20) / (uint64_t(ix->dim) * 4));
	RX_CUDA(stage.ensure(std::min(slice, cnt) * ix->dim));
	for (uint64_t off = 0; off < cnt; off += slice) {
		const uint64_t m = std::min(slice, cnt - off);
		RX_CUDA(cudaStreamSynchronize(st));  // the previous slice has left the staging buffer
		prepareRows(ix, vecs, normCoefs, rows, first + off, m, stage.p);
		RX_CUDA(cudaMemcpyAsync(d_out + off * ix->dim, stage.p, m * ix->dim * 4, cudaMemcpyHostToDevice, st));
	}
	RX_CUDA(cudaStreamSynchronize(st));
	return 0;
}

int checkFinite(const rxgpu_index* ix, uint64_t n, const float* vecs, const float* normCoefs) {
	const uint32_t dim = ix->dim;
	const bool scaled = ix->metric == RXGPU_COS && normCoefs;
	for (uint64_t i = 0; i < n; ++i) {
		const float k = scaled ? normCoefs[i] : 1.f;
		for (uint32_t j = 0; j < dim; ++j) {
			if (!std::isfinite(vecs[i * dim + j] * k)) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF training input contains NaN's or Inf's");
			}
		}
	}
	return 0;
}

// split_clusters (Clustering.cpp:247-294) on FAISS's float histogram: the (empty, split) pairs in order, hassign updated as FAISS does
std::vector<uint2> chooseSplits(std::vector<float>& hassign, uint64_t n) {
	const size_t k = hassign.size();
	std::vector<uint2> splits;
	std::mt19937 mt(1234u);  // RandomGenerator rng(1234)
	for (size_t ci = 0; ci < k; ++ci) {
		if (hassign[ci] != 0) {
			continue;
		}
		size_t cj = 0;
		for (;; cj = (cj + 1) % k) {
			const float p = float((double(hassign[cj]) - 1.0) / double(float(n - k)));
			const float r = float(mt()) / float(mt.max());
			if (r < p) {
				break;
			}
		}
		splits.push_back(make_uint2(uint32_t(ci), uint32_t(cj)));
		hassign[ci] = hassign[cj] / 2;
		hassign[cj] -= hassign[ci];
	}
	return splits;
}

// the radix sort's scratch bytes for nx (centroid, point) pairs and the end bit that covers nlist centroids
struct KmeansSort {
	size_t bytes = 0;
	int endBit = 1;
};
int kmeansSort(uint64_t nx, uint32_t nlist, cudaStream_t st, KmeansSort& ks) {
	while ((1u << ks.endBit) < nlist) {
		++ks.endBit;
	}
	RX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, ks.bytes, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
											static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), int(nx), 0, ks.endBit, st));
	return 0;
}
// errSystem unless the device has room for the training set and one iteration's scratch (the points, their keys, (centroid, point) pairs
// twice for the sort, the centroids) plus `extra` bytes, for each of `sharers` trainings that allocate on this device at once; checked
// before anything reads the input
int checkTrainMemory(const rxgpu_index* ix, uint64_t nx, uint32_t nlist, const KmeansSort& ks, uint64_t extra, uint32_t sharers) {
	const uint64_t need =
		(nx * ix->dim * 4 + nx * (8 + 16) + ks.bytes + uint64_t(nlist) * (ix->pitch * 4 + 8) + (uint64_t(64) << 20) + extra) * sharers;
	size_t freeB = 0, totalB = 0;
	RX_CUDA(cudaMemGetInfo(&freeB, &totalB));
	if (need > freeB) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: not enough device memory for the IVF training set (" + std::to_string(need >> 20) + " MB needed, " +
										   std::to_string(freeB >> 20) + " MB free)");
	}
	return 0;
}

// writes the assignment keys of the caller's share of the points against the centroids (cent, cnorm) to keys
using KmeansAssign = std::function<int(const float* cent, const float* cnorm, uint64_t* keys)>;
// completes keys[0, nx) with the other ranks' shares
using KmeansExchange = std::function<int(uint64_t* keys)>;

// The k-means from its initial centroids on (faiss::Clustering::train_encoded after the sample and the init): `cent` [nlist][pitch]
// holds the initial centroids as prepared rows, `x` the nx prepared points and `keys` room for their keys (both when there are
// iterations).  Renormalises the initial centroids (spherical), runs the Lloyd iterations and leaves the index as
// rxgpu_ivf_create(nlist, centroids) would.  An iteration's keys come from `assign` then, when set, `exchange`; the update after them is
// this one code on every rank of a sharded training, so the same keys give the same centroids everywhere.
int kmeansRun(rxgpu_index* ix, uint32_t nlist, const KmeansPlan& plan, int niter, const KmeansSort& ks, DevBuf<float>& cent, DevBuf<float>& x,
			  DevBuf<uint64_t>& keys, const KmeansAssign& assign, const KmeansExchange& exchange, float* out_centroids,
			  rxgpu_ivf_train_stats* stats) {
	const bool spherical = ix->metric != RXGPU_L2;  // IndexIVF sets cp.spherical for METRIC_INNER_PRODUCT (IndexIVF.cpp:179-182)
	const uint32_t dim = ix->dim, pitch = ix->pitch;
	const uint64_t nx = plan.nx;
	cudaStream_t st = ix->stream;
	if (stats) {
		std::fill(stats, stats + niter, rxgpu_ivf_train_stats{0.0, 0, 0.f, 0.f, 0.f});
	}
	if (spherical && !plan.copy) {  // post_process_centroids of the initial centroids
		kmeans_renorm_kernel<<<(nlist + 7u) / 8u, 256, 0, st>>>(cent.p, pitch, dim, nlist);
		RX_CUDA(cudaGetLastError());
	}
	if (!plan.copy && niter > 0) {
		DevBuf<float> cnorm;
		DevBuf<uint32_t> assign1, point, assign2, point2, off;
		DevBuf<uint2> splits;
		DevBuf<unsigned char> cubTmp;
		RX_CUDA(assign1.ensure(nx));
		RX_CUDA(point.ensure(nx));
		RX_CUDA(assign2.ensure(nx));
		RX_CUDA(point2.ensure(nx));
		RX_CUDA(off.ensure(size_t(nlist) + 1));
		RX_CUDA(cubTmp.ensure(std::max<size_t>(ks.bytes, 1)));
		if (ix->metric == RXGPU_COS) {
			RX_CUDA(cnorm.ensure(nlist));
		}
		cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
		struct EventsGuard {
			cudaEvent_t* e;
			~EventsGuard() {
				for (int i = 0; i < 6; ++i) {
					if (e[i]) {
						cudaEventDestroy(e[i]);
					}
				}
			}
		} evGuard{ev};
		for (int i = 0; i < 6; ++i) {
			RX_CUDA(cudaEventCreate(&ev[i]));
		}
		std::vector<uint64_t> hkeys(nx);
		std::vector<uint32_t> counts(nlist), hoff(size_t(nlist) + 1);
		std::vector<float> hassign(nlist);
		size_t sortBytes = ks.bytes;
		for (int it = 0; it < niter; ++it) {
			// the centroids as the index holds them for the search: Cosine norm coefficients (IndexFlatCosine::add)
			if (ix->metric == RXGPU_COS) {
				RX_CUDA(launchNormCoefs(cent.p, pitch, dim, 0, nlist, cnorm.p, st));
			}
			RX_CUDA(cudaEventRecord(ev[0], st));
			if (int rc = assign(cent.p, cnorm.p, keys.p)) {
				return rc;
			}
			RX_CUDA(cudaEventRecord(ev[1], st));
			if (exchange) {
				if (int rc = exchange(keys.p)) {
					return rc;
				}
			}
			RX_CUDA(cudaEventRecord(ev[5], st));
			kmeans_split_keys_kernel<<<unsigned((nx + 255) / 256), 256, 0, st>>>(keys.p, uint32_t(nx), assign1.p, point.p);
			RX_CUDA(cudaGetLastError());
			RX_CUDA(cub::DeviceRadixSort::SortPairs(cubTmp.p, sortBytes, assign1.p, assign2.p, point.p, point2.p, int(nx), 0, ks.endBit, st));
			RX_CUDA(cudaEventRecord(ev[2], st));
			RX_CUDA(cudaEventSynchronize(ev[2]));  // the host clock below starts once the device work before it is done
			// the host's part: the keys back, the objective, the histogram, split_clusters' choices, the offsets out
			const auto h0 = std::chrono::steady_clock::now();
			RX_CUDA(cudaMemcpyAsync(hkeys.data(), keys.p, nx * 8, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			// objective (in FAISS's convention) and the histogram
			double obj = 0.0;
			std::fill(counts.begin(), counts.end(), 0u);
			for (uint64_t i = 0; i < nx; ++i) {
				const float d = key_dist(uint32_t(hkeys[i] >> 32), false);
				obj += ix->metric == RXGPU_L2 ? double(d) : -double(d);
				counts[uint32_t(hkeys[i])]++;
			}
			hoff[0] = 0;
			for (uint32_t c = 0; c < nlist; ++c) {
				hoff[c + 1] = hoff[c] + counts[c];
				hassign[c] = float(std::min<uint32_t>(counts[c], 1u << 24));
			}
			const std::vector<uint2> sp = chooseSplits(hassign, nx);
			RX_CUDA(cudaMemcpyAsync(off.p, hoff.data(), hoff.size() * 4, cudaMemcpyHostToDevice, st));
			if (!sp.empty()) {
				RX_CUDA(splits.ensure(sp.size()));
				RX_CUDA(cudaMemcpyAsync(splits.p, sp.data(), sp.size() * sizeof(uint2), cudaMemcpyHostToDevice, st));
			}
			RX_CUDA(cudaStreamSynchronize(st));
			const float hostMs = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - h0).count();
			RX_CUDA(cudaEventRecord(ev[3], st));
			kmeans_update_kernel<<<dim3(nlist, (dim + 127u) / 128u), 128, 0, st>>>(x.p, dim, point2.p, off.p, cent.p, pitch);
			RX_CUDA(cudaGetLastError());
			if (!sp.empty()) {
				kmeans_split_kernel<<<(dim + 127u) / 128u, 128, 0, st>>>(splits.p, uint32_t(sp.size()), dim, cent.p, pitch);
				RX_CUDA(cudaGetLastError());
			}
			if (spherical) {
				kmeans_renorm_kernel<<<(nlist + 7u) / 8u, 256, 0, st>>>(cent.p, pitch, dim, nlist);
				RX_CUDA(cudaGetLastError());
			}
			RX_CUDA(cudaEventRecord(ev[4], st));
			RX_CUDA(cudaStreamSynchronize(st));
			if (stats) {
				float a = 0.f, u0 = 0.f, u1 = 0.f;
				RX_CUDA(cudaEventElapsedTime(&a, ev[0], ev[1]));
				RX_CUDA(cudaEventElapsedTime(&u0, ev[5], ev[2]));
				RX_CUDA(cudaEventElapsedTime(&u1, ev[3], ev[4]));
				stats[it] = rxgpu_ivf_train_stats{obj, int32_t(sp.size()), a, u0 + u1, hostMs};
			}
		}
	}
	std::vector<float> hc(size_t(nlist) * dim);
	RX_CUDA(cudaMemcpy2DAsync(hc.data(), size_t(dim) * 4, cent.p, size_t(pitch) * 4, size_t(dim) * 4, nlist, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	// the scratch goes before the lists are made
	x.release();
	keys.release();
	if (int rc = rxgpu_ivf_create(ix, nlist, hc.data())) {
		return rc;
	}
	if (out_centroids) {
		std::copy(hc.begin(), hc.end(), out_centroids);
	}
	return 0;
}

}  // namespace

extern "C" {

int rxgpu_kmeans_plan(uint64_t n, uint32_t nlist, int32_t seed, int32_t max_points_per_centroid, int32_t* out_sample, int32_t* out_init) {
	if (!out_init) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (int rc = checkPlanArgs(n, nlist, seed, max_points_per_centroid)) {
		return rc;
	}
	try {
		const KmeansPlan p = kmeansPlan(n, nlist, seed, max_points_per_centroid);
		if (out_sample) {
			if (p.sample.empty()) {
				for (uint64_t i = 0; i < n; ++i) {
					out_sample[i] = int32_t(i);
				}
			} else {
				std::copy(p.sample.begin(), p.sample.end(), out_sample);
			}
		}
		std::copy(p.init.begin(), p.init.end(), out_init);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_ivf_train(rxgpu_index* ix, uint32_t nlist, uint64_t n, const float* vecs, const float* norm_coefs, const rxgpu_ivf_train_params* params,
					float* out_centroids, rxgpu_ivf_train_stats* stats) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->size != 0 || ix->ivf) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: rxgpu_ivf_train needs an empty index with no IVF lists attached");
	}
	const rxgpu_ivf_train_params prm = params ? *params : rxgpu_ivf_train_params{10, 1234, 256};
	if (!vecs && n) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (prm.niter < 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: niter must be >= 0");
	}
	if (int rc = checkPlanArgs(n, nlist, prm.seed, prm.max_points_per_centroid)) {
		return rc;
	}
	if (int rc = ivfCheckCoarseDim(ix->dim)) {
		return rc;
	}
	const uint32_t dim = ix->dim, pitch = ix->pitch;
	cudaStream_t st = ix->stream;
	const uint64_t nx = std::min<uint64_t>(n, uint64_t(nlist) * uint64_t(prm.max_points_per_centroid));
	KmeansSort ks;
	if (int rc = kmeansSort(nx, nlist, st, ks)) {
		return rc;
	}
	if (int rc = checkTrainMemory(ix, nx, nlist, ks, 0, 1)) {
		return rc;
	}
	if (int rc = checkFinite(ix, n, vecs, norm_coefs)) {
		return rc;
	}
	try {
		const KmeansPlan plan = kmeansPlan(n, nlist, prm.seed, prm.max_points_per_centroid);
		DevBuf<float> x, cent;
		DevBuf<uint64_t> keys;
		PinBuf<float> stage;
		RX_CUDA(cent.ensure(size_t(nlist) * pitch));
		RX_CUDA(cudaMemsetAsync(cent.p, 0, size_t(nlist) * pitch * 4, st));
		// initial centroids: input rows (the sample's perm[c]-th, prepared as the sample is)
		{
			RX_CUDA(x.ensure(size_t(nlist) * dim));
			if (int rc = uploadRows(ix, vecs, norm_coefs, plan.init.data(), 0, nlist, x.p, stage, st)) {
				return rc;
			}
			RX_CUDA(cudaMemcpy2DAsync(cent.p, size_t(pitch) * 4, x.p, size_t(dim) * 4, size_t(dim) * 4, nlist, cudaMemcpyDeviceToDevice, st));
		}
		if (!plan.copy && prm.niter > 0) {
			x.release();
			RX_CUDA(x.ensure(size_t(nx) * dim));
			if (int rc = uploadRows(ix, vecs, norm_coefs, plan.sample.empty() ? nullptr : plan.sample.data(), 0, nx, x.p, stage, st)) {
				return rc;
			}
			RX_CUDA(keys.ensure(nx));
		}
		const KmeansAssign assign = [&](const float* c, const float* cn, uint64_t* k) -> int {
			RX_CUDA(ivfAssignRows(ix, c, cn, nlist, x.p, uint32_t(nx), k, st));
			return 0;
		};
		return kmeansRun(ix, nlist, plan, prm.niter, ks, cent, x, keys, assign, nullptr, out_centroids, stats);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_sharded_ivf_train(rxgpu_comm* c, rxgpu_index* ix, uint32_t nlist, uint64_t n_local, const float* vecs_local,
							const float* norm_coefs_local, const rxgpu_ivf_train_params* params, float* out_centroids, rxgpu_ivf_train_stats* stats) {
	if (!c) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null communicator");
	}
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	const rxgpu_ivf_train_params prm = params ? *params : rxgpu_ivf_train_params{10, 1234, 256};
	// what this rank alone can find wrong travels with its row count and parameters, so every rank learns it from the one exchange
	int status = 0;
	std::string why;
	if (ix->device != commDevice(c)) {
		status = fail(RXGPU_ERR_PARAMS, "rxgpu: the shard lives on another device than its communicator");
	} else if (ix->size != 0 || ix->ivf) {
		status = fail(RXGPU_ERR_LOGIC, "rxgpu: rxgpu_sharded_ivf_train needs an empty index with no IVF lists attached");
	} else if (!vecs_local && n_local) {
		status = fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (status) {
		why = g_err;
	}
	const uint32_t R = uint32_t(commSize(c)), me = uint32_t(commRank(c)), dim = ix->dim, pitch = ix->pitch;
	cudaStream_t st = ix->stream;
	std::lock_guard<std::mutex> lck(commMutex(c));
	try {
		// ---- 1. every rank's row count, parameters, status and device (ranks on one device share its memory)
		struct Hello {
			uint64_t n;
			uint32_t nlist, dim, metric;
			int32_t niter, seed, maxPpc, status, pad;
			cudaUUID_t device;
		};
		static_assert(sizeof(Hello) == 56, "Hello layout");
		std::vector<Hello> hello(R);
		DevBuf<Hello> dHello;
		RX_CUDA(dHello.ensure(size_t(R) + 1));
		cudaDeviceProp prop{};
		RX_CUDA(cudaGetDeviceProperties(&prop, ix->device));
		const Hello mine{n_local, nlist, dim, uint32_t(ix->metric), prm.niter, prm.seed, prm.max_points_per_centroid, status, 0, prop.uuid};
		RX_CUDA(cudaMemcpyAsync(dHello.p + R, &mine, sizeof(Hello), cudaMemcpyHostToDevice, st));
		if (int rc = commAllGather(c, dHello.p + R, dHello.p, sizeof(Hello), st)) {
			return rc;
		}
		RX_CUDA(cudaMemcpyAsync(hello.data(), dHello.p, size_t(R) * sizeof(Hello), cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		uint64_t N = 0, base = 0;
		uint32_t sharers = 0;
		std::vector<uint64_t> bases(R);
		for (uint32_t r = 0; r < R; ++r) {
			const Hello& h = hello[r];
			sharers += std::memcmp(&h.device, &prop.uuid, sizeof(cudaUUID_t)) == 0 ? 1u : 0u;
			if (h.status) {
				return fail(h.status, r == me ? why : "rxgpu: sharded IVF training failed on rank " + std::to_string(r));
			}
			if (h.nlist != nlist || h.dim != dim || h.metric != uint32_t(ix->metric) || h.niter != prm.niter || h.seed != prm.seed ||
				h.maxPpc != prm.max_points_per_centroid) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: the ranks of a sharded IVF training disagree on nlist, dim, metric or the parameters");
			}
			bases[r] = N;
			N += h.n;
		}
		base = bases[me];
		// ---- 2. the checks of rxgpu_ivf_train on the whole input: the same verdict on every rank
		if (prm.niter < 0) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: niter must be >= 0");
		}
		if (int rc = checkPlanArgs(N, nlist, prm.seed, prm.max_points_per_centroid)) {
			return rc;
		}
		if (int rc = ivfCheckCoarseDim(dim)) {
			return rc;
		}
		// ---- 3. the training rows (the sample; the first nlist rows in the copy case): which rank owns each, where it lands in the all-gather
		const KmeansPlan plan = kmeansPlan(N, nlist, prm.seed, prm.max_points_per_centroid);
		const uint64_t nx = plan.nx;
		std::vector<uint8_t> owner(nx);
		std::vector<uint64_t> owned(R, 0);
		for (uint64_t pos = 0; pos < nx; ++pos) {
			const uint64_t row = gatheredRow(plan, pos);
			const uint32_t r = uint32_t(std::upper_bound(bases.begin(), bases.end(), row) - bases.begin()) - 1;
			owner[pos] = uint8_t(r);
			owned[r]++;
		}
		const uint64_t maxc = *std::max_element(owned.begin(), owned.end());
		const uint64_t slice = (nx + R - 1) / R;  // the points each rank assigns
		// ---- 4. the checks of this rank alone, agreed before the first large exchange: the largest error code wins on every rank.  The
		// memory check counts every rank on this device: they allocate at the same time.
		KmeansSort ks;
		status = kmeansSort(nx, nlist, st, ks);
		if (!status) {
			status = checkTrainMemory(ix, nx, nlist, ks, (uint64_t(R) + 1) * maxc * dim * 4 + nx * 8 + (uint64_t(R) * slice - nx) * 8, sharers);
		}
		if (!status) {
			status = checkFinite(ix, n_local, vecs_local, norm_coefs_local);
		}
		if (status) {
			why = g_err;
		}
		{
			DevBuf<uint32_t> dStatus;
			RX_CUDA(dStatus.ensure(1));
			const uint32_t s32 = uint32_t(status);
			uint32_t all = 0;
			RX_CUDA(cudaMemcpyAsync(dStatus.p, &s32, 4, cudaMemcpyHostToDevice, st));
			if (int rc = commAllReduce(c, dStatus.p, 1, CommOp::MaxU32, st)) {
				return rc;
			}
			RX_CUDA(cudaMemcpyAsync(&all, dStatus.p, 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			if (all) {
				return fail(int(all), uint32_t(status) == all ? why : "rxgpu: sharded IVF training failed on another rank");
			}
		}
		// ---- 5. one all-gather of every rank's training rows (prepared as rxgpu_ivf_train prepares them), then plan order on the device
		DevBuf<float> x, cent;
		DevBuf<uint64_t> keys, from;
		{
			std::vector<int32_t> rows;
			rows.reserve(owned[me]);
			std::vector<uint64_t> hfrom(nx);
			std::vector<uint64_t> seen(R, 0);
			for (uint64_t pos = 0; pos < nx; ++pos) {
				const uint32_t r = owner[pos];
				hfrom[pos] = uint64_t(r) * maxc + seen[r]++;
				if (r == me) {
					rows.push_back(int32_t(gatheredRow(plan, pos) - base));
				}
			}
			DevBuf<float> send, recv;
			PinBuf<float> stage;
			RX_CUDA(send.ensure(std::max<uint64_t>(maxc, 1) * dim));
			RX_CUDA(recv.ensure(std::max<uint64_t>(maxc, 1) * dim * R));
			RX_CUDA(from.ensure(nx));
			if (!rows.empty()) {
				if (int rc = uploadRows(ix, vecs_local, norm_coefs_local, rows.data(), 0, rows.size(), send.p, stage, st)) {
					return rc;
				}
			}
			if (int rc = commAllGather(c, send.p, recv.p, maxc * dim * 4, st)) {
				return rc;
			}
			RX_CUDA(cudaMemcpyAsync(from.p, hfrom.data(), nx * 8, cudaMemcpyHostToDevice, st));
			RX_CUDA(x.ensure(size_t(nx) * dim));
			kmeans_gather_rows_kernel<<<unsigned(nx), 128, 0, st>>>(recv.p, dim, from.p, x.p, dim);
			RX_CUDA(cudaGetLastError());
			// the initial centroids are training rows: plan.initPos
			for (uint32_t i = 0; i < nlist; ++i) {
				hfrom[i] = uint64_t(plan.initPos[i]);
			}
			RX_CUDA(cudaMemcpyAsync(from.p, hfrom.data(), size_t(nlist) * 8, cudaMemcpyHostToDevice, st));
			RX_CUDA(cent.ensure(size_t(nlist) * pitch));
			RX_CUDA(cudaMemsetAsync(cent.p, 0, size_t(nlist) * pitch * 4, st));
			kmeans_gather_rows_kernel<<<nlist, 128, 0, st>>>(x.p, dim, from.p, cent.p, pitch);
			RX_CUDA(cudaGetLastError());
			RX_CUDA(cudaStreamSynchronize(st));  // the host vectors and the exchange buffers go
		}
		from.release();
		// ---- 6. the iterations: rank r assigns the points [r * slice, (r + 1) * slice), one all-gather completes the keys
		if (!plan.copy && prm.niter > 0) {
			RX_CUDA(keys.ensure(size_t(R) * slice));
		}
		const uint64_t lo = std::min<uint64_t>(nx, uint64_t(me) * slice), cnt = std::min<uint64_t>(nx, lo + slice) - lo;
		const KmeansAssign assign = [&](const float* cp, const float* cn, uint64_t* k) -> int {
			if (cnt) {
				RX_CUDA(ivfAssignRows(ix, cp, cn, nlist, x.p + lo * dim, uint32_t(cnt), k + lo, st));
			}
			return 0;
		};
		const KmeansExchange exchange = [&](uint64_t* k) -> int { return R > 1 ? commAllGather(c, k + uint64_t(me) * slice, k, slice * 8, st) : 0; };
		return kmeansRun(ix, nlist, plan, prm.niter, ks, cent, x, keys, assign, exchange, out_centroids, stats);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_ivf_assign(const rxgpu_index* ix, uint64_t n, const float* vecs, const float* norm_coefs, uint32_t* out_list_nos, float* out_dist) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	IvfCentroids ic{};
	if (int rc = ivfCentroids(ix, ic)) {
		return rc;
	}
	if (n == 0) {
		return 0;
	}
	if (!vecs || !out_list_nos) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (int rc = ivfCheckCoarseDim(ix->dim)) {
		return rc;
	}
	cudaStream_t st = ix->stream;
	const bool negZero = ix->metric != RXGPU_L2;
	try {
		const uint64_t chunk = std::min<uint64_t>(n, std::max<uint64_t>(16, (uint64_t(256) << 20) / (uint64_t(ix->dim) * 4)));
		DevBuf<float> x;
		DevBuf<uint64_t> keys;
		PinBuf<float> stage;
		RX_CUDA(x.ensure(chunk * ix->dim));
		RX_CUDA(keys.ensure(chunk));
		std::vector<uint64_t> hk(chunk);
		for (uint64_t off = 0; off < n; off += chunk) {
			const uint64_t m = std::min(chunk, n - off);
			if (int rc = uploadRows(ix, vecs, norm_coefs, nullptr, off, m, x.p, stage, st)) {
				return rc;
			}
			RX_CUDA(ivfAssignRows(ix, ic.centroids, ic.cnorm, ic.nlist, x.p, uint32_t(m), keys.p, st));
			RX_CUDA(cudaMemcpyAsync(hk.data(), keys.p, m * 8, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			for (uint64_t i = 0; i < m; ++i) {
				out_list_nos[off + i] = uint32_t(hk[i]);
				if (out_dist) {
					out_dist[off + i] = key_dist(uint32_t(hk[i] >> 32), negZero);
				}
			}
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_ivf_add_assign(rxgpu_index* ix, uint64_t n, const uint64_t* labels, const float* vecs, const float* norm_coefs, uint32_t* out_list_nos) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	IvfCentroids ic{};
	if (int rc = ivfCentroids(ix, ic)) {
		return rc;
	}
	if (!ic.own) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: rxgpu_ivf_add needs lists made by rxgpu_ivf_create");
	}
	if (n == 0) {
		return 0;
	}
	if (!labels || !vecs) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		std::vector<uint32_t> lists(n);
		if (int rc = rxgpu_ivf_assign(ix, n, vecs, norm_coefs, lists.data(), nullptr)) {
			return rc;
		}
		if (int rc = rxgpu_ivf_add(ix, n, lists.data(), labels, vecs)) {
			return rc;
		}
		if (out_list_nos) {
			std::copy(lists.begin(), lists.end(), out_list_nos);
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

}  // extern "C"
