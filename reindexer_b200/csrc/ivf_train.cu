// librxgpu: IVF training and list assignment on the device (rxgpu_ivf_train, rxgpu_ivf_assign, rxgpu_ivf_add_assign, rxgpu_kmeans_plan)
// -- faiss::Clustering::train as IndexIVFFlat::train reaches it, and quantizer->assign as IndexIVF::add_with_ids calls it.  The
// assignment is the coarse pass's distance kernel in argmin mode (ivf_coarse.cuh), launched by ivf.cu (ivfAssignRows); the update,
// split and renormalisation kernels are ivf_train.cuh's.  The host keeps what FAISS decides with its RNG: the sample, the initial centroids and which cluster an empty one
// splits.
#include <cuda_runtime.h>

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
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
	std::vector<int32_t> sample;  // empty: no subsampling, the sample is the input
	std::vector<int32_t> init;    // [nlist] input rows
	uint64_t nx = 0;
	bool copy = false;            // nx == nlist: the centroids are the first nlist input rows, no iterations
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
	if (p.nx == nlist) {
		p.copy = true;
		for (uint32_t c = 0; c < nlist; ++c) {
			p.init[c] = int32_t(c);
		}
		return p;
	}
	const std::vector<int32_t> perm = randPerm(p.nx, int64_t(seed) + 1);
	for (uint32_t c = 0; c < nlist; ++c) {
		p.init[c] = p.sample.empty() ? perm[c] : p.sample[perm[c]];
	}
	return p;
}

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
	const bool spherical = ix->metric != RXGPU_L2;  // IndexIVF sets cp.spherical for METRIC_INNER_PRODUCT (IndexIVF.cpp:179-182)
	const uint32_t dim = ix->dim, pitch = ix->pitch;
	cudaStream_t st = ix->stream;
	// the training set and one iteration's scratch: the points, their keys, (centroid, point) pairs twice for the sort; checked before
	// anything reads the input
	const uint64_t nx = std::min<uint64_t>(n, uint64_t(nlist) * uint64_t(prm.max_points_per_centroid));
	size_t sortBytes = 0;
	int endBit = 1;
	while ((1u << endBit) < nlist) {
		++endBit;
	}
	RX_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr),
											static_cast<uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), int(nx), 0, endBit, st));
	{
		const uint64_t need = nx * dim * 4 + nx * (8 + 16) + sortBytes + uint64_t(nlist) * (pitch * 4 + 8) + (uint64_t(64) << 20);
		size_t freeB = 0, totalB = 0;
		RX_CUDA(cudaMemGetInfo(&freeB, &totalB));
		if (need > freeB) {
			return fail(RXGPU_ERR_SYSTEM, "rxgpu: not enough device memory for the IVF training set (" + std::to_string(need >> 20) + " MB needed, " +
											   std::to_string(freeB >> 20) + " MB free)");
		}
	}
	if (int rc = checkFinite(ix, n, vecs, norm_coefs)) {
		return rc;
	}
	try {
		const KmeansPlan plan = kmeansPlan(n, nlist, prm.seed, prm.max_points_per_centroid);
		if (stats) {
			std::fill(stats, stats + prm.niter, rxgpu_ivf_train_stats{0.0, 0, 0.f, 0.f, 0.f});
		}
		DevBuf<float> x, cent, cnorm;
		DevBuf<uint64_t> keys;
		DevBuf<uint32_t> assign, point, assign2, point2, off;
		DevBuf<uint2> splits;
		DevBuf<unsigned char> cubTmp;
		PinBuf<float> stage;
		RX_CUDA(cent.ensure(size_t(nlist) * pitch));
		RX_CUDA(cudaMemsetAsync(cent.p, 0, size_t(nlist) * pitch * 4, st));
		// initial centroids: input rows (the sample's perm[c]-th, prepared as the sample is), then post_process_centroids
		{
			RX_CUDA(x.ensure(size_t(nlist) * dim));
			if (int rc = uploadRows(ix, vecs, norm_coefs, plan.init.data(), 0, nlist, x.p, stage, st)) {
				return rc;
			}
			RX_CUDA(cudaMemcpy2DAsync(cent.p, size_t(pitch) * 4, x.p, size_t(dim) * 4, size_t(dim) * 4, nlist, cudaMemcpyDeviceToDevice, st));
		}
		if (spherical && !plan.copy) {
			kmeans_renorm_kernel<<<(nlist + 7u) / 8u, 256, 0, st>>>(cent.p, pitch, dim, nlist);
			RX_CUDA(cudaGetLastError());
		}
		if (!plan.copy && prm.niter > 0) {
			x.release();
			RX_CUDA(x.ensure(size_t(nx) * dim));
			if (int rc = uploadRows(ix, vecs, norm_coefs, plan.sample.empty() ? nullptr : plan.sample.data(), 0, nx, x.p, stage, st)) {
				return rc;
			}
			RX_CUDA(keys.ensure(nx));
			RX_CUDA(assign.ensure(nx));
			RX_CUDA(point.ensure(nx));
			RX_CUDA(assign2.ensure(nx));
			RX_CUDA(point2.ensure(nx));
			RX_CUDA(off.ensure(size_t(nlist) + 1));
			RX_CUDA(cubTmp.ensure(std::max<size_t>(sortBytes, 1)));
			if (ix->metric == RXGPU_COS) {
				RX_CUDA(cnorm.ensure(nlist));
			}
			cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
			struct EventsGuard {
				cudaEvent_t* e;
				~EventsGuard() {
					for (int i = 0; i < 5; ++i) {
						if (e[i]) {
							cudaEventDestroy(e[i]);
						}
					}
				}
			} evGuard{ev};
			for (int i = 0; i < 5; ++i) {
				RX_CUDA(cudaEventCreate(&ev[i]));
			}
			std::vector<uint64_t> hkeys(nx);
			std::vector<uint32_t> counts(nlist), hoff(size_t(nlist) + 1);
			std::vector<float> hassign(nlist);
			for (int it = 0; it < prm.niter; ++it) {
				// the centroids as the index holds them for the search: Cosine norm coefficients (IndexFlatCosine::add)
				if (ix->metric == RXGPU_COS) {
					RX_CUDA(launchNormCoefs(cent.p, pitch, dim, 0, nlist, cnorm.p, st));
				}
				RX_CUDA(cudaEventRecord(ev[0], st));
				RX_CUDA(ivfAssignRows(ix, cent.p, cnorm.p, nlist, x.p, uint32_t(nx), keys.p, st));
				RX_CUDA(cudaEventRecord(ev[1], st));
				kmeans_split_keys_kernel<<<unsigned((nx + 255) / 256), 256, 0, st>>>(keys.p, uint32_t(nx), assign.p, point.p);
				RX_CUDA(cudaGetLastError());
				RX_CUDA(cub::DeviceRadixSort::SortPairs(cubTmp.p, sortBytes, assign.p, assign2.p, point.p, point2.p, int(nx), 0, endBit, st));
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
					RX_CUDA(cudaEventElapsedTime(&u0, ev[1], ev[2]));
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
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
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
