// TEST INFRASTRUCTURE.  IvfIndex's two index builds (cpp_src/core/index/float_vector/ivf_index.cc) run through the IVF adapter's
// GpuIvfMap::TrainAndFill (reindexer_b200/host/gpu_ivf.h), beside the reference flow on the CPU, compiled against the reference's vendored
// FAISS headers:
//   * the training upsert (:96-107): once the flat space holds more than 39 x centroids rows, a new IndexIVFFlat is trained on all of
//     them (trainIdx: hashtable direct map, idx.train(n, x, norms)) and filled with add_with_ids(n, x, norms, ids);
//   * RebuildCentroids (:637-684): train on max(rows x dataPart, 39 x centroids) rows gathered from the direct map, then add every row.
// Checked per metric: every id sits in the same list in the adapter's FAISS direct map and on the device (an independent device
// assignment over the adapter's centroids), upserts and searches after the build need no import (DeviceImports() == 0), and recall@10 at
// nprobe 16 against the exact neighbours is within 0.02 of the CPU-trained reference index.  Built by tests/cpp/ivf_train.mk only where
// the reference tree exists.
#include <algorithm>
#include <cstdio>
#include <numeric>
#include <random>
#include <set>
#include <vector>

#include "gpu_ivf.h"
#include "faiss/IndexFlat.h"
#include "tools/normalize.h"

namespace {

std::unique_ptr<faiss::IndexFlat> newSpace(size_t dim, int metric) {  // IvfIndex::newSpace, ivf_index.cc:686-695
	if (metric == 0) {
		return std::make_unique<faiss::IndexFlatL2>(dim);
	}
	if (metric == 1) {
		return std::make_unique<faiss::IndexFlatIP>(dim);
	}
	return std::make_unique<faiss::IndexFlatCosine>(dim);
}
std::unique_ptr<faiss::IndexIVFFlat> newIvf(faiss::IndexFlat* space, size_t dim, size_t nlist, int metric) {
	return std::make_unique<faiss::IndexIVFFlat>(space, dim, nlist, metric == 0 ? faiss::METRIC_L2 : faiss::METRIC_INNER_PRODUCT, metric == 2);
}

// exact top-10 ids of every query over all rows (fp64), in the metric's order
std::vector<std::set<faiss::idx_t>> exactTop(int metric, size_t dim, const std::vector<float>& x, const std::vector<faiss::idx_t>& ids,
											 const std::vector<float>& q, size_t nq) {
	const size_t n = ids.size();
	std::vector<std::set<faiss::idx_t>> out(nq);
	std::vector<std::pair<double, faiss::idx_t>> d(n);
	for (size_t j = 0; j < nq; ++j) {
		for (size_t i = 0; i < n; ++i) {
			double s = 0, nn = 0;
			for (size_t c = 0; c < dim; ++c) {
				const double a = x[i * dim + c], b = q[j * dim + c];
				s += metric == 0 ? (a - b) * (a - b) : -a * b;
				nn += a * a;
			}
			d[i] = {metric == 2 && nn > 0 ? s / std::sqrt(nn) : s, ids[i]};
		}
		std::partial_sort(d.begin(), d.begin() + 10, d.end());
		for (size_t r = 0; r < 10; ++r) {
			out[j].insert(d[r].second);
		}
	}
	return out;
}

template <typename Map>
double recall(const Map& m, const std::vector<float>& q, size_t nq, const std::vector<std::set<faiss::idx_t>>& truth) {
	faiss::IVFSearchParameters p;
	p.nprobe = 16;
	std::vector<float> d(nq * 10);
	std::vector<faiss::idx_t> l(nq * 10);
	m.search(faiss::idx_t(nq), q.data(), 10, d.data(), l.data(), &p);
	size_t hit = 0;
	for (size_t j = 0; j < nq; ++j) {
		for (size_t r = 0; r < 10; ++r) {
			hit += truth[j].count(l[j * 10 + r]);
		}
	}
	return double(hit) / double(nq * 10);
}

// every id's list in the adapter's direct map equals an independent device assignment over the adapter's own centroids
bool sameLists(const reindexer::GpuIvfMap& gpu, int metric, size_t dim, const std::vector<float>& x, const std::vector<faiss::idx_t>& ids) {
	const faiss::IndexIVFFlat& idx = *gpu;
	std::vector<float> cent(idx.nlist * dim);
	idx.quantizer->reconstruct_n(0, faiss::idx_t(idx.nlist), cent.data());
	rxgpu_index* ix = nullptr;
	if (rxgpu_index_create(&ix, rxgpu_metric(metric), uint32_t(dim), 16, 0, 0) != RXGPU_OK || rxgpu_ivf_create(ix, uint32_t(idx.nlist), cent.data()) != RXGPU_OK) {
		return false;
	}
	std::vector<uint32_t> lists(ids.size());
	const bool ok = rxgpu_ivf_assign(ix, ids.size(), x.data(), nullptr, lists.data(), nullptr) == RXGPU_OK;
	rxgpu_index_destroy(ix);
	for (size_t i = 0; ok && i < ids.size(); ++i) {
		const auto it = idx.direct_map.hashtable.find(ids[i]);
		if (it == idx.direct_map.hashtable.end() || faiss::lo_listno(it->second) != faiss::idx_t(lists[i])) {
			return false;
		}
	}
	return ok && size_t(idx.ntotal) == ids.size();
}

int runMetric(int metric) {
	const size_t dim = 16, nlist = 64, ntrain = 39 * nlist, nextra = 800, nq = 200;
	std::mt19937 rng(4400 + metric);
	std::normal_distribution<float> gauss(0.f, 1.f);
	// rows around 256 random centres, so that IVF recall at nprobe 16 means something
	std::vector<float> centres(256 * dim);
	for (float& v : centres) {
		v = 3.f * gauss(rng);
	}
	auto rows = [&](size_t n) {
		std::vector<float> out(n * dim);
		for (size_t i = 0; i < n; ++i) {
			const size_t c = rng() % 256;
			for (size_t j = 0; j < dim; ++j) {
				out[i * dim + j] = centres[c * dim + j] + gauss(rng);
			}
		}
		return out;
	};
	std::vector<float> x = rows(ntrain + 1), extra = rows(nextra), q = rows(nq);
	if (metric == 2) {  // FloatVectorIndex normalises the key for Cosine
		std::vector<float> qn(dim);
		for (size_t j = 0; j < nq; ++j) {
			reindexer::ann::NormalizeCopyVector(q.data() + j * dim, int32_t(dim), qn.data());
			std::copy(qn.begin(), qn.end(), q.begin() + j * dim);
		}
	}
	std::vector<faiss::idx_t> ids(ntrain + 1 + nextra);
	for (size_t i = 0; i < ids.size(); ++i) {
		ids[i] = faiss::idx_t(i) << 32;
	}
	std::vector<float> norms;  // the flat space's norm coefficients, as IvfIndex hands them over (Cosine)
	for (size_t i = 0; metric == 2 && i < ids.size(); ++i) {
		const float* v = i <= ntrain ? x.data() + i * dim : extra.data() + (i - ntrain - 1) * dim;
		norms.push_back(reindexer::ann::CalculateL2Module(v, int32_t(dim)));
	}
	const size_t n0 = ntrain + 1;
	const float* nm = metric == 2 ? norms.data() : nullptr;

	// the training upsert: the reference on the CPU, the adapter on the device
	auto refSpace = newSpace(dim, metric);
	auto ref = newIvf(refSpace.get(), dim, nlist, metric);
	ref->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
	ref->train(faiss::idx_t(n0), x.data(), nm);
	ref->add_with_ids(faiss::idx_t(n0), x.data(), nm, ids.data());
	auto devSpace = newSpace(dim, metric);
	reindexer::GpuIvfMap gpu;
	gpu.TrainAndFill(newIvf(devSpace.get(), dim, nlist, metric), x.data(), nm, n0, ids.data());
	std::vector<faiss::idx_t> firstIds(ids.begin(), ids.begin() + n0);
	bool ok = sameLists(gpu, metric, dim, x, firstIds);
	// upserts on the trained index, one add_with_ids per row (IvfIndex::upsert)
	for (size_t i = 0; i < nextra; ++i) {
		const float* en = nm ? nm + n0 + i : nullptr;
		ref->add_with_ids(1, extra.data() + i * dim, en, &ids[n0 + i]);
		gpu.add_with_ids(1, extra.data() + i * dim, en, &ids[n0 + i]);
	}
	std::vector<float> all(x);
	all.insert(all.end(), extra.begin(), extra.end());
	const auto truth = exactTop(metric, dim, all, ids, q, nq);
	const double rRef1 = recall(*ref, q, nq, truth), rGpu1 = recall(gpu, q, nq, truth);
	ok = ok && gpu.DeviceImports() == 0 && rGpu1 >= rRef1 - 0.02;

	// RebuildCentroids(dataPart = 0.5): train on max(rows / 2, 39 x nlist) rows taken in direct-map order, then add every row
	std::vector<float> data;
	std::vector<float> dnorms;
	std::vector<faiss::idx_t> order;
	for (const auto& [id, lo] : gpu->direct_map.hashtable) {
		const auto* v = reinterpret_cast<const float*>(gpu->invlists->get_single_code(faiss::lo_listno(lo), faiss::lo_offset(lo)));
		data.insert(data.end(), v, v + dim);
		if (metric == 2) {
			dnorms.push_back(*gpu->invlists->get_single_norm(faiss::lo_listno(lo), faiss::lo_offset(lo)));
		}
		order.push_back(id);
	}
	const size_t vecs = std::min(order.size(), std::max(order.size() / 2, ntrain));
	auto rebuildRefSpace = newSpace(dim, metric);
	auto rebuiltRef = newIvf(rebuildRefSpace.get(), dim, nlist, metric);
	rebuiltRef->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
	rebuiltRef->train(faiss::idx_t(vecs), data.data(), metric == 2 ? dnorms.data() : nullptr);
	for (size_t i = 0; i < order.size(); ++i) {
		rebuiltRef->add_with_ids(1, data.data() + i * dim, metric == 2 ? dnorms.data() + i : nullptr, &order[i]);
	}
	auto rebuildSpace = newSpace(dim, metric);
	gpu.TrainAndFill(newIvf(rebuildSpace.get(), dim, nlist, metric), data.data(), metric == 2 ? dnorms.data() : nullptr, order.size(),
					 order.data(), vecs);
	ok = ok && sameLists(gpu, metric, dim, data, order);
	const double rRef2 = recall(*rebuiltRef, q, nq, truth), rGpu2 = recall(gpu, q, nq, truth);
	ok = ok && gpu.DeviceImports() == 0 && rGpu2 >= rRef2 - 0.02;
	std::printf("metric %d: %zu centroids; training upsert on %zu rows + %zu upserts: recall@10 (nprobe 16) device %.4f, CPU %.4f; "
				"RebuildCentroids on %zu of %zu rows: device %.4f, CPU %.4f; device imports %zu -> %s %s\n",
				metric, nlist, n0, nextra, rGpu1, rRef1, vecs, order.size(), rGpu2, rRef2, gpu.DeviceImports(), ok ? "MATCH" : "MISMATCH",
				gpu.LastDeviceError().c_str());
	return ok ? 0 : 1;
}

}  // namespace

int main() {
	int bad = 0;
	for (const int metric : {0, 1, 2}) {
		bad += runMetric(metric);
	}
	return bad;
}
