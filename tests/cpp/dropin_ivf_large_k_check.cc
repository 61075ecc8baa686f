// TEST INFRASTRUCTURE.  The IVF adapter (reindexer_b200/host/gpu_ivf.h) at the large k IvfIndex asks for when other conditions filter
// the KNN result (k = 300, 1000, 10000 at nprobe 16 and 32), compiled against the reference's vendored FAISS headers and driven beside a
// plain faiss::IndexIVFFlat with the same trained centroids, through bursts of upserts and deletes like IvfIndex::upsert / del
// (cpp_src/core/index/float_vector/ivf_index.cc:87-132).  Built by tests/cpp/ivf_large_k.mk only where the reference tree exists.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <map>
#include <random>
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

struct Cpu {
	std::unique_ptr<faiss::IndexFlat> space;
	std::unique_ptr<faiss::IndexIVFFlat> map;
};

Cpu make(size_t dim, size_t nlist, int metric) {
	Cpu c;
	c.space = newSpace(dim, metric);
	c.map = std::make_unique<faiss::IndexIVFFlat>(c.space.get(), dim, nlist, metric == 0 ? faiss::METRIC_L2 : faiss::METRIC_INNER_PRODUCT, metric == 2);
	c.map->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
	return c;
}

// FAISS-shaped results (ids -1 past the count) agree: the same number of results, distances within fp noise
// position by position, and ids equal except for rows whose distance is within fp noise of the k-th (the cut may trade such rows)
bool sameKnn(const std::vector<float>& da, const std::vector<faiss::idx_t>& ia, const std::vector<float>& db, const std::vector<faiss::idx_t>& ib) {
	size_t na = 0, nb = 0;
	while (na < ia.size() && ia[na] >= 0) {
		++na;
	}
	while (nb < ib.size() && ib[nb] >= 0) {
		++nb;
	}
	if (na != nb) {
		return false;
	}
	for (size_t j = na; j < ia.size(); ++j) {
		if (ia[j] != -1 || ib[j] != -1) {
			return false;
		}
	}
	auto noise = [](float d) { return 1e-4f * std::max(std::abs(d), 1e-2f) + 2e-6f; };
	for (size_t j = 0; j < na; ++j) {
		if (std::abs(da[j] - db[j]) > noise(da[j])) {
			return false;
		}
	}
	if (na == 0) {
		return true;
	}
	std::map<faiss::idx_t, float> a, b;
	for (size_t j = 0; j < na; ++j) {
		a.emplace(ia[j], da[j]);
		b.emplace(ib[j], db[j]);
	}
	const float last = da[na - 1];
	for (const auto& [id, d] : a) {
		if (!b.count(id) && std::abs(d - last) > noise(last)) {
			return false;
		}
	}
	for (const auto& [id, d] : b) {
		if (!a.count(id) && std::abs(d - last) > noise(last)) {
			return false;
		}
	}
	return a.size() == na && b.size() == nb;  // no id twice
}

int runMetric(int metric) {
	const size_t dim = 32, nlist = 64, n0 = 40000, extra = 4000, nq = 6;
	std::mt19937 rng(4321 + metric);
	std::normal_distribution<float> gauss(0.f, 1.f);
	std::vector<float> centers(128 * dim);
	for (auto& v : centers) {
		v = gauss(rng);
	}
	auto makeVec = [&](float* out) {
		const size_t c = rng() % 128;
		for (size_t i = 0; i < dim; ++i) {
			out[i] = centers[c * dim + i] + 0.4f * gauss(rng);
		}
	};
	std::vector<float> vecs((n0 + extra) * dim);
	for (size_t i = 0; i < n0 + extra; ++i) {
		makeVec(vecs.data() + i * dim);
	}
	std::vector<faiss::idx_t> ids(n0 + extra);
	for (size_t i = 0; i < ids.size(); ++i) {
		ids[i] = faiss::idx_t(i) << 32;  // FloatVectorId numbers: row id in the upper half
	}
	Cpu ref = make(dim, nlist, metric);
	ref.map->train(faiss::idx_t(n0), vecs.data());
	Cpu mine = make(dim, nlist, metric);  // the adapter's CPU half gets the SAME trained centroids
	std::vector<float> cent(nlist * dim);
	ref.map->quantizer->reconstruct_n(0, faiss::idx_t(nlist), cent.data());
	mine.map->quantizer->add(faiss::idx_t(nlist), cent.data());
	mine.map->is_trained = true;
	ref.map->add_with_ids(faiss::idx_t(n0), vecs.data(), ids.data());
	mine.map->add_with_ids(faiss::idx_t(n0), vecs.data(), ids.data());
	reindexer::GpuIvfMap gpu(std::move(mine.map));

	std::vector<float> queries(nq * dim), qn(dim);
	for (size_t q = 0; q < nq; ++q) {
		makeVec(queries.data() + q * dim);
		if (metric == 2) {  // FloatVectorIndex normalises the key for Cosine (ivf_index.cc:307-316 via NormalizeCopyVector)
			reindexer::ann::NormalizeCopyVector(queries.data() + q * dim, int32_t(dim), qn.data());
			std::copy(qn.begin(), qn.end(), queries.begin() + q * dim);
		}
	}
	size_t searches = 0, same = 0;
	auto compare = [&]() {
		for (const size_t nprobe : {size_t(16), size_t(32)}) {
			faiss::IVFSearchParameters params;
			params.nprobe = nprobe;
			for (const size_t k : {size_t(300), size_t(1000), size_t(10000)}) {
				for (size_t q = 0; q < nq; ++q) {
					std::vector<float> da(k), db(k);
					std::vector<faiss::idx_t> ia(k), ib(k);
					ref.map->search(1, queries.data() + q * dim, faiss::idx_t(k), da.data(), ia.data(), &params);
					gpu.search(1, queries.data() + q * dim, faiss::idx_t(k), db.data(), ib.data(), &params);
					same += sameKnn(da, ia, db, ib);
					++searches;
				}
			}
		}
	};
	compare();
	size_t done = n0;
	std::vector<faiss::idx_t> alive(ids.begin(), ids.begin() + n0);
	for (const size_t burst : {size_t(1), size_t(999), size_t(3000)}) {
		for (size_t i = done; i < done + burst; ++i) {  // IvfIndex::upsert: one add_with_ids per row
			ref.map->add_with_ids(1, vecs.data() + i * dim, &ids[i]);
			gpu.add_with_ids(1, vecs.data() + i * dim, &ids[i]);
			alive.push_back(ids[i]);
		}
		done += burst;
		for (size_t r = 0; r < alive.size() / 10; ++r) {  // IvfIndex::del
			const size_t at = rng() % alive.size();
			const faiss::idx_t id = alive[at];
			alive[at] = alive.back();
			alive.pop_back();
			ref.map->remove_ids(faiss::IDSelectorArray{1, &id});
			gpu.remove_ids(faiss::IDSelectorArray{1, &id});
		}
		compare();
	}
	const bool ok = same == searches && gpu.DeviceImports() == 1 && size_t(gpu->ntotal) == alive.size();
	std::printf("metric %d: %zu knn searches at k = 300 / 1000 / 10000, nprobe 16 / 32: identical %zu, device imports %zu, rows %zu -> %s %s\n",
				metric, searches, same, gpu.DeviceImports(), alive.size(), ok ? "MATCH" : "MISMATCH", gpu.LastDeviceError().c_str());
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
