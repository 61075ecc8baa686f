// TEST INFRASTRUCTURE.  The IVF adapter (reindexer_b200/host/gpu_ivf.h) over an IvfIndex-shaped faiss::IndexIVFFlat with 20 000
// centroids (above the 16 384 the device path once stopped at), compiled against the reference's vendored FAISS headers and driven
// beside a plain faiss::IndexIVFFlat with the same centroids (a pre-filled quantizer, no k-means), through bursts of upserts and
// deletes like IvfIndex::upsert / del (cpp_src/core/index/float_vector/ivf_index.cc:87-132).  After each burst, search (k = 10 and
// k = 1000) and range_search must agree with FAISS (ids may differ only within fp noise of the distances).  Built by
// tests/cpp/ivf_many_centroids.mk only where the reference tree exists.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <map>
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

struct Cpu {
	std::unique_ptr<faiss::IndexFlat> space;
	std::unique_ptr<faiss::IndexIVFFlat> map;
};

Cpu make(size_t dim, const std::vector<float>& cent, int metric) {
	const size_t nlist = cent.size() / dim;
	Cpu c;
	c.space = newSpace(dim, metric);
	c.space->add(faiss::idx_t(nlist), cent.data());
	c.map = std::make_unique<faiss::IndexIVFFlat>(c.space.get(), dim, nlist, metric == 0 ? faiss::METRIC_L2 : faiss::METRIC_INNER_PRODUCT, metric == 2);
	c.map->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
	return c;
}

float noise(float d) { return 1e-4f * std::max(std::abs(d), 1e-2f) + 2e-6f; }

// one query's KNN lists agree: the same count, distances within fp noise place by place, and the same ids wherever the distance is
// clear of the last one (a group of equal distances at the k-th place may trade members)
bool sameKnn(size_t k, const float* da, const faiss::idx_t* ia, const float* db, const faiss::idx_t* ib) {
	size_t na = 0, nb = 0;
	while (na < k && ia[na] >= 0) {
		++na;
	}
	while (nb < k && ib[nb] >= 0) {
		++nb;
	}
	if (na != nb) {
		return false;
	}
	std::set<faiss::idx_t> sa, sb;
	for (size_t j = 0; j < na; ++j) {
		if (std::abs(da[j] - db[j]) > noise(da[j])) {
			return false;
		}
		if (std::abs(da[j] - da[na - 1]) > noise(da[na - 1])) {
			sa.insert(ia[j]);
			sb.insert(ib[j]);
		}
	}
	return sa == sb;
}

// the matches of query q agree: distances of common ids within fp noise, ids on one side only within fp noise of the radius
bool sameRange(const faiss::RangeSearchResult& a, const faiss::RangeSearchResult& b, size_t q, float radius) {
	std::map<faiss::idx_t, float> ma, mb;
	for (size_t i = a.lims[q]; i < a.lims[q + 1]; ++i) {
		ma.emplace(a.labels[i], a.distances[i]);
	}
	for (size_t i = b.lims[q]; i < b.lims[q + 1]; ++i) {
		mb.emplace(b.labels[i], b.distances[i]);
	}
	if (ma.size() != a.lims[q + 1] - a.lims[q] || mb.size() != b.lims[q + 1] - b.lims[q]) {
		return false;  // an id twice
	}
	for (const auto& [id, d] : ma) {
		const auto it = mb.find(id);
		if (it == mb.end() ? std::abs(d - radius) > noise(radius) : std::abs(d - it->second) > noise(d)) {
			return false;
		}
	}
	for (const auto& [id, d] : mb) {
		if (!ma.count(id) && std::abs(d - radius) > noise(radius)) {
			return false;
		}
	}
	return true;
}

int runMetric(int metric) {
	const size_t dim = 8, nlist = 20000, n0 = 30000, extra = 3000, nq = 8;
	std::mt19937 rng(9100 + metric);
	std::normal_distribution<float> gauss(0.f, 1.f);
	auto fill = [&](float* out, size_t n) {
		for (size_t i = 0; i < n; ++i) {
			out[i] = gauss(rng);
		}
	};
	std::vector<float> cent(nlist * dim), vecs((n0 + extra) * dim), queries(nq * dim);
	fill(cent.data(), cent.size());
	fill(vecs.data(), vecs.size());
	fill(queries.data(), queries.size());
	std::vector<float> qn(dim);
	for (size_t q = 0; q < nq && metric == 2; ++q) {  // FloatVectorIndex normalises the key for Cosine (ivf_index.cc:307-316)
		reindexer::ann::NormalizeCopyVector(queries.data() + q * dim, int32_t(dim), qn.data());
		std::copy(qn.begin(), qn.end(), queries.begin() + q * dim);
	}
	std::vector<faiss::idx_t> ids(n0 + extra);
	for (size_t i = 0; i < ids.size(); ++i) {
		ids[i] = faiss::idx_t(i) << 32;  // FloatVectorId numbers: row id in the upper half
	}
	Cpu ref = make(dim, cent, metric);
	Cpu mine = make(dim, cent, metric);
	ref.map->add_with_ids(faiss::idx_t(n0), vecs.data(), ids.data());
	mine.map->add_with_ids(faiss::idx_t(n0), vecs.data(), ids.data());
	reindexer::GpuIvfMap gpu(std::move(mine.map));

	size_t checks = 0, agree = 0;
	auto compare = [&]() {
		for (const size_t nprobe : {size_t(8), size_t(64)}) {
			faiss::IVFSearchParameters params;
			params.nprobe = nprobe;
			for (const size_t k : {size_t(10), size_t(1000)}) {
				std::vector<float> dw(nq * k), dg(nq * k);
				std::vector<faiss::idx_t> iw(nq * k), ig(nq * k);
				ref.map->search(faiss::idx_t(nq), queries.data(), faiss::idx_t(k), dw.data(), iw.data(), &params);
				gpu.search(faiss::idx_t(nq), queries.data(), faiss::idx_t(k), dg.data(), ig.data(), &params);
				bool ok = true;
				for (size_t q = 0; q < nq; ++q) {
					ok = ok && sameKnn(k, dw.data() + q * k, iw.data() + q * k, dg.data() + q * k, ig.data() + q * k);
				}
				agree += ok;
				++checks;
				// range at query 0's last distance (FAISS' convention): its k-th, or its last probed row
				size_t last = k - 1;
				while (last > 0 && iw[last] < 0) {
					--last;
				}
				const float radius = dw[last];
				faiss::RangeSearchResult want(nq), got(nq);
				ref.map->range_search(faiss::idx_t(nq), queries.data(), radius, &want, &params);
				gpu.range_search(faiss::idx_t(nq), queries.data(), radius, &got, &params);
				ok = true;
				for (size_t q = 0; q < nq; ++q) {
					ok = ok && sameRange(want, got, q, radius);
				}
				agree += ok;
				++checks;
			}
		}
	};
	compare();
	size_t done = n0;
	std::vector<faiss::idx_t> alive(ids.begin(), ids.begin() + n0);
	for (const size_t burst : {size_t(1), size_t(999), size_t(2000)}) {
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
	const bool ok = agree == checks && gpu.DeviceImports() == 1 && size_t(gpu->ntotal) == alive.size() && gpu->nlist == nlist;
	std::printf("metric %d: %zu centroids, %zu search / range checks (k 10 / 1000, nprobe 8 / 64) through 4 bursts: agree with faiss %zu, "
				"device imports %zu, rows %zu -> %s %s\n",
				metric, nlist, checks, agree, gpu.DeviceImports(), alive.size(), ok ? "MATCH" : "MISMATCH", gpu.LastDeviceError().c_str());
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
