// TEST INFRASTRUCTURE.  The IVF adapter (reindexer_b200/host/gpu_ivf.h) answering range_search for a batch of queries (n > 1: one
// rxgpu_ivf_search_range_batch call, and a second one for the queries with more than 256 matches), compiled against the reference's
// vendored FAISS headers and driven beside a plain faiss::IndexIVFFlat with the same trained centroids, through bursts of upserts and
// deletes like IvfIndex::upsert / del (cpp_src/core/index/float_vector/ivf_index.cc:87-132).  Each batch must agree with FAISS' own
// range_search and be identical to n one-query adapter calls.  Built by tests/cpp/ivf_range.mk only where the reference tree exists.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
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

float noise(float d) { return 1e-4f * std::max(std::abs(d), 1e-2f) + 2e-6f; }

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

// query q of the batch holds exactly the single call's result, in the same order, with the same distance bits
bool identical(const faiss::RangeSearchResult& batch, size_t q, const faiss::RangeSearchResult& one) {
	const size_t n = batch.lims[q + 1] - batch.lims[q];
	return n == one.lims[1] && std::equal(one.labels, one.labels + n, batch.labels + batch.lims[q]) &&
		   std::memcmp(one.distances, batch.distances + batch.lims[q], n * sizeof(float)) == 0;
}

int runMetric(int metric) {
	const size_t dim = 32, nlist = 64, n0 = 40000, extra = 4000, nq = 40;
	std::mt19937 rng(8765 + metric);
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
	size_t batches = 0, agree = 0, same = 0, compared = 0, above256 = 0;
	auto compare = [&]() {
		for (const size_t nprobe : {size_t(16), size_t(32)}) {
			faiss::IVFSearchParameters params;
			params.nprobe = nprobe;
			// radii at the 100th and the 1000th neighbour of query 0 (FAISS' convention): some queries above 256 matches, some below
			for (const size_t rank : {size_t(100), size_t(1000)}) {
				std::vector<float> kd(rank);
				std::vector<faiss::idx_t> ki(rank);
				ref.map->search(1, queries.data(), faiss::idx_t(rank), kd.data(), ki.data(), &params);
				const float radius = kd[rank - 1];
				faiss::RangeSearchResult want(nq), got(nq);
				ref.map->range_search(faiss::idx_t(nq), queries.data(), radius, &want, &params);
				gpu.range_search(faiss::idx_t(nq), queries.data(), radius, &got, &params);
				bool ok = true, ident = true;
				for (size_t q = 0; q < nq; ++q) {
					ok = ok && sameRange(want, got, q, radius);
					faiss::RangeSearchResult one(1);
					gpu.range_search(1, queries.data() + q * dim, radius, &one, &params);
					ident = ident && identical(got, q, one);
					above256 += got.lims[q + 1] - got.lims[q] > 256;
					++compared;
				}
				agree += ok;
				same += ident;
				++batches;
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
	const bool ok = agree == batches && same == batches && above256 > 0 && above256 < compared && gpu.DeviceImports() == 1 &&
					size_t(gpu->ntotal) == alive.size();
	std::printf("metric %d: %zu range batches of %zu queries, nprobe 16 / 32: agree with faiss %zu, identical to single calls %zu, "
				"queries above 256 matches %zu of %zu, device imports %zu, rows %zu -> %s %s\n",
				metric, batches, nq, agree, same, above256, compared, gpu.DeviceImports(), alive.size(), ok ? "MATCH" : "MISMATCH",
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
