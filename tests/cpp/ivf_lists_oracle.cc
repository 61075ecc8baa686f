// TEST INFRASTRUCTURE.  An IVF oracle over GIVEN centroids and list assignments: the reference's vendored FAISS (linked from
// oracle/_ref/liboracle_ref_ivf.so), driven like reindexer::IvfIndex drives it, but without k-means, which cannot train 20 000 to
// 131 072 centroids in test time.  The quantizer (IndexFlatL2 / IP / Cosine, IvfIndex::newSpace, ivf_index.cc:686-695) holds the
// centroids, the index is marked trained, the rows go to the given lists through IndexIVFFlat::add_core (Cosine: CalculateL2Module
// norms, as IvfIndex hands them over), and the direct map is a hashtable, as IvfIndex::trainIdx sets it.  Upserts, deletes and
// searches then go through FAISS exactly as in the oracle's own facade.  Built by tests/cpp/ivf_lists_oracle.mk where the reference
// tree exists; wrapped by tests/ivf_lists_oracle.py.
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "faiss/IndexFlat.h"
#include "faiss/IndexIVFFlat.h"
#include "faiss/impl/AuxIndexStructures.h"
#include "faiss/invlists/DirectMap.h"
#include "tools/normalize.h"

namespace {
thread_local std::string g_err;

struct ListsIvf {
	std::unique_ptr<faiss::IndexFlat> space;
	std::unique_ptr<faiss::IndexIVFFlat> map;
	size_t dim = 0;
	int metric = 0;
};

template <typename Fn>
int guarded(Fn&& fn) noexcept {
	try {
		fn();
		return 0;
	} catch (const std::exception& e) {
		g_err = e.what();
	} catch (...) {
		g_err = "unknown exception";
	}
	return 1;
}

std::vector<float> norms(const ListsIvf& h, size_t n, const float* vecs) {
	std::vector<float> out;
	if (h.metric == 2) {
		out.resize(n);
		for (size_t i = 0; i < n; ++i) {
			out[i] = reindexer::ann::CalculateL2Module(vecs + i * h.dim, int32_t(h.dim));
		}
	}
	return out;
}
}  // namespace

extern "C" {

const char* ivf_lists_last_error() { return g_err.c_str(); }

// metric: 0 = L2, 1 = InnerProduct, 2 = Cosine (reindexer::VectorMetric); row i goes to list list_nos[i] with id ids[i]
void* ivf_lists_create(int metric, size_t dim, size_t nlist, const float* centroids, size_t n, const int64_t* list_nos, const int64_t* ids,
					   const float* vecs) {
	ListsIvf* out = nullptr;
	guarded([&] {
		auto h = std::make_unique<ListsIvf>();
		h->dim = dim;
		h->metric = metric;
		if (metric == 0) {
			h->space = std::make_unique<faiss::IndexFlatL2>(dim);
		} else if (metric == 1) {
			h->space = std::make_unique<faiss::IndexFlatIP>(dim);
		} else if (metric == 2) {
			h->space = std::make_unique<faiss::IndexFlatCosine>(dim);
		} else {
			throw std::runtime_error("ivf_lists_create: unknown metric");
		}
		h->space->add(faiss::idx_t(nlist), centroids);  // IndexFlatCosine computes the centroids' norm coefficients here
		h->map = std::make_unique<faiss::IndexIVFFlat>(h->space.get(), dim, nlist, metric == 0 ? faiss::METRIC_L2 : faiss::METRIC_INNER_PRODUCT,
														metric == 2);
		h->map->is_trained = true;
		h->map->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
		const std::vector<float> nv = norms(*h, n, vecs);
		h->map->add_core(faiss::idx_t(n), vecs, nv.empty() ? nullptr : nv.data(), reinterpret_cast<const faiss::idx_t*>(ids),
						 reinterpret_cast<const faiss::idx_t*>(list_nos));
		out = h.release();
	});
	return out;
}
void ivf_lists_destroy(void* h) { delete static_cast<ListsIvf*>(h); }

// IvfIndex::upsert on a trained index: map_->add_with_ids(1, vect, &id) (ivf_index.cc:87-91), the quantizer choosing the list
int ivf_lists_add(void* hv, size_t n, const float* vecs, const int64_t* ids) {
	auto* h = static_cast<ListsIvf*>(hv);
	return guarded([&] {
		const std::vector<float> nv = norms(*h, n, vecs);
		for (size_t i = 0; i < n; ++i) {
			const faiss::idx_t id = ids[i];
			if (h->metric == 2) {
				h->map->add_with_ids(1, vecs + i * h->dim, &nv[i], &id);
			} else {
				h->map->add_with_ids(1, vecs + i * h->dim, &id);
			}
		}
	});
}
// IvfIndex::del: map_->remove_ids(IDSelectorArray{1, &id}) (ivf_index.cc:120-124)
int ivf_lists_remove(void* hv, int64_t id) {
	auto* h = static_cast<ListsIvf*>(hv);
	return guarded([&] {
		const faiss::idx_t fid = id;
		h->map->remove_ids(faiss::IDSelectorArray{1, &fid});
	});
}
// the list every id lives in, from the direct map
int ivf_lists_list_of(const void* hv, size_t n, const int64_t* ids, uint32_t* list_nos) {
	auto* h = static_cast<const ListsIvf*>(hv);
	return guarded([&] {
		for (size_t i = 0; i < n; ++i) {
			const auto it = h->map->direct_map.hashtable.find(ids[i]);
			if (it == h->map->direct_map.hashtable.end()) {
				throw std::runtime_error("ivf_lists_list_of: unknown id");
			}
			list_nos[i] = uint32_t(faiss::lo_listno(it->second));
		}
	});
}
// nq queries, k results each, best first in FAISS' convention (L2: squared distance ascending, IP / Cosine: similarity descending),
// id -1 past the end
int ivf_lists_search(const void* hv, size_t nq, const float* queries, size_t k, size_t nprobe, float* dists, int64_t* ids) {
	auto* h = static_cast<const ListsIvf*>(hv);
	return guarded([&] {
		faiss::IVFSearchParameters p;
		p.nprobe = nprobe;
		h->map->search(faiss::idx_t(nq), queries, faiss::idx_t(k), dists, reinterpret_cast<faiss::idx_t*>(ids), &p);
	});
}
// map_->range_search(1, key, radius, &result, &params) (ivf_index.cc:211-212); returns the number of results, writes at most maxOut
// (unsorted); radius in FAISS' convention (L2: dis < radius, IP / Cosine: dis > radius)
int64_t ivf_lists_range_search(const void* hv, const float* query, float radius, size_t nprobe, size_t maxOut, float* dists, int64_t* ids) {
	auto* h = static_cast<const ListsIvf*>(hv);
	int64_t n = -1;
	guarded([&] {
		faiss::IVFSearchParameters p;
		p.nprobe = nprobe;
		faiss::RangeSearchResult res(1);
		h->map->range_search(1, query, radius, &res, &p);
		n = int64_t(res.lims[1] - res.lims[0]);
		for (int64_t i = 0; i < n && size_t(i) < maxOut; ++i) {
			dists[i] = res.distances[res.lims[0] + i];
			ids[i] = res.labels[res.lims[0] + i];
		}
	});
	return n;
}

}  // extern "C"
