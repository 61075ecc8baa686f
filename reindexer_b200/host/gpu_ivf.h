// Drop-in replacement for the `std::unique_ptr<faiss::IndexIVFFlat> map_` member of reindexer::IvfIndex
// (cpp_src/core/index/float_vector/ivf_index.h:75, used at ivf_index.cc:87-132 upsert / del, :150-300 search / range_search through the
// `const auto& map` templates, :309-316, :420-429): the CPU faiss::IndexIVFFlat stays the row store (getView, reconstruct, index cache,
// clone, RebuildCentroids read its inverted lists and direct map through operator->), the four calls on the query/update path --
//   search(1, key, k, dists, ids, &IVFSearchParameters{nprobe})      range_search(1, key, radius, &result, &params)
//   add_with_ids(1, vec[, norm], &id)                                 remove_ids(IDSelectorArray{1, &id})
// -- are served by librxgpu (include/rxgpu.h: rxgpu_ivf_create / _add / _remove / _search_knn_large_k / _search_range, and
// _search_range_batch for range_search with n > 1).  The device lists are filled once, from the trained index, by the first search, or
// built on the device together with the CPU index by TrainAndFill (rxgpu_ivf_train / _add_assign); after that every upsert / delete
// patches them in place (the list number
// is read back from FAISS' direct map, so both sides agree on the assignment bit for bit).  Distances follow FAISS' conventions
// (L2: squared distance ascending; inner product / cosine: +similarity descending, labels -1 past the end).
// Meant to be dropped into cpp_src/core/index/float_vector/; compiled only where the reference tree is available
// (tests/cpp/dropin_ivf_check.cc does so in the authoring container).  INTEGRATION.md section 8 shows the patch.
#pragma once

#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <vector>

#include "faiss/IndexIVFFlat.h"
#include "faiss/impl/AuxIndexStructures.h"
#include "faiss/impl/IDSelector.h"
#include "faiss/invlists/DirectMap.h"
#include "rxgpu.h"
#include "tools/normalize.h"

namespace reindexer {

class [[nodiscard]] GpuIvfMap {
public:
	GpuIvfMap() = default;
	explicit GpuIvfMap(std::unique_ptr<faiss::IndexIVFFlat> idx) : cpu_(std::move(idx)) {}
	GpuIvfMap(const GpuIvfMap&) = delete;
	GpuIvfMap& operator=(const GpuIvfMap&) = delete;
	GpuIvfMap& operator=(std::unique_ptr<faiss::IndexIVFFlat>&& idx) noexcept {  // map_ = std::move(idx), ivf_index.cc:104,609,681
		releaseDevice();
		cpu_ = std::move(idx);
		return *this;
	}
	~GpuIvfMap() { releaseDevice(); }

	explicit operator bool() const noexcept { return bool(cpu_); }
	faiss::IndexIVFFlat* operator->() const noexcept { return cpu_.get(); }
	faiss::IndexIVFFlat& operator*() const noexcept { return *cpu_; }
	faiss::IndexIVFFlat* get() const noexcept { return cpu_.get(); }
	void reset() noexcept {
		releaseDevice();
		cpu_.reset();
	}

	void add_with_ids(faiss::idx_t n, const float* x, const faiss::idx_t* ids) { add_with_ids(n, x, nullptr, ids); }
	void add_with_ids(faiss::idx_t n, const float* x, const float* norms, const faiss::idx_t* ids) {
		if (norms) {
			cpu_->add_with_ids(n, x, norms, ids);
		} else {
			cpu_->add_with_ids(n, x, ids);
		}
		std::lock_guard<std::mutex> lck(mtx_);
		if (!gpu_) {
			return;  // filled from the CPU index by the first search
		}
		std::vector<uint32_t> lists(n);
		std::vector<uint64_t> labels(n);
		for (faiss::idx_t i = 0; i < n; ++i) {
			lists[i] = listOf(ids[i]);
			labels[i] = uint64_t(ids[i]);
		}
		if (rxgpu_ivf_add(gpu_, uint64_t(n), lists.data(), labels.data(), x) != RXGPU_OK) {
			lastError_ = rxgpu_last_error();
			releaseDevice();  // rebuilt from the CPU index by the next search
		}
	}
	size_t remove_ids(const faiss::IDSelector& sel) {
		const auto* arr = dynamic_cast<const faiss::IDSelectorArray*>(&sel);
		if (!arr) {
			throw std::logic_error("GpuIvfMap: remove_ids takes an IDSelectorArray (what IvfIndex::del passes)");
		}
		std::vector<faiss::idx_t> present;
		for (size_t i = 0; i < arr->n; ++i) {
			if (cpu_->direct_map.hashtable.find(arr->ids[i]) != cpu_->direct_map.hashtable.end()) {
				present.push_back(arr->ids[i]);
			}
		}
		const size_t removed = cpu_->remove_ids(sel);
		std::lock_guard<std::mutex> lck(mtx_);
		for (const faiss::idx_t id : present) {
			if (gpu_ && rxgpu_ivf_remove(gpu_, uint64_t(id)) != RXGPU_OK) {
				lastError_ = rxgpu_last_error();
				releaseDevice();
			}
		}
		return removed;
	}

	void search(faiss::idx_t n, const float* x, faiss::idx_t k, float* distances, faiss::idx_t* labels,
				const faiss::SearchParameters* params = nullptr) const {
		ensureDevice();
		const uint32_t nprobe = nprobeOf(params);
		std::vector<uint64_t> lab(size_t(n) * k);
		std::vector<uint32_t> cnt(n);
		// any k (IvfIndex asks for large k when other conditions filter the KNN result): k <= 256 at nprobe <= 1024 takes the fused path
		check(rxgpu_ivf_search_knn_large_k(gpu_, uint32_t(n), x, uint32_t(k), nprobe, distances, lab.data(), cnt.data()));
		const bool similarity = cpu_->metric_type != faiss::METRIC_L2;
		for (faiss::idx_t q = 0; q < n; ++q) {
			for (faiss::idx_t j = 0; j < k; ++j) {
				const size_t at = size_t(q) * k + j;
				if (j < cnt[q]) {
					labels[at] = faiss::idx_t(lab[at]);
					if (similarity) {
						distances[at] = -distances[at];
					}
				} else {  // faiss pads with -1 and the heap's neutral value
					labels[at] = -1;
					distances[at] = similarity ? -std::numeric_limits<float>::max() : std::numeric_limits<float>::max();
				}
			}
		}
	}
	void range_search(faiss::idx_t n, const float* x, float radius, faiss::RangeSearchResult* result,
					  const faiss::SearchParameters* params = nullptr) const {
		ensureDevice();
		const uint32_t nprobe = nprobeOf(params);
		const bool similarity = cpu_->metric_type != faiss::METRIC_L2;
		std::vector<std::vector<float>> d(n);
		std::vector<std::vector<uint64_t>> l(n);
		if (n > 1) {  // one coarse pass and one scan of the probed lists for the whole batch
			rangeBatch(n, x, similarity ? -radius : radius, nprobe, d, l);
			for (faiss::idx_t q = 0; q < n; ++q) {
				result->lims[q] = d[q].size();
			}
		} else {
			for (faiss::idx_t q = 0; q < n; ++q) {
				uint64_t total = 0;
				d[q].resize(256);
				l[q].resize(256);
				const float r = similarity ? -radius : radius;  // map space: dist < r
				check(rxgpu_ivf_search_range(gpu_, x + size_t(q) * cpu_->d, r, nprobe, d[q].size(), d[q].data(), l[q].data(), &total));
				if (total > d[q].size()) {
					d[q].resize(total);
					l[q].resize(total);
					check(rxgpu_ivf_search_range(gpu_, x + size_t(q) * cpu_->d, r, nprobe, d[q].size(), d[q].data(), l[q].data(), &total));
				}
				d[q].resize(total);
				l[q].resize(total);
				result->lims[q] = total;
			}
		}
		result->do_allocation();  // turns the counts in lims into offsets and allocates labels / distances
		for (faiss::idx_t q = 0; q < n; ++q) {
			for (size_t i = 0; i < d[q].size(); ++i) {
				result->labels[result->lims[q] + i] = faiss::idx_t(l[q][i]);
				result->distances[result->lims[q] + i] = similarity ? -d[q][i] : d[q][i];
			}
		}
	}

	// Building the index on the device -- replaces IvfIndex::trainIdx followed by add_with_ids of every row (the training upsert,
	// ivf_index.cc:97-102, and RebuildCentroids, :671-679): `idx` is the new, untrained IndexIVFFlat over its empty quantizer.  The
	// centroids are trained on the first `ntrain` rows (all n by default; RebuildCentroids trains on a part) by rxgpu_ivf_train with
	// idx.cp's niter / seed / max_points_per_centroid, added to idx.quantizer, and both are marked trained; every row is then assigned
	// on the device (rxgpu_ivf_add_assign) and its list handed to idx.add_core, so FAISS's lists and the device's are the same by
	// construction.  This map then owns idx and keeps the device index it built: the next search needs no import.  Cosine: norms are
	// the rows' norm coefficients as IvfIndex passes them, or NULL (computed here as add_with_ids does).  Throws on any error, leaving
	// this map as it was.
	void TrainAndFill(std::unique_ptr<faiss::IndexIVFFlat> idx, const float* x, const float* norms, size_t n, const faiss::idx_t* ids,
					  size_t ntrain = 0) {
		ntrain = ntrain ? ntrain : n;
		const auto metric = idx->metric_type == faiss::METRIC_L2 ? RXGPU_L2 : idx->is_cosine ? RXGPU_COS : RXGPU_IP;
		const size_t dim = size_t(idx->d), nlist = idx->nlist;
		if (idx->direct_map.type != faiss::DirectMap::Type::Hashtable) {
			idx->set_direct_map_type(faiss::DirectMap::Type::Hashtable);  // as IvfIndex::trainIdx sets it
		}
		rxgpu_index* ix = nullptr;
		check(rxgpu_index_create(&ix, metric, uint32_t(dim), 16, deviceFromEnv(), 0));
		std::unique_ptr<rxgpu_index, void (*)(rxgpu_index*)> guard(ix, rxgpu_index_destroy);
		const rxgpu_ivf_train_params prm{int32_t(idx->cp.niter), int32_t(idx->cp.seed), int32_t(idx->cp.max_points_per_centroid)};
		std::vector<float> centroids(nlist * dim);
		check(rxgpu_ivf_train(ix, uint32_t(nlist), uint64_t(ntrain), x, norms, &prm, centroids.data(), nullptr));
		idx->quantizer->reset();
		idx->quantizer->add(faiss::idx_t(nlist), centroids.data());  // IndexFlatCosine computes the centroids' norm coefficients here
		idx->quantizer->is_trained = true;
		idx->is_trained = true;
		std::vector<uint64_t> labels(ids, ids + n);
		std::vector<uint32_t> lists(n);
		check(rxgpu_ivf_add_assign(ix, uint64_t(n), labels.data(), x, norms, lists.data()));
		std::vector<float> coefs;
		if (metric == RXGPU_COS && !norms) {  // IndexIVF::add_with_ids without norms: the coefficients of NormalizeVector
			coefs.resize(n);
			std::vector<float> row(dim);
			for (size_t i = 0; i < n; ++i) {
				coefs[i] = reindexer::ann::NormalizeCopyVector(x + i * dim, int32_t(dim), row.data());
			}
			norms = coefs.data();
		}
		const std::vector<faiss::idx_t> listNos(lists.begin(), lists.end());
		idx->add_core(faiss::idx_t(n), x, metric == RXGPU_COS ? norms : nullptr, ids, listNos.data());
		std::lock_guard<std::mutex> lck(mtx_);
		releaseDevice();
		cpu_ = std::move(idx);
		gpu_ = guard.release();
	}

	size_t DeviceImports() const noexcept { return imports_; }
	const std::string& LastDeviceError() const noexcept { return lastError_; }

private:
	// n queries in one rxgpu_ivf_search_range_batch with room for 256 matches each, then one more batch of only the queries with more,
	// with room for the largest of them; r in map space.  d[q] / l[q] receive all matches of query q, best first.
	void rangeBatch(faiss::idx_t n, const float* x, float r, uint32_t nprobe, std::vector<std::vector<float>>& d,
					std::vector<std::vector<uint64_t>>& l) const {
		const size_t dim = cpu_->d;
		uint64_t room = 256;
		std::vector<float> rad(n, r), bd(size_t(n) * room);
		std::vector<uint64_t> bl(size_t(n) * room), cnt(n);
		check(rxgpu_ivf_search_range_batch(gpu_, uint32_t(n), x, rad.data(), nprobe, room, bd.data(), bl.data(), cnt.data()));
		std::vector<faiss::idx_t> more;
		uint64_t most = 0;
		for (faiss::idx_t q = 0; q < n; ++q) {
			if (cnt[q] > room) {
				more.push_back(q);
				most = std::max(most, cnt[q]);
				continue;
			}
			d[q].assign(bd.begin() + size_t(q) * room, bd.begin() + size_t(q) * room + cnt[q]);
			l[q].assign(bl.begin() + size_t(q) * room, bl.begin() + size_t(q) * room + cnt[q]);
		}
		if (more.empty()) {
			return;
		}
		room = most;
		std::vector<float> mq(more.size() * dim);
		for (size_t i = 0; i < more.size(); ++i) {
			std::copy(x + size_t(more[i]) * dim, x + size_t(more[i] + 1) * dim, mq.begin() + i * dim);
		}
		bd.assign(more.size() * room, 0.f);
		bl.assign(more.size() * room, 0);
		check(rxgpu_ivf_search_range_batch(gpu_, uint32_t(more.size()), mq.data(), rad.data(), nprobe, room, bd.data(), bl.data(), cnt.data()));
		for (size_t i = 0; i < more.size(); ++i) {
			d[more[i]].assign(bd.begin() + i * room, bd.begin() + i * room + cnt[i]);
			l[more[i]].assign(bl.begin() + i * room, bl.begin() + i * room + cnt[i]);
		}
	}
	static void check(int rc) {
		if (rc != RXGPU_OK) {
			throw std::runtime_error(rxgpu_last_error());
		}
	}
	static int deviceFromEnv() {
		const char* e = std::getenv("RX_GPU_DEVICE");
		return e ? std::atoi(e) : 0;
	}
	uint32_t nprobeOf(const faiss::SearchParameters* params) const {
		if (const auto* p = dynamic_cast<const faiss::IVFSearchParameters*>(params)) {
			return uint32_t(p->nprobe);
		}
		return uint32_t(cpu_->nprobe);
	}
	uint32_t listOf(faiss::idx_t id) const {
		const auto it = cpu_->direct_map.hashtable.find(id);
		if (it == cpu_->direct_map.hashtable.end()) {
			throw std::logic_error("GpuIvfMap: the id is missing from FAISS' direct map (set_direct_map_type(Hashtable) is required)");
		}
		return uint32_t(faiss::lo_listno(it->second));
	}
	void releaseDevice() noexcept {
		if (gpu_) {
			rxgpu_index_destroy(gpu_);
			gpu_ = nullptr;
		}
	}
	// one import of the trained index: centroids from the coarse quantiser, then every inverted list as one batch
	void ensureDevice() const {
		std::lock_guard<std::mutex> lck(mtx_);
		if (gpu_) {
			return;
		}
		const faiss::IndexIVFFlat& idx = *cpu_;
		const auto metric = idx.metric_type == faiss::METRIC_L2 ? RXGPU_L2 : idx.is_cosine ? RXGPU_COS : RXGPU_IP;
		rxgpu_index* ix = nullptr;
		check(rxgpu_index_create(&ix, metric, uint32_t(idx.d), 16, deviceFromEnv(), 0));
		std::unique_ptr<rxgpu_index, void (*)(rxgpu_index*)> guard(ix, rxgpu_index_destroy);
		std::vector<float> centroids(idx.nlist * size_t(idx.d));
		idx.quantizer->reconstruct_n(0, faiss::idx_t(idx.nlist), centroids.data());
		check(rxgpu_ivf_create(ix, uint32_t(idx.nlist), centroids.data()));
		std::vector<uint32_t> lists;
		std::vector<uint64_t> labels;
		for (size_t l = 0; l < idx.nlist; ++l) {
			const size_t sz = idx.invlists->list_size(l);
			if (!sz) {
				continue;
			}
			faiss::InvertedLists::ScopedCodes codes(idx.invlists, l);
			faiss::InvertedLists::ScopedIds ids(idx.invlists, l);
			lists.assign(sz, uint32_t(l));
			labels.assign(ids.get(), ids.get() + sz);
			check(rxgpu_ivf_add(ix, sz, lists.data(), labels.data(), reinterpret_cast<const float*>(codes.get())));
		}
		gpu_ = guard.release();
		++imports_;
	}

	std::unique_ptr<faiss::IndexIVFFlat> cpu_;
	mutable rxgpu_index* gpu_ = nullptr;
	mutable std::mutex mtx_;
	mutable size_t imports_ = 0;
	mutable std::string lastError_;
};

}  // namespace reindexer
