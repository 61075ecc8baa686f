// Drop-in `Map` for HnswIndexBase<Map> (cpp_src/core/index/float_vector/hnsw_index.h:13-57) with the member surface of
// hnswlib::HierarchicalNSW<synchronization> (cpp_src/core/index/float_vector/hnswlib/hnsw.h:13-73): graph CONSTRUCTION stays with
// the reference's own inserter (HierarchicalNSWImpl::addPoint, hnswalg.h:1695-1852 -- heuristic neighbour selection, level RNG seeded
// with 100, tombstone replacement), SEARCH runs on the GPU through librxgpu (include/rxgpu.h: rxgpu_hnsw_import / _search_knn /
// _search_range / _mark_deleted / _update).  The device copy (rows in internal-id order + level-0 slab + upper levels) is imported by
// the first search; after that single-writer inserts patch it in place (rxgpu_hnsw_update: the inserted row and the lists of the nodes
// the reference's inserter rewrote), MarkDelete sets a tombstone bit (like hnswalg.h:1303-1335).  Concurrent bulk inserts, resizes and
// cache loads re-import -- unless device building is switched on (constructor flag, RX_GPU_HNSW_BUILD at the patch site): then
// AddPointConcurrent only stages (label, vector), and the first other member call sorts the staged rows by label, appends them to the
// device copy and inserts them there with rxgpu_hnsw_build, then writes the new nodes and every list they changed back into the host
// graph with addPoint's bookkeeping.  The host graph then equals the device graph list for list and no import follows.  That graph
// differs from the one the reference's inserter would build (DESIGN.md §3.8), so the switch is off by default.
// Meant to be dropped into cpp_src/core/index/float_vector/hnswlib/ next to hnsw.h; it includes the reference's own headers and is
// therefore compiled only where that tree is available (tests/cpp/dropin_hnsw_check.cc does so in the authoring container).
// INTEGRATION.md section 5 shows the patch of hnsw_index.cc.
//
// Not on the device (explicit, never silent): scalar quantisation (QuantizationAvailable() is false, Quantize throws) and
// streaming search (Begin/ContinueStreamingSearch run the reference's own routine on the host graph this adapter keeps for inserts).
#pragma once

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <memory>
#include <mutex>
#include <optional>
#include <stdexcept>
#include <numeric>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "core/index/float_vector/float_vector_id.h"
#include "core/index/float_vector/hnswlib/hnswalg.h"
#include "core/keyvalue/float_vector.h"
#include "rxgpu.h"

namespace hnswlib {

template <Synchronization synchronization>
class [[nodiscard]] GpuHnsw {
	using Cpu = HierarchicalNSWImpl<float, synchronization>;

public:
	GpuHnsw(reindexer::IsArray, reindexer::VectorMetric metric, size_t dim, size_t maxElements, size_t M, size_t efConstruction,
			bool deviceBuild = false)
		: metric_(metric),
		  dim_(dim),
		  cpu_(std::make_unique<Cpu>(metric, dim, maxElements, M, efConstruction, kHnswRandomSeed, reindexer::ReplaceDeleted_True)),
		  deviceBuild_(deviceBuild) {}
	GpuHnsw(const GpuHnsw& other, size_t newCapacity)
		: metric_(other.metric_),
		  dim_(other.dim_),
		  cpu_((other.materialise(), std::make_unique<Cpu>(*other.cpu_, newCapacity))),
		  deviceBuild_(other.deviceBuild_) {}  // device copy: lazily
	GpuHnsw& operator=(GpuHnsw&& o) noexcept {
		releaseDevice();
		metric_ = o.metric_;
		dim_ = o.dim_;
		cpu_ = std::move(o.cpu_);
		gpu_ = std::exchange(o.gpu_, nullptr);
		dirty_.store(o.dirty_.load());
		hasPending_.store(o.hasPending_.load());
		pendingRows_ = std::move(o.pendingRows_);
		pendingLists_ = std::move(o.pendingLists_);
		deviceCapacity_ = o.deviceCapacity_;
		deviceBuild_ = o.deviceBuild_;
		stagedLabels_ = std::move(o.stagedLabels_);
		stagedRows_ = std::move(o.stagedRows_);
		stagedIndex_ = std::move(o.stagedIndex_);
		stagedCount_.store(o.stagedCount_.load());
		return *this;
	}
	~GpuHnsw() { releaseDevice(); }

	// staged rows count: upsertConcurrent's capacity check (hnsw_index.cc:106) sees them
	size_t MaxElements() const noexcept { return cpu_->MaxElements(); }
	size_t CurrentElementCount() const noexcept { return cpu_->CurrentElementCount() + stagedCount_.load(std::memory_order_acquire); }
	size_t DeletedCountUnsafe() const {
		materialise();
		return cpu_->DeletedCountUnsafe();
	}
	size_t AllocatedMemSize() const {
		materialise();
		return cpu_->AllocatedMemSize();
	}
	size_t ElementSize() const noexcept { return cpu_->ElementSize(); }
	size_t DeviceMemSize() const {
		materialise();
		return gpu_ ? rxgpu_index_device_bytes(gpu_) : 0;
	}
	labeltype ExternalLabel(tableint internalId) const {
		materialise();
		return cpu_->ExternalLabel(internalId);
	}
	bool IsMarkedDeleted(tableint internalId) const {
		materialise();
		return cpu_->IsMarkedDeleted(internalId);
	}
	const float* FloatPtrByExternalLabel(labeltype label) const {
		materialise();
		return cpu_->FloatPtrByExternalLabel(label);
	}
	size_t GetHash(reindexer::FloatVectorId id) const {
		materialise();
		return cpu_->GetHash(id.AsNumber());
	}

	void MarkDelete(reindexer::FloatVectorId id) {
		materialise();
		const labeltype label = id.AsNumber();
		if (gpu_ && !dirty_.load(std::memory_order_acquire) && hasPending_.load(std::memory_order_acquire)) {
			try {
				flushPending();  // the label may belong to a row that is not on the device yet
			} catch (const std::exception& e) {
				lastPatchError_ = e.what();
				dirty_.store(true, std::memory_order_release);
			}
		}
		cpu_->MarkDelete(label);  // throws "markDelete: Label not found: ..." / "... already deleted" like the reference
		if (gpu_ && !dirty_.load(std::memory_order_acquire)) {
			if (rxgpu_hnsw_mark_deleted(gpu_, label) != RXGPU_OK) {
				lastPatchError_ = rxgpu_last_error();
				dirty_.store(true, std::memory_order_release);  // the device copy is rebuilt by the next search
			}
		}
	}
	// Single-writer insert (the namespace's exclusive lock): the device copy is patched in place by the next search -- the nodes whose
	// lists addPoint / updatePoint rewrote are known exactly (one-hop neighbours before and after the call), so an upsert costs O(M) small copies, not a re-import.
	void AddPointNoLock(reindexer::ConstFloatVectorView vect, reindexer::FloatVectorId id) {
		materialise();
		const labeltype label = id.AsNumber();
		if (!gpu_ || dirty_.load(std::memory_order_acquire)) {
			cpu_->AddPointNoLock(vect.Data(), label);
			dirty_.store(true, std::memory_order_release);
			return;
		}
		// which slot the reference will write (hnswalg.h:1401-1470): a vacant tombstone first, else the label's own node, else a new one
		const size_t before = cpu_->cur_element_count.load();
		const auto known = cpu_->label_lookup_.find(label);
		const bool vacant = !cpu_->deleted_elements.empty();
		bool trackable = !(vacant && known != cpu_->label_lookup_.end());
		tableint node = vacant ? *cpu_->deleted_elements.begin() : known != cpu_->label_lookup_.end() ? known->second : tableint(before);
		std::vector<tableint> touched;
		if (node < before) {
			neighboursOf(node, touched);  // updatePoint re-selects the lists of the old one-hop neighbours (hnswalg.h:1512-1583)
		}
		cpu_->AddPointNoLock(vect.Data(), label);
		trackable = trackable && cpu_->cur_element_count.load() == (node < before ? before : before + 1) && cpu_->MaxElements() == deviceCapacity_;
		if (!trackable) {
			lastPatchError_ = "insert not trackable (label lives in another slot while a tombstone is vacant, or the map was resized)";
			dirty_.store(true, std::memory_order_release);
			return;
		}
		neighboursOf(node, touched);  // mutuallyConnectNewElement rewrote the lists of the selected neighbours (hnswalg.h:1070-1180)
		std::lock_guard<std::mutex> lck(mtx_);
		pendingRows_.push_back(node);
		pendingLists_.insert(pendingLists_.end(), touched.begin(), touched.end());
		if (pendingLists_.size() > std::max<size_t>(4096, before / 4)) {  // a bulk load: one import is cheaper than the patches
			dirty_.store(true, std::memory_order_release);
		}
		hasPending_.store(true, std::memory_order_release);
	}
	// The transaction's inserter threads (TransactionConcurrentInserter).  Device building: a new label on a map without tombstones is
	// only staged, never touching the device; an existing label, or a map whose tombstones replace_deleted would reuse, takes the
	// reference's path.  Without device building, concurrent inserts interleave their list rewrites, so the set of touched nodes is not
	// known per call: full re-import.
	void AddPointConcurrent(reindexer::ConstFloatVectorView vect, reindexer::FloatVectorId id) {
		const labeltype label = id.AsNumber();
		if (deviceBuild_) {
			std::lock_guard<std::mutex> lck(stageMtx_);  // also orders the reference's path below after the label_lookup_ read
			if (cpu_->DeletedCountUnsafe() == 0 && cpu_->label_lookup_.find(label) == cpu_->label_lookup_.end()) {
				if (const auto it = stagedIndex_.find(label); it != stagedIndex_.end()) {  // staged twice: the later vector wins
					std::copy(vect.Data(), vect.Data() + dim_, stagedRows_.begin() + it->second * dim_);
					return;
				}
				if (cpu_->CurrentElementCount() + stagedLabels_.size() >= cpu_->MaxElements()) {
					throw std::runtime_error("The number of elements exceeds the specified limit");  // hnswalg.h:1730
				}
				stagedIndex_.emplace(label, stagedLabels_.size());
				stagedLabels_.push_back(label);
				stagedRows_.insert(stagedRows_.end(), vect.Data(), vect.Data() + dim_);
				stagedCount_.store(stagedLabels_.size(), std::memory_order_release);
				return;
			}
			cpu_->AddPointConcurrent(vect.Data(), label);
			dirty_.store(true, std::memory_order_release);
			return;
		}
		cpu_->AddPointConcurrent(vect.Data(), label);
		dirty_.store(true, std::memory_order_release);
	}
	void ResizeIndex(size_t newMaxElements) {
		materialise();
		cpu_->ResizeIndex(newMaxElements);
		dirty_.store(true, std::memory_order_release);  // the device copy is re-imported at the new capacity
	}
	void SaveIndex(IWriter& writer, const std::atomic_int32_t& cancel) const {
		materialise();
		writer.PutVarUInt(uint32_t(0));  // not quantised (HierarchicalNSW::serializeQuantizingParams, hnsw.cc:52-58)
		cpu_->SaveIndex(writer, cancel);
	}
	void LoadIndex(IReader& reader) {
		materialise();
		if (reader.GetVarUInt() != 0) {
			throw std::runtime_error("GpuHnsw: quantised HNSW caches are not supported on the device path");
		}
		cpu_ = std::make_unique<Cpu>(reader, metric_, dim_, kHnswRandomSeed, reindexer::ReplaceDeleted_True, std::nullopt);
		dirty_.store(true, std::memory_order_release);
	}
	void Reset() noexcept {
		stagedLabels_.clear();
		stagedRows_.clear();
		stagedIndex_.clear();
		stagedCount_.store(0);
		releaseDevice();
		cpu_.reset();
	}

	// returns the reference's max-heap (worst on top) so that HnswIndexBase::select drains it unchanged
	SearchResultQueue SearchKnn(const float* queryData, std::optional<float> /*queryDataNorm*/, size_t k, size_t ef = 0) const {
		using pair_t = std::pair<float, labeltype>;
		materialise();
		if (cpu_->CurrentElementCount() == 0) {
			return SearchResultQueue();  // hnswalg.h:1989-1991
		}
		ensureDevice();
		const size_t n = std::min<size_t>(k, cpu_->CurrentElementCount());
		std::vector<float> dists(std::max<size_t>(n, 1));
		std::vector<uint64_t> labels(std::max<size_t>(n, 1));
		uint32_t count = 0;
		check(rxgpu_hnsw_search_knn(gpu_, 1, queryData, uint32_t(n), uint32_t(ef), dists.data(), labels.data(), &count, nullptr));
		std::vector<pair_t> container;
		container.reserve(count);
		for (uint32_t i = 0; i < count; ++i) {
			container.emplace_back(dists[i], labels[i]);
		}
		return SearchResultQueue(std::less<pair_t>(), std::move(container));
	}
	SearchResultQueue SearchRange(const float* queryData, std::optional<float> /*queryDataNorm*/, float radius, size_t ef) const {
		using pair_t = std::pair<float, labeltype>;
		materialise();
		if (cpu_->CurrentElementCount() == 0) {
			return SearchResultQueue();  // hnswalg.h:2017-2019
		}
		ensureDevice();
		uint64_t total = 0;
		std::vector<float> dists(256);
		std::vector<uint64_t> labels(256);
		check(rxgpu_hnsw_search_range(gpu_, queryData, radius, uint32_t(ef), dists.size(), dists.data(), labels.data(), &total));
		if (total > dists.size()) {
			dists.resize(total);
			labels.resize(total);
			check(rxgpu_hnsw_search_range(gpu_, queryData, radius, uint32_t(ef), dists.size(), dists.data(), labels.data(), &total));
		}
		std::vector<pair_t> container;
		container.reserve(total);
		for (uint64_t i = 0; i < total; ++i) {
			container.emplace_back(dists[i], labels[i]);
		}
		return SearchResultQueue(std::less<pair_t>(), std::move(container));
	}
	// streaming search: the reference's own routine on the host graph (hnswalg.h:1865-1975)
	StreamingSearchSession BeginStreamingSearch(const float* queryData, std::optional<float> queryDataNorm, StreamingSearchOptions opts) const {
		materialise();
		return cpu_->BeginStreamingSearch(queryData, queryDataNorm, opts);
	}
	StreamingBatch ContinueStreamingSearch(StreamingSearchSession& session, size_t batchSize) const {
		return cpu_->ContinueStreamingSearch(session, batchSize);
	}

	bool IsQuantized() const noexcept { return false; }
	bool QuantizationAvailable() const noexcept { return false; }
	void Quantize(const QuantizationConfig&) { throw std::logic_error("GpuHnsw: scalar quantisation is not available on the device path"); }
	void SwitchMapOnQuantized() {}

	// number of times the device copy was (re)built -- exposed for tests
	size_t DeviceImports() const noexcept { return imports_.load(); }
	// nodes patched in place since the last import
	const std::string& LastPatchError() const noexcept { return lastPatchError_; }  // why the copy was last scheduled for a re-import
	size_t DevicePatchedNodes() const noexcept { return gpu_ ? size_t(rxgpu_hnsw_update_count(gpu_)) : 0; }
	// rows inserted by rxgpu_hnsw_build, and the graphs themselves -- exposed for tests
	size_t DeviceBuiltRows() const noexcept { return builtRows_.load(); }
	const Cpu& HostGraph() const {
		materialise();
		return *cpu_;
	}
	const rxgpu_index* DeviceIndex() const {
		materialise();
		return gpu_;
	}

private:
	constexpr static int kHnswRandomSeed = 100;  // hnsw.h:73

	static rxgpu_metric toMetric(reindexer::VectorMetric m) {
		switch (m) {
			case reindexer::VectorMetric::L2:
				return RXGPU_L2;
			case reindexer::VectorMetric::InnerProduct:
				return RXGPU_IP;
			case reindexer::VectorMetric::Cosine:
				return RXGPU_COS;
		}
		std::abort();
	}
	static int deviceFromEnv() {
		const char* e = std::getenv("RX_GPU_DEVICE");
		return e ? std::atoi(e) : 0;
	}
	static void check(int rc) {
		if (rc != RXGPU_OK) {
			throw std::runtime_error(rxgpu_last_error());
		}
	}
	void releaseDevice() const noexcept {
		if (gpu_) {
			rxgpu_index_destroy(gpu_);
			gpu_ = nullptr;
		}
	}

	// Searches run concurrently under the namespace's shared lock; inserts under its exclusive lock.  The first search after an
	// insertion rebuilds the device copy; the others wait on the mutex.
	void neighboursOf(tableint node, std::vector<tableint>& out) const {
		const Cpu& g = *cpu_;
		for (int lvl = 0; lvl <= g.element_levels_[node]; ++lvl) {
			const auto* ll = lvl == 0 ? g.get_linklist0(node) : g.get_linklist(node, lvl);
			const unsigned cnt = g.getListCount(ll);
			for (unsigned j = 0; j < cnt; ++j) {
				out.push_back(readLinkListNeighbor(ll, j));
			}
		}
	}
	// pushes the current lists of every touched node (and the rows of the inserted ones) to the device copy
	void flushPending() const {
		std::lock_guard<std::mutex> lck(mtx_);
		flushPendingLocked();
	}
	void flushPendingLocked() const {
		if (!hasPending_.load(std::memory_order_acquire)) {
			return;
		}
		const Cpu& g = *cpu_;
		const size_t m0 = g.maxM0_, m = g.M_;
		std::vector<tableint> rows = pendingRows_, lists = pendingLists_;
		std::sort(rows.begin(), rows.end());
		rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
		std::sort(lists.begin(), lists.end());
		lists.erase(std::unique(lists.begin(), lists.end()), lists.end());
		std::vector<tableint> order = rows;  // rows first, in internal-id order (appends must arrive that way)
		for (const tableint v : lists) {
			if (!std::binary_search(rows.begin(), rows.end(), v)) {
				order.push_back(v);
			}
		}
		size_t slots = 0;
		for (const tableint v : order) {
			slots += size_t(g.element_levels_[v]);
		}
		std::vector<uint32_t> level0(order.size() * (1 + m0)), upper(slots * (1 + m));
		std::vector<rxgpu_hnsw_node_update> upd(order.size());
		size_t slot = 0;
		for (size_t i = 0; i < order.size(); ++i) {
			const tableint v = order[i];
			uint32_t* dst0 = level0.data() + i * (1 + m0);
			const auto* ll0 = g.get_linklist0(v);
			const unsigned cnt0 = g.getListCount(ll0);
			dst0[0] = cnt0;
			for (size_t j = 0; j < cnt0; ++j) {
				dst0[1 + j] = readLinkListNeighbor(ll0, j);
			}
			rxgpu_hnsw_node_update& u = upd[i];
			u.node = v;
			u.level = g.element_levels_[v];
			u.level0 = dst0;
			u.upper = u.level > 0 ? upper.data() + slot * (1 + m) : nullptr;
			for (int lvl = 1; lvl <= u.level; ++lvl, ++slot) {
				const auto* ll = g.get_linklist(v, lvl);
				const unsigned cnt = g.getListCount(ll);
				uint32_t* dst = upper.data() + slot * (1 + m);
				dst[0] = cnt;
				for (size_t j = 0; j < cnt; ++j) {
					dst[1 + j] = readLinkListNeighbor(ll, j);
				}
			}
			const bool isRow = i < rows.size();
			u.vec = isRow ? reinterpret_cast<const float*>(g.getDataByInternalId(v)) : nullptr;
			u.deleted = g.IsMarkedDeleted(v) ? 1 : 0;
			u.label = u.deleted ? ((uint64_t(1) << 63) | uint64_t(v)) : uint64_t(g.ExternalLabel(v));
		}
		check(rxgpu_hnsw_update(gpu_, g.maxlevel_, uint32_t(g.enterpoint_node_), uint32_t(upd.size()), upd.data()));
		pendingRows_.clear();
		pendingLists_.clear();
		hasPending_.store(false, std::memory_order_release);
	}

	// Inserts the staged rows: sorted by label (so the graph depends on the set of rows, not on thread timing), appended to the device
	// copy brought up to date first, levels drawn from the host graph's own generator as addPoint would draw them, rxgpu_hnsw_build,
	// then the new nodes and every old node their lists name are read back and written into the host graph.  When the device step
	// fails the rows go through the reference's inserter instead and the device copy is rebuilt by the next search.
	void materialise() const {
		if (stagedCount_.load(std::memory_order_acquire) == 0) {
			return;
		}
		std::lock_guard<std::mutex> lck(stageMtx_);
		const size_t cnt = stagedLabels_.size();
		if (cnt == 0) {
			return;
		}
		std::vector<size_t> order(cnt);
		std::iota(order.begin(), order.end(), size_t(0));
		std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return stagedLabels_[a] < stagedLabels_[b]; });
		std::vector<uint64_t> labels(cnt);
		std::vector<float> rows(cnt * dim_);
		for (size_t i = 0; i < cnt; ++i) {
			labels[i] = stagedLabels_[order[i]];
			std::copy_n(stagedRows_.begin() + order[i] * dim_, dim_, rows.begin() + i * dim_);
		}
		stagedLabels_.clear();
		stagedRows_.clear();
		stagedIndex_.clear();
		Cpu& g = *cpu_;
		const size_t first = g.cur_element_count.load();
		std::vector<int32_t> levels(cnt);
		for (auto& l : levels) {
			l = g.template getRandomLevel<DummyLocker>(g.mult_);
		}
		try {
			buildOnDevice(first, labels, rows, levels);
		} catch (const std::exception& e) {
			lastPatchError_ = e.what();
			for (size_t i = 0; i < cnt; ++i) {
				if (g.label_lookup_.find(labels[i]) == g.label_lookup_.end()) {
					g.AddPointNoLock(rows.data() + i * dim_, labels[i]);
				}
			}
			dirty_.store(true, std::memory_order_release);
		}
		stagedCount_.store(0, std::memory_order_release);
	}
	void buildOnDevice(size_t first, const std::vector<uint64_t>& labels, const std::vector<float>& rows, const std::vector<int32_t>& levels) const {
		Cpu& g = *cpu_;
		const size_t cnt = labels.size(), m0 = g.maxM0_, m = g.M_;
		if (first == 0) {  // nothing to import: a fresh device index
			std::lock_guard<std::mutex> lk(mtx_);
			releaseDevice();
			pendingRows_.clear();
			pendingLists_.clear();
			hasPending_.store(false, std::memory_order_release);
			rxgpu_index* ix = nullptr;
			check(rxgpu_index_create(&ix, toMetric(metric_), uint32_t(dim_), g.MaxElements(), deviceFromEnv(), 0));
			gpu_ = ix;
			deviceCapacity_ = g.MaxElements();
			dirty_.store(false, std::memory_order_release);
		} else {
			if (first + cnt > deviceCapacity_) {
				dirty_.store(true, std::memory_order_release);  // re-imported at the map's capacity
			}
			ensureDevice();
		}
		check(rxgpu_index_upsert_batch(gpu_, cnt, labels.data(), rows.data()));
		rxgpu_hnsw_build_stats st{};
		check(rxgpu_hnsw_build(gpu_, uint32_t(m), uint32_t(g.ef_construction_), first, levels.data(), 0, &st));
		// the new nodes, then every old node one of their lists names: only those lists changed
		std::vector<uint32_t> nodes(cnt);
		std::iota(nodes.begin(), nodes.end(), uint32_t(first));
		rxgpu_hnsw_graph info{};
		std::vector<uint32_t> l0, up;
		std::vector<int32_t> lv;
		std::vector<int64_t> off;
		auto read = [&](const std::vector<uint32_t>& which) {
			l0.assign(which.size() * (1 + m0), 0u);
			lv.assign(which.size(), 0);
			off.assign(which.size() + 1, 0);
			check(rxgpu_hnsw_export(gpu_, which.size(), which.data(), l0.data(), lv.data(), off.data(), nullptr, &info));
			up.assign(std::max<int64_t>(off[which.size()], 1) * (1 + m), 0u);
			check(rxgpu_hnsw_export(gpu_, which.size(), which.data(), nullptr, nullptr, nullptr, up.data(), nullptr));
		};
		read(nodes);
		std::vector<uint32_t> oldNodes;
		for (size_t i = 0; i < cnt; ++i) {
			for (uint32_t j = 1; j <= l0[i * (1 + m0)]; ++j) {
				oldNodes.push_back(l0[i * (1 + m0) + j]);
			}
			for (int64_t s = off[i]; s < off[i + 1]; ++s) {
				for (uint32_t j = 1; j <= up[s * (1 + m)]; ++j) {
					oldNodes.push_back(up[s * (1 + m) + j]);
				}
			}
		}
		oldNodes.erase(std::remove_if(oldNodes.begin(), oldNodes.end(), [&](uint32_t v) { return v >= first; }), oldNodes.end());
		std::sort(oldNodes.begin(), oldNodes.end());
		oldNodes.erase(std::unique(oldNodes.begin(), oldNodes.end()), oldNodes.end());
		const std::vector<uint32_t> newL0 = l0, newUp = up;
		const std::vector<int64_t> newOff = off;
		// addPoint's bookkeeping for every new node (hnswalg.h:1727-1775)
		for (size_t i = 0; i < cnt; ++i) {
			const tableint id = tableint(first + i);
			const float* data = rows.data() + i * dim_;
			g.label_lookup_[labels[i]] = id;
			g.cur_element_count++;
			g.fstdistfunc_.AddNorm(data, id);
			g.element_levels_[id] = levels[i];
			std::memset(g.data_level0_memory_ + size_t(id) * g.size_data_per_element_, 0, g.size_data_per_element_);
			g.setExternalLabel(id, labels[i]);
			g.setHashByInternalId(id, g.CalcHash(data));
			std::memcpy(g.getDataByInternalId(id), data, g.data_size_);
			if (levels[i]) {
				g.linkLists_[id] = static_cast<char*>(malloc(g.size_links_per_element_ * levels[i] + 1));
				if (g.linkLists_[id] == nullptr) {
					throw std::runtime_error("Not enough memory: addPoint failed to allocate linklist");
				}
				std::memset(g.linkLists_[id], 0, g.size_links_per_element_ * levels[i] + 1);
			}
		}
		auto write = [&](tableint v, const uint32_t* list0, const uint32_t* upper, int level) {
			auto put = [&](linklistsizeint* ll, const uint32_t* src) {
				g.setListCount(ll, (unsigned short)src[0]);
				for (uint32_t j = 0; j < src[0]; ++j) {
					writeLinkListNeighbor(ll, j, src[1 + j]);
				}
			};
			put(g.get_linklist0(v), list0);
			for (int l = 1; l <= level; ++l) {
				put(g.get_linklist(v, l), upper + size_t(l - 1) * (1 + m));
			}
		};
		for (size_t i = 0; i < cnt; ++i) {
			write(tableint(first + i), newL0.data() + i * (1 + m0), newUp.data() + newOff[i] * (1 + m), levels[i]);
		}
		if (!oldNodes.empty()) {
			read(oldNodes);
			for (size_t i = 0; i < oldNodes.size(); ++i) {
				write(tableint(oldNodes[i]), l0.data() + i * (1 + m0), up.data() + off[i] * (1 + m), lv[i]);
			}
		}
		g.maxlevel_ = info.maxlevel;
		g.enterpoint_node_ = tableint(info.enterpoint);
		builtRows_.fetch_add(cnt);
	}

	void ensureDevice() const {
		if (gpu_ && !dirty_.load(std::memory_order_acquire) && !hasPending_.load(std::memory_order_acquire)) {
			return;
		}
		std::lock_guard<std::mutex> lck(mtx_);
		if (gpu_ && !dirty_.load(std::memory_order_acquire)) {
			try {
				flushPendingLocked();
				return;
			} catch (const std::exception& e) {  // e.g. the slab of upper-level lists is full: rebuild the copy from the host graph
				lastPatchError_ = e.what();
				dirty_.store(true, std::memory_order_release);
			}
		}
		pendingRows_.clear();
		pendingLists_.clear();
		hasPending_.store(false, std::memory_order_release);
		const Cpu& g = *cpu_;
		const size_t n = g.cur_element_count.load();
		const size_t m0 = g.maxM0_, m = g.M_;
		if (gpu_) {
			rxgpu_index_destroy(gpu_);
			gpu_ = nullptr;
		}
		rxgpu_index* ix = nullptr;
		check(rxgpu_index_create(&ix, toMetric(metric_), uint32_t(dim_), std::max(n, g.MaxElements()), deviceFromEnv(), 0));
		deviceCapacity_ = std::max(n, g.MaxElements());
		std::unique_ptr<rxgpu_index, void (*)(rxgpu_index*)> guard(ix, rxgpu_index_destroy);
		// rows in internal-id order (internal id i = row i), in slices; a tombstone keeps its slot but gets a label of its own:
		// with replace_deleted the same external label may live again in another slot (hnswalg.h:1710-1760)
		std::vector<uint32_t> level0(n * (1 + m0));
		std::vector<int32_t> levels(n);
		std::vector<int64_t> upperOffsets(n + 1);
		std::vector<uint32_t> upper;
		std::vector<uint64_t> labels(n);
		std::vector<tableint> deleted;
		int64_t slot = 0;
		for (size_t i = 0; i < n; ++i) {
			slot += g.element_levels_[i];
		}
		upper.resize(size_t(slot) * (1 + m));
		slot = 0;
		for (size_t i = 0; i < n; ++i) {
			const auto* ll0 = g.get_linklist0(tableint(i));
			const unsigned cnt0 = g.getListCount(ll0);
			uint32_t* dst0 = level0.data() + i * (1 + m0);
			dst0[0] = cnt0;
			for (size_t j = 0; j < m0; ++j) {
				dst0[1 + j] = j < cnt0 ? readLinkListNeighbor(ll0, j) : 0u;
			}
			levels[i] = g.element_levels_[i];
			upperOffsets[i] = slot;
			for (int lvl = 1; lvl <= g.element_levels_[i]; ++lvl, ++slot) {
				const auto* ll = g.get_linklist(tableint(i), lvl);
				const unsigned cnt = g.getListCount(ll);
				uint32_t* dst = upper.data() + size_t(slot) * (1 + m);
				dst[0] = cnt;
				for (size_t j = 0; j < m; ++j) {
					dst[1 + j] = j < cnt ? readLinkListNeighbor(ll, j) : 0u;
				}
			}
			if (g.IsMarkedDeleted(tableint(i))) {
				labels[i] = (uint64_t(1) << 63) | uint64_t(i);
				deleted.push_back(tableint(i));
			} else {
				labels[i] = g.ExternalLabel(tableint(i));
			}
		}
		upperOffsets[n] = slot;
		const size_t slice = std::max<size_t>(1, (size_t(64) << 20) / (dim_ * sizeof(float)));
		std::vector<float> rows(std::min(slice, n) * dim_);
		for (size_t base = 0; base < n; base += slice) {
			const size_t cnt = std::min(slice, n - base);
			for (size_t i = 0; i < cnt; ++i) {
				std::memcpy(rows.data() + i * dim_, g.getDataByInternalId(tableint(base + i)), dim_ * sizeof(float));
			}
			check(rxgpu_index_upsert_batch(ix, cnt, labels.data() + base, rows.data()));
		}
		rxgpu_hnsw_graph graph{};
		graph.n = uint32_t(n);
		graph.M = uint32_t(m);
		graph.maxM0 = uint32_t(m0);
		graph.maxlevel = g.maxlevel_;
		graph.enterpoint = uint32_t(g.enterpoint_node_);
		graph.upper_slots = uint64_t(slot);
		graph.level0 = level0.data();
		graph.levels = levels.data();
		graph.upper_offsets = upperOffsets.data();
		graph.upper = upper.empty() ? nullptr : upper.data();
		check(rxgpu_hnsw_import(ix, &graph));
		for (const tableint i : deleted) {
			check(rxgpu_hnsw_mark_deleted(ix, labels[i]));
		}
		gpu_ = guard.release();
		imports_.fetch_add(1);
		dirty_.store(false, std::memory_order_release);
	}

	reindexer::VectorMetric metric_;
	size_t dim_;
	std::unique_ptr<Cpu> cpu_;
	mutable rxgpu_index* gpu_ = nullptr;
	mutable std::atomic<bool> dirty_{true};        // the device copy must be rebuilt from the host graph
	mutable std::atomic<bool> hasPending_{false};  // ... or only patched: rows written / nodes whose lists were rewritten since
	mutable std::vector<tableint> pendingRows_, pendingLists_;
	mutable size_t deviceCapacity_ = 0;
	mutable std::string lastPatchError_;
	mutable std::atomic<size_t> imports_{0};
	mutable std::mutex mtx_;
	bool deviceBuild_ = false;
	mutable std::mutex stageMtx_;  // the staged rows (AddPointConcurrent) and their materialisation
	mutable std::vector<labeltype> stagedLabels_;
	mutable std::vector<float> stagedRows_;
	mutable std::unordered_map<labeltype, size_t> stagedIndex_;
	mutable std::atomic<size_t> stagedCount_{0};
	mutable std::atomic<size_t> builtRows_{0};
};

}  // namespace hnswlib
