// TEST INFRASTRUCTURE.  GpuHnsw<OnInsertions> with device building switched on, driven like TransactionConcurrentInserter drives the
// reference's map (AddPointConcurrent from 8 threads), in three rounds onto a growing map, beside HierarchicalNSW<OnInsertions> fed the
// same rows by the same threads.  Checks, per metric: the host graph equals the exported device graph list for list; no import
// happened; recall@10 of the reference's SearchKnn on the host graph and of the adapter's device SearchKnn within 0.01 of the reference
// map's; a SaveIndex / LoadIndex round trip searches the same; an existing label and a map with tombstones take the reference's path;
// with the switch off the rows go through the reference's inserter and the first search imports.  One MATCH / MISMATCH line per check.
// Built by tests/cpp/hnsw_build.mk only where the reference tree exists.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <optional>
#include <random>
#include <span>
#include <string>
#include <thread>
#include <vector>

#include "core/index/float_vector/hnswlib/hnsw.h"
#include "gpu_hnsw.h"

namespace {

constexpr size_t kDim = 32, kRound = 4000, kRounds = 3, kThreads = 8, kCap = 16000, kQueries = 300, kK = 10, kEf = 64;
using Sync = hnswlib::Synchronization;

struct Token {
	uint64_t u = 0;
	int64_t i = 0;
	float f = 0.f;
	std::string s;
};
class MemWriter final : public hnswlib::IWriter {
public:
	std::vector<Token> tokens;
	void PutVarUInt(uint64_t v) override { tokens.push_back(Token{v, 0, 0.f, {}}); }
	void PutVarUInt(uint32_t v) override { tokens.push_back(Token{v, 0, 0.f, {}}); }
	void PutVarInt(int64_t v) override { tokens.push_back(Token{0, v, 0.f, {}}); }
	void PutVarInt(int32_t v) override { tokens.push_back(Token{0, v, 0.f, {}}); }
	void PutVString(std::string_view v) override { tokens.push_back(Token{0, 0, 0.f, std::string(v)}); }
	void PutFloat(float v) override { tokens.push_back(Token{0, 0, v, {}}); }
	void AppendPKByID(hnswlib::labeltype label) override { tokens.push_back(Token{label, 0, 0.f, {}}); }
};
class MemReader final : public hnswlib::IReader {
public:
	MemReader(const std::vector<Token>& t, const std::vector<std::vector<float>>& rows) : tokens_(t), rows_(rows) {}
	uint64_t GetVarUInt() override { return tokens_[pos_++].u; }
	int64_t GetVarInt() override { return tokens_[pos_++].i; }
	std::string_view GetVString() override { return tokens_[pos_++].s; }
	float GetFloat() override { return tokens_[pos_++].f; }
	hnswlib::labeltype ReadPkEncodedData(float* destBuf) override {
		const uint64_t label = tokens_[pos_++].u;
		const auto& v = rows_[size_t(label >> 32)];
		std::memcpy(destBuf, v.data(), v.size() * sizeof(float));
		return label;
	}
	bool WithQuantizer() const override { return false; }

private:
	const std::vector<Token>& tokens_;
	const std::vector<std::vector<float>>& rows_;
	size_t pos_ = 0;
};

reindexer::FloatVectorId fid(size_t i) { return reindexer::FloatVectorId{reindexer::IdType::FromNumber(int(i)), 0}; }
reindexer::ConstFloatVectorView view(const std::vector<float>& v) { return reindexer::ConstFloatVectorView{std::span<const float>{v}}; }

int failures = 0;
void report(bool ok, const std::string& what) {
	std::printf("%s %s\n", ok ? "MATCH" : "MISMATCH", what.c_str());
	failures += ok ? 0 : 1;
}

template <typename Map>
void insertConcurrent(Map& map, const std::vector<std::vector<float>>& rows, size_t begin, size_t end) {
	std::vector<std::thread> th;
	for (size_t t = 0; t < kThreads; ++t) {
		th.emplace_back([&, t] {
			for (size_t i = begin + t; i < end; i += kThreads) {
				map.AddPointConcurrent(view(rows[i]), fid(i));
			}
		});
	}
	for (auto& x : th) {
		x.join();
	}
}

std::vector<uint64_t> labelsOf(hnswlib::SearchResultQueue q) {
	std::vector<uint64_t> out;
	while (!q.empty()) {
		out.push_back(q.top().second);
		q.pop();
	}
	return out;
}

double recall(const std::vector<std::vector<uint64_t>>& found, const std::vector<std::vector<uint64_t>>& truth) {
	double hit = 0;
	for (size_t q = 0; q < truth.size(); ++q) {
		for (const uint64_t l : found[q]) {
			hit += std::count(truth[q].begin(), truth[q].end(), l) ? 1 : 0;
		}
	}
	return hit / double(truth.size() * kK);
}

// every list, level, the top level and the enter point of the host graph against the device graph
template <typename G>
bool sameGraph(const G& g, const rxgpu_index* ix) {
	rxgpu_hnsw_graph info{};
	if (rxgpu_hnsw_export(ix, 0, nullptr, nullptr, nullptr, nullptr, nullptr, &info) != RXGPU_OK) {
		return false;
	}
	const size_t n = g.cur_element_count.load(), m0 = g.maxM0_, m = g.M_;
	if (info.n != n || info.maxlevel != g.maxlevel_ || info.enterpoint != g.enterpoint_node_) {
		return false;
	}
	std::vector<uint32_t> l0(n * (1 + m0));
	std::vector<int32_t> lv(n);
	std::vector<int64_t> off(n + 1);
	rxgpu_hnsw_export(ix, n, nullptr, l0.data(), lv.data(), off.data(), nullptr, nullptr);
	std::vector<uint32_t> up(std::max<int64_t>(off[n], 1) * (1 + m));
	rxgpu_hnsw_export(ix, n, nullptr, nullptr, nullptr, nullptr, up.data(), nullptr);
	auto same = [&](const auto* ll, const uint32_t* dev) {
		const unsigned cnt = g.getListCount(ll);
		if (cnt != dev[0]) {
			return false;
		}
		for (unsigned j = 0; j < cnt; ++j) {
			if (hnswlib::readLinkListNeighbor(ll, j) != dev[1 + j]) {
				return false;
			}
		}
		return true;
	};
	for (size_t v = 0; v < n; ++v) {
		if (lv[v] != g.element_levels_[v] || !same(g.get_linklist0(hnswlib::tableint(v)), l0.data() + v * (1 + m0))) {
			return false;
		}
		for (int l = 1; l <= lv[v]; ++l) {
			if (!same(g.get_linklist(hnswlib::tableint(v), l), up.data() + size_t(off[v] + l - 1) * (1 + m))) {
				return false;
			}
		}
	}
	return true;
}

void run(reindexer::VectorMetric metric, const char* name) {
	std::mt19937 rng(7);
	std::normal_distribution<float> nd(0.f, 1.f);
	auto make = [&](size_t n) {
		std::vector<std::vector<float>> out(n, std::vector<float>(kDim));
		for (auto& r : out) {
			for (auto& x : r) {
				x = nd(rng);
			}
		}
		return out;
	};
	const auto rows = make(kRound * kRounds);
	const auto queries = make(kQueries);
	auto dist = [&](const std::vector<float>& q, const std::vector<float>& r) {
		float s = 0.f;
		for (size_t j = 0; j < kDim; ++j) {
			s += metric == reindexer::VectorMetric::L2 ? (q[j] - r[j]) * (q[j] - r[j]) : -q[j] * r[j];
		}
		return s;
	};
	hnswlib::GpuHnsw<Sync::OnInsertions> dev(reindexer::IsArray_False, metric, kDim, kCap, 16, 200, true);
	hnswlib::HierarchicalNSW<Sync::OnInsertions> ref(reindexer::IsArray_False, metric, kDim, kCap, 16, 200);
	bool graphs = true, imports = true;
	for (size_t r = 0; r < kRounds; ++r) {
		insertConcurrent(dev, rows, r * kRound, (r + 1) * kRound);
		insertConcurrent(ref, rows, r * kRound, (r + 1) * kRound);
		imports = imports && dev.CurrentElementCount() == (r + 1) * kRound;
		(void)dev.SearchKnn(queries[0].data(), std::nullopt, kK, kEf);  // materialises the round
		graphs = graphs && sameGraph(dev.HostGraph(), dev.DeviceIndex());
		imports = imports && dev.DeviceImports() == 0 && dev.DeviceBuiltRows() == (r + 1) * kRound;
	}
	report(graphs, std::string(name) + " host graph == device graph after each of 3 rounds");
	report(imports, std::string(name) + " no import, every row built on the device, staged rows counted");
	std::vector<std::vector<uint64_t>> truth(kQueries), fRef(kQueries), fHost(kQueries), fDev(kQueries);
	for (size_t q = 0; q < kQueries; ++q) {
		std::vector<std::pair<float, uint64_t>> all;
		for (size_t i = 0; i < rows.size(); ++i) {
			all.emplace_back(dist(queries[q], rows[i]), fid(i).AsNumber());
		}
		std::partial_sort(all.begin(), all.begin() + kK, all.end());
		for (size_t j = 0; j < kK; ++j) {
			truth[q].push_back(all[j].second);
		}
		fRef[q] = labelsOf(ref.SearchKnn(queries[q].data(), std::nullopt, kK, kEf));
		fHost[q] = labelsOf(dev.HostGraph().SearchKnn(queries[q].data(), std::nullopt, kK, kEf));
		fDev[q] = labelsOf(dev.SearchKnn(queries[q].data(), std::nullopt, kK, kEf));
	}
	const double rRef = recall(fRef, truth), rHost = recall(fHost, truth), rDev = recall(fDev, truth);
	std::printf("%s recall@10 ef %zu: reference map %.4f, host graph %.4f, device %.4f\n", name, kEf, rRef, rHost, rDev);
	report(rHost >= rRef - 0.01 && rDev >= rRef - 0.01, std::string(name) + " recall within 0.01 of HierarchicalNSW<OnInsertions>");

	MemWriter w;
	std::atomic_int32_t cancel{0};
	dev.SaveIndex(w, cancel);
	hnswlib::GpuHnsw<Sync::OnInsertions> loaded(reindexer::IsArray_False, metric, kDim, kCap, 16, 200, true);
	MemReader rd(w.tokens, rows);
	loaded.LoadIndex(rd);
	bool same = sameGraph(loaded.HostGraph(), dev.DeviceIndex());
	for (size_t q = 0; q < kQueries && same; ++q) {
		same = labelsOf(loaded.SearchKnn(queries[q].data(), std::nullopt, kK, kEf)) == fDev[q];
	}
	report(same, std::string(name) + " SaveIndex / LoadIndex round trip searches the same");

	// an existing label: the reference's path (updatePoint), nothing built on the device
	const size_t built = dev.DeviceBuiltRows();
	std::vector<float> moved(kDim, 0.25f);
	dev.AddPointConcurrent(view(moved), fid(17));
	const float* got = dev.FloatPtrByExternalLabel(fid(17).AsNumber());
	bool fallback = std::equal(moved.begin(), moved.end(), got) && dev.DeviceBuiltRows() == built && dev.CurrentElementCount() == rows.size();
	// tombstones: replace_deleted reuses the slot, nothing built on the device
	dev.MarkDelete(fid(5));
	std::vector<float> fresh(kDim, -0.5f);
	dev.AddPointConcurrent(view(fresh), fid(rows.size() + 1));
	got = dev.FloatPtrByExternalLabel(fid(rows.size() + 1).AsNumber());
	fallback = fallback && std::equal(fresh.begin(), fresh.end(), got) && dev.DeviceBuiltRows() == built &&
			   dev.CurrentElementCount() == rows.size() && !dev.SearchKnn(fresh.data(), std::nullopt, kK, kEf).empty();
	report(fallback, std::string(name) + " existing label and tombstones take the reference's path");

	// switch off: as before, the reference's inserter and an import at the first search
	hnswlib::GpuHnsw<Sync::OnInsertions> off(reindexer::IsArray_False, metric, kDim, kCap, 16, 200);
	insertConcurrent(off, rows, 0, kRound);
	(void)off.SearchKnn(queries[0].data(), std::nullopt, kK, kEf);
	report(off.DeviceImports() == 1 && off.DeviceBuiltRows() == 0 && off.CurrentElementCount() == kRound &&
			   sameGraph(off.HostGraph(), off.DeviceIndex()),
		   std::string(name) + " switch off: reference inserter, one import");
}

}  // namespace

int main() {
	if (rxgpu_device_count() < 1) {
		std::printf("no CUDA device\n");
		return 2;
	}
	run(reindexer::VectorMetric::L2, "L2");
	run(reindexer::VectorMetric::InnerProduct, "IP");
	return failures ? 1 : 0;
}
