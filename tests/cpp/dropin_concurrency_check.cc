// TEST INFRASTRUCTURE.  The drop-in adapters (reindexer_b200/host/gpu_bruteforce.h, gpu_hnsw.h, gpu_ivf.h) under the reference's lock
// discipline: one std::shared_mutex plays the namespace lock, R reader threads take it shared and search, and between rounds one writer
// takes it exclusive and mutates (upserts, deletes, tombstones reused by inserts, an IVF add / remove burst, one resize).  So every round
// opens with all readers racing on the adapter's lazy device copy: GpuHnsw patches it in place or re-imports it, GpuIvfMap rebuilds it.
// Every reader's answer must be bit-identical to the adapter's answer computed serially at the same epoch, and that serial answer must
// match the reference map (BruteforceSearch, HierarchicalNSW, faiss::IndexIVFFlat) under the criteria of the sibling dropin_*_check.cc.
// One MATCH / MISMATCH line per adapter and metric.  Built by tests/cpp/concurrency.mk only where the reference tree exists.
#include <algorithm>
#include <barrier>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <random>
#include <shared_mutex>
#include <span>
#include <string>
#include <thread>
#include <vector>

#include "core/index/float_vector/hnswlib/bruteforce.h"
#include "core/index/float_vector/hnswlib/hnsw.h"
#include "faiss/IndexFlat.h"
#include "gpu_bruteforce.h"
#include "gpu_hnsw.h"
#include "gpu_ivf.h"

namespace {

constexpr int kReaders = 6;
constexpr size_t kDim = 32;
using Hits = std::vector<std::pair<float, uint64_t>>;
using Answers = std::vector<Hits>;  // one entry per call of a reader's schedule

// small integers (bit-equal distances, ties at the k-th place), or for HNSW continuous values: the reference's heaps pop equal distances
// in no defined order, so a graph search is compared with it only where distances are distinct
std::vector<float> vec(std::mt19937& rng, bool continuous = false) {
	std::uniform_int_distribution<int> v(-3, 3);
	std::normal_distribution<float> g(0.f, 1.f);
	std::vector<float> out(kDim);
	for (auto& x : out) {
		x = continuous ? g(rng) : float(v(rng));
	}
	return out;
}

bool bitsEqual(const Answers& a, const Answers& b) {
	if (a.size() != b.size()) {
		return false;
	}
	for (size_t i = 0; i < a.size(); ++i) {
		if (a[i].size() != b[i].size()) {
			return false;
		}
		for (size_t j = 0; j < a[i].size(); ++j) {
			if (a[i][j].second != b[i][j].second || std::memcmp(&a[i][j].first, &b[i][j].first, sizeof(float)) != 0) {
				return false;
			}
		}
	}
	return true;
}

// R readers start together, each under the shared lock, each running `calls` (one Hits per call); returns whether every reader's answers
// equal the serial answers computed afterwards at the same epoch (no writer in between), and those serial answers
bool raceRound(std::shared_mutex& ns, const std::function<Answers()>& calls, Answers& serial) {
	std::vector<Answers> got(kReaders);
	std::vector<std::string> errors(kReaders);
	std::barrier start(kReaders);
	std::vector<std::thread> th;
	for (int r = 0; r < kReaders; ++r) {
		th.emplace_back([&, r] {
			start.arrive_and_wait();
			try {
				std::shared_lock lck(ns);
				got[r] = calls();
			} catch (const std::exception& e) {
				errors[r] = e.what();
			}
		});
	}
	for (auto& t : th) {
		t.join();
	}
	{
		std::shared_lock lck(ns);
		serial = calls();
	}
	bool ok = true;
	for (int r = 0; r < kReaders; ++r) {
		if (!errors[r].empty() || !bitsEqual(got[r], serial)) {
			std::printf("  reader %d differs from the serial answer at the same epoch %s\n", r, errors[r].c_str());
			ok = false;
		}
	}
	return ok;
}

template <typename Q>
Hits drain(Q res) {
	Hits r(res.size());
	for (auto i = res.size(); !res.empty(); res.pop()) {
		r[--i] = res.top();
	}
	return r;
}

// the serial GPU answers against the reference's: the share of identical id lists, and distances within fp noise
bool closeToReference(const Answers& ref, const Answers& gpu, double minShare) {
	if (ref.size() != gpu.size()) {
		return false;
	}
	size_t same = 0, close = 0;
	for (size_t i = 0; i < ref.size(); ++i) {
		bool ids = ref[i].size() == gpu[i].size(), dists = ids;
		for (size_t j = 0; ids && j < ref[i].size(); ++j) {
			ids = ref[i][j].second == gpu[i][j].second;
		}
		for (size_t j = 0; dists && j < ref[i].size(); ++j) {
			dists = std::abs(ref[i][j].first - gpu[i][j].first) <= 1e-4f * std::abs(ref[i][j].first) + 2e-6f;
		}
		same += ids;
		close += dists;
	}
	return same >= minShare * ref.size() && close >= minShare * ref.size();
}

reindexer::FloatVectorId fid(size_t i) { return reindexer::FloatVectorId{reindexer::IdType::FromNumber(int(i)), 0}; }

// ---------------------------------------------------------------------------------------------------------------- brute force + HNSW

// drives the adapter and the reference map through the same rounds (kHnsw: GpuHnsw / HierarchicalNSW, else the brute-force maps)
template <typename Gpu, typename Ref, bool kHnsw>
bool runHnswlib(reindexer::VectorMetric metric, const char* name) {
	const size_t n0 = kHnsw ? 3000 : 6000, k = 10, ef = 64, nq = 12;
	std::mt19937 rng(metric == reindexer::VectorMetric::L2 ? 11 : 12);
	auto make = [&]<typename M>(M*) {
		if constexpr (kHnsw) {
			return std::make_unique<M>(reindexer::IsArray_False, metric, kDim, n0 + 64, 16, 200);
		} else {
			return std::make_unique<M>(metric, kDim, n0 + 64);
		}
	};
	auto gpu = make((Gpu*)nullptr);
	auto ref = make((Ref*)nullptr);
	std::vector<std::vector<float>> rows;
	auto upsert = [&](size_t id, const std::vector<float>& v) {
		gpu->AddPointNoLock(reindexer::ConstFloatVectorView{std::span<const float>{v}}, fid(id));
		ref->AddPointNoLock(reindexer::ConstFloatVectorView{std::span<const float>{v}}, fid(id));
	};
	auto remove = [&](size_t id) {
		if constexpr (kHnsw) {
			gpu->MarkDelete(fid(id));
			ref->MarkDelete(fid(id));
		} else {
			gpu->RemovePoint(fid(id).AsNumber());
			ref->RemovePoint(fid(id).AsNumber());
		}
	};
	for (size_t i = 0; i < n0; ++i) {
		rows.push_back(vec(rng, kHnsw));
		upsert(i, rows.back());
	}
	std::vector<std::vector<float>> queries;
	for (size_t q = 0; q < nq; ++q) {
		queries.push_back(vec(rng, kHnsw));
	}
	const float radius = kHnsw ? (metric == reindexer::VectorMetric::L2 ? 40.f : -9.f) : (metric == reindexer::VectorMetric::L2 ? 60.f : -12.f);
	auto callsOf = [&](auto& map) {
		return [&]() {
			Answers out;
			for (const auto& q : queries) {
				if constexpr (kHnsw) {
					out.push_back(drain(map->SearchKnn(q.data(), std::nullopt, k, ef)));
					out.push_back(drain(map->SearchRange(q.data(), std::nullopt, radius, ef)));
				} else {
					out.push_back(drain(map->SearchKnn(q.data(), std::nullopt, k)));
					out.push_back(drain(map->SearchRange(q.data(), std::nullopt, radius, 0)));
				}
			}
			return out;
		};
	};
	std::shared_mutex ns;
	bool ok = true;
	size_t next = n0;
	for (int round = 0; round < 6; ++round) {
		size_t importsBefore = 0, patchedBefore = 0;
		if constexpr (kHnsw) {
			importsBefore = gpu->DeviceImports();
			patchedBefore = gpu->DevicePatchedNodes();
		}
		if (round > 0) {  // the writer, under the exclusive lock
			std::unique_lock lck(ns);
			if (round == 4) {
				gpu->ResizeIndex(gpu->MaxElements() + 200);
				ref->ResizeIndex(ref->MaxElements() + 200);
			}
			for (size_t j = 0; j < 24; ++j) {
				if (j % 6 == 2) {
					remove(next - 3);  // a tombstone, reused by a later insert in HNSW
				} else if (j % 6 == 4) {
					rows[next - 5] = vec(rng, kHnsw);  // the same id again with another vector
					upsert(next - 5, rows[next - 5]);
				} else {
					rows.push_back(vec(rng, kHnsw));
					upsert(next++, rows.back());
				}
			}
		}
		Answers serial;
		ok = raceRound(ns, callsOf(gpu), serial) && ok;
		const Answers want = callsOf(ref)();
		if (!closeToReference(want, serial, kHnsw ? 0.9 : 1.0)) {
			std::printf("  round %d: the serial answer does not match the reference map\n", round);
			ok = false;
		}
		if constexpr (kHnsw) {
			// the first round imports once; steady-state rounds patch in place; the resize round re-imports exactly once, however many
			// readers raced into the lazy copy
			const size_t imports = gpu->DeviceImports() - importsBefore;
			const size_t patched = imports ? 0 : gpu->DevicePatchedNodes() - patchedBefore;  // an import starts a fresh device copy and count
			const bool expect = round == 0 || round == 4 ? imports == 1 : imports == 0 && patched > 0;
			std::printf("  %s round %d: %zu import(s), %zu nodes patched%s\n", name, round, imports, patched,
						expect ? "" : (" -- unexpected: " + gpu->LastPatchError()).c_str());
			ok = ok && expect;
		}
	}
	return ok;
}

// ---------------------------------------------------------------------------------------------------------------- IVF

bool runIvf(int metric) {
	const size_t nlist = 64, n0 = 20000, nq = 40, k = 10;
	std::mt19937 rng(900 + metric);
	std::normal_distribution<float> gauss(0.f, 1.f);
	auto space = [&]() -> std::unique_ptr<faiss::IndexFlat> {
		if (metric == 0) {
			return std::make_unique<faiss::IndexFlatL2>(kDim);
		}
		return std::make_unique<faiss::IndexFlatIP>(kDim);
	};
	const auto fm = metric == 0 ? faiss::METRIC_L2 : faiss::METRIC_INNER_PRODUCT;
	auto refSpace = space(), mineSpace = space();
	auto ref = std::make_unique<faiss::IndexIVFFlat>(refSpace.get(), kDim, nlist, fm);
	auto mine = std::make_unique<faiss::IndexIVFFlat>(mineSpace.get(), kDim, nlist, fm);
	ref->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
	mine->set_direct_map_type(faiss::DirectMap::Type::Hashtable);
	std::vector<float> vecs((n0 + 4000) * kDim);
	for (auto& v : vecs) {
		v = gauss(rng);
	}
	std::vector<faiss::idx_t> ids(n0 + 4000);
	for (size_t i = 0; i < ids.size(); ++i) {
		ids[i] = faiss::idx_t(i) << 32;
	}
	ref->train(faiss::idx_t(n0), vecs.data());
	std::vector<float> cent(nlist * kDim);
	ref->quantizer->reconstruct_n(0, faiss::idx_t(nlist), cent.data());
	mine->quantizer->add(faiss::idx_t(nlist), cent.data());
	mine->is_trained = true;
	ref->nprobe = mine->nprobe = 8;
	ref->add_with_ids(faiss::idx_t(n0), vecs.data(), ids.data());
	mine->add_with_ids(faiss::idx_t(n0), vecs.data(), ids.data());
	reindexer::GpuIvfMap gpu(std::move(mine));
	std::vector<float> queries(nq * kDim);
	for (auto& v : queries) {
		v = gauss(rng);
	}
	const float radius = metric == 0 ? 22.f : 6.f;
	auto callsOf = [&](auto search, auto range) {
		return [&, search, range]() {
			Answers out;
			for (size_t n : {size_t(1), nq}) {  // one query per call and a batch of 40
				for (size_t q0 = 0; q0 < nq; q0 += n) {
					std::vector<float> d(n * k);
					std::vector<faiss::idx_t> l(n * k);
					search(faiss::idx_t(n), queries.data() + q0 * kDim, faiss::idx_t(k), d.data(), l.data());
					for (size_t q = 0; q < n; ++q) {
						Hits h;
						for (size_t j = 0; j < k && l[q * k + j] >= 0; ++j) {
							h.emplace_back(d[q * k + j], uint64_t(l[q * k + j]));
						}
						out.push_back(std::move(h));
					}
					faiss::RangeSearchResult rr{faiss::idx_t(n)};
					range(faiss::idx_t(n), queries.data() + q0 * kDim, radius, &rr);
					for (size_t q = 0; q < n; ++q) {
						Hits h;
						for (size_t i = rr.lims[q]; i < rr.lims[q + 1]; ++i) {
							h.emplace_back(rr.distances[i], uint64_t(rr.labels[i]));
						}
						std::sort(h.begin(), h.end(), [](const auto& a, const auto& b) { return a.second < b.second; });
						out.push_back(std::move(h));
					}
				}
			}
			return out;
		};
	};
	auto gpuCalls = callsOf([&](faiss::idx_t n, const float* x, faiss::idx_t kk, float* d, faiss::idx_t* l) { gpu.search(n, x, kk, d, l); },
							[&](faiss::idx_t n, const float* x, float r, faiss::RangeSearchResult* rr) { gpu.range_search(n, x, r, rr); });
	auto refCalls = callsOf([&](faiss::idx_t n, const float* x, faiss::idx_t kk, float* d, faiss::idx_t* l) { ref->search(n, x, kk, d, l); },
							[&](faiss::idx_t n, const float* x, float r, faiss::RangeSearchResult* rr) { ref->range_search(n, x, r, rr); });
	std::shared_mutex ns;
	bool ok = true;
	size_t next = n0;
	for (int round = 0; round < 5; ++round) {
		if (round > 0) {  // an add_with_ids / remove_ids burst under the exclusive lock
			std::unique_lock lck(ns);
			const size_t burst = 1 + size_t(round) * 300;
			gpu.add_with_ids(faiss::idx_t(burst), vecs.data() + next * kDim, ids.data() + next);
			ref->add_with_ids(faiss::idx_t(burst), vecs.data() + next * kDim, ids.data() + next);
			next += burst;
			for (size_t j = 0; j < 50; ++j) {
				const faiss::idx_t id = ids[(rng() % next)];
				faiss::IDSelectorArray sel(1, &id);
				gpu.remove_ids(sel);
				ref->remove_ids(sel);
			}
		}
		Answers serial;
		ok = raceRound(ns, gpuCalls, serial) && ok;
		if (!closeToReference(refCalls(), serial, 0.95)) {
			std::printf("  ivf round %d: the serial answer does not match faiss::IndexIVFFlat\n", round);
			ok = false;
		}
	}
	return ok;
}

}  // namespace

int main() {
	int bad = 0;
	for (auto metric : {reindexer::VectorMetric::L2, reindexer::VectorMetric::InnerProduct}) {
		const int m = int(metric);
		bool ok = runHnswlib<hnswlib::GpuBruteforceSearch, hnswlib::BruteforceSearch, false>(metric, "bruteforce");
		std::printf("GpuBruteforceSearch metric %d: 6 rounds x %d readers -> %s\n", m, kReaders, ok ? "MATCH" : "MISMATCH");
		bad += !ok;
		ok = runHnswlib<hnswlib::GpuHnsw<hnswlib::Synchronization::None>, hnswlib::HierarchicalNSW<hnswlib::Synchronization::None>, true>(
			metric, "hnsw");
		std::printf("GpuHnsw metric %d: 6 rounds x %d readers -> %s\n", m, kReaders, ok ? "MATCH" : "MISMATCH");
		bad += !ok;
	}
	for (int metric : {0, 1}) {
		const bool ok = runIvf(metric);
		std::printf("GpuIvfMap metric %d: 5 rounds x %d readers -> %s\n", metric, kReaders, ok ? "MATCH" : "MISMATCH");
		bad += !ok;
	}
	return bad;
}
