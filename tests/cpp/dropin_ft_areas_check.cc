// TEST INFRASTRUCTURE.  The highlight-area side of the ft_fast adapter: GpuFtMerger<IdCont>::MergeAreas against the reference's own
// ft::Merger<IdCont, ft::MergeDataAreas<Area>, OffsetT>::Merge on the SAME ft::QueryMergeData built from the reference's own containers
// (IdRelVec and PackedIdRelVec).  It diffs the merge entries (ids, order, uint8 ranks, field, rank bits) and, per entry and field,
// GetAreas(f)->GetData(); and it checks that MergeableAreas refuses phrases, maxAreasInDoc outside [1, 64] and maxTotalAreasToCache >= 0.
// The problems, containers and queries are dropin_ft_check.cc's (included, its main renamed).  Built by tests/cpp/areas.mk.
#define main dropin_ft_check_main
#include "dropin_ft_check.cc"
#undef main

namespace {

int g_areaRuns = 0, g_areaNonEmpty = 0, g_areasCompared = 0;

template <typename IdCont>
bool runAreasCase(const Problem& p, int maxAreas, const char* name) {
	using reindexer::Area;
	using AreasData = reindexer::ft::MergeDataAreas<Area>;
	std::vector<IdCont> conts(p.lists.size());
	for (size_t i = 0; i < p.lists.size(); ++i) {
		buildCont(p.lists[i], conts[i]);
	}
	reindexer::FtMergeStatuses::Statuses excluded(p.totalDocs, false);
	for (uint32_t d = 0; d < p.totalDocs; ++d) {
		if (p.excluded[d]) {
			excluded.set(d);
		}
	}
	reindexer::ft::GpuFtMerger<IdCont> gpu(p.totalDocs, p.nfields, p.stats);
	bool ok = true;
	for (auto rst : {reindexer::RankSortType::RankAndID, reindexer::RankSortType::IDOnly}) {
		auto qRef = buildQuery(p, conts);
		auto qGpu = buildQuery(p, conts);
		reindexer::FTConfig cfg = p.cfg;
		cfg.maxAreasInDoc = maxAreas;
		if (!reindexer::ft::GpuFtMerger<IdCont>::MergeableAreas(qGpu, cfg)) {
			std::printf("%s: a phrase-free query with maxAreasInDoc %d refused -> MISMATCH\n", name, maxAreas);
			return false;
		}
		reindexer::RdxContext ctx;
		auto excludedRef = excluded;
		const auto maxMerged = std::min<uint64_t>(cfg.mergeLimit, qRef.totalORVids);
		auto call = [&](auto& merger) {
			switch (cfg.bm25Config.bm25Type) {
				case reindexer::FTConfig::Bm25Config::Bm25Type::classic:
					return merger.template Merge<reindexer::Bm25Classic>(qRef, rst, p.stats);
				case reindexer::FTConfig::Bm25Config::Bm25Type::wordCount:
					return merger.template Merge<reindexer::TermCount>(qRef, rst, p.stats);
				default:
					return merger.template Merge<reindexer::Bm25Rx>(qRef, rst, p.stats);
			}
		};
		auto runRef = [&]() -> AreasData {
			if (maxMerged < 0xFFFF) {  // Selector::Process, selecterimpl.h:637-644
				reindexer::ft::Merger<IdCont, AreasData, uint16_t> m(p.totalDocs, &cfg, excludedRef, p.nfields, maxAreas, false, ctx);
				return call(m);
			}
			reindexer::ft::Merger<IdCont, AreasData, uint32_t> m(p.totalDocs, &cfg, excludedRef, p.nfields, maxAreas, false, ctx);
			return call(m);
		};
		AreasData ref = runRef();
		AreasData res = gpu.MergeAreas(qGpu, rst, excluded, cfg);
		bool same = ref.size() == res.size();
		for (size_t i = 0; same && i < ref.size(); ++i) {
			same = ref[i].id.ToNumber() == res[i].id.ToNumber() && ref[i].normalizedProc == res[i].normalizedProc && ref[i].field == res[i].field &&
				   ref[i].proc == res[i].proc;
			auto& ra = ref.vectorAreas[ref[i].areaIndex];
			auto& ga = res.vectorAreas[res[i].areaIndex];
			for (uint32_t f = 0; same && f < p.nfields; ++f) {
				const auto* rf = ra.GetAreas(f);
				const auto* gf = ga.GetAreas(f);
				const size_t rn = rf ? rf->GetData().size() : 0, gn = gf ? gf->GetData().size() : 0;
				same = rn == gn;
				for (size_t k = 0; same && k < rn; ++k) {
					const Area &x = rf->GetData()[k], &y = gf->GetData()[k];
					same = x.start == y.start && x.end == y.end && x.arrayIdx == y.arrayIdx;
					++g_areasCompared;
				}
			}
		}
		if (!same) {
			std::printf("%s maxAreasInDoc %d rst %d: reference %zu docs, device %zu docs -> MISMATCH\n", name, maxAreas, int(rst), ref.size(),
						res.size());
		}
		ok = ok && same;
		g_areaNonEmpty += !ref.empty();
		++g_areaRuns;
	}
	return ok;
}

// MergeableAreas: the phrase / maxAreasInDoc / maxTotalAreasToCache cases that keep ft::Merger
template <typename IdCont>
bool checkMergeable(const Problem& p) {
	std::vector<IdCont> conts(p.lists.size());
	for (size_t i = 0; i < p.lists.size(); ++i) {
		buildCont(p.lists[i], conts[i]);
	}
	const auto q = buildQuery(p, conts);
	bool hasPhrase = false;
	for (const auto& t : p.terms) {
		hasPhrase |= t.phraseNum != 0;
	}
	reindexer::FTConfig cfg = p.cfg;
	bool ok = true;
	for (int a : {-1, 0, 1, 5, 64, 65}) {
		for (int cache : {-1, 0, 1000}) {
			cfg.maxAreasInDoc = a;
			cfg.maxTotalAreasToCache = cache;
			const bool want = !hasPhrase && a >= 1 && a <= 64 && cache < 0;
			ok = ok && reindexer::ft::GpuFtMerger<IdCont>::MergeableAreas(q, cfg) == want;
		}
	}
	return ok;
}

}  // namespace

int main() {
	int bad = 0, cases = 0, mergeable = 0;
	const int areasPool[] = {1, 2, 3, 5, 64};
	for (uint32_t seed = 0; seed < 24; ++seed) {
		const uint32_t nfields = 1 + seed % 3, nterms = 1 + seed % 4;
		const Problem withPhrases = makeProblem(seed, 300 + 97 * seed, nfields, nterms, seed % 4 == 1 ? 25 : 20000, seed % 3 == 2 ? 0.5 : 0.0);
		const bool m = checkMergeable<reindexer::IdRelVec>(withPhrases) && checkMergeable<reindexer::PackedIdRelVec>(withPhrases);
		if (!m) {
			std::printf("seed %u: MergeableAreas -> MISMATCH\n", seed);
		}
		bad += !m;
		mergeable += 2;
		Problem p = withPhrases;  // the phrase's terms as plain terms
		for (auto& t : p.terms) {
			t.phraseNum = 0;
			t.distance = 0;
		}
		const int maxAreas = areasPool[seed % 5];
		const bool a = runAreasCase<reindexer::IdRelVec>(p, maxAreas, "IdRelVec");
		const bool b = runAreasCase<reindexer::PackedIdRelVec>(p, maxAreas, "PackedIdRelVec");
		bad += !a + !b;
		cases += 2;
	}
	bad += g_areaNonEmpty * 10 < g_areaRuns * 8;  // most results must be non-empty for the comparison to mean something
	std::printf("ft areas adapter: %d of %d merges non-empty, %d areas compared, %d MergeableAreas checks; ", g_areaNonEmpty, g_areaRuns,
				g_areasCompared, mergeable);
	std::printf("ft areas adapter: %d cases (IdRelVec and PackedIdRelVec, maxAreasInDoc 1..64, AND/OR/NOT, preselect cut, all bm25 variants, "
				"multi-word synonyms with suppressed subterms): %s\n",
				cases, bad ? "MISMATCH" : "MATCH MATCH MATCH MATCH");
	return bad;
}
