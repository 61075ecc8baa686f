// Drop-in replacement for ft::Merger<IdCont, ft::MergeData, OffsetT>::Merge at the ft_fast seam
// Selector<IdCont>::mergeResults (cpp_src/core/ft/ft_fast/selecterimpl.h:609-627): takes exactly what the reference hands its merger --
// ft::QueryMergeData<IdCont> (querymergedata.h:13-242), FtMergeStatuses::Statuses, FTConfig, a DocsStatsGetter duck-type
// (index/indextext/indextext.h:245-258) -- converts it to the C ABI of librxgpu (include/rxgpu.h: rxgpu_ft_*) and returns ft::MergeData
// (phrasemerger.h:57-78).  One GpuFtMerger lives next to the index's DataHolder: document statistics are uploaded once per commit,
// every posting list (IdRelVec or PackedIdRelVec) once at its first use (keyed by the container's address, which is stable until the
// next commit rebuilds the holder -- the owner then calls Reset()).
// Meant to be dropped into cpp_src/core/ft/ft_fast/; it includes the reference's own headers and is compiled only where that tree is
// available (tests/cpp/dropin_ft_check.cc does so in the authoring container).  INTEGRATION.md section 6 shows the patch.
//
// Covered on the device: query parts that are plain terms with their variant subterms (AND / OR / NOT), the preselect step, all three
// BM25 variants, summationRanksByFieldsRatio, multi-word synonyms (with their suppressed subterms), phrases.  MergeAreas serves the
// highlight result type ft::MergeDataAreas<Area> (FtCtxType::kFtArea: queries with highlight() / snippet()) for the queries
// MergeableAreas accepts: no phrase, maxAreasInDoc in [1, 64], maxTotalAreasToCache < 0.  The caller keeps ft::Merger for the rest and
// for MergeDataAreas<AreaDebug> (an explicit dispatch on the result type at the seam).
#pragma once

#include <cstdlib>
#include <stdexcept>
#include <unordered_map>
#include <vector>

// clang-format off
#include "tools/float_comparison.h"
#include "core/ft/ft_fast/mergerimpl.h"
// clang-format on
#include "core/ft/idrelset.h"
#include "rxgpu.h"

namespace reindexer {
namespace ft {

template <typename IdCont>
class [[nodiscard]] GpuFtMerger {
public:
	template <typename DocsStatsGetter>
	GpuFtMerger(size_t totalNumDocs, size_t fieldSize, const DocsStatsGetter& stats) : totalDocs_(uint32_t(totalNumDocs)), nfields_(uint32_t(fieldSize)) {
		std::vector<uint32_t> words(size_t(totalDocs_) * nfields_);
		std::vector<uint8_t> removed(totalDocs_);
		std::vector<float> avg(nfields_);
		for (uint32_t d = 0; d < totalDocs_; ++d) {
			removed[d] = stats.DocRemoved(d) ? 1 : 0;
			for (uint32_t f = 0; f < nfields_; ++f) {
				words[size_t(d) * nfields_ + f] = uint32_t(stats.NumWordsInField(d, f));
			}
		}
		for (uint32_t f = 0; f < nfields_; ++f) {
			avg[f] = stats.AvgWordsCount(f);
		}
		check(rxgpu_ft_create(&h_, totalDocs_, nfields_, words.data(), avg.data(), removed.data(), deviceFromEnv()));
	}
	GpuFtMerger(const GpuFtMerger&) = delete;
	GpuFtMerger& operator=(const GpuFtMerger&) = delete;
	~GpuFtMerger() { rxgpu_ft_destroy(h_); }

	// what Merge covers: every QueryMergeData (terms, phrases, multi-word synonyms) whose result type is ft::MergeData; the area
	// result types go through MergeableAreas / MergeAreas, or stay with ft::Merger -- the caller dispatches on the result type
	static bool Mergeable(const QueryMergeData<IdCont>&) noexcept { return true; }
	// what MergeAreas covers (otherwise ft::Merger<IdCont, MergeDataAreas<Area>, OffsetT> stays in charge):
	//  - no phrase: PhraseMerger's areas (phrasemerger.h:168-206) depend on the permutation an unstable sort leaves among equal positions;
	//  - maxAreasInDoc in [1, 64]: 0 divides by zero in AreasInField::Insert, negative values make the ring unbounded;
	//  - maxTotalAreasToCache < 0: IndexText::doSelectKey (indextext.cc:691-705) admits a result to the cache by its area count BEFORE
	//    the commit, which the committed AreasInDocument objects built here cannot report.
	static bool MergeableAreas(const QueryMergeData<IdCont>& q, const FTConfig& cfg) noexcept {
		for (const auto& qp : q.queryParts) {
			if (qp.IsPhrase()) {
				return false;
			}
		}
		return cfg.maxAreasInDoc >= 1 && cfg.maxAreasInDoc <= 64 && cfg.maxTotalAreasToCache < 0;
	}

	MergeData Merge(QueryMergeData<IdCont>& q, RankSortType rankSortType, const FtMergeStatuses::Statuses& docsExcluded, const FTConfig& cfg) {
		MergeData out;
		if (q.Empty() || totalDocs_ == 0) {
			return out;  // Merger::Merge, mergerimpl.h:472-474
		}
		Converted cv;
		convert(q, docsExcluded, cfg, cv);
		std::vector<rxgpu_ft_merge_info> res(cv.maxOut);
		uint64_t n = 0;
		check(rxgpu_ft_merge_query(h_, &cv.c, &cv.query, cv.excludedPtr(), int(rankSortType), cv.maxOut, res.data(), &n));
		out.reserve(n);
		for (uint64_t i = 0; i < n && i < cv.maxOut; ++i) {
			MergeInfo mi;
			mi.id = IdType::FromNumber(res[i].id);
			mi.proc = res[i].proc;
			mi.field = res[i].field;
			mi.normalizedProc = res[i].normalized_proc;
			out.emplace_back(mi);
		}
		return out;
	}

	// Merger<IdCont, MergeDataAreas<Area>, OffsetT>::Merge for a query MergeableAreas accepts.  Every document's areas come back
	// committed; its AreasInDocument is rebuilt by inserting them in start order (they never touch and there are at most maxAreasInDoc
	// of them, so AreasInField::Insert appends each unchanged) and committing, which leaves GetAreas(f)->GetData() equal to the
	// reference's.  Nothing after the merger inserts areas again (InsertArea / AddWord are called from ft_fast/ only).
	MergeDataAreas<Area> MergeAreas(QueryMergeData<IdCont>& q, RankSortType rankSortType, const FtMergeStatuses::Statuses& docsExcluded,
									const FTConfig& cfg) {
		MergeDataAreas<Area> out;
		if (q.Empty() || totalDocs_ == 0) {
			return out;
		}
		if (!MergeableAreas(q, cfg)) {
			throw std::runtime_error("GpuFtMerger: MergeAreas called for a query MergeableAreas refuses");
		}
		Converted cv;
		convert(q, docsExcluded, cfg, cv);
		const int maxAreas = cfg.maxAreasInDoc;
		std::vector<rxgpu_ft_merge_info> res(cv.maxOut);
		std::vector<uint32_t> begin(cv.maxOut * nfields_ + 1);
		std::vector<rxgpu_ft_area> areas(cv.maxOut * nfields_ * size_t(maxAreas));
		uint64_t n = 0;
		check(rxgpu_ft_merge_query_areas(h_, &cv.c, &cv.query, cv.excludedPtr(), int(rankSortType), maxAreas, cv.maxOut, res.data(),
										 begin.data(), areas.data(), nullptr, &n));
		const uint64_t m = std::min<uint64_t>(n, cv.maxOut);
		out.reserve(m);
		out.vectorAreas.reserve(m);
		for (uint64_t i = 0; i < m; ++i) {
			MergeInfoAreas mi;
			mi.id = IdType::FromNumber(res[i].id);
			mi.proc = res[i].proc;
			mi.field = res[i].field;
			mi.normalizedProc = res[i].normalized_proc;
			mi.areaIndex = uint32_t(i);
			auto& doc = out.vectorAreas.emplace_back();
			doc.ReserveField(int(nfields_));
			for (uint32_t f = 0; f < nfields_; ++f) {
				for (uint32_t a = begin[i * nfields_ + f]; a < begin[i * nfields_ + f + 1]; ++a) {
					[[maybe_unused]] const bool ok = doc.InsertArea(Area(areas[a].start, areas[a].end, 0), f, 0.f, maxAreas);
				}
			}
			doc.Commit();
			out.emplace_back(mi);
		}
		return out;
	}

	// the holder was rebuilt (commit): cached posting ids refer to containers that no longer exist
	void Reset() { cache_.clear(); }
	size_t UploadedLists() const noexcept { return cache_.size(); }

private:
	// the C ABI view of one merge (the arrays outlive the call; filled in place, never moved)
	struct Converted {
		struct TermArrays {
			std::vector<float> boosts, procs;
			std::vector<uint8_t> needSum, suppressed;
			std::vector<uint32_t> lists, synIds;
		};
		std::vector<rxgpu_ft_field_config> fields;
		rxgpu_ft_config c{};
		std::vector<TermArrays> arrays;
		std::vector<rxgpu_ft_term> terms;
		std::vector<std::vector<rxgpu_ft_term>> synTerms;
		std::vector<rxgpu_ft_synonym> syns;
		rxgpu_ft_query query{};
		std::vector<uint8_t> excluded;
		bool anyExcluded = false;
		uint64_t maxOut = 0;
		const uint8_t* excludedPtr() const noexcept { return anyExcluded ? excluded.data() : nullptr; }
	};
	void convert(QueryMergeData<IdCont>& q, const FtMergeStatuses::Statuses& docsExcluded, const FTConfig& cfg, Converted& cv) {
		// mergerimpl.h:479 sorts the subterms AFTER the phrases were merged (Merger::init): plain and synonym terms are sorted here with
		// the same (unstable) sort on the same data and the library keeps that order; phrase terms are handed over in their own order
		for (auto& qp : q.queryParts) {
			if (qp.IsTerm()) {
				qp.SortSubterms();
			}
		}
		for (auto& syn : q.synonyms) {
			for (auto& term : syn.Terms()) {
				term.SortSubterms();
			}
		}
		cv.fields.resize(nfields_);
		for (uint32_t f = 0; f < nfields_; ++f) {
			const auto& fc = cfg.fieldsCfg[f];
			cv.fields[f] = rxgpu_ft_field_config{fc.bm25Boost, fc.bm25Weight, fc.termLenBoost, fc.termLenWeight, fc.positionBoost, fc.positionWeight};
		}
		rxgpu_ft_config& c = cv.c;
		c.merge_limit = uint32_t(cfg.mergeLimit);
		c.min_rank = int32_t(cfg.minRank);
		c.bm25_k1 = cfg.bm25Config.bm25k1;
		c.bm25_b = cfg.bm25Config.bm25b;
		switch (cfg.bm25Config.bm25Type) {
			case FTConfig::Bm25Config::Bm25Type::rx:
				c.bm25_type = 0;
				break;
			case FTConfig::Bm25Config::Bm25Type::classic:
				c.bm25_type = 1;
				break;
			case FTConfig::Bm25Config::Bm25Type::wordCount:
				c.bm25_type = 2;
				break;
		}
		c.distance_boost = cfg.distanceBoost;
		c.distance_weight = cfg.distanceWeight;
		c.full_match_boost = cfg.fullMatchBoost;
		c.nfields = nfields_;
		c.fields = cv.fields.data();
		c.summation_ranks_by_fields_ratio = cfg.summationRanksByFieldsRatio;

		// flat copies of the query parts and of the multi-word synonyms' terms
		size_t nSynTerms = 0;
		for (auto& syn : q.synonyms) {
			nSynTerms += syn.NumTerms();
		}
		size_t nQueryTerms = 0;
		for (auto& qp : q.queryParts) {
			nQueryTerms += qp.IsPhrase() ? qp.Phrase().NumTerms() : 1;
		}
		cv.arrays.resize(nQueryTerms + nSynTerms);
		size_t next = 0;
		auto convertTerm = [&](TermResults<IdCont>& tr) {
			typename Converted::TermArrays& a = cv.arrays[next++];
			const FtDslOpts& o = tr.Opts();
			a.boosts.resize(nfields_);
			a.needSum.resize(nfields_);
			for (uint32_t f = 0; f < nfields_; ++f) {
				a.boosts[f] = o.fieldsOpts[f].boost;
				a.needSum[f] = o.fieldsOpts[f].needSumRank ? 1 : 0;
			}
			bool anySuppressed = false;
			for (const SubtermResults<IdCont>& st : tr) {
				a.lists.push_back(postingsId(&st.Occurences()));
				a.procs.push_back(st.Proc());
				a.suppressed.push_back(st.Suppressed() ? 1 : 0);
				anySuppressed |= st.Suppressed();
			}
			rxgpu_ft_term t{};
			t.op = int32_t(o.op);
			t.boost = o.boost;
			t.term_len_boost = o.termLenBoost;
			t.field_boosts = a.boosts.data();
			t.nsubterms = uint32_t(a.lists.size());
			t.postings = a.lists.data();
			t.procs = a.procs.data();
			t.need_sum_rank = a.needSum.data();
			t.suppressed = anySuppressed ? a.suppressed.data() : nullptr;
			return t;
		};
		cv.terms.reserve(cv.arrays.size());
		int32_t phraseNum = 0;
		for (auto& qp : q.queryParts) {
			if (qp.IsPhrase()) {  // the phrase's terms follow one another under one phrase number, like in the DSL
				++phraseNum;
				auto& ph = qp.Phrase();
				for (size_t i = 0; i < ph.NumTerms(); ++i) {
					rxgpu_ft_term t = convertTerm(ph.Term(i));
					t.phrase_num = phraseNum;
					t.distance = int32_t(ph.Term(i).Distance());
					cv.terms.push_back(t);
				}
				continue;
			}
			typename Converted::TermArrays& a = cv.arrays[next];
			rxgpu_ft_term t = convertTerm(qp.Term());
			for (const size_t id : qp.SynonymsIds()) {
				a.synIds.push_back(uint32_t(id));
			}
			t.nsynonyms = uint32_t(a.synIds.size());
			t.synonym_ids = a.synIds.empty() ? nullptr : a.synIds.data();
			cv.terms.push_back(t);
		}
		cv.synTerms.resize(q.synonyms.size());
		cv.syns.resize(q.synonyms.size());
		for (size_t y = 0; y < q.synonyms.size(); ++y) {
			for (auto& tr : q.synonyms[y].Terms()) {
				cv.synTerms[y].push_back(convertTerm(tr));
			}
			cv.syns[y] = rxgpu_ft_synonym{uint32_t(cv.synTerms[y].size()), cv.synTerms[y].data()};
		}
		cv.query = rxgpu_ft_query{uint32_t(cv.terms.size()), cv.terms.data(), uint32_t(cv.syns.size()), cv.syns.empty() ? nullptr : cv.syns.data()};
		cv.excluded.assign(totalDocs_, 0);
		for (uint32_t d = 0; d < totalDocs_ && d < docsExcluded.size(); ++d) {
			cv.excluded[d] = docsExcluded[d] ? 1 : 0;
			cv.anyExcluded |= cv.excluded[d] != 0;
		}
		cv.maxOut = std::min<uint64_t>(cfg.mergeLimit, q.totalORVids) + 1;
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
	// one posting list -> SoA arrays (the iterator of either container decodes; positions keep the reference's order) -> HBM, once
	uint32_t postingsId(const IdCont* list) {
		if (const auto it = cache_.find(list); it != cache_.end()) {
			return it->second;
		}
		std::vector<uint32_t> docs, begin{0}, positions;
		docs.reserve(list->size());
		begin.reserve(list->size() + 1);
		for (auto&& rel : *list) {
			docs.push_back(uint32_t(rel.Id()));
			for (const PosType& p : rel.Pos()) {
				if (p.pos() >= (1u << 24) || p.field() > 255u || p.arrayIdx() != 0) {
					throw std::runtime_error("GpuFtMerger: word position / field / array index outside the device posting format");
				}
				positions.push_back(uint32_t(p.pos()) | (uint32_t(p.field()) << 24));
			}
			begin.push_back(uint32_t(positions.size()));
		}
		rxgpu_ft_postings pl{uint32_t(docs.size()), docs.data(), begin.data(), positions.data()};
		uint32_t id = 0;
		check(rxgpu_ft_add_postings(h_, &pl, &id));
		cache_.emplace(list, id);
		return id;
	}

	uint32_t totalDocs_, nfields_;
	rxgpu_ft_index* h_ = nullptr;
	std::unordered_map<const IdCont*, uint32_t> cache_;
};

}  // namespace ft
}  // namespace reindexer
