// ORACLE / TEST INFRASTRUCTURE ONLY -- never linked into the product (librxgpu.so).
//
// extern "C" facade over the *unmodified* reference merger with highlight areas, compiled in place from /root/reference/cpp_src:
//   ft::Merger<IdCont, ft::MergeDataAreas<Area>, OffsetT>::Merge       core/ft/ft_fast/mergerimpl.h:466-566, merger.h:196-205
//   AreasInDocument / AreasInField (Insert ring, Commit)               core/ft/areaholder.h
// The problem description, the posting containers and the configuration are built by the helpers of ref_ft_facade.cc, which this
// file includes; it goes into its own library (oracle/_ref/liboracle_ref_ft_areas.so, built by oracle/areas.mk).
#include "ref_ft_facade.cc"

namespace {

template <typename IdCont>
void buildQuery(const Stats& stats, std::vector<IdCont>& lists, uint32_t nterms, const ft_term* terms, uint32_t nsyn, const ft_synonym* syns,
				reindexer::ft::QueryMergeData<IdCont>& q) {
	for (uint32_t y = 0; y < nsyn; ++y) {  // the selecter appends synonyms while it walks the terms (selecterimpl.h:440-466,580-603)
		reindexer::ft::Synonym<IdCont> syn;
		for (uint32_t t = 0; t < syns[y].nterms; ++t) {
			auto tr = makeTerm(syns[y].terms[t], stats.nfields, lists);
			q.totalORVids += tr.MaxVDocs();
			syn.AddTerm(std::move(tr));
		}
		q.synonyms.emplace_back(std::move(syn));
	}
	reindexer::ft::PhraseResults<IdCont> nextPhrase;  // grouped like the selecter does (selecterimpl.h:546-566)
	int curPhraseNum = 0;
	for (uint32_t t = 0; t < nterms; ++t) {
		auto tr = makeTerm(terms[t], stats.nfields, lists);
		q.totalORVids += tr.MaxVDocs();
		if (terms[t].phrase_num != 0) {
			if (nextPhrase.NumTerms() && curPhraseNum != terms[t].phrase_num) {
				q.queryParts.emplace_back(std::move(nextPhrase));
				nextPhrase.clear();
			}
			curPhraseNum = terms[t].phrase_num;
			nextPhrase.Add(std::move(tr));
			continue;
		}
		if (nextPhrase.NumTerms()) {
			q.queryParts.emplace_back(std::move(nextPhrase));
			nextPhrase.clear();
		}
		q.queryParts.emplace_back(std::move(tr));
		for (uint32_t y = 0; y < terms[t].nsynonyms; ++y) {
			q.queryParts.back().AddSynonymId(terms[t].synonym_ids[y]);
		}
	}
	if (nextPhrase.NumTerms()) {
		q.queryParts.emplace_back(std::move(nextPhrase));
		nextPhrase.clear();
	}
}

using AreasData = reindexer::ft::MergeDataAreas<reindexer::Area>;

template <typename IdCont, typename OffsetT>
AreasData runMergeAreas(uint32_t totalDocs, const Stats& stats, const uint8_t* excluded, std::vector<IdCont>& lists, reindexer::FTConfig& cfg,
						uint32_t nterms, const ft_term* terms, uint32_t nsyn, const ft_synonym* syns, int rankSortType, int maxAreasInDoc,
						int64_t* ns) {
	reindexer::ft::QueryMergeData<IdCont> q;
	buildQuery(stats, lists, nterms, terms, nsyn, syns, q);
	reindexer::FtMergeStatuses::Statuses docsExcluded(totalDocs, false);
	if (excluded) {
		for (uint32_t i = 0; i < totalDocs; ++i) {
			if (excluded[i]) {
				docsExcluded.set(i);
			}
		}
	}
	reindexer::RdxContext ctx;
	reindexer::ft::Merger<IdCont, AreasData, OffsetT> m(totalDocs, &cfg, docsExcluded, stats.nfields, maxAreasInDoc, false, ctx);
	const auto t0 = std::chrono::steady_clock::now();
	const auto type = cfg.bm25Config.bm25Type;
	using Bm25Type = reindexer::FTConfig::Bm25Config::Bm25Type;
	AreasData out = type == Bm25Type::classic	  ? m.template Merge<reindexer::Bm25Classic>(q, reindexer::RankSortType(rankSortType), stats)
					: type == Bm25Type::wordCount ? m.template Merge<reindexer::TermCount>(q, reindexer::RankSortType(rankSortType), stats)
												  : m.template Merge<reindexer::Bm25Rx>(q, reindexer::RankSortType(rankSortType), stats);
	*ns = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
	return out;
}

template <typename IdCont>
AreasData dispatchAreas(uint32_t totalDocs, const Stats& stats, const uint8_t* excluded, uint32_t nlists, const ft_postings* lists,
						reindexer::FTConfig& cfg, uint32_t nterms, const ft_term* terms, uint32_t nsyn, const ft_synonym* syns, int rankSortType,
						int maxAreasInDoc, int64_t* ns) {
	std::vector<IdCont> conts(nlists);
	for (uint32_t i = 0; i < nlists; ++i) {
		buildList(lists[i], conts[i]);
	}
	uint64_t totalOR = 0;
	auto count = [&](const ft_term& t) {
		for (uint32_t s = 0; s < t.nsubterms; ++s) {
			totalOR += lists[t.postings[s]].ndocs;
		}
	};
	for (uint32_t t = 0; t < nterms; ++t) {
		count(terms[t]);
	}
	for (uint32_t y = 0; y < nsyn; ++y) {
		for (uint32_t t = 0; t < syns[y].nterms; ++t) {
			count(syns[y].terms[t]);
		}
	}
	const uint64_t maxMerged = std::min<uint64_t>(cfg.mergeLimit, totalOR);  // selecterimpl.h:637-644
	if (maxMerged < 0xFFFF) {
		return runMergeAreas<IdCont, uint16_t>(totalDocs, stats, excluded, conts, cfg, nterms, terms, nsyn, syns, rankSortType, maxAreasInDoc, ns);
	}
	return runMergeAreas<IdCont, uint32_t>(totalDocs, stats, excluded, conts, cfg, nterms, terms, nsyn, syns, rankSortType, maxAreasInDoc, ns);
}

}  // namespace

extern "C" {

// ft::Merger<IdCont, MergeDataAreas<Area>, OffsetT>::Merge on one problem with FTConfig::maxAreasInDoc = max_areas_in_doc.
// For returned entry i: out[i]; out_raw_count[i] = vectorAreas[areaIndex].GetAreasCount() taken before any GetAreas (the uncommitted
// ring sizes); then, per field f, GetAreas(f)->GetData() (the commit) as (start, end) pairs at out_areas[2 * out_area_begin[i * nfields + f]]
// (min(n, max_out) * nfields + 1 offsets).  area_cap = room of out_areas in pairs.  Returns 0 on success.
int ref_ft_merge_query_areas(uint32_t total_docs, uint32_t nfields, const uint32_t* words, const float* avg, const uint8_t* removed,
							 const uint8_t* excluded, uint32_t nlists, const ft_postings* lists, const ft_config* cfg, uint32_t nterms,
							 const ft_term* terms, uint32_t nsyn, const ft_synonym* syns, int rank_sort_type, int packed, int32_t max_areas_in_doc,
							 uint64_t max_out, ft_merge_info* out, uint32_t* out_area_begin, uint32_t* out_areas, uint64_t area_cap,
							 uint32_t* out_raw_count, uint64_t* out_n, int64_t* merge_ns) {
	try {
		reindexer::FTConfig c(nfields);
		fillConfig(c, cfg);
		c.bm25Config.bm25Type = reindexer::FTConfig::Bm25Config::Bm25Type(cfg->bm25_type == 1	? 0
																		   : cfg->bm25_type == 2 ? 2
																								 : 1);
		c.maxAreasInDoc = max_areas_in_doc;
		Stats stats{words, avg, removed, nfields};
		int64_t ns = 0;
		AreasData res = packed ? dispatchAreas<reindexer::PackedIdRelVec>(total_docs, stats, excluded, nlists, lists, c, nterms, terms, nsyn,
																		  syns, rank_sort_type, max_areas_in_doc, &ns)
							   : dispatchAreas<reindexer::IdRelVec>(total_docs, stats, excluded, nlists, lists, c, nterms, terms, nsyn, syns,
																	rank_sort_type, max_areas_in_doc, &ns);
		if (merge_ns) {
			*merge_ns = ns;
		}
		*out_n = res.size();
		uint64_t at = 0;
		size_t i = 0;
		for (; i < res.size() && i < max_out; ++i) {
			out[i].id = res[i].id.ToNumber();
			out[i].proc = res[i].proc;
			out[i].field = res[i].field;
			out[i].normalized_proc = res[i].normalizedProc;
			auto& doc = res.vectorAreas.at(res[i].areaIndex);
			out_raw_count[i] = uint32_t(doc.GetAreasCount());
			for (uint32_t f = 0; f < nfields; ++f) {
				out_area_begin[i * nfields + f] = uint32_t(at);
				const auto* fa = doc.GetAreas(f);
				if (!fa) {
					continue;
				}
				for (const auto& a : fa->GetData()) {
					if (a.arrayIdx != 0 || at >= area_cap) {
						g_err = a.arrayIdx != 0 ? "an area with an array index" : "out_areas too small";
						return 1;
					}
					out_areas[2 * at] = a.start;
					out_areas[2 * at + 1] = a.end;
					++at;
				}
			}
		}
		out_area_begin[i * nfields] = uint32_t(at);
		return 0;
	} catch (const std::exception& e) {
		g_err = e.what();
		return 1;
	}
}

}  // extern "C"
