// ft_fast full-text merge on the device: BM25 / rank scoring over posting lists.
//
// Replaces ft::Merger::Merge (cpp_src/core/ft/ft_fast/mergerimpl.h:466-566) for term-only queries:
//   buildRestrictingBitmask :326-384      -> ft_mask_* kernels (bitset ops on a docs-wide bitmap in HBM)
//   preselectMostRelevantDocs :386-464    -> ft_score_pass (integer u16 scores) + ft_hist (65536-bin histogram) + ordered threshold
//   mergeTerm :107-192 / mergeSimple :194-250 -> ft_rank_pass (calcTermRank phrasemergerimpl.h:13-91 with fp64 BM25, bm25.h:13-27,
//                                            PositionsDistance :20-37) + ordered slot assignment (block scan) = addDoc order
//   addFullMatchBoost merger.h:100-109    -> ft_full_match
//   postProcessResults merger.h:111-155   -> host (<= mergeLimit entries): minRank filter with the reference's swap-removal order,
//                                            uint8 normalisation, optional sort
// Every posting list is streamed with coalesced loads (SoA: doc ids | position offsets | packed positions), one thread per
// posting, per-document state (slot, score, mask bit) gathered from HBM.  The reference's order dependences are kept exactly:
// subterms are processed in the reference's order, one pass per subterm, and new documents receive their slots in ascending
// document order through an exclusive scan -- so the merge_limit cut-off and the output order are the reference's.
// Floating point follows the reference expression by expression with explicitly rounded operations (no FMA contraction):
// BM25 in fp64, the products in fp32, idf (two logs) computed once per subterm on the host.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <numeric>
#include <vector>

#include <cub/cub.cuh>

#include "internal.h"
#include "../host/packed_postings.h"

using namespace rxgpu;

namespace {

constexpr int kFtThreads = 256;
constexpr uint32_t kNoSlot = 0xFFFFFFFFu;  // idoffsets_ entry of a document that is not in the merge yet
constexpr int kMaxFtFields = 64;  // kMaxFtCompositeFields = 63 (ft/idrelset.h:11)

struct DevList {
	uint32_t ndocs = 0;
	uint64_t npos = 0;
	uint32_t* doc_ids = nullptr;
	uint32_t* pos_begin = nullptr;
	uint32_t* positions = nullptr;
	bool owned = true;  // false: the arrays live in a slab of rxgpu_ft_add_postings_packed_batch
	uint32_t max_doc_npos = 0;  // most positions any document has in this list (sizes the phrase merger's per-document buffers)
};

struct FieldCfgF {  // FTFieldConfig members converted to float where the reference's bound(float, float, float) takes them
	float bm25_weight, bm25_boost, pos_weight, pos_boost, len_weight, len_boost;
};

struct TermParams {
	float field_boosts[kMaxFtFields];
	FieldCfgF fc[kMaxFtFields];
	float boost, term_len_boost, proc;
	double idf, k1, b;
	int bm25_type;
	uint32_t nfields;
	float dist_weight, dist_boost;
	unsigned long long need_sum_mask;  // FtDslFieldOpts::needSumRank per field (bit f)
	double sum_ratio;                  // FTConfig::summationRanksByFieldsRatio (0 = off)
};

struct MergeState {
	// per document (total_docs)
	uint32_t* mask;      // restrictingMask_
	uint32_t* tmask;     // per-term scratch mask
	uint32_t* idoff;     // idoffsets_: slot or sentinel
	uint16_t* score;     // preselect scores
	// per merged document (max_merged)
	int32_t* md_id;
	float* md_proc;
	uint8_t* md_field;
	unsigned long long* last_ptr;  // MergerDocumentData::lastTermPositions as (pointer, count) into the posting arrays
	uint32_t* last_n;
	unsigned long long* next_ptr;
	uint32_t* next_n;
	float* ext_rank;
	uint16_t* ext_cnt;
	uint16_t* ext_last_term;
	uint32_t* n_docs;  // device counter numDocs()
};

// MergeDataAreas<Area> (areaholder.h:54-162): per merged document one AreasInDocument, i.e. per field an AreasInField ring of A areas
// (A = maxAreasInDoc) and its index_, and one maxTermRank_.  Only the slots that ft_assign hands out are initialised.
constexpr int kMaxAreasInDoc = 64;
struct AreaState {
	uint2* ring;         // [max_merged][nfields][A] (start, end); arrayIdx is always 0 in this posting format
	uint32_t* idx;       // [max_merged][nfields] AreasInField::index_ (insertions); the ring holds min(index_, A) areas
	float* max_rank;     // [max_merged] AreasInDocument::maxTermRank_
	uint32_t nfields, A;
};

// ---- exactly rounded helpers -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float bound_f(float k, float weight, float boost) {  // ftconfig.h:146
	const float kbw = __fmul_rn(__fmul_rn(k, boost), weight);
	return __double2float_rn(__dadd_rn(__dsub_rn(1.0, double(weight)), double(kbw)));
}
__device__ __forceinline__ float pos2rank(unsigned pos) {  // ftconfig.h:127-144
	if (pos <= 10) {
		return __double2float_rn(__dsub_rn(1.0, __ddiv_rn(double(pos), 100.0)));
	}
	if (pos <= 100) {
		return __double2float_rn(__dsub_rn(0.9, __ddiv_rn(double(pos), 1000.0)));
	}
	if (pos <= 1000) {
		return __double2float_rn(__dsub_rn(0.8, __ddiv_rn(double(pos), 10000.0)));
	}
	if (pos <= 10000) {
		return __double2float_rn(__dsub_rn(0.7, __ddiv_rn(double(pos), 100000.0)));
	}
	if (pos <= 100000) {
		return __double2float_rn(__dsub_rn(0.6, __ddiv_rn(double(pos), 1000000.0)));
	}
	return 0.5f;
}
__device__ __forceinline__ double bm25_get(const TermParams& t, double termCountInDoc, double wordsInDoc, double avgDocLen) {  // bm25.h
	if (t.bm25_type == 2) {
		return termCountInDoc;
	}
	const double tf = t.bm25_type == 0 ? termCountInDoc : __ddiv_rn(termCountInDoc, wordsInDoc);
	const double num = __dmul_rn(__dmul_rn(t.idf, tf), __dadd_rn(t.k1, 1.0));
	const double inner = __dadd_rn(__dsub_rn(1.0, t.b), __ddiv_rn(__dmul_rn(t.b, wordsInDoc), avgDocLen));
	return __ddiv_rn(num, __dadd_rn(tf, __dmul_rn(t.k1, inner)));
}

// calcTermRank (phrasemergerimpl.h:13-91), incl. the summation of the other fields' ranks (summationRanksByFieldsRatio > 0 and fields
// with needSumRank; at most kMaxSumFields of them, checked on the host)
constexpr int kMaxSumFields = 16;
__device__ __forceinline__ float calc_term_rank(const TermParams& t, const uint32_t* words, const float* avg, uint32_t doc,
												const uint32_t* pos, uint32_t npos, uint8_t* fieldOut) {
	uint8_t best_field = 0;
	float termRank = 0.f;
	const bool summing = t.sum_ratio > 0.0 && t.need_sum_mask != 0ull;
	float ranks[kMaxSumFields];  // descending (insertion): the reference sorts them before the weighted sum
	int nranks = 0;
	bool sumWinner = false;
	for (uint32_t idx = 0; idx < npos;) {
		const uint32_t f = pos[idx] >> 24;
		const uint32_t begin = idx;
		++idx;
		while (idx < npos && (pos[idx] >> 24) == f) {
			++idx;
		}
		if (t.field_boosts[f] == 0.f) {
			continue;
		}
		const float bm25 = __double2float_rn(bm25_get(t, double(idx - begin), double(words[size_t(doc) * t.nfields + f]), double(avg[f])));
		const float normBm25 = bound_f(bm25, t.fc[f].bm25_weight, t.fc[f].bm25_boost);
		const float positionRank = bound_f(pos2rank(pos[begin] & 0xFFFFFFu), t.fc[f].pos_weight, t.fc[f].pos_boost);
		const float termLenBoost = bound_f(t.term_len_boost, t.fc[f].len_weight, t.fc[f].len_boost);
		const float tmp = __fmul_rn(__fmul_rn(__fmul_rn(t.field_boosts[f], normBm25), termLenBoost), positionRank);
		const bool needSum = summing && ((t.need_sum_mask >> f) & 1ull);
		if (tmp > termRank) {
			best_field = uint8_t(f);
			termRank = tmp;
			sumWinner = needSum;
		}
		if (needSum && nranks < kMaxSumFields) {
			int j = nranks++;
			for (; j > 0 && ranks[j - 1] < tmp; --j) {
				ranks[j] = ranks[j - 1];
			}
			ranks[j] = tmp;
		}
	}
	if (summing && termRank > 0.f) {  // :70-78
		float k = __double2float_rn(t.sum_ratio);
		for (int i = sumWinner ? 1 : 0; i < nranks; ++i) {
			termRank = __fadd_rn(termRank, __fmul_rn(k, ranks[i]));
			k = __double2float_rn(__dmul_rn(double(k), t.sum_ratio));
		}
	}
	*fieldOut = best_field;
	return __fmul_rn(__fmul_rn(t.boost, t.proc), termRank);
}

// PosType::fullField() (idrelset.h:20) narrows (arrayIdx | field << 28) to 32 bits: with no array indexes only the low four bits of the
// field survive, so fields 16 apart compare equal there.  Kept, because the ranks depend on it.
__device__ __forceinline__ bool same_full_field(uint32_t a, uint32_t b) { return (((a ^ b) >> 24) & 0xFu) == 0u; }
// PositionsDistance (mergerimpl.h:20-37): the walk advances by word position (fullPos() truncates the field away), a pair counts
// only when the fields match
__device__ __forceinline__ unsigned positions_distance(const uint32_t* a, uint32_t na, const uint32_t* b, uint32_t nb) {
	unsigned res = 0xFFFFFFFFu;
	uint32_t i = 0, j = 0;
	while (i < na && j < nb) {
		const uint32_t pa = a[i] & 0xFFFFFFu, pb = b[j] & 0xFFFFFFu;
		const bool sign = pa > pb;
		if (same_full_field(a[i], b[j])) {
			const unsigned dst = sign ? pa - pb : pb - pa;
			if (dst < res) {
				res = dst;
				if (res <= 1) {
					break;
				}
			}
		}
		if (sign) {
			j++;
		} else {
			i++;
		}
	}
	return res == 0xFFFFFFFFu ? 0 : res;
}

// ---- kernels -----------------------------------------------------------------------------------------------------------------------
__global__ void ft_mask_init(uint32_t* mask, const uint8_t* excluded, uint32_t total_docs, uint32_t words) {
	for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) {
		uint32_t bits = 0;
		for (uint32_t b = 0; b < 32; ++b) {
			const uint32_t d = w * 32 + b;
			if (d < total_docs && !(excluded && excluded[d])) {
				bits |= 1u << b;
			}
		}
		mask[w] = bits;
	}
}
__global__ void ft_fill_u32(uint32_t* p, uint32_t v, uint64_t n) {
	for (uint64_t i = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; i < n; i += uint64_t(gridDim.x) * blockDim.x) {
		p[i] = v;
	}
}
// calcTermBitmask (mergerimpl.h:252-274)
__global__ void ft_and_mark(DevList l, TermParams t, int all_positive, uint32_t* tmask) {
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < l.ndocs; i += gridDim.x * blockDim.x) {
		bool relevant = all_positive;
		for (uint32_t p = l.pos_begin[i]; !relevant && p < l.pos_begin[i + 1]; ++p) {
			relevant = t.field_boosts[l.positions[p] >> 24] != 0.f;
		}
		if (relevant) {
			const uint32_t d = l.doc_ids[i];
			atomicOr(&tmask[d >> 5], 1u << (d & 31));
		}
	}
}
__global__ void ft_mask_and(uint32_t* mask, const uint32_t* tmask, uint32_t words) {
	for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) {
		mask[w] &= tmask[w];
	}
}
// excludeTermFromBitmask (mergerimpl.h:276-287)
__global__ void ft_not_clear(DevList l, uint32_t* mask) {
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < l.ndocs; i += gridDim.x * blockDim.x) {
		const uint32_t d = l.doc_ids[i];
		atomicAnd(&mask[d >> 5], ~(1u << (d & 31)));
	}
}
// restrictingMask_.PopCount() > cfg_->mergeLimit (mergerimpl.h:486-489), decided where the count lives
__global__ void ft_decide_preselect(const unsigned long long* popc, uint32_t merge_limit, uint32_t* flag) { *flag = *popc > merge_limit ? 1u : 0u; }
__global__ void ft_popcount(const uint32_t* mask, uint32_t words, unsigned long long* out) {
	__shared__ unsigned long long s_sum;
	if (threadIdx.x == 0) {
		s_sum = 0;
	}
	__syncthreads();
	unsigned long long c = 0;
	for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) {
		c += __popc(mask[w]);
	}
	for (int off = 16; off > 0; off >>= 1) {
		c += __shfl_xor_sync(0xffffffffu, c, off);
	}
	if ((threadIdx.x & 31) == 0 && c) {
		atomicAdd(&s_sum, c);
	}
	__syncthreads();
	if (threadIdx.x == 0 && s_sum) {  // one global atomic per block: 19 000 warps on one address were most of this kernel's time
		atomicAdd(out, s_sum);
	}
}
// static_cast<uint16_t>(proc) of calcTermScores as the reference's x86-64 build executes it: cvttss2si truncates to int32, NaN and
// values outside [-2^31, 2^31) give INT32_MIN, and the low 16 bits are kept.  A negative boost thus scores up to 16383 there and a
// proc >= 65536 wraps; the device's own float -> u16 conversion saturates instead, so the conversion is written out.
__device__ __forceinline__ uint32_t proc_to_u16(float proc) {
	const int32_t i = proc >= -2147483648.f && proc < 2147483648.f ? __float2int_rz(proc) : INT32_MIN;
	return uint32_t(i) & 0xFFFFu;
}
// calcTermScores (mergerimpl.h:289-324): one pass per subterm; a document scores once per term (tmask)
__global__ void ft_score_pass(DevList l, TermParams t, int all_same, const uint32_t* mask, uint32_t* tmask, uint16_t* score, const uint32_t* enabled) {
	if (enabled && !*enabled) {  // preselect decided on the device (ft_decide_preselect): the host enqueues the whole query ahead
		return;
	}
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < l.ndocs; i += gridDim.x * blockDim.x) {
		const uint32_t d = l.doc_ids[i];
		const uint32_t bit = 1u << (d & 31);
		if (!(mask[d >> 5] & bit)) {
			continue;
		}
		float maxBoost = t.field_boosts[0];
		if (!all_same) {
			maxBoost = 0.f;
			for (uint32_t p = l.pos_begin[i]; p < l.pos_begin[i + 1]; ++p) {
				maxBoost = fmaxf(maxBoost, t.field_boosts[l.positions[p] >> 24]);
			}
		}
		if (maxBoost > 0.f) {
			if (!(atomicOr(&tmask[d >> 5], bit) & bit)) {  // docs are unique inside one list: exactly one thread scores d in this pass
				const float proc = __fmul_rn(__fmul_rn(t.proc, maxBoost), t.boost);
				uint32_t p16 = proc_to_u16(proc);
				p16 = min(p16, 65535u / 4u);
				p16 = min(p16, 65535u - uint32_t(score[d]));
				score[d] = uint16_t(score[d] + p16);
			}
		}
	}
}
// ---- preselect, per-document passes.  A thread owns one mask word = 32 consecutive documents (64 bytes of u16 scores as four
// 128-bit loads); the score array is padded to a whole number of mask words.
struct Scores32 {
	uint32_t w[16];
	__device__ __forceinline__ uint32_t at(int i) const { return (w[i >> 1] >> ((i & 1) * 16)) & 0xFFFFu; }
	__device__ __forceinline__ bool any() const {
		uint32_t o = 0;
#pragma unroll
		for (int i = 0; i < 16; ++i) {
			o |= w[i];
		}
		return o != 0;
	}
};
__device__ __forceinline__ Scores32 load_scores32(const uint16_t* score, uint32_t word) {
	const uint4* p = reinterpret_cast<const uint4*>(score + size_t(word) * 32);
	Scores32 r;
#pragma unroll
	for (int j = 0; j < 4; ++j) {
		const uint4 v = __ldg(p + j);
		r.w[j * 4 + 0] = v.x;
		r.w[j * 4 + 1] = v.y;
		r.w[j * 4 + 2] = v.z;
		r.w[j * 4 + 3] = v.w;
	}
	return r;
}
// zero scores outside the mask / of removed docs and build the 65536-bin histogram (mergerimpl.h:416-423).  Scores cluster on a
// handful of values (sums of a few subterm procs), so the histogram is privatised: a persistent grid keeps the low 8192 bins in
// shared memory and flushes them once; only scores >= 8192 go to the global bins directly.
constexpr uint32_t kFtHistSmemBins = 8192;
__global__ void __launch_bounds__(kFtThreads) ft_hist(uint16_t* score, const uint32_t* mask, const uint8_t* removed, uint32_t words,
													  unsigned long long* hist, uint32_t* max_score, const uint32_t* enabled) {
	if (enabled && !*enabled) {  // preselect decided on the device (ft_decide_preselect): the host enqueues the whole query ahead
		return;
	}
	__shared__ uint32_t s_hist[kFtHistSmemBins];
	for (uint32_t i = threadIdx.x; i < kFtHistSmemBins; i += blockDim.x) {
		s_hist[i] = 0;
	}
	__syncthreads();
	uint32_t top = 0;  // the highest score seen: ft_pick_threshold only walks the bins below it
	for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) {
		const Scores32 sc = load_scores32(score, w);
		if (!sc.any()) {
			continue;
		}
		const uint32_t m = mask[w];
#pragma unroll
		for (int i = 0; i < 32; ++i) {
			const uint32_t s = sc.at(i);
			if (s) {
				const uint32_t d = w * 32u + i;
				if (!((m >> i) & 1u) || (removed && removed[d])) {
					score[d] = 0;
				} else if (s < kFtHistSmemBins) {
					atomicAdd(&s_hist[s], 1u);
					top = max(top, s);
				} else {
					atomicAdd(&hist[s], 1ull);
					top = max(top, s);
				}
			}
		}
	}
	top = __reduce_max_sync(0xffffffffu, top);
	if ((threadIdx.x & 31) == 0 && top) {
		atomicMax(max_score, top);
	}
	__syncthreads();
	for (uint32_t i = threadIdx.x; i < kFtHistSmemBins; i += blockDim.x) {
		if (s_hist[i]) {
			atomicAdd(&hist[i], (unsigned long long)s_hist[i]);
		}
	}
}
// threshold of the counting sort (mergerimpl.h:425-446), on the device so the merge does not stop for the host:
//   A(sc) = number of docs with score > sc;  minScore = the smallest sc >= 1 with A(sc) < maxMerged (sc = 65535 always qualifies);
//   minScoreDocs = maxMerged - A(minScore).   thr[0] = minScore, thr[1] = minScoreDocs.  One block of 1024 threads, 64 bins each.
__global__ void __launch_bounds__(1024) ft_pick_threshold(const unsigned long long* hist, uint32_t max_merged, const uint32_t* max_score,
														  uint32_t* thr, const uint32_t* enabled) {
	if (enabled && !*enabled) {  // preselect decided on the device (ft_decide_preselect): the host enqueues the whole query ahead
		return;
	}
	// Scores are walked from the highest one present downwards, 1024 bins per round (thread t of a round looks at score hi - t: coalesced
	// loads, one block-wide inclusive scan per round): A(sc) = docs above the round + the scan up to t - the bin itself.  A(sc) only grows
	// as sc falls, so the qualifying scores of a round are a prefix of its threads; the walk ends in the first round that holds a
	// non-qualifying score or reaches sc = 1.  A handful of terms gives a few hundred occupied bins: one round.
	__shared__ unsigned long long s_warp[32];
	__shared__ unsigned long long s_above;
	__shared__ uint32_t s_min, s_docs, s_stop;
	const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
	const uint32_t top = min(65535u, *max_score);
	if (t == 0) {
		s_above = 0;
		s_min = 1;              // every score down to 1 qualifies unless a round says otherwise
		s_docs = max_merged;    // minScoreDocs for that case: A(1) is subtracted below
		s_stop = 0;
	}
	__syncthreads();
	for (int64_t hi = top; hi >= 1; hi -= 1024) {
		const int64_t sc = hi - int64_t(t);
		const unsigned long long cnt = sc >= 1 ? hist[sc] : 0ull;
		unsigned long long incl = cnt;
		for (int off = 1; off < 32; off <<= 1) {
			const unsigned long long y = __shfl_up_sync(0xffffffffu, incl, off);
			if (lane >= uint32_t(off)) {
				incl += y;
			}
		}
		if (lane == 31) {
			s_warp[warp] = incl;
		}
		__syncthreads();
		unsigned long long before = s_above;
		for (uint32_t x = 0; x < warp; ++x) {
			before += s_warp[x];
		}
		const unsigned long long a = before + incl - cnt;  // docs with a score above sc
		const bool ok = sc >= 1 && a < max_merged;
		const bool next_ok = sc - 1 >= 1 && a + cnt < max_merged;  // the score below me (the next thread's, or the next round's first)
		if (ok && !next_ok) {  // exactly one thread over all rounds: the smallest qualifying score
			s_min = uint32_t(sc);
			s_docs = uint32_t(max_merged - a);
			s_stop = 1;
		}
		__syncthreads();
		if (s_stop) {
			break;
		}
		if (t == 0) {
			unsigned long long sum = s_above;
			for (uint32_t x = 0; x < 32; ++x) {
				sum += s_warp[x];
			}
			s_above = sum;
		}
		__syncthreads();
	}
	if (t == 0) {
		thr[0] = s_min;
		thr[1] = s_stop ? s_docs : uint32_t(s_above < max_merged ? max_merged - s_above : 0ull);
	}
}
// ordered cut at the threshold score: keep score > min, and the first `budget` docs (ascending id) with score == min (:448-462).
// Block b owns a contiguous chunk of mask words: pass 1 counts its threshold docs, pass 2 ranks them behind the earlier blocks.
__device__ __forceinline__ uint32_t ft_chunk_words(uint32_t words) {
	const uint32_t per = (words + gridDim.x - 1) / gridDim.x;
	return (per + kFtThreads - 1) / kFtThreads * kFtThreads;
}
__device__ __forceinline__ void ft_classify(const Scores32& sc, uint32_t m, uint32_t min_score, uint32_t& eq, uint32_t& gt) {
	eq = gt = 0;
#pragma unroll
	for (int i = 0; i < 32; ++i) {
		const uint32_t s = sc.at(i);
		eq |= uint32_t(s == min_score) << i;
		gt |= uint32_t(s > min_score) << i;
	}
	eq &= m;
	gt &= m;
}
__global__ void __launch_bounds__(kFtThreads) ft_thresh_count(const uint16_t* score, const uint32_t* mask, uint32_t words, const uint32_t* thr,
															  uint32_t* block_counts, const uint32_t* enabled) {
	if (enabled && !*enabled) {  // preselect decided on the device (ft_decide_preselect): the host enqueues the whole query ahead
		return;
	}
	__shared__ uint32_t s_cnt;
	if (threadIdx.x == 0) {
		s_cnt = 0;
	}
	__syncthreads();
	const uint32_t min_score = thr[0];
	const uint32_t chunk = ft_chunk_words(words);
	const uint32_t begin = blockIdx.x * chunk, end = min(words, begin + chunk);
	uint32_t cnt = 0;
	for (uint32_t w = begin + threadIdx.x; w < end; w += blockDim.x) {
		const uint32_t m = mask[w];
		if (m) {
			uint32_t eq, gt;
			ft_classify(load_scores32(score, w), m, min_score, eq, gt);
			cnt += __popc(eq);
		}
	}
	for (int off = 16; off > 0; off >>= 1) {
		cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
	}
	if ((threadIdx.x & 31) == 0 && cnt) {
		atomicAdd(&s_cnt, cnt);
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		block_counts[blockIdx.x] = s_cnt;
	}
}
__global__ void __launch_bounds__(kFtThreads) ft_thresh_apply(const uint16_t* score, uint32_t* mask, uint32_t words, const uint32_t* thr,
															  const uint32_t* block_counts, const uint32_t* enabled) {
	if (enabled && !*enabled) {  // preselect decided on the device (ft_decide_preselect): the host enqueues the whole query ahead
		return;
	}
	__shared__ uint32_t s_warp[kFtThreads / 32];
	__shared__ uint32_t s_base;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t min_score = thr[0], budget = thr[1];
	{  // threshold docs in the chunks of all earlier blocks
		uint32_t before = 0;
		for (uint32_t b = threadIdx.x; b < blockIdx.x; b += blockDim.x) {
			before += block_counts[b];
		}
		for (int off = 16; off > 0; off >>= 1) {
			before += __shfl_xor_sync(0xffffffffu, before, off);
		}
		if (threadIdx.x == 0) {
			s_base = 0;
		}
		__syncthreads();
		if (lane == 0 && before) {
			atomicAdd(&s_base, before);
		}
		__syncthreads();
	}
	uint32_t running = s_base;
	const uint32_t chunk = ft_chunk_words(words);
	const uint32_t begin = blockIdx.x * chunk, end = min(words, begin + chunk);
	for (uint32_t w0 = begin; w0 < end; w0 += blockDim.x) {
		const uint32_t w = w0 + threadIdx.x;
		uint32_t m = 0, eq = 0, gt = 0;
		if (w < end) {
			m = mask[w];
			if (m) {
				ft_classify(load_scores32(score, w), m, min_score, eq, gt);
			}
		}
		// exclusive block scan of popc(eq)
		const uint32_t cnt = __popc(eq);
		uint32_t incl = cnt;
		for (int off = 1; off < 32; off <<= 1) {
			const uint32_t y = __shfl_up_sync(0xffffffffu, incl, off);
			if (lane >= off) {
				incl += y;
			}
		}
		if (lane == 31) {
			s_warp[warp] = incl;
		}
		__syncthreads();
		uint32_t warp_off = 0, total = 0;
#pragma unroll
		for (int x = 0; x < kFtThreads / 32; ++x) {
			const uint32_t v = s_warp[x];
			warp_off += x < warp ? v : 0;
			total += v;
		}
		__syncthreads();
		const uint32_t rank0 = running + warp_off + incl - cnt;
		uint32_t keep_eq = eq;
		const uint32_t allowed = budget > rank0 ? budget - rank0 : 0;
		while (uint32_t(__popc(keep_eq)) > allowed) {  // keep the lowest ids
			keep_eq &= ~(0x80000000u >> __clz(keep_eq));
		}
		if (w < end && m != (gt | keep_eq)) {
			mask[w] = gt | keep_eq;
		}
		running += total;
	}
}
// exclusive scan of block counts, single block (counts <= ~200k entries)
__global__ void ft_scan_blocks(uint32_t* counts, uint32_t n, uint32_t* total) {
	// one block; a thread owns kItems consecutive counts per round (a round = blockDim.x * kItems counts: 19 532 block counts of a
	// 5 M-posting list are 3 rounds of 8192 instead of 20 rounds of 1024, each with its three barriers)
	constexpr uint32_t kItems = 8;
	__shared__ uint32_t s_warp[32];
	__shared__ uint32_t s_carry;
	if (threadIdx.x == 0) {
		s_carry = 0;
	}
	__syncthreads();
	for (uint32_t base = 0; base < n; base += blockDim.x * kItems) {
		const uint32_t i0 = base + threadIdx.x * kItems;
		uint32_t v[kItems];
		uint32_t mine = 0;
#pragma unroll
		for (uint32_t x = 0; x < kItems; ++x) {
			v[x] = i0 + x < n ? counts[i0 + x] : 0;
			mine += v[x];
		}
		uint32_t x = mine;
		for (int off = 1; off < 32; off <<= 1) {
			const uint32_t y = __shfl_up_sync(0xffffffffu, x, off);
			if ((threadIdx.x & 31) >= off) {
				x += y;
			}
		}
		if ((threadIdx.x & 31) == 31) {
			s_warp[threadIdx.x >> 5] = x;
		}
		__syncthreads();
		if (threadIdx.x < 32) {
			uint32_t w = threadIdx.x < (blockDim.x >> 5) ? s_warp[threadIdx.x] : 0;
			for (int off = 1; off < 32; off <<= 1) {
				const uint32_t y = __shfl_up_sync(0xffffffffu, w, off);
				if (threadIdx.x >= off) {
					w += y;
				}
			}
			s_warp[threadIdx.x] = w;
		}
		__syncthreads();
		const uint32_t warp_off = (threadIdx.x >> 5) ? s_warp[(threadIdx.x >> 5) - 1] : 0;
		const uint32_t incl = s_carry + warp_off + x;
		uint32_t run = incl - mine;  // exclusive prefix of my first item
#pragma unroll
		for (uint32_t y = 0; y < kItems; ++y) {
			if (i0 + y < n) {
				counts[i0 + y] = run;
			}
			run += v[y];
		}
		__syncthreads();
		if (threadIdx.x == blockDim.x - 1) {
			s_carry = incl;
		}
		__syncthreads();
	}
	if (threadIdx.x == 0 && total) {
		*total = s_carry;
	}
}
__device__ __forceinline__ uint32_t block_exclusive_rank(bool flag, uint32_t* s_warp) {
	const unsigned m = __ballot_sync(0xffffffffu, flag);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	if (lane == 0) {
		s_warp[warp] = __popc(m);
	}
	__syncthreads();
	uint32_t off = 0;
	for (int w = 0; w < warp; ++w) {
		off += s_warp[w];
	}
	__syncthreads();
	return off + __popc(m & ((1u << lane) - 1u));
}
// switchToNextWord (merger.h:220-228)
__global__ void ft_switch(MergeState st) {
	const uint32_t n = *st.n_docs;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (st.next_n[i]) {
			st.last_ptr[i] = st.next_ptr[i];
			st.last_n[i] = st.next_n[i];
			st.next_n[i] = 0;
			st.ext_rank[i] = 0.f;
		}
	}
}

// Merger::addAreas (ft_fast/merger.h:196-205): AddWord(Area(pos, pos + 1, 0), field, rank) for every position of the posting in posting
// order, through AreasInField::Insert (areaholder.h:77-94); the first refused area ends the walk, later fields included.  Then
// UpdateRank(rank).  One thread per slot and pass: a document occurs once per posting list.
__device__ __forceinline__ void add_areas(const AreaState& as, uint32_t slot, const uint32_t* pos, uint32_t npos, float rank) {
	const uint32_t A = as.A;
	const float maxRank = as.max_rank[slot];
	for (uint32_t k = 0; k < npos; ++k) {
		const uint32_t f = pos[k] >> 24, p = pos[k] & 0xFFFFFFu;
		const size_t fi = size_t(slot) * as.nfields + f;
		uint2* ring = as.ring + fi * A;
		const uint32_t idx = as.idx[fi];
		if (idx > 0) {  // Area::Concat (areaholder.h:14-29) of the last written area with (p, p + 1)
			uint2 last = ring[(idx - 1) % A];
			if ((p <= last.y && p >= last.x) || (p + 1 <= last.y && p + 1 >= last.x) || (last.x > p && last.y < p + 1)) {
				last.x = min(last.x, p);
				last.y = max(last.y, p + 1);
				ring[(idx - 1) % A] = last;
				continue;
			}
		}
		if (idx >= A && !(rank > maxRank)) {
			break;  // the ring is full and the rank does not beat the document's best term
		}
		ring[idx % A] = make_uint2(p, p + 1);
		as.idx[fi] = idx + 1;
	}
	if (rank > maxRank) {
		as.max_rank[slot] = rank;
	}
}

// one subterm pass of mergeTerm / mergeSimple: rank every posting, update documents already merged in place, flag new ones.
// kAreas: also add the posting's areas to documents already merged (addDocAreas)
template <bool kAreas>
__global__ void ft_rank_pass(DevList l, TermParams t, MergeState st, const uint32_t* words, const float* avg, const uint8_t* removed,
							 int check_removed, int simple, uint32_t sentinel, uint16_t qp_idx, float* tmp_rank, uint8_t* tmp_field,
							 uint32_t* block_counts, const uint32_t* preselected, AreaState as) {
	if (preselected && *preselected) {
		check_removed = 0;  // needToCheckRemoved_ = false after preselectMostRelevantDocs (mergerimpl.h:463)
	}
	__shared__ uint32_t s_cnt;
	if (threadIdx.x == 0) {
		s_cnt = 0;
	}
	__syncthreads();
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	bool is_new = false;
	if (i < l.ndocs) {
		const uint32_t d = l.doc_ids[i];
		bool ok = (st.mask[d >> 5] >> (d & 31)) & 1u;
		if (ok && check_removed && removed && removed[d]) {
			ok = false;
		}
		if (ok) {
			const uint32_t* pos = l.positions + l.pos_begin[i];
			const uint32_t npos = l.pos_begin[i + 1] - l.pos_begin[i];
			uint8_t field;
			const float rank = calc_term_rank(t, words, avg, d, pos, npos, &field);
			if (rank != 0.f) {
				const uint32_t slot = st.idoff ? st.idoff[d] : sentinel;
				if (slot == sentinel) {
					is_new = true;
					tmp_rank[i] = rank;
					tmp_field[i] = field;
				} else if (simple) {  // mergeSimple :236-241
					if (st.md_proc[slot] < rank) {
						st.md_proc[slot] = rank;
						st.md_field[slot] = field;
					}
				} else {  // mergeTerm :167-188
					if (st.ext_last_term[slot] < qp_idx) {
						st.ext_cnt[slot]++;
						st.ext_last_term[slot] = qp_idx;
					}
					unsigned distance = positions_distance(reinterpret_cast<const uint32_t*>(st.last_ptr[slot]), st.last_n[slot], pos, npos);
					distance = max(distance, 1u);
					const float normDist = bound_f(__double2float_rn(__ddiv_rn(1.0, double(float(distance)))), t.dist_weight, t.dist_boost);
					const float finalRank = __fmul_rn(normDist, rank);
					if (finalRank > st.ext_rank[slot]) {
						float p = st.md_proc[slot];
						p = __fsub_rn(p, st.ext_rank[slot]);
						p = __fadd_rn(p, finalRank);
						st.md_proc[slot] = p;
						st.next_ptr[slot] = reinterpret_cast<unsigned long long>(pos);
						st.next_n[slot] = npos;
						st.ext_rank[slot] = finalRank;
					}
				}
				if constexpr (kAreas) {
					if (!is_new) {
						add_areas(as, slot, pos, npos, rank);
					}
				}
			}
		}
		if (!is_new) {
			tmp_rank[i] = 0.f;  // 0 marks "not a new document" for ft_assign
		}
	}
	const unsigned m = __ballot_sync(0xffffffffu, is_new);
	if ((threadIdx.x & 31) == 0 && m) {
		atomicAdd(&s_cnt, __popc(m));
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		block_counts[blockIdx.x] = s_cnt;
	}
}
// addDoc in ascending document order (merger.h:160-179): slot = numDocs() + exclusive rank; the merge_limit cut-off drops the rest.
// kAreas: the new slot's areas start empty and receive the posting's (addLastDocAreas)
template <bool kAreas>
__global__ void ft_assign(DevList l, MergeState st, int simple, uint32_t max_merged, uint16_t qp_idx, const float* tmp_rank,
						  const uint8_t* tmp_field, const uint32_t* block_offsets, AreaState as) {
	__shared__ uint32_t s_warp[kFtThreads / 32];
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	const bool is_new = i < l.ndocs && tmp_rank[i] != 0.f;
	const uint32_t slot = *st.n_docs + block_offsets[blockIdx.x] + block_exclusive_rank(is_new, s_warp);
	if (is_new && slot < max_merged) {
		const uint32_t d = l.doc_ids[i];
		st.md_id[slot] = int32_t(d);
		st.md_proc[slot] = tmp_rank[i];
		st.md_field[slot] = tmp_field[i];
		if (st.idoff) {
			st.idoff[d] = slot;
		}
		if (!simple) {
			st.last_n[slot] = 0;
			st.last_ptr[slot] = 0;
			st.next_ptr[slot] = reinterpret_cast<unsigned long long>(l.positions + l.pos_begin[i]);
			st.next_n[slot] = l.pos_begin[i + 1] - l.pos_begin[i];
			st.ext_rank[slot] = tmp_rank[i];
			st.ext_cnt[slot] = 1;
			st.ext_last_term[slot] = qp_idx;
		}
		if constexpr (kAreas) {
			for (uint32_t f = 0; f < as.nfields; ++f) {
				as.idx[size_t(slot) * as.nfields + f] = 0;
			}
			as.max_rank[slot] = 0.f;
			add_areas(as, slot, l.positions + l.pos_begin[i], l.pos_begin[i + 1] - l.pos_begin[i], tmp_rank[i]);
		}
	}
}
// AreasInDocument::Commit (areaholder.h:64-75, 124-129) of every merged document: one warp per slot, lane = field.  Sorted by start,
// each field's areas fold into the union of touching intervals (Concat of a neighbour with an equal or lower start merges exactly when
// the neighbour's end reaches this start), which no order of equal starts changes.  cnt[slot][field] = committed areas (0 past numDocs;
// cnt[max_merged * nfields] = 0 closes the scan), raw[slot] = GetAreasCount() before the commit.
__global__ void ft_areas_commit(AreaState as, const uint32_t* n_docs, uint32_t max_merged, uint32_t* cnt, uint32_t* raw) {
	const uint32_t n = *n_docs, lane = threadIdx.x & 31, A = as.A, nf = as.nfields;
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		cnt[size_t(max_merged) * nf] = 0;
	}
	for (uint32_t slot = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; slot < max_merged; slot += (gridDim.x * blockDim.x) >> 5) {
		uint32_t rawSum = 0;
		for (uint32_t f = lane; f < nf; f += 32) {
			const size_t fi = size_t(slot) * nf + f;
			if (slot >= n) {
				cnt[fi] = 0;
				continue;
			}
			uint2* ring = as.ring + fi * A;
			const uint32_t sz = min(as.idx[fi], A);
			rawSum += sz;
			for (uint32_t j = 1; j < sz; ++j) {  // insertion sort by start, <= 64 entries
				const uint2 v = ring[j];
				uint32_t k = j;
				for (; k > 0 && ring[k - 1].x > v.x; --k) {
					ring[k] = ring[k - 1];
				}
				ring[k] = v;
			}
			uint32_t out = 0;
			if (sz) {
				uint2 cur = ring[0];
				for (uint32_t j = 1; j < sz; ++j) {
					const uint2 v = ring[j];
					if (cur.y >= v.x) {
						cur.y = max(cur.y, v.y);
					} else {
						ring[out++] = cur;
						cur = v;
					}
				}
				ring[out++] = cur;
			}
			cnt[fi] = out;
		}
		for (int off = 16; off > 0; off >>= 1) {
			rawSum += __shfl_down_sync(0xffffffffu, rawSum, off);
		}
		if (lane == 0 && slot < n) {
			raw[slot] = rawSum;
		}
	}
}
// the committed areas of every (slot, field) at its offset of the slot-ordered CSR (off = exclusive scan of ft_areas_commit's cnt)
__global__ void ft_areas_emit(AreaState as, const uint32_t* n_docs, const uint32_t* cnt, const uint32_t* off, uint2* out) {
	const uint64_t total = uint64_t(*n_docs) * as.nfields;
	for (uint64_t fi = blockIdx.x * uint64_t(blockDim.x) + threadIdx.x; fi < total; fi += uint64_t(gridDim.x) * blockDim.x) {
		const uint2* ring = as.ring + fi * as.A;
		uint2* dst = out + off[fi];
		for (uint32_t j = 0; j < cnt[fi]; ++j) {
			dst[j] = ring[j];
		}
	}
}
__global__ void ft_reset_idoff(const int32_t* md_id, const uint32_t* n_docs, uint32_t* idoff) {
	const uint32_t n = *n_docs;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		idoff[md_id[i]] = kNoSlot;
	}
}
__global__ void ft_bump_count(uint32_t* n_docs, const uint32_t* total_new, uint32_t max_merged) {
	*n_docs = min(*n_docs + *total_new, max_merged);
}
__global__ void ft_mask_or(uint32_t* mask, const uint32_t* other, uint32_t words) {
	for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < words; w += gridDim.x * blockDim.x) {
		mask[w] |= other[w];
	}
}
// a suppressed subterm of a multi-word synonym (QueryMergeData::SupressDuplicatesInSynonyms, querymergedata.h:221-241): it only counts
// towards termsCounter of documents that are already merged (mergerimpl.h:144-151)
__global__ void ft_suppressed_pass(DevList l, MergeState st, const uint8_t* removed, int check_removed, uint32_t sentinel, uint16_t qp_idx,
								   const uint32_t* preselected) {
	if (preselected && *preselected) {
		check_removed = 0;
	}
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= l.ndocs) {
		return;
	}
	const uint32_t d = l.doc_ids[i];
	if (!((st.mask[d >> 5] >> (d & 31)) & 1u) || (check_removed && removed && removed[d])) {
		return;
	}
	const uint32_t slot = st.idoff[d];
	if (slot != sentinel && st.ext_last_term[slot] < qp_idx) {
		st.ext_cnt[slot]++;
		st.ext_last_term[slot] = qp_idx;
	}
}
// after the terms of one multi-word synonym: documents added since the synonyms began either hold all of its terms or start counting
// again (mergerimpl.h:517-525)
__global__ void ft_syn_mark(MergeState st, const uint32_t* before, uint16_t num_terms, uint8_t* full) {
	const uint32_t n = *st.n_docs;
	for (uint32_t i = *before + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (st.ext_cnt[i] < num_terms) {
			st.ext_cnt[i] = 0;
		} else {
			full[i] = 1;
		}
	}
}
// documents that hold only a part of a multi-word synonym leave the result (mergerimpl.h:539-560): marked with proc = -inf, which the
// post-processing drops (device) or filters in order (host)
__global__ void ft_syn_finish(MergeState st, const uint32_t* before, const uint8_t* full) {
	const uint32_t n = *st.n_docs;
	for (uint32_t i = *before + blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (!full[i]) {
			st.md_proc[i] = -INFINITY;
		}
	}
}
__global__ void ft_copy_u32(uint32_t* dst, const uint32_t* src) { *dst = *src; }

// ---- phrases: PhraseMerger (phrasemerger.h:285-399, phrasemergerimpl.h:166-312) and Merger::mergePhrase (mergerimpl.h:41-90) ------------
// Per merged document the phrase merger keeps two position sets (lastPhrasePositions / nextPhrasePositions); here they are rows of two
// [slots][cap] arrays, cap = the most positions one document can collect in one term (known from the lists).
struct PhraseState {
	uint32_t* pre;    // preselectedDocs_
	uint32_t* idoff;  // idoffsets_ (sentinel = kNoSlot)
	int32_t* id;
	float* proc;
	uint8_t* field;
	float* rank;
	uint32_t* last;
	uint32_t* last_n;
	uint32_t* next;
	uint32_t* next_n;
	uint32_t cap, max_merged;
	uint32_t* n;  // NumDocsMerged()
};
__global__ void ft_phrase_mark(DevList l, const uint8_t* removed, uint32_t* bits) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < l.ndocs) {
		const uint32_t d = l.doc_ids[i];
		if (!(removed && removed[d])) {
			atomicOr(&bits[d >> 5], 1u << (d & 31));
		}
	}
}
// first term of a phrase, one subterm pass (phrasemergerimpl.h:203-221): ranks, documents already merged updated in place, new ones flagged
__global__ void ft_phrase_first_pass(DevList l, TermParams t, PhraseState ps, const uint32_t* words, const float* avg, float* tmp_rank,
									 uint8_t* tmp_field, uint32_t* block_counts) {
	__shared__ uint32_t s_cnt;
	if (threadIdx.x == 0) {
		s_cnt = 0;
	}
	__syncthreads();
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	bool is_new = false;
	if (i < l.ndocs) {
		const uint32_t d = l.doc_ids[i];
		tmp_rank[i] = 0.f;
		if ((ps.pre[d >> 5] >> (d & 31)) & 1u) {
			const uint32_t* pos = l.positions + l.pos_begin[i];
			const uint32_t npos = l.pos_begin[i + 1] - l.pos_begin[i];
			uint8_t field;
			const float rank = calc_term_rank(t, words, avg, d, pos, npos, &field);
			if (rank != 0.f) {
				const uint32_t slot = ps.idoff[d];
				if (slot == kNoSlot) {
					is_new = true;
					tmp_rank[i] = rank;
					tmp_field[i] = field;
				} else {
					if (rank > ps.rank[slot]) {
						ps.rank[slot] = rank;
						ps.proc[slot] = rank;
					}
					uint32_t n = ps.next_n[slot];  // AddPositions: appended, sorted and deduplicated at the end of the term
					for (uint32_t k = 0; k < npos && n < ps.cap; ++k) {
						ps.next[size_t(slot) * ps.cap + n++] = pos[k];
					}
					ps.next_n[slot] = n;
				}
			}
		}
	}
	const unsigned m = __ballot_sync(0xffffffffu, is_new);
	if ((threadIdx.x & 31) == 0 && m) {
		atomicAdd(&s_cnt, __popc(m));
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		block_counts[blockIdx.x] = s_cnt;
	}
}
__global__ void ft_phrase_first_assign(DevList l, PhraseState ps, const float* tmp_rank, const uint8_t* tmp_field, const uint32_t* block_offsets) {
	__shared__ uint32_t s_warp[kFtThreads / 32];
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	const bool is_new = i < l.ndocs && tmp_rank[i] != 0.f;
	const uint32_t slot = *ps.n + block_offsets[blockIdx.x] + block_exclusive_rank(is_new, s_warp);
	if (is_new && slot < ps.max_merged) {
		const uint32_t d = l.doc_ids[i];
		ps.id[slot] = int32_t(d);
		ps.proc[slot] = tmp_rank[i];
		ps.field[slot] = tmp_field[i];
		ps.rank[slot] = tmp_rank[i];
		ps.idoff[d] = slot;
		const uint32_t* pos = l.positions + l.pos_begin[i];
		const uint32_t npos = min(l.pos_begin[i + 1] - l.pos_begin[i], ps.cap);
		for (uint32_t k = 0; k < npos; ++k) {
			ps.next[size_t(slot) * ps.cap + k] = pos[k];
		}
		ps.next_n[slot] = npos;
		ps.last_n[slot] = 0;
	}
}
// a later term of the phrase, one subterm pass (phrasemergerimpl.h:222-241): MergePositionsWithDist (phrasemerger.h:23-54) against the
// positions the previous term left, rank scaled by the smallest distance
__global__ void ft_phrase_next_pass(DevList l, TermParams t, PhraseState ps, uint32_t dist, const uint32_t* words, const float* avg) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= l.ndocs) {
		return;
	}
	const uint32_t d = l.doc_ids[i];
	if (!((ps.pre[d >> 5] >> (d & 31)) & 1u)) {
		return;
	}
	const uint32_t slot = ps.idoff[d];
	if (slot == kNoSlot) {
		return;
	}
	const uint32_t* pos = l.positions + l.pos_begin[i];
	const uint32_t npos = l.pos_begin[i + 1] - l.pos_begin[i];
	uint8_t field;
	const float rank = calc_term_rank(t, words, avg, d, pos, npos, &field);
	if (rank == 0.f) {
		return;
	}
	const uint32_t* left = ps.last + size_t(slot) * ps.cap;
	const uint32_t nl = ps.last_n[slot];
	uint32_t* out = ps.next + size_t(slot) * ps.cap;
	uint32_t no = ps.next_n[slot];
	unsigned minDist = 0x7FFFFFFFu;  // std::numeric_limits<int>::max()
	uint32_t r = 0;
	for (uint32_t a = 0; a < nl; ++a) {
		const uint32_t lp = left[a] & 0xFFFFFFu;  // fullPos(): the word position (the field is compared separately)
		while (r < npos && (pos[r] & 0xFFFFFFu) < lp) {
			++r;
		}
		if (r == npos) {
			break;
		}
		while (r < npos && same_full_field(pos[r], left[a]) && (pos[r] & 0xFFFFFFu) - lp <= dist) {
			minDist = min((pos[r] & 0xFFFFFFu) - lp, minDist);
			if (no < ps.cap) {
				out[no++] = pos[r];
			}
			++r;
		}
	}
	ps.next_n[slot] = no;
	if (no == 0) {
		return;
	}
	const int md = int(minDist);
	const float normDist = bound_f(__double2float_rn(__ddiv_rn(1.0, double(md < 1 ? 1 : md))), t.dist_weight, t.dist_boost);
	const float finalRank = __fmul_rn(normDist, rank);
	if (finalRank > ps.rank[slot]) {
		float p = ps.proc[slot];
		p = __fsub_rn(p, ps.rank[slot]);
		ps.rank[slot] = finalRank;
		ps.proc[slot] = __fadd_rn(p, finalRank);
	}
}
// end of a phrase term (phrasemergerimpl.h:245-259): documents without a continuation drop out, the others SwitchPositions (sort, unique)
__global__ void ft_phrase_end_term(PhraseState ps) {
	const uint32_t n = min(*ps.n, ps.max_merged);
	for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < n; slot += gridDim.x * blockDim.x) {
		uint32_t* nx = ps.next + size_t(slot) * ps.cap;
		const uint32_t cnt = ps.next_n[slot];
		if (cnt == 0) {
			const uint32_t d = uint32_t(ps.id[slot]);
			atomicAnd(&ps.pre[d >> 5], ~(1u << (d & 31)));
			ps.proc[slot] = 0.f;
			ps.last_n[slot] = 0;
			ps.rank[slot] = 0.f;
			continue;
		}
		for (uint32_t a = 1; a < cnt; ++a) {  // insertion sort: a handful of positions per document
			const uint32_t v = nx[a];
			uint32_t b = a;
			for (; b > 0 && nx[b - 1] > v; --b) {
				nx[b] = nx[b - 1];
			}
			nx[b] = v;
		}
		uint32_t* ls = ps.last + size_t(slot) * ps.cap;
		uint32_t m = 0;
		for (uint32_t a = 0; a < cnt; ++a) {
			if (a == 0 || nx[a] != nx[a - 1]) {
				ls[m++] = nx[a];
			}
		}
		ps.last_n[slot] = m;
		ps.next_n[slot] = 0;
		ps.rank[slot] = 0.f;
	}
}
// GetMergedDocsBitmask / ExcludeMergedDocsFromBitmask (phrasemerger.h:311-329)
__global__ void ft_phrase_bits(PhraseState ps, uint32_t* bits, int set) {
	const uint32_t n = min(*ps.n, ps.max_merged);
	for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < n; slot += gridDim.x * blockDim.x) {
		if (ps.proc[slot] > 0.f) {
			const uint32_t d = uint32_t(ps.id[slot]);
			if (set) {
				atomicOr(&bits[d >> 5], 1u << (d & 31));
			} else {
				atomicAnd(&bits[d >> 5], ~(1u << (d & 31)));
			}
		}
	}
}
// GetMergedDocsScore (phrasemerger.h:331-338)
__global__ void ft_phrase_score(PhraseState ps, uint16_t* score, uint32_t phrase_proc, const uint32_t* enabled) {
	if (enabled && !*enabled) {  // preselect decided on the device (ft_decide_preselect): the host enqueues the whole query ahead
		return;
	}
	const uint32_t n = min(*ps.n, ps.max_merged);
	for (uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x; slot < n; slot += gridDim.x * blockDim.x) {
		if (ps.proc[slot] > 0.f) {
			const uint32_t d = uint32_t(ps.id[slot]);
			const uint32_t cur = score[d];
			score[d] = uint16_t(cur + min(phrase_proc, 65535u - cur));
		}
	}
}
// Merger::mergePhrase (mergerimpl.h:41-90): the phrase's documents enter the merge in the phrase merger's order
__global__ void ft_phrase_merge_pass(PhraseState ps, MergeState st, uint16_t qp_idx, uint8_t* flags, uint32_t* block_counts) {
	__shared__ uint32_t s_cnt;
	if (threadIdx.x == 0) {
		s_cnt = 0;
	}
	__syncthreads();
	const uint32_t n = min(*ps.n, ps.max_merged);
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	bool is_new = false;
	if (i < n) {
		const float proc = ps.proc[i];
		const uint32_t d = uint32_t(ps.id[i]);
		if (proc != 0.f && ((st.mask[d >> 5] >> (d & 31)) & 1u)) {
			const uint32_t slot = st.idoff[d];
			if (slot == kNoSlot) {
				is_new = true;
			} else {
				if (st.ext_last_term[slot] < qp_idx) {
					st.ext_cnt[slot]++;
					st.ext_last_term[slot] = qp_idx;
				}
				st.md_proc[slot] = __fadd_rn(st.md_proc[slot], proc);
				st.last_ptr[slot] = reinterpret_cast<unsigned long long>(ps.last + size_t(i) * ps.cap);
				st.last_n[slot] = ps.last_n[i];
				st.ext_rank[slot] = 0.f;
			}
		}
	}
	if (i < ps.max_merged) {
		flags[i] = is_new ? 1 : 0;
	}
	const unsigned m = __ballot_sync(0xffffffffu, is_new);
	if ((threadIdx.x & 31) == 0 && m) {
		atomicAdd(&s_cnt, __popc(m));
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		block_counts[blockIdx.x] = s_cnt;
	}
}
__global__ void ft_phrase_merge_assign(PhraseState ps, MergeState st, uint32_t max_merged, uint16_t qp_idx, const uint8_t* flags,
									   const uint32_t* block_offsets) {
	__shared__ uint32_t s_warp[kFtThreads / 32];
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	const bool is_new = i < ps.max_merged && flags[i];
	const uint32_t slot = *st.n_docs + block_offsets[blockIdx.x] + block_exclusive_rank(is_new, s_warp);
	if (is_new && slot < max_merged) {
		const uint32_t d = uint32_t(ps.id[i]);
		st.md_id[slot] = int32_t(d);
		st.md_proc[slot] = ps.proc[i];
		st.md_field[slot] = ps.field[i];
		st.idoff[d] = slot;
		st.last_ptr[slot] = reinterpret_cast<unsigned long long>(ps.last + size_t(i) * ps.cap);
		st.last_n[slot] = ps.last_n[i];
		st.next_ptr[slot] = 0;
		st.next_n[slot] = 0;
		st.ext_rank[slot] = 0.f;  // MergerDocumentData(phraseDocMergeDataExt.rank): the phrase merger left 0 there
		st.ext_cnt[slot] = 1;
		st.ext_last_term[slot] = qp_idx;
	}
}
// addFullMatchBoost (merger.h:100-109) with canBeBoostedByFullMatch (mergerimpl.h:533-537)
__global__ void ft_full_match(MergeState st, const uint32_t* words, uint32_t nfields, uint32_t num_terms, uint32_t need_cnt, int simple,
							  double boost) {
	const uint32_t n = *st.n_docs;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const bool can = simple || st.ext_cnt[i] == need_cnt;
		if (can && words[size_t(st.md_id[i]) * nfields + st.md_field[i]] == num_terms) {
			st.md_proc[i] = __double2float_rn(__dmul_rn(double(st.md_proc[i]), boost));
		}
	}
}


// ---- device-side postProcessResults + IndexText::afterSelect / sortAfterSelect (merger.h:111-155, indextext.cc:480-611) ----------------
// d_post: [0] scale (float bits) [1] rows total (u32)
__global__ void ft_post_scale(const float* proc, const uint32_t* n_docs, uint32_t* d_post) {
	__shared__ float s_max[32];
	const uint32_t n = *n_docs;
	float m = 0.f;
	for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
		m = fmaxf(m, proc[i]);
	}
	for (int off = 16; off > 0; off >>= 1) {
		m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
	}
	if ((threadIdx.x & 31) == 0) {
		s_max[threadIdx.x >> 5] = m;
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		for (uint32_t w = 0; w < blockDim.x / 32; ++w) {
			m = fmaxf(m, s_max[w]);
		}
		// scalingFactor = maxProc > 255 ? 255.0 / maxProc : 1.0 (a float: the double quotient is narrowed at the assignment)
		const float scale = m > 255.f ? __double2float_rn(__ddiv_rn(255.0, double(m))) : 1.0f;
		d_post[0] = __float_as_uint(scale);
		d_post[2] = __float_as_uint(m);  // >= 0: its bits order like the value (the shards' maxima are combined with an integer max)
	}
}
// docid-range shards: the scaling factor again, from the maximum over ALL shards (d_post[2] after the all-reduce)
__global__ void ft_post_rescale(uint32_t* d_post) {
	const float m = __uint_as_float(d_post[2]);
	d_post[0] = __float_as_uint(m > 255.f ? __double2float_rn(__ddiv_rn(255.0, double(m))) : 1.0f);
}
// docid-range shards, ordered cut of the preselect: this shard's threshold documents rank behind those of the lower shards
__global__ void ft_sum_u32(const uint32_t* v, uint32_t n, uint32_t* out) {
	__shared__ uint32_t s_sum;
	if (threadIdx.x == 0) {
		s_sum = 0;
	}
	__syncthreads();
	uint32_t c = 0;
	for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
		c += v[i];
	}
	for (int off = 16; off > 0; off >>= 1) {
		c += __shfl_xor_sync(0xffffffffu, c, off);
	}
	if ((threadIdx.x & 31) == 0 && c) {
		atomicAdd(&s_sum, c);
	}
	__syncthreads();
	if (threadIdx.x == 0) {
		*out = s_sum;
	}
}
__global__ void ft_shard_budget(uint32_t* thr, const uint32_t* counts, uint32_t rank) {
	unsigned long long before = 0;
	for (uint32_t r = 0; r < rank; ++r) {
		before += counts[r];
	}
	thr[1] = thr[1] > before ? uint32_t(thr[1] - before) : 0u;
}
// rows a merged document contributes: 0 when its rank is below minRank, else its row ids that pass the external statuses
__global__ void ft_post_count(const int32_t* md_id, const float* proc, const uint32_t* n_docs, float min_proc, const uint32_t* row_begin,
							  const int32_t* row_ids, const uint8_t* row_status, uint32_t cap, uint32_t* cnt) {
	const uint32_t n = *n_docs;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += gridDim.x * blockDim.x) {
		uint32_t c = 0;
		if (i < n && !(proc[i] < min_proc)) {
			const uint32_t d = uint32_t(md_id[i]);
			if (!row_begin) {
				c = (!row_status || row_status[d]) ? 1u : 0u;
			} else {
				for (uint32_t r = row_begin[d]; r < row_begin[d + 1]; ++r) {
					c += (!row_status || row_status[row_ids[r]]) ? 1u : 0u;
				}
			}
		}
		cnt[i] = c;
	}
}
// key per row: RankAndID -> (255 - rank) << 32 | rowId   (rank descending, row id ascending, indextext.cc:487-498)
//              IDOnly    -> rowId << 8 | rank           (row id ascending)
__global__ void ft_post_emit(const int32_t* md_id, const float* proc, const uint32_t* n_docs, const uint32_t* d_post, const uint32_t* row_begin,
							 const int32_t* row_ids, const uint8_t* row_status, const uint32_t* cnt, const uint32_t* off, int rank_and_id,
							 unsigned long long* keys, uint32_t* rows_total, uint32_t row_base) {
	const uint32_t n = *n_docs;
	const float scale = __uint_as_float(d_post[0]);
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (i + 1 == n) {
			*rows_total = off[i] + cnt[i];
		}
		if (cnt[i] == 0) {
			continue;
		}
		const uint32_t rank = uint32_t(uint8_t(__fmul_rn(proc[i], scale)));  // normalizedProc = static_cast<uint8_t>(proc * scalingFactor)
		const uint32_t d = uint32_t(md_id[i]);
		uint32_t o = off[i];
		if (!row_begin) {  // vdoc i is row i (+ the first document of this docid-range shard)
			const unsigned long long row = (unsigned long long)d + row_base;
			keys[o] = rank_and_id ? ((unsigned long long)(255u - rank) << 32) | row : (row << 8) | rank;
		} else {
			for (uint32_t r = row_begin[d]; r < row_begin[d + 1]; ++r) {
				const uint32_t row = uint32_t(row_ids[r]);
				if (!row_status || row_status[row]) {
					keys[o++] = rank_and_id ? ((unsigned long long)(255u - rank) << 32) | row : ((unsigned long long)row << 8) | rank;
				}
			}
		}
	}
}

// ---- device decoder of the reference's packed posting lists (PackedIdRelVec; IdRelType::unpackWithoutArrayIdxs, idrelset.cc:185-235,
// state chain idrelset.h:172-211, varints tools/varint.h:122-175).  The stream has no skip pointers, so one thread walks one list; a
// commit uploads thousands of lists, which is where the parallelism comes from.  Pass 1 validates and counts, pass 2 writes the SoA.
struct PackedCursor {
	const uint8_t* p;
	const uint8_t* end;
	bool ok;
	__device__ uint32_t get() {
		uint32_t v = 0;
		for (unsigned shift = 0; shift < 35; shift += 7) {
			if (p == end) {
				ok = false;
				return 0;
			}
			const uint8_t b = *p++;
			v |= uint32_t(b & 0x7f) << shift;
			if (!(b & 0x80)) {
				return v;
			}
		}
		ok = false;
		return 0;
	}
};
// status: 0 ok, 1 malformed / count mismatch, 2 field or position outside the SoA range, 3 document ids not ascending below total_docs
template <bool kWrite>
__global__ void ft_packed_decode(const uint8_t* bytes, const unsigned long long* byte_off, const uint32_t* counts, uint32_t nlists,
								 uint32_t total_docs, uint32_t nfields, unsigned long long* npos_out, uint32_t* status, uint32_t* max_doc_npos,
								 const unsigned long long* doc_off, const unsigned long long* pos_off, uint32_t* doc_ids, uint32_t* pos_begin,
								 uint32_t* positions) {
	const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
	if (l >= nlists) {
		return;
	}
	PackedCursor c{bytes + byte_off[l], bytes + byte_off[l + 1], true};
	uint32_t lastId = 0, lastField = 0, ndocs = 0, st = 0, maxDoc = 0;
	unsigned long long npos = 0;
	uint32_t* d_docs = kWrite ? doc_ids + doc_off[l] : nullptr;
	uint32_t* d_begin = kWrite ? pos_begin + doc_off[l] + l : nullptr;  // every list owns count + 1 offsets
	uint32_t* d_pos = kWrite ? positions + pos_off[l] : nullptr;
	if (kWrite) {
		d_begin[0] = 0;
	}
	while (c.p != c.end && st == 0) {
		uint32_t id = c.get();
		const uint32_t head = c.get();
		if (head & 1) {
			id += lastId;
		}
		uint32_t field = lastField;
		if (!(head & 2)) {
			field = c.get();
		}
		uint32_t size = 1;
		if (!(head & 4)) {
			size = c.get() + 1;
		}
		if (!c.ok) {
			st = 1;
			break;
		}
		uint32_t pf = field, ps = head >> 3;
		for (uint32_t i = 0; i < size; ++i) {
			if (i) {
				uint32_t next = c.get();
				const bool same = next & 1;
				next >>= 1;
				if (same) {
					next += ps;
				} else {
					pf = c.get() + pf;
				}
				ps = next;
				if (!c.ok) {
					st = 1;
					break;
				}
			}
			if (pf >= nfields || pf > 0xFFu || ps > 0xFFFFFFu) {
				st = 2;
				break;
			}
			if (kWrite) {
				d_pos[npos] = ps | (pf << 24);
			}
			++npos;
		}
		if (st) {
			break;
		}
		if (id >= total_docs || (ndocs && id <= lastId) || ndocs >= counts[l]) {
			st = ndocs >= counts[l] ? 1 : 3;
			break;
		}
		if (kWrite) {
			d_docs[ndocs] = id;
			d_begin[ndocs + 1] = uint32_t(npos);
		}
		maxDoc = max(maxDoc, size);
		++ndocs;
		lastId = id;
		lastField = field;
	}
	if (st == 0 && ndocs != counts[l]) {
		st = 1;
	}
	if (!kWrite) {
		npos_out[l] = npos;
		status[l] = st;
		max_doc_npos[l] = maxDoc;
	}
}

unsigned gridFor(uint64_t n, int sm) { return unsigned(std::min<uint64_t>((n + kFtThreads - 1) / kFtThreads, uint64_t(sm) * 16)); }

thread_local rxgpu_ft_stats g_ft_stats{};

}  // namespace

struct rxgpu_ft_index {
	int device = 0;
	int sm_count = 132;
	uint32_t total_docs = 0, nfields = 0;
	DevBuf<uint32_t> words;
	DevBuf<float> avg;
	DevBuf<uint8_t> removed;
	bool has_removed = false;
	std::vector<DevList> lists;
	std::vector<void*> slabs;  // batch uploads: one allocation per array kind and batch
	uint32_t max_list = 0;
	cudaStream_t stream = nullptr;
	std::mutex mtx;  // one merge at a time per index (the per-document scratch below is shared)
	// scratch
	DevBuf<uint32_t> mask, tmask, idoff, block_counts, scalar_u32;
	DevBuf<uint32_t> syn_masks, tmask2;  // multi-word synonyms: one document mask per synonym + a per-term scratch
	DevBuf<uint8_t> syn_full;            // MergerDocumentData::containsFullMultiWordSynonym per merged document
	struct PhraseBufs {                  // one PhraseMerger (phrasemerger.h:285-399)
		DevBuf<uint32_t> pre, last, last_n, next, next_n, n;
		DevBuf<int32_t> id;
		DevBuf<float> proc, rank;
		DevBuf<uint8_t> field, flags;
		uint32_t cap = 0, max_merged = 0, phrase_proc = 0, num_merged = 0;
	};
	std::vector<std::unique_ptr<PhraseBufs>> phrases;
	DevBuf<uint32_t> p_idoff, p_term_mask;  // the phrase mergers' idoffsets_ (shared, cleaned after each) and nextTermDocs_
	bool p_idoff_clean = false;
	bool idoff_clean = false;  // idoff holds kNoSlot everywhere
	PinBuf<int32_t> h_id;  // results of the last merge (pinned: one asynchronous copy per array, one synchronisation per query)
	PinBuf<float> h_proc;
	PinBuf<uint8_t> h_field;
	PinBuf<uint32_t> h_n;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	DevBuf<uint16_t> score;
	DevBuf<unsigned long long> hist, popc;
	DevBuf<unsigned long long> shard_counts, shard_keys;  // docid-range shards: exchanged counts, gathered result keys
	DevBuf<uint32_t> shard_u32;
	DevBuf<uint8_t> excluded, tmp_field, md_field;
	DevBuf<float> tmp_rank, md_proc, ext_rank;
	DevBuf<int32_t> md_id;
	DevBuf<unsigned long long> last_ptr, next_ptr;
	DevBuf<uint32_t> last_n, next_n;
	DevBuf<uint16_t> ext_cnt, ext_last_term;
	// vdoc -> row ids (IndexText::vdocs_[vdoc].RowIds(), rxgpu_ft_set_rows) and the scratch of rxgpu_ft_select
	DevBuf<uint32_t> row_begin;
	DevBuf<int32_t> row_ids;
	bool has_rows = false;
	uint64_t max_row = 0, max_rows_per_doc = 1;
	DevBuf<uint8_t> row_status, sort_tmp;
	DevBuf<uint32_t> post_cnt, post_off, post_scalars;
	DevBuf<unsigned long long> post_keys, post_keys_sorted;
	PinBuf<unsigned long long> h_keys;
	PinBuf<uint32_t> h_post;
	// rxgpu_ft_merge_query_areas: the AreaState of every slot, the committed counts and their scan, the slot-ordered CSR of areas
	DevBuf<uint2> area_ring, area_out;
	DevBuf<uint32_t> area_idx, area_cnt, area_off, area_raw;
	DevBuf<float> area_max;
	PinBuf<uint32_t> h_area_off, h_area_raw;
	PinBuf<uint2> h_areas;
	~rxgpu_ft_index() {
		cudaSetDevice(device);
		for (auto& l : lists) {
			if (l.owned) {
				cudaFree(l.doc_ids);
				cudaFree(l.pos_begin);
				cudaFree(l.positions);
			}
		}
		for (void* p : slabs) {
			cudaFree(p);
		}
		if (ev0) {
			cudaEventDestroy(ev0);
			cudaEventDestroy(ev1);
		}
		if (stream) {
			cudaStreamDestroy(stream);
		}
	}
};

extern "C" {

int rxgpu_ft_create(rxgpu_ft_index** out, uint32_t total_docs, uint32_t nfields, const uint32_t* words_in_field, const float* avg_words,
					const uint8_t* removed, int device) {
	if (!out || !words_in_field || !avg_words) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	*out = nullptr;
	if (nfields == 0 || nfields > uint32_t(kMaxFtFields)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: full-text index needs 1..64 fields");
	}
	if (rxgpu_device_count() <= device || device < 0) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: no usable CUDA device (this library has no CPU fallback)");
	}
	RX_CUDA(cudaSetDevice(device));
	auto ft = std::make_unique<rxgpu_ft_index>();
	ft->device = device;
	ft->total_docs = total_docs;
	ft->nfields = nfields;
	cudaDeviceProp prop{};
	RX_CUDA(cudaGetDeviceProperties(&prop, device));
	ft->sm_count = prop.multiProcessorCount;
	RX_CUDA(cudaStreamCreateWithFlags(&ft->stream, cudaStreamNonBlocking));
	const size_t nw = std::max<size_t>(1, size_t(total_docs) * nfields);
	RX_CUDA(ft->words.ensure(nw));
	RX_CUDA(ft->avg.ensure(nfields));
	RX_CUDA(cudaMemcpy(ft->words.p, words_in_field, size_t(total_docs) * nfields * 4, cudaMemcpyHostToDevice));
	RX_CUDA(cudaMemcpy(ft->avg.p, avg_words, nfields * 4, cudaMemcpyHostToDevice));
	if (removed) {
		RX_CUDA(ft->removed.ensure(std::max<size_t>(1, total_docs)));
		RX_CUDA(cudaMemcpy(ft->removed.p, removed, total_docs, cudaMemcpyHostToDevice));
		ft->has_removed = true;
	}
	*out = ft.release();
	return 0;
}

void rxgpu_ft_destroy(rxgpu_ft_index* ft) { delete ft; }

int rxgpu_ft_add_postings(rxgpu_ft_index* ft, const rxgpu_ft_postings* list, uint32_t* out_id) {
	if (!ft || !list || !out_id) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	RX_CUDA(cudaSetDevice(ft->device));
	if (list->ndocs && (!list->doc_ids || !list->pos_begin)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	DevList l;
	l.ndocs = list->ndocs;
	l.npos = list->ndocs ? list->pos_begin[list->ndocs] : 0;
	// the kernels index positions[] with these offsets: they must start at 0 and never decrease
	if (list->ndocs && list->pos_begin[0] != 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: posting list: pos_begin must start at 0");
	}
	for (uint32_t i = 0; i < list->ndocs; ++i) {
		if (list->pos_begin[i + 1] < list->pos_begin[i]) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: posting list: pos_begin must be non-decreasing");
		}
		l.max_doc_npos = std::max(l.max_doc_npos, list->pos_begin[i + 1] - list->pos_begin[i]);
	}
	if (l.npos && !list->positions) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	for (uint32_t i = 0; i < list->ndocs; ++i) {
		if (list->doc_ids[i] >= ft->total_docs || (i && list->doc_ids[i] <= list->doc_ids[i - 1])) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: posting list must hold ascending document ids below total_docs");
		}
	}
	for (uint64_t p = 0; p < l.npos; ++p) {
		if ((list->positions[p] >> 24) >= ft->nfields) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: posting position refers to a field outside the index");
		}
	}
	RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&l.doc_ids), std::max<size_t>(1, l.ndocs) * 4));
	RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&l.pos_begin), (size_t(l.ndocs) + 1) * 4));
	RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&l.positions), std::max<uint64_t>(1, l.npos) * 4));
	if (l.ndocs) {
		RX_CUDA(cudaMemcpy(l.doc_ids, list->doc_ids, size_t(l.ndocs) * 4, cudaMemcpyHostToDevice));
		RX_CUDA(cudaMemcpy(l.pos_begin, list->pos_begin, (size_t(l.ndocs) + 1) * 4, cudaMemcpyHostToDevice));
		RX_CUDA(cudaMemcpy(l.positions, list->positions, l.npos * 4, cudaMemcpyHostToDevice));
	} else {
		const uint32_t zero = 0;
		RX_CUDA(cudaMemcpy(l.pos_begin, &zero, 4, cudaMemcpyHostToDevice));
	}
	ft->lists.push_back(l);
	ft->max_list = std::max(ft->max_list, l.ndocs);
	*out_id = uint32_t(ft->lists.size() - 1);
	return 0;
}

int rxgpu_ft_decode_packed(const uint8_t* data, uint64_t len, uint32_t count, uint32_t* doc_ids, uint32_t* pos_begin, uint32_t* positions,
						   uint64_t max_positions, uint64_t* npos) {
	if ((len && !data) || !npos) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		DecodedPostings d;
		const int rc = decodePackedPostings(data, len, count, d);
		if (rc == -2) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: packed posting list holds a field > 255 or a word position >= 2^24");
		}
		if (rc) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: malformed packed posting list (or it contains array indexes / a different record count)");
		}
		*npos = d.positions.size();
		if (doc_ids) {
			std::copy(d.doc_ids.begin(), d.doc_ids.end(), doc_ids);
		}
		if (pos_begin) {
			std::copy(d.pos_begin.begin(), d.pos_begin.end(), pos_begin);
		}
		if (positions) {
			std::copy(d.positions.begin(), d.positions.begin() + std::min<uint64_t>(max_positions, d.positions.size()), positions);
		}
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_ft_add_postings_packed(rxgpu_ft_index* ft, const uint8_t* data, uint64_t len, uint32_t count, uint32_t* out_id) {
	if (!ft || !out_id || (len && !data)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	try {
		DecodedPostings d;
		const int rc = decodePackedPostings(data, len, count, d);
		if (rc == -2) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: packed posting list holds a field > 255 or a word position >= 2^24");
		}
		if (rc) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: malformed packed posting list (or it contains array indexes / a different record count)");
		}
		rxgpu_ft_postings l{};
		l.ndocs = uint32_t(d.doc_ids.size());
		l.doc_ids = d.doc_ids.data();
		l.pos_begin = d.pos_begin.data();
		l.positions = d.positions.data();
		return rxgpu_ft_add_postings(ft, &l, out_id);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_ft_add_postings_packed_batch(rxgpu_ft_index* ft, uint32_t nlists, const uint8_t* const* data, const uint64_t* lens,
									   const uint32_t* counts, uint32_t* out_ids) {
	if (!ft || (nlists && (!data || !lens || !counts || !out_ids))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (nlists == 0) {
		return 0;
	}
	RX_CUDA(cudaSetDevice(ft->device));
	// One thread decodes one list; a list longer than this would hold the whole batch back, so it takes the host decoder instead
	// (an explicit split by size, both sides produce the same arrays)
	constexpr uint64_t kDeviceDecodeMaxBytes = 256u << 10;
	try {
		std::vector<uint32_t> dev;  // indexes of the lists decoded on the device
		uint64_t bytes = 0;
		for (uint32_t i = 0; i < nlists; ++i) {
			if (lens[i] && !data[i]) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
			}
			if (lens[i] <= kDeviceDecodeMaxBytes) {
				dev.push_back(i);
				bytes += lens[i];
			}
		}
		const size_t firstId = ft->lists.size();
		std::vector<DevList> fresh;
		std::vector<void*> slabs;
		auto dropSlabs = [&] {
			for (void* p : slabs) {
				cudaFree(p);
			}
		};
		const uint32_t nd = uint32_t(dev.size());
		std::vector<DevList> devLists(nd);
		if (nd) {
			std::vector<uint8_t> blob(std::max<uint64_t>(bytes, 1));
			std::vector<unsigned long long> byteOff(size_t(nd) + 1, 0), docOff(size_t(nd) + 1, 0), posOff(size_t(nd) + 1, 0), npos(nd);
			std::vector<uint32_t> cnt(nd), status(nd);
			for (uint32_t j = 0; j < nd; ++j) {
				const uint32_t i = dev[j];
				if (lens[i]) {
					std::memcpy(blob.data() + byteOff[j], data[i], lens[i]);
				}
				byteOff[j + 1] = byteOff[j] + lens[i];
				cnt[j] = counts[i];
				docOff[j + 1] = docOff[j] + counts[i];
			}
			DevBuf<uint8_t> dBlob;
			DevBuf<unsigned long long> dByteOff, dNpos, dDocOff, dPosOff;
			DevBuf<uint32_t> dCnt, dStatus;
			RX_CUDA(dBlob.ensure(blob.size()));
			RX_CUDA(dByteOff.ensure(byteOff.size()));
			RX_CUDA(dNpos.ensure(nd));
			RX_CUDA(dDocOff.ensure(docOff.size()));
			RX_CUDA(dPosOff.ensure(posOff.size()));
			RX_CUDA(dCnt.ensure(nd));
			RX_CUDA(dStatus.ensure(nd));
			cudaStream_t st = ft->stream;
			RX_CUDA(cudaMemcpyAsync(dBlob.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
			RX_CUDA(cudaMemcpyAsync(dByteOff.p, byteOff.data(), byteOff.size() * 8, cudaMemcpyHostToDevice, st));
			RX_CUDA(cudaMemcpyAsync(dCnt.p, cnt.data(), size_t(nd) * 4, cudaMemcpyHostToDevice, st));
			const unsigned grid = (nd + 63) / 64;
			DevBuf<uint32_t> dMaxDoc;
			std::vector<uint32_t> maxDoc(nd);
			RX_CUDA(dMaxDoc.ensure(nd));
			ft_packed_decode<false><<<grid, 64, 0, st>>>(dBlob.p, dByteOff.p, dCnt.p, nd, ft->total_docs, ft->nfields, dNpos.p, dStatus.p, dMaxDoc.p,
														   nullptr, nullptr, nullptr, nullptr, nullptr);
			RX_CUDA(cudaMemcpyAsync(maxDoc.data(), dMaxDoc.p, size_t(nd) * 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaGetLastError());
			RX_CUDA(cudaMemcpyAsync(npos.data(), dNpos.p, size_t(nd) * 8, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaMemcpyAsync(status.data(), dStatus.p, size_t(nd) * 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			for (uint32_t j = 0; j < nd; ++j) {
				if (status[j] == 2) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: packed posting list holds a field outside the index / > 255 or a word position >= 2^24");
				}
				if (status[j] == 3) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: posting list must hold ascending document ids below total_docs");
				}
				if (status[j]) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: malformed packed posting list (or it contains array indexes / a different record count)");
				}
				if (npos[j] > 0xFFFFFFFFull) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: posting list with more than 2^32 positions");
				}
				posOff[j + 1] = posOff[j] + npos[j];
			}
			uint32_t *docs = nullptr, *begin = nullptr, *pos = nullptr;
			RX_CUDA(cudaMalloc(reinterpret_cast<void**>(&docs), std::max<uint64_t>(docOff[nd], 1) * 4));
			slabs.push_back(docs);
			cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&begin), (docOff[nd] + nd) * 4);
			if (e == cudaSuccess) {
				slabs.push_back(begin);
				e = cudaMalloc(reinterpret_cast<void**>(&pos), std::max<uint64_t>(posOff[nd], 1) * 4);
			}
			if (e != cudaSuccess) {
				dropSlabs();
				return fail(RXGPU_ERR_SYSTEM, std::string("CUDA error: ") + cudaGetErrorString(e) + " at cudaMalloc (posting slab)");
			}
			slabs.push_back(pos);
			cudaMemcpyAsync(dDocOff.p, docOff.data(), docOff.size() * 8, cudaMemcpyHostToDevice, st);
			cudaMemcpyAsync(dPosOff.p, posOff.data(), posOff.size() * 8, cudaMemcpyHostToDevice, st);
			ft_packed_decode<true><<<grid, 64, 0, st>>>(dBlob.p, dByteOff.p, dCnt.p, nd, ft->total_docs, ft->nfields, nullptr, nullptr, nullptr,
														  dDocOff.p, dPosOff.p, docs, begin, pos);
			e = cudaGetLastError();
			if (e == cudaSuccess) {
				e = cudaStreamSynchronize(st);
			}
			if (e != cudaSuccess) {
				dropSlabs();
				return fail(RXGPU_ERR_SYSTEM, std::string("CUDA error: ") + cudaGetErrorString(e) + " at the packed decode");
			}
			for (uint32_t j = 0; j < nd; ++j) {
				DevList& l = devLists[j];
				l.ndocs = cnt[j];
				l.npos = npos[j];
				l.doc_ids = docs + docOff[j];
				l.pos_begin = begin + docOff[j] + j;
				l.positions = pos + posOff[j];
				l.owned = false;
				l.max_doc_npos = maxDoc[j];
			}
		}
		// commit: ids in the caller's order; the long lists go through the host decoder one by one
		uint32_t j = 0;
		for (uint32_t i = 0; i < nlists; ++i) {
			if (j < nd && dev[j] == i) {
				ft->lists.push_back(devLists[j]);
				ft->max_list = std::max(ft->max_list, devLists[j].ndocs);
				out_ids[i] = uint32_t(ft->lists.size() - 1);
				++j;
			} else if (int rc = rxgpu_ft_add_postings_packed(ft, data[i], lens[i], counts[i], &out_ids[i])) {
				// roll back: nothing of a failed batch stays (slab-backed entries are dropped with their slabs)
				while (ft->lists.size() > firstId) {
					DevList& l = ft->lists.back();
					if (l.owned) {
						cudaFree(l.doc_ids);
						cudaFree(l.pos_begin);
						cudaFree(l.positions);
					}
					ft->lists.pop_back();
				}
				dropSlabs();
				return rc;
			}
		}
		ft->slabs.insert(ft->slabs.end(), slabs.begin(), slabs.end());
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

void rxgpu_ft_last_stats(rxgpu_ft_stats* out) {
	if (out) {
		*out = g_ft_stats;
	}
}

}  // extern "C"

namespace {
struct SelectReq {  // rxgpu_ft_select: post-processing and IndexText::afterSelect on the device
	const uint8_t* row_status;
	uint64_t limit;
	int32_t* out_row_ids;
	float* out_ranks;
};
// One docid-range shard of a namespace (SURVEY 8e): this index holds the documents [doc_base, doc_base + total_docs) with LOCAL ids, the
// posting lists restricted to them, the GLOBAL average field lengths.  The merge then needs five exchanges with the other shards, all
// tiny: (1) document and posting counts (BM25's IDF, maxMerged and the preselect estimate are namespace-wide), (2) the popcount of the
// restricting mask, (3) the 65 536-bin score histogram and the highest score, (4) how many documents AT the threshold score the lower
// shards hold (the ordered cut keeps the lowest ids), (5) the largest rank (uint8 normalisation) -- and at the end the shards' first
// `limit` rows are gathered and merged.  Everything else is per document.  After the preselect at most maxMerged documents survive in
// all shards together, so the slot order inside a shard never decides anything the select output shows.
struct FtShard {
	rxgpu_comm* comm;
	uint32_t doc_base;
};
struct AreasReq {  // rxgpu_ft_merge_query_areas: MergeDataAreas<Area> with maxAreasInDoc = A
	uint32_t A;
	uint32_t* out_begin;
	rxgpu_ft_area* out_areas;
	uint32_t* out_raw;
};
// SortSubterms: proc descending (querymergedata.h); stable here, the reference's pdqsort is not -- equal procs are a don't-care of the
// reference itself
struct Sub {
	uint32_t list;
	float proc;
	bool suppressed;
	uint64_t gdocs;  // documents of the list over the whole namespace (= the list's length unless the index is one shard of several)
};
// What the query asks for, checked: built by parseQuery and buildSubterms, read by every later stage of the merge
struct QueryPlan {
	// the query parts, then the terms of the multi-word synonyms in the order Merger::Merge walks them (mergerimpl.h:510-515); the
	// terms of synonym y are terms[synBegin[y], synBegin[y + 1])
	std::vector<rxgpu_ft_term> terms;
	std::vector<uint32_t> synBegin;
	uint32_t nterms = 0, nsyn = 0, nall = 0;
	// query parts: a plain term, or a phrase = consecutive terms that share a non-zero phrase_num (FtDslOpts::phraseNum; the selecter
	// groups them the same way, selecterimpl.h:548-558).  head[t]: term t opens a part; inPhrase[t]: it belongs to a phrase;
	// phraseLen[t]: the number of terms of the phrase term t opens
	std::vector<uint8_t> head, inPhrase;
	std::vector<uint32_t> phraseLen;
	uint32_t nparts = 0, nphrases = 0;
	std::vector<std::vector<Sub>> subs;  // per term of `terms`
	uint32_t N = 0;                      // documents of this index
	uint64_t gN = 0;                     // documents of the whole namespace
	uint32_t maxMerged = 0;
	bool simple = false, trivial = false;

	bool empty() const { return nparts == 0 || (nparts == 1 && terms[0].op == 3) || N == 0; }  // QueryMergeData::Empty(), mergerimpl.h:472
};
// The query flattened and split into parts, with every check in the merge's order (an empty query skips those of its terms)
int parseQuery(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, int rank_sort_type, uint64_t* out_n,
			   const SelectReq* sel, const FtShard* sh, QueryPlan& q) {
	if (!ft || !cfg || !out_n || !query || (query->nterms && !query->terms) || (query->nsynonyms && !query->synonyms)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	const uint32_t nterms = query->nterms;
	q.nterms = nterms;
	q.nsyn = query->nsynonyms;
	q.terms.assign(query->terms, query->terms + nterms);
	q.synBegin.assign(q.nsyn + 1, nterms);
	for (uint32_t y = 0; y < q.nsyn; ++y) {
		if (query->synonyms[y].nterms == 0 || !query->synonyms[y].terms) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: a multi-word synonym without terms");
		}
		q.terms.insert(q.terms.end(), query->synonyms[y].terms, query->synonyms[y].terms + query->synonyms[y].nterms);
		q.synBegin[y + 1] = uint32_t(q.terms.size());
	}
	q.nall = uint32_t(q.terms.size());
	if (cfg->nfields != ft->nfields || !cfg->fields) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: config field count differs from the index");
	}
	if (rank_sort_type == 2) {
		return fail(RXGPU_ERR_LOGIC, "RankSortType::ExternalExpression not implemented.");  // merger.h:151
	}
	RX_CUDA(cudaSetDevice(ft->device));
	g_ft_stats = rxgpu_ft_stats{};
	*out_n = 0;
	q.N = ft->total_docs;
	q.gN = q.N;
	if (sh && (!sel || q.nsyn || q.N == 0)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: a sharded merge serves the select path, query parts without multi-word synonyms, non-empty shards");
	}
	const rxgpu_ft_term* terms = q.terms.data();
	q.head.assign(nterms, 1);
	q.inPhrase.assign(nterms, 0);
	q.phraseLen.assign(nterms, 0);
	for (uint32_t t = 0; t < nterms; ++t) {
		if (terms[t].phrase_num != 0) {
			q.inPhrase[t] = 1;
			if (t > 0 && terms[t - 1].phrase_num == terms[t].phrase_num) {
				q.head[t] = 0;
			}
		}
		q.nparts += q.head[t];
	}
	for (uint32_t t = 0; t < nterms; ++t) {
		if (q.head[t] && q.inPhrase[t]) {
			uint32_t e = t + 1;
			while (e < nterms && !q.head[e]) {
				++e;
			}
			q.phraseLen[t] = e - t;
			++q.nphrases;
			if (q.phraseLen[t] < 2) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: a phrase needs at least two terms");
			}
			for (uint32_t u = t; u < e; ++u) {
				if (terms[u].nsynonyms || terms[u].distance < 0) {
					return fail(RXGPU_ERR_PARAMS, "rxgpu: malformed phrase term (synonym ids / negative distance)");
				}
			}
		}
	}
	if (sh && q.nphrases) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: phrases are not served by the sharded merge (a phrase's slot order is global)");
	}
	if (q.empty()) {
		return 0;
	}
	for (uint32_t t = 0; t < q.nall; ++t) {
		if (terms[t].op < 1 || terms[t].op > 3 || !terms[t].field_boosts || (terms[t].nsubterms && (!terms[t].postings || !terms[t].procs))) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: malformed query term");
		}
		if (terms[t].nsynonyms && (t >= q.nterms || !terms[t].synonym_ids)) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: synonym ids belong to query parts only");
		}
		for (uint32_t y = 0; y < terms[t].nsynonyms; ++y) {
			if (terms[t].synonym_ids[y] >= q.nsyn) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: unknown synonym id");
			}
		}
		for (uint32_t s = 0; s < terms[t].nsubterms; ++s) {
			if (terms[t].postings[s] >= ft->lists.size()) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: unknown posting list id");
			}
		}
		uint32_t summed = 0;
		for (uint32_t f = 0; terms[t].need_sum_rank && f < ft->nfields; ++f) {
			summed += terms[t].need_sum_rank[f] ? 1u : 0u;
		}
		if (summed > uint32_t(kMaxSumFields)) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: at most 16 fields of a term may carry needSumRank on the device path");
		}
	}
	if (!(cfg->summation_ranks_by_fields_ratio >= 0.0)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: summation_ranks_by_fields_ratio must be >= 0");
	}
	return 0;
}

// Every term's subterms with their namespace-wide document counts, sorted, and what Merger::init derives from them
int buildSubterms(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, const FtShard* sh, QueryPlan& q) {
	const rxgpu_ft_term* terms = q.terms.data();
	std::vector<unsigned long long> counts;
	if (sh) {  // exchange 1: the shards' document and posting counts, summed
		counts.push_back(q.N);
		for (uint32_t t = 0; t < q.nall; ++t) {
			for (uint32_t s = 0; s < terms[t].nsubterms; ++s) {
				counts.push_back(ft->lists[terms[t].postings[s]].ndocs);
			}
		}
		RX_CUDA(ft->shard_counts.ensure(counts.size()));
		RX_CUDA(cudaMemcpyAsync(ft->shard_counts.p, counts.data(), counts.size() * 8, cudaMemcpyHostToDevice, ft->stream));
		if (int rc = commAllReduce(sh->comm, ft->shard_counts.p, counts.size(), CommOp::SumU64, ft->stream)) {
			return rc;
		}
		RX_CUDA(cudaMemcpyAsync(counts.data(), ft->shard_counts.p, counts.size() * 8, cudaMemcpyDeviceToHost, ft->stream));
		RX_CUDA(cudaStreamSynchronize(ft->stream));
		q.gN = counts[0];
	}
	q.subs.resize(q.nall);
	uint64_t totalORVids = 0;  // selecterimpl.h:443,462,546,595: the synonyms' terms count as well
	size_t at = 1;
	for (uint32_t t = 0; t < q.nall; ++t) {
		for (uint32_t s = 0; s < terms[t].nsubterms; ++s) {
			const uint32_t list = terms[t].postings[s];
			const uint64_t gdocs = sh ? counts[at++] : ft->lists[list].ndocs;  // exchanged, or the list's length
			q.subs[t].push_back(Sub{list, terms[t].procs[s], terms[t].suppressed && terms[t].suppressed[s], gdocs});
			totalORVids += q.subs[t].back().gdocs;
		}
		if (t < q.nterms && q.inPhrase[t]) {
			continue;  // PhraseMerger::Merge runs inside Merger::init (merger.h:84-90), BEFORE SortSubterms: the caller's order stands
		}
		std::stable_sort(q.subs[t].begin(), q.subs[t].end(), [](const Sub& a, const Sub& b) { return a.proc > b.proc; });
	}
	q.maxMerged = uint32_t(std::min<uint64_t>(cfg->merge_limit, totalORVids));  // init(), merger.h:66-67
	q.simple = q.nparts == 1 && !q.inPhrase[0] && terms[0].op != 3 && q.nsyn == 0;  // QueryMergeData::Simple()
	q.trivial = q.simple && terms[0].nsubterms == 1;
	return 0;
}

uint64_t bytesOfPass(const DevList& l) { return uint64_t(l.ndocs) * 20 + l.npos * 4; }

// After a pass that adds documents (enqueued by the caller): its block counts scanned, the assign kernel, *n raised (capped at cap)
template <class... P, class... A>
void enqueueNewDocs(cudaStream_t st, unsigned lb, uint32_t* blockCounts, uint32_t* n, uint32_t* totalNew, uint32_t cap, void (*assign)(P...),
					A... args) {
	ft_scan_blocks<<<1, 1024, 0, st>>>(blockCounts, lb, totalNew);
	assign<<<lb, kFtThreads, 0, st>>>(args...);
	ft_bump_count<<<1, 1, 0, st>>>(n, totalNew, cap);
	g_ft_stats.launches += 3;
}

// The device state the stages of one merge share, and the stages from the scratch on
struct MergeRun {
	const QueryPlan& q;
	rxgpu_ft_index* ft;
	const rxgpu_ft_config* cfg;
	const FtShard* sh;
	const AreasReq* areas;
	cudaStream_t st;
	int sm;
	const rxgpu_ft_term* terms = q.terms.data();
	uint32_t mwords = (q.N + 31) / 32;                      // words of a document mask
	size_t areaFields = size_t(q.maxMerged) * ft->nfields;  // (slot, field) pairs
	const uint8_t* d_excluded = nullptr;
	MergeState ms{};
	AreaState as{};
	std::vector<PhraseState> pstates;
	std::vector<int> phraseOf = std::vector<int>(q.nterms, -1);  // head term -> index into ft->phrases
	const uint32_t* preselFlag = nullptr;  // set when preselectMostRelevantDocs may run: the device word that says whether it does

	// The scratch, MergeState and AreaState; then the stream's first work: the clock, the counters, the slot table, the restricting mask
	int setUp(const uint8_t* excluded) {
		const uint32_t N = q.N, maxMerged = q.maxMerged;
		const uint32_t nblocks_list = (ft->max_list + kFtThreads - 1) / kFtThreads + 1;
		const uint32_t nblocks_docs = (N + kFtThreads - 1) / kFtThreads + 1;
		RX_CUDA(ft->mask.ensure(mwords));
		RX_CUDA(ft->tmask.ensure(mwords));
		RX_CUDA(ft->block_counts.ensure(std::max(nblocks_list, nblocks_docs)));
		RX_CUDA(ft->scalar_u32.ensure(8));
		if (q.nsyn) {
			RX_CUDA(ft->syn_masks.ensure(size_t(q.nsyn) * mwords));
			RX_CUDA(ft->tmask2.ensure(mwords));
			RX_CUDA(ft->syn_full.ensure(maxMerged));
		}
		RX_CUDA(ft->popc.ensure(1));
		RX_CUDA(ft->tmp_rank.ensure(std::max<size_t>(1, ft->max_list)));
		RX_CUDA(ft->tmp_field.ensure(std::max<size_t>(1, ft->max_list)));
		RX_CUDA(ft->md_id.ensure(maxMerged));
		RX_CUDA(ft->md_proc.ensure(maxMerged));
		RX_CUDA(ft->md_field.ensure(maxMerged));
		if (!q.trivial) {
			RX_CUDA(ft->idoff.ensure(N));
		}
		if (!q.simple) {
			RX_CUDA(ft->last_ptr.ensure(maxMerged));
			RX_CUDA(ft->next_ptr.ensure(maxMerged));
			RX_CUDA(ft->last_n.ensure(maxMerged));
			RX_CUDA(ft->next_n.ensure(maxMerged));
			RX_CUDA(ft->ext_rank.ensure(maxMerged));
			RX_CUDA(ft->ext_cnt.ensure(maxMerged));
			RX_CUDA(ft->ext_last_term.ensure(maxMerged));
		}
		if (areas) {
			RX_CUDA(ft->area_ring.ensure(areaFields * areas->A));
			RX_CUDA(ft->area_out.ensure(areaFields * areas->A));
			RX_CUDA(ft->area_idx.ensure(areaFields));
			RX_CUDA(ft->area_cnt.ensure(areaFields + 1));
			RX_CUDA(ft->area_off.ensure(areaFields + 1));
			RX_CUDA(ft->area_raw.ensure(maxMerged));
			RX_CUDA(ft->area_max.ensure(maxMerged));
			RX_CUDA(ft->h_area_off.ensure(areaFields + 1));
			RX_CUDA(ft->h_area_raw.ensure(maxMerged));
			as = AreaState{ft->area_ring.p, ft->area_idx.p, ft->area_max.p, ft->nfields, areas->A};
		}
		if (excluded) {
			RX_CUDA(ft->excluded.ensure(N));
			RX_CUDA(cudaMemcpyAsync(ft->excluded.p, excluded, N, cudaMemcpyHostToDevice, st));
			d_excluded = ft->excluded.p;
		}
		ms.mask = ft->mask.p;
		ms.tmask = ft->tmask.p;
		ms.idoff = q.trivial ? nullptr : ft->idoff.p;
		ms.md_id = ft->md_id.p;
		ms.md_proc = ft->md_proc.p;
		ms.md_field = ft->md_field.p;
		ms.last_ptr = ft->last_ptr.p;
		ms.last_n = ft->last_n.p;
		ms.next_ptr = ft->next_ptr.p;
		ms.next_n = ft->next_n.p;
		ms.ext_rank = ft->ext_rank.p;
		ms.ext_cnt = ft->ext_cnt.p;
		ms.ext_last_term = ft->ext_last_term.p;
		ms.n_docs = ft->scalar_u32.p;  // [0] numDocs(); [1] new docs of the current pass

		if (!ft->ev0) {
			RX_CUDA(cudaEventCreate(&ft->ev0));
			RX_CUDA(cudaEventCreate(&ft->ev1));
		}
		RX_CUDA(ft->h_id.ensure(maxMerged));
		RX_CUDA(ft->h_proc.ensure(maxMerged));
		RX_CUDA(ft->h_field.ensure(maxMerged));
		RX_CUDA(ft->h_n.ensure(2));
		RX_CUDA(cudaEventRecord(ft->ev0, st));
		RX_CUDA(cudaMemsetAsync(ft->scalar_u32.p, 0, 32, st));
		if (!q.trivial) {  // idoffsets_: every merge leaves the table clean again (ft_reset_idoff), so the 4 N byte fill runs only once
			if (!ft->idoff_clean) {
				ft_fill_u32<<<gridFor(N, sm), kFtThreads, 0, st>>>(ft->idoff.p, kNoSlot, N);
				g_ft_stats.launches++;
			}
			ft->idoff_clean = false;
		}
		ft_mask_init<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(ft->mask.p, d_excluded, N, mwords);
		g_ft_stats.launches++;
		return 0;
	}

	TermParams termParams(uint32_t t, const Sub& sub) const {
		const rxgpu_ft_term& term = q.terms[t];
		const uint32_t nfields = ft->nfields;
		TermParams p{};
		for (uint32_t f = 0; f < nfields; ++f) {
			p.field_boosts[f] = term.field_boosts[f];
			p.fc[f] = FieldCfgF{float(cfg->fields[f].bm25_weight),     float(cfg->fields[f].bm25_boost),     float(cfg->fields[f].position_weight),
								float(cfg->fields[f].position_boost), float(cfg->fields[f].term_len_weight), float(cfg->fields[f].term_len_boost)};
		}
		p.boost = term.boost;
		p.term_len_boost = term.term_len_boost;
		p.proc = sub.proc;
		p.k1 = cfg->bm25_k1;
		p.b = cfg->bm25_b;
		p.bm25_type = cfg->bm25_type;
		p.nfields = nfields;
		p.dist_weight = float(cfg->distance_weight);
		p.dist_boost = float(cfg->distance_boost);
		p.sum_ratio = cfg->summation_ranks_by_fields_ratio;
		for (uint32_t f = 0; term.need_sum_rank && f < nfields; ++f) {
			p.need_sum_mask |= term.need_sum_rank[f] ? (1ull << f) : 0ull;
		}
		const double totalDocCount = double(q.gN - 1), matched = double(sub.gdocs);  // mergerimpl.h:122-124 (namespace-wide counts)
		if (cfg->bm25_type == 0) {  // Bm25Rx::IDF (bm25.h:21-27), on the host: the same libm as the reference
			double f = std::log((totalDocCount - matched + 1) / matched) / std::log(1 + totalDocCount);
			p.idf = f < 0.2 ? 0.2 : f;
		} else if (cfg->bm25_type == 1) {
			p.idf = std::log(totalDocCount / (matched + 1)) + 1;
		}
		return p;
	}

	// calcTermBitmask for every subterm of term t: the documents with a position in a field of non-zero boost are set in dst
	void markTermDocs(uint32_t t, uint32_t* dst) const {
		int allPositive = 1;
		for (uint32_t f = 0; f < ft->nfields; ++f) {
			allPositive &= q.terms[t].field_boosts[f] != 0.f;
		}
		for (const Sub& sub : q.subs[t]) {
			const DevList& l = ft->lists[sub.list];
			if (l.ndocs) {
				ft_and_mark<<<gridFor(l.ndocs, sm), kFtThreads, 0, st>>>(l, termParams(t, sub), allPositive, dst);
				g_ft_stats.launches++;
				g_ft_stats.postings_scanned += l.ndocs;
				g_ft_stats.algorithmic_bytes += bytesOfPass(l);
			}
		}
	}

	// PhraseMerger::Merge for every phrase part (Merger::init, merger.h:82-90) -- before anything else, on docsExcluded as given
	int mergePhrases() {
		if (!q.nphrases) {
			return 0;
		}
		const uint32_t N = q.N;
		while (ft->phrases.size() < q.nphrases) {
			ft->phrases.emplace_back(std::make_unique<rxgpu_ft_index::PhraseBufs>());
		}
		RX_CUDA(ft->p_idoff.ensure(N));
		RX_CUDA(ft->p_term_mask.ensure(mwords));
		if (!ft->p_idoff_clean) {
			ft_fill_u32<<<gridFor(N, sm), kFtThreads, 0, st>>>(ft->p_idoff.p, kNoSlot, N);
			g_ft_stats.launches++;
			ft->p_idoff_clean = true;
		}
		uint32_t pi = 0;
		for (uint32_t t = 0; t < q.nterms; ++t) {
			if (!(q.head[t] && q.inPhrase[t])) {
				continue;
			}
			const uint32_t len = q.phraseLen[t];
			rxgpu_ft_index::PhraseBufs& pb = *ft->phrases[pi];
			phraseOf[t] = int(pi++);
			// init (phrasemerger.h:341-358)
			uint64_t firstVDocs = 0;
			for (const Sub& sub : q.subs[t]) {
				firstVDocs += ft->lists[sub.list].ndocs;
			}
			pb.max_merged = uint32_t(std::min<uint64_t>(cfg->merge_limit, firstVDocs));
			long long sumProc = 0;  // PhraseResults::CalcProc16 (querymergedata.h:121-131): the FIRST subterm of every term
			uint64_t cap = 1;
			for (uint32_t u = t; u < t + len; ++u) {
				if (!q.subs[u].empty()) {
					sumProc += (long long)(q.subs[u][0].proc);
				}
				uint64_t c = 0;
				for (const Sub& sub : q.subs[u]) {
					c += ft->lists[sub.list].max_doc_npos;
				}
				cap = std::max(cap, c);
			}
			if (sumProc < 0 || sumProc >= 65535) {
				return fail(RXGPU_ERR_PARAMS, "rxgpu: the procs of a phrase's terms do not fit 16 bits (PhraseResults::CalcProc16)");
			}
			pb.phrase_proc = uint32_t(sumProc);
			const uint64_t slots = std::max<uint32_t>(pb.max_merged, 1);
			if (slots * cap * 8 > (uint64_t(4) << 30)) {
				return fail(RXGPU_ERR_LOGIC, "rxgpu: the phrase's position buffers would exceed 4 GiB on the device (merge_limit x positions per document)");
			}
			pb.cap = uint32_t(cap);
			RX_CUDA(pb.pre.ensure(mwords));
			RX_CUDA(pb.n.ensure(2));
			RX_CUDA(pb.id.ensure(slots));
			RX_CUDA(pb.proc.ensure(slots));
			RX_CUDA(pb.rank.ensure(slots));
			RX_CUDA(pb.field.ensure(slots));
			RX_CUDA(pb.flags.ensure(slots));
			RX_CUDA(pb.last_n.ensure(slots));
			RX_CUDA(pb.next_n.ensure(slots));
			RX_CUDA(pb.last.ensure(slots * cap));
			RX_CUDA(pb.next.ensure(slots * cap));
			RX_CUDA(cudaMemsetAsync(pb.n.p, 0, 8, st));
			PhraseState ps{pb.pre.p, ft->p_idoff.p, pb.id.p, pb.proc.p, pb.field.p, pb.rank.p, pb.last.p, pb.last_n.p,
						   pb.next.p, pb.next_n.p, pb.cap, pb.max_merged, pb.n.p};
			// preselectDocsContainingAllTerms (phrasemergerimpl.h:262-300): AND of the terms' document sets, removed documents leave with
			// the last term, excluded ones at the end
			ft_mask_init<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(pb.pre.p, d_excluded, N, mwords);
			g_ft_stats.launches++;
			for (uint32_t u = t; u < t + len; ++u) {
				RX_CUDA(cudaMemsetAsync(ft->p_term_mask.p, 0, size_t(mwords) * 4, st));
				for (const Sub& sub : q.subs[u]) {
					const DevList& l = ft->lists[sub.list];
					if (l.ndocs) {
						ft_phrase_mark<<<gridFor(l.ndocs, sm), kFtThreads, 0, st>>>(l, u + 1 == t + len && ft->has_removed ? ft->removed.p : nullptr,
																					  ft->p_term_mask.p);
						g_ft_stats.launches++;
						g_ft_stats.postings_scanned += l.ndocs;
					}
				}
				ft_mask_and<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(pb.pre.p, ft->p_term_mask.p, mwords);
				g_ft_stats.launches++;
			}
			// mergePhraseTerm for every term (phrasemergerimpl.h:166-259)
			for (uint32_t u = t; u < t + len; ++u) {
				for (const Sub& sub : q.subs[u]) {
					const DevList& l = ft->lists[sub.list];
					if (!l.ndocs) {
						continue;
					}
					const unsigned lb = (l.ndocs + kFtThreads - 1) / kFtThreads;
					if (u == t) {
						if (pb.max_merged == 0) {
							continue;
						}
						ft_phrase_first_pass<<<lb, kFtThreads, 0, st>>>(l, termParams(u, sub), ps, ft->words.p, ft->avg.p, ft->tmp_rank.p,
																		 ft->tmp_field.p, ft->block_counts.p);
						enqueueNewDocs(st, lb, ft->block_counts.p, pb.n.p, pb.n.p + 1, pb.max_merged, ft_phrase_first_assign, l, ps, ft->tmp_rank.p,
									   ft->tmp_field.p, ft->block_counts.p);
					} else {
						ft_phrase_next_pass<<<lb, kFtThreads, 0, st>>>(l, termParams(u, sub), ps, uint32_t(q.terms[u].distance), ft->words.p,
																		ft->avg.p);
					}
					g_ft_stats.launches++;
					g_ft_stats.postings_scanned += l.ndocs;
					g_ft_stats.algorithmic_bytes += bytesOfPass(l);
				}
				ft_phrase_end_term<<<gridFor(std::max<uint32_t>(pb.max_merged, 1), sm), kFtThreads, 0, st>>>(ps);
				g_ft_stats.launches++;
			}
			ft_reset_idoff<<<gridFor(std::max<uint32_t>(pb.max_merged, 1), sm), kFtThreads, 0, st>>>(pb.id.p, pb.n.p, ft->p_idoff.p);
			g_ft_stats.launches++;
			RX_CUDA(cudaMemcpyAsync(&pb.num_merged, pb.n.p, 4, cudaMemcpyDeviceToHost, st));  // NumDocsMerged() feeds estimateNumDocsInMerge
			pstates.push_back(ps);
		}
		RX_CUDA(cudaGetLastError());
		RX_CUDA(cudaStreamSynchronize(st));
		return 0;
	}

	// buildRestrictingBitmask (mergerimpl.h:326-384)
	int buildRestrictingBitmask() {
		std::vector<uint8_t> synMaskDone(q.nsyn, 0);
		for (uint32_t t = 0; t < q.nterms; ++t) {
			if (!q.head[t] || terms[t].op != 2) {
				continue;
			}
			RX_CUDA(cudaMemsetAsync(ft->tmask.p, 0, size_t(mwords) * 4, st));
			if (q.inPhrase[t]) {  // phraseMergers_[i].GetMergedDocsBitmask (mergerimpl.h:346-347)
				const PhraseState& ps = pstates[phraseOf[t]];
				ft_phrase_bits<<<gridFor(std::max<uint32_t>(ps.max_merged, 1), sm), kFtThreads, 0, st>>>(ps, ft->tmask.p, 1);
				ft_mask_and<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(ft->mask.p, ft->tmask.p, mwords);
				g_ft_stats.launches += 2;
				continue;
			}
			markTermDocs(t, ft->tmask.p);
			for (uint32_t y = 0; y < terms[t].nsynonyms; ++y) {  // termMask |= AND over the synonym's terms (mergerimpl.h:352-363)
				const uint32_t sy = terms[t].synonym_ids[y];
				uint32_t* synMask = ft->syn_masks.p + size_t(sy) * mwords;
				if (!synMaskDone[sy]) {
					for (uint32_t u = q.synBegin[sy]; u < q.synBegin[sy + 1]; ++u) {
						uint32_t* dst = u == q.synBegin[sy] ? synMask : ft->tmask2.p;
						RX_CUDA(cudaMemsetAsync(dst, 0, size_t(mwords) * 4, st));
						markTermDocs(u, dst);
						if (u != q.synBegin[sy]) {
							ft_mask_and<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(synMask, ft->tmask2.p, mwords);
							g_ft_stats.launches++;
						}
					}
					synMaskDone[sy] = 1;
				}
				ft_mask_or<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(ft->tmask.p, synMask, mwords);
				g_ft_stats.launches++;
			}
			ft_mask_and<<<gridFor(mwords, sm), kFtThreads, 0, st>>>(ft->mask.p, ft->tmask.p, mwords);
			g_ft_stats.launches++;
		}
		for (uint32_t t = 0; t < q.nterms; ++t) {
			if (!q.head[t] || terms[t].op != 3) {
				continue;
			}
			if (q.inPhrase[t]) {  // ExcludeMergedDocsFromBitmask (mergerimpl.h:378-379)
				const PhraseState& ps = pstates[phraseOf[t]];
				ft_phrase_bits<<<gridFor(std::max<uint32_t>(ps.max_merged, 1), sm), kFtThreads, 0, st>>>(ps, ft->mask.p, 0);
				g_ft_stats.launches++;
				continue;
			}
			for (const Sub& sub : q.subs[t]) {
				const DevList& l = ft->lists[sub.list];
				if (l.ndocs) {
					ft_not_clear<<<gridFor(l.ndocs, sm), kFtThreads, 0, st>>>(l, ft->mask.p);
					g_ft_stats.launches++;
					g_ft_stats.postings_scanned += l.ndocs;
				}
			}
		}
		return 0;
	}

	// estimateNumDocsInMerge (merger.h:239-267), then if needed preselectMostRelevantDocs (mergerimpl.h:386-464) with exchanges 2-4
	int preselectMostRelevantDocs() {
		const uint32_t nterms = q.nterms, nall = q.nall;
		uint64_t estOr = 0, estAnd = UINT64_MAX;
		for (uint32_t t = 0; t < nterms; ++t) {
			if (!q.head[t] || terms[t].op == 3) {
				continue;
			}
			uint64_t nd = 0;
			for (const Sub& sub : q.subs[t]) {
				nd += sub.gdocs;
			}
			if (q.inPhrase[t]) {
				nd = ft->phrases[phraseOf[t]]->num_merged;  // phraseMergers_[i].NumDocsMerged() (merger.h:252)
			}
			for (uint32_t y = 0; y < terms[t].nsynonyms; ++y) {  // + the first term of each of its synonyms (merger.h:253-256)
				for (const Sub& sub : q.subs[q.synBegin[terms[t].synonym_ids[y]]]) {
					nd += sub.gdocs;
				}
			}
			if (terms[t].op == 2) {
				estAnd = std::min(estAnd, nd);
			} else {
				estOr += nd;
			}
		}
		const uint64_t est = std::min<uint64_t>(std::min(estOr, estAnd), q.gN);
		if (!(est > cfg->merge_limit && q.gN > cfg->merge_limit && !std::getenv("REINDEXER_NO_2PHASE_FT_MERGE"))) {
			return 0;
		}
		uint32_t* d_presel = ft->scalar_u32.p + 6;  // [6] 1 when preselectMostRelevantDocs runs
		RX_CUDA(cudaMemsetAsync(ft->popc.p, 0, 8, st));
		ft_popcount<<<std::min<unsigned>(gridFor(mwords, sm), unsigned(sm) * 4), kFtThreads, 0, st>>>(ft->mask.p, mwords, ft->popc.p);
		if (sh) {  // exchange 2: restrictingMask_.PopCount() over all shards
			if (int rc = commAllReduce(sh->comm, ft->popc.p, 1, CommOp::SumU64, st)) {
				return rc;
			}
		}
		ft_decide_preselect<<<1, 1, 0, st>>>(ft->popc.p, cfg->merge_limit, d_presel);
		g_ft_stats.launches += 2;
		preselFlag = d_presel;  // the last condition is known on the device only: the kernels below test it, the host does not wait
		RX_CUDA(ft->score.ensure(size_t(mwords) * 32));
		RX_CUDA(ft->hist.ensure(65536));
		RX_CUDA(cudaMemsetAsync(ft->score.p, 0, size_t(mwords) * 64, st));
		RX_CUDA(cudaMemsetAsync(ft->hist.p, 0, 65536 * 8, st));
		for (uint32_t tt = 0; tt < nall; ++tt) {
			const uint32_t t = tt < nall - nterms ? nterms + tt : tt - (nall - nterms);  // the synonyms' terms first (mergerimpl.h:392-396)
			if (t < nterms && (!q.head[t] || terms[t].op == 3)) {
				continue;
			}
			if (t < nterms && q.inPhrase[t]) {  // GetMergedDocsScore (mergerimpl.h:408-409)
				const PhraseState& ps = pstates[phraseOf[t]];
				ft_phrase_score<<<gridFor(std::max<uint32_t>(ps.max_merged, 1), sm), kFtThreads, 0, st>>>(ps, ft->score.p,
																										   ft->phrases[phraseOf[t]]->phrase_proc, preselFlag);
				g_ft_stats.launches++;
				continue;
			}
			RX_CUDA(cudaMemsetAsync(ft->tmask.p, 0, size_t(mwords) * 4, st));
			int allSame = 1;
			for (uint32_t f = 0; f < ft->nfields; ++f) {
				allSame &= terms[t].field_boosts[f] == terms[t].field_boosts[0];
			}
			for (const Sub& sub : q.subs[t]) {
				const DevList& l = ft->lists[sub.list];
				if (l.ndocs) {
					ft_score_pass<<<gridFor(l.ndocs, sm), kFtThreads, 0, st>>>(l, termParams(t, sub), allSame, ft->mask.p, ft->tmask.p, ft->score.p,
																				preselFlag);
					g_ft_stats.launches++;
					g_ft_stats.postings_scanned += l.ndocs;
					g_ft_stats.algorithmic_bytes += bytesOfPass(l);
				}
			}
		}
		const unsigned pg = unsigned(sm) * 4;    // persistent grid of the per-document passes
		uint32_t* d_thr = ft->scalar_u32.p + 2;  // [2] minScore, [3] minScoreDocs
		RX_CUDA(ft->block_counts.ensure(pg));
		ft_hist<<<pg, kFtThreads, 0, st>>>(ft->score.p, ft->mask.p, ft->has_removed ? ft->removed.p : nullptr, mwords, ft->hist.p, ft->scalar_u32.p + 5,
										   preselFlag);
		if (sh) {  // exchange 3: the score histogram and the highest score of the whole namespace -> the same threshold on every shard
			if (int rc = commAllReduce(sh->comm, ft->hist.p, 65536, CommOp::SumU64, st)) {
				return rc;
			}
			if (int rc = commAllReduce(sh->comm, ft->scalar_u32.p + 5, 1, CommOp::MaxU32, st)) {
				return rc;
			}
		}
		ft_pick_threshold<<<1, 1024, 0, st>>>(ft->hist.p, q.maxMerged, ft->scalar_u32.p + 5, d_thr, preselFlag);
		ft_thresh_count<<<pg, kFtThreads, 0, st>>>(ft->score.p, ft->mask.p, mwords, d_thr, ft->block_counts.p, preselFlag);
		if (sh) {  // exchange 4: the documents AT the threshold score are kept in ascending GLOBAL id order = lower shards first
			const uint32_t R = uint32_t(commSize(sh->comm));
			RX_CUDA(ft->shard_u32.ensure(size_t(R) + 1));
			ft_sum_u32<<<1, 256, 0, st>>>(ft->block_counts.p, pg, ft->shard_u32.p + R);
			if (int rc = commAllGather(sh->comm, ft->shard_u32.p + R, ft->shard_u32.p, 4, st)) {
				return rc;
			}
			ft_shard_budget<<<1, 1, 0, st>>>(d_thr, ft->shard_u32.p, uint32_t(commRank(sh->comm)));
			g_ft_stats.launches += 2;
		}
		ft_thresh_apply<<<pg, kFtThreads, 0, st>>>(ft->score.p, ft->mask.p, mwords, d_thr, ft->block_counts.p, preselFlag);
		g_ft_stats.launches += 4;
		g_ft_stats.algorithmic_bytes += uint64_t(q.N) * 6;
		return 0;
	}

	// The mergeSimple / mergeTerm passes of every query part and synonym term, mergePhrase for the phrases, the synonyms' marks
	int mergeTerms() {
		const uint32_t nterms = q.nterms, nsyn = q.nsyn, maxMerged = q.maxMerged;
		const uint8_t* d_removed = ft->has_removed ? ft->removed.p : nullptr;
		const int checkRemoved = 1;
		const auto rankPass = areas ? ft_rank_pass<true> : ft_rank_pass<false>;
		const auto assign = areas ? ft_assign<true> : ft_assign<false>;
		uint16_t qpIdx = 0;
		uint32_t* d_total_new = ft->scalar_u32.p + 1;  // [1] new docs of the current pass
		uint32_t* d_before = ft->scalar_u32.p + 4;     // [4] numDocsBeforeSynonyms
		for (uint32_t t = 0; t < q.nall; ++t) {
			if (t == nterms) {
				ft_copy_u32<<<1, 1, 0, st>>>(d_before, ms.n_docs);
				RX_CUDA(cudaMemsetAsync(ft->syn_full.p, 0, maxMerged, st));
				g_ft_stats.launches++;
			}
			if (t < nterms && !q.head[t]) {
				continue;  // inside a phrase: merged with its head
			}
			// mergeTerm returns at once for OpNot (mergerimpl.h:113-115); a NOT query part does not even take an index (:497-499)
			const bool isNot = terms[t].op == 3;
			if (!isNot || t >= nterms) {
				++qpIdx;
			}
			if (t < nterms && q.inPhrase[t]) {
				if (!isNot) {  // mergePhrase (mergerimpl.h:41-90): no switchToNextWord, the phrase's last positions become the document's
					const PhraseState& ps = pstates[phraseOf[t]];
					uint8_t* flags = ft->phrases[phraseOf[t]]->flags.p;
					const unsigned lb = (std::max<uint32_t>(ps.max_merged, 1) + kFtThreads - 1) / kFtThreads;
					RX_CUDA(ft->block_counts.ensure(lb + 1));
					ft_phrase_merge_pass<<<lb, kFtThreads, 0, st>>>(ps, ms, qpIdx, flags, ft->block_counts.p);
					g_ft_stats.launches++;
					enqueueNewDocs(st, lb, ft->block_counts.p, ms.n_docs, d_total_new, maxMerged, ft_phrase_merge_assign, ps, ms, maxMerged, qpIdx, flags,
								   ft->block_counts.p);
				}
				continue;
			}
			if (!q.simple && !isNot) {
				ft_switch<<<gridFor(maxMerged, sm), kFtThreads, 0, st>>>(ms);
				g_ft_stats.launches++;
			}
			for (const Sub& sub : q.subs[t]) {
				if (isNot) {
					break;
				}
				const DevList& l = ft->lists[sub.list];
				if (!l.ndocs) {
					continue;
				}
				const unsigned lb = (l.ndocs + kFtThreads - 1) / kFtThreads;
				if (sub.suppressed) {
					ft_suppressed_pass<<<lb, kFtThreads, 0, st>>>(l, ms, d_removed, checkRemoved, kNoSlot, qpIdx, preselFlag);
					g_ft_stats.launches++;
					g_ft_stats.postings_scanned += l.ndocs;
					g_ft_stats.algorithmic_bytes += uint64_t(l.ndocs) * 8;
					continue;
				}
				rankPass<<<lb, kFtThreads, 0, st>>>(l, termParams(t, sub), ms, ft->words.p, ft->avg.p, d_removed, checkRemoved, q.simple ? 1 : 0,
													kNoSlot, qpIdx, ft->tmp_rank.p, ft->tmp_field.p, ft->block_counts.p, preselFlag, as);
				enqueueNewDocs(st, lb, ft->block_counts.p, ms.n_docs, d_total_new, maxMerged, assign, l, ms, q.simple ? 1 : 0, maxMerged, qpIdx,
							   ft->tmp_rank.p, ft->tmp_field.p, ft->block_counts.p, as);
				g_ft_stats.launches++;
				g_ft_stats.postings_scanned += l.ndocs;
				g_ft_stats.algorithmic_bytes += bytesOfPass(l) + uint64_t(l.ndocs) * 9;
			}
			for (uint32_t y = 0; y < nsyn; ++y) {
				if (t + 1 == q.synBegin[y + 1]) {  // the last term of synonym y
					ft_syn_mark<<<gridFor(maxMerged, sm), kFtThreads, 0, st>>>(ms, d_before, uint16_t(q.synBegin[y + 1] - q.synBegin[y]), ft->syn_full.p);
					g_ft_stats.launches++;
				}
			}
		}
		return 0;
	}

	// canBeBoostedByFullMatch, the synonyms' finish, the slot table cleaned, the areas committed
	int finish() {
		const uint32_t maxMerged = q.maxMerged;
		const uint32_t* d_before = ft->scalar_u32.p + 4;
		// canBeBoostedByFullMatch: termsCounter == queryParts.size() (NOT parts never count); QueryLength() == nterms: every phrase counts
		// its terms (querymergedata.h:212-219)
		ft_full_match<<<gridFor(maxMerged, sm), kFtThreads, 0, st>>>(ms, ft->words.p, ft->nfields, q.simple ? 1u : q.nterms, q.nparts, q.simple ? 1 : 0,
																	 cfg->full_match_boost);
		g_ft_stats.launches++;
		if (q.nsyn) {
			ft_syn_finish<<<gridFor(maxMerged, sm), kFtThreads, 0, st>>>(ms, d_before, ft->syn_full.p);
			g_ft_stats.launches++;
		}
		if (!q.trivial) {
			ft_reset_idoff<<<gridFor(maxMerged, sm), kFtThreads, 0, st>>>(ms.md_id, ms.n_docs, ft->idoff.p);
			g_ft_stats.launches++;
		}
		if (areas) {  // commit every slot's areas, then the slot-ordered CSR: offsets by an exclusive scan over (slot, field), areas by emit
			ft_areas_commit<<<gridFor(uint64_t(maxMerged) * 32, sm), kFtThreads, 0, st>>>(as, ms.n_docs, maxMerged, ft->area_cnt.p, ft->area_raw.p);
			size_t tmpBytes = 0;
			cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, ft->area_cnt.p, ft->area_off.p, areaFields + 1, st);
			RX_CUDA(ft->sort_tmp.ensure(tmpBytes));
			cub::DeviceScan::ExclusiveSum(ft->sort_tmp.p, tmpBytes, ft->area_cnt.p, ft->area_off.p, areaFields + 1, st);
			ft_areas_emit<<<gridFor(areaFields, sm), kFtThreads, 0, st>>>(as, ms.n_docs, ft->area_cnt.p, ft->area_off.p, ft->area_out.p);
			g_ft_stats.launches += 3;
		}
		RX_CUDA(cudaGetLastError());
		return 0;
	}

	// The end of every call after its copies: one synchronisation, then the bookkeeping of a success (*flag: copy of scalar_u32[6])
	int endCall(const uint32_t* flag) {
		RX_CUDA(cudaStreamSynchronize(st));
		RX_CUDA(cudaEventElapsedTime(&g_ft_stats.device_ms, ft->ev0, ft->ev1));
		ft->idoff_clean = !q.trivial;
		g_ft_stats.preselected = preselFlag ? *flag : 0;
		return 0;
	}

	// postProcessResults (drop ranks below minRank, uint8 normalisation by the global maximum) + afterSelect (vdoc -> row ids, optional
	// external statuses) + sortAfterSelect ((rank desc, row id asc) or row id asc) without leaving the device; only the first `limit` rows
	// travel back.  A shard runs exchange 5 on the way and gathers every shard's first rows at the end.
	int select(const SelectReq* sel, bool rankAndId, uint64_t* out_n) {
		const uint32_t maxMerged = q.maxMerged;
		RX_CUDA(ft->post_scalars.ensure(4));
		RX_CUDA(ft->post_cnt.ensure(maxMerged));
		RX_CUDA(ft->post_off.ensure(maxMerged));
		RX_CUDA(ft->h_post.ensure(4));
		const uint8_t* d_status = nullptr;
		if (sel->row_status) {
			const uint64_t nrows = ft->has_rows ? ft->max_row + 1 : q.N;
			RX_CUDA(ft->row_status.ensure(nrows));
			RX_CUDA(cudaMemcpyAsync(ft->row_status.p, sel->row_status, nrows, cudaMemcpyHostToDevice, st));
			d_status = ft->row_status.p;
		}
		const uint32_t* rb = ft->has_rows ? ft->row_begin.p : nullptr;
		const int32_t* ri = ft->has_rows ? ft->row_ids.p : nullptr;
		ft_post_scale<<<1, 1024, 0, st>>>(ms.md_proc, ms.n_docs, ft->post_scalars.p);
		if (sh) {  // exchange 5: the uint8 normalisation divides by the largest rank of the whole namespace
			if (int rc = commAllReduce(sh->comm, ft->post_scalars.p + 2, 1, CommOp::MaxU32, st)) {
				return rc;
			}
			ft_post_rescale<<<1, 1, 0, st>>>(ft->post_scalars.p);
			g_ft_stats.launches++;
		}
		ft_post_count<<<gridFor(maxMerged, sm), kFtThreads, 0, st>>>(ms.md_id, ms.md_proc, ms.n_docs, float(cfg->min_rank), rb, ri, d_status, maxMerged,
																	 ft->post_cnt.p);
		size_t tmpBytes = 0;
		cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, ft->post_cnt.p, ft->post_off.p, int(maxMerged), st);
		RX_CUDA(ft->sort_tmp.ensure(tmpBytes));
		cub::DeviceScan::ExclusiveSum(ft->sort_tmp.p, tmpBytes, ft->post_cnt.p, ft->post_off.p, int(maxMerged), st);
		g_ft_stats.launches += 3;
		// Key capacity: every merged document contributes at most max_rows_per_doc rows.  When that bound is small the whole chain
		// (emit -> sort -> copy of the first `limit` keys) is enqueued without stopping for the host; unused slots hold a key above every
		// valid one.  Otherwise the row total is read back first to size the sort.
		const uint64_t capBound = uint64_t(maxMerged) * (ft->has_rows ? std::max<uint64_t>(ft->max_rows_per_doc, 1) : 1);
		uint32_t rowsTotal = 0, nMerged = maxMerged;
		uint64_t sortItems = capBound;
		const bool noSync = capBound <= (1u << 20);
		if (!noSync) {
			RX_CUDA(cudaMemcpyAsync(ft->h_post.p, ms.n_docs, 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaMemcpyAsync(ft->h_post.p + 1, ft->scalar_u32.p + 6, 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			nMerged = ft->h_post.p[0];
			if (nMerged) {
				uint32_t lastOff = 0, lastCnt = 0;
				RX_CUDA(cudaMemcpyAsync(&lastOff, ft->post_off.p + (nMerged - 1), 4, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaMemcpyAsync(&lastCnt, ft->post_cnt.p + (nMerged - 1), 4, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaStreamSynchronize(st));
				rowsTotal = lastOff + lastCnt;
			}
			sortItems = rowsTotal;
		}
		if (sortItems) {
			RX_CUDA(ft->post_keys.ensure(sortItems));
			RX_CUDA(ft->post_keys_sorted.ensure(sortItems));
			if (noSync) {
				RX_CUDA(cudaMemsetAsync(ft->post_keys.p, 0xFF, sortItems * 8, st));  // padding: bits 0..40 all set > any valid 40-bit key
				RX_CUDA(cudaMemsetAsync(ft->post_scalars.p + 1, 0, 4, st));
			}
			ft_post_emit<<<gridFor(nMerged, sm), kFtThreads, 0, st>>>(ms.md_id, ms.md_proc, ms.n_docs, ft->post_scalars.p, rb, ri, d_status, ft->post_cnt.p,
																	   ft->post_off.p, rankAndId ? 1 : 0, ft->post_keys.p, ft->post_scalars.p + 1,
																	   sh ? sh->doc_base : 0u);
			size_t sortBytes = 0;
			cub::DeviceRadixSort::SortKeys(nullptr, sortBytes, ft->post_keys.p, ft->post_keys_sorted.p, int(sortItems), 0, 41, st);
			RX_CUDA(ft->sort_tmp.ensure(sortBytes));
			cub::DeviceRadixSort::SortKeys(ft->sort_tmp.p, sortBytes, ft->post_keys.p, ft->post_keys_sorted.p, int(sortItems), 0, 41, st);
			g_ft_stats.launches += 2;
		}
		RX_CUDA(cudaGetLastError());
		const uint64_t lim = sel->limit;
		const uint32_t R = sh ? uint32_t(commSize(sh->comm)) : 1;
		if (sh) {  // the shards' first `limit` rows (keys are globally comparable: rank and GLOBAL row id) gathered; the row totals summed
			RX_CUDA(ft->shard_keys.ensure(std::max<uint64_t>(lim, 1) * (R + 1)));
			unsigned long long* snd = ft->shard_keys.p + lim * R;
			if (lim) {
				RX_CUDA(cudaMemsetAsync(snd, 0xFF, lim * 8, st));
				const uint64_t have = std::min<uint64_t>(sortItems, lim);
				if (have) {
					RX_CUDA(cudaMemcpyAsync(snd, ft->post_keys_sorted.p, have * 8, cudaMemcpyDeviceToDevice, st));
				}
				if (int rc = commAllGather(sh->comm, snd, ft->shard_keys.p, lim * 8, st)) {
					return rc;
				}
			}
			if (!noSync) {  // the row total was read back to size the sort: put it where the other path leaves it
				RX_CUDA(cudaMemcpyAsync(ft->post_scalars.p + 1, &rowsTotal, 4, cudaMemcpyHostToDevice, st));
			} else if (!sortItems) {
				RX_CUDA(cudaMemsetAsync(ft->post_scalars.p + 1, 0, 4, st));
			}
			if (int rc = commAllReduce(sh->comm, ft->post_scalars.p + 1, 1, CommOp::SumU32, st)) {
				return rc;
			}
		}
		RX_CUDA(cudaEventRecord(ft->ev1, st));
		// one copy of the first rows (of every shard, on a shard) and, unless it was read back already, of the row total
		const bool readTotal = sh || noSync;
		const uint64_t nkeys = sh ? lim * R : std::min<uint64_t>(noSync ? sortItems : rowsTotal, lim);
		RX_CUDA(ft->h_keys.ensure(std::max<uint64_t>(nkeys, 1)));
		if (nkeys) {
			RX_CUDA(cudaMemcpyAsync(ft->h_keys.p, sh ? ft->shard_keys.p : ft->post_keys_sorted.p, nkeys * 8, cudaMemcpyDeviceToHost, st));
		}
		if (readTotal) {
			RX_CUDA(cudaMemcpyAsync(ft->h_post.p, ft->post_scalars.p + 1, 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaMemcpyAsync(ft->h_post.p + 1, ft->scalar_u32.p + 6, 4, cudaMemcpyDeviceToHost, st));
		}
		if (int rc = endCall(ft->h_post.p + 1)) {
			return rc;
		}
		const uint64_t total = readTotal ? ft->h_post.p[0] : rowsTotal;
		const unsigned long long* keys = ft->h_keys.p;
		uint64_t nout = std::min<uint64_t>(total, lim);
		std::vector<unsigned long long> all;
		if (sh) {  // every shard's slice is sorted and row ids are disjoint: a plain sort of <= R x limit keys
			for (uint64_t i = 0; i < lim * R; ++i) {
				if (ft->h_keys.p[i] != ~0ull) {
					all.push_back(ft->h_keys.p[i]);
				}
			}
			std::sort(all.begin(), all.end());
			keys = all.data();
			nout = std::min<uint64_t>(all.size(), lim);
		}
		for (uint64_t i = 0; i < nout; ++i) {  // a RankAndID key is (255 - rank) << 32 | row id, an IDOnly key row id << 8 | rank
		sel->out_row_ids[i] = int32_t(uint32_t(rankAndId ? keys[i] : keys[i] >> 8));
		sel->out_ranks[i] = float(rankAndId ? 255u - uint32_t(keys[i] >> 32) : uint32_t(keys[i] & 0xFF));
	}
		*out_n = total;
		return 0;
	}

	// The merge's own output: the merged documents (<= merge_limit entries, 9 bytes each) and their areas come back in full -- their
	// number is not known before the copy -- and postProcessResults (merger.h:111-155) runs on the host
	int postProcessResults(int rank_sort_type, uint64_t max_out, rxgpu_ft_merge_info* out, uint64_t* out_n) {
		const size_t maxMerged = q.maxMerged;
		RX_CUDA(cudaEventRecord(ft->ev1, st));
		RX_CUDA(cudaMemcpyAsync(ft->h_n.p, ms.n_docs, 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(ft->h_n.p + 1, ft->scalar_u32.p + 6, 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(ft->h_id.p, ms.md_id, maxMerged * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(ft->h_proc.p, ms.md_proc, maxMerged * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(ft->h_field.p, ms.md_field, maxMerged, cudaMemcpyDeviceToHost, st));
		if (areas) {
			RX_CUDA(cudaMemcpyAsync(ft->h_area_off.p, ft->area_off.p, (areaFields + 1) * 4, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaMemcpyAsync(ft->h_area_raw.p, ft->area_raw.p, maxMerged * 4, cudaMemcpyDeviceToHost, st));
		}
		if (int rc = endCall(ft->h_n.p + 1)) {
			return rc;
		}
		const uint32_t n = ft->h_n.p[0];
		if (areas) {  // the number of committed areas is known now: they follow in one copy
			const uint32_t totalAreas = ft->h_area_off.p[size_t(n) * ft->nfields];
			RX_CUDA(ft->h_areas.ensure(std::max<uint32_t>(totalAreas, 1)));
			if (totalAreas) {
				RX_CUDA(cudaMemcpyAsync(ft->h_areas.p, ft->area_out.p, size_t(totalAreas) * 8, cudaMemcpyDeviceToHost, st));
				RX_CUDA(cudaStreamSynchronize(st));
			}
		}
		try {
			const int32_t* ids = ft->h_id.p;
			const float* procs = ft->h_proc.p;
			const uint8_t* fields = ft->h_field.p;
			std::vector<rxgpu_ft_merge_info> md;
			std::vector<uint32_t> slotOf;  // areas: the slot of md[i] (MergeInfo::areaIndex), moved with it
			md.reserve(n);
			float maxProc = 0.f;
			for (uint32_t i = 0; i < n; ++i) {
				if (q.nsyn && procs[i] == -INFINITY) {
					continue;  // held only a part of a multi-word synonym: removed in order (mergerimpl.h:539-560)
				}
				md.push_back(rxgpu_ft_merge_info{ids[i], procs[i], fields[i], 0});
				maxProc = std::max(maxProc, procs[i]);
				if (areas) {
					slotOf.push_back(i);
				}
			}
			const float scalingFactor = maxProc > 255 ? float(255.0 / maxProc) : 1.0f;
			const float minProc = float(cfg->min_rank);
			size_t passed = md.size();
			while (passed > 0 && md[passed - 1].proc < minProc) {
				passed--;
			}
			for (size_t i = 0; i + 1 < passed; i++) {
				if (md[i].proc < minProc) {
					md[i] = md[passed - 1];
					if (areas) {
						slotOf[i] = slotOf[passed - 1];
					}
					passed--;
					while (passed > i && md[passed - 1].proc < minProc) {
						passed--;
					}
				}
			}
			md.resize(passed);
			for (auto& m : md) {
				m.normalized_proc = uint8_t(m.proc * scalingFactor);
				m.proc = m.normalized_proc;
			}
			if (rank_sort_type == 0 || rank_sort_type == 4) {  // RankOnly / IDAndPositions: one stable order for the entries and their slots
				std::vector<uint32_t> perm(md.size());
				std::iota(perm.begin(), perm.end(), 0u);
				std::stable_sort(perm.begin(), perm.end(), [&](uint32_t l, uint32_t r) { return md[l].normalized_proc > md[r].normalized_proc; });
				std::vector<rxgpu_ft_merge_info> mdSorted;
				std::vector<uint32_t> slotSorted;
				for (uint32_t i : perm) {
					mdSorted.push_back(md[i]);
					if (areas) {
						slotSorted.push_back(slotOf[i]);
					}
				}
				md.swap(mdSorted);
				slotOf.swap(slotSorted);
			}
			*out_n = md.size();
			for (size_t i = 0; i < md.size() && i < max_out; ++i) {
				out[i] = md[i];
			}
			if (areas) {  // gather the slot-ordered CSR into the output order
				const uint32_t nf = ft->nfields;
				const uint32_t* off = ft->h_area_off.p;
				uint32_t at = 0;
				size_t i = 0;
				for (; i < md.size() && i < max_out; ++i) {
					const size_t s = slotOf[i];
					for (uint32_t f = 0; f < nf; ++f) {
						areas->out_begin[i * nf + f] = at;
						for (uint32_t a = off[s * nf + f]; a < off[s * nf + f + 1]; ++a) {
							areas->out_areas[at++] = rxgpu_ft_area{ft->h_areas.p[a].x, ft->h_areas.p[a].y};
						}
					}
					if (areas->out_raw) {
						areas->out_raw[i] = ft->h_area_raw.p[s];
					}
				}
				areas->out_begin[i * nf] = at;
			}
		} catch (const std::bad_alloc&) {
			return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
		}
		return 0;
	}
};

int ftMergeImpl(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded, int rank_sort_type,
				uint64_t max_out, rxgpu_ft_merge_info* out, uint64_t* out_n, const SelectReq* sel, const FtShard* sh = nullptr,
				const AreasReq* areas = nullptr) {
	QueryPlan q;
	if (int rc = parseQuery(ft, cfg, query, rank_sort_type, out_n, sel, sh, q); rc || q.empty()) {
		return rc;
	}
	std::lock_guard<std::mutex> lck(ft->mtx);
	if (int rc = buildSubterms(ft, cfg, sh, q); rc || q.maxMerged == 0) {
		return rc;
	}
	MergeRun r{q, ft, cfg, sh, areas, ft->stream, ft->sm_count};
	if (int rc = r.setUp(excluded)) {
		return rc;
	}
	if (int rc = r.mergePhrases()) {
		return rc;
	}
	if (!q.simple) {
		if (int rc = r.buildRestrictingBitmask()) {
			return rc;
		}
		if (int rc = r.preselectMostRelevantDocs()) {
			return rc;
		}
	}
	if (int rc = r.mergeTerms()) {
		return rc;
	}
	if (int rc = r.finish()) {
		return rc;
	}
	return sel ? r.select(sel, rank_sort_type == 1, out_n) : r.postProcessResults(rank_sort_type, max_out, out, out_n);
}
}  // namespace

extern "C" {

int rxgpu_ft_merge(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, uint32_t nterms, const rxgpu_ft_term* terms, const uint8_t* excluded,
				   int rank_sort_type, uint64_t max_out, rxgpu_ft_merge_info* out, uint64_t* out_n) {
	const rxgpu_ft_query q{nterms, terms, 0, nullptr};
	return rxgpu_ft_merge_query(ft, cfg, &q, excluded, rank_sort_type, max_out, out, out_n);
}
int rxgpu_ft_merge_query(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded, int rank_sort_type,
						 uint64_t max_out, rxgpu_ft_merge_info* out, uint64_t* out_n) {
	return ftMergeImpl(ft, cfg, query, excluded, rank_sort_type, max_out, out, out_n, nullptr);
}
int rxgpu_ft_merge_query_areas(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded,
							   int rank_sort_type, int32_t max_areas_in_doc, uint64_t max_out, rxgpu_ft_merge_info* out,
							   uint32_t* out_area_begin, rxgpu_ft_area* out_areas, uint32_t* out_raw_count, uint64_t* out_n) {
	if (!ft || !cfg || !query || !out_n || !out_area_begin || (query->nterms && !query->terms) || (max_out && (!out || !out_areas))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (max_areas_in_doc < 1 || max_areas_in_doc > kMaxAreasInDoc) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: max_areas_in_doc must lie in [1, 64]");
	}
	for (uint32_t t = 0; t < query->nterms; ++t) {
		if (query->terms[t].phrase_num != 0) {  // PhraseMerger's areas depend on an unstable sort's order (DESIGN.md §8.1)
			return fail(RXGPU_ERR_PARAMS, "rxgpu: areas are not served for queries with phrases");
		}
	}
	const AreasReq req{uint32_t(max_areas_in_doc), out_area_begin, out_areas, out_raw_count};
	const int rc = ftMergeImpl(ft, cfg, query, excluded, rank_sort_type, max_out, out, out_n, nullptr, nullptr, &req);
	if (rc == 0 && *out_n == 0) {
		out_area_begin[0] = 0;
	}
	return rc;
}

int rxgpu_ft_set_rows(rxgpu_ft_index* ft, const uint32_t* row_begin, const int32_t* row_ids) {
	if (!ft) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	RX_CUDA(cudaSetDevice(ft->device));
	std::lock_guard<std::mutex> lck(ft->mtx);
	if (!row_begin) {
		ft->has_rows = false;
		return 0;
	}
	const uint32_t n = ft->total_docs;
	if (row_begin[0] != 0) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: row_begin must start at 0");
	}
	uint64_t maxRow = 0, maxPerDoc = 1;
	for (uint32_t d = 0; d < n; ++d) {
		if (row_begin[d + 1] < row_begin[d]) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: row_begin must be non-decreasing");
		}
		maxPerDoc = std::max<uint64_t>(maxPerDoc, row_begin[d + 1] - row_begin[d]);
	}
	const uint64_t total = row_begin[n];
	if (total && !row_ids) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	for (uint64_t i = 0; i < total; ++i) {
		if (row_ids[i] < 0) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: negative row id");
		}
		maxRow = std::max<uint64_t>(maxRow, uint64_t(row_ids[i]));
	}
	RX_CUDA(ft->row_begin.ensure(size_t(n) + 1));
	RX_CUDA(ft->row_ids.ensure(std::max<uint64_t>(total, 1)));
	RX_CUDA(cudaMemcpy(ft->row_begin.p, row_begin, (size_t(n) + 1) * 4, cudaMemcpyHostToDevice));
	if (total) {
		RX_CUDA(cudaMemcpy(ft->row_ids.p, row_ids, total * 4, cudaMemcpyHostToDevice));
	}
	ft->max_row = maxRow;
	ft->max_rows_per_doc = maxPerDoc;
	ft->has_rows = true;
	return 0;
}

static int ftSelectCheck(int rank_sort_type, uint64_t limit, const int32_t* out_row_ids, const float* out_ranks) {
	if (rank_sort_type != 1 && rank_sort_type != 3) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: rxgpu_ft_select orders by RankAndID (1) or IDOnly (3); use rxgpu_ft_merge for the other sort types");
	}
	if (limit && (!out_row_ids || !out_ranks)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	return 0;
}
int rxgpu_ft_select(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, uint32_t nterms, const rxgpu_ft_term* terms, const uint8_t* excluded,
					const uint8_t* row_status, int rank_sort_type, uint64_t limit, int32_t* out_row_ids, float* out_ranks, uint64_t* out_n) {
	const rxgpu_ft_query q{nterms, terms, 0, nullptr};
	return rxgpu_ft_select_query(ft, cfg, &q, excluded, row_status, rank_sort_type, limit, out_row_ids, out_ranks, out_n);
}
int rxgpu_ft_select_query(rxgpu_ft_index* ft, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded,
						  const uint8_t* row_status, int rank_sort_type, uint64_t limit, int32_t* out_row_ids, float* out_ranks, uint64_t* out_n) {
	if (int rc = ftSelectCheck(rank_sort_type, limit, out_row_ids, out_ranks)) {
		return rc;
	}
	const SelectReq sel{row_status, limit, out_row_ids, out_ranks};
	return ftMergeImpl(ft, cfg, query, excluded, rank_sort_type, 0, nullptr, out_n, &sel);
}

int rxgpu_sharded_ft_select(rxgpu_comm* comm, rxgpu_ft_index* shard, uint32_t doc_base, const rxgpu_ft_config* cfg, uint32_t nterms,
							const rxgpu_ft_term* terms, const uint8_t* excluded, const uint8_t* row_status, int rank_sort_type, uint64_t limit,
							int32_t* out_row_ids, float* out_ranks, uint64_t* out_n) {
	if (!comm || !shard) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (int rc = ftSelectCheck(rank_sort_type, limit, out_row_ids, out_ranks)) {
		return rc;
	}
	if (limit > (1u << 20)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: the sharded select gathers `limit` rows per shard: limit <= 2^20");
	}
	if (commDevice(comm) != shard->device) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: the shard lives on another device than its communicator");
	}
	std::lock_guard<std::mutex> lck(commMutex(comm));
	const SelectReq sel{row_status, limit, out_row_ids, out_ranks};
	const rxgpu_ft_query q{nterms, terms, 0, nullptr};
	const FtShard sh{comm, doc_base};
	return ftMergeImpl(shard, cfg, &q, excluded, rank_sort_type, 0, nullptr, out_n, &sel, &sh);
}

}  // extern "C"
