"""Random ft_fast merge problems for the oracle pin tests and the GPU parity tests (test infrastructure)."""
import numpy as np

from oracle import ft_oracle as F


def random_problem(seed, total_docs=400, nfields=1, nterms=3, max_sub=3, density=0.2, merge_limit=20000, ops=None, removed_frac=0.0,
                   excluded_frac=0.0, field_boost_zero=False, max_pos=3, doc_len=(3, 40)):
    rng = np.random.default_rng(seed)
    words = rng.integers(doc_len[0], doc_len[1], size=(total_docs, nfields)).astype(np.uint32)
    words[0] = 0
    removed = (rng.random(total_docs) < removed_frac).astype(np.uint8) if removed_frac else None
    excluded = (rng.random(total_docs) < excluded_frac).astype(np.uint8) if excluded_frac else None
    p = F.FtProblem(total_docs, words, removed=removed, excluded=excluded)
    p.cfg["merge_limit"] = merge_limit
    procs_pool = [100.0, 90.0, 85.0, 80.0, 72.0, 65.0, 57.0, 50.0, 43.0, 31.0]
    for t in range(nterms):
        nsub = int(rng.integers(1, max_sub + 1))
        subs = []
        procs = rng.choice(procs_pool, size=nsub, replace=False)  # distinct procs: SortSubterms is unstable for ties
        for s in range(nsub):
            dens = density * float(rng.uniform(0.3, 1.5)) / (1 + s)
            ndocs = max(1, int(dens * (total_docs - 1)))
            docs = np.sort(rng.choice(np.arange(1, total_docs), size=min(ndocs, total_docs - 1), replace=False))
            pos_lists = []
            for d in docs:
                npos = int(rng.integers(1, max_pos + 1))
                pp = []
                for _ in range(npos):
                    f = int(rng.integers(0, nfields))
                    pp.append((int(rng.integers(0, max(int(words[d, f]), 1))), f))
                pos_lists.append(pp)
            subs.append((p.add_list(docs, pos_lists), float(procs[s])))
        op = ops[t] if ops else int(rng.choice([F.OP_OR, F.OP_OR, F.OP_AND, F.OP_NOT])) if t else F.OP_OR
        fb = np.ones(nfields, np.float32)
        if nfields > 1:
            fb = rng.choice([1.0, 0.5, 2.0, 1.5], size=nfields).astype(np.float32)
            if field_boost_zero:
                fb[int(rng.integers(0, nfields))] = 0.0
        p.add_term(subs, op=op, boost=float(rng.choice([1.0, 1.0, 0.7, 1.3])), term_len_boost=float(rng.choice([1.0, 0.8, 0.5])),
                   field_boosts=fb)
    return p


def add_random_synonyms(p, seed, nsyn=2, density=0.25, suppress=True):
    """Multi-word synonyms on top of random_problem: every synonym has 2-3 terms of 1-2 subterms each, is attached to one or two
    OR / AND query parts (PhraseOrTerm::AddSynonymId), and may carry a suppressed subterm that re-uses a posting list of the query
    (what QueryMergeData::SupressDuplicatesInSynonyms marks)."""
    rng = np.random.default_rng(seed ^ 0x5A17)
    total_docs, nfields = p.total_docs, p.nfields
    hosts = [i for i, t in enumerate(p.terms) if t["op"] != F.OP_NOT]
    for y in range(nsyn):
        terms = []
        for _ in range(int(rng.integers(2, 4))):
            subs = []
            procs = rng.choice([60.0, 52.0, 45.0, 38.0, 33.0], size=2, replace=False)
            for s_ in range(int(rng.integers(1, 3))):
                ndocs = max(1, int(density * float(rng.uniform(0.4, 1.4)) * (total_docs - 1)))
                docs = np.sort(rng.choice(np.arange(1, total_docs), size=min(ndocs, total_docs - 1), replace=False))
                pos_lists = [[(int(rng.integers(0, max(int(p.words[d, f]), 1))), f) for f in [int(rng.integers(0, nfields))]
                              for _ in range(int(rng.integers(1, 3)))] for d in docs]
                subs.append((p.add_list(docs, pos_lists), float(procs[s_])))
            if suppress and rng.random() < 0.4:  # a word of the query repeated inside the synonym
                host = p.terms[int(rng.choice(hosts))]
                subs.append((int(host["postings"][0]), 29.0, True))
            terms.append(dict(subterms=subs, op=F.OP_OR, boost=float(rng.choice([1.0, 0.8])), term_len_boost=1.0,
                              field_boosts=np.ones(nfields, np.float32)))
        sid = p.add_synonym(terms)
        for h in rng.choice(hosts, size=min(len(hosts), int(rng.integers(1, 3))), replace=False):
            p.terms[int(h)]["synonym_ids"] = np.append(p.terms[int(h)]["synonym_ids"], np.uint32(sid)).astype(np.uint32)
    return p


def corpus_problem(seed, total_docs=600, nfields=2, vocab=24, merge_limit=20000, removed_frac=0.0, excluded_frac=0.0, with_synonym=False):
    """A problem built from an actual token corpus, so that PHRASES match: every document holds random words of a small vocabulary in
    every field; posting lists are derived from it.  The query mixes one or two phrases (2-3 terms, distances 1-3, 1-2 variant subterms
    per term, in the caller's -- unsorted -- order) with plain terms under OR / AND / NOT."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(4, 22, size=(total_docs, nfields))
    lens[0] = 0
    words = lens.astype(np.uint32)
    removed = (rng.random(total_docs) < removed_frac).astype(np.uint8) if removed_frac else None
    excluded = (rng.random(total_docs) < excluded_frac).astype(np.uint8) if excluded_frac else None
    p = F.FtProblem(total_docs, words, removed=removed, excluded=excluded)
    p.cfg["merge_limit"] = merge_limit
    tokens = [[rng.integers(0, vocab, size=lens[d, f]) for f in range(nfields)] for d in range(total_docs)]
    list_of_word = {}

    def postings(w):
        if w not in list_of_word:
            docs, pos_lists = [], []
            for d in range(1, total_docs):
                pp = [(int(i), f) for f in range(nfields) for i in np.nonzero(tokens[d][f] == w)[0]]
                if pp:
                    docs.append(d)
                    pos_lists.append(pp)
            list_of_word[w] = p.add_list(docs, pos_lists)
        return list_of_word[w]

    def subterms(primary):
        subs = [(postings(int(primary)), float(rng.choice([100.0, 90.0, 85.0])))]
        if rng.random() < 0.5:  # a variant (typo / stem) of lower relevancy, possibly listed FIRST
            v = (postings(int(rng.integers(0, vocab))), float(rng.choice([72.0, 65.0, 57.0])))
            subs = [v] + subs if rng.random() < 0.5 else subs + [v]
        return subs

    nparts = int(rng.integers(1, 4))
    phrase_num = 0
    for part in range(nparts):
        op = F.OP_OR if part == 0 else int(rng.choice([F.OP_OR, F.OP_OR, F.OP_AND, F.OP_NOT]))
        fb = rng.choice([1.0, 0.5, 2.0], size=nfields).astype(np.float32) if nfields > 1 else np.ones(1, np.float32)
        if part == 0 or rng.random() < 0.5:  # a phrase taken from a real document, so that it occurs
            phrase_num += 1
            d, f = int(rng.integers(1, total_docs)), int(rng.integers(0, nfields))
            n = int(rng.integers(2, 4))
            at = int(rng.integers(0, max(1, lens[d, f] - 2 * n)))
            step = int(rng.integers(1, 3))
            chosen = [int(tokens[d][f][min(at + k * step, lens[d, f] - 1)]) for k in range(n)]
            for k, w in enumerate(chosen):
                p.add_term(subterms(w), op=op, boost=float(rng.choice([1.0, 0.8])), term_len_boost=float(rng.choice([1.0, 0.9])),
                           field_boosts=fb, phrase_num=phrase_num, distance=int(rng.integers(1, 4)) if k else 0)
        else:
            syn = ()
            if with_synonym and op != F.OP_NOT:
                syn = (p.add_synonym([dict(subterms=[(postings(int(rng.integers(0, vocab))), 45.0)], field_boosts=np.ones(nfields, np.float32))
                                      for _ in range(2)]),)
            p.add_term(subterms(int(rng.integers(0, vocab))), op=op, boost=1.0, term_len_boost=1.0, field_boosts=fb, synonym_ids=syn)
    return p


def bulk_list(p, rng, docs, npos=1, max_pos=40, nfields=None, fields=None, first_pos=None):
    """add_list without a per-document Python loop: docs ascending and unique, npos positions per document (a scalar or one count per
    document) in random fields below nfields (or the given per-document `fields`) at word positions below max_pos, duplicates merged.
    first_pos (per document) moves the positions of a document up by that much and adds first_pos itself in the document's first
    field (field 0, or fields[i]), so it is that field's first position."""
    docs = np.ascontiguousarray(docs, np.uint32)
    nfields = p.nfields if nfields is None else nfields
    cnt = np.broadcast_to(np.asarray(npos, np.int64), docs.shape)
    assert (cnt >= 1).all()
    owner = np.repeat(np.arange(len(docs)), cnt)
    f = rng.integers(0, nfields, size=len(owner)) if fields is None else np.asarray(fields, np.int64)[owner]
    pos = rng.integers(0, max_pos, size=len(owner))
    if first_pos is not None:
        pos = np.minimum(pos + np.asarray(first_pos, np.int64)[owner], (1 << 24) - 1)
    packed = (f.astype(np.uint64) << 24) | pos.astype(np.uint64)
    if first_pos is not None:
        f0 = np.zeros(len(docs), np.int64) if fields is None else np.asarray(fields, np.int64)
        owner = np.concatenate([owner, np.arange(len(docs))])
        packed = np.concatenate([packed, (f0.astype(np.uint64) << 24) | np.asarray(first_pos, np.uint64)])
    order = np.lexsort((packed, owner))
    owner, packed = owner[order], packed[order]
    keep = np.ones(len(owner), bool)
    keep[1:] = (owner[1:] != owner[:-1]) | (packed[1:] != packed[:-1])
    owner, packed = owner[keep], packed[keep].astype(np.uint32)
    begin = np.zeros(len(docs) + 1, np.uint32)
    begin[1:] = np.cumsum(np.bincount(owner, minlength=len(docs)))
    return p.add_list_arrays(docs, begin, packed)


def random_words(rng, total_docs, nfields, lo=3, hi=40):
    words = rng.integers(lo, hi, size=(total_docs, nfields)).astype(np.uint32)
    words[0] = 0
    return words


def score_problem(scores, saturated=None, seed=0, nfields=1, merge_limit=20000, excluded=None, removed=None, max_pos=40):
    """OR terms whose preselect scores are chosen per document (scores[d] in 0..65535).  Term b (b = 0..13) holds the documents whose
    remainder has bit b set, with subterm proc 1 and term boost 2^b; up to four more terms of boost 16384 add 65535 / 4 = 16383 each
    (the per-subterm cap).  So calcTermScores (mergerimpl.h:289-324) gives document d exactly scores[d].  Documents marked `saturated`
    are put into five capped terms instead: 5 x 16383 saturates the u16 sum at 65535."""
    scores = np.asarray(scores, np.int64)
    total_docs = len(scores)
    assert scores[0] == 0 and (scores >= 0).all() and (scores <= 65535).all()
    caps = np.minimum(scores // 16383, 4)
    target = scores - caps * 16383
    if saturated is not None:
        caps = np.where(saturated, 5, caps)
        target = np.where(saturated, 0, target)
    rng = np.random.default_rng(seed)
    p = F.FtProblem(total_docs, random_words(rng, total_docs, nfields), removed=removed, excluded=excluded)
    p.cfg["merge_limit"] = merge_limit
    assert (target < 16384).all()
    for b in range(14):
        docs = np.nonzero((target >> b) & 1)[0]
        if len(docs):
            p.add_term([(bulk_list(p, rng, docs, npos=rng.integers(1, 3, size=len(docs)), max_pos=max_pos), 1.0)], boost=float(1 << b))
    for c in range(int(caps.max())):
        docs = np.nonzero(caps > c)[0]
        p.add_term([(bulk_list(p, rng, docs, max_pos=max_pos), 1.0)], boost=16384.0)
    return p


def planted_scores(n, seed, top, thr, run_start, run_len, frac=0.3, above=0.02):
    """preselect scores for score_problem: a fraction of the documents below thr, a few in (thr, top], document 1 at top and a run
    of run_len consecutive documents from run_start at exactly thr (so the threshold's documents fill whole mask words)"""
    rng = np.random.default_rng(seed)
    s = np.zeros(n, np.int64)
    lo = rng.random(n) < frac
    s[lo] = rng.integers(1, max(thr, 2), size=int(lo.sum()))
    if top > thr:
        hi = rng.random(n) < above
        s[hi] = rng.integers(thr + 1, top + 1, size=int(hi.sum()))
    s[run_start:run_start + run_len] = thr
    s[1] = top
    s[0] = 0
    return s


def cut_limit(scores, thr, cut_id):
    """the merge_limit that makes thr the threshold score and keeps the threshold's documents up to and including cut_id"""
    eq = np.nonzero(scores == thr)[0]
    assert cut_id in eq
    return int((scores > thr).sum()) + int(np.searchsorted(eq, cut_id, side="right"))


def ref_u16(proc):
    """static_cast<uint16_t>(float) as the reference's x86-64 build executes it: cvttss2si truncates to int32 (NaN and values outside
    [-2^31, 2^31) give INT32_MIN), then the low 16 bits are kept"""
    x = np.asarray(proc, np.float32).astype(np.float64)
    ok = (x >= -2.0 ** 31) & (x < 2.0 ** 31)
    i = np.where(ok, np.trunc(np.where(ok, x, 0.0)), -2.0 ** 31).astype(np.int64)
    return (i & 0xFFFF).astype(np.int64)


def _per_doc(lst, fb, any_nonzero):
    """per document of a list: whether a position lies in a field of non-zero boost (calcTermBitmask), or the largest field boost
    over its positions, starting from 0 (maxFieldsBoost)"""
    d, b, q = lst
    assert (np.diff(b.astype(np.int64)) > 0).all()
    if not len(d):
        return np.zeros(0, bool if any_nonzero else np.float32)
    v = np.asarray(fb, np.float32)[q >> 24]
    if any_nonzero:
        return np.logical_or.reduceat(v != 0, b[:-1].astype(np.int64))
    return np.maximum(np.maximum.reduceat(v, b[:-1].astype(np.int64)), np.float32(0))


def preselect_plan(p, to_u16=None):
    """numpy restatement of buildRestrictingBitmask, estimateNumDocsInMerge, calcTermScores and the threshold walk of
    preselectMostRelevantDocs (mergerimpl.h:289-464, merger.h:239-267) for plain OR / AND / NOT terms.  Used to prove that a
    problem reaches a boundary of the device's preselect: the top score, the threshold (minScore) and the budget of documents kept
    at the threshold, and which documents hold that score.  to_u16 replaces the reference's float -> u16 conversion (ref_u16)."""
    assert not p.synonyms and not any(t.get("phrase_num", 0) for t in p.terms)
    N = p.total_docs
    mask = np.ones(N, bool) if p.excluded is None else p.excluded == 0
    for t in p.terms:
        if t["op"] == F.OP_AND:
            tm = np.zeros(N, bool)
            for li in t["postings"]:
                d = p.lists[int(li)][0]
                tm[d if (t["field_boosts"] != 0).all() else d[_per_doc(p.lists[int(li)], t["field_boosts"], True)]] = True
            mask &= tm
    for t in p.terms:
        if t["op"] == F.OP_NOT:
            for li in t["postings"]:
                mask[p.lists[int(li)][0]] = False
    est_or, est_and = 0, None
    for t in p.terms:
        if t["op"] == F.OP_NOT:
            continue
        nd = sum(len(p.lists[int(li)][0]) for li in t["postings"])
        if t["op"] == F.OP_AND:
            est_and = nd if est_and is None else min(est_and, nd)
        else:
            est_or += nd
    est = min(est_or if est_and is None else min(est_or, est_and), N)
    total_or = sum(len(p.lists[int(li)][0]) for t in p.terms for li in t["postings"])
    ml = p.cfg["merge_limit"]
    max_merged = min(ml, total_or)
    popcount = int(mask.sum())
    simple = len(p.terms) == 1 and p.terms[0]["op"] != F.OP_NOT
    score = np.zeros(N, np.int64)
    for t in p.terms:
        if t["op"] == F.OP_NOT:
            continue
        fb = np.asarray(t["field_boosts"], np.float32)
        tmask = np.zeros(N, bool)
        for li, sp in zip(t["postings"], t["procs"]):
            d = p.lists[int(li)][0].astype(np.int64)
            mb = np.full(len(d), fb[0], np.float32) if (fb == fb[0]).all() else _per_doc(p.lists[int(li)], fb, False)
            sel = mask[d] & (mb > 0) & ~tmask[d]
            proc = (np.float32(sp) * mb[sel]).astype(np.float32) * np.float32(t["boost"])
            p16 = np.minimum((to_u16 or ref_u16)(proc), 65535 // 4)
            dd = d[sel]
            score[dd] += np.minimum(p16, 65535 - score[dd])
            tmask[dd] = True
    if p.removed is not None:
        score[p.removed != 0] = 0
    score[~mask] = 0
    hist = np.bincount(score, minlength=65536)
    min_score, budget, taken = 65535, 0, 0
    for sc in range(65535, 0, -1):
        if taken >= max_merged:
            break
        min_score, budget = sc, max_merged - taken
        taken += int(hist[sc])
    eq = np.nonzero(mask & (score == min_score))[0]
    return dict(preselect=(not simple) and est > ml and N > ml and popcount > ml, popcount=popcount, estimate=est, max_merged=max_merged,
                score=score, top=int(score.max()), min_score=min_score, budget=budget, eq=eq, positive=int((score > 0).sum()),
                kept=int((score > min_score).sum()) + min(budget, len(eq)))


def assert_same_merge(a, b, rank_sort_type, ctx=""):
    """a, b: MERGE_INFO arrays.  RankAndID / IDOnly keep the merge order (deterministic); RankOnly / IDAndPositions are sorted by an
    unstable sort, so equal ranks compare as sets."""
    assert len(a) == len(b), (ctx, len(a), len(b))
    if rank_sort_type in (F.RANK_AND_ID, F.ID_ONLY):
        assert (a["id"] == b["id"]).all(), ctx
        assert (a["normalized_proc"] == b["normalized_proc"]).all(), (ctx, a[:8], b[:8])
        assert (a["field"] == b["field"]).all(), ctx
        assert (a["proc"] == b["proc"]).all(), ctx
    else:
        assert (a["normalized_proc"] == b["normalized_proc"]).all(), ctx
        oa, ob = np.lexsort((a["id"], -a["normalized_proc"].astype(int))), np.lexsort((b["id"], -b["normalized_proc"].astype(int)))
        assert (a["id"][oa] == b["id"][ob]).all() and (a["field"][oa] == b["field"][ob]).all(), ctx


def load_golden_problem(g, name):
    """Rebuild an FtProblem from tests/golden/ft_golden.npz (inputs are stored, not regenerated)."""
    words = g[f"{name}/words"]
    rem, exc = g[f"{name}/removed"], g[f"{name}/excluded"]
    p = F.FtProblem(words.shape[0], words, avg=g[f"{name}/avg"], removed=rem if len(rem) else None, excluded=exc if len(exc) else None)
    for i in range(int(g[f"{name}/nlists"])):
        p.add_list_arrays(g[f"{name}/list{i}/docs"], g[f"{name}/list{i}/begin"], g[f"{name}/list{i}/pos"])
    for i in range(int(g[f"{name}/nterms"])):
        op, boost, tlb = g[f"{name}/term{i}/scalars"]
        p.terms.append(dict(op=int(op), boost=float(boost), term_len_boost=float(tlb), field_boosts=g[f"{name}/term{i}/field_boosts"],
                            postings=g[f"{name}/term{i}/postings"], procs=g[f"{name}/term{i}/procs"]))
    p.cfg["merge_limit"] = int(g[f"{name}/merge_limit"])
    return p


def gpu_merge(prob, rank_sort_type=F.RANK_AND_ID, packed=None, batch=False):
    """Run one problem through the product (rxgpu_ft_*); returns (result, stats).  packed: per-list byte streams of the reference's
    PackedIdRelVec -- the lists are then uploaded through rxgpu_ft_add_postings_packed."""
    import reindexer_b200 as rx

    ft = rx.GpuFtIndex(prob.total_docs, prob.words, prob.avg, prob.removed)
    if packed is not None and batch:  # the raw streams travel to the device and are decoded there (rxgpu_ft_add_postings_packed_batch)
        ids = ft.add_postings_packed_batch(packed, [len(l[0]) for l in prob.lists])
    elif packed is not None:
        ids = [ft.add_postings_packed(packed[i], len(prob.lists[i][0])) for i in range(len(prob.lists))]
    else:
        ids = [ft.add_postings(d, b, p) for d, b, p in prob.lists]
    terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in prob.terms]
    syns = [[dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in syn] for syn in prob.synonyms]
    res = ft.merge(prob.cfg, prob.field_cfg, terms, excluded=prob.excluded, rank_sort_type=rank_sort_type, synonyms=syns or None)
    st = ft.last_stats()
    ft.close()
    return res, st
