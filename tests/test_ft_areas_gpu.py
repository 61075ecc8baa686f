"""GPU tests of rxgpu_ft_merge_query_areas: the ft_fast merge with highlight areas (MergeDataAreas<Area>) checked exactly against the
reference's own merger (oracle/_ref/liboracle_ref_ft_areas.so): the merge infos bit for bit, every returned document's committed areas
per field, and its area count before the commit.  RankAndID / IDOnly compare entry by entry; RankOnly / IDAndPositions are ordered by an
unstable sort in the reference, so there the areas are compared by document id.  The problems are dense in positions (short documents,
up to 12 positions per posting), so that Concat, duplicate words and ring overwrites are frequent."""
import ctypes as C

import numpy as np
import pytest
from ft_helpers import add_random_synonyms, assert_same_merge, corpus_problem, cut_limit, planted_scores, preselect_plan, random_problem, \
    score_problem

import reindexer_b200 as rx
from oracle import ft_areas_oracle as FA
from oracle import ft_oracle as F

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not FA.ref_available(), reason="needs oracle/_ref (the reference's own merger)")]
ALL_RST = (F.RANK_AND_ID, F.RANK_ONLY, F.ID_ONLY, F.ID_AND_POSITIONS)
AS = (1, 2, 3, 5, 64)


def token_problem(seed, total_docs=300, nfields=3, vocab=12, nterms=3, ops=None, removed_frac=0.0, excluded_frac=0.0, zero_boost=False,
                  max_len=12):
    """A phrase-free query over an actual token corpus: every field of every document holds 1..max_len words of a small vocabulary, the
    posting lists are derived from it, so the words of one query stand next to each other and their areas touch.  Each term holds its
    word and maybe a variant (another word, lower proc); the parts are OR / AND / NOT."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, max_len + 1, size=(total_docs, nfields))
    lens[0] = 0
    removed = (rng.random(total_docs) < removed_frac).astype(np.uint8) if removed_frac else None
    excluded = (rng.random(total_docs) < excluded_frac).astype(np.uint8) if excluded_frac else None
    p = F.FtProblem(total_docs, lens.astype(np.uint32), removed=removed, excluded=excluded)
    tokens = [[rng.integers(0, vocab, size=lens[d, f]) for f in range(nfields)] for d in range(total_docs)]
    cache = {}

    def postings(w):
        if w not in cache:
            docs, pos_lists = [], []
            for d in range(1, total_docs):
                pp = [(int(i), f) for f in range(nfields) for i in np.nonzero(tokens[d][f] == w)[0]]
                if pp:
                    docs.append(d)
                    pos_lists.append(pp)
            cache[w] = p.add_list(docs, pos_lists)
        return cache[w]

    for t in range(nterms):
        subs = [(postings(int(rng.integers(0, vocab))), float(rng.choice([100.0, 90.0])))]
        if rng.random() < 0.5:
            subs.append((postings(int(rng.integers(0, vocab))), float(rng.choice([72.0, 57.0]))))
        op = ops[t] if ops else (F.OP_OR if t == 0 else int(rng.choice([F.OP_OR, F.OP_OR, F.OP_AND, F.OP_NOT])))
        fb = rng.choice([1.0, 0.5, 2.0], size=nfields).astype(np.float32)
        if zero_boost and nfields > 1:
            fb[int(rng.integers(0, nfields))] = 0.0
        p.add_term(subs, op=op, boost=float(rng.choice([1.0, 0.8, 1.3])), term_len_boost=float(rng.choice([1.0, 0.9])), field_boosts=fb)
    return p


def gpu_areas(p, runs, packed=False, batch=False):
    """one device index for the problem; runs: (A, rank_sort_type) pairs.  Returns [(infos, begin, areas, raw, plain)] where plain is
    rxgpu_ft_merge_query's result on the same index right after the areas call"""
    ft = rx.GpuFtIndex(p.total_docs, p.words, p.avg, p.removed)
    try:
        if packed:
            streams = [F.ref_pack_list(*l) for l in p.lists]
            if batch:
                ids = ft.add_postings_packed_batch(streams, [len(l[0]) for l in p.lists])
            else:
                ids = [ft.add_postings_packed(streams[i], len(p.lists[i][0])) for i in range(len(p.lists))]
        else:
            ids = [ft.add_postings(d, b, q) for d, b, q in p.lists]
        terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in p.terms]
        syns = [[dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in syn] for syn in p.synonyms]
        out = []
        for A, rst in runs:
            res = ft.merge_areas(p.cfg, p.field_cfg, terms, max_areas_in_doc=A, excluded=p.excluded, rank_sort_type=rst, synonyms=syns or None)
            plain = ft.merge(p.cfg, p.field_cfg, terms, excluded=p.excluded, rank_sort_type=rst, synonyms=syns or None)
            out.append(res + (plain,))
        return out
    finally:
        ft.close()


def same_bits(a, b):
    return len(a) == len(b) and (a["id"] == b["id"]).all() and (a["proc"].view(np.uint32) == b["proc"].view(np.uint32)).all() and \
        (a["field"] == b["field"]).all() and (a["normalized_proc"] == b["normalized_proc"]).all()


def per_entry(infos, begin, areas, nf):
    return [[areas[begin[i * nf + f]:begin[i * nf + f + 1]].tolist() for f in range(nf)] for i in range(len(infos))]


def assert_same_areas(p, ref, got, rst, ctx):
    ri, rb, ra, rr, _ = ref
    gi, gb, ga, gr, plain = got
    assert same_bits(gi, plain), (ctx, "areas call and plain merge differ")
    assert_same_merge(ri, gi, rst, ctx=ctx)
    nf = p.nfields
    if rst in (F.RANK_AND_ID, F.ID_ONLY):
        assert same_bits(ri, gi), ctx
        assert (rb == gb).all() and (ra == ga).all() and (rr == gr).all(), (ctx, per_entry(ri, rb, ra, nf)[:3], per_entry(gi, gb, ga, nf)[:3])
    else:
        want = {int(d): (a, int(r)) for d, a, r in zip(ri["id"], per_entry(ri, rb, ra, nf), rr)}
        have = {int(d): (a, int(r)) for d, a, r in zip(gi["id"], per_entry(gi, gb, ga, nf), gr)}
        assert want == have, ctx


def check(p, runs, packed=False, batch=False, ctx=""):
    got = gpu_areas(p, runs, packed=packed, batch=batch)
    for (A, rst), g in zip(runs, got):
        ref = FA.ref_merge_areas(p, A, rst, packed=packed)
        assert_same_areas(p, ref, g, rst, ctx=f"{ctx} A={A} rst={rst}")
    return got


# ---- the grid -------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nfields", [1, 3, 64])
@pytest.mark.parametrize("A", AS)
def test_token_corpus(A, nfields):
    """OR / AND / NOT over a token corpus; removed and excluded documents, a zero field boost, all three BM25 types, min_rank"""
    for seed in range(10):
        p = token_problem(7000 + 100 * A + 10 * nfields + seed, total_docs=200 if nfields == 64 else 300, nfields=nfields,
                          vocab=8 if nfields == 64 else 12, nterms=1 + seed % 3, removed_frac=0.1 if seed % 4 == 1 else 0.0,
                          excluded_frac=0.15 if seed % 4 == 2 else 0.0, zero_boost=seed % 4 == 3, max_len=6 if nfields == 64 else 12)
        p.cfg["bm25_type"] = seed % 3
        p.cfg["min_rank"] = (0, 5, 30)[seed % 3]
        check(p, [(A, ALL_RST[seed % 4])], ctx=f"token seed {seed} nfields {nfields}")


@pytest.mark.parametrize("A", AS)
def test_dense_random_problems(A):
    """random_problem with up to 12 positions per posting in documents of 2..14 words, with OR / AND / NOT"""
    for seed in range(10):
        nf = (1, 3)[seed % 2]
        p = random_problem(500 + 10 * A + seed, total_docs=250, nfields=nf, nterms=1 + seed % 4, max_sub=3, density=0.3, max_pos=12,
                           doc_len=(2, 14), field_boost_zero=seed % 3 == 0, removed_frac=0.05 * (seed % 2), excluded_frac=0.05 * (seed % 3 == 1))
        check(p, [(A, F.RANK_AND_ID), (A, F.RANK_ONLY)] if seed % 2 else [(A, F.ID_ONLY)], ctx=f"dense seed {seed}")


@pytest.mark.parametrize("A", AS)
def test_multi_word_synonyms(A):
    """multi-word synonyms, some with a suppressed subterm that repeats a word of the query (ft_suppressed_pass adds no areas); documents
    holding part of a synonym leave the result and take their areas with them"""
    for seed in range(8):
        p = random_problem(900 + 10 * A + seed, total_docs=300, nfields=(1, 3)[seed % 2], nterms=1 + seed % 3, max_sub=2, density=0.25,
                           max_pos=10, doc_len=(2, 14), ops=[F.OP_OR, F.OP_AND if seed % 2 else F.OP_OR, F.OP_NOT])
        add_random_synonyms(p, seed, nsyn=1 + seed % 2)
        check(p, [(A, F.RANK_AND_ID), (A, F.ID_AND_POSITIONS)], ctx=f"synonyms seed {seed}")


@pytest.mark.parametrize("mode", ["idrelvec", "packed", "packed_batch"])
def test_posting_containers(mode):
    """IdRelVec, PackedIdRelVec uploaded through the host decoder, and packed streams decoded on the device"""
    for seed in range(10):
        p = token_problem(3000 + seed, total_docs=300, nfields=(1, 3)[seed % 2], nterms=1 + seed % 3)
        check(p, [(AS[seed % 5], F.RANK_AND_ID)], packed=mode != "idrelvec", batch=mode == "packed_batch", ctx=f"{mode} seed {seed}")


def test_merge_limit_cut_mid_pass():
    """merge_limit below the documents of the first pass: ft_assign's cut drops documents in the middle of a pass, and they get no
    areas from later passes either"""
    for seed in range(10):  # one term (mergeSimple, never preselected) or two and three (mergeTerm, the preselect may run first)
        p = token_problem(4000 + seed, total_docs=400, nfields=3, nterms=1 if seed % 2 == 0 else 2 + seed % 4 // 2, ops=[F.OP_OR] * 3)
        first = len(p.lists[int(p.terms[0]["postings"][0])][0])
        p.cfg["merge_limit"] = max(1, first // 2 + seed)
        got = check(p, [(AS[seed % 5], F.RANK_AND_ID)], ctx=f"cut seed {seed}")
        assert len(got[0][0]) <= p.cfg["merge_limit"]


def test_min_rank_swap_removal():
    """min_rank drops entries with the reference's swap-removal: the areas must follow the entries that move"""
    for seed in range(10):
        p = random_problem(4500 + seed, total_docs=300, nfields=3, nterms=3, max_sub=2, density=0.3, max_pos=12, doc_len=(2, 14),
                           ops=[F.OP_OR, F.OP_OR, F.OP_OR])
        ref, _ = F.ref_merge(p)
        p.cfg["min_rank"] = int(np.percentile(ref["proc"], 50)) if len(ref) else 5  # half of the documents fall below
        check(p, [(AS[seed % 5], F.RANK_AND_ID), (AS[seed % 5], F.RANK_ONLY)], ctx=f"min_rank seed {seed}")


@pytest.mark.parametrize("preselect", [True, False])
def test_preselect_shapes(preselect):
    """the preselect keeps the merge_limit best documents, the threshold's documents cut in the middle of a mask word; without it
    (merge_limit = popcount) every document merges"""
    n = 6000
    thr = 300
    s = planted_scores(n, 17, 2000, thr, run_start=2000, run_len=900, frac=0.3, above=0.05)
    cut_id = int(np.nonzero(s == thr)[0][400])
    p = score_problem(s, seed=17, merge_limit=cut_limit(s, thr, cut_id), max_pos=12)
    p.cfg["min_rank"] = 0
    if not preselect:
        p.cfg["merge_limit"] = preselect_plan(p)["popcount"]
    plan = preselect_plan(p)
    assert plan["preselect"] == preselect
    for A in (1, 5):
        got = check(p, [(A, F.RANK_AND_ID), (A, F.ID_ONLY)], ctx=f"preselect {preselect}")
        assert len(got[0][0]) > 0


def test_empty_results():
    """no posting survives: every document excluded, a NOT-only query, an AND of disjoint words, an empty list"""
    p = token_problem(5000, total_docs=100, nfields=2, nterms=2, ops=[F.OP_OR, F.OP_OR])
    p.excluded = np.ones(p.total_docs, np.uint8)
    got = check(p, [(5, F.RANK_AND_ID)], ctx="all excluded")
    assert len(got[0][0]) == 0 and got[0][1].tolist() == [0]
    q = token_problem(5001, total_docs=100, nfields=2, nterms=1, ops=[F.OP_NOT])
    assert len(check(q, [(5, F.RANK_AND_ID)], ctx="not only")[0][0]) == 0
    r = F.FtProblem(10, np.full((10, 1), 5, np.uint32))
    r.add_term([(r.add_list([1, 2], [[(0, 0)], [(1, 0)]]), 100.0)], op=F.OP_AND)
    r.add_term([(r.add_list([3, 4], [[(0, 0)], [(1, 0)]]), 100.0)], op=F.OP_AND)
    assert len(check(r, [(3, F.RANK_AND_ID)], ctx="disjoint and")[0][0]) == 0
    e = F.FtProblem(10, np.full((10, 1), 5, np.uint32))
    e.add_term([(e.add_list(np.zeros(0, np.uint32), []), 100.0)])
    assert len(check(e, [(3, F.RANK_AND_ID)], ctx="empty list")[0][0]) == 0


def test_corpus_problems_without_phrases():
    """corpus_problem's queries with every phrase taken apart into plain terms: words that stand next to each other in real documents,
    variants listed before their word, and synonyms"""
    for seed in range(12):
        p = corpus_problem(6000 + seed, total_docs=300, nfields=2, vocab=10, with_synonym=True)
        p.terms = [dict(t, phrase_num=0, distance=0) for t in p.terms]
        check(p, [(AS[seed % 5], F.RANK_AND_ID)], ctx=f"corpus seed {seed}")


# ---- boundaries -----------------------------------------------------------------------------------------------------------------------
def raw_call(ft, p, terms, A, max_out=64):
    """rxgpu_ft_merge_query_areas with sentinel-filled outputs; returns (rc, outputs)"""
    c, arr, keep = ft._config_and_terms(p.cfg, p.field_cfg, terms)
    q = ft._query(arr, len(terms), [], keep)
    infos = np.full(max_out * 12, 0x5A, np.uint8)  # rxgpu_ft_merge_info[max_out] as raw bytes
    begin = np.full(max_out * p.nfields + 1, 0xDEADBEEF, np.uint32)
    areas = np.full((max(max_out * p.nfields * 64, 1), 2), 0xDEADBEEF, np.uint32)
    raw = np.full(max_out, 0xDEADBEEF, np.uint32)
    n = C.c_uint64(777)
    u32p = C.POINTER(C.c_uint32)
    rc = ft._lib.rxgpu_ft_merge_query_areas(ft._h, C.byref(c), C.byref(q), None, F.RANK_AND_ID, A, max_out, infos.ctypes.data,
                                            begin.ctypes.data_as(u32p), areas.ctypes.data, raw.ctypes.data_as(u32p), C.byref(n))
    return rc, (infos, begin, areas, raw, n.value)


def untouched(outs):
    infos, begin, areas, raw, n = outs
    return n == 777 and (infos == 0x5A).all() and (begin == 0xDEADBEEF).all() and (areas == 0xDEADBEEF).all() and \
        (raw == 0xDEADBEEF).all()


def test_refused_calls_change_nothing_and_leave_the_merge_intact():
    p = token_problem(8000, total_docs=200, nfields=3, nterms=3, ops=[F.OP_OR, F.OP_AND, F.OP_OR])
    ft = rx.GpuFtIndex(p.total_docs, p.words, p.avg, p.removed)
    try:
        ids = [ft.add_postings(d, b, q) for d, b, q in p.lists]
        terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in p.terms]
        before = ft.merge(p.cfg, p.field_cfg, terms)
        assert len(before) > 0
        for A in (0, 65, -1):
            rc, outs = raw_call(ft, p, terms, A)
            assert rc == 3, (A, rc)  # errParams
            assert untouched(outs), A
            assert same_bits(ft.merge(p.cfg, p.field_cfg, terms), before), A
        phrase = [dict(t, phrase_num=1 if i < 2 else 0, distance=1 if i == 1 else 0, op=F.OP_OR) for i, t in enumerate(terms)]
        rc, outs = raw_call(ft, p, phrase, 5)
        assert rc == 3 and untouched(outs)
        with pytest.raises(rx.RxGpuError) as e:
            ft.merge_areas(p.cfg, p.field_cfg, phrase, max_areas_in_doc=5)
        assert e.value.code == 3
        assert same_bits(ft.merge(p.cfg, p.field_cfg, terms), before)
        for A in AS:  # an areas call leaves the plain merge's scratch as it found it
            infos, begin, areas, raw = ft.merge_areas(p.cfg, p.field_cfg, terms, max_areas_in_doc=A)
            assert same_bits(infos, before), A
            assert same_bits(ft.merge(p.cfg, p.field_cfg, terms), before), A
            ref = FA.ref_merge_areas(p, A)
            assert (ref[1] == begin).all() and (ref[2] == areas).all() and (ref[3] == raw).all(), A
        # max_out below the result: the first max_out entries and their areas
        full = ft.merge_areas(p.cfg, p.field_cfg, terms, max_areas_in_doc=3)
        cut = ft.merge_areas(p.cfg, p.field_cfg, terms, max_areas_in_doc=3, max_out=5)
        assert same_bits(cut[0], full[0][:5]) and (cut[1] == full[1][:5 * 3 + 1]).all() and (cut[2] == full[2][:cut[1][-1]]).all()
        assert (cut[3] == full[3][:5]).all()
    finally:
        ft.close()
