"""GPU tests of the ft_fast merge (rxgpu_ft_merge / rxgpu_ft_select) at the shape and value boundaries of its kernels, each compared
exactly (ids, order, field, proc bits, uint8 rank) with the reference's own merger (or the C port when oracle/_ref is absent).  Every
test also asserts that its problem reached the boundary it is named after: the preselect's scores, threshold and budget are computed
by the numpy restatement ft_helpers.preselect_plan, and the grid shapes from the device's SM count."""
import numpy as np
import pytest
from ft_helpers import (assert_same_merge, bulk_list, corpus_problem, cut_limit, gpu_merge, planted_scores, preselect_plan, random_words,
                        score_problem)
from test_ft_boundaries_pin import BOOSTS, boost_problem, saturating_u16, threshold_cases

import reindexer_b200 as rx
from oracle import ft_oracle as F

pytestmark = pytest.mark.gpu
ALL_RST = (F.RANK_AND_ID, F.RANK_ONLY, F.ID_ONLY)
needs_ref = pytest.mark.skipif(not F.ref_available(), reason="oracle/_ref not built (the C port does not restate phrases / packing)")


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def check(p, rsts=ALL_RST, preselected=None, ctx=""):
    for rst in rsts:
        a, _ = F.best_merge(p, rst)
        b, st = gpu_merge(p, rst)
        assert_same_merge(a, b, rst, ctx=f"{ctx} rst {rst}")
        if preselected is not None:
            assert st["preselected"] == int(preselected), (ctx, st)
    return a


def assert_cut_mid_word(plan):
    """the budget for the threshold's documents runs out inside a mask word: the last kept and the first dropped one share it"""
    eq, k = plan["eq"], plan["budget"]
    assert 0 < k < len(eq) and eq[k - 1] // 32 == eq[k] // 32, (k, len(eq))
    return int(eq[k - 1])


# ---- preselect ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1])
def test_preselect_threshold_walk(seed):
    """ft_score_pass caps and saturation, ft_hist's shared / global bins (scores 8191 / 8192), ft_pick_threshold over several
    1024-bin rounds, on the round edges top-1023 / top-1024, in the saturated top bin and down to score 1"""
    for name, p in threshold_cases(seed=seed):
        plan = preselect_plan(p)
        assert plan["preselect"]
        if name == "to_one":
            assert plan["min_score"] == 1 and plan["positive"] < plan["max_merged"] < plan["popcount"]
        else:
            assert_cut_mid_word(plan)
            gap = {"deep": 21000, "edge1023": 1023, "edge1024": 1024, "at8192": 12000 - 8192, "below8192": 1, "top": 0}[name]
            assert plan["top"] - plan["min_score"] == gap and plan["top"] >= 8192, name
            assert name != "at8192" or plan["min_score"] == 8192
            assert name != "below8192" or (plan["min_score"] == 8191 and plan["top"] == 8192)
        check(p, preselected=True, ctx=name)


def test_preselect_saturated_scores():
    """five capped terms (5 x 16383) saturate the u16 score at 65535; the threshold falls inside that bin"""
    rng = np.random.default_rng(3)
    n = 40000
    s = np.where(rng.random(n) < 0.2, rng.integers(1, 65535, size=n), 0)
    s[0] = 0
    sat = np.zeros(n, bool)
    sat[1000:1600] = True
    s[sat] = 0
    p = score_problem(s, saturated=sat, merge_limit=300)
    p.cfg["min_rank"] = 0
    plan = preselect_plan(p)
    assert plan["top"] == 65535 and plan["min_score"] == 65535 and plan["budget"] == 300 and (s == 65535).sum() <= 1
    check(p, preselected=True)


def test_preselect_decision_edges():
    """merge_limit = popcount - 1 (preselect), popcount and popcount + 1 (none), and an estimate above merge_limit with the popcount
    at or below it (excluded documents, an AND term)"""
    rng = np.random.default_rng(5)
    n = 5000
    s = np.where(rng.random(n) < 0.5, rng.integers(1, 3000, size=n), 0)
    s[0] = 0
    p = score_problem(s)
    p.cfg["min_rank"] = 0
    pop = preselect_plan(p)["popcount"]
    assert pop == n
    for ml, want in ((pop - 1, True), (pop, False), (pop + 1, False)):
        p.cfg["merge_limit"] = ml
        plan = preselect_plan(p)
        assert plan["estimate"] > pop - 1 and plan["preselect"] == want
        check(p, rsts=(F.RANK_AND_ID,), preselected=want, ctx=f"merge_limit {ml}")
    ex = (rng.random(n) < 0.5).astype(np.uint8)
    q = score_problem(s, excluded=ex)
    q.cfg.update(min_rank=0, merge_limit=int((ex == 0).sum()))
    plan = preselect_plan(q)
    assert plan["estimate"] > q.cfg["merge_limit"] >= plan["popcount"] and not plan["preselect"]
    check(q, rsts=(F.RANK_AND_ID,), preselected=False, ctx="excluded")


def test_preselect_cut_inside_block_chunks():
    """ft_thresh_count / ft_thresh_apply with a persistent grid of 4 x SMs blocks: more than pg x 256 mask words, so one block's chunk
    holds several 256-word steps; the budget runs out inside the second step of block 1's chunk, in the middle of a word, with
    threshold documents in block 0's chunk ahead of it"""
    pg = 4 * sm_count()
    words = pg * 256 * 2 + 300
    n = words * 32
    chunk = -(-(-(-words // pg)) // 256) * 256
    assert chunk >= 3 * 256
    cut_word = chunk + 256 + 100
    cut_id = cut_word * 32 + 13
    thr = 3000
    s = planted_scores(n, 11, 12000, thr, run_start=cut_id - 3000, run_len=6000, frac=0.004, above=0.004)
    s[5000:6000] = thr
    p = score_problem(s, seed=11, merge_limit=cut_limit(s, thr, cut_id))
    p.cfg["min_rank"] = 0
    plan = preselect_plan(p)
    assert plan["preselect"] and plan["min_score"] == thr and assert_cut_mid_word(plan) == cut_id
    assert words > pg * 256 and chunk + 256 <= cut_word < chunk + 512
    check(p, rsts=(F.RANK_AND_ID, F.ID_ONLY), preselected=True)


def test_out_of_range_boosts_convert_like_the_reference():
    """a term boost that takes subterm proc x boost below 0 or past 65536, 2^31 and 2^32: the preselect score is the reference
    build's static_cast<uint16_t> (cvttss2si, low 16 bits), not a saturating conversion"""
    for i, b in enumerate(BOOSTS):
        p = boost_problem(i, b)
        plan = preselect_plan(p)
        assert plan["preselect"]
        if b != 700.005:  # a saturating conversion would keep other documents
            sat = preselect_plan(p, to_u16=saturating_u16)
            assert not np.array_equal(plan["score"], sat["score"])
        check(p, rsts=(F.RANK_AND_ID, F.RANK_ONLY), preselected=True, ctx=f"boost {b}")


# ---- slot order and cut-off --------------------------------------------------------------------------------------------------------
def test_list_longer_than_one_scan_round():
    """a list of more than 8192 blocks of 256 postings: ft_scan_blocks carries between its rounds; ft_score_pass and ft_and_mark
    stride over more than 16 x SMs x 256 postings"""
    rng = np.random.default_rng(17)
    n = 2_500_000
    big = 8192 * 256 + 70_001
    assert big > 16 * sm_count() * 256
    words = random_words(rng, n, 1)
    p = F.FtProblem(n, words)
    docs = np.sort(rng.choice(np.arange(1, n), size=big, replace=False))
    lb = bulk_list(p, rng, docs, npos=rng.integers(1, 3, size=big))
    ls = bulk_list(p, rng, np.sort(rng.choice(np.arange(1, n), size=50_000, replace=False)), npos=2)
    p.add_term([(lb, 100.0)])
    p.cfg.update(merge_limit=3_000_000, min_rank=0)
    a = check(p, rsts=(F.RANK_AND_ID,), ctx="simple")
    assert len(a) == big and -(-big // 256) > 8192
    p.add_term([(ls, 90.0)], op=F.OP_OR)
    check(p, rsts=(F.RANK_AND_ID,), preselected=False, ctx="two terms")
    p.cfg["merge_limit"] = 100_000
    plan = preselect_plan(p)
    assert plan["preselect"]
    check(p, rsts=(F.RANK_AND_ID,), preselected=True, ctx="preselect")


@pytest.mark.parametrize("total", [1, 2, 32, 33])
def test_tiny_corpora_and_last_document(total):
    rng = np.random.default_rng(total)
    p = F.FtProblem(total, random_words(rng, total, 2))
    p.add_term([(bulk_list(p, rng, np.arange(total), npos=2), 100.0)], field_boosts=np.array([1.0, 2.0], np.float32))
    p.add_term([(bulk_list(p, rng, np.array([total - 1]), npos=1), 90.0)], op=F.OP_OR)
    p.cfg["min_rank"] = 0
    a = check(p)
    assert (total - 1) in a["id"].tolist()


@pytest.mark.parametrize("ndocs", [1, 255, 256, 257])
def test_list_lengths_around_a_block(ndocs):
    rng = np.random.default_rng(ndocs)
    n = 3000
    p = F.FtProblem(n, random_words(rng, n, 1))
    l1 = bulk_list(p, rng, np.sort(rng.choice(np.arange(1, n), size=ndocs, replace=False)), npos=rng.integers(1, 4, size=ndocs))
    l2 = bulk_list(p, rng, np.sort(rng.choice(np.arange(1, n), size=ndocs, replace=False)), npos=1)
    p.add_term([(l1, 100.0), (l2, 80.0)])
    p.add_term([(l2, 70.0)], op=F.OP_OR)
    p.cfg["min_rank"] = 0
    check(p, ctx="whole")
    for ml in (max(1, ndocs // 2), max(1, ndocs - 1), ndocs + 1):  # merge_limit ends a pass inside a block
        p.cfg["merge_limit"] = ml
        check(p, ctx=f"merge_limit {ml}")


def test_more_than_255_query_parts():
    """qp_idx, ext_cnt and ext_last_term are 16-bit: 300 query parts (OR, AND, NOT) over overlapping lists"""
    rng = np.random.default_rng(300)
    n = 4000
    p = F.FtProblem(n, random_words(rng, n, 1))
    common = np.sort(rng.choice(np.arange(1, n), size=1500, replace=False))
    for t in range(300):
        docs = np.union1d(common[:1200], rng.choice(np.arange(1, n), size=40, replace=False)).astype(np.uint32)
        op = F.OP_OR if t == 0 or t % 7 else (F.OP_AND if t % 2 else F.OP_NOT)
        p.add_term([(bulk_list(p, rng, docs if op != F.OP_NOT else docs[-3:], npos=1), float(100 - t % 50))], op=op)
    assert len(p.terms) > 255
    p.cfg["min_rank"] = 0
    check(p, rsts=(F.RANK_AND_ID, F.RANK_ONLY))
    p.cfg["merge_limit"] = 500
    check(p, rsts=(F.RANK_AND_ID,))


# ---- ranking -----------------------------------------------------------------------------------------------------------------------
POS_EDGES = [0, 10, 11, 100, 101, 1000, 1001, 10000, 10001, 100000, 100001, (1 << 24) - 1]


@pytest.mark.parametrize("nfields", [17, 33, 64])
def test_many_fields_and_position_edges(nfields):
    """pos2rank at each edge of its steps, fields 16 apart (PosType::fullField compares only 4 field bits in PositionsDistance),
    field boosts and field configs indexed up to 63, and documents with hundreds of positions of one term"""
    rng = np.random.default_rng(nfields)
    n = 3000
    p = F.FtProblem(n, random_words(rng, n, nfields, 5, 400))
    fb = rng.choice([0.0, 0.5, 1.0, 1.5, 2.0], size=nfields).astype(np.float32)
    fb[[0, 16, nfields - 1]] = [1.0, 2.0, 1.5]
    for f in range(nfields):
        p.field_cfg[f].update(bm25_weight=float(rng.uniform(0.05, 0.5)), position_weight=float(rng.uniform(0.05, 0.5)),
                              term_len_weight=0.3, bm25_boost=float(rng.uniform(0.8, 1.5)))
    docs = np.arange(1, n)
    first = np.asarray(POS_EDGES)[rng.integers(0, len(POS_EDGES), size=len(docs))]
    fields = rng.choice([0, 16, nfields - 1, nfields - 17, int(rng.integers(0, nfields))], size=len(docs)) % nfields
    heavy = rng.random(len(docs)) < 0.05
    npos = np.where(heavy, rng.integers(200, 400, size=len(docs)), rng.integers(1, 4, size=len(docs)))
    l0 = bulk_list(p, rng, docs, npos=npos, max_pos=400, fields=fields, first_pos=first)
    l1 = bulk_list(p, rng, docs[rng.random(len(docs)) < 0.6], npos=3, max_pos=30, fields=None)
    d2 = docs[rng.random(len(docs)) < 0.6]
    l2 = bulk_list(p, rng, d2, npos=2, max_pos=30, fields=(fields[d2 - 1] + 16) % nfields)  # the same positions 16 fields apart
    p.add_term([(l0, 100.0), (l1, 72.0)], field_boosts=fb)
    p.add_term([(l2, 90.0)], op=F.OP_OR, field_boosts=fb, boost=1.3)
    p.cfg.update(min_rank=0, distance_weight=0.5, distance_boost=1.5)
    assert (np.diff(p.lists[l0][1]) >= 200).any() and max(fields) >= 16
    check(p, rsts=(F.RANK_AND_ID, F.RANK_ONLY))
    p.cfg["merge_limit"] = 700
    check(p, rsts=(F.RANK_AND_ID,))
    # exactly 16 needSumRank fields are served; 17 are refused
    p.cfg.update(summation_ranks_by_fields_ratio=0.5, merge_limit=20000)
    ns = np.zeros(nfields, np.uint8)
    ns[rng.choice(nfields, size=16, replace=False)] = 1
    for t in p.terms:
        t["need_sum_rank"] = ns
    check(p, rsts=(F.RANK_AND_ID,), ctx="16 sum fields")
    ns17 = ns.copy()
    ns17[np.nonzero(ns == 0)[0][0]] = 1
    p.terms[0]["need_sum_rank"] = ns17
    with pytest.raises(rx.RxGpuError):
        gpu_merge(p)


@pytest.mark.parametrize("bm25_type", [0, 1, 2])
def test_zero_word_counts_and_bm25_knobs(bm25_type):
    """words_in_field = 0 and avg = 0 (inf / NaN inside BM25 in fp64), b = 0, b = 1, k1 = 0"""
    rng = np.random.default_rng(40 + bm25_type)
    n = 2000
    words = random_words(rng, n, 2)
    words[rng.random((n, 2)) < 0.2] = 0
    for avg in (None, np.array([0.0, 7.5], np.float32)):
        p = F.FtProblem(n, words, avg=avg)
        l0 = bulk_list(p, rng, np.sort(rng.choice(np.arange(1, n), size=900, replace=False)), npos=rng.integers(1, 5, size=900))
        l1 = bulk_list(p, rng, np.sort(rng.choice(np.arange(1, n), size=700, replace=False)), npos=2)
        p.add_term([(l0, 100.0)], field_boosts=np.array([1.0, 1.5], np.float32))
        p.add_term([(l1, 85.0)], op=F.OP_OR)
        for k1, b in ((2.0, 0.75), (2.0, 0.0), (2.0, 1.0), (0.0, 0.75)):
            p.cfg.update(bm25_type=bm25_type, bm25_k1=k1, bm25_b=b, min_rank=0)
            check(p, rsts=(F.RANK_AND_ID,), ctx=f"avg {avg} k1 {k1} b {b}")


# ---- post-processing and select ----------------------------------------------------------------------------------------------------
def test_scale_switch_min_rank_and_limits():
    """the largest proc exactly 255.0f and the next float above it (the scaling switch of postProcessResults), ranks exactly at
    min_rank, and select limits 0, 1, n and n + 1"""
    n = 400
    rng = np.random.default_rng(9)
    for top in (np.float32(255.0), np.nextafter(np.float32(255.0), np.float32(1e9))):
        p = F.FtProblem(n, random_words(rng, n, 1))
        procs = [float(top), 200.0, 100.0, float(np.nextafter(np.float32(100.0), np.float32(0))), 50.0, 7.0]
        sub = [(bulk_list(p, rng, np.arange(1 + 60 * k, 60 * (k + 1)), npos=1), pr) for k, pr in enumerate(procs)]
        p.add_term(sub)
        p.field_cfg[0].update(bm25_weight=0.0, position_weight=0.0, term_len_weight=0.0)  # every factor of the rank is 1
        for min_rank in (0, 100, 99):
            p.cfg["min_rank"] = min_rank
            a = check(p, rsts=(F.RANK_AND_ID, F.RANK_ONLY))
            # 255.0 keeps scalingFactor 1; the next float scales every proc by 255 / max
            assert a["proc"].max() == np.float32(255.0) and (a["proc"] == np.float32(200.0)).any() == (top == np.float32(255.0))
            # minRank filters the unscaled procs: a proc of exactly 100 stays and, scaled, ranks 99
            assert min_rank == 0 or a["normalized_proc"].min() == {100: 100 if top == np.float32(255.0) else 99, 99: 99}[min_rank]
        ft = rx.GpuFtIndex(p.total_docs, p.words, p.avg)
        ids = [ft.add_postings(*lst) for lst in p.lists]
        terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in p.terms]
        want = F.after_select_order(a)
        for limit in (0, 1, len(want), len(want) + 1):
            got_ids, got_ranks, tot = ft.select(p.cfg, p.field_cfg, terms, limit)
            m = min(limit, len(want))
            assert tot == len(want) and len(got_ids) == m
            assert (got_ids == want["id"][:m]).all() and (got_ranks == want["normalized_proc"][:m].astype(np.float32)).all()
        ft.close()


def test_sharded_select_with_high_preselect_scores():
    """rxgpu_sharded_ft_select with scores >= 8192 in the exchanged histogram and the threshold's documents cut inside a shard"""
    from test_ft_sharded_gpu import run_sharded, run_whole

    n, thr = 20000, 9000
    s = planted_scores(n, 21, 30000, thr, run_start=11000, run_len=400)
    p = score_problem(s, seed=21, merge_limit=cut_limit(s, thr, 11000 + 201))
    p.cfg["min_rank"] = 0
    plan = preselect_plan(p)
    assert plan["top"] >= 8192 and plan["min_score"] == thr and assert_cut_mid_word(plan) == 11201
    ref = F.after_select_order(F.best_merge(p)[0])
    for rst in (F.RANK_AND_ID, F.ID_ONLY):
        whole, st = run_whole(p, 5000, rst)
        assert st["preselected"] == 1 and whole[2] == len(ref)
        if rst == F.RANK_AND_ID:
            assert (whole[0] == ref["id"][:5000]).all()
        for bounds in ([0, 7000, 11100, n], [0, 11201, 11202, n]):
            for ids, ranks, tot in run_sharded(p, bounds, 5000, rst):
                assert tot == whole[2] and (ids == whole[0]).all() and (ranks == whole[1]).all(), bounds


# ---- phrases, packed lists, parameters ---------------------------------------------------------------------------------------------
@needs_ref
def test_phrase_proc_sum_limits():
    """the first-subterm procs of a phrase's terms must fit 16 bits: 65534 is served (and feeds ft_phrase_score under the preselect),
    65535 is refused"""
    served = preselected = 0
    for seed in range(12):
        p = corpus_problem(seed, total_docs=800, nfields=1 + seed % 2, merge_limit=30 if seed % 2 else 20000)
        phrase = [t for t in p.terms if t.get("phrase_num", 0) == 1]
        share = [65534 // len(phrase) + (1 if k < 65534 % len(phrase) else 0) for k in range(len(phrase))]
        for t, v in zip(phrase, share):
            t["procs"] = np.asarray([float(v)] + [float(x) for x in t["procs"][1:]], np.float32)
        assert sum(int(t["procs"][0]) for t in phrase) == 65534
        for rst in (F.RANK_AND_ID, F.RANK_ONLY):
            a, _ = F.ref_merge(p, rst)
            b, st = gpu_merge(p, rst)
            assert_same_merge(a, b, rst, ctx=f"seed {seed}")
        served += 1
        preselected += st["preselected"]
        phrase[0]["procs"] = phrase[0]["procs"] + np.float32(1.0)
        with pytest.raises(rx.RxGpuError):
            gpu_merge(p)
    assert served == 12 and preselected > 0


@needs_ref
def test_packed_batch_decoder_split():
    """rxgpu_ft_add_postings_packed_batch decodes lists of at most 256 KiB on the device and longer ones on the host: one list of
    exactly 262144 bytes and one of 262145 give the merges of the plain upload"""
    n = 400_000
    rng = np.random.default_rng(4)
    words = random_words(rng, n, 1, 300, 400)

    def stream(ndocs, k):
        d = np.arange(1, ndocs + 1, dtype=np.uint32)
        pos = np.full(ndocs, 5, np.uint32)
        pos[:k] = 300
        return (d, np.arange(ndocs + 1, dtype=np.uint32), pos), F.ref_pack_list(d, np.arange(ndocs + 1, dtype=np.uint32), pos)

    def exact(target):
        lo, hi = 1, n - 2
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if len(stream(mid, 0)[1]) <= target else (lo, mid - 1)
        for nd in range(lo, lo - 8, -1):
            for k in range(0, 400):
                soa, s = stream(nd, k)
                if len(s) == target:
                    return soa, s
                if len(s) > target:
                    break
        raise AssertionError(f"no stream of {target} bytes")

    lists = [exact(256 << 10), exact((256 << 10) + 1)]
    assert [len(s) for _, s in lists] == [262144, 262145]
    p = F.FtProblem(n, words)
    a = rx.GpuFtIndex(n, words, p.avg)
    ids = a.add_postings_packed_batch([s for _, s in lists], [len(soa[0]) for soa, _ in lists])
    for (soa, _), lid in zip(lists, ids):
        q = F.FtProblem(n, words)
        q.add_term([(q.add_list_arrays(*soa), 100.0)])
        q.cfg["min_rank"] = 0
        want, _ = F.best_merge(q)
        got = a.merge(q.cfg, q.field_cfg, [dict(q.terms[0], postings=[lid])])
        assert_same_merge(want, got, F.RANK_AND_ID)
        assert len(got) == min(len(soa[0]), q.cfg["merge_limit"])
    a.close()


def test_field_count_edges():
    words = np.ones((10, 64), np.uint32)
    rx.GpuFtIndex(10, words, np.ones(64, np.float32)).close()
    for nf in (0, 65):
        with pytest.raises(rx.RxGpuError):
            rx.GpuFtIndex(10, np.ones((10, nf), np.uint32), np.ones(max(nf, 1), np.float32))
