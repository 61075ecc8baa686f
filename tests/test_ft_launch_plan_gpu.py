"""The full-text merge's launch plan, pinned: a fixed sequence of calls on one fresh index (merge, merge with synonyms, with areas,
select, sharded select; plain, trivial, AND / OR / NOT, phrase, synonym and preselect queries) must report, after every call, the
kernel launches, the preselect decision, the postings scanned and the algorithmic bytes that tests/golden/ft_launch_plan.npz holds
(written by tests/golden/make_ft_launch_plan.py).  The other tests pin what the merge returns; this one catches a launch that is
dropped or doubled without changing a result.  The calls run in the recorded order: the first merge on an index also fills its slot
table (idoff), so what a call launches depends on the calls before it.  The selects whose row total is read back before the sort
(more possible keys than the device sorts without asking) also have their rows pinned: no other test reaches that path."""
import os

import numpy as np
import pytest
from ft_helpers import add_random_synonyms, corpus_problem, random_problem

from oracle import ft_oracle as F

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ft_launch_plan.npz")
FIELDS = ("launches", "preselected", "postings_scanned", "algorithmic_bytes")  # device_ms is a time, not part of the plan
T = 600  # documents of the index: every problem below is built over the same ids, its lists are added to the one index


def run_plan():
    """([(call name, [launches, preselected, postings_scanned, algorithmic_bytes])] in call order, {call name: (row ids, ranks, total)}
    of the selects that read the row total back first)"""
    import reindexer_b200 as rx

    simple = random_problem(3, total_docs=T, nfields=2, nterms=1, max_sub=3, removed_frac=0.05)
    trivial = random_problem(2, total_docs=T, nfields=2, nterms=1, max_sub=1)
    ops = random_problem(3, total_docs=T, nfields=2, nterms=4, ops=[F.OP_OR, F.OP_AND, F.OP_NOT, F.OP_OR], excluded_frac=0.05,
                         field_boost_zero=True)
    presel = random_problem(4, total_docs=T, nfields=2, nterms=3, ops=[F.OP_OR] * 3, merge_limit=40, density=0.5)
    presel_and = random_problem(5, total_docs=T, nfields=2, nterms=3, ops=[F.OP_OR, F.OP_AND, F.OP_NOT], merge_limit=40, density=0.5)
    phrases = corpus_problem(6, total_docs=T, nfields=2)
    phrases_presel = corpus_problem(7, total_docs=T, nfields=2, merge_limit=30)
    phrases_syn = corpus_problem(9, total_docs=T, nfields=2, with_synonym=True)
    syn = add_random_synonyms(random_problem(9, total_docs=T, nfields=2, nterms=3, ops=[F.OP_OR, F.OP_AND, F.OP_OR]), 9)
    syn_presel = add_random_synonyms(random_problem(10, total_docs=T, nfields=2, nterms=3, ops=[F.OP_OR] * 3, merge_limit=40,
                                                    density=0.5), 10)
    assert len(simple.terms[0]["postings"]) > 1 and len(trivial.terms[0]["postings"]) == 1
    assert any(t["phrase_num"] for t in phrases.terms) and any(t["phrase_num"] for t in phrases_syn.terms) and phrases_syn.synonyms
    assert any(s.get("suppressed") is not None for y in syn.synonyms for s in y)

    ft = rx.GpuFtIndex(T, simple.words, simple.avg, simple.removed)

    def upload(p):
        ids = [ft.add_postings(d, b, q) for d, b, q in p.lists]
        remap = lambda ts: [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in ts]  # noqa: E731
        return p, remap(p.terms), [remap(y) for y in p.synonyms] or None

    q = {name: upload(p) for name, p in (("simple", simple), ("trivial", trivial), ("ops", ops), ("presel", presel),
                                         ("presel_and", presel_and), ("phrases", phrases), ("phrases_presel", phrases_presel),
                                         ("phrases_syn", phrases_syn), ("syn", syn), ("syn_presel", syn_presel))}
    status = (np.random.default_rng(11).random(T) < 0.8).astype(np.uint8)
    plan, rows = [], {}

    def merge(name, key, rank_sort_type=F.RANK_AND_ID):
        p, terms, syns = q[key]
        ft.merge(p.cfg, p.field_cfg, terms, excluded=p.excluded, rank_sort_type=rank_sort_type, synonyms=syns)
        record(name)

    def areas(name, key):
        p, terms, syns = q[key]
        ft.merge_areas(p.cfg, p.field_cfg, terms, max_areas_in_doc=3, excluded=p.excluded, synonyms=syns)
        record(name)

    def select(name, key, rank_sort_type=F.RANK_AND_ID, row_status=None):
        p, terms, syns = q[key]
        out = ft.select(p.cfg, p.field_cfg, terms, 50, excluded=p.excluded, row_status=row_status, rank_sort_type=rank_sort_type,
                        synonyms=syns)
        record(name)
        return out

    def sharded_select(name, key, row_status=None):
        p, terms, _ = q[key]
        out = ft.sharded_select(comm, 0, p.cfg, p.field_cfg, terms, 50, excluded=p.excluded, row_status=row_status)
        record(name)
        return out

    def record(name):
        st = ft.last_stats()
        plan.append((name, [int(st[f]) for f in FIELDS]))

    comm = None
    try:
        merge("simple", "simple")
        merge("simple_again", "simple")
        merge("trivial", "trivial")
        merge("and_or_not", "ops")
        merge("and_or_not_rank_only", "ops", F.RANK_ONLY)
        merge("preselect", "presel")
        merge("preselect_and_not", "presel_and")
        merge("phrases", "phrases")
        merge("phrases_preselect", "phrases_presel")
        merge("phrases_synonyms", "phrases_syn")
        merge("synonyms", "syn")
        merge("synonyms_preselect", "syn_presel", F.RANK_ONLY)
        areas("areas_simple", "simple")
        areas("areas_and_or_not", "ops")
        areas("areas_preselect", "presel")
        areas("areas_synonyms", "syn")
        select("select_trivial", "trivial")
        select("select", "ops")
        select("select_id_only", "presel", F.ID_ONLY)
        select("select_synonyms", "syn_presel")
        select("select_phrases", "phrases")
        select("select_row_status", "ops", row_status=status)
        p, terms, _ = q["ops"]
        ft.merge(p.cfg, p.field_cfg, [])
        record("empty_query")
        ft.merge(p.cfg, p.field_cfg, [dict(terms[2])])
        record("not_only")
        ft.merge(dict(p.cfg, merge_limit=0), p.field_cfg, terms, excluded=p.excluded)
        record("merge_limit_zero")
        (comm,) = rx.ShardComm.local_group(1)
        sharded_select("sharded_select", "ops")
        sharded_select("sharded_select_preselect", "presel")
        nrows = np.random.default_rng(12).integers(0, 3, size=T).astype(np.uint32)
        row_begin = np.concatenate([[0], np.cumsum(nrows)]).astype(np.uint32)
        ft.set_rows(row_begin, np.arange(int(row_begin[-1]), dtype=np.int32))
        select("select_rows_row_status", "ops", row_status=(np.arange(int(row_begin[-1])) % 5 != 0).astype(np.uint8))
        # document 1 owns 8192 rows: merged documents x rows per document exceeds 2^20 keys, so the row total is read back to size the sort
        nrows[1] = 8192
        row_begin = np.concatenate([[0], np.cumsum(nrows)]).astype(np.uint32)
        ft.set_rows(row_begin, np.arange(int(row_begin[-1]), dtype=np.int32))
        big_status = (np.arange(int(row_begin[-1])) % 7 != 0).astype(np.uint8)
        rows["select_read_back_first"] = select("select_read_back_first", "ops", row_status=big_status)
        rows["sharded_select_read_back_first"] = sharded_select("sharded_select_read_back_first", "ops", row_status=big_status)
    finally:
        if comm is not None:
            comm.close()
        ft.close()
    return plan, rows


def test_launch_plan_matches_golden():
    g = np.load(GOLDEN)
    plan, rows = run_plan()
    assert [n for n, _ in plan] == g["names"].tolist()
    got = np.array([s for _, s in plan], np.int64)
    diff = [(n, dict(zip(FIELDS, got[i].tolist())), dict(zip(FIELDS, g["stats"][i].tolist()))) for i, (n, _) in enumerate(plan)
            if (got[i] != g["stats"][i]).any()]
    assert not diff, diff
    for name, (ids, ranks, n) in rows.items():
        assert n == g[f"{name}/n"] and (ids == g[f"{name}/ids"]).all() and (ranks == g[f"{name}/ranks"]).all(), name
