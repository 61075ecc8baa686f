"""GPU tests of the batched HNSW range search (rxgpu_hnsw_search_range_batch, reindexer_b200/csrc/hnsw.cu).

Every query of a batch must come back bit-identical to its own rxgpu_hnsw_search_range call: labels, distance bits and out_n.
On the synthetic graphs of test_hnsw_exact_gpu.py the exact scan's table gives every distance the kernels see, so each returned
distance must equal its table entry, and every query whose ef-search took no decision between equal distances must return the
replay of the reference's SearchRange (tests/hnsw_replay.py).  On graphs built by the reference's CPU code the batch must return
the reference's set wherever the seeds agree."""
import numpy as np
import pytest
from helpers import ATOL, RTOL, prep_query
from hnsw_replay import search_range
from test_hnsw_exact_gpu import delete, fp32_table, make_index, random_graph, rows_for, rows_of, run_knn, slots_with_one_cta_per_sm

import reindexer_b200 as rx
from oracle import oracle as O
from reindexer_b200 import binding as B

pytestmark = pytest.mark.gpu

F = np.float32
METRICS = [rx.L2, rx.IP, rx.COS]
MNAME = {rx.L2: "l2", rx.IP: "ip", rx.COS: "cos"}


def same_as_single(gpu, queries, radii, ef, max_out, D, L, N, ctx=""):
    """row q of the batch == rxgpu_hnsw_search_range(queries[q], radii[q], ef, max_out); singles are cached by query row"""
    cache = {}
    for q in range(len(queries)):
        key = (queries[q].tobytes(), F(radii[q]).tobytes())
        if key not in cache:
            cache[key] = gpu.hnsw_search_range(queries[q], float(radii[q]), ef, max_out)
        d, lab, n = cache[key]
        m = min(n, max_out)
        assert int(N[q]) == n, (ctx, q, int(N[q]), n)
        assert (L[q, :m] == lab).all(), (ctx, q, L[q, :m][:8], lab[:8])
        assert (D[q, :m].view(np.uint32) == d.view(np.uint32)).all(), (ctx, q)


def halfway(table_q, i):
    """a radius strictly between the i-th and (i+1)-th distinct table distances: no comparison depends on rounding"""
    srt = np.unique(table_q)
    r = F((np.float64(srt[i]) + np.float64(srt[i + 1])) / 2)
    assert srt[i] < r < srt[i + 1]
    return r


# ---------------------------------------------------------------------------------------------------------------- replay


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("share", [0.0, 0.3])
def test_batch_matches_replay_and_single_calls(metric, share):
    """one batch mixes -inf, 0, a radius between two table distances, +inf and NaN; every max_out from 0 to a whole answer"""
    dim, n = 12, 2500
    rows = rows_for(metric, 51, n, dim)
    g = random_graph(51, n, 20, M=10, maxlevel=2, fill="mixed")
    gpu = make_index(metric, rows, g)
    base = rows_for(metric, 52, 6, dim)
    table = fp32_table(gpu, metric, rows, base)
    deleted = delete(gpu, n, np.nonzero(np.random.default_rng(53).random(n) < share)[0]) if share else frozenset()
    pick, radii = [], []
    for q in range(len(base)):
        for r in (-np.inf, 0.0, halfway(table[q], 40), np.inf, np.nan):
            pick.append(q)
            radii.append(r)
    pick, radii = np.array(pick), np.array(radii, F)
    queries = base[pick]
    for ef in (1, 32):
        reps = [search_range(g, lambda ids, q=q: table[q][ids], radii[i], ef, deleted) for i, q in enumerate(pick)]
        totals = [len(r.top) for r in reps]
        some = next((t for t, r in zip(totals, radii) if np.isfinite(r) and t > 1), 2)  # a bounded answer
        for max_out in sorted({0, 1, some - 1, some, max(totals) - 1, max(totals)}):
            D, L, N = gpu.hnsw_search_range_batch(queries, radii, ef, max_out)
            ctx = (MNAME[metric], share, ef, max_out)
            for i, q in enumerate(pick):
                m = min(int(N[i]), max_out)
                rows_q = rows_of(L[i, :m])
                assert (D[i, :m].view(np.uint32) == table[q, rows_q].view(np.uint32)).all(), (ctx, i)
                assert not (set(rows_q.tolist()) & deleted), (ctx, i)
                if np.isnan(radii[i]) or radii[i] == -np.inf:
                    assert N[i] == 0, (ctx, i)
                if reps[i].tie:
                    continue
                assert N[i] == totals[i], (ctx, i, N[i], totals[i])
                assert (rows_q == np.array([v for _, v in reps[i].top[:max_out]], np.int64)).all(), (ctx, i)
            same_as_single(gpu, queries, radii, ef, max_out, D, L, N, ctx)


# ---------------------------------------------------------------------------------------------------------------- reference


@pytest.mark.skipif(not O.ref_knn_available(), reason="needs oracle/_ref (reference HNSW build)")
@pytest.mark.parametrize("metric,dim", [(rx.L2, 48), (rx.IP, 64), (rx.COS, 96)])
def test_batch_matches_reference(metric, dim):
    n, ef, nq = 15000, 64, 40
    vecs, labels = O.synth_matrix(1300 + metric, n, dim), O.row_labels(n)
    ref = O.RefHnsw(metric, dim, n, M=16, ef_construction=200, seed=100, multithread=False)
    ref.add_batch(labels, vecs)
    g = ref.export(with_vectors=False)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(labels, vecs)
    gpu.hnsw_import(g)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(1400 + metric, nq, dim)])
    db, lb, _ = gpu.search_knn(queries, 201)
    js = np.array([[3, 40, 120, 200][i % 4] for i in range(nq)])
    radii = np.array([(np.float64(db[i, j - 1]) + np.float64(db[i, j])) / 2 for i, j in enumerate(js)], F)
    D, L, N = gpu.hnsw_search_range_batch(queries, radii, ef, n)
    same_as_single(gpu, queries, radii, ef, n, D, L, N, "reference graph")
    same = 0
    for i in range(nq):
        m = int(N[i])
        d, lab = D[i, :m], L[i, :m]
        dr, lr, tr = ref.search_range(queries[i], float(radii[i]), ef)
        assert (np.diff(d) >= 0).all() and (d < radii[i]).all()
        assert set(lab.tolist()) <= set(lb[i, :js[i]].tolist()), "a result outside the exact radius ball"
        if m == tr and (lab == lr).all():
            same += 1
            assert np.allclose(d, dr, rtol=RTOL, atol=ATOL)
    assert same >= nq - 2, (same, nq)
    assert N.max() >= 20, N  # the expansion really found neighbourhoods, not just seeds


# ---------------------------------------------------------------------------------------------------------------- independence


def test_queries_are_independent():
    """copies of one query and queries with overlapping closures: a shared or stale visited bitmap would drop nodes from some copies"""
    metric, dim, n = rx.L2, 10, 3000
    rows = rows_for(metric, 81, n, dim)
    g = random_graph(81, n, 32, M=16, maxlevel=2)
    gpu = make_index(metric, rows, g)
    rng = np.random.default_rng(82)
    near = (rows[7] + rng.standard_normal((20, dim)).astype(F) * 0.05).astype(F)  # closures around one row overlap
    queries = np.concatenate([np.repeat(rows[11:12], 40, axis=0), near, np.repeat(near[:3], 10, axis=0)])
    table = fp32_table(gpu, metric, rows, queries)
    radii = np.array([halfway(table[q], 150) for q in range(len(queries))], F)
    for ef in (1, 16):
        D, L, N = gpu.hnsw_search_range_batch(queries, radii, ef, 200)
        assert N.max() > 50, N
        for q in range(1, 40):
            assert N[q] == N[0] and (L[q] == L[0]).all() and (D[q].view(np.uint32) == D[0].view(np.uint32)).all(), (ef, q)
        for c in range(3):
            for j in range(10):
                q = 60 + c * 10 + j
                assert N[q] == N[40 + c] and (L[q] == L[40 + c]).all(), (ef, q)
        same_as_single(gpu, queries, radii, ef, 200, D, L, N, ("independent", ef))
        reps = [search_range(g, lambda ids, q=q: table[q][ids], radii[q], ef) for q in range(40, 60)]
        for q, rep in zip(range(40, 60), reps):
            if not rep.tie:
                assert N[q] == len(rep.top) and (rows_of(L[q, :min(N[q], 200)]) == [v for _, v in rep.top[:200]]).all(), (ef, q)


# ---------------------------------------------------------------------------------------------------------------- shapes


def test_batch_sizes():
    metric, dim, n = rx.IP, 16, 2000
    rows = rows_for(metric, 91, n, dim)
    g = random_graph(91, n, 24, M=12, maxlevel=2)
    gpu = make_index(metric, rows, g)
    base = rows_for(metric, 92, 33, dim)
    table = fp32_table(gpu, metric, rows, base)
    radii = np.array([halfway(table[q], 30 + q) for q in range(len(base))], F)
    for nq in (0, 1, 2, 31, 32, 33):
        D, L, N = gpu.hnsw_search_range_batch(base[:nq], radii[:nq], 8, 64)
        assert D.shape == (nq, 64) and N.shape == (nq,)
        same_as_single(gpu, base[:nq], radii[:nq], 8, 64, D, L, N, nq)


def test_batch_spanning_several_chunks(monkeypatch):
    """with one CTA per SM the bitmaps (one per query of a chunk) are fewer than the queries: the batch runs in several chunks"""
    slots = slots_with_one_cta_per_sm(monkeypatch)
    metric, dim, n = rx.L2, 12, 5000
    rows = rows_for(metric, 3, n, dim)
    g = random_graph(3, n, 48, M=24, maxlevel=3)
    gpu = make_index(metric, rows, g)
    base = rows_for(metric, 4, 16, dim)
    table = fp32_table(gpu, metric, rows, base)
    radii = np.array([halfway(table[q], 20 + 17 * q) for q in range(len(base))], F)
    nq = 2 * slots + 7
    pick = np.arange(nq) % len(base)
    D, L, N = gpu.hnsw_search_range_batch(base[pick], radii[pick], 24, 300)
    same_as_single(gpu, base[pick], radii[pick], 24, 300, D, L, N, "chunks")
    assert rx.last_search_stats()["passes"] >= 3  # three chunks, each at least one level


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("dim", [1, 127, 128, 129, 1000, 2048])
def test_dimensions(metric, dim):
    n = 1000 if dim >= 1000 else 2000
    rows = rows_for(metric, dim, n, dim, zero_rows=2)
    g = random_graph(dim + 10 * metric, n, 32, M=16, maxlevel=3)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, dim + 1, 12, dim)
    table = fp32_table(gpu, metric, rows, queries)
    radii = np.array([halfway(table[q], 25) if len(np.unique(table[q])) > 26 else np.inf for q in range(len(queries))], F)
    D, L, N = gpu.hnsw_search_range_batch(queries, radii, 16, 100)
    for q in range(len(queries)):
        rows_q = rows_of(L[q, :min(N[q], 100)])
        assert (D[q, :len(rows_q)].view(np.uint32) == table[q, rows_q].view(np.uint32)).all(), (dim, q)
    same_as_single(gpu, queries, radii, 16, 100, D, L, N, dim)


def test_two_components_and_an_isolated_node():
    metric, dim, n = rx.L2, 16, 3000
    rows = rows_for(metric, 95, n, dim)
    g = random_graph(95, n, 16, M=8, maxlevel=2, fill="mixed", split=n // 3, isolated=True)
    gpu = make_index(metric, rows, g)
    queries = np.concatenate([rows_for(metric, 96, 8, dim), rows[[5, n // 3 + 5, n - 1]]])
    table = fp32_table(gpu, metric, rows, queries)
    radii = np.concatenate([[halfway(table[q], 60) for q in range(8)], [np.inf, np.inf, np.inf]]).astype(F)
    for ef in (1, 64):
        D, L, N = gpu.hnsw_search_range_batch(queries, radii, ef, n)
        same_as_single(gpu, queries, radii, ef, n, D, L, N, ef)
        for q in range(len(queries)):
            rep = search_range(g, lambda ids, q=q: table[q][ids], radii[q], ef)
            if not rep.tie:
                assert N[q] == len(rep.top) and (rows_of(L[q, :N[q]]) == [v for _, v in rep.top]).all(), (ef, q)
        assert N[8:].max() < n - 1 and n - 1 not in rows_of(L[8, :N[8]]).tolist()  # a +inf radius floods one component only


# ---------------------------------------------------------------------------------------------------------------- overflow


def test_overflowing_regions_are_answered_again():
    """a component of more than 4096 nodes under a +inf radius overflows its region (max_out 3 keeps it at 4096 entries): those
    queries are answered again without a bound; the other queries of the batch stay on the bounded path"""
    metric, dim, n = rx.L2, 8, 9000
    rows = rows_for(metric, 101, n, dim)
    g = random_graph(101, n, 16, M=8, maxlevel=2)
    gpu = make_index(metric, rows, g)
    base = rows_for(metric, 102, 6, dim)
    table = fp32_table(gpu, metric, rows, base, envelope=False)
    radii = np.array([np.inf, halfway(table[1], 30), np.inf, halfway(table[3], 90), np.inf, 0.0], F)
    want = [search_range(g, lambda ids, q=q: table[q][ids], radii[q], 16) for q in range(len(base))]
    comp = len(want[0].top)  # the enter point's component
    assert comp > 8192, comp  # more than a region holds at max_out 3 (4096 entries) and at max_out 4096 (8192)
    for max_out in (3, 4096):
        D, L, N = gpu.hnsw_search_range_batch(base, radii, 16, max_out)
        st = rx.last_search_stats()
        floods = [q for q in range(len(base)) if radii[q] == np.inf]
        assert all(N[q] == comp for q in floods), (N, comp)
        assert st["tc_fallbacks"] == len(floods), st
        for q in range(len(base)):
            if not want[q].tie:
                assert N[q] == len(want[q].top) and (rows_of(L[q, :min(N[q], max_out)]) == [v for _, v in want[q].top[:max_out]]).all()
        same_as_single(gpu, base, radii, 16, max_out, D, L, N, max_out)


# ---------------------------------------------------------------------------------------------------------------- maintenance


def test_after_mark_deleted_and_update():
    metric, dim, n = rx.IP, 16, 3000
    rows = rows_for(metric, 111, n, dim)
    g = random_graph(111, n, 24, M=12, maxlevel=2)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 112, 24, dim)
    table = fp32_table(gpu, metric, rows, queries)
    radii = np.array([halfway(table[q], 50) for q in range(len(queries))], F)
    deleted = delete(gpu, n, np.nonzero(np.random.default_rng(113).random(n) < 0.2)[0])
    # rewrite the level-0 lists of 200 nodes in place (the device copy is patched, not re-imported)
    rng = np.random.default_rng(114)
    nodes = rng.choice(n, 200, replace=False)
    g2 = dict(g, level0=g["level0"].copy())
    for v in nodes:
        cnt = int(rng.integers(1, 25))
        nb = rng.choice(np.delete(np.arange(n), v), cnt, replace=False)
        g2["level0"][v] = 0
        g2["level0"][v, 0] = cnt
        g2["level0"][v, 1:1 + cnt] = nb
    gpu.hnsw_update(g2, nodes, deleted=sorted(deleted))
    for ef in (1, 32):
        D, L, N = gpu.hnsw_search_range_batch(queries, radii, ef, 500)
        same_as_single(gpu, queries, radii, ef, 500, D, L, N, ef)
        for q in range(len(queries)):
            rep = search_range(g2, lambda ids, q=q: table[q][ids], radii[q], ef, deleted)
            assert not (set(rows_of(L[q, :min(N[q], 500)]).tolist()) & deleted)
            if not rep.tie:
                assert N[q] == len(rep.top) and (rows_of(L[q, :N[q]]) == [v for _, v in rep.top]).all(), (ef, q)


# ---------------------------------------------------------------------------------------------------------------- search state


def test_knn_after_range_batch_sees_clean_bitmaps(monkeypatch):
    """the closure borrows the search kernel's visited bitmaps: after range batches that clear them by their matches' lists and
    in full (an overflow), a KNN batch over every slot must still match the replay, and a range batch must repeat itself"""
    slots = slots_with_one_cta_per_sm(monkeypatch)
    metric, dim, n = rx.L2, 8, 6000
    rows = rows_for(metric, 121, n, dim)
    g = random_graph(121, n, 32, M=16, maxlevel=3)
    gpu = make_index(metric, rows, g)
    base = rows_for(metric, 122, 16, dim)
    table = fp32_table(gpu, metric, rows, base, envelope=False)
    radii = np.array([np.inf if q % 5 == 0 else halfway(table[q], 100) for q in range(len(base))], F)
    pick = np.arange(slots + 3) % len(base)
    first = gpu.hnsw_search_range_batch(base[pick], radii[pick], 32, 2)
    assert rx.last_search_stats()["tc_fallbacks"] > 0
    again = gpu.hnsw_search_range_batch(base[pick], radii[pick], 32, 2)
    for a, b in zip(first, again):
        assert (a.view(np.uint8) == b.view(np.uint8)).all()
    knn_pick = np.arange(3 * slots) % len(base)
    reps, _ = run_knn(gpu, g, table, base, 10, 200)
    d, lab, cnt = gpu.hnsw_search_knn(base[knn_pick], 10, 200)
    for i, q in enumerate(knn_pick):
        if not reps[q].tie:
            assert (rows_of(lab[i, :cnt[i]]) == [v for _, v in reps[q].top]).all(), i


# ---------------------------------------------------------------------------------------------------------------- errors


def test_errors():
    metric, dim, n = rx.L2, 8, 500
    rows = rows_for(metric, 131, n, dim)
    q = rows_for(metric, 132, 4, dim)
    plain = rx.GpuBruteforceSearch(metric, dim, n)
    plain.add_points(O.row_labels(n), rows)
    with pytest.raises(rx.RxGpuError) as e:
        plain.hnsw_search_range_batch(q, 1.0, 8, 10)
    assert e.value.code == 4 and "no HNSW graph" in e.value.what
    empty = rx.GpuBruteforceSearch(metric, dim, 10)
    D, L, N = empty.hnsw_search_range_batch(q, 1.0, 8, 10)
    assert (N == 0).all()
    gpu = make_index(metric, rows, random_graph(131, n, 8, M=4, maxlevel=1))
    lib = gpu._lib
    r = np.ones(4, F)
    d = np.zeros((4, 10), F)
    lab = np.zeros((4, 10), np.uint64)
    cnt = np.zeros(4, np.uint64)
    args = [B._p(q, B._f32p), B._p(r, B._f32p), 8, 10, B._p(d, B._f32p), B._p(lab, B._u64p), B._p(cnt, B._u64p)]
    for i in (0, 1, 4, 5, 6):
        bad = list(args)
        bad[i] = None
        assert lib.rxgpu_hnsw_search_range_batch(gpu._h, 4, *bad) == 3, i
    assert lib.rxgpu_hnsw_search_range_batch(gpu._h, 0, None, None, 8, 10, None, None, None) == 0
    assert lib.rxgpu_hnsw_search_range_batch(gpu._h, 4, args[0], args[1], 8, 0, None, None, args[6]) == 0  # counts only
    with pytest.raises(rx.RxGpuError, match="ef must be <= 1024"):
        gpu.hnsw_search_range_batch(q, 1.0, 1025, 10)
    D, L, N = gpu.hnsw_search_range_batch(q, 1.0, 0, 10)  # ef 0 is ef 1
    D1, L1, N1 = gpu.hnsw_search_range_batch(q, 1.0, 1, 10)
    assert (N == N1).all() and (L == L1).all()
