"""GPU tests of the batched range search (rxgpu_search_range_batch).  On the tensor-core filter path every query's answer must equal
rxgpu_search_range for that query alone: the same total, the same distance bits and the same label order, with the filter deciding
the ordinary queries itself rather than handing them to the exact scan."""
import ctypes as C
import functools

import numpy as np
import pytest
from helpers import ATOL, RTOL, prep_query

import reindexer_b200 as rx
from reindexer_b200 import binding as B
from oracle import oracle as O

pytestmark = pytest.mark.gpu

RANKS = (1, 10, 100, 1000)


@functools.lru_cache(maxsize=2)
def synth_rows(n, dim, seed):
    rows = O.synth_matrix(seed, n, dim)
    rows[n - 300:] = rows[:300]  # duplicated rows: equal distances under different labels
    return rows


def make_index(metric, rows, labels, extra_capacity=0):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], len(rows) + extra_capacity)
    gpu.add_points(labels, rows)
    return gpu


def make_queries(metric, seed, nq, dim):
    q = O.synth_matrix(seed, nq, dim)
    return np.stack([prep_query(metric, x) for x in q]) if metric == rx.COS else q


def exact_knn_dists(gpu, queries, k):
    gpu.set_tensor_core_filter(2)
    d, _, c = gpu.search_knn(queries, k)
    assert (c == k).all()
    return d


def rank_radii(d, nq):
    """radius of query i: its r-th best distance (a row exactly there is excluded), every other group one ulp above it"""
    r = np.empty(nq, np.float32)
    for i in range(nq):
        r[i] = d[i, RANKS[i % len(RANKS)] - 1]
        if (i // len(RANKS)) % 2:
            r[i] = np.nextafter(r[i], np.float32(np.inf))
    return r


def assert_same_as_single(gpu, queries, radii, max_out, D, L, N, which=None):
    for q in range(len(queries)) if which is None else which:
        d, l, n = gpu.search_range(queries[q], float(radii[q]), max_out)
        assert N[q] == n, (q, N[q], n)
        m = min(n, max_out)
        assert (L[q, :m] == l).all(), (q, np.argwhere(L[q, :m] != l)[:5])
        assert (D[q, :m].view(np.uint32) == d.view(np.uint32)).all(), q


@pytest.mark.parametrize("dim", [64, 200, 768, 1000])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_range_batch_matches_single_query(metric, dim):
    n, nq, max_out = 50000, 64, 2000
    rows = synth_rows(n, dim, 0x7A0 + dim)
    labels = O.row_labels(n)[np.random.default_rng(dim).permutation(n)]  # label order differs from row order
    gpu = make_index(metric, rows, labels)
    queries = make_queries(metric, 0x7A1 + dim + metric, nq, dim)
    queries[5] = prep_query(metric, rows[7])  # a duplicated row: its twin ties with it under a different label
    d = exact_knn_dists(gpu, queries, 1000)
    radii = rank_radii(d, nq)
    radii[56] = d[56, 0] - abs(d[56, 0]) - 1.0  # below the best: no match
    radii[57] = np.nan
    radii[58] = np.inf
    radii[59] = -np.inf
    gpu.set_tensor_core_filter(1)
    D, L, N = gpu.search_range_batch(queries, radii, max_out)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    assert N[56] == 0 and N[57] == 0 and N[59] == 0 and N[58] == n
    assert_same_as_single(gpu, queries, radii, max_out, D, L, N)
    gpu.close()


def test_range_batch_arguments():
    n, dim = 5000, 32
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.append_synth(0x7B0, 0, n)
    D, L, N = gpu.search_range_batch(np.zeros((0, dim), np.float32), np.zeros(0, np.float32), 10)  # zero queries
    assert D.shape == (0, 10) and len(N) == 0
    q = O.synth_matrix(0x7B1, 4, dim)
    r = np.full(4, 5.0, np.float32)
    out_n = np.zeros(4, np.uint64)
    lib = B.lib()
    rc = lib.rxgpu_search_range_batch(gpu._h, 4, B._p(q, B._f32p), B._p(r, B._f32p), 0, None, None, B._p(out_n, B._u64p))
    assert rc == 0  # max_out = 0: no result rows, the totals still filled
    _, _, N = gpu.search_range_batch(q, r, 10)
    assert (out_n == N).all() and N.sum() > 0
    for args in ((None, r, out_n), (q, None, out_n), (q, r, None)):
        p = [None if a is None else B._p(a, B._u64p if a is out_n else B._f32p) for a in args]
        assert lib.rxgpu_search_range_batch(gpu._h, 4, p[0], p[1], 0, None, None, p[2]) == 3
    d10 = np.zeros((4, 10), np.float32)
    assert lib.rxgpu_search_range_batch(gpu._h, 4, B._p(q, B._f32p), B._p(r, B._f32p), 10, B._p(d10, B._f32p), None,
                                        B._p(out_n, B._u64p)) == 3
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_range_batch_overflow_and_truncation(metric):
    """a radius whose candidates overflow the list falls back to the exact scan; max_out below the match count truncates"""
    n, dim, nq, max_out = 50000, 96, 64, 100  # candidate lists of 4096
    rows = synth_rows(n, dim, 0x7C0)
    gpu = make_index(metric, rows, O.row_labels(n))
    queries = make_queries(metric, 0x7C1, nq, dim)
    d = exact_knn_dists(gpu, queries, 1000)
    radii = d[:, 999].copy()  # about 999 matches per query, 100 returned
    radii[:4] = exact_knn_dists(gpu, queries[:4], 20000)[:, -1]  # about 20 000 matches: more candidates than the list holds
    gpu.set_tensor_core_filter(1)
    D, L, N = gpu.search_range_batch(queries, radii, max_out)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] >= 4, st
    assert (N[:4] > 4096).all() and (N[4:] > max_out).all()
    assert_same_as_single(gpu, queries, radii, max_out, D, L, N)
    gpu.close()


def test_range_batch_after_removes_and_upserts():
    n, dim, nq, max_out = 30000, 96, 64, 2000
    rng = np.random.default_rng(11)
    rows = O.synth_matrix(0x7D0, n, dim)
    labels = O.row_labels(n)
    gpu = make_index(rx.L2, rows, labels, extra_capacity=100)
    queries = make_queries(rx.L2, 0x7D1, nq, dim)
    gpu.set_tensor_core_filter(1)
    gpu.search_range_batch(queries, np.full(nq, 1.0, np.float32), max_out)  # builds the shadow
    for lab in rng.choice(labels, 200, replace=False):
        gpu.remove_point(int(lab))  # swap-removes
    upd = rng.choice(labels, 100, replace=False)
    new = O.row_labels(100, first_row=n)
    vecs = O.synth_matrix(0x7D2, 200, dim)
    gpu.add_points(np.concatenate([upd, new]), vecs)  # rewrites and appends
    d = exact_knn_dists(gpu, queries, 1000)
    radii = rank_radii(d, nq)
    gpu.set_tensor_core_filter(1)
    D, L, N = gpu.search_range_batch(queries, radii, max_out)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    assert_same_as_single(gpu, queries, radii, max_out, D, L, N)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_range_batch_ties_ordered_by_label(metric):
    n, dim, nq, max_out = 30000, 64, 64, 4000
    rng = np.random.default_rng(metric + 5)
    rows = rng.integers(-2, 3, size=(n, dim)).astype(np.float32)
    gpu = make_index(metric, rows, O.row_labels(n)[rng.permutation(n)])
    queries = rng.integers(-2, 3, size=(nq, dim)).astype(np.float32)
    d = exact_knn_dists(gpu, queries, 1000)
    radii = rank_radii(d, nq)
    gpu.set_tensor_core_filter(1)
    D, L, N = gpu.search_range_batch(queries, radii, max_out)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1, st
    assert_same_as_single(gpu, queries, radii, max_out, D, L, N)
    gpu.close()


@pytest.mark.skipif(not O.ref_knn_available(), reason="oracle/_ref not built")
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_range_batch_against_reference(metric):
    n, dim, nq = 20000, 200, 64
    rows = O.synth_matrix(0x7E0, n, dim)
    labels = O.row_labels(n)
    gpu = make_index(metric, rows, labels)
    ref = O.RefBF(metric, dim, n)
    assert ref.add_batch(labels, rows) == 0
    queries = make_queries(metric, 0x7E1 + metric, nq, dim)
    d = exact_knn_dists(gpu, queries, 1001)
    ranks = np.array([RANKS[i % 4] for i in range(nq)])
    radii = ((d[np.arange(nq), ranks - 1] + d[np.arange(nq), ranks]) / 2).astype(np.float32)
    gpu.set_tensor_core_filter(1)
    D, L, N = gpu.search_range_batch(queries, radii, n)
    assert rx.last_search_stats()["tc_used"] == 1
    for q in range(nq):
        rd, rl = ref.search_range(queries[q], float(radii[q]))
        mine = dict(zip(L[q, :N[q]].tolist(), D[q, :N[q]].tolist()))
        theirs = dict(zip(rl.tolist(), rd.tolist()))
        noise = RTOL * max(abs(float(radii[q])), 1e-2)
        for lab in set(mine) ^ set(theirs):  # only a row within fp noise of the radius may fall on either side
            assert abs(mine.get(lab, theirs.get(lab)) - radii[q]) <= noise, (q, lab)
        common = sorted(set(mine) & set(theirs))
        assert np.allclose([mine[x] for x in common], [theirs[x] for x in common], rtol=RTOL, atol=ATOL), q
    gpu.close()


def test_range_batch_keeps_single_query_state():
    """the retained result of rxgpu_search_range and the KNN tie replay from the filter's lists are unaffected by a range batch"""
    n, dim, nq, k = 30000, 64, 64, 10
    rng = np.random.default_rng(3)
    rows = rng.integers(-2, 3, size=(n, dim)).astype(np.float32)
    gpu = make_index(rx.L2, rows, O.row_labels(n)[rng.permutation(n)])
    queries = rng.integers(-2, 3, size=(nq, dim)).astype(np.float32)
    gpu.set_tensor_core_filter(1)
    d0, l0, c0 = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tie_from_lists"] > 0, st  # integer rows: ties straddle the k-th place
    r0 = float(d0[0, k - 1]) + 0.5  # integer distances: at least k matches
    sd, sl, sn = gpu.search_range(queries[0], r0, 1)
    assert sn >= k
    gpu.search_range_batch(queries, d0[:, k - 1] + 1.0, 1000)
    assert rx.last_search_stats()["tc_used"] == 1
    rd, rl = np.zeros(sn, np.float32), np.zeros(sn, np.uint64)
    assert B.lib().rxgpu_last_range_results(0, sn, B._p(rd, B._f32p), B._p(rl, B._u64p)) == 0
    assert rl[0] == sl[0] and rd[0] == sd[0]
    full_d, full_l, _ = gpu.search_range(queries[0], r0, sn)
    assert (rl == full_l).all() and (rd.view(np.uint32) == full_d.view(np.uint32)).all()
    d1, l1, c1 = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tie_from_lists"] == st["tie_from_lists"]
    assert (c0 == c1).all() and (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all()
    gpu.close()


@pytest.mark.parametrize("mode", [1, 4])  # single CTAs, clusters of two
def test_range_batch_larger_than_one_launch(mode):
    n, dim, nq, max_out = 20000, 64, 40000, 50
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.append_synth(0x7F0, 0, n)
    queries = O.synth_matrix(0x7F1, nq, dim)
    radii = exact_knn_dists(gpu, queries, 10)[:, 9]
    D0, L0, N0 = gpu.search_range_batch(queries, radii, max_out)  # mode 2: the exact scan per query
    assert rx.last_search_stats()["tc_used"] == 0
    gpu.set_tensor_core_filter(mode)
    D, L, N = gpu.search_range_batch(queries, radii, max_out)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0 and st["passes"] >= 2, st
    assert st["tc_cluster"] == (2 if mode == 4 else 1), st
    assert (N == N0).all() and N.sum() > 8 * nq
    assert (L == L0).all() and (D.view(np.uint32) == D0.view(np.uint32)).all()
    assert_same_as_single(gpu, queries, radii, max_out, D, L, N, which=range(0, nq, 997))
    gpu.close()


def test_range_batch_automatic_routing():
    """mode 0: the filter serves batches of >= 64 queries on >= 100k rows; anything smaller takes the exact scan, same results"""
    dim, max_out = 64, 200
    queries = O.synth_matrix(0x801, 64, dim)
    for n, nq, tc in ((100000, 64, 1), (100000, 63, 0), (99999, 64, 0)):
        gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
        gpu.append_synth(0x800, 0, n)
        radii = exact_knn_dists(gpu, queries[:nq], 100)[:, 99]
        gpu.set_tensor_core_filter(0)
        D, L, N = gpu.search_range_batch(queries[:nq], radii, max_out)
        assert rx.last_search_stats()["tc_used"] == tc, (n, nq)
        assert_same_as_single(gpu, queries[:nq], radii, max_out, D, L, N)
        gpu.close()
