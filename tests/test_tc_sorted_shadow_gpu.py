"""GPU tests of the int8 filter's sorted shadow: the rows sit in slots sorted by their scale, each 64-slot block is tested against one
integer threshold per query, and the slots of mutated indexes go dead or are appended unsorted.  Every answer must stay bit-identical
to the exact scan (tensor-core filter off) for all three metrics, through non-finite and all-zero rows, swap-removes, upserts,
appends and a whole rebuild, at staged k and at every query-block count of every cluster shape."""
import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu

METRICS = [rx.L2, rx.IP, rx.COS]


def queries_for(metric, q):
    return np.stack([prep_query(metric, x) if np.any(x) else x for x in q]) if metric == rx.COS else q


def assert_filter_exact(gpu, queries, k, ctx=""):
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    gpu.set_tensor_core_filter(1)
    d1, l1, c1 = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 1, ctx
    assert (c0 == c1).all(), ctx
    assert (l0 == l1).all(), (ctx, np.argwhere(l0 != l1)[:5])
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all(), ctx
    return d1, l1


def mixed_rows(rng, n, dim):
    rows = O.synth_matrix(0x5047 + dim, n, dim) * (10.0 ** rng.uniform(-2, 2, size=(n, 1)))
    rows[rng.integers(0, n, 40)] = 0.0                              # all-zero rows (zero-norm rows for Cosine)
    rows[rng.integers(0, n, 8), rng.integers(0, dim, 8)] = np.inf   # non-finite rows
    rows[rng.integers(0, n, 8), rng.integers(0, dim, 8)] = -np.inf
    rows[rng.integers(0, n, 8), rng.integers(0, dim, 8)] = np.nan
    rows[rng.integers(0, n, 16)] *= 1e-30                           # scales near the bottom of fp32
    return rows.astype(np.float32)


def edge_queries(rng, rows, nq, dim):
    q = O.synth_matrix(0x5048 + dim, nq, dim)
    near = rows[rng.integers(0, len(rows), nq // 2)]
    ok = np.isfinite(near).all(axis=1)
    q[: nq // 2][ok] = near[ok]  # a row itself: its score sits at the top of the query's list, next to its ties
    q[nq - 1] = 0.0
    return q.astype(np.float32)


@pytest.mark.parametrize("metric", METRICS)
def test_sorted_shadow_exact_on_mixed_rows(metric):
    rng = np.random.default_rng(11 + metric)
    n, dim, nq = 20000, 96, 160
    rows = mixed_rows(rng, n, dim)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    assert_filter_exact(gpu, queries_for(metric, edge_queries(rng, rows, nq, dim)), 10, f"metric {metric}")
    gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_sorted_shadow_mutations_match_rebuild(metric):
    rng = np.random.default_rng(23 + metric)
    n, dim, nq = 16000, 64, 128
    rows = O.synth_matrix(0x5049, n, dim)
    labels = O.row_labels(n)
    queries = queries_for(metric, edge_queries(rng, rows, nq, dim))
    gpu = rx.GpuBruteforceSearch(metric, dim, n + 4096)
    gpu.add_points(labels, rows)
    assert_filter_exact(gpu, queries, 10, "built")
    # swap-removes: the last row, rows in the middle of sorted blocks; upserts of existing labels; a small append
    gpu.remove_point(int(labels[-1]))
    for lab in rng.choice(labels[: n // 2], 30, replace=False):
        gpu.remove_point(int(lab))
    up = rng.choice(labels[: n // 2], 20, replace=False)
    gpu.add_points(up, O.synth_matrix(0x504A, len(up), dim) * 3.0)
    extra = O.row_labels(n + 300)[n:]
    gpu.add_points(extra, O.synth_matrix(0x504B, 300, dim))
    d_inc, l_inc = assert_filter_exact(gpu, queries, 10, "incremental")
    # the same index built at once (a resize rebuilds the shadow whole): the same bits
    gpu.resize_index(n + 8192)
    d_full, l_full = assert_filter_exact(gpu, queries, 10, "rebuilt")
    assert (l_inc == l_full).all() and (d_inc.view(np.uint32) == d_full.view(np.uint32)).all()
    # removes until the dead slots force a whole rebuild, then search again
    for lab in rng.choice(labels[n // 2: -1], 3000, replace=False):
        gpu.remove_point(int(lab))
    assert_filter_exact(gpu, queries, 10, "after many removes")
    gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_sorted_shadow_staged_and_range(metric):
    rng = np.random.default_rng(31 + metric)
    n, dim, nq = 30000, 64, 96
    rows = O.synth_matrix(0x504C, n, dim) * (10.0 ** rng.uniform(-1, 1, size=(n, 1))).astype(np.float32)
    queries = queries_for(metric, edge_queries(rng, rows, nq, dim))
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    assert_filter_exact(gpu, queries, 300, "staged k = 300")
    d, _ = assert_filter_exact(gpu, queries, 10, "k = 10")
    radius = np.where(np.isfinite(d[:, -1]), d[:, -1], 0.0).astype(np.float32)
    gpu.set_tensor_core_filter(2)
    r0 = gpu.search_range_batch(queries, radius, 256)
    gpu.set_tensor_core_filter(1)
    r1 = gpu.search_range_batch(queries, radius, 256)
    for a, b in zip(r0, r1):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))
    gpu.close()


@pytest.mark.parametrize("mode", [3, 4, 5])
def test_sorted_shadow_every_query_block_count(mode):
    rng = np.random.default_rng(41 + mode)
    n, dim = 40000, 128
    rows = O.synth_matrix(0x504D, n, dim)
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    for blocks in range(1, 10):
        queries = edge_queries(rng, rows, 128 * blocks - 5, dim)
        gpu.set_tensor_core_filter(2)
        d0, l0, _ = gpu.search_knn(queries, 10)
        gpu.set_tensor_core_filter(mode)
        d1, l1, _ = gpu.search_knn(queries, 10)
        assert rx.last_search_stats()["tc_used"] == 1
        assert (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all(), (mode, blocks)
    gpu.close()
