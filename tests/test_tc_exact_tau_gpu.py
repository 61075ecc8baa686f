"""GPU tests of the int8 filter's bound list of EXACT distances (knn_tc.cuh header: tc_init_tau seeds it with the exact k1 best of the
first rows, the bookkeepers insert the exact distances of the rows they rescore).  Its threshold only decides which rows are
candidates; the answers must stay bit-identical to the exact scan (filter mode 2): labels, order, counts and distance bits, on data
built so that the lists see every kind of entry -- tie runs at the k-th place (the tie replay reads the candidate lists), rings kept
full by near-duplicates, Cosine rows at the norm coefficient's 1e-5 edge, zero rows, NaN and infinite components, lists that
overflow into the exact scan, and an index smaller than the seed."""
import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KS = (1, 10, 63, 127)


def exact_and_filter(gpu, queries, k, mode, max_fallbacks=0):
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 0
    gpu.set_tensor_core_filter(mode)
    d1, l1, c1 = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_kernel"] == 1, st  # the filter answered, with the production kernel
    assert st["tc_fallbacks"] <= max_fallbacks, st
    assert (c0 == c1).all(), (k, np.argwhere(c0 != c1)[:5])
    assert (l0 == l1).all(), (k, np.argwhere(l0 != l1)[:5])
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all(), k
    return st


def index_of(metric, rows):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], len(rows))
    gpu.add_points(O.row_labels(len(rows)), rows)
    return gpu


@pytest.mark.parametrize("mode", [3, 4])  # single CTAs, clusters of two
@pytest.mark.parametrize("dim", [64, 768, 1000, 2048])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_exact_bound_list_is_bit_identical(metric, dim, mode):
    n, nq = 6000, 200  # more rows than the seed: the bookkeepers rescore and insert
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0xE7A0 + dim, 0, n)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(0xE7A1 + dim, nq, dim)])
    for k in KS:
        st = exact_and_filter(gpu, queries, k, mode)
        assert st["tc_cluster"] == (2 if mode == 4 else 1), st
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_exact_bound_list_several_launches(metric):
    n, dim, nq = 20000, 64, 40000  # 313 query blocks: more than one launch holds
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0xE7A2 + metric, 0, n)
    queries = O.synth_matrix(0xE7A3 + metric, nq, dim)
    st = exact_and_filter(gpu, queries, 10, 3)
    assert st["passes"] >= 2, st
    gpu.close()


@pytest.mark.parametrize("mode", [3, 4])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_exact_bound_list_tie_runs(metric, mode):
    """integer rows over a few values: long runs of equal distances straddle the k-th place, so the bound list holds equal
    entries and the tie replay takes its rows from the candidate lists"""
    rng = np.random.default_rng(70 + metric)
    n, dim, nq = 8000, 64, 160
    rows = rng.integers(-1, 2, size=(n, dim)).astype(np.float32)
    rows[rng.integers(0, n, size=2000)] = rows[rng.integers(0, n, size=2000)]  # duplicated rows: exact ties
    queries = rng.integers(-1, 2, size=(nq, dim)).astype(np.float32)
    gpu = index_of(metric, rows)
    for k in KS:
        exact_and_filter(gpu, queries, k, mode, max_fallbacks=nq)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_exact_bound_list_near_duplicates(metric):
    """every row a near-copy of one vector: every pair passes the block test, every rescored row beats the threshold for a while,
    and the candidate queues stay full"""
    rng = np.random.default_rng(80 + metric)
    n, dim, nq = 6000, 128, 256
    base = O.synth_matrix(0xE7A4, 1, dim)[0]
    rows = (base + rng.normal(0, 1e-4, size=(n, dim))).astype(np.float32)
    queries = np.stack([prep_query(metric, q) for q in (base + rng.normal(0, 1e-2, size=(nq, dim))).astype(np.float32)])
    gpu = index_of(metric, rows)
    for k in (10, 127):
        exact_and_filter(gpu, queries, k, 3, max_fallbacks=nq)
    gpu.close()


def test_exact_bound_list_cosine_norm_edge_and_zero_rows():
    """Cosine rows whose squared norm sits just inside and just outside the 1e-5 window of the norm coefficient's shortcut, and
    all-zero rows (coefficient 1, distance -0)"""
    rng = np.random.default_rng(90)
    n, dim, nq = 6000, 96, 160
    rows = O.synth_matrix(0xE7A5, n, dim).astype(np.float64)
    rows /= np.linalg.norm(rows, axis=1, keepdims=True)
    scale = np.sqrt(1.0 + rng.choice([-1.2e-5, -0.8e-5, 0.0, 0.8e-5, 1.2e-5], size=(n, 1)))
    rows = (rows * scale).astype(np.float32)
    rows[rng.choice(n, size=300, replace=False)] = 0.0
    queries = np.stack([prep_query(rx.COS, q) for q in O.synth_matrix(0xE7A6, nq, dim)])
    gpu = index_of(rx.COS, rows)
    for k in KS:
        exact_and_filter(gpu, queries, k, 3, max_fallbacks=nq)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_exact_bound_list_non_finite_rows(metric):
    """rows with a NaN, +inf or -inf component: their distances are NaN or infinite, never inserted into the bound list as NaN"""
    rng = np.random.default_rng(100 + metric)
    n, dim, nq = 6000, 64, 160
    rows = O.synth_matrix(0xE7A7, n, dim)
    for bad in (np.nan, np.inf, -np.inf):
        at = rng.choice(n, size=60, replace=False)
        rows[at, rng.integers(0, dim, size=60)] = bad
    queries = O.synth_matrix(0xE7A8, nq, dim)
    gpu = index_of(metric, rows)
    for k in (1, 10, 127):
        exact_and_filter(gpu, queries, k, 3, max_fallbacks=nq)
    gpu.close()


def test_exact_bound_list_l2_offset_rows_overflow():
    """L2 rows and queries far from the origin (+1000 in every component): the error bound admits every row, the candidate lists
    overflow and the exact scan answers those queries"""
    n, dim, nq = 6000, 64, 160
    rows = (O.synth_matrix(0xE7A9, n, dim) + 1000.0).astype(np.float32)
    queries = (O.synth_matrix(0xE7AA, nq, dim) + 1000.0).astype(np.float32)
    gpu = index_of(rx.L2, rows)
    st = exact_and_filter(gpu, queries, 10, 3, max_fallbacks=nq)
    assert st["tc_fallbacks"] > 0, st
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_exact_bound_list_index_smaller_than_seed(metric):
    n, dim, nq = 700, 128, 130
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0xE7AB + metric, 0, n)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(0xE7AC, nq, dim)])
    for k in KS:
        exact_and_filter(gpu, queries, k, 3)
    gpu.close()
