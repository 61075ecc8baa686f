"""GPU tests of the int8 filter's KNN step around the filter kernel (knn_tc.cuh): the seed (tc_seed_slices over query tiles and
512-row slices, merged by tc_seed_merge) and the re-rank of only the candidates whose lower bound is at or below the query's final
threshold.  Neither may change an answer: labels, order, counts and distance bits equal the exact scan's (filter mode 2) at every
batch, k, dimension and index size around the seed's tiles and slices, and the rows the re-rank gathers include every row of the
answer."""
import ctypes

import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O
from reindexer_b200 import binding as B

pytestmark = pytest.mark.gpu

NQS = (1, 15, 16, 17, 64, 1000, 1024)  # one seed query tile is 16 queries
KS = (1, 11, 127, 128)                 # k1 up to the bound list's 128 entries
GATHERED = 41                          # knn_tc.cuh: kTcDgGathered, in CTA 0's slots of the diagnostic counters


def same_as_exact(gpu, queries, k, max_fallbacks=0):
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 0
    gpu.set_tensor_core_filter(1)
    d1, l1, c1 = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_kernel"] == 1, st
    assert st["tc_fallbacks"] <= max_fallbacks, st
    ctx = (len(queries), k)
    assert (c0 == c1).all(), (ctx, np.argwhere(c0 != c1)[:5])
    assert (l0 == l1).all(), (ctx, np.argwhere(l0 != l1)[:5])
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all(), ctx
    return st


# fewer rows than one seed slice, than the seed, exactly the seed, and one row more
@pytest.mark.parametrize("n", [300, 4095, 4096, 4097])
@pytest.mark.parametrize("dim", [64, 768, 1000])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_step_matches_exact_scan(metric, dim, n):
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0x57E0 + dim + n, 0, n)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(0x57E1 + dim, max(NQS), dim)])
    for nq in NQS:
        for k in KS:
            same_as_exact(gpu, queries[:nq], k)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_step_near_duplicates_and_non_finite_rows(metric):
    """near-duplicate rows keep many candidates at the final threshold; rows with NaN and infinite components give NaN or infinite
    distances and bounds, which the seed sorts last and the re-rank keeps"""
    rng = np.random.default_rng(0x57E2 + metric)
    n, dim, nq = 9000, 64, 300
    base = rng.standard_normal((60, dim)).astype(np.float32)
    rows = base[rng.integers(0, 60, size=n)] + 1e-4 * rng.standard_normal((n, dim)).astype(np.float32)
    if metric != rx.COS:
        rows[rng.integers(0, n, size=40), rng.integers(0, dim, size=40)] = np.nan
        rows[rng.integers(0, n, size=40), rng.integers(0, dim, size=40)] = np.inf
    queries = np.stack([prep_query(metric, q) for q in base[rng.integers(0, 60, size=nq)]])
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    for k in (1, 11, 128):
        same_as_exact(gpu, queries, k, max_fallbacks=nq)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_step_tie_replay_from_lists(metric):
    """integer rows over a few values: runs of equal distances straddle the k-th place, so the tie replay reads the full
    candidate lists after the re-rank gathered only the rows under the final threshold"""
    rng = np.random.default_rng(0x57E3 + metric)
    n, dim, nq = 8000, 64, 160
    rows = rng.integers(-1, 2, size=(n, dim)).astype(np.float32)
    rows[rng.integers(0, n, size=2000)] = rows[rng.integers(0, n, size=2000)]
    queries = rng.integers(-1, 2, size=(nq, dim)).astype(np.float32)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    replays = 0
    for k in (1, 11, 127):
        st = same_as_exact(gpu, queries, k, max_fallbacks=nq)
        replays += st["tie_from_lists"]
    assert replays > 0
    gpu.close()


def test_rerank_gathers_a_subset_holding_the_answer(monkeypatch):
    """with the stamped diagnostic filter (real results), the re-rank counts the rows it gathers: at most the candidates in the
    lists, at least every row of the answers, and far fewer than the candidates once tau has tightened past the seed's"""
    torch = pytest.importorskip("torch")
    monkeypatch.setenv("RXGPU_TC_DIAG", "1")
    lib = B.lib()
    n, dim, nq, k = 200000, 128, 256, 11
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.append_synth(0x57E4, 0, n)
    queries = O.synth_matrix(0x57E5, nq, dim)
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    gpu.set_tensor_core_filter(1)
    counters = torch.zeros(1 << 22, dtype=torch.int64, device="cuda:0")
    B._check(lib.rxgpu_tc_diag(1, ctypes.c_void_p(counters.data_ptr())))
    try:
        d1, l1, c1 = gpu.search_knn(queries, k)
        st = rx.last_search_stats()
    finally:
        B._check(lib.rxgpu_tc_diag(0, None))
    torch.cuda.synchronize()
    assert st["tc_used"] == 1 and st["tc_kernel"] == 2 and st["tc_fallbacks"] == 0, st
    assert (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all() and (c0 == c1).all()
    gathered = int(counters[GATHERED].item())
    assert int(c1.sum()) <= gathered <= st["tc_candidates"], (gathered, st)
    assert gathered < st["tc_candidates"], (gathered, st)
    gpu.close()
