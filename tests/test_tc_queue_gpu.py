"""GPU tests of the int8 filter's candidate queue under back-pressure.  Every row is a near-duplicate of one vector and so are the
queries, so every (query, row) pair passes the block test: each 64-row block hands 64 x 128 hits to a queue of at most 512 records,
and the consumers wait on a full queue all the time.  No hit may be dropped: KNN (bound list), staged KNN (k + 1 > 128, fixed
thresholds) and range batches must stay bit-identical to the exact scan, with single CTAs and with clusters of two, and the filter
must decide every query itself (3000 rows stay under the 4096-entry candidate lists, so no query falls back to the exact scan)."""
import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu

N, DIM, NQ = 3000, 96, 256


def near_duplicates(seed, n):
    rng = np.random.default_rng(seed)
    base = O.synth_matrix(0x0DD + seed, 1, DIM)[0].astype(np.float64)
    return (base + rng.normal(0, 1e-3, size=(n, DIM))).astype(np.float32)


def setup(metric):
    rows = near_duplicates(1, N)
    queries = near_duplicates(1, NQ + 7)[7:]  # the same centre, other noise
    if metric == rx.COS:
        queries = np.stack([prep_query(metric, q) for q in queries])
    gpu = rx.GpuBruteforceSearch(metric, DIM, N)
    gpu.add_points(O.row_labels(N), rows)
    return gpu, queries


def same(a, b):
    for x, y in zip(a, b):
        assert x.shape == y.shape
        assert (x.view(np.uint8) == y.view(np.uint8)).all()


@pytest.mark.parametrize("mode", [3, 4], ids=["single", "cluster2"])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS], ids=["l2", "ip", "cos"])
def test_full_queue_knn_and_staged(metric, mode):
    gpu, queries = setup(metric)
    for k in (10, 300):
        gpu.set_tensor_core_filter(2)
        ref = gpu.search_knn(queries, k)
        gpu.set_tensor_core_filter(mode)
        got = gpu.search_knn(queries, k)
        st = rx.last_search_stats()
        assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, (k, st)
        assert st["tc_candidates"] >= NQ * N // 2, (k, st)  # the pairs really crowded the queue
        if mode == 4:
            assert st["tc_cluster"] == 2, st
        same(ref, got)
    gpu.close()


@pytest.mark.parametrize("mode", [3, 4], ids=["single", "cluster2"])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS], ids=["l2", "ip", "cos"])
def test_full_queue_range(metric, mode):
    gpu, queries = setup(metric)
    gpu.set_tensor_core_filter(2)
    d, _, _ = gpu.search_knn(queries, 50)
    radii = np.nextafter(d[:, -1], np.float32(np.inf)).astype(np.float32)  # about 50 matches per query
    ref = gpu.search_range_batch(queries, radii, 64)
    gpu.set_tensor_core_filter(mode)
    got = gpu.search_range_batch(queries, radii, 64)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    assert (got[2] >= 50).all()
    same(ref, got)
    gpu.close()
