"""GPU tests of KNN with k + 1 in (128, 1024] on the tensor-core filter: staged exact thresholds (DESIGN 3.2).  Every answer must be
bit-identical to the exact scan (filter mode 2): the same labels in the same order, the same distance bits and the same counts.

Stages: the seed is the exact top-k1 of the first 2 k1 rows, and every stage's prefix is 4 times the previous one, the last one all
rows, so a search over n rows takes max(1, ceil(log4(n / (2 k1)))) filter stages (`stages` below)."""
import numpy as np
import pytest
from helpers import assert_same_knn, prep_query
from test_size_gpu import _ref_bf_filled, _threads
from test_tc_int8_bound_gpu import adversarial_queries, adversarial_rows

import reindexer_b200 as rx
from reindexer_b200 import binding as B
from oracle import oracle as O

pytestmark = pytest.mark.gpu

KS = (127, 128, 255, 256, 300, 1000, 1023)


def stages(n, k):
    rows, s = min(n, 2 * (k + 1)), 0
    while True:
        rows, s = min(n, rows * 4), s + 1
        if rows == n:
            return s


def tie_heavy(n, dim, seed):
    """integer-valued rows: every summation order gives the same fp32 sums, so bit-equal distances abound"""
    return np.random.default_rng(seed).integers(-2, 3, size=(n, dim)).astype(np.float32)


def make_queries(metric, seed, nq, dim):
    q = O.synth_matrix(seed, nq, dim)
    return np.stack([prep_query(metric, x) for x in q]) if metric == rx.COS else q


def exact(gpu, queries, k):
    gpu.set_tensor_core_filter(2)
    out = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 0
    return out


def assert_identical(a, b):
    (d0, l0, c0), (d1, l1, c1) = a, b
    assert (c0 == c1).all()
    assert (l0 == l1).all(), np.argwhere(l0 != l1)[:5]
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all()


@pytest.mark.parametrize("mode", [3, 4])
@pytest.mark.parametrize("dim", [64, 200, 768, 1000])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_large_k_matches_exact_scan(metric, dim, mode):
    # 40 000 rows: k = 127 runs on the bound list; k = 128 .. 300 take 4 filter stages, k = 1000 and 1023 take 3.  160 queries make
    # two query blocks, so mode 4 runs clusters of two
    n, nq = 40000, 160
    rows = O.synth_matrix(0x1A00 + dim, n, dim)
    rows[n - 500:] = rows[:500]  # duplicated rows: equal distances under different labels
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    queries = make_queries(metric, 0x1A01 + dim, nq, dim)
    for k in KS:
        ref = exact(gpu, queries, k)
        gpu.set_tensor_core_filter(mode)
        got = gpu.search_knn(queries, k)
        st = rx.last_search_stats()
        assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, (k, st)
        assert st["tc_cluster"] == (2 if mode == 4 else 1), st
        if k + 1 > 128:
            assert stages(n, k) >= 2
        assert_identical(ref, got)
    gpu.close()


def test_large_k_automatic_routing():
    n, dim = 100000, 64
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.append_synth(0x1B00, 0, n)
    queries = O.synth_matrix(0x1B01, 64, dim)
    gpu.set_tensor_core_filter(0)
    got = gpu.search_knn(queries, 1023)  # 64 queries, 100 k rows, k + 1 = 1024: the filter, 3 stages
    assert rx.last_search_stats()["tc_used"] == 1
    gpu.search_knn(queries[:63], 1023)
    assert rx.last_search_stats()["tc_used"] == 0
    gpu.search_knn(queries, 1024)
    assert rx.last_search_stats()["tc_used"] == 0
    assert_identical(exact(gpu, queries, 1023), got)
    gpu.close()


@pytest.mark.parametrize("k", [300, 777])
@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_large_k_ties_replayed_from_lists(metric, k):
    # 30 000 rows minus 300 swap-removed: 3 filter stages at k = 300 and at k = 777
    n, dim, nq = 30000, 32, 64
    rng = np.random.default_rng(k + metric)
    vecs, labels = tie_heavy(n, dim, 7 + k), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(labels, vecs)
    cpu = O.best_bf(metric, dim, n)
    cpu.add_batch(labels, vecs)
    for lab in rng.choice(labels, 300, replace=False):
        gpu.remove_point(int(lab))
        cpu.remove(int(lab))
    queries = tie_heavy(nq, dim, 8 + k)
    ref = exact(gpu, queries, k)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    assert st["tie_replays"] > 0 and st["tie_from_lists"] == st["tie_replays"], st
    assert_identical(ref, got)
    for i in range(0, nq, 8):
        dr, lr = cpu.search_knn(queries[i], k)
        assert (got[1][i] == lr).all(), i
        assert (got[0][i].view(np.uint32) == np.asarray(dr, np.float32).view(np.uint32)).all(), i
    gpu.close()


def test_large_k_overflow_falls_back_to_exact_scan():
    """25 000 copies of each of four rows: every copy is a candidate of a query next to it, more than the last stage's list of
    64 k1 = 19 264 entries holds, so those queries are answered by the exact scan"""
    n, dim, nq, k = 120000, 64, 64, 300
    base = O.synth_matrix(0x1C00, 4, dim)
    vecs = np.concatenate([np.repeat(base, 25000, axis=0), O.synth_matrix(0x1C01, n - 100000, dim)])
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.add_points(O.row_labels(n), vecs)
    queries = np.concatenate([base + 0.001, O.synth_matrix(0x1C02, nq - 4, dim)]).astype(np.float32)
    ref = exact(gpu, queries, k)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] >= 4, st
    assert_identical(ref, got)
    gpu.close()


def test_large_k_after_upserts_and_removes():
    n, dim, nq, k = 40000, 96, 64, 300
    rng = np.random.default_rng(5)
    labels = O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n + 100)
    gpu.add_points(labels, O.synth_matrix(0x1D00, n, dim))
    queries = O.synth_matrix(0x1D01, nq, dim)
    gpu.set_tensor_core_filter(1)
    gpu.search_knn(queries, k)  # builds the shadow
    for lab in rng.choice(labels, 200, replace=False):
        gpu.remove_point(int(lab))  # swap-removes
    upd = rng.choice(labels, 50, replace=False)
    vecs = (queries[rng.integers(0, nq, size=150)] * 3.0).astype(np.float32)
    gpu.add_points(np.concatenate([upd, O.row_labels(100, first_row=n)]), vecs)  # rewrites and appends next to the queries
    ref = exact(gpu, queries, k)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 1
    assert_identical(ref, got)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_large_k_on_int8_stress_rows(metric):
    n, dim, nq, k = 24000, 96, 160, 300
    rng = np.random.default_rng(dim * 7 + metric)
    rows = adversarial_rows(rng, n, dim)
    queries = adversarial_queries(rng, rows, nq, dim)
    if metric == rx.COS:
        queries = np.stack([prep_query(metric, q) if np.any(q) else q for q in queries])
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    ref = exact(gpu, queries, k)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] <= nq // 4, st
    assert_identical(ref, got)
    gpu.close()


def test_large_k_batch_larger_than_one_launch():
    n, dim, nq, k = 20000, 64, 40000, 200  # 313 query blocks of 128: several filter launches per stage
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.append_synth(0x1E00, 0, n)
    queries = O.synth_matrix(0x1E01, nq, dim)
    ref = exact(gpu, queries, k)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    assert_identical(ref, got)
    gpu.close()


def test_large_k_sharded_single_rank_ties():
    n, dim, nq, k = 30000, 32, 64, 300
    vecs, labels = tie_heavy(n, dim, 17), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.add_points(labels, vecs)
    gpu.set_tensor_core_filter(1)
    queries = tie_heavy(nq, dim, 18)
    comm = B.ShardComm(1, 0, None, 0)
    d1, l1, c1 = comm.search_knn(gpu, queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tie_replays"] > 0 and st["tie_from_lists"] == st["tie_replays"], st
    assert_identical(gpu.search_knn(queries, k), (d1, l1, c1))
    comm.close()
    gpu.close()


def test_large_k_device_entry_point():
    import torch

    n, dim, nq, k1 = 50000, 96, 128, 501
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.append_synth(0x1F00, 0, n)
    dq = torch.from_numpy(O.synth_matrix(0x1F01, nq, dim)).cuda()
    outs = []
    for mode in (2, 1):
        gpu.set_tensor_core_filter(mode)
        od = torch.zeros((nq, k1), dtype=torch.float32, device="cuda")
        oi = torch.zeros((nq, k1), dtype=torch.int32, device="cuda")
        ol = torch.zeros((nq, k1), dtype=torch.int64, device="cuda")
        oc = torch.zeros((nq,), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        gpu.search_knn_device(nq, dq.data_ptr(), k1, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr())
        assert rx.last_search_stats()["tc_used"] == (mode == 1)
        outs.append([t.cpu().numpy() for t in (od, oi, ol, oc)])
    (d0, i0, l0, c0), (d1, i1, l1, c1) = outs
    assert (c0 == k1).all() and (c0 == c1).all() and (i0 == i1).all() and (l0 == l1).all()
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all()
    gpu.close()


@pytest.mark.skipif(not O.ref_knn_available(), reason="oracle/_ref not built")
def test_large_k_one_million_rows_vs_reference():
    n, dim, k, seed = 1_000_000, 768, 1000, 0x51EE
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.append_synth(seed, 0, n)
    cpu = _ref_bf_filled(O.IP, dim, n, seed)
    batch = O.synth_matrix(seed + 1, 128, dim)
    d, l, c = gpu.search_knn(batch, k)  # automatic mode: 128 queries on 1M rows, k + 1 = 1001 -> staged thresholds, 5 stages
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    dr, lr, cr = cpu.search_knn_batch(batch[:12], k, _threads())
    for i in range(12):
        assert_same_knn(d[i], l[i], dr[i], lr[i], ctx=f"batch query {i}")
