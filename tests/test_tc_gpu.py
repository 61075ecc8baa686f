"""GPU tests of the tensor-core filter path (wgmma + TMA + mbarrier, knn_tc.cuh): for large query batches the bf16 tensor-core
scores only SELECT candidates under a certified error bound; the exact fp32 routine re-ranks them.  So the answers must be
bit-identical to the exact scan (same labels, same order, same distance bits) -- and therefore match the oracle like it does."""
import numpy as np
import pytest
from helpers import assert_same_knn, prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def both_paths(gpu, queries, k):
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    s0 = rx.last_search_stats()
    gpu.set_tensor_core_filter(1)
    d1, l1, c1 = gpu.search_knn(queries, k)
    s1 = rx.last_search_stats()
    assert s0["tc_used"] == 0 and s1["tc_used"] == 1, (s0, s1)
    return (d0, l0, c0), (d1, l1, c1), s1


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("n,dim,nq,k", [(20000, 128, 64, 10), (30000, 100, 100, 10), (12000, 768, 96, 10), (9000, 64, 300, 15),
                                        (5000, 200, 33, 1), (30000, 768, 400, 10), (40000, 256, 700, 5), (6000, 1000, 150, 10),
                                        (60000, 128, 520, 40), (50000, 96, 200, 63), (80000, 64, 260, 100), (45000, 160, 130, 127),
                                        (20000, 64, 32, 10)])  # the last one: a query block of 32 (wgmma N = 32)
def test_tc_path_is_bit_identical_to_exact_scan(metric, n, dim, nq, k):
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0xABC0 + dim, 0, n)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(0xABC1 + dim, nq, dim)])
    (d0, l0, c0), (d1, l1, c1), st = both_paths(gpu, queries, k)
    assert (c0 == c1).all() and (c0 == k).all()
    assert (l0 == l1).all(), np.argwhere(l0 != l1)[:5]
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all()
    assert st["tc_fallbacks"] == 0 and 0 < st["tc_candidates"] < nq * 4096, st
    # every cluster shape gives the same bits: 3 = single CTAs, 4 = clusters of up to two CTAs sharing every row tile (TMA multicast)
    for mode in (3, 4):
        gpu.set_tensor_core_filter(mode)
        d2, l2, c2 = gpu.search_knn(queries, k)
        s2 = rx.last_search_stats()
        assert s2["tc_kernel"] == 1 and s2["tc_cluster"] == (2 if mode == 4 and nq > 128 else 1), (mode, s2)
        assert (l2 == l0).all() and (d2.view(np.uint32) == d0.view(np.uint32)).all(), mode
    assert st["tc_kernel"] == 1
    assert st["tc_cluster"] == 1, st  # default: single CTAs


def test_tc_path_matches_oracle():
    n, dim, nq, k = 15000, 96, 80, 10
    vecs, labels = O.synth_matrix(31, n, dim), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.add_points(labels, vecs)
    gpu.set_tensor_core_filter(1)
    cpu = O.best_bf(rx.IP, dim, n)
    cpu.add_batch(labels, vecs)
    queries = O.synth_matrix(32, nq, dim)
    d, l, c = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 1
    for i in range(0, nq, 7):
        dr, lr = cpu.search_knn(queries[i], k)
        assert_same_knn(d[i], l[i], dr, lr, ctx=f"q{i}")


def test_tc_overflow_falls_back_to_exact_scan_and_ties_still_replay():
    """pathological data: thousands of identical rows => every one of them is a candidate => the list overflows => those queries
    are answered by the exact scan; the reference's tie rule is still applied on top (duplicates tie at the k-th place)"""
    n, dim, nq, k = 24000, 64, 64, 10
    base = O.synth_matrix(41, 4, dim)
    vecs = np.concatenate([np.repeat(base, 5000, axis=0), O.synth_matrix(42, n - 20000, dim)])
    labels = O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.add_points(labels, vecs)
    queries = np.concatenate([base + 0.001, O.synth_matrix(43, nq - 4, dim)]).astype(np.float32)
    (d0, l0, c0), (d1, l1, c1), st = both_paths(gpu, queries, k)
    assert st["tc_fallbacks"] >= 4
    assert (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all()
    cpu = O.best_bf(rx.L2, dim, n)
    cpu.add_batch(labels, vecs)
    for i in range(6):
        dr, lr = cpu.search_knn(queries[i], k)
        assert (l1[i] == lr).all()


def test_tc_shadow_follows_index_mutations():
    n, dim, nq, k = 20000, 128, 64, 10
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n + 100)
    gpu.append_synth(51, 0, n)
    queries = O.synth_matrix(52, nq, dim)
    both_paths(gpu, queries, k)
    # plant rows after the shadow was built: they must be found through the tensor-core path too
    planted = (queries[:8] * 4.0).astype(np.float32)
    gpu.add_points(O.row_labels(8, first_row=n), planted)
    gpu.remove_point(int(O.row_labels(1, first_row=5)[0]))
    (d0, l0, c0), (d1, l1, c1), st = both_paths(gpu, queries, k)
    assert (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all()
    assert all(l1[i, 0] == (n + i) << 32 for i in range(8))


def test_tc_shadow_incremental_updates_equal_a_rebuild():
    """the bf16 shadow is brought up to date row by row (the mutations log the rows they rewrite): after rounds of upserts of existing
    labels, appended runs, swap-removes and a resize the tensor-core path must still equal the exact scan bit for bit -- and equal a
    second index built from scratch with the same final content"""
    rng = np.random.default_rng(9)
    n, dim, nq, k = 30000, 96, 128, 10
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n + 4000)
    vecs = O.synth_matrix(61, n, dim)
    labels = O.row_labels(n)
    gpu.add_points(labels, vecs)
    queries = O.synth_matrix(62, nq, dim)
    both_paths(gpu, queries, k)  # builds the shadow
    next_row = n
    for rnd in range(4):
        hit = rng.choice(n, size=40, replace=False)  # rewrite existing rows close to some queries
        newv = (queries[rng.integers(0, nq, size=40)] + rng.normal(0, 0.01, size=(40, dim))).astype(np.float32)
        gpu.add_points(labels[hit], newv)
        fresh = (queries[rng.integers(0, nq, size=300)] * rng.uniform(0.9, 1.1, size=(300, 1))).astype(np.float32)
        gpu.add_points(O.row_labels(300, first_row=next_row), fresh)
        next_row += 300
        for lab in labels[rng.choice(n, size=25, replace=False)]:
            gpu.remove_point(int(lab))
        if rnd == 2:
            gpu.resize_index(n + 8000)  # the shadow is rebuilt at the new capacity
        (d0, l0, c0), (d1, l1, c1), st = both_paths(gpu, queries, k)
        assert (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all(), rnd
    gpu.close()
