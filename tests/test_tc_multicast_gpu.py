"""GPU tests of the int8 filter in clusters of up to four CTAs (knn_tc.cuh, kCluster = 1, 2, 4): the CTAs of a cluster own
consecutive query blocks, walk the same 64-row blocks, fetch 1/C of every stage each and multicast it to all C.  Modes 3, 4 and 5 of
rxgpu_set_tensor_core_filter take single CTAs, clusters of up to two and clusters of up to four; every one must return the exact
scan's labels and distance bits, with no fallback, on the shapes that reach the edges of the cluster coupling: every query-block
count from 1 to 9 (every padding case at C = 2 and C = 4), a batch of several launches, walkers of every block count residue mod 3,
partial last tiles, every ring shape (1, 6, 10, 12, 13 and 16 K chunks per block), and near-duplicate rows that keep the candidate
queues full while the cluster's CTAs wait on each other's stage releases."""
import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu

MODES = (3, 4, 5)
CLUSTER_MAX = {3: 1, 4: 2, 5: 4}


def tc_query_block(nq, kchunks):
    """the query block index.cu's tcQueryBlock picks, from tc_smem_bytes (knn_tc.cuh)"""
    def smem(nqb):
        return 1024 + nqb * kchunks * 128 + 12 * 8192 + 256 + nqb * 40 + 64

    nqb = min(128, (nq + 31) // 32 * 32)
    while nqb >= 32 and smem(nqb) > 227 * 1024:
        nqb -= 32
    blocks = (nq + nqb - 1) // nqb
    return min(nqb, ((nq + blocks - 1) // blocks + 31) // 32 * 32)


def expected_cluster(mode, nblocks, ntiles):
    """index.cu's tcClusterSize: the largest C <= the mode's maximum whose padding is at most one block and fewer than the batch's"""
    c = CLUSTER_MAX[mode]
    while c > 1:
        pad = (c - nblocks % c) % c
        if ntiles >= 2 and pad <= 1 and pad < nblocks:
            return c
        c //= 2
    return 1


def same_bits(ref, got, ctx):
    for x, y in zip(ref, got):
        assert x.shape == y.shape, ctx
        assert (x.view(np.uint8) == y.view(np.uint8)).all(), ctx


def check(gpu, queries, ks, n, dim, with_range=True):
    """KNN at every k in ks and one range batch, in modes 3 / 4 / 5 against the exact scan; returns the cluster sizes taken"""
    nq = len(queries)
    nblocks = -(-nq // tc_query_block(nq, (dim + 127) // 128))
    ntiles = -(-n // 128)
    taken = set()
    knn10 = None
    for k in ks:
        gpu.set_tensor_core_filter(2)
        ref = gpu.search_knn(queries, k)
        assert rx.last_search_stats()["tc_used"] == 0
        if knn10 is None:
            knn10 = ref
        for mode in MODES:
            gpu.set_tensor_core_filter(mode)
            got = gpu.search_knn(queries, k)
            st = rx.last_search_stats()
            assert st["tc_used"] == 1 and st["tc_kernel"] == 1 and st["tc_fallbacks"] == 0, (mode, k, st)
            assert st["tc_cluster"] == expected_cluster(mode, nblocks, ntiles), (mode, k, nblocks, st)
            taken.add(st["tc_cluster"])
            same_bits(ref, got, (mode, k))
    if with_range:
        d, _, c = knn10
        # radii just above the 4th exact distance (or the last one found): every query has matches
        radii = np.array([np.nextafter(d[q, min(3, int(c[q]) - 1)], np.float32(np.inf)) for q in range(nq)], np.float32)
        gpu.set_tensor_core_filter(2)
        ref = gpu.search_range_batch(queries, radii, 64)
        for mode in MODES:
            gpu.set_tensor_core_filter(mode)
            got = gpu.search_range_batch(queries, radii, 64)
            st = rx.last_search_stats()
            assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, (mode, st)
            assert st["tc_cluster"] == expected_cluster(mode, nblocks, ntiles), (mode, st)
            same_bits(ref, got, ("range", mode))
    return taken


def make_index(metric, n, dim, seed):
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(seed, 0, n)
    return gpu


def make_queries(metric, nq, dim, seed):
    return np.stack([prep_query(metric, q) for q in O.synth_matrix(seed, nq, dim)]).astype(np.float32)


# 1..9 query blocks of 128: at C = 4 the counts 3 and 7 are padded with one block and 1, 2, 5, 6 and 9 fall back to C = 2
# (padded at 3, 5, 7 and 9); one block is never paired with a padding block
@pytest.mark.parametrize("nblocks", range(1, 10))
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS], ids=["l2", "ip", "cos"])
def test_query_block_counts(metric, nblocks):
    n, dim, nq = 20000, 96, 128 * nblocks - 5
    gpu = make_index(metric, n, dim, 0x3C00 + nblocks)
    queries = make_queries(metric, nq, dim, 0x3C01 + nblocks)
    taken = check(gpu, queries, (10, 127, 300), n, dim)
    if nblocks in (3, 4, 7, 8):
        assert 4 in taken
    gpu.close()


# 8 query blocks (two groups of four): rows 100 = one tile whose second half is empty (no cluster: one tile); 2000, 2600, 4500,
# 6000 = 16 to 47 tiles over the walkers, so walkers get 1, 2 or 3 tiles (2, 4, 6 blocks: every residue mod 3), with partial last
# tiles (2600: the last tile's second half is empty); 70000 = long walks
@pytest.mark.parametrize("n", [100, 2000, 2600, 4500, 6000, 70000])
@pytest.mark.parametrize("metric", [rx.IP, rx.L2], ids=["ip", "l2"])
def test_walker_block_counts(metric, n):
    dim, nq = 96, 1019
    gpu = make_index(metric, n, dim, 0x3D00 + n)
    queries = make_queries(metric, nq, dim, 0x3D01 + n)
    check(gpu, queries, (10,), n, dim)
    gpu.close()


# kchunks = 1, 6, 10 (query block 96 and an 11-stage ring), 12 (as many chunks as the ring has stages), 13 and 16 (a block wraps the
# ring); 8 query blocks of whatever size the dimension allows
@pytest.mark.parametrize("dim", [64, 768, 1200, 1536, 1600, 2048])
def test_chunk_counts(dim):
    n = 30000
    nq = 8 * tc_query_block(1024, (dim + 127) // 128) - 3
    gpu = make_index(rx.IP, n, dim, 0x3E00 + dim)
    queries = make_queries(rx.IP, nq, dim, 0x3E01 + dim)
    taken = check(gpu, queries, (10, 300), n, dim)
    assert 4 in taken
    gpu.close()


def test_batch_larger_than_one_launch():
    n, dim, nq = 20000, 64, 312 * 128 - 5  # 312 query blocks: more clusters of four than are resident at once
    gpu = make_index(rx.IP, n, dim, 0x3F00)
    queries = make_queries(rx.IP, nq, dim, 0x3F01)
    gpu.set_tensor_core_filter(2)
    ref = gpu.search_knn(queries, 10)
    gpu.set_tensor_core_filter(5)
    got = gpu.search_knn(queries, 10)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0 and st["passes"] >= 2 and st["tc_cluster"] == 4, st
    same_bits(ref, got, "several launches")
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS], ids=["l2", "ip", "cos"])
def test_near_duplicates_fill_the_queues(metric):
    """every row and query is a near-duplicate of one vector, so every (query, row) pair passes the block test and the consumers
    wait on full candidate queues throughout, holding their stages -- and so the stages of the other CTAs of their cluster"""
    n, dim, nq = 3000, 96, 4 * 128
    rng = np.random.default_rng(7)
    base = O.synth_matrix(0x0DE, 1, dim)[0].astype(np.float64)
    rows = (base + rng.normal(0, 1e-3, size=(n, dim))).astype(np.float32)
    queries = (base + rng.normal(0, 1e-3, size=(nq, dim))).astype(np.float32)
    if metric == rx.COS:
        queries = np.stack([prep_query(metric, q) for q in queries])
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    taken = check(gpu, queries, (10, 300), n, dim)
    assert 4 in taken
    gpu.set_tensor_core_filter(5)
    gpu.search_knn(queries, 10)
    st = rx.last_search_stats()
    assert st["tc_cluster"] == 4 and st["tc_candidates"] >= nq * n // 2, st  # the pairs really crowded the queues
    gpu.close()
