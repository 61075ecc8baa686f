"""GPU tests of the int8 filter's block walk (knn_tc.cuh): one stage ring consumed in block order, and three consumer warpgroups that
take turns issuing their blocks' MMAs (warpgroup i % 3 owns the walker's block i).  The shapes reach the edges of that walk: walkers
with no block at all and with block counts of every residue mod 3, a last tile whose second half lies beyond the rows, a block of
one K chunk, blocks of as many chunks as the ring has stages and of more, and an odd number of query blocks under clusters of two.
Every answer must carry the exact scan's bits, and the filter must have answered every query itself (no fallback)."""
import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def tc_query_block(nq, kchunks):
    """the query block index.cu's tcQueryBlock picked before the ring was shared by three warpgroups (two rings of six stages,
    two copies of the per-query thresholds); the three-warpgroup layout keeps it at every dimension"""
    def smem(nqb):
        return 1024 + nqb * kchunks * 128 + 12 * 8192 + 256 + nqb * 40 + 64

    nqb = min(128, (nq + 31) // 32 * 32)
    while nqb >= 32 and smem(nqb) > 227 * 1024:
        nqb -= 32
    blocks = (nq + nqb - 1) // nqb
    return min(nqb, ((nq + blocks - 1) // blocks + 31) // 32 * 32)


def make_index(metric, n, dim, seed):
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(seed, 0, n)
    return gpu


def make_queries(metric, nq, dim, seed):
    return np.stack([prep_query(metric, q) for q in O.synth_matrix(seed, nq, dim)]).astype(np.float32)


def same_bits(a, b, ctx):
    (d0, l0, c0), (d1, l1, c1) = a, b
    assert (c0 == c1).all(), ctx
    assert (l0 == l1).all(), (ctx, np.argwhere(l0 != l1)[:5])
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all(), ctx


def filter_stats(expect_cluster=None):
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_kernel"] == 1 and st["tc_fallbacks"] == 0, st
    if expect_cluster is not None:
        assert st["tc_cluster"] == expect_cluster, st
    return st


def check_knn(gpu, queries, k, clusters):
    gpu.set_tensor_core_filter(2)
    ref = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 0
    for mode in (3, 4):
        gpu.set_tensor_core_filter(mode)
        got = gpu.search_knn(queries, k)
        filter_stats(clusters if mode == 4 else 1)
        same_bits(ref, got, (mode, k))
    return ref


def check_range(gpu, queries, knn_ref, clusters):
    d, _, c = knn_ref
    # radii between the 3rd and the 4th exact distance (or just above the last one found): every query has matches
    radii = np.array([np.nextafter(d[q, min(3, int(c[q]) - 1)], np.float32(np.inf)) for q in range(len(queries))], np.float32)
    max_out = 64
    gpu.set_tensor_core_filter(2)
    ref = gpu.search_range_batch(queries, radii, max_out)
    for mode in (3, 4):
        gpu.set_tensor_core_filter(mode)
        got = gpu.search_range_batch(queries, radii, max_out)
        filter_stats(clusters if mode == 4 else 1)
        D0, L0, N0 = ref
        D1, L1, N1 = got
        assert (N0 == N1).all(), mode
        for q in range(len(queries)):
            m = int(min(N0[q], max_out))
            assert (L0[q, :m] == L1[q, :m]).all(), (mode, q)
            assert (D0[q, :m].view(np.uint32) == D1[q, :m].view(np.uint32)).all(), (mode, q)


# rows: 100 = one tile whose second half is empty (the walker's second block has no row); 3000 = 24 tiles, most walkers get no
# block; 20000, 40000, 53700 and 70000 = walkers of 1 to 4 tiles (2 to 8 blocks: every residue mod 3), with a partial last tile
@pytest.mark.parametrize("n", [100, 3000, 20000, 40000, 53700, 70000])
@pytest.mark.parametrize("metric", [rx.IP, rx.L2])
def test_walker_block_counts(metric, n):
    dim, nq = 96, 96
    gpu = make_index(metric, n, dim, 0x7A00 + n)
    queries = make_queries(metric, nq, dim, 0x7A01 + n)
    ref = check_knn(gpu, queries, 10, clusters=1)
    check_range(gpu, queries, ref, clusters=1)
    gpu.close()


# kchunks = 1, 6, 12 (as many chunks as the ring has stages), 13 and 16 (more chunks than stages: a block wraps the ring)
@pytest.mark.parametrize("dim", [64, 768, 1536, 1600, 2048])
def test_chunk_counts(dim):
    n, nq = 30000, 160
    gpu = make_index(rx.IP, n, dim, 0x7B00 + dim)
    queries = make_queries(rx.IP, nq, dim, 0x7B01 + dim)
    ref = check_knn(gpu, queries, 10, clusters=2)
    check_range(gpu, queries, ref, clusters=2)
    check_knn(gpu, queries, 300, clusters=2)  # staged thresholds (k + 1 > 128)
    gpu.close()


@pytest.mark.parametrize("metric", [rx.IP, rx.COS])
def test_odd_query_block_count_in_clusters_of_two(metric):
    n, dim, nq = 45000, 256, 3 * 128 - 5  # three query blocks of 128: the cluster of two pads the last one
    gpu = make_index(metric, n, dim, 0x7C00)
    queries = make_queries(metric, nq, dim, 0x7C01)
    ref = check_knn(gpu, queries, 10, clusters=2)
    assert rx.last_search_stats()["query_tile"] == 2 * 128
    check_range(gpu, queries, ref, clusters=2)
    check_knn(gpu, queries, 500, clusters=2)
    gpu.close()


def test_every_dimension_keeps_its_query_block_and_queues():
    """The layout depends on the dimension only through kchunks = ceil(dim / 128): one batch of 1024 queries per kchunks covers
    every dimension from 1 to 2048.  Each must take the query block it took with two consumer warpgroups, and tcPrepare must find
    room for three queues of at least kTcQueueMin records (it refuses the launch otherwise)."""
    assert sorted({(dim + 127) // 128 for dim in range(1, 2049)}) == list(range(1, 17))
    nq = 1024
    for kchunks in range(1, 17):
        dim = kchunks * 128
        gpu = make_index(rx.IP, 2000, dim, 0x7D00 + dim)
        queries = make_queries(rx.IP, nq, dim, 0x7D01 + dim)
        gpu.set_tensor_core_filter(3)
        got = gpu.search_knn(queries, 4)
        st = filter_stats(1)
        assert st["query_tile"] == tc_query_block(nq, kchunks), (dim, st)
        gpu.set_tensor_core_filter(2)
        same_bits(gpu.search_knn(queries, 4), got, dim)
        gpu.close()
