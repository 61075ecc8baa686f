"""rxgpu_hnsw_build on the device: the exported graph equals the model of tests/hnsw_build_model.py list for list, builds are
deterministic, the graph is well formed at 200k rows, searches on it recall as well as on the reference's own graphs, it is searched
without an import, and every error leaves the index as it was."""
import numpy as np
import pytest

import reindexer_b200 as rx
from oracle import oracle as O

import hnsw_build_model as model

pytestmark = pytest.mark.gpu

F = np.float32


def labels(n, base=0):
    return (np.arange(base, base + n, dtype=np.uint64) << np.uint64(32))


def rows_for(seed, n, dim):
    return (np.random.default_rng(seed).standard_normal((n, dim)) * 0.5).astype(F)


def index_with(metric, rows, capacity=None):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], capacity or len(rows))
    gpu.add_points(labels(len(rows)), rows)
    return gpu


def graph_bytes(g):
    return [np.ascontiguousarray(g[k]).tobytes() for k in ("level0", "levels", "upper_offsets", "upper")] + [
        (g["n"], g["maxlevel"], g["enterpoint"])]


# ---------------------------------------------------------------------------------------------------------------- exact replay

REPLAY = [
    (rx.L2, 8, 16, 64, 2000),
    (rx.IP, 100, 2, 4, 2000),
    (rx.COS, 768, 32, 200, 1200),
    (rx.L2, 1, 2, 4, 1500),
    (rx.COS, 8, 16, 200, 2000),
    (rx.IP, 768, 16, 64, 1200),
    (rx.L2, 100, 32, 200, 2000),
    (rx.COS, 100, 2, 64, 2000),
    (rx.L2, 768, 2, 200, 1200),
]


@pytest.mark.parametrize("metric,dim,M,efc,n", REPLAY)
def test_exact_replay_from_scratch(metric, dim, M, efc, n):
    rows = rows_for(1000 * dim + M, n, dim)
    gpu = index_with(metric, rows)
    D = model.distance_table(gpu, metric, rows)
    levels, ends = rx.hnsw_build_plan(M, n)
    st = gpu.hnsw_build(M, efc)
    g, mst = model.build(D, M, efc, levels)
    model.assert_same_graph(gpu.hnsw_export(), g, (metric, dim, M, efc))
    assert st["batches"] == len(ends) and st["rows"] == n
    assert st["reverse_links"] == mst["reverse_links"] and st["lists_pruned"] == mst["lists_pruned"]
    assert st["distances"] > 0 and st["search_select_ms"] > 0
    gpu.close()


@pytest.mark.parametrize("metric,dim,M,efc", [(rx.L2, 16, 16, 64), (rx.COS, 100, 8, 200), (rx.IP, 8, 32, 4)])
def test_exact_replay_onto_a_reference_graph(metric, dim, M, efc):
    if not O.ref_knn_available():
        pytest.skip("the reference's HNSW is not built")
    n0, n = 1000, 2500
    rows = rows_for(77 + dim, n, dim)
    if metric == rx.COS:
        rows /= np.linalg.norm(rows.astype(np.float64), axis=1, keepdims=True).astype(F)
    ref = O.RefHnsw(metric, dim, n0, M=M, ef_construction=efc, seed=100)
    ref.add_batch(labels(n0), rows[:n0])
    rg = ref.export(with_vectors=False)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(labels(n0), rows[:n0])
    gpu.hnsw_import(rg)
    gpu.add_points(labels(n - n0, n0), rows[n0:])
    D = model.distance_table(gpu, metric, rows)
    levels, _ = rx.hnsw_build_plan(M, n, first=n0, maxlevel=int(rg["maxlevel"]), seed=7)
    st = gpu.hnsw_build(M, efc, first=n0, levels=levels)
    g, mst = model.build(D, M, efc, levels, model.Graph.from_dict(rg))
    model.assert_same_graph(gpu.hnsw_export(), g, (metric, dim, M, efc))
    assert st["rows"] == n - n0 and st["lists_pruned"] == mst["lists_pruned"]
    gpu.close()


@pytest.mark.parametrize("metric,M", [(rx.L2, 2), (rx.COS, 2), (rx.IP, 16)])
def test_exact_replay_with_duplicated_rows(metric, M):
    """a run of identical rows lands in one batch: ties everywhere, and one list receives far more links than Mcurmax"""
    n, dim = 3000, 12
    rows = rows_for(31 + M, n, dim)
    rows[2400:2700] = rows[7]
    rows[100:400:3] = rows[11]
    gpu = index_with(metric, rows)
    D = model.distance_table(gpu, metric, rows)
    levels, _ = rx.hnsw_build_plan(M, n)
    st = gpu.hnsw_build(M, 64)
    g, mst = model.build(D, M, 64, levels)
    model.assert_same_graph(gpu.hnsw_export(), g, (metric, M))
    assert mst["longest_segment"] > 2 * M, mst
    assert st["lists_pruned"] == mst["lists_pruned"] > 0
    gpu.close()


def test_exact_replay_with_a_list_receiving_more_than_64_links():
    """past 64 x 64 rows a batch holds more than 64 rows: a run of identical rows there sends them all to the same lists, so one
    reverse-link segment is longer than one distance gather"""
    n, dim, M = 4600, 6, 2
    rows = rows_for(57, n, dim)
    rows[4200:4500] = rows[9]
    gpu = index_with(rx.L2, rows)
    D = model.distance_table(gpu, rx.L2, rows)
    levels, _ = rx.hnsw_build_plan(M, n)
    st = gpu.hnsw_build(M, 32)
    g, mst = model.build(D, M, 32, levels)
    model.assert_same_graph(gpu.hnsw_export(), g, "long segment")
    assert mst["longest_segment"] > 64, mst
    assert st["lists_pruned"] == mst["lists_pruned"]
    gpu.close()


def test_append_needs_the_covered_rows_unchanged():
    dim, n0 = 16, 2000
    rows = rows_for(61, n0 + 500, dim)
    for mutate in ("upsert", "remove"):
        gpu = rx.GpuBruteforceSearch(rx.L2, dim, n0 + 500)
        gpu.add_points(labels(n0), rows[:n0])
        gpu.hnsw_build(16, 64)
        if mutate == "upsert":
            gpu.add_points(labels(1, 10), rows[n0 + 499:])  # row 10 rewritten in place
        else:
            gpu.remove_point(int(labels(1, 10)[0]))  # the last row moves into row 10
            gpu.add_points(labels(1, n0 + 1), rows[n0 + 1:n0 + 2])
        gpu.add_points(labels(400, n0 + 2), rows[n0 + 2:n0 + 402])
        with pytest.raises(rx.RxGpuError) as e:
            gpu.hnsw_build(16, 64, first=n0)
        assert e.value.code == 4, mutate
        gpu.close()
    gpu = index_with(rx.L2, rows[:n0], capacity=n0 + 500)  # appends alone are fine
    gpu.hnsw_build(16, 64)
    gpu.add_points(labels(500, n0), rows[n0:])
    gpu.hnsw_build(16, 64, first=n0)
    gpu.close()


def test_export_of_listed_nodes():
    rows = rows_for(3, 1500, 16)
    gpu = index_with(rx.L2, rows)
    gpu.hnsw_build(8, 32)
    full = gpu.hnsw_export()
    nodes = np.array([1499, 3, 0, 700, 3], np.uint32)
    part = gpu.hnsw_export(nodes)
    assert (part["level0"] == full["level0"][nodes]).all() and (part["levels"] == full["levels"][nodes]).all()
    for i, v in enumerate(nodes):
        a = part["upper"][part["upper_offsets"][i]:part["upper_offsets"][i + 1]]
        b = full["upper"][full["upper_offsets"][v]:full["upper_offsets"][v + 1]]
        assert (a == b).all()
    gpu.close()


# ---------------------------------------------------------------------------------------------------------------- determinism, search


def test_two_builds_give_the_same_bytes():
    rows = rows_for(9, 60_000, 48)
    a, b = index_with(rx.COS, rows), index_with(rx.COS, rows)
    a.hnsw_build(16, 100)
    b.hnsw_build(16, 100)
    assert graph_bytes(a.hnsw_export()) == graph_bytes(b.hnsw_export())
    a.close()
    b.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_searchable_without_import(metric):
    n, dim = 30_000, 32
    rows = rows_for(11 + metric, n, dim)
    built = index_with(metric, rows)
    built.hnsw_build(12, 80)
    imported = index_with(metric, rows)
    imported.hnsw_import(built.hnsw_export())
    q = rows_for(12, 256, dim)
    if metric == rx.COS:
        q = model.staged_rows(rx.COS, q)
    d1, l1, c1 = built.hnsw_search_knn(q, 10, 64)
    d2, l2, c2 = imported.hnsw_search_knn(q, 10, 64)
    assert (c1 == c2).all() and (l1 == l2).all() and (d1.view(np.uint32) == d2.view(np.uint32)).all()
    r1 = built.hnsw_search_range_batch(q[:16], np.full(16, d1[:16, 5].max(), F), 32, 1000)
    r2 = imported.hnsw_search_range_batch(q[:16], np.full(16, d1[:16, 5].max(), F), 32, 1000)
    for x, y in zip(r1, r2):
        assert (np.asarray(x) == np.asarray(y)).all()
    built.close()
    imported.close()


def test_invariants_at_200k_rows():
    n, dim, M = 200_000, 64, 16
    rows = rows_for(21, n, dim)
    gpu = index_with(rx.L2, rows)
    st = gpu.hnsw_build(M, 100)
    g = gpu.hnsw_export()
    lv = g["levels"]
    assert st["rows"] == n and int(lv[g["enterpoint"]]) == g["maxlevel"] == lv.max()

    def check(lists, owners, level, cap):
        cnt = lists[:, 0].astype(np.int64)
        assert (cnt <= cap).all() and (cnt >= 1).all(), level
        ids = lists[:, 1:]
        used = np.arange(ids.shape[1])[None, :] < cnt[:, None]
        assert (ids[used] < n).all(), level
        assert not (used & (ids == owners[:, None])).any(), ("self link", level)
        s = np.sort(np.where(used, ids.astype(np.int64), -1 - np.arange(ids.shape[1])[None, :]), axis=1)
        assert not (s[:, 1:] == s[:, :-1]).any(), ("duplicate", level)
        assert (lv[ids[used]] >= level).all(), ("neighbour below the list's level", level)

    check(g["level0"], np.arange(n), 0, 2 * M)
    for level in range(1, g["maxlevel"] + 1):
        owners = np.nonzero(lv >= level)[0]
        if len(owners) > 1:
            check(g["upper"][g["upper_offsets"][owners] + level - 1], owners, level, M)
    gpu.close()


# ---------------------------------------------------------------------------------------------------------------- quality


def recall(found, truth):
    return np.mean([len(set(f.tolist()) & set(t.tolist())) / len(t) for f, t in zip(found, truth)])


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_recall_against_the_reference_inserters(metric):
    if not O.ref_knn_available():
        pytest.skip("the reference's HNSW is not built")
    n, dim, M, efc = 200_000, 128, 16, 200
    rows = O.synth_matrix(0xB0D + metric, n, dim)
    if metric == rx.COS:
        rows = model.staged_rows(rx.COS, rows)
    q = O.synth_matrix(0xB0E + metric, 1024, dim)
    if metric == rx.COS:
        q = model.staged_rows(rx.COS, q)
    dev = index_with(metric, rows)
    dev.set_tensor_core_filter(2)
    _, truth, _ = dev.search_knn(q, 10)
    dev.hnsw_build(M, efc)
    graphs = {}
    import os
    for name, mt in (("single", False), ("multi", True)):
        ref = O.RefHnsw(metric, dim, n, M=M, ef_construction=efc, seed=100, multithread=mt)
        ref.add_batch(labels(n), rows, threads=os.cpu_count() if mt else 1)
        graphs[name] = index_with(metric, rows)
        graphs[name].hnsw_import(ref.export(with_vectors=False))
        del ref
    for ef in (64, 128):
        r_dev = recall(dev.hnsw_search_knn(q, 10, ef)[1], truth)
        for name, gi in graphs.items():
            r_ref = recall(gi.hnsw_search_knn(q, 10, ef)[1], truth)
            assert r_dev >= r_ref - 0.01, (metric, ef, name, r_dev, r_ref)
    dev.close()
    for gi in graphs.values():
        gi.close()


# ---------------------------------------------------------------------------------------------------------------- errors


def assert_unchanged(gpu, before, q, res):
    assert graph_bytes(gpu.hnsw_export()) == graph_bytes(before)
    d, l, c = gpu.hnsw_search_knn(q, 5, 32)
    assert (l == res[1]).all() and (d.view(np.uint32) == res[0].view(np.uint32)).all()


def test_errors_leave_the_index_unchanged():
    dim, n0, n = 16, 3000, 4000
    rows = rows_for(41, n, dim)
    fresh = index_with(rx.L2, rows[:100])
    for kw in (dict(M=1, ef_construction=64), dict(M=33, ef_construction=64), dict(M=16, ef_construction=3),
               dict(M=16, ef_construction=1025), dict(M=16, ef_construction=64, first=5),
               dict(M=16, ef_construction=64, levels=np.r_[np.zeros(99), -1].astype(np.int32))):
        with pytest.raises(rx.RxGpuError) as e:
            fresh.hnsw_build(**kw)
        assert e.value.code == 3, kw
    with pytest.raises(rx.RxGpuError) as e:  # no graph was left behind
        fresh.hnsw_export()
    assert e.value.code == 4
    fresh.close()
    wide = index_with(rx.L2, rows_for(42, 64, 12288))
    with pytest.raises(rx.RxGpuError) as e:  # dimension and ef beyond the shared-memory budget
        wide.hnsw_build(16, 1024)
    assert e.value.code == 3
    wide.close()

    # a workspace that does not fit: a visited bitmap per resident warp over 150M rows of capacity is more HBM than the card has
    big = rx.GpuBruteforceSearch(rx.L2, dim, 150_000_000)
    big.add_points(labels(100), rows[:100])
    with pytest.raises(rx.RxGpuError) as e:
        big.hnsw_build(16, 64)
    assert e.value.code == 37
    with pytest.raises(rx.RxGpuError) as e:
        big.hnsw_export()
    assert e.value.code == 4
    big.close()

    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.add_points(labels(n0), rows[:n0])
    gpu.hnsw_build(16, 64)
    gpu.add_points(labels(n - n0, n0), rows[n0:])
    for kw in (dict(M=16, ef_construction=64, first=0), dict(M=8, ef_construction=64, first=n0),
               dict(M=16, ef_construction=64, first=n0, levels=np.r_[np.zeros(n - n0 - 1), -1].astype(np.int32))):
        with pytest.raises(rx.RxGpuError) as e:
            gpu.hnsw_build(**kw)
        assert e.value.code == 3, kw
    gpu.hnsw_build(16, 64, first=n0)  # and the append itself still runs
    gpu.close()

    # the same checks on a graph whose rows are unchanged since the build, so its searches still run
    q = rows_for(43, 8, dim)
    gpu = index_with(rx.L2, rows[:n0])
    gpu.hnsw_build(16, 64)
    before, res = gpu.hnsw_export(), gpu.hnsw_search_knn(q, 5, 32)
    with pytest.raises(rx.RxGpuError) as e:
        gpu.hnsw_build(8, 64, first=n0)
    assert e.value.code == 3
    assert_unchanged(gpu, before, q, res)
    gpu.hnsw_mark_deleted(int(labels(1, 17)[0]))
    before, res = gpu.hnsw_export(), gpu.hnsw_search_knn(q, 5, 32)
    with pytest.raises(rx.RxGpuError) as e:  # tombstones: replace_deleted would reuse their slots, the builder only appends
        gpu.hnsw_build(16, 64, first=n0)
    assert e.value.code == 4
    assert_unchanged(gpu, before, q, res)
    gpu.close()
