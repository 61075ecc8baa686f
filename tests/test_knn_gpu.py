"""GPU parity tests (run with -m gpu on an H100): the CUDA brute-force path, called through the C ABI, against the oracle
(the reference's own code in oracle/_ref when present, else the pinned C port) and the committed golden fixtures."""
import threading

import numpy as np
import pytest
from conftest import GOLDEN_SYNTH_CASES, GOLDEN_TIE_CASES
from helpers import ATOL, RTOL, assert_same_knn, numpy_dists, prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def build_pair(metric, vecs, labels, capacity=None, host_mirror=False):
    n, dim = vecs.shape
    cap = capacity or n
    gpu = rx.GpuBruteforceSearch(metric, dim, cap, host_mirror=host_mirror)
    gpu.add_points(labels, vecs)
    cpu = O.best_bf(metric, dim, cap)
    assert cpu.add_batch(labels, vecs) == 0
    return gpu, cpu


def compare_queries(metric, gpu, cpu, queries, k, exact_ids=False):
    qs = np.stack([prep_query(metric, q) for q in queries])
    d, l, c = gpu.search_knn(qs, k)
    for i in range(len(qs)):
        dr, lr = cpu.search_knn(qs[i], k)
        assert c[i] == len(dr)
        if exact_ids:
            assert (l[i, :c[i]] == lr).all(), (i, l[i, :c[i]], lr)
            assert np.allclose(d[i, :c[i]], dr, rtol=RTOL, atol=ATOL)
        else:
            assert_same_knn(d[i, :c[i]], l[i, :c[i]], dr, lr, ctx=f"query {i}")


@pytest.mark.parametrize("name", GOLDEN_SYNTH_CASES)
def test_golden_synth(golden, name):
    metric, n, dim, k, nq, seed = (int(x) for x in golden[f"{name}/meta"])
    vecs, queries, labels = O.synth_matrix(seed, n, dim), O.synth_matrix(seed + 1, nq, dim), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(labels, vecs)
    qs = np.stack([prep_query(metric, q, use_ref=False) for q in queries])
    d, l, c = gpu.search_knn(qs, k)
    for i in range(nq):
        cnt = int(golden[f"{name}/count"][i])
        assert c[i] == cnt
        assert_same_knn(d[i, :cnt], l[i, :cnt], golden[f"{name}/dist"][i, :cnt], golden[f"{name}/label"][i, :cnt], ctx=f"{name} q{i}")
    rd, rl, total = gpu.search_range(qs[0], float(golden[f"{name}/range_radius"]))
    assert total == len(golden[f"{name}/range_label"])
    assert (rl == golden[f"{name}/range_label"]).all()
    assert np.allclose(rd, golden[f"{name}/range_dist"], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("name", GOLDEN_TIE_CASES)
def test_golden_ties_bit_exact(golden, name):
    """integer-valued vectors: every summation order gives the same sums, so labels AND their order must match exactly,
    including which of several bit-equal distances survive (the reference's heap tie rule)."""
    metric, n, dim, k, nq, _ = (int(x) for x in golden[f"{name}/meta"])
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(golden[f"{name}/labels"], golden[f"{name}/vecs"])
    for lab in golden[f"{name}/removes"]:
        gpu.remove_point(int(lab))
    qs = np.stack([prep_query(metric, q, use_ref=False) for q in golden[f"{name}/queries"]])
    d, l, c = gpu.search_knn(qs, k)
    replays = 0
    for i in range(nq):
        assert c[i] == k
        assert (l[i] == golden[f"{name}/label"][i]).all(), (name, i, l[i], golden[f"{name}/label"][i])
        assert np.allclose(d[i], golden[f"{name}/dist"][i], rtol=RTOL, atol=ATOL)
        # single-query calls agree with the batched call and report their tie replays
        d1, l1 = gpu.search_knn(qs[i], k)
        replays += rx.last_search_stats()["tie_replays"]
        assert (l1 == l[i]).all()
    assert replays > 0, "tie-heavy fixture never hit the replay path"


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("dim", [1, 3, 17, 100, 128, 130, 384, 768, 1000])
def test_parity_dims(metric, dim):
    n = 3000 if dim < 500 else 1500
    vecs, labels = O.synth_matrix(1000 + dim, n, dim), O.row_labels(n)
    gpu, cpu = build_pair(metric, vecs, labels)
    compare_queries(metric, gpu, cpu, O.synth_matrix(2000 + dim, 7, dim), 10)


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("k,nq", [(1, 1), (2, 3), (10, 1), (10, 2), (10, 9), (37, 5), (100, 4), (254, 2)])
def test_parity_k_and_batch(metric, k, nq):
    n, dim = 5000, 64
    vecs, labels = O.synth_matrix(77, n, dim), O.row_labels(n)
    gpu, cpu = build_pair(metric, vecs, labels)
    compare_queries(metric, gpu, cpu, O.synth_matrix(78, nq, dim), k)
    for qt in (1, 2, 4):  # every query-tile variant gives the same answer
        gpu.set_query_tile(qt)
        compare_queries(metric, gpu, cpu, O.synth_matrix(78, nq, dim), k)


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("k", [255, 256, 300, 1000, 2500, 6000])
def test_parity_large_k(metric, k):
    """k + 1 > 256 is answered in rounds of 256 results (one pass per round, floor key between rounds); the reference's tests go to
    k = 1000 (gtests/tests/unit/float_vector_index.cc)."""
    n, dim = 5000, 64
    vecs, labels = O.synth_matrix(177, n, dim), O.row_labels(n)
    gpu, cpu = build_pair(metric, vecs, labels)
    compare_queries(metric, gpu, cpu, O.synth_matrix(178, 3, dim), k)
    assert rx.last_search_stats()["passes"] >= (min(k + 1, n) + 255) // 256


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
@pytest.mark.parametrize("k", [300, 777])
def test_large_k_ties_bit_exact(metric, k):
    """tie-heavy integer vectors with k beyond one round: labels and order equal the reference's heap result bit for bit, including
    the tie replay over a first-k-rows scan that itself spans several rounds"""
    n, dim = 4000, 6
    rng = np.random.default_rng(4242 + k)
    vecs = rng.integers(-2, 3, size=(n, dim)).astype(np.float32)
    labels = O.row_labels(n)[rng.permutation(n)]
    gpu, cpu = build_pair(metric, vecs, labels)
    for lab in labels[rng.choice(n, 40, replace=False)]:
        gpu.remove_point(int(lab))
        cpu.remove(int(lab))
    qs = rng.integers(-2, 3, size=(4, dim)).astype(np.float32)
    compare_queries(metric, gpu, cpu, qs, k, exact_ids=True)
    d1, l1 = gpu.search_knn(qs[0], k)
    assert rx.last_search_stats()["tie_replays"] == 1


def test_batch_equals_single_queries_bitwise():
    n, dim = 20000, 128
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.add_points(O.row_labels(n), O.synth_matrix(5, n, dim))
    qs = O.synth_matrix(6, 11, dim)
    d, l, c = gpu.search_knn(qs, 10)
    for i in range(len(qs)):
        d1, l1 = gpu.search_knn(qs[i], 10)
        assert (l1 == l[i]).all() and (d1 == d[i]).all()  # identical per-row arithmetic in every kernel variant


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_empty_small_and_k_larger_than_n(metric):
    dim = 32
    gpu = rx.GpuBruteforceSearch(metric, dim, 64)
    q = prep_query(metric, O.synth(1, 0, dim))
    d, l = gpu.search_knn(q, 10)
    assert len(d) == 0
    rd, rl, total = gpu.search_range(q, 1e9)
    assert total == 0
    vecs, labels = O.synth_matrix(3, 7, dim), O.row_labels(7)
    gpu.add_points(labels, vecs)
    cpu = O.best_bf(metric, dim, 64)
    cpu.add_batch(labels, vecs)
    for k in (1, 6, 7, 8, 50):
        d, l = gpu.search_knn(q, k)
        dr, lr = cpu.search_knn(q, k)
        assert len(d) == len(dr) == min(k, 7) and (l == lr).all()
    d, l, c = gpu.search_knn(np.stack([q, q]), 0)
    assert (c == 0).all()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_maintenance_semantics(metric):
    """upsert of existing labels, swap-with-last deletes (internal order changes!), resize, clone, capacity errors."""
    rng = np.random.default_rng(5 + metric)
    n, dim, cap = 2000, 48, 2100
    vecs, labels = O.synth_matrix(40 + metric, n, dim), O.row_labels(n)
    gpu, cpu = build_pair(metric, vecs, labels, capacity=cap, host_mirror=True)
    queries = O.synth_matrix(50 + metric, 6, dim)
    for lab in labels[rng.choice(n, 300, replace=False)]:
        gpu.remove_point(int(lab))
        cpu.remove(int(lab))
    gpu.remove_point(1 << 60)  # unknown label: no-op like the reference
    newl = np.concatenate([labels[rng.choice(n, 40, replace=False)], O.row_labels(60, first_row=n + 10)])
    newl = np.unique(newl)
    present = np.array([cpu.get(int(x)) is not None for x in newl])
    newv = O.synth_matrix(60 + metric, len(newl), dim)
    gpu.add_points(newl, newv)
    cpu.add_batch(newl, newv)
    assert present.any() and (~present).any()
    assert gpu.size() == cpu.size()
    compare_queries(metric, gpu, cpu, queries, 10)
    # single-row upserts, including a duplicate label inside one batch (last write wins, applied in order)
    gpu.add_point(newv[0], int(newl[1]))
    cpu.add(newv[0], int(newl[1]))
    dupl = np.array([newl[2], newl[2], newl[3]], np.uint64)
    dupv = O.synth_matrix(61 + metric, 3, dim)
    gpu.add_points(dupl, dupv)
    cpu.add_batch(dupl, dupv)
    compare_queries(metric, gpu, cpu, queries, 10)
    assert np.array_equal(gpu.float_ptr_by_external_label(int(newl[2])), dupv[1])
    assert gpu.element_size() == cpu.element_size() == dim * 4 + 8
    # clone is a deep copy
    clone = gpu.clone(cap + 100)
    assert clone.max_elements() == cap + 100 and clone.size() == gpu.size()
    gpu.remove_point(int(newl[0]))
    cpu_before = cpu.clone(cap + 100)
    cpu.remove(int(newl[0]))
    compare_queries(metric, clone, cpu_before, queries, 10)
    compare_queries(metric, gpu, cpu, queries, 10)
    # resize
    gpu.resize_index(cap * 2)
    cpu.resize(cap * 2)
    assert gpu.max_elements() == cap * 2
    compare_queries(metric, gpu, cpu, queries, 10)
    with pytest.raises(rx.RxGpuError) as e:
        gpu.resize_index(10)
    assert "Cannot resize, max element is less than the current number of elements" in e.value.what
    small = rx.GpuBruteforceSearch(metric, dim, 2)
    small.add_points(labels[:2], vecs[:2])
    with pytest.raises(rx.RxGpuError) as e:
        small.add_point(vecs[2], int(labels[2]))
    assert "The number of elements exceeds the specified limit" in e.value.what
    small.add_point(vecs[2], int(labels[1]))  # upsert of a present label still fits
    with pytest.raises(rx.RxGpuError) as e:
        small.float_ptr_by_external_label(12345)
    assert "Label not found" in e.value.what


def test_get_without_host_mirror():
    n, dim = 100, 20
    vecs, labels = O.synth_matrix(9, n, dim), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.add_points(labels, vecs)
    for i in (0, 57, 99):
        assert np.array_equal(gpu.float_ptr_by_external_label(int(labels[i])), vecs[i])


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_range_search(metric):
    n, dim = 4000, 40
    vecs, labels = O.synth_matrix(300 + metric, n, dim), O.row_labels(n)
    gpu, cpu = build_pair(metric, vecs, labels)
    q = prep_query(metric, O.synth(301, 0, dim))
    dr, lr = cpu.search_knn(q, 200)
    for cut in (0, 1, 17, 150):
        # radii sit halfway between neighbouring distances (or clearly below the best) so fp noise cannot move a row across
        radius = float((dr[cut] + dr[cut + 1]) / 2) if cut else float(dr[0] - 0.01 * abs(dr[0]) - 1e-3)
        d, l, total = gpu.search_range(q, radius)
        dc, lc = cpu.search_range(q, radius)
        assert total == len(lc) == (cut + 1 if cut else 0)
        assert (l == lc).all() and np.allclose(d, dc, rtol=RTOL, atol=ATOL)
    d, l, total = gpu.search_range(q, float(dr[150]), max_out=10)  # truncated output keeps the best
    assert total >= 150 and len(l) == 10 and (l == lr[:10]).all()


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_select_matches_reference_contract(metric):
    """FloatVectorIndex::Select contract as the reference's tests assert it (float_vector_index.cc:32-86): rank monotone
    (ascending for L2, descending for IP / Cosine), ties by ascending row id, Cosine in [-1, 1], radius respected; checked
    against the oracle's restatement of HnswIndexBase::select on the oracle's own search results."""
    n, dim, k = 3000, 24, 25
    base = O.synth_matrix(400 + metric, n // 3, dim)
    vecs = np.repeat(base, 3, axis=0)  # array-style duplicates: rowId r has arrayIdx 0..2 with identical vectors
    labels = (np.repeat(np.arange(n // 3), 3).astype(np.uint64) << np.uint64(32)) | np.tile(np.arange(3), n // 3).astype(np.uint64)
    perm = np.random.default_rng(3).permutation(n)
    vecs, labels = vecs[perm], labels[perm]
    gpu, cpu = build_pair(metric, vecs, labels)
    for q in O.synth_matrix(401 + metric, 5, dim):
        qn = prep_query(metric, q)
        dr, lr = cpu.search_knn(qn, k)
        for is_array in (False, True):
            ids, ranks = gpu.select(q, k=k, is_array=is_array)
            ids_o, ranks_o = O.select_postprocess(metric, dr, lr, is_array=is_array, k=k)
            assert ids.tolist() == ids_o.tolist()
            assert np.allclose(ranks, ranks_o, rtol=RTOL, atol=ATOL)
            sign = 1 if metric == rx.L2 else -1
            assert (np.diff(sign * ranks) >= 0).all()
            if metric == rx.COS:
                assert (np.abs(ranks) <= 1 + 1e-5).all()
            if is_array:
                assert len(set(ids.tolist())) == len(ids)
        ids_raw, _ = gpu.select(q, k=k, raw=True)
        assert ids_raw.tolist() == O.select_postprocess(metric, dr, lr, raw=True, k=k)[0].tolist()
        # radius (user space: +IP / +cos, squared L2) and k + radius
        cut = 11
        r_map = float((dr[cut] + dr[cut + 1]) / 2)
        r_user = r_map if metric == rx.L2 else -r_map
        ids, ranks = gpu.select(q, radius=r_user)
        assert len(ids) == cut + 1 and ((ranks < r_user).all() if metric == rx.L2 else (ranks > r_user).all())
        ids2, _ = gpu.select(q, k=5, radius=r_user)
        assert ids2.tolist() == ids[:5].tolist()


def test_concurrent_searches_are_reentrant():
    """the reference issues K / K+R / R queries from 4 threads against one index (float_vector_index.cc:257-294, :548)"""
    n, dim = 30000, 64
    vecs, labels = O.synth_matrix(500, n, dim), O.row_labels(n)
    gpu, cpu = build_pair(rx.L2, vecs, labels)
    queries = O.synth_matrix(501, 32, dim)
    expected = [cpu.search_knn(q, 10) for q in queries]
    errors = []

    def worker(tid):
        try:
            for rep in range(6):
                for i in range(tid, len(queries), 4):
                    d, l = gpu.search_knn(queries[i], 10)
                    assert_same_knn(d, l, expected[i][0], expected[i][1], ctx=f"thread {tid} q{i}")
                    rd, rl, total = gpu.search_range(queries[i], float(expected[i][0][3] + expected[i][0][4]) / 2)
                    assert total == 4
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]


def test_device_resident_api_and_shard_merge():
    """rxgpu_search_knn_device on two shards of one data set + rxgpu_merge_shards == one index over everything."""
    import torch

    n, dim, k, nq = 12000, 96, 10, 6
    vecs, labels = O.synth_matrix(600, n, dim), O.row_labels(n)
    full, cpu = build_pair(rx.IP, vecs, labels)
    half = n // 2
    shards = [rx.GpuBruteforceSearch(rx.IP, dim, half) for _ in range(2)]
    shards[0].add_points(labels[:half], vecs[:half])
    shards[1].add_points(labels[half:], vecs[half:])
    queries = O.synth_matrix(601, nq, dim)
    dq = torch.from_numpy(queries).cuda()
    k1 = k + 1
    D = np.zeros((2, nq, k1), np.float32)
    I = np.zeros((2, nq, k1), np.uint32)
    L = np.zeros((2, nq, k1), np.uint64)
    Cn = np.zeros((2, nq), np.uint32)
    for s, sh in enumerate(shards):
        od = torch.zeros((nq, k1), dtype=torch.float32, device="cuda")
        oi = torch.zeros((nq, k1), dtype=torch.int32, device="cuda")
        ol = torch.zeros((nq, k1), dtype=torch.int64, device="cuda")
        oc = torch.zeros((nq,), dtype=torch.int32, device="cuda")
        sh.search_knn_device(nq, dq.data_ptr(), k1, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr(),
                             torch.cuda.current_stream().cuda_stream)
        D[s], I[s] = od.cpu().numpy(), oi.cpu().numpy().view(np.uint32)
        L[s], Cn[s] = ol.cpu().numpy().view(np.uint64), oc.cpu().numpy().view(np.uint32)
    od, og, ol, oc, nt = rx.merge_shards(k, D, I, L, Cn, np.array([0, half], np.uint64))
    d_full, l_full, c_full = full.search_knn(queries, k)
    assert not nt.any()
    assert (ol == l_full).all() and (od == d_full).all() and (oc == k).all()
    for i in range(nq):
        dr, lr = cpu.search_knn(queries[i], k)
        assert_same_knn(od[i], ol[i], dr, lr)


def test_full_size_properties():
    """BASELINE config 1 shape (768-dim, inner product, k=10) at a size that needs the device generator: properties that do
    not need a CPU scan of everything -- planted neighbours are found, returned distances recompute on the host from the
    generator, no sampled row beats the k-th, shard merge equals the single index, rows sorted."""
    dim, k = 768, 10
    free_b, _ = __import__("torch").cuda.mem_get_info()
    n = 10_000_000 if free_b > 70e9 else 2_000_000
    seed, nq = 0x5EED0001, 8
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n + 16)
    gpu.append_synth(seed, 0, n)
    assert gpu.size() == n
    queries = O.synth_matrix(seed + 1, nq, dim)
    # plant: row n+i = 3 * query_i  => inner product 3*|q|^2, far above any random row
    planted = (queries * 3.0).astype(np.float32)
    gpu.add_points(O.row_labels(nq, first_row=n), planted)
    d, l, c = gpu.search_knn(queries, k)
    stats = rx.last_search_stats()
    assert (c == k).all() and stats["passes"] == 2 and stats["query_tile"] == 4
    rng = np.random.default_rng(1)
    sample_rows = np.sort(rng.choice(n, 4096, replace=False))
    sample = np.stack([O.synth(seed, int(r) * dim, dim) for r in sample_rows])
    for i in range(nq):
        assert l[i, 0] == (n + i) << 32
        assert abs(d[i, 0] + 3 * float(queries[i].astype(np.float64) @ queries[i].astype(np.float64))) < 1e-3 * abs(d[i, 0])
        assert (np.diff(d[i]) >= 0).all()
        rows = (l[i, 1:] >> np.uint64(32)).astype(np.int64)
        assert len(set(rows.tolist())) == k - 1 and (rows < n + nq).all()

        def row_vec(r):  # other queries' planted rows (3 * q_j, large norm) may legitimately rank high too
            return planted[r - n] if r >= n else O.synth(seed, int(r) * dim, dim)

        recomputed = np.array([-(row_vec(int(r)).astype(np.float64) @ queries[i].astype(np.float64)) for r in rows])
        assert np.allclose(d[i, 1:], recomputed, rtol=RTOL, atol=ATOL)
        assert (numpy_dists(rx.IP, queries[i], sample) >= d[i, -1] - 1e-4).all()  # nothing sampled beats the k-th
    # range over the full index: strictly-below-radius rows are exactly the first m of the knn answer
    radius = float((d[0, 4] + d[0, 5]) / 2)
    rd, rl, total = gpu.search_range(queries[0], radius)
    assert total == 5 and (rl == l[0, :5]).all()
