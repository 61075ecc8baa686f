"""GPU tests of the IVF search at any k (rxgpu_ivf_search_knn_large_k): one distance pass writes every probed row's key, an exact radix
select keeps the k best per query.  Compared with the reference's own FAISS (oracle/_ref: faiss::IndexIVFFlat trained and filled like
reindexer::IvfIndex, lists imported into the device index as in test_ivf_gpu.py), with the fused path where both serve a call, with the
exact brute-force scan at full probe, and with a numpy model of the tie rule on integer-valued rows."""
import numpy as np
import pytest
from helpers import ATOL, RTOL, prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not O.ref_ivf_available(), reason="needs oracle/_ref (reference FAISS build)")]

KEY_CAP = 1 << 26  # keys per query chunk of the select path (kIvfKeyCap, DESIGN.md §8.1)


def build(metric, n, dim, nlist, seed):
    vecs, labels = O.synth_matrix(seed, n, dim), O.row_labels(n)
    ref = O.RefIvf(metric, dim, nlist)
    ref.train_add(labels, vecs)
    st = ref.export()
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(st["labels"], st["vecs"])  # rows grouped by list, label = FAISS id
    gpu.ivf_import(st["centroids"], st["list_sizes"])
    return ref, gpu, st


def assert_matches_faiss(ref, metric, queries, k, nprobe, d, l, c, ctx=""):
    for i, q in enumerate(queries):
        dr, lr = ref.search(q, k, nprobe)
        assert c[i] == len(lr), (ctx, k, nprobe, i, c[i], len(lr))
        dr_map = dr if metric == rx.L2 else -dr  # FAISS reports +IP / +cos (descending); the map space is the negation (ascending)
        assert np.allclose(d[i, :c[i]], dr_map, rtol=RTOL, atol=ATOL), (ctx, k, nprobe, i)
        if not (l[i, :c[i]] == lr).all():  # ids may differ only where neighbouring distances are within fp noise
            bad = np.nonzero(l[i, :c[i]] != lr)[0]
            assert set(l[i, :c[i]]) == set(lr) or np.allclose(d[i, bad], dr_map[bad], rtol=1e-5), (ctx, k, nprobe, i)


def same_bits(a, b):
    (d0, l0, c0), (d1, l1, c1) = a, b
    assert (c0 == c1).all()
    for i in range(len(c0)):
        assert (l0[i, :c0[i]] == l1[i, :c1[i]]).all(), i
        assert (d0[i, :c0[i]].view(np.uint32) == d1[i, :c1[i]].view(np.uint32)).all(), i


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("dim", [32, 96, 768])
def test_large_k_matches_reference_faiss(metric, dim):
    n, nlist = (20000, 32) if dim < 500 else (8000, 16)
    ref, gpu, _ = build(metric, n, dim, nlist, 5100 + dim + metric)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(5200 + dim, 6, dim)])
    for k in (257, 300, 1000, 4096):
        for nprobe in (1, 4, nlist // 2, nlist):
            d, l, c = gpu.ivf_search_knn_large_k(queries, k, nprobe)
            assert_matches_faiss(ref, metric, queries, k, nprobe, d, l, c)
            st = rx.last_search_stats()
            assert st["passes"] == 1 and st["algorithmic_bytes"] >= int(c.sum()) * dim * 4


def int_rows(seed, n, dim, lo=-2, hi=3):
    return np.random.default_rng(seed).integers(lo, hi, size=(n, dim)).astype(np.float32)


def int_index(metric, n, dim, nlist, seed):
    """integer-valued rows and centroids (every distance exact in fp32, ties everywhere) in the imported layout: the rows of list l are
    one contiguous block, so internal row = index row; labels a random permutation so that label order differs from row order"""
    rng = np.random.default_rng(seed)
    sizes = rng.multinomial(n, np.ones(nlist) / nlist).astype(np.uint64)
    vecs = int_rows(seed + 1, n, dim)
    cents = int_rows(seed + 2, nlist, dim)
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(32)) | np.uint64(7)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(labels, vecs)
    gpu.ivf_import(cents, sizes)
    return gpu, vecs, cents, labels, sizes


def model(metric, q, vecs, cents, labels, sizes, k, nprobe):
    """numpy model of the IVF order: probed lists by (centroid distance, list), probed rows cut at k by (distance, row), the result
    ordered by (distance, label)"""
    q64 = q.astype(np.float64)
    dist = (lambda x: ((x.astype(np.float64) - q64) ** 2).sum(1)) if metric == rx.L2 else (lambda x: -(x.astype(np.float64) @ q64))
    cd = dist(cents)
    lists = sorted(range(len(cents)), key=lambda c: (cd[c], c))[:nprobe]
    begin = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
    rows = np.concatenate([np.arange(begin[c], begin[c + 1]) for c in lists])
    rd = dist(vecs[rows])
    order = np.lexsort((rows, rd))[:k]
    sel_rows, sel_d = rows[order], rd[order]
    fin = np.lexsort((labels[sel_rows], sel_d))
    return sel_d[fin].astype(np.float32), labels[sel_rows][fin], len(rows), rd


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_tie_rule_against_numpy_model(metric):
    # 100 000 rows: nprobe = nlist gives one query 100 000 keys (the multi-CTA select), nlist / 4 about 25 000 (one CTA per query)
    n, dim, nlist = 100000, 8, 16
    gpu, vecs, cents, labels, sizes = int_index(metric, n, dim, nlist, 61 + metric)
    queries = int_rows(71 + metric, 4, dim)
    straddles = 0
    for nprobe in (nlist // 4, nlist):
        for k in (257, 1000, 4099, 65535):
            d, l, c = gpu.ivf_search_knn_large_k(queries, k, nprobe)
            for i, q in enumerate(queries):
                md, ml, probed, rd = model(metric, q, vecs, cents, labels, sizes, k, nprobe)
                assert c[i] == min(k, probed), (nprobe, k, i)
                assert (d[i, :c[i]] == md).all() and (l[i, :c[i]] == ml).all(), (nprobe, k, i)
                srt = np.sort(rd)
                straddles += k < probed and srt[k - 1] == srt[k]
    assert straddles >= 8  # the cut fell inside a group of equal distances (the row word of the key decided)


def test_routing_gives_the_fused_path_bits():
    ref, gpu, _ = build(rx.L2, 12000, 48, 24, 811)
    queries = O.synth_matrix(812, 20, 48)
    tie, *_ = int_index(rx.IP, 30000, 8, 12, 813)
    tq = int_rows(814, 20, 8)
    for g, qs in ((gpu, queries), (tie, tq)):
        for k in (1, 10, 255, 256):
            for nprobe in (1, 5, 12):
                same_bits(g.ivf_search_knn_large_k(qs, k, nprobe), g.ivf_search_knn(qs, k, nprobe))


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_full_probe_is_the_exact_scan(metric):
    nlist = 20
    ref, gpu, _ = build(metric, 16000, 64, nlist, 900 + metric)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(901 + metric, 8, 64)])
    for k in (257, 1000, 5000):
        d, l, c = gpu.ivf_search_knn_large_k(queries, k, nlist)
        db, lb, cb = gpu.search_knn(queries, k)
        assert (c == k).all() and (cb == k).all()
        assert (l == lb).all() and (d.view(np.uint32) == db.view(np.uint32)).all(), k


def test_edges_and_errors():
    gpu, vecs, cents, labels, sizes = int_index(rx.L2, 20000, 8, 10, 333)
    q = int_rows(334, 3, 8)
    d, l, c = gpu.ivf_search_knn_large_k(q, 65535, 1)  # k above the probed rows: all of them
    for i in range(3):
        md, ml, probed, _ = model(rx.L2, q[i], vecs, cents, labels, sizes, 65535, 1)
        assert c[i] == probed and (l[i, :probed] == ml).all()
    d, l, c = gpu.ivf_search_knn_large_k(q, 65535, 10)
    assert (c == 20000).all()
    for k in (0, 65536):
        with pytest.raises(rx.RxGpuError):
            gpu.ivf_search_knn_large_k(q, k, 4)
    d, l, c = gpu.ivf_search_knn_large_k(np.zeros((0, 8), np.float32), 300, 4)  # nq = 0: nothing to do
    assert len(c) == 0
    gpu.add_point(vecs[0], int(labels[5]))  # a row was overwritten: the imported lists are stale
    with pytest.raises(rx.RxGpuError) as e:
        gpu.ivf_search_knn_large_k(q, 300, 4)
    assert "changed after the IVF lists were imported" in e.value.what
    fresh = rx.GpuBruteforceSearch(rx.L2, 8, 10)
    fresh.add_point(vecs[0], 1)
    with pytest.raises(rx.RxGpuError) as e:
        fresh.ivf_search_knn_large_k(q, 300, 4)
    assert "no IVF lists imported" in e.value.what


def test_nprobe_above_the_merge_fan_in():
    nlist = 2048
    ref, gpu, _ = build(rx.L2, 40000, 8, nlist, 1200)
    queries = O.synth_matrix(1201, 6, 8)
    for k, nprobe in ((100, 1500), (300, 1100), (1000, nlist)):
        d, l, c = gpu.ivf_search_knn_large_k(queries, k, nprobe)
        assert_matches_faiss(ref, rx.L2, queries, k, nprobe, d, l, c, "nprobe > 1024")
    with pytest.raises(rx.RxGpuError):
        gpu.ivf_search_knn(queries, 100, 1500)  # the fused path keeps its limit


def test_batches_equal_single_queries():
    ref, gpu, _ = build(rx.IP, 30000, 40, 32, 1300)
    queries = O.synth_matrix(1301, 300, 40)
    for k, nprobe in ((1000, 8), (300, 32)):
        single = [gpu.ivf_search_knn_large_k(q, k, nprobe) for q in queries]
        for nq in (1, 2, 33, 300):
            d, l, c = gpu.ivf_search_knn_large_k(queries[:nq], k, nprobe)
            for i in range(nq):
                same_bits((d[i:i + 1], l[i:i + 1], c[i:i + 1]), single[i])


def test_batch_above_the_key_cap_is_split():
    """1M rows, nprobe = nlist: every query has 1M keys (the multi-CTA select), 70 queries exceed the key workspace and run in chunks"""
    n, dim, nlist, nq, k = 1 << 20, 16, 64, 70, 1000
    assert nq * n > KEY_CAP
    vecs = O.synth_matrix(1400, n, dim)
    labels = O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, n)
    gpu.add_points(labels, vecs)
    gpu.ivf_import(O.synth_matrix(1401, nlist, dim), np.full(nlist, n // nlist, np.uint64))
    queries = O.synth_matrix(1402, nq, dim)
    batch = gpu.ivf_search_knn_large_k(queries, k, nlist)
    same_bits(batch, gpu.search_knn(queries, k))  # full probe = the exact scan
    for i in (0, 33, 69):
        same_bits(tuple(x[i:i + 1] for x in batch), gpu.ivf_search_knn_large_k(queries[i], k, nlist))


@pytest.mark.parametrize("metric,dim,nlist", [(rx.L2, 40, 24), (rx.COS, 96, 12)])
def test_mutable_lists_large_k_follow_reference(metric, dim, nlist):
    n0, seed = 8000, 1500 + dim
    vecs, labels = O.synth_matrix(seed, n0 + 3000, dim), O.row_labels(n0 + 3000)
    ref = O.RefIvf(metric, dim, nlist)
    ref.train_add(labels[:n0], vecs[:n0])
    st = ref.export()
    gpu = rx.GpuBruteforceSearch(metric, dim, 16)  # rows live in the lists, not in the flat index
    gpu.ivf_create(st["centroids"])
    gpu.ivf_add(ref.list_of(labels[:n0]), labels[:n0], vecs[:n0])
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(seed + 1, 10, dim)])
    rng = np.random.default_rng(seed)
    alive = set(labels[:n0].tolist())

    def check(ctx):
        for nprobe in (3, nlist):
            d, l, c = gpu.ivf_search_knn_large_k(queries, 1000, nprobe)
            assert_matches_faiss(ref, metric, queries, 1000, nprobe, d, l, c, ctx)

    check("initial fill")
    done = n0
    for burst in (1, 40, 900, 2059):
        new = slice(done, done + burst)
        ref.add(labels[new], vecs[new])
        gpu.ivf_add(ref.list_of(labels[new]), labels[new], vecs[new])
        alive |= set(labels[new].tolist())
        done += burst
        for v in rng.choice(sorted(alive), size=min(len(alive) // 10, 300), replace=False):
            ref.remove(int(v))
            gpu.ivf_remove(int(v))
            alive.discard(int(v))
        check(f"after {done - n0} upserts")
