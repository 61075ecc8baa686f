"""GPU tests of IVF indexes with more than 16 384 centroids (up to the reference's 131 072): the coarse pass tiled over (query tile x
centroid slice) with a radix select of the nprobe nearest centroids per query (reindexer_b200/csrc/ivf_coarse.cuh).  Compared with a
numpy model of the tie rule on integer-valued rows, with the reference's own FAISS over the same centroids and lists
(tests/ivf_lists_oracle.py: no k-means), with the exact scan at full probe, and with single-query calls."""
import numpy as np
import pytest
import ivf_lists_oracle as LO
from helpers import prep_query
from test_ivf_large_k_gpu import KEY_CAP, assert_matches_faiss, int_index, int_rows, same_bits

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu
needs_faiss = pytest.mark.skipif(not LO.available(), reason="needs tests/cpp/_build/libivf_lists_oracle.so (reference FAISS build)")

MAX_NLIST = 131072  # the reference's centroids_count bound (kIvfNCentroidsMax)
ERR_PARAMS = 3


def dist64(metric, x, q):
    q64 = q.astype(np.float64)
    return ((x.astype(np.float64) - q64) ** 2).sum(1) if metric == rx.L2 else -(x.astype(np.float64) @ q64)


def probed(metric, q, vecs, cents, sizes, nprobe):
    """rows of the nprobe lists nearest under (centroid distance, centroid id), their distances, and the sorted centroid distances"""
    cd = dist64(metric, cents, q)
    order = np.lexsort((np.arange(len(cents)), cd))
    mask = np.zeros(len(cents), bool)
    mask[order[:nprobe]] = True
    rows = np.nonzero(np.repeat(mask, sizes.astype(np.int64)))[0]
    return rows, dist64(metric, vecs[rows], q), cd[order]


def knn_model(rows, rd, labels, k):
    order = np.lexsort((rows, rd))[:k]
    sel_rows, sel_d = rows[order], rd[order]
    fin = np.lexsort((labels[sel_rows], sel_d))
    return sel_d[fin].astype(np.float32), labels[sel_rows][fin]


def range_model(rows, rd, labels, radius):
    hit = rd < radius
    r, d = rows[hit], rd[hit]
    fin = np.lexsort((labels[r], d))
    return d[fin].astype(np.float32), labels[r][fin]


@pytest.fixture(scope="module", params=[16385, 40000, MAX_NLIST])
def tie_index(request):
    out = {}
    for metric in (rx.L2, rx.IP):
        out[metric] = int_index(metric, 200000, 8, request.param, 2100 + request.param % 97 + metric)
    return request.param, out


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_tie_rule_against_numpy_model(tie_index, metric):
    nlist, idx = tie_index
    gpu, vecs, cents, labels, sizes = idx[metric]
    queries = int_rows(2200 + nlist % 89 + metric, 3, 8)
    ties = 0
    for nprobe in (1, 7, 1024, 1025, nlist):
        model = [probed(metric, q, vecs, cents, sizes, nprobe) for q in queries]
        ties += sum(nprobe < nlist and cds[nprobe - 1] == cds[nprobe] for _, _, cds in model)
        calls = [(256, gpu.ivf_search_knn_large_k(queries, 256, nprobe))]  # nprobe <= 1024: the fused path itself
        if nprobe <= 1024:
            calls.append((10, gpu.ivf_search_knn(queries, 10, nprobe)))
        for k in (257, 4099):
            calls.append((k, gpu.ivf_search_knn_large_k(queries, k, nprobe)))
        for k, (d, l, c) in calls:
            for i in range(len(queries)):
                md, ml = knn_model(model[i][0], model[i][1], labels, k)
                assert c[i] == len(md), (nlist, nprobe, k, i)
                assert (d[i, :c[i]] == md).all() and (l[i, :c[i]] == ml).all(), (nlist, nprobe, k, i)
        # range: the radius at the j-th model distance (strict: that group is out) and one ulp above it (the group is in)
        radii = []
        for rows, rd, _ in model:
            srt = np.sort(rd).astype(np.float32)
            r = srt[min(50, len(srt) - 1)] if len(srt) else np.float32(1.0)
            radii.append(r)
        radii = np.array(radii, np.float32)
        for rr in (radii, np.nextafter(radii, np.float32(np.inf))):
            bd, bl, bn = gpu.ivf_search_range_batch(queries, rr, nprobe, 100000)
            for i in range(len(queries)):
                md, ml = range_model(model[i][0], model[i][1], labels, rr[i])
                assert bn[i] == len(md), (nlist, nprobe, i)
                assert (bd[i, :bn[i]] == md).all() and (bl[i, :bn[i]] == ml).all(), (nlist, nprobe, i)
                sd, sl, _ = gpu.ivf_search_range(queries[i], float(rr[i]), nprobe)
                assert (sd == md).all() and (sl == ml).all(), (nlist, nprobe, i)
    assert ties >= 3  # the nprobe-th place fell inside a group of equal centroid distances: the centroid id decided


def grouped(list_nos, labels, vecs, nlist):
    """rows grouped by list (the imported layout), with the list sizes"""
    order = np.argsort(list_nos, kind="stable")
    return labels[order], vecs[order], np.bincount(list_nos, minlength=nlist).astype(np.uint64)


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("dim,nlist", [(16, 40000), (129, 30000), (768, 20000)])
def test_matches_reference_faiss(metric, dim, nlist):
    """random centroids and rows, lists drawn at random: FAISS and the device probe the same lists wherever centroid distances are apart
    by more than fp noise (at these nlist, the gap at the nprobe-th place is orders of magnitude wider)"""
    rng = np.random.default_rng(2300 + dim + metric)
    n = 60000 if dim < 500 else 30000
    cents = O.synth_matrix(2301 + dim, nlist, dim)
    vecs = O.synth_matrix(2302 + dim, n, dim)
    labels = O.row_labels(n)
    list_nos = rng.integers(0, nlist, n).astype(np.int64)
    ref = LO.ListsIvf(metric, cents, list_nos, labels, vecs)
    gl, gv, sizes = grouped(list_nos, labels, vecs, nlist)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(gl, gv)
    gpu.ivf_import(cents, sizes)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(2303 + dim, 6, dim)])
    for nprobe in (16, 300):
        for k in (10, 1000):
            d, l, c = gpu.ivf_search_knn_large_k(queries, k, nprobe)
            assert_matches_faiss(ref, metric, queries, k, nprobe, d, l, c, f"nlist {nlist}")
        d, l, c = gpu.ivf_search_knn(queries, 10, nprobe)
        assert_matches_faiss(ref, metric, queries, 10, nprobe, d, l, c, f"nlist {nlist} fused")
        for i, q in enumerate(queries[:2]):  # radius halfway between the 10th and 11th distance: clear of fp noise on both sides
            radius = float((d[i, 9] + np.float32(gpu.ivf_search_knn(q, 11, nprobe)[0][0, 10])) / 2)
            _, gl_, _ = gpu.ivf_search_range(q, radius, nprobe)
            _, rl = ref.range_search(q, radius if metric == rx.L2 else -radius, nprobe)
            assert set(gl_.tolist()) == set(rl.tolist()) == set(l[i].tolist()), (nlist, nprobe, i)
    st = rx.last_search_stats()
    assert st["algorithmic_bytes"] >= nlist * dim * 4  # the centroids, read once per query tile


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_full_probe_is_the_exact_scan(metric):
    n, dim, nlist = 100000, 64, 32768
    vecs, labels = O.synth_matrix(2400 + metric, n, dim), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(labels, vecs)
    sizes = np.random.default_rng(2401).multinomial(n, np.ones(nlist) / nlist).astype(np.uint64)
    gpu.ivf_import(O.synth_matrix(2402, nlist, dim), sizes)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(2403 + metric, 8, dim)])
    for k in (10, 1000):
        d, l, c = gpu.ivf_search_knn_large_k(queries, k, nlist)
        db, lb, cb = gpu.search_knn(queries, k)
        assert (c == k).all() and (cb == k).all()
        assert (l == lb).all() and (d.view(np.uint32) == db.view(np.uint32)).all(), k


def test_batches_equal_single_queries_across_key_chunks():
    """600 queries x 131 072 centroids = 78.6M coarse keys: above the key workspace, the coarse pass runs in two query chunks"""
    n, dim, nlist, nq = 300000, 24, MAX_NLIST, 600
    assert nq * nlist > KEY_CAP
    vecs, labels = O.synth_matrix(2500, n, dim), O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.add_points(labels, vecs)
    sizes = np.random.default_rng(2501).multinomial(n, np.ones(nlist) / nlist).astype(np.uint64)
    gpu.ivf_import(O.synth_matrix(2502, nlist, dim), sizes)
    queries = O.synth_matrix(2503, nq, dim)
    knn = gpu.ivf_search_knn(queries, 10, 32)
    st = rx.last_search_stats()
    assert st["launches"] == 2 * 4 + 2  # two coarse chunks (distances, select, sort, emit), list scans, merge
    big = gpu.ivf_search_knn_large_k(queries, 300, 1500)
    radii = knn[0][:, 9].copy()
    rb = gpu.ivf_search_range_batch(queries, radii, 32, 64)
    for i in list(range(0, nq, 23)) + [511, 512, nq - 1]:
        same_bits(tuple(x[i:i + 1] for x in knn), gpu.ivf_search_knn(queries[i], 10, 32))
        same_bits(tuple(x[i:i + 1] for x in big), gpu.ivf_search_knn_large_k(queries[i], 300, 1500))
        sd, sl, _ = gpu.ivf_search_range(queries[i], float(radii[i]), 32)
        assert rb[2][i] == len(sd) and (rb[1][i, :min(64, len(sd))] == sl[:64]).all(), i
        assert (rb[0][i, :min(64, len(sd))].view(np.uint32) == sd[:64].view(np.uint32)).all(), i


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.COS])
def test_mutable_lists_follow_reference_and_fresh_import(metric):
    """random rows (no bit-equal distances: the slab's row order and a fresh import's agree on every cut)"""
    dim, nlist, n0 = 16, 32768, 40000
    rng = np.random.default_rng(2600 + metric)
    total = n0 + 6000
    cents = O.synth_matrix(2601, nlist, dim)
    vecs = O.synth_matrix(2602, total, dim)
    labels = (rng.permutation(total).astype(np.uint64) << np.uint64(32)) | np.uint64(5)
    list0 = rng.integers(0, nlist, n0).astype(np.int64)
    ref = LO.ListsIvf(metric, cents, list0, labels[:n0], vecs[:n0])
    gpu = rx.GpuBruteforceSearch(metric, dim, 16)  # rows live in the lists
    gpu.ivf_create(cents)
    gpu.ivf_add(list0.astype(np.uint32), labels[:n0], vecs[:n0])
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(2603, 8, dim)])
    alive = {int(labels[i]): i for i in range(n0)}
    lists = {int(labels[i]): int(list0[i]) for i in range(n0)}

    def check(ctx):
        idx = np.array(sorted(alive.values()), np.int64)
        ln = np.array([lists[int(labels[i])] for i in idx], np.int64)
        gl, gv, sizes = grouped(ln, labels[idx], vecs[idx], nlist)
        fresh = rx.GpuBruteforceSearch(metric, dim, len(idx))
        fresh.add_points(gl, gv)
        fresh.ivf_import(cents, sizes)
        for k, nprobe in ((10, 8), (1000, 64), (100, 2000)):
            got = gpu.ivf_search_knn_large_k(queries, k, nprobe)
            same_bits(got, fresh.ivf_search_knn_large_k(queries, k, nprobe))
            assert_matches_faiss(ref, metric, queries, k, nprobe, *got, ctx)
        fresh.close()

    check("initial fill")
    done = n0
    for burst in (1, 500, 5499):
        new = slice(done, done + burst)
        ref.add(labels[new], vecs[new])
        ln = ref.list_of(labels[new])
        gpu.ivf_add(ln, labels[new], vecs[new])
        for j, lab in enumerate(labels[new]):
            alive[int(lab)] = done + j
            lists[int(lab)] = int(ln[j])
        done += burst
        for v in rng.choice(sorted(alive), size=min(len(alive) // 10, 2000), replace=False):
            ref.remove(int(v))
            gpu.ivf_remove(int(v))
            del alive[int(v)]
        check(f"after {done - n0} upserts")
    assert gpu.ivf_list_stats()["relocations"] > 0


def test_bounds_and_errors():
    dim = 8
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, 16)
    gpu.ivf_create(int_rows(2700, MAX_NLIST, dim))  # the reference's bound is accepted
    with pytest.raises(rx.RxGpuError) as e:
        gpu.ivf_create(int_rows(2701, MAX_NLIST + 1, dim))
    assert e.value.code == ERR_PARAMS and "131072" in e.value.what
    flat = rx.GpuBruteforceSearch(rx.L2, dim, 100)
    flat.add_points(O.row_labels(100), int_rows(2702, 100, dim))
    sizes = np.zeros(MAX_NLIST + 1, np.uint64)
    sizes[0] = 100
    with pytest.raises(rx.RxGpuError) as e:
        flat.ivf_import(int_rows(2703, MAX_NLIST + 1, dim), sizes)
    assert e.value.code == ERR_PARAMS
    q = int_rows(2704, 2, dim)
    with pytest.raises(rx.RxGpuError) as e:
        flat.ivf_search_knn(q, 10, 4)
    assert "no IVF lists imported" in e.value.what
    flat.ivf_import(int_rows(2705, MAX_NLIST, dim), sizes[:MAX_NLIST])
    d, l, c = flat.ivf_search_knn_large_k(q, 10, MAX_NLIST)  # every list probed: all 100 rows compete
    assert (c == 10).all()
    flat.add_point(int_rows(2706, 1, dim)[0], int(O.row_labels(100)[5]))  # a row was overwritten: the imported lists are stale
    for call in (lambda: flat.ivf_search_knn(q, 10, 4), lambda: flat.ivf_search_knn_large_k(q, 300, 4),
                 lambda: flat.ivf_search_range(q[0], 1.0, 4), lambda: flat.ivf_search_range_batch(q, 1.0, 4, 10)):
        with pytest.raises(rx.RxGpuError) as e:
            call()
        assert "changed after the IVF lists were imported" in e.value.what
