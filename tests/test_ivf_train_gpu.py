"""GPU tests of IVF training and list assignment on the device (rxgpu_ivf_train / _assign / _add_assign, reindexer_b200/csrc/
ivf_train.cu): bit-identical to the reference's FAISS k-means where every assignment is unambiguous (tests/ivf_train_oracle.py), the
assignment equal to the coarse pass's first probe and the update equal to a numpy restatement at the shape boundaries, determinism, the
error cases, and adds through the device's assignment against FAISS filled with the same lists (tests/ivf_lists_oracle.py)."""
import ctypes as C

import ivf_lists_oracle as LO
import ivf_train_oracle as TO
import numpy as np
import pytest

import reindexer_b200 as rx
from oracle import oracle as O
from test_ivf_large_k_gpu import assert_matches_faiss

pytestmark = pytest.mark.gpu
needs_faiss = pytest.mark.skipif(not (TO.available() and LO.available()), reason="needs the reference FAISS build (tests/cpp/_build)")
ERR_PARAMS, ERR_LOGIC, ERR_SYSTEM = 3, 4, 37
COARSE_MAX_DIM = 51200  # the coarse pass stages one query of at most 400 x 128 floats in shared memory


def normalized(metric, x):
    """the vectors as the coarse quantiser sees them: Cosine normalised as rxgpu_select_knn normalises a query"""
    return np.stack([O.normalize_copy(v, use_ref=False)[0] for v in x]) if metric == rx.COS else x


def sites(seed, nlist, n, dim, metric):
    """n points that are duplicates of nlist + nlist / 2 integer sites spread far apart: every distance the assignment compares differs
    by far more than FAISS's BLAS-formula rounding, and duplicated initial centroids force empty clusters and splits"""
    rng = np.random.default_rng(seed)
    s = set()
    while len(s) < nlist + nlist // 2:
        s.add(tuple(int(v) for v in rng.integers(-500, 501, dim)))
    s = np.array(sorted(s), np.float32)
    idx = rng.integers(0, len(s), n)
    idx[:min(n, len(s))] = np.arange(min(n, len(s)))
    rng.shuffle(idx)
    return s[idx]


def ambiguous(metric, x, c):
    """points whose two nearest distinct centroids are within fp32 rounding of each other (in fp64)"""
    x64, c64 = x.astype(np.float64), c.astype(np.float64)
    if metric == rx.L2:
        d = ((x64[:, None, :] - c64[None]) ** 2).sum(2)
    else:
        d = -(x64 @ (c64 / np.linalg.norm(c64, axis=1, keepdims=True)).T) if metric == rx.COS else -(x64 @ c64.T)
    if d.shape[1] < 2:
        return 0
    o = np.argsort(d, 1, kind="stable")
    s = np.take_along_axis(d, o, 1)
    same = (c[o[:, 0]] == c[o[:, 1]]).all(1)
    return int(((s[:, 1] - s[:, 0] < 1e-5 * (np.abs(s[:, 0]) + 1)) & ~same).sum())


def ulp_diff(a, b):
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def train(metric, x, nlist, **kw):
    g = rx.GpuBruteforceSearch(metric, x.shape[1], 1)
    c, st = g.ivf_train(nlist, x, **kw)
    return g, c, st


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("mult", [1, 39, 300])
def test_bit_identical_to_faiss_when_unambiguous(metric, mult):
    nlist, dim = 8, 4
    x = sites(7 + metric, nlist, nlist * mult, dim, metric)
    sample, _ = rx.kmeans_plan(len(x), nlist)
    xt = normalized(metric, x)[sample]
    splits = 0
    for niter in range(11):
        want, _, nsplit = TO.train(metric, x, nlist, niter=niter)
        assert ambiguous(metric, xt, want) == 0, "test data: FAISS's iteration %d has near-tied assignments" % niter
        if niter not in (0, 1, 10):
            continue
        g, got, st = train(metric, x, nlist, niter=niter)
        if metric == rx.L2:
            assert (got.view(np.uint32) == want.view(np.uint32)).all(), niter
        else:
            assert ulp_diff(got, want).max() <= 2, (niter, ulp_diff(got, want).max())
        if mult > 1:
            assert [s["nsplit"] for s in st] == nsplit[:niter].tolist()
            splits = sum(nsplit)
        assert g.ivf_size() == 0 and g.size() == 0
        # the trained lists answer like rxgpu_ivf_create over the same centroids
        ln, _ = g.ivf_assign(x)
        g2 = rx.GpuBruteforceSearch(metric, dim, 1)
        g2.ivf_create(got)
        assert (g2.ivf_assign(x)[0] == ln).all()
        g.close()
        g2.close()
    if mult > 1:
        assert splits > 0  # the data does exercise split_clusters


# (nlist, dim) over the boundaries of the assignment kernel's centroid groups, the coarse pass's slices and its query staging
SHAPES = [(1, 1), (2, 3), (4095, 128), (4096, 3), (4097, 768), (16385, 128), (131072, 128), (2, COARSE_MAX_DIM), (4097, 1)]


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{a}x{b}" for a, b in SHAPES])
def test_assignment_is_the_first_probe_and_update_matches_numpy(metric, shape):
    nlist, dim = shape
    n = max(2 * nlist + 3, 64) if dim < 10000 else 40
    x = O.synth_matrix(0x7A1 + nlist + dim + metric, n, dim)
    g0, c0, _ = train(metric, x, nlist, niter=0)
    sample, init = rx.kmeans_plan(n, nlist)
    xs = normalized(metric, x)
    if metric == rx.L2:
        assert (c0 == x[init]).all()
    ln, dist = g0.ivf_assign(x)
    # the coarse pass itself: list c holds the single row "centroid c, label c"; the nearest row at nprobe 1 is the first probe's
    # (the list scan's fused top-k stages a query in at most 100 KB of shared memory: the widest shape is compared with fp64 instead)
    if dim <= 16384:
        probe = rx.GpuBruteforceSearch(metric, dim, 1)
        probe.ivf_create(c0)
        probe.ivf_add(np.arange(nlist), np.arange(nlist), c0)
        _, lab, cnt = probe.ivf_search_knn(xs, 1, 1)
        assert (cnt == 1).all() and (lab[:, 0] == ln).all()
        probe.close()
    else:
        c64 = c0.astype(np.float64)
        if metric == rx.COS:
            c64 = c64 / np.linalg.norm(c64, axis=1, keepdims=True)
        d64 = ((xs.astype(np.float64)[:, None, :] - c64[None]) ** 2).sum(2) if metric == rx.L2 else -(xs.astype(np.float64) @ c64.T)
        clear = np.sort(d64, 1)[:, 1] - np.sort(d64, 1)[:, 0] > 1e-5 * (np.abs(d64).max(1) + 1e-3)
        assert clear.mean() >= 0.9 and (d64.argmin(1) == ln)[clear].all()
    # one iteration from the same start: the update of the device's own assignment, summed in ascending point order in fp32
    g1, c1, st = train(metric, x, nlist, niter=1)
    if st[0]["nsplit"] == 0:  # duplicates among the initial centroids leave clusters empty; their splits are checked against FAISS
        a, xt = ln[sample], xs[sample]
        order = np.argsort(a, kind="stable")
        counts = np.bincount(a, minlength=nlist)
        starts = np.searchsorted(a[order], np.arange(nlist))
        sums = np.zeros((nlist, dim), np.float32)
        for r in range(counts.max()):
            cl = np.nonzero(counts > r)[0]
            sums[cl] += xt[order[starts[cl] + r]]
        want = sums * (np.float32(1) / np.maximum(counts, 1).astype(np.float32))[:, None]
        if metric == rx.L2:
            assert (c1.view(np.uint32) == want.view(np.uint32)).all()
        else:  # spherical: renormalised with an fp64 norm, rounded once
            w64 = want.astype(np.float64)
            want = (w64 / np.sqrt((w64 ** 2).sum(1, keepdims=True))).astype(np.float32)
            assert ulp_diff(c1, want).max() <= 1
    g0.close()
    g1.close()


def test_deterministic_and_stats():
    x = O.synth_matrix(0xD5, 20000, 64)
    for metric in (rx.L2, rx.COS):
        ga, ca, sa = train(metric, x, 300, niter=5)
        gb, cb, sb = train(metric, x, 300, niter=5)
        assert (ca.view(np.uint32) == cb.view(np.uint32)).all()
        assert [s["obj"] for s in sa] == [s["obj"] for s in sb] and [s["nsplit"] for s in sa] == [s["nsplit"] for s in sb]
        assert all(s["assign_ms"] > 0 and s["update_ms"] > 0 for s in sa)
        if metric == rx.L2:  # Lloyd iterations never make the objective worse
            assert sa[-1]["obj"] <= sa[0]["obj"]
        assert (ga.ivf_assign(x)[0] == gb.ivf_assign(x)[0]).all()
        ga.close()
        gb.close()


def _unchanged(g):
    assert g.ivf_size() == 0
    with pytest.raises(rx.RxGpuError) as e:
        g.ivf_assign(np.zeros((1, g.dim), np.float32))
    assert e.value.code == ERR_LOGIC


def test_errors_leave_the_index_unchanged():
    dim = 16
    x = O.synth_matrix(0xE1, 500, dim)
    g = rx.GpuBruteforceSearch(rx.COS, dim, 1000)
    bad = x.copy()
    bad[77, 3] = np.nan
    inf = x.copy()
    inf[5, 0] = np.inf
    cases = [(dict(nlist=10, vecs=bad), ERR_PARAMS), (dict(nlist=10, vecs=inf), ERR_PARAMS), (dict(nlist=600, vecs=x), ERR_PARAMS),
             (dict(nlist=0, vecs=x), ERR_PARAMS), (dict(nlist=131073, vecs=x), ERR_PARAMS), (dict(nlist=10, vecs=x, seed=-1), ERR_PARAMS),
             (dict(nlist=10, vecs=x, max_points_per_centroid=0), ERR_PARAMS), (dict(nlist=10, vecs=x, niter=-1), ERR_PARAMS),
             (dict(nlist=10, vecs=x, norm_coefs=np.full(500, np.nan, np.float32)), ERR_PARAMS)]
    for kw, code in cases:
        with pytest.raises(rx.RxGpuError) as e:
            g.ivf_train(**kw)
        assert e.value.code == code, kw
        _unchanged(g)
    # more points than device memory can hold: refused before the input is read (the array is one row long)
    lib = rx.lib()
    one = np.zeros(dim, np.float32)
    prm = rx.binding.IvfTrainParams(1, 1234, 2**31 - 1)
    big = rx.GpuBruteforceSearch(rx.L2, COARSE_MAX_DIM, 1)
    rc = lib.rxgpu_ivf_train(big._h, 10, 2**31 - 1, one.ctypes.data_as(C.POINTER(C.c_float)), None, C.byref(prm), None, None)
    assert rc == ERR_SYSTEM
    _unchanged(big)
    big.close()
    # a dimension beyond the coarse pass
    wide = rx.GpuBruteforceSearch(rx.L2, COARSE_MAX_DIM + 128, 1)
    with pytest.raises(rx.RxGpuError) as e:
        wide.ivf_train(2, np.zeros((4, COARSE_MAX_DIM + 128), np.float32))
    assert e.value.code == ERR_PARAMS
    wide.close()
    # errLogic: an index with rows, or one with lists already
    g.add_points(np.arange(3, dtype=np.uint64), x[:3])
    with pytest.raises(rx.RxGpuError) as e:
        g.ivf_train(10, x)
    assert e.value.code == ERR_LOGIC
    g.close()
    h = rx.GpuBruteforceSearch(rx.L2, dim, 1)
    c, _ = h.ivf_train(10, x, niter=2)
    with pytest.raises(rx.RxGpuError) as e:
        h.ivf_train(10, x)
    assert e.value.code == ERR_LOGIC
    assert h.ivf_size() == 0 and (h.ivf_assign(x)[0] < 10).all()
    h.close()


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_add_assign_and_search_against_faiss_over_the_same_lists(metric):
    dim, nlist, n = 32, 64, 6000
    x = O.synth_matrix(0xADD0 + metric, n, dim)
    labels = (np.arange(n, dtype=np.uint64) * np.uint64(7919)) | np.uint64(1 << 40)
    a, c, _ = train(metric, x, nlist, niter=4)
    b, c2, _ = train(metric, x, nlist, niter=4)
    assert (c.view(np.uint32) == c2.view(np.uint32)).all()
    lists = a.ivf_add_assign(labels, x)
    ln, _ = b.ivf_assign(x)
    b.ivf_add(ln, labels, x)
    assert (lists == ln).all() and a.ivf_size() == n
    # all or nothing: a duplicate id refuses the whole batch
    with pytest.raises(rx.RxGpuError) as e:
        a.ivf_add_assign(np.array([1, labels[0]], np.uint64), x[:2])
    assert e.value.code == ERR_LOGIC and a.ivf_size() == n
    q = O.synth_matrix(0xADD9, 50, dim)
    qs = normalized(metric, q)
    da, la, ca = a.ivf_search_knn(qs, 10, 8)
    db, lb, cb = b.ivf_search_knn(qs, 10, 8)
    assert (la == lb).all() and (da.view(np.uint32) == db.view(np.uint32)).all()
    ref = LO.ListsIvf(metric, c, lists, labels, x)
    assert (ref.list_of(labels) == lists).all()
    assert_matches_faiss(ref, metric, qs, 10, 8, da, la, ca, "add_assign")
    a.close()
    b.close()


def exact_top10(metric, x, q):
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    if metric == rx.L2:
        d = (x64 ** 2).sum(1)[None] - 2 * q64 @ x64.T
    else:
        d = -(q64 @ (x64 / np.linalg.norm(x64, axis=1, keepdims=True) if metric == rx.COS else x64).T)
    return np.argsort(d, 1, kind="stable")[:, :10]


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_quality_against_faiss_on_unseparated_data(metric):
    """the objective within 0.5 % of FAISS's, and recall@10 at nprobe 16 of an index trained and filled on the device within 0.02 of
    the index FAISS trains and fills (add_with_ids: its own quantizer picks the lists)"""
    dim, nlist = 32, 256
    x = O.synth_matrix(0x9A0 + metric, 39 * nlist, dim)
    labels = np.arange(len(x), dtype=np.uint64)
    want, obj, _ = TO.train(metric, x, nlist)
    g = rx.GpuBruteforceSearch(metric, dim, 1)
    got, st = g.ivf_train(nlist, x)
    assert abs(st[-1]["obj"] - obj[-1]) <= 0.005 * abs(obj[-1]), (st[-1]["obj"], obj[-1])
    g.ivf_add_assign(labels, x)
    ref = LO.ListsIvf(metric, want, np.zeros(0, np.int64), np.zeros(0, np.uint64), np.zeros((0, dim), np.float32))
    ref.add(labels, x)
    q = normalized(metric, O.synth_matrix(0x9AF, 300, dim))
    truth = exact_top10(metric, x, q)
    _, lg, _ = g.ivf_search_knn(q, 10, 16)
    _, lr = ref.search_batch(q, 10, 16)
    rec_dev = np.mean([len(set(truth[i]) & set(lg[i].tolist())) for i in range(len(q))]) / 10
    rec_ref = np.mean([len(set(truth[i]) & set(lr[i].tolist())) for i in range(len(q))]) / 10
    assert rec_dev >= rec_ref - 0.02, (rec_dev, rec_ref)
    g.close()
