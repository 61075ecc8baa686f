"""GPU tests of the IVF range batch (rxgpu_ivf_search_range_batch): one coarse pass and one key pass over the probed lists serve the
whole batch, then each query's matches are counted, kept, sorted by (distance, label) and cut at max_out on the device.  Every query
must be bit-identical to its own rxgpu_ivf_search_range call; the match sets are also held against the reference's FAISS, the fp64
envelope and, at full probe, the exact brute-force scan."""
import numpy as np
import pytest
from helpers import prep_query
from test_fp64_envelope_gpu import Envelope, assert_identical, check_range, ivf_index, probed_rows, queries_for
from test_ivf_gpu import build
from test_ivf_large_k_gpu import int_index, int_rows, model

import reindexer_b200 as rx
from oracle import oracle as O
from reindexer_b200 import binding as B

pytestmark = pytest.mark.gpu
needs_faiss = pytest.mark.skipif(not O.ref_ivf_available(), reason="needs oracle/_ref (reference FAISS build)")

KEY_CAP = 1 << 26   # keys per query chunk (kIvfKeyCap, DESIGN.md §8.1)
SLOT_CAP = 1 << 24  # survivors per sort sub-chunk (kIvfSlotCap)


def singles(gpu, queries, radii, nprobe, max_out):
    """one rxgpu_ivf_search_range call per query, shaped like the batch"""
    nq = len(queries)
    d = np.zeros((nq, max_out), np.float32)
    l = np.zeros((nq, max_out), np.uint64)
    n = np.zeros(nq, np.uint64)
    for q in range(nq):
        dq, lq, n[q] = gpu.ivf_search_range(queries[q], float(radii[q]), nprobe, max_out=max_out)
        d[q, :len(dq)], l[q, :len(lq)] = dq, lq
    return d, l, n


def assert_batch_is_singles(gpu, queries, radii, nprobe, max_out, ctx=""):
    batch = gpu.ivf_search_range_batch(queries, radii, nprobe, max_out)
    st = rx.last_search_stats()
    assert st["passes"] == (1 if len(queries) else 0) and st["tc_fallbacks"] == 0, (ctx, st)
    assert_identical(batch, singles(gpu, queries, radii, nprobe, max_out), ctx)
    return batch


def mixed_radii(gpu, queries, nprobe):
    """per query, cycling: -inf, NaN, 0, -0, +inf and the j-th best probed distance (j = 1, 10, 100, 1000) and one ulp above it"""
    d, _, c = gpu.ivf_search_knn_large_k(queries, 1000, nprobe)
    out = []
    for q in range(len(queries)):
        kind = q % 13
        if kind < 5:
            out.append([-np.inf, np.nan, 0.0, -0.0, np.inf][kind])
            continue
        j = [1, 10, 100, 1000][(kind - 5) // 2]
        r = np.float32(d[q, min(j, int(c[q])) - 1]) if c[q] else np.float32(1.0)
        out.append(np.nextafter(r, np.float32(np.inf)) if kind % 2 == 0 else r)
    return np.array(out, np.float32)


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("dim", [16, 128, 129])
def test_batch_is_the_single_call(metric, dim):
    nlist = 24
    ref, gpu, st = build(metric, 6000, dim, nlist, 7100 + dim + metric)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(7200 + dim, 26, dim)])
    for nprobe in (1, 3, nlist, nlist + 5):
        radii = mixed_radii(gpu, queries, nprobe)
        for max_out in (0, 1, 40, 6000):
            d, l, n = assert_batch_is_singles(gpu, queries, radii, nprobe, max_out, (metric, dim, nprobe, max_out))
        _, _, probed = gpu.ivf_search_knn_large_k(queries, 65535, nprobe)  # 6000 rows: k above them returns every probed row
        assert (n[np.isnan(radii) | (radii == -np.inf)] == 0).all()
        assert (n[radii == np.inf] == probed[radii == np.inf]).all() and n.max() > 0


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_match_sets_are_the_reference_faiss(metric):
    n, dim, nlist, nprobe = 8000, 40, 16, 5
    ref, gpu, st = build(metric, n, dim, nlist, 7300 + metric)
    at = (st["labels"] >> np.uint64(32)).astype(np.int64)  # the rows back in insertion order: label >> 32 is the row
    vecs = np.zeros((n, dim), np.float32)
    vecs[at] = st["vecs"]
    lists = np.zeros(n, np.int64)
    lists[at] = np.repeat(np.arange(nlist), st["list_sizes"].astype(np.int64))
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(7400 + metric, 30, dim)])
    allowed, clear = probed_rows(metric, st["centroids"], queries, lists, nprobe)
    assert clear.sum() >= 10
    kd, _, _ = gpu.ivf_search_knn(queries, 60, nprobe)
    j = np.array([5, 20, 59])[np.arange(len(queries)) % 3]
    radii = ((kd[np.arange(len(queries)), j - 1].astype(np.float64) + kd[np.arange(len(queries)), j]) / 2).astype(np.float32)
    d, l, c = gpu.ivf_search_range_batch(queries, radii, nprobe, 100)
    for q in np.nonzero(clear)[0]:
        fd, fl = ref.range_search(queries[q], float(radii[q]) if metric == rx.L2 else -float(radii[q]), nprobe)
        assert c[q] == len(fl) == j[q] and sorted(l[q, :c[q]].tolist()) == sorted(fl.tolist()), q
    env = Envelope(metric, vecs, queries[clear]).restrict(allowed[clear])
    check_range(env, radii[clear], d[clear], l[clear], c[clear])


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_own_lists_inside_the_fp64_envelope(metric):
    """mutable lists with empty lists among them, radii at the j-th best fp64 distance: every certain match returned, every returned
    row possible, distances inside the envelope"""
    dim, nlist, n, nprobe = 48, 40, 12000, 6
    gpu, cents, rows, lists = ivf_index(metric, dim, nlist, n, 0x7500 + metric)
    queries = queries_for(metric, 0x7501 + metric, 24, dim)
    allowed, clear = probed_rows(metric, cents, queries, lists, nprobe)
    env = Envelope(metric, rows, queries[clear]).restrict(allowed[clear])
    srt = np.sort(env.mid, axis=1)
    radii = np.full(len(queries), np.float32(1.0))
    radii[clear] = [np.float32(srt[i, [1, 10, 100][i % 3] - 1]) for i in range(int(clear.sum()))]
    d, l, c = assert_batch_is_singles(gpu, queries, radii, nprobe, 500)
    check_range(env, radii[clear], d[clear], l[clear], c[clear])
    gpu.close()


@needs_faiss
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_full_probe_is_the_exact_scan(metric):
    nlist = 20
    ref, gpu, _ = build(metric, 16000, 64, nlist, 7600 + metric)
    queries = np.stack([prep_query(metric, q) for q in O.synth_matrix(7601 + metric, 10, 64)])
    radii = mixed_radii(gpu, queries, nlist)
    d, l, c = gpu.ivf_search_range_batch(queries, radii, nlist, 1200)
    for q in range(len(queries)):
        dq, lq, nq_ = gpu.search_range(queries[q], float(radii[q]), max_out=1200)
        assert c[q] == nq_ and (l[q, :len(lq)] == lq).all() and (d[q, :len(dq)].view(np.uint32) == dq.view(np.uint32)).all(), q


def tie_radii(vecs, queries, metric, rng):
    """radii among the integer distances, so that many equal distances lie below each radius"""
    q64 = queries.astype(np.float64)
    v = vecs[rng.choice(len(vecs), 200, replace=False)].astype(np.float64)
    dist = ((q64[:, None, :] - v[None]) ** 2).sum(2) if metric == rx.L2 else -(q64 @ v.T)
    return np.array([np.float32(np.median(dist[i]) + 0.5) for i in range(len(queries))], np.float32)


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_cut_follows_distance_then_label_on_imported_lists(metric):
    """integer rows: groups of bit-equal distances straddle the max_out cut; labels are a permutation, so label order differs from
    row order, and the cut must follow (distance, label) as the single call does"""
    n, dim, nlist, nprobe = 30000, 6, 12, 5
    gpu, vecs, cents, labels, sizes = int_index(metric, n, dim, nlist, 7700 + metric)
    queries = int_rows(7701 + metric, 12, dim)
    radii = tie_radii(vecs, queries, metric, np.random.default_rng(7702))
    straddles = 0
    for max_out in (1, 37, 500, 4000):
        d, l, c = assert_batch_is_singles(gpu, queries, radii, nprobe, max_out, max_out)
        for i, q in enumerate(queries):
            md, ml, probed, _ = model(metric, q, vecs, cents, labels, sizes, n, nprobe)
            hit = md < radii[i]
            assert c[i] == hit.sum(), (max_out, i)
            m = min(int(c[i]), max_out)
            assert (d[i, :m] == md[hit][:m]).all() and (l[i, :m] == ml[hit][:m]).all(), (max_out, i)
            straddles += m < c[i] and md[hit][m - 1] == md[hit][m]
    assert straddles >= 8


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_cut_follows_distance_then_label_on_mutable_lists(metric):
    """integer rows in mutable lists, after bursts of adds and removes that relocate lists in the slab: slab order differs from label
    order"""
    dim, nlist = 6, 10
    rng = np.random.default_rng(7800 + metric)
    cents = int_rows(7801, nlist, dim)
    n = 20000
    rows = int_rows(7802 + metric, n, dim)
    labels = (rng.permutation(n).astype(np.uint64) << np.uint64(32)) | np.uint64(3)
    lists = rng.integers(0, nlist, n).astype(np.uint32)
    gpu = rx.GpuBruteforceSearch(metric, dim, 16)
    gpu.ivf_create(cents)
    queries = int_rows(7803 + metric, 9, dim)
    alive = set()
    done = 0
    for burst in (3000, 1, 777, 6000, 10222):
        gpu.ivf_add(lists[done:done + burst], labels[done:done + burst], rows[done:done + burst])
        alive |= set(labels[done:done + burst].tolist())
        done += burst
        for v in rng.choice(sorted(alive), size=len(alive) // 8, replace=False):
            gpu.ivf_remove(int(v))
            alive.discard(int(v))
        radii = tie_radii(rows, queries, metric, rng)
        for max_out in (1, 100, 3000):
            assert_batch_is_singles(gpu, queries, radii, 4, max_out, (done, max_out))
    assert gpu.ivf_list_stats()["relocations"] > 0
    gpu.close()


@pytest.mark.parametrize("metric", [rx.L2, rx.COS])
def test_batch_sizes_and_independence(metric):
    dim, nlist = 24, 30
    gpu, cents, rows, lists = ivf_index(metric, dim, nlist, 9000, 0x7900 + metric, empty_every=4)
    queries = queries_for(metric, 0x7901 + metric, 33, dim)
    radii = mixed_radii(gpu, queries, 2)
    d, l, c = gpu.ivf_search_range_batch(queries[:0], radii[:0], 2, 10)  # nq = 0: nothing to do
    assert d.shape == (0, 10) and len(c) == 0
    for nq in range(1, 34):
        assert_batch_is_singles(gpu, queries[:nq], radii[:nq], 2 if nq % 2 else 1, 25, nq)
    full = gpu.ivf_search_range_batch(queries, radii, 3, 300)
    perm = np.random.default_rng(0x7902).permutation(len(queries))
    shuffled = gpu.ivf_search_range_batch(queries[perm], radii[perm], 3, 300)
    assert_identical(shuffled, tuple(x[perm] for x in full))
    gpu.close()


def test_chunks_with_a_query_above_the_key_cap_and_the_survivor_cap():
    """one list of more than 2^26 rows: a query probing it is a key chunk of its own, and its 2^24+ matches a sort of its own; the
    queries around it probe a small list and share chunks"""
    dim, big, small = 4, KEY_CAP + (1 << 20), 3000
    rng = np.random.default_rng(0x7A00)
    iv = rng.integers(-2, 3, size=(big + small, dim), dtype=np.int8)
    iv[big:] += 40
    vecs = iv.astype(np.float32)
    labels = (np.arange(big + small, dtype=np.uint64)[::-1].copy() << np.uint64(32))
    gpu = rx.GpuBruteforceSearch(rx.L2, dim, big + small)
    gpu.add_points(labels, vecs)
    gpu.ivf_import(np.array([[0.0] * dim, [40.0] * dim], np.float32), np.array([big, small], np.uint64))
    near_big = rng.integers(-1, 2, size=(2, dim)).astype(np.float32)
    near_small = rng.integers(39, 42, size=(4, dim)).astype(np.float32)
    queries = np.concatenate([near_small[:2], near_big[:1], near_small[2:3], near_big[1:], near_small[3:]])
    radii = np.full(len(queries), np.float32(6.5))
    for i, qi in enumerate((2, 4)):  # integer distances: the radius just above the one where the matches pass 2^24
        d2 = ((iv[:big].astype(np.int16) - near_big[i].astype(np.int16)) ** 2).sum(1)
        cum = np.cumsum(np.bincount(d2))
        radii[qi] = np.float32(np.searchsorted(cum, SLOT_CAP, side="right") + 0.5)
        del d2
    d, l, c = gpu.ivf_search_range_batch(queries, radii, 1, 1000)
    st = rx.last_search_stats()
    assert st["passes"] == 1 and st["tc_fallbacks"] == 0
    assert c[2] > SLOT_CAP and c[4] > SLOT_CAP
    assert_identical((d, l, c), singles(gpu, queries, radii, 1, 1000))
    gpu.close()


def test_errors():
    gpu, vecs, cents, labels, sizes = int_index(rx.L2, 4000, 8, 6, 0x7B00)
    q = int_rows(0x7B01, 3, 8)
    r = np.full(3, np.float32(10.0))
    lib = B.lib()
    qp, rp = B._p(np.ascontiguousarray(q), B._f32p), B._p(r, B._f32p)
    d = np.zeros((3, 5), np.float32)
    l = np.zeros((3, 5), np.uint64)
    n = np.zeros(3, np.uint64)
    dp, lp, np_ = B._p(d, B._f32p), B._p(l, B._u64p), B._p(n, B._u64p)
    for args in ((qp, rp, 2, 5, dp, lp, None), (qp, rp, 2, 5, None, lp, np_), (qp, rp, 2, 5, dp, None, np_), (qp, None, 2, 5, dp, lp, np_),
                 (None, rp, 2, 5, dp, lp, np_)):
        assert lib.rxgpu_ivf_search_range_batch(gpu._h, 3, *args) == 3
        assert b"null argument" in lib.rxgpu_last_error()
    assert lib.rxgpu_ivf_search_range_batch(gpu._h, 3, qp, rp, 2, 0, None, None, np_) == 0  # max_out = 0: outputs not needed
    gpu.add_point(vecs[0], int(labels[5]))  # a row was overwritten: the imported lists are stale
    with pytest.raises(rx.RxGpuError) as e:
        gpu.ivf_search_range_batch(q, r, 2, 5)
    assert "changed after the IVF lists were imported" in e.value.what
    fresh = rx.GpuBruteforceSearch(rx.L2, 8, 10)
    fresh.add_point(vecs[0], 1)
    with pytest.raises(rx.RxGpuError) as e:
        fresh.ivf_search_range_batch(q, r, 2, 5)
    assert "no IVF lists imported" in e.value.what
