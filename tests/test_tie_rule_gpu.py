"""GPU tests of the reference's KNN tie rule (bruteforce.cc:103-127) on every path that replays it, at every k and shard boundary.

When bit-equal distances straddle the k-th place, which rows survive depends on internal order and labels.  The library replays that
rule in four places: the exact tie-rows scan, the filter's bound lists (k <= 127, and k = 128 on the lists the staged scan wrote),
the staged lists through knn_select_topk (128 < k < 1024), and the host closed form fed shard by shard in rxgpu_sharded_search_knn.
Every answer here is compared with the heap applied literally (test_tie_rule_pin.literal_heap): labels, order, counts and distance
bits.  Integer-valued rows and queries make every fp32 sum exact, so the model's distances are the library's (tests/index_model.py);
float rows take their distance table from the exact scan, certified against the fp64 envelope of test_fp64_envelope_gpu.

Tie shapes are laid out on purpose (shaped_index): for each designed query, `m` strictly closer rows and a run of tied rows around
the k-th place -- (a) the run before the closer rows (evictions), (b) after them, (c) longer than k, (d) one row too long, and for
inner product (f) a tie at d* = 0 on zero rows.  Cosine rows of one level are copies under different labels (g); (e), every row at
one distance, has an index of its own.  Labels are always a permutation of internal order.  A zero dot product gives -(+0) = -0 on
every device path, as in the reference; zeros of both signs in one list are built directly as shard payloads."""
import numpy as np
import pytest
from test_fp64_envelope_gpu import Envelope, check_knn
from test_sharded_range_gpu import collective, make_shards
from test_tie_rule_pin import literal_heap

import reindexer_b200 as rx
from index_model import IndexModel
from oracle import oracle as O

pytestmark = pytest.mark.gpu

F = np.float32
KS = (1, 2, 127, 128, 129, 255, 256, 1022, 1023, 1024, 4095)
NQ = 160
DIM = 64
BLOCK = 8
METRICS = (rx.L2, rx.IP, rx.COS)


# ---------------------------------------------------------------------------------------------------------------- the model


def model_dists(metric, rows, queries):
    """fp32 distances [nq, n] in internal order, exact for integer-valued rows and queries (IndexModel.distances, batched)"""
    v64, q64 = rows.astype(np.float64), queries.astype(np.float64)
    if metric == rx.L2:
        return ((q64 ** 2).sum(1)[:, None] + (v64 ** 2).sum(1)[None, :] - 2.0 * (q64 @ v64.T)).astype(F)
    d = -(q64 @ v64.T).astype(F)
    if metric == rx.COS:
        s = (v64 * v64).sum(1).astype(F)
        long = (s > 0) & (np.abs(F(1) - s) > F(1e-5))
        coef = np.where(long, (1.0 / np.sqrt(np.where(long, s, F(1))).astype(np.float64)).astype(F), F(1))
        d = d * coef.astype(F)[None, :]
    return d.astype(F)


def heap_answers(d, labels, k):
    """the literal heap per query: (dist [nq, k], labels [nq, k], counts)"""
    nq = d.shape[0]
    kk = max(min(k, d.shape[1]), 1)
    od, ol, oc = np.zeros((nq, kk), F), np.zeros((nq, kk), np.uint64), np.zeros(nq, np.uint32)
    for q in range(nq):
        idx = literal_heap(d[q], labels, k)
        od[q, :len(idx)], ol[q, :len(idx)], oc[q] = d[q, idx], labels[idx], len(idx)
    return od, ol, oc


def assert_equal_answers(want, got, ctx=""):
    (d0, l0, c0), (d1, l1, c1) = want, got
    assert (c0 == c1).all(), (ctx, np.argwhere(c0 != c1)[:5])
    for q in range(len(c0)):
        m = int(c0[q])
        assert (l0[q, :m] == l1[q, :m]).all(), (ctx, q, l0[q, :m][l0[q, :m] != l1[q, :m]][:5])
        assert (d0[q, :m].view(np.uint32) == d1[q, :m].view(np.uint32)).all(), (ctx, q)


def straddles(d, k):
    """per query: bit-equal (float-equal) distances at the k-th and (k+1)-th place"""
    s = np.sort(d, axis=1)
    return (s[:, k - 1] == s[:, k]) if k < d.shape[1] else np.zeros(len(d), bool)


def evictions(dq, k):
    """tieReplay's E for one query: rows strictly below d* that are not among the first k rows with dist <= d*"""
    dstar = np.sort(dq)[k - 1]
    first = np.nonzero(dq <= dstar)[0][:k]
    return int((dq < dstar).sum() - (dq[first] < dstar).sum())


# ---------------------------------------------------------------------------------------------------------------- data


def level_row(metric, qblock, j):
    """a row at level j of a designed query: distance strictly increasing with j for all three metrics"""
    v = qblock.copy()
    v[0] -= np.sign(qblock[0]) * j
    return v


def shaped_index(metric, k, seed, nbg=3000):
    """integer rows and NQ queries; returns rows, labels, queries, {shape: (query, first internal row, end row of its rows)}.
    Coordinate 0 separates the designed rows (0) from the background (-2); shape s owns coordinates 1 + 8 s .. 8 + 8 s."""
    rng = np.random.default_rng(seed)
    m = k // 2
    plans = {  # (closer rows at level 0, tied rows at level 1, order)
        "a": (m, k - m + 3, "ties first"),
        "b": (m, k - m + 3, "closer first"),
        "c": (k // 3, 2 * k + 5, "mixed"),
        "d": (m, k + 1 - m, "mixed"),
    }
    if metric == rx.IP:
        plans["f"] = (m, k - m + 4, "zero ties")
    parts, spans, qs = [], {}, []
    pos = 0
    for s, (shape, (nlow, ntie, order)) in enumerate(plans.items()):
        q = np.zeros(DIM, F)
        q[0] = 1
        sl = slice(1 + BLOCK * s, 1 + BLOCK * (s + 1))
        q[sl] = -3 if shape == "f" else 3
        def rows_at(j, cnt):
            r = np.zeros((cnt, DIM), F)
            r[:, sl] = level_row(metric, q[sl], j)
            return r
        low = rows_at(0, nlow)
        tie = np.zeros((ntie, DIM), F) if shape == "f" else rows_at(1, ntie)
        far = -rows_at(0, 4) if shape == "f" else rows_at(2, 4)  # above d* = 0 for (f)
        if order == "ties first":
            blk = np.concatenate([tie, low, far])
        elif order == "closer first":
            blk = np.concatenate([low, tie, far])
        else:
            blk = np.concatenate([low, tie, far])[rng.permutation(nlow + ntie + 4)]
        parts.append(blk)
        spans[shape] = (len(qs), pos, pos + len(blk))
        qs.append(q)
        pos += len(blk)
    bg = np.zeros((nbg, DIM), F)
    bg[:, 0] = -2
    bg[:, 1 + BLOCK * 5:] = rng.integers(-2, 3, size=(nbg, DIM - 1 - BLOCK * 5))
    rows = np.concatenate(parts + [bg])
    n = len(rows)
    more = np.zeros((NQ - len(qs), DIM), F)
    more[:, 1 + BLOCK * 5:] = rng.integers(-2, 3, size=(NQ - len(qs), DIM - 1 - BLOCK * 5))
    queries = np.concatenate([np.stack(qs), more]).astype(F)
    labels = O.row_labels(n)[rng.permutation(n)]
    return rows, labels, queries, spans


def index_of(metric, rows, labels, mode=2):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], max(len(rows), 1))
    if len(rows):
        gpu.add_points(labels, rows)
    gpu.set_tensor_core_filter(mode)
    return gpu


def check_designed(metric, k, d, spans):
    """the designed queries straddle the k-th place as laid out"""
    for shape, (q, _, _) in spans.items():
        assert straddles(d[q:q + 1], k)[0], (shape, k)
        e = evictions(d[q], k)
        if shape == "b":
            assert e == 0, (shape, k, e)
        if shape == "a" and k >= 8:
            assert e > 0, (shape, k, e)
        if shape == "f":
            assert np.sort(d[q])[k - 1] == 0, k


def sample_vs_model_and_reference(metric, rows, labels, queries, got, qsel):
    """IndexModel.knn (the heap restated over the model's rows) and the reference's own bruteforce on a few queries"""
    model = IndexModel(metric, rows.shape[1], len(rows))
    model.upsert(labels, rows)
    ref = O.best_bf(metric, rows.shape[1], len(rows))
    ref.add_batch(labels, rows)
    d, l, c = got
    k = d.shape[1]
    for q in qsel:
        md, ml = model.knn(queries[q], k)
        assert c[q] == len(ml) and (l[q, :c[q]] == ml).all() and (d[q, :c[q]].view(np.uint32) == md.view(np.uint32)).all(), q
        rd, rl = ref.search_knn(queries[q], k)
        assert (l[q, :c[q]] == rl).all() and (d[q, :c[q]].view(np.uint32) == np.asarray(rd, F).view(np.uint32)).all(), q


# ---------------------------------------------------------------------------------------------------------------- single index


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("metric", METRICS)
def test_single_index_every_list_form(metric, k):
    rows, labels, queries, spans = shaped_index(metric, k, 100 * k + metric)
    d = model_dists(metric, rows, queries)
    check_designed(metric, k, d, spans)
    want = heap_answers(d, labels, k)
    gpu = index_of(metric, rows, labels)
    ntie = int(straddles(d, k).sum())
    for mode in (2, 1, 3, 4):
        gpu.set_tensor_core_filter(mode)
        got = gpu.search_knn(queries, k)
        st = rx.last_search_stats()
        assert_equal_answers(want, got, (mode, k))
        filt = mode != 2 and k + 1 <= 1024
        assert st["tc_used"] == int(filt), (mode, k, st)
        assert st["tie_replays"] == ntie and ntie >= len(spans), (mode, k, st, ntie)
        if filt:
            # k = 127: bound lists; k = 128: the staged scan (k + 1 > 128) and the bound-list tie pass over its lists; larger: staged
            assert st["tc_fallbacks"] == 0 and st["tc_cluster"] == (2 if mode == 4 else 1), (mode, k, st)
            assert st["tie_from_lists"] == st["tie_replays"], (mode, k, st)
        else:
            assert st["tie_from_lists"] == 0, (mode, k, st)
        if mode == 2:
            sample_vs_model_and_reference(metric, rows, labels, queries, got, [q for q, _, _ in spans.values()][:3])
    if metric == rx.IP:
        q = spans["f"][0]
        zeros = got[0][q][got[0][q] == 0]
        assert len(zeros) and np.signbit(zeros).all()  # -(+0), as the reference computes it
    gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_every_row_at_one_distance(metric):
    """(e): all rows are copies of one vector under shuffled labels, so every k below n is a straddling tie"""
    n, dim = 4000, 16  # at most 4096 candidates: no list overflows
    rng = np.random.default_rng(metric)
    rows = np.repeat(rng.integers(-2, 3, size=(1, dim)).astype(F), n, axis=0)
    labels = O.row_labels(n)[rng.permutation(n)]
    queries = rng.integers(-2, 3, size=(NQ, dim)).astype(F)
    d = model_dists(metric, rows, queries)
    gpu = index_of(metric, rows, labels)
    for k in KS[:-1]:
        want = heap_answers(d, labels, k)
        for mode in (2, 1, 4):
            gpu.set_tensor_core_filter(mode)
            got = gpu.search_knn(queries, k)
            st = rx.last_search_stats()
            assert_equal_answers(want, got, (mode, k))
            assert st["tie_replays"] == NQ, (mode, k, st)
            assert st["tie_from_lists"] == (NQ if mode != 2 and k + 1 <= 1024 else 0), (mode, k, st)
    gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_k_clamped_to_the_size(metric):
    """k in {n - 1, n, n + 5}: kEff = min(k, n); the two farthest rows are copies, so k = n - 1 straddles them"""
    n, dim = 600, 16
    rng = np.random.default_rng(7 + metric)
    rows = rng.integers(-2, 3, size=(n, dim)).astype(F)
    rows[-2:] = -9 if metric == rx.L2 else 0
    rows[-2:, 0] = 9  # far from every query under L2; a distinct direction under IP / cosine
    labels = O.row_labels(n)[rng.permutation(n)]
    queries = rng.integers(-2, 3, size=(NQ, dim)).astype(F)
    d = model_dists(metric, rows, queries)
    gpu = index_of(metric, rows, labels)
    for k in (n - 1, n, n + 5):
        want = heap_answers(d, labels, k)
        for mode in (2, 1, 3):
            gpu.set_tensor_core_filter(mode)
            got = gpu.search_knn(queries, k)
            st = rx.last_search_stats()
            assert_equal_answers(want, got, (mode, k))
            assert (got[2] == min(k, n)).all()
            assert st["tc_used"] == int(mode != 2), st
            assert st["tie_replays"] == int(straddles(d, min(k, n)).sum()), (k, st)
            if k == n - 1 and metric == rx.L2:
                assert st["tie_replays"] == NQ, st
            if mode != 2:
                assert st["tie_from_lists"] == st["tie_replays"], st
    gpu.close()


# ---------------------------------------------------------------------------------------------------------------- list overflow


def overflow_data(dim, seed):
    """integer rows in {-2..2}; base b is 6 along coordinate b.  Base 0 has 34000 exact copies on every other row of the first 68000
    (more candidates than a list of 256 k1 = 32768 at k = 127 holds), bases 2..11 have 150 copies each further on.  Query 0 sits on
    base 0, the others on bases 2..11: every query ties at k = 127, and query 0's list overflows."""
    rng = np.random.default_rng(seed)
    n = 80000
    rows = rng.integers(-2, 3, size=(n, dim)).astype(F)
    bases = np.zeros((12, dim), F)
    bases[np.arange(12), np.arange(12)] = 6
    rows[0:68000:2] = bases[0]
    for b in range(2, 12):
        rows[rng.choice(np.arange(68000, n), 150, replace=False)] = bases[b]
    queries = np.concatenate([bases[:1], bases[2 + np.arange(63) % 10]]).astype(F)
    labels = O.row_labels(n)[rng.permutation(n)]
    return rows, labels, queries


def float_table(metric, rows, labels, queries):
    """every row's fp32 distance in internal order, from the exact scan (range batch, radius +inf), certified by the fp64 envelope"""
    n = len(rows)
    gpu = index_of(metric, rows, labels, mode=2)
    dd, ll, cc = gpu.search_range_batch(queries, np.inf, n)
    assert (cc == n).all() and rx.last_search_stats()["tc_used"] == 0
    pos = {int(x): i for i, x in enumerate(labels)}
    row_of = lambda lab: np.array([pos.get(int(x), -1) for x in np.ravel(lab)], np.int64)  # noqa: E731
    check_knn(Envelope(metric, rows, queries), dd, ll, cc.astype(np.int64), n, ctx="table", row_of=row_of)
    d = np.zeros((len(queries), n), F)
    for q in range(len(queries)):
        d[q, row_of(ll[q])] = dd[q]
    gpu.close()
    return d


@pytest.mark.parametrize("dim", [64, 768])
def test_overflowed_lists_take_the_exact_tie_scan(dim):
    k, metric = 127, rx.L2
    rows, labels, queries = overflow_data(dim, 0x7100 + dim)
    d = float_table(metric, rows, labels, queries)
    assert straddles(d, k).all()
    want = heap_answers(d, labels, k)
    gpu = index_of(metric, rows, labels, mode=1)
    got = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert_equal_answers(want, got, dim)
    # every query ties; one whose list overflowed takes the exact tie scan, every other one replays from its list
    assert st["tc_used"] == 1 and st["tc_fallbacks"] >= 1, st
    assert st["tie_replays"] == len(queries) and st["tie_from_lists"] == len(queries) - st["tc_fallbacks"], st
    gpu.close()


# ---------------------------------------------------------------------------------------------------------------- tie rows


def test_search_tie_rows_device():
    import torch

    n, dim = 6000, 16
    rng = np.random.default_rng(3)
    rows = rng.integers(-2, 3, size=(n, dim)).astype(F)
    rows[::7] = 0  # zero rows: a zero distance for inner product
    labels = O.row_labels(n)[rng.permutation(n)]
    query = rng.integers(-2, 3, size=(1, dim)).astype(F)
    query[0, :4] = -2
    gpu = index_of(rx.IP, rows, labels)
    d = model_dists(rx.IP, rows, query)[0]
    vals = np.unique(d)
    mid = vals[np.searchsorted(vals, 0) - 3]
    dstars = [mid, F((mid + vals[np.searchsorted(vals, mid) + 1]) / 2), F(0.0), F(-0.0), F(-np.inf), F(np.inf)]
    dq = torch.from_numpy(query).cuda()
    for k in (1, 128, 1023, 5000):
        od = torch.zeros(k, dtype=torch.float32, device="cuda")
        oi = torch.zeros(k, dtype=torch.int32, device="cuda")
        ol = torch.zeros(k, dtype=torch.int64, device="cuda")
        oc = torch.zeros(1, dtype=torch.int32, device="cuda")
        for ds in dstars:
            torch.cuda.synchronize()
            gpu.search_tie_rows_device(dq.data_ptr(), float(ds), k, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr())
            want = np.nonzero(d <= ds)[0][:k]
            c = int(oc.cpu().item())
            assert c == len(want), (k, ds, c, len(want))
            assert (oi.cpu().numpy()[:c] == want).all(), (k, ds)
            assert (ol.cpu().numpy().view(np.uint64)[:c] == labels[want]).all(), (k, ds)
            assert (od.cpu().numpy()[:c].view(np.uint32) == d[want].view(np.uint32)).all(), (k, ds)
    assert (d == 0).sum() > 800 and np.signbit(d[d == 0]).all()
    gpu.close()


# ---------------------------------------------------------------------------------------------------------------- sharded


def shard_cuts(n, R, k, spans, seed):
    """R shards: one cut inside the tie run of shape (c); then a shard of exactly k + 1 rows, one of fewer, an empty one; the
    remaining cuts mostly inside the designed tie runs, so runs cross one and several cuts"""
    if R == 1:
        return [0, n]
    rng = np.random.default_rng(seed)
    _, c0, c1 = spans["c"]
    x = c0 + (c1 - c0) // 3
    cuts = [0, x]
    if R >= 5:
        cuts += [x + k + 1, x + k + 1 + max(k // 2, 1), x + k + 1 + max(k // 2, 1)]
    lo = cuts[-1] + 1
    hi = max(s[2] for s in spans.values())
    extra = R - len(cuts)
    cuts += sorted(int(v) for v in rng.choice(np.arange(lo, hi if hi - lo > extra else n), extra, replace=False))
    cuts.append(n)
    assert len(cuts) == R + 1 and all(a <= b for a, b in zip(cuts, cuts[1:]))
    return cuts


def sharded_knn(shards, queries, k, dq=None):
    if dq is None:
        return collective(shards, lambda comm, shard: comm.search_knn(shard, queries, k))
    return collective(shards, lambda comm, shard: comm.search_knn(shard, dq.data_ptr(), k, nq=len(queries)))


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("metric", METRICS)
def test_sharded_every_rank_equals_the_heap(metric, k):
    import torch

    rows, labels, queries, spans = shaped_index(metric, k, 200 * k + metric)
    d = model_dists(metric, rows, queries)
    want = heap_answers(d, labels, k)
    whole = index_of(metric, rows, labels)
    assert_equal_answers(want, whole.search_knn(queries, k), "whole")
    ntie = int(straddles(d, k).sum())
    dq = torch.from_numpy(queries).cuda()
    torch.cuda.synchronize()
    for R in (1, 2, 5, 32):
        cuts = shard_cuts(len(rows), R, k, spans, R + k)
        tc = [(1, 2, 3, 4)[r % 4] for r in range(R)]
        shards = make_shards(metric, rows, labels, cuts, tc)
        for dev in ((False, True) if R in (2, 5) else (False,)):  # device-resident queries on two group sizes
            res = sharded_knn(shards, queries, k, dq if dev else None)
            for r, (got, st) in enumerate(res):
                assert_equal_answers(want, got, (R, r, dev, cuts[r:r + 2]))
                assert st["tie_replays"] == ntie, (R, r, st)
                size = cuts[r + 1] - cuts[r]
                filt = tc[r] != 2 and k + 1 <= 1024 and size > 0
                assert st["tc_used"] == int(filt), (R, r, st)
                if filt and size >= k + 1:
                    assert st["tc_fallbacks"] == 0 and st["tie_from_lists"] == ntie, (R, r, size, st)
                else:  # a shard shorter than k + 1 may leave the staged lists for the exact scan: then all its tie rows come from there
                    assert st["tie_from_lists"] == (ntie if filt and st["tc_fallbacks"] == 0 else 0), (R, r, size, st)
        for s in shards:
            s.close()
    whole.close()


def test_sharded_overflow_on_one_shard():
    """shard 0 holds more copies of base 0 than a list holds: its list overflows for query 0, so it answers every tied query with
    the exact tie scan; a shard without an overflowed list answers them all from its lists"""
    k, metric = 127, rx.L2
    rows, labels, queries = overflow_data(64, 0x7200)
    n = len(rows)
    d = float_table(metric, rows, labels, queries)
    want = heap_answers(d, labels, k)
    ntie = int(straddles(d, k).sum())
    for cuts in ([0, 70000, 75000, n], [0, 68000, n - 300, n]):
        shards = make_shards(metric, rows, labels, cuts, [1, 1, 3])
        res = sharded_knn(shards, queries, k)
        for r, (got, st) in enumerate(res):
            assert_equal_answers(want, got, (cuts, r))
            assert st["tie_replays"] == ntie == len(queries), st
        assert res[0][1]["tc_fallbacks"] >= 1 and res[0][1]["tie_from_lists"] == 0, res[0][1]
        for r, (_, st) in enumerate(res):  # the list source is decided per shard for all tied queries at once
            assert st["tc_used"] == 1 and st["tie_from_lists"] == (ntie if st["tc_fallbacks"] == 0 else 0), (r, st)
        for s in shards:
            s.close()


def test_sharded_refuses_33_ranks_and_k_65536():
    from reindexer_b200 import binding as B

    with pytest.raises(rx.RxGpuError) as e:
        B.ShardComm.local_group(33)
    assert e.value.code == 3
    rows = np.random.default_rng(1).integers(-2, 3, size=(300, 16)).astype(F)
    labels = O.row_labels(300)
    shards = make_shards(rx.L2, rows, labels, [0, 100, 300], 2)
    queries = rows[:3].copy()
    # k >= 65536 is refused even though the shards hold 300 rows (documented in rxgpu.h); 5000 > 300 is served and clamped
    res = collective(shards, lambda comm, shard: _expect_refusal(comm, shard, queries))
    d = model_dists(rx.L2, rows, queries)
    want = heap_answers(d, labels, 5000)
    for (got, _) in res:
        assert_equal_answers(want, tuple(x[:, :300] if x.ndim == 2 else x for x in got))
        assert (got[2] == 300).all()
    for s in shards:
        s.close()


def _expect_refusal(comm, shard, queries):
    with pytest.raises(rx.RxGpuError) as e:
        comm.search_knn(shard, queries, 65536)
    assert e.value.code == 3
    return comm.search_knn(shard, queries, 5000)


@pytest.mark.parametrize("k", [10, 128, 1023])
def test_public_two_step_path(k):
    """search_knn_device per shard, merge_shards, search_tie_rows_device per shard and tie_replay, assembled as rxgpu.h documents,
    equal the sharded call"""
    import torch

    metric = rx.IP
    rows, labels, queries, spans = shaped_index(metric, k, 300 + k)
    n = len(rows)
    cuts = shard_cuts(n, 5, k, spans, 9)
    shards = make_shards(metric, rows, labels, cuts, [1, 2, 3, 4, 1])
    want = sharded_knn(shards, queries, k)[0][0]
    k1, nq, R = k + 1, len(queries), len(shards)
    dq = torch.from_numpy(queries).cuda()
    dist, idx, lab = np.zeros((R, nq, k1), F), np.zeros((R, nq, k1), np.uint32), np.zeros((R, nq, k1), np.uint64)
    cnt = np.zeros((R, nq), np.uint32)
    for s, sh in enumerate(shards):
        od = torch.zeros((nq, k1), dtype=torch.float32, device="cuda")
        oi = torch.zeros((nq, k1), dtype=torch.int32, device="cuda")
        ol = torch.zeros((nq, k1), dtype=torch.int64, device="cuda")
        oc = torch.zeros(nq, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        sh.search_knn_device(nq, dq.data_ptr(), k1, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr())
        dist[s], idx[s], lab[s], cnt[s] = od.cpu().numpy(), oi.cpu().numpy(), ol.cpu().numpy().view(np.uint64), oc.cpu().numpy()
    md, mg, ml, mc, tie = rx.merge_shards(k, dist, idx, lab, cnt, np.array(cuts[:-1], np.uint64))
    assert tie.sum() >= len(spans)
    od_t = torch.zeros(k, dtype=torch.float32, device="cuda")
    oi_t = torch.zeros(k, dtype=torch.int32, device="cuda")
    ol_t = torch.zeros(k, dtype=torch.int64, device="cuda")
    oc_t = torch.zeros(1, dtype=torch.int32, device="cuda")
    for q in np.nonzero(tie)[0]:
        dstar = md[q, k - 1]
        low = md[q, :k] < dstar
        fd, fg, fl = [], [], []
        for s, sh in enumerate(shards):
            if cuts[s + 1] == cuts[s]:
                continue
            torch.cuda.synchronize()
            sh.search_tie_rows_device(dq[q].data_ptr(), float(dstar), k, od_t.data_ptr(), oi_t.data_ptr(), ol_t.data_ptr(), oc_t.data_ptr())
            c = int(oc_t.cpu().item())
            fd += list(od_t.cpu().numpy()[:c])
            fg += list(oi_t.cpu().numpy()[:c].astype(np.uint64) + np.uint64(cuts[s]))
            fl += list(ol_t.cpu().numpy().view(np.uint64)[:c])
        rd, rl = rx.tie_replay(k, dstar, (md[q, :k][low], mg[q, :k][low], ml[q, :k][low]), (fd[:k], fg[:k], fl[:k]))
        md[q, :len(rd)], ml[q, :len(rl)], mc[q] = rd, rl, len(rl)
    assert_equal_answers(want, (md, ml, mc), k)
    for s in shards:
        s.close()


# ---------------------------------------------------------------------------------------------------------------- device merge


def payload(lists, sizes, nq, k1):
    """rxgpu_shard_payload_bytes layout: [dist nq*k1][idx nq*k1][label nq*k1][count nq][size], 16-byte aligned sections"""
    up = lambda x: (x + 15) & ~15  # noqa: E731
    n = nq * k1
    off_idx = up(n * 4)
    off_label = up(off_idx + n * 4)
    off_count = up(off_label + n * 8)
    off_size = up(off_count + nq * 4)
    nbytes = up(off_size + 16)
    assert nbytes == rx.binding.lib().rxgpu_shard_payload_bytes(nq, k1)
    out = np.zeros((len(lists), nbytes), np.uint8)
    for s, (dist, idx, lab, cnt) in enumerate(lists):
        out[s, :n * 4] = dist.reshape(-1).view(np.uint8)
        out[s, off_idx:off_idx + n * 4] = idx.reshape(-1).view(np.uint8)
        out[s, off_label:off_label + n * 8] = lab.reshape(-1).view(np.uint8)
        out[s, off_count:off_count + nq * 4] = cnt.view(np.uint8)
        out[s, off_size:off_size + 8] = np.array([sizes[s]], np.uint64).view(np.uint8)
    return out


def random_shard_lists(rng, R, nq, k1, counts):
    """per shard and query: counts[s][q] entries ascending under (dist, local row) from a few values with zeros of both signs"""
    vals = F([-1.0, -0.0, 0.0, 2.0])
    lists, sizes = [], []
    for s in range(R):
        dist, idx = np.zeros((nq, k1), F), np.zeros((nq, k1), np.uint32)
        lab = np.zeros((nq, k1), np.uint64)
        cnt = np.array([counts[s][q] for q in range(nq)], np.uint32)
        size = int(cnt.max(initial=0)) + int(rng.integers(0, 3))
        for q in range(nq):
            c = int(cnt[q])
            loc = np.sort(rng.choice(size, c, replace=False)) if c else np.zeros(0, np.int64)
            dd = rng.choice(vals, c).astype(F)
            o = sorted(range(c), key=lambda i: (float(dd[i]), int(loc[i])))
            dist[q, :c], idx[q, :c] = dd[o], loc[o]
            lab[q, :c] = (np.uint64(s) << np.uint64(40)) | (loc[o].astype(np.uint64) * np.uint64(7919) % np.uint64(1 << 30))
        lists.append((dist, idx, lab, cnt))
        sizes.append(size)
    return lists, sizes


@pytest.mark.parametrize("k", [1, 1023, 5000])
def test_merge_shards_device_at_its_limits(k):
    import torch

    rng = np.random.default_rng(k)
    R, nq, k1 = 32, 9, k + 1
    counts = [[0] * nq for _ in range(R)]
    for s in range(R):
        for q in range(nq):
            counts[s][q] = [0, int(rng.integers(0, max(k // 8, 2))), min(k1, int(rng.integers(0, k1 + 1))), k1][q % 4]
            if q == nq - 1:
                counts[s][q] = 0  # every count 0
    lists, sizes = random_shard_lists(rng, R, nq, k1, counts)
    # query 1: the k-th and (k+1)-th are -0 and +0 from two shards (a float tie with different bits)
    for s in range(R):
        lists[s][3][1] = 0
    d0, i0, l0, c0 = lists[0]
    d1, i1, l1, c1 = lists[1]
    c0[1], c1[1] = k, 1
    d0[1, :k], i0[1, :k] = np.concatenate([np.full(k - 1, -1.0, F), F([-0.0])]), np.arange(k)
    d1[1, 0], i1[1, 0] = F(0.0), 0
    sizes[0] = max(sizes[0], k)
    l0[1, :k] = np.arange(k, dtype=np.uint64) + np.uint64(1 << 50)
    l1[1, 0] = 3
    pay = payload(lists, sizes, nq, k1)
    dpay = torch.from_numpy(pay).cuda()
    od = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    og = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    ol = torch.zeros((nq, k), dtype=torch.int64, device="cuda")
    oc = torch.zeros(nq, dtype=torch.int32, device="cuda")
    ot = torch.zeros(nq, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rx.binding._check(rx.binding.lib().rxgpu_merge_shards_device(R, nq, k, k1, dpay.data_ptr(), od.data_ptr(), og.data_ptr(), ol.data_ptr(),
                                                                  oc.data_ptr(), ot.data_ptr(), None))
    torch.cuda.synchronize()
    gd, gg, gl = od.cpu().numpy(), og.cpu().numpy().view(np.uint64), ol.cpu().numpy().view(np.uint64)
    gc, gt = oc.cpu().numpy(), ot.cpu().numpy()
    base = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.uint64)
    hd, hg, hl, hc, ht = rx.merge_shards(k, np.stack([x[0] for x in lists]), np.stack([x[1] for x in lists]),
                                         np.stack([x[2] for x in lists]), np.stack([x[3] for x in lists]), base)
    assert (gc == hc).all() and (gt == ht).all(), (gc, hc, gt, ht)
    assert ht[1] == 1 and gc[nq - 1] == 0
    for q in range(nq):
        c = int(hc[q])
        o = sorted(range(c), key=lambda j: (float(gd[q, j]), int(gl[q, j])))  # the device leaves runs of equal distances by row
        assert (gg[q, o] == hg[q, :c]).all() and (gl[q, o] == hl[q, :c]).all(), q
        assert (gd[q, o].view(np.uint32) == hd[q, :c].view(np.uint32)).all(), q
