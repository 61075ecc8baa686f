"""GPU tests of the sharded range batch (rxgpu_sharded_search_range_batch) and of the sharded KNN on in-process rank groups.  The shards
are in-process ranks on cuda:0 (ShardComm.local_group, one thread per rank), so one GPU runs every cross-shard path: the local range
batch of each shard, the all-reduces of the totals and of the payload width, the all-gather and the device merge.  The reference answer
is rxgpu_search_range_batch (or rxgpu_search_knn) on one index holding all rows; equal means the same totals, the same labels in the
same order and the same distance bits, on every rank.  The NCCL run with one process per GPU is tests/mp_sharded_range_nccl.py,
launched by test_two_ranks_nccl when the box has two GPUs."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from reindexer_b200 import binding as B
from reindexer_b200.sharded import ShardedBruteforceSearch
from oracle import oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RANKS = (1, 10, 100)


def uneven_cuts(n, R, seed, empty=None):
    """row boundaries of R shards of uneven sizes; shard `empty` gets no rows"""
    w = np.random.default_rng(seed).uniform(0.4, 1.6, R)
    if empty is not None:
        w[empty] = 0.0
    return [0] + [int(x) for x in np.round(np.cumsum(w) / w.sum() * n)[:-1]] + [n]


def make_shards(metric, rows, labels, cuts, tc):
    shards = []
    for r in range(len(cuts) - 1):
        a, b = cuts[r], cuts[r + 1]
        s = rx.GpuBruteforceSearch(metric, rows.shape[1], max(b - a, 1))
        if b > a:
            s.add_points(labels[a:b], rows[a:b])
        s.set_tensor_core_filter(tc[r] if isinstance(tc, (list, tuple)) else tc)
        shards.append(s)
    return shards


def collective(shards, call):
    """call(comm, shard) on every rank, each from its own thread; returns [(result, last_search_stats)] by rank"""
    R = len(shards)
    comms = B.ShardComm.local_group(R)
    out, err = [None] * R, [None] * R

    def work(r):
        try:
            res = call(comms[r], shards[r])
            out[r] = (res, rx.last_search_stats())
        except Exception as e:  # noqa: BLE001 - reported by the main thread
            err[r] = e

    threads = [threading.Thread(target=work, args=(r,), daemon=True) for r in range(R)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads), "a rank is stuck in a collective"
    for c in comms:
        c.close()
    for e in err:
        if e is not None:
            raise e
    return out


def sharded_range(shards, queries, radii, max_out):
    return collective(shards, lambda comm, shard: comm.search_range_batch(shard, queries, radii, max_out))


def assert_same_range(want, got, max_out, ctx=""):
    D0, L0, N0 = want
    D, L, N = got
    assert (N == N0).all(), (ctx, np.argwhere(N != N0)[:5])
    valid = np.arange(max_out)[None, :] < np.minimum(N0, max_out)[:, None]
    assert (~valid | (L == L0)).all(), (ctx, np.argwhere(valid & (L != L0))[:5])
    assert (~valid | (D.view(np.uint32) == D0.view(np.uint32))).all(), (ctx, np.argwhere(valid & (D.view(np.uint32) != D0.view(np.uint32)))[:5])


def check_all_ranks(whole, queries, radii, max_out, results, singles=()):
    want = whole.search_range_batch(queries, radii, max_out)
    for r, (got, _) in enumerate(results):
        assert_same_range(want, got, max_out, ctx=("rank", r))
    D, L, N = results[0][0]
    for q in singles:  # one query at a time through rxgpu_search_range
        d, l, n = whole.search_range(queries[q], float(radii[q]), max_out)
        m = min(n, max_out)
        assert N[q] == n and (L[q, :m] == l).all() and (D[q, :m].view(np.uint32) == d.view(np.uint32)).all(), q
    return want


def rank_radii(d, nq):
    """radius of query i: its r-th best distance, r in RANKS (a row exactly there is excluded); every other group one ulp above"""
    r = np.empty(nq, np.float32)
    for i in range(nq):
        r[i] = d[i, RANKS[i % len(RANKS)] - 1]
        if (i // len(RANKS)) % 2:
            r[i] = np.nextafter(r[i], np.float32(np.inf))
    return r


def whole_index(metric, rows, labels):
    whole = rx.GpuBruteforceSearch(metric, rows.shape[1], len(rows))
    whole.add_points(labels, rows)
    whole.set_tensor_core_filter(2)  # the exact scan: a reference independent of the filter
    return whole


def exact_knn_dists(whole, queries, k):
    d, _, c = whole.search_knn(queries, k)
    assert (c == k).all()
    return d


def close_all(*objs):
    for o in objs:
        for x in (o if isinstance(o, list) else [o]):
            x.close()


@pytest.mark.parametrize("metric,dim,R", [(rx.L2, 64, 2), (rx.L2, 200, 5), (rx.L2, 768, 3), (rx.IP, 64, 3), (rx.IP, 200, 1),
                                          (rx.IP, 768, 2), (rx.COS, 64, 5), (rx.COS, 200, 2), (rx.COS, 768, 3)])
def test_filter_path_equals_single_index(metric, dim, R):
    n, nq, max_out = 30000 if dim < 768 else 20000, 64, 500
    rng = np.random.default_rng(dim + 7 * R + metric)
    rows = O.synth_matrix(0x9A0 + dim, n, dim)
    rows[n - 200:] = rows[:200]  # duplicated rows in other shards: equal distances under different labels
    labels = O.row_labels(n)[rng.permutation(n)]  # label order is not shard order
    whole = whole_index(metric, rows, labels)
    queries = np.stack([prep_query(metric, x) for x in O.synth_matrix(0x9A1 + dim + metric, nq, dim)])
    queries[5] = prep_query(metric, rows[7])
    d = exact_knn_dists(whole, queries, 100)
    radii = rank_radii(d, nq)
    radii[60] = d[60, 0] - abs(d[60, 0]) - 1.0  # below the best: no match
    radii[61], radii[62], radii[63] = np.nan, np.inf, -np.inf
    shards = make_shards(metric, rows, labels, uneven_cuts(n, R, dim), 1)
    res = sharded_range(shards, queries, radii, max_out)
    for _, st in res:
        assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    D0, L0, N0 = check_all_ranks(whole, queries, radii, max_out, res, singles=(0, 1, 2, 5, 33, 60, 62))
    assert N0[60] == N0[61] == N0[63] == 0 and N0[62] == n
    close_all(whole, shards)


@pytest.mark.parametrize("R,empty", [(1, None), (2, None), (3, None), (5, None), (2, 0), (3, 1), (5, 4)])
def test_exact_path_and_empty_shard(R, empty):
    """few queries: every shard takes the exact scan; shard `empty` holds no rows at all"""
    n, dim, nq, max_out = 12000, 96, 6, 300
    rows = O.synth_matrix(0x9B0, n, dim)
    labels = O.row_labels(n)[np.random.default_rng(R).permutation(n)]
    whole = whole_index(rx.L2, rows, labels)
    queries = O.synth_matrix(0x9B1, nq, dim)
    d = exact_knn_dists(whole, queries, 1000)
    radii = np.array([d[0, 0], d[1, 9], d[2, 99], d[3, 999], np.nextafter(d[4, 99], np.float32(np.inf)), np.inf], np.float32)
    shards = make_shards(rx.L2, rows, labels, uneven_cuts(n, R, 5, empty=empty), 0)
    res = sharded_range(shards, queries, radii, max_out)
    for _, st in res:
        assert st["tc_used"] == 0, st
    D0, L0, N0 = check_all_ranks(whole, queries, radii, max_out, res, singles=range(nq))
    assert N0[3] > max_out and N0[5] == n  # truncated by max_out
    close_all(whole, shards)


def test_mixed_paths_in_one_call():
    """the filter on some shards and the exact scan on others: a row's distance has the same bits on either path"""
    n, dim, nq, max_out, R = 40000, 128, 64, 1000, 4
    rows = O.synth_matrix(0x9C0, n, dim)
    labels = O.row_labels(n)[np.random.default_rng(9).permutation(n)]
    whole = whole_index(rx.IP, rows, labels)
    queries = O.synth_matrix(0x9C1, nq, dim)
    radii = rank_radii(exact_knn_dists(whole, queries, 100), nq)
    shards = make_shards(rx.IP, rows, labels, uneven_cuts(n, R, 2), [1, 2, 1, 2])
    res = sharded_range(shards, queries, radii, max_out)
    assert [st["tc_used"] for _, st in res] == [1, 0, 1, 0]
    check_all_ranks(whole, queries, radii, max_out, res, singles=(0, 31, 63))
    close_all(whole, shards)


@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
@pytest.mark.parametrize("tc", [1, 2])
def test_ties_across_shards(metric, tc):
    """integer rows: masses of bit-equal distances, spread over the shards, ordered by label; IP rows with zero dot products give
    zero distances on every shard"""
    n, dim, nq, max_out, R = 24000, 32, 64 if tc == 1 else 4, 20000, 3
    rng = np.random.default_rng(metric + 3 * tc)
    rows = rng.integers(-2, 3, size=(n, dim)).astype(np.float32)
    queries = rng.integers(-2, 3, size=(nq, dim)).astype(np.float32)
    if metric == rx.IP:
        rows[::50] = 0.0  # zero rows: every dot product with them is zero
        rows[1::50, : dim // 2] = 0.0
        queries[:, dim // 2:] = 0.0  # ... and half-zero rows against half-zero queries too
    labels = O.row_labels(n)[rng.permutation(n)]
    whole = whole_index(metric, rows, labels)
    d = exact_knn_dists(whole, queries, 1000)
    radii = rank_radii(d, nq)
    if metric == rx.IP:
        radii[: nq // 2] = np.float32(0.5)  # every row with a dot product >= 0 matches: the zero distances of all shards meet
    cuts = uneven_cuts(n, R, 4)
    shards = make_shards(metric, rows, labels, cuts, tc)
    res = sharded_range(shards, queries, radii, max_out)
    D0, L0, N0 = check_all_ranks(whole, queries, radii, max_out, res, singles=(0, 1, nq - 1))
    shard_of = {int(l): s for s in range(R) for l in labels[cuts[s]:cuts[s + 1]]}
    spans = 0
    for q in range(nq):  # runs of equal distances whose members come from more than one shard
        m = int(min(N0[q], max_out))
        for v in np.unique(D0[q, :m]):
            spans += len({shard_of[int(l)] for l in L0[q, :m][D0[q, :m] == v]}) > 1
    assert spans > nq
    if metric == rx.IP:
        assert (D0[: nq // 2, :] == 0).any()
    close_all(whole, shards)


def test_list_overflow_on_one_shard():
    """radii wide enough that the big shard's candidate lists overflow: that shard answers those queries with the exact scan"""
    n, dim, nq, max_out = 40000, 64, 64, 100  # lists of 4096 candidates
    rows = O.synth_matrix(0x9D0, n, dim)
    labels = O.row_labels(n)
    whole = whole_index(rx.L2, rows, labels)
    queries = O.synth_matrix(0x9D1, nq, dim)
    d = exact_knn_dists(whole, queries, 1000)
    radii = d[:, 499].copy()
    radii[:4] = exact_knn_dists(whole, queries[:4], 20000)[:, -1]  # about 18 000 of the matches on shard 0, 2 000 on shard 1
    shards = make_shards(rx.L2, rows, labels, [0, 36000, n], 1)
    res = sharded_range(shards, queries, radii, max_out)
    assert res[0][1]["tc_used"] == 1 and res[0][1]["tc_fallbacks"] >= 4, res[0][1]
    assert res[1][1]["tc_used"] == 1 and res[1][1]["tc_fallbacks"] == 0, res[1][1]
    D0, L0, N0 = check_all_ranks(whole, queries, radii, max_out, res, singles=(0, 3, 4))
    assert (N0[:4] > 4096).all()
    close_all(whole, shards)


def test_no_match_anywhere_and_special_radii():
    """no shard has a match (the agreed width is 0): totals 0, the output rows untouched"""
    n, dim, nq, max_out = 20000, 64, 64, 50
    rows = O.synth_matrix(0x9E0, n, dim)
    labels = O.row_labels(n)
    queries = O.synth_matrix(0x9E1, nq, dim)
    for tc in (1, 2):
        shards = make_shards(rx.L2, rows, labels, uneven_cuts(n, 3, 1), tc)
        radii = np.full(nq, -1.0, np.float32)
        radii[::3], radii[1::3] = np.nan, -np.inf
        res = sharded_range(shards, queries, radii, max_out)
        for (D, L, N), _ in res:
            assert (N == 0).all() and (D == 0).all() and (L == 0).all()
        close_all(shards)


def test_max_out_zero_nq_zero_and_arguments():
    n, dim, nq = 20000, 64, 64
    rows = O.synth_matrix(0x9F0, n, dim)
    labels = O.row_labels(n)
    whole = whole_index(rx.IP, rows, labels)
    queries = O.synth_matrix(0x9F1, nq, dim)
    radii = np.ascontiguousarray(exact_knn_dists(whole, queries, 10)[:, 9])  # passed to the C call as a pointer
    _, _, N0 = whole.search_range_batch(queries, radii, 10)
    shards = make_shards(rx.IP, rows, labels, uneven_cuts(n, 2, 3), 1)
    lib = B.lib()
    qp, rp = B._p(queries, B._f32p), B._p(radii, B._f32p)

    def max_out_zero(comm, shard):
        out_n = np.zeros(nq, np.uint64)
        B._check(lib.rxgpu_sharded_search_range_batch(comm._h, shard._h, nq, qp, 0, rp, 0, None, None, B._p(out_n, B._u64p)))
        return out_n

    for out_n, _ in collective(shards, max_out_zero):
        assert (out_n == N0).all()
    for (D, L, N), _ in collective(shards, lambda comm, shard: comm.search_range_batch(shard, queries[:0], radii[:0], 10)):
        assert D.shape == (0, 10) and len(N) == 0
    (comm,) = B.ShardComm.local_group(1)
    out_n = np.zeros(nq, np.uint64)
    d10 = np.zeros((nq, 10), np.float32)
    np_ = B._p(out_n, B._u64p)
    assert lib.rxgpu_sharded_search_range_batch(None, shards[0]._h, nq, qp, 0, rp, 0, None, None, np_) == 3
    assert lib.rxgpu_sharded_search_range_batch(comm._h, shards[0]._h, nq, None, 0, rp, 0, None, None, np_) == 3
    assert lib.rxgpu_sharded_search_range_batch(comm._h, shards[0]._h, nq, qp, 0, None, 0, None, None, np_) == 3
    assert lib.rxgpu_sharded_search_range_batch(comm._h, shards[0]._h, nq, qp, 0, rp, 0, None, None, None) == 3
    assert lib.rxgpu_sharded_search_range_batch(comm._h, shards[0]._h, nq, qp, 0, rp, 10, B._p(d10, B._f32p), None, np_) == 3
    comm.close()
    close_all(whole, shards)


def test_shard_on_another_device():
    if rx.device_count() < 2:
        pytest.skip("needs two GPUs")
    (comm,) = B.ShardComm.local_group(1, devices=[0])
    shard = rx.GpuBruteforceSearch(rx.L2, 16, 100, device=1)
    shard.append_synth(1, 0, 100)
    with pytest.raises(rx.RxGpuError) as e:
        comm.search_range_batch(shard, np.zeros((2, 16), np.float32), 1.0, 10)
    assert e.value.code == 3 and "another device" in e.value.what
    close_all(shard, comm)


def test_device_queries_and_sharded_search_object():
    import torch

    n, dim, nq, max_out = 30000, 96, 64, 200
    rows = O.synth_matrix(0xA00, n, dim)
    labels = O.row_labels(n)[np.random.default_rng(1).permutation(n)]
    whole = whole_index(rx.IP, rows, labels)
    queries = O.synth_matrix(0xA01, nq, dim)
    radii = rank_radii(exact_knn_dists(whole, queries, 100), nq)
    shards = make_shards(rx.IP, rows, labels, uneven_cuts(n, 3, 6), 1)
    dq = torch.from_numpy(queries).cuda()
    torch.cuda.synchronize()
    res = collective(shards, lambda comm, shard: comm.search_range_batch(shard, dq.data_ptr(), radii, max_out, nq=nq))
    want = check_all_ranks(whole, queries, radii, max_out, res)
    one = ShardedBruteforceSearch(whole, n)  # single rank, the C path
    assert one.comm is not None
    assert_same_range(want, one.search_range_batch(queries, radii, max_out), max_out)
    assert_same_range(want, one.search_range_batch(dq, radii, max_out), max_out)
    cpu_mode = ShardedBruteforceSearch(whole, n, local_search=lambda q, k1: None)  # the CPU / gloo mode has no range exchange
    with pytest.raises(NotImplementedError):
        cpu_mode.search_range_batch(queries, radii, max_out)
    one.comm.close()
    close_all(whole, shards)


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("tc", [0, 1])
def test_sharded_knn_in_process(R, tc):
    """rxgpu_sharded_search_knn on in-process ranks: the exchanges and the cross-shard tie replay run through the host rendezvous"""
    n, dim, k = 24000, 32, 10
    nq = 96 if tc else 5
    rng = np.random.default_rng(40 + R + tc)
    rows = rng.integers(-2, 3, size=(n, dim)).astype(np.float32)
    queries = rng.integers(-2, 3, size=(nq, dim)).astype(np.float32)
    labels = O.row_labels(n)[rng.permutation(n)]
    whole = whole_index(rx.L2, rows, labels)
    d0, l0, c0 = whole.search_knn(queries, k)
    shards = make_shards(rx.L2, rows, labels, uneven_cuts(n, R, 8), tc)
    res = collective(shards, lambda comm, shard: comm.search_knn(shard, queries, k))
    for r, ((d1, l1, c1), st) in enumerate(res):
        assert (c0 == c1).all() and (l0 == l1).all() and (d0.view(np.uint32) == d1.view(np.uint32)).all(), r
        assert st["tie_replays"] > 0, st  # integer rows tie at the k-th place
        assert st["tc_used"] == tc, st
        if tc:
            assert st["tie_from_lists"] == st["tie_replays"], st
    close_all(whole, shards)


def test_size_1m_four_shards():
    """1M x 768 inner product in four shards of 250k rows, 1024 queries, radius at each query's 10th-best distance: the filter on
    every rank, and the whole batch equal to the single index's"""
    n, dim, nq, max_out, R = 1_000_000, 768, 1024, 4096, 4
    whole = rx.GpuBruteforceSearch(rx.IP, dim, n)
    whole.append_synth(0xA10, 0, n)
    queries = O.synth_matrix(0xA11, nq, dim)
    d, _, c = whole.search_knn(queries, 10)
    assert (c == 10).all()
    radii = np.ascontiguousarray(d[:, 9])
    want = whole.search_range_batch(queries, radii, max_out)
    assert rx.last_search_stats()["tc_used"] == 1
    whole.close()
    shards = []
    for r in range(R):
        s = rx.GpuBruteforceSearch(rx.IP, dim, n // R)
        s.append_synth(0xA10, r * (n // R), n // R)  # rows and labels of rows [r n/R, (r+1) n/R) of the whole index
        shards.append(s)
    res = sharded_range(shards, queries, radii, max_out)
    for r, (got, st) in enumerate(res):
        assert st["tc_used"] == 1, (r, st)
        assert_same_range(want, got, max_out, ctx=r)
    assert want[2].sum() >= 9 * nq
    close_all(shards)


def test_two_ranks_nccl():
    if rx.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29619", os.path.join(ROOT, "tests", "mp_sharded_range_nccl.py")], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "mp_sharded_range_nccl ok" in r.stdout
