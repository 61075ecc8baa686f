"""GPU tests of the sharded IVF index: rxgpu_sharded_ivf_train, rxgpu_sharded_ivf_search_knn and rxgpu_sharded_ivf_search_range_batch.
The ranks are threads of one process on cuda:0 (ShardComm.local_group), so one GPU runs every cross-shard path.  The reference is one
index over all rows: rxgpu_ivf_train on the concatenation of the ranks' rows in rank order, rxgpu_ivf_add_assign of every row, then
rxgpu_ivf_search_knn_large_k / rxgpu_ivf_search_range_batch.  Equal means the same bits: centroids, per-iteration obj / nsplit, labels in
the same order and distance bits, on every rank.  The NCCL run with one process per GPU is tests/mp_sharded_ivf_nccl.py, launched by
test_two_ranks_nccl when the box has two GPUs."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import reindexer_b200 as rx
from reindexer_b200 import binding as B

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cuts_of(n, R, seed, empty=None):
    """row boundaries of R shards of uneven sizes; shard `empty` gets no rows"""
    w = np.random.default_rng(seed).uniform(0.3, 1.7, R)
    if empty is not None:
        w[empty] = 0.0
    return [0] + [int(x) for x in np.round(np.cumsum(w) / w.sum() * n)[:-1]] + [n]


def collective(R, call):
    """call(comm, r) on every rank of a fresh local group, each from its own thread (joined with a timeout: a stuck rank fails the
    test); returns ([result or None], [exception or None]) by rank"""
    comms = B.ShardComm.local_group(R)
    out, err = [None] * R, [None] * R

    def work(r):
        try:
            out[r] = call(comms[r], r)
        except Exception as e:  # noqa: BLE001 - reported by the caller
            err[r] = e

    threads = [threading.Thread(target=work, args=(r,), daemon=True) for r in range(R)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads), "a rank is stuck in a collective"
    for c in comms:
        c.close()
    return out, err


def ok(res):
    out, err = res
    for e in err:
        if e is not None:
            raise e
    return out


def data(seed, n, dim, dup=0):
    rng = np.random.default_rng(seed)
    x = rng.normal(0, 1, size=(n, dim)).astype(np.float32)
    x[: n // 3] += 2.0  # not one blob: some lists fill, some stay small
    if dup:
        x[-dup:] = x[0]  # identical rows: empty clusters that k-means must split
    return x


def norm_coefs(x):
    return (1.0 / np.linalg.norm(x, axis=1)).astype(np.float32)


def shards_for(metric, dim, R):
    return [rx.GpuBruteforceSearch(metric, dim, 1) for _ in range(R)]


def close(*objs):
    for o in objs:
        o.close()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- the assumption
@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
def test_assignment_key_does_not_depend_on_the_batch(metric):
    """A point's assignment (list and distance bits) is the same whether it is assigned alone, in a slice or in the whole batch: the
    sharded training assigns slices of the sample and relies on it."""
    dim, nlist = 48, 300
    x = data(1, 4000, dim)
    g = rx.GpuBruteforceSearch(metric, dim, 1)
    g.ivf_train(nlist, x, niter=2)
    l0, d0 = g.ivf_assign(x)
    for lo, hi in ((0, 1), (17, 18), (5, 12), (100, 1333), (3999, 4000), (1234, 4000)):
        l1, d1 = g.ivf_assign(x[lo:hi])
        assert (l1 == l0[lo:hi]).all() and (bits(d1) == bits(d0[lo:hi])).all(), (lo, hi)
    g.close()


# ---------------------------------------------------------------------------------------------------------------- training
TRAIN_CASES = [  # (metric, R, empty rank, n, dim, nlist, niter, max_points_per_centroid, with norm_coefs, duplicated rows)
    (rx.L2, 1, None, 3000, 24, 40, 6, 256, False, 0),
    (rx.L2, 2, None, 5000, 24, 40, 6, 50, False, 0),          # subsampled
    (rx.IP, 3, 1, 4000, 32, 64, 5, 256, False, 0),            # one empty rank
    (rx.COS, 5, None, 4500, 20, 50, 4, 40, False, 0),
    (rx.COS, 3, 0, 4500, 20, 50, 4, 256, True, 0),
    (rx.L2, 3, None, 2000, 16, 100, 8, 256, False, 1500),    # most rows identical: empty clusters split
    (rx.IP, 2, None, 2000, 16, 64, 0, 256, False, 0),         # niter = 0: the initial centroids
    (rx.L2, 3, 2, 64, 16, 64, 5, 256, False, 0),              # n == nlist: the centroids are the rows
    (rx.L2, 2, None, 262147, 4, 131072, 1, 256, False, 0),    # the largest nlist
    (rx.L2, 3, None, 300, 16, 150, 5, 1, False, 0),           # subsampled to nlist rows: the first 150 rows, over two ranks
    (rx.COS, 3, 0, 500, 16, 40, 3, 1, True, 0),               # the same with rank 0 empty, Cosine with norm_coefs
]


@pytest.mark.parametrize("case", range(len(TRAIN_CASES)))
def test_train_is_bit_identical_to_one_index(case):
    metric, R, empty, n, dim, nlist, niter, ppc, with_nc, dup = TRAIN_CASES[case]
    x = data(10 + case, n, dim, dup)
    nc = norm_coefs(x) * np.float32(1.5) if with_nc else None
    one = rx.GpuBruteforceSearch(metric, dim, 1)
    c0, s0 = one.ivf_train(nlist, x, norm_coefs=nc, niter=niter, max_points_per_centroid=ppc)
    cuts = cuts_of(n, R, case, empty)
    shards = shards_for(metric, dim, R)

    def run(comm, r):
        a, b = cuts[r], cuts[r + 1]
        return comm.ivf_train(shards[r], nlist, x[a:b], None if nc is None else nc[a:b], niter=niter, max_points_per_centroid=ppc)

    out = ok(collective(R, run))
    if dup:
        assert sum(s["nsplit"] for s in s0) > 0
    for r, (c, s) in enumerate(out):
        assert (bits(c) == bits(c0)).all(), (case, r, np.argwhere(bits(c) != bits(c0))[:4])
        assert [(t["obj"], t["nsplit"]) for t in s] == [(t["obj"], t["nsplit"]) for t in s0], (case, r)
        assert shards[r].ivf_size() == 0
    close(one, *shards)


# ---------------------------------------------------------------------------------------------------------------- search
class World:
    """R trained shards with their rows assigned (rank r holds rows [cuts[r], cuts[r + 1])), and one index over all rows"""

    def __init__(self, metric, R, n, dim, nlist, seed, empty=None, x=None, labels=None, cuts=None):
        self.metric, self.R, self.dim, self.nlist = metric, R, dim, nlist
        self.x = data(seed, n, dim) if x is None else x
        n = len(self.x)
        self.labels = (np.random.default_rng(seed).permutation(n).astype(np.uint64) << np.uint64(20)) + np.uint64(3) if labels is None else labels
        self.cuts = cuts_of(n, R, seed, empty) if cuts is None else cuts
        self.one = rx.GpuBruteforceSearch(metric, dim, 1)
        c0, _ = self.one.ivf_train(nlist, self.x, niter=4)
        self.one.ivf_add_assign(self.labels, self.x)
        self.shards = shards_for(metric, dim, R)
        out = ok(collective(R, lambda comm, r: comm.ivf_train(self.shards[r], nlist, self.part(r, self.x), niter=4)))
        assert all((bits(c) == bits(c0)).all() for c, _ in out)
        for r in range(R):
            if self.cuts[r + 1] > self.cuts[r]:
                self.shards[r].ivf_add_assign(self.part(r, self.labels), self.part(r, self.x))

    def part(self, r, a):
        return a[self.cuts[r]:self.cuts[r + 1]]

    def knn(self, q, k, nprobe):
        return collective(self.R, lambda comm, r: comm.ivf_search_knn(self.shards[r], q, k, nprobe))

    def range(self, q, radii, nprobe, max_out):
        return collective(self.R, lambda comm, r: comm.ivf_search_range_batch(self.shards[r], q, radii, nprobe, max_out))

    def model_knn(self, q, k, nprobe):
        """the (distance, rank, local row) model from each shard's own full answer: the k best by (distance, rank), then (distance,
        label) -- valid while no two rows of one shard tie"""
        per = []
        for r, s in enumerate(self.shards):
            m = s.ivf_size()
            if m == 0:
                continue
            d, l, c = s.ivf_search_knn_large_k(q, m, nprobe)
            per.append((d, l, c, r))
        res = []
        for i in range(len(q)):
            d = np.concatenate([p[0][i, :p[2][i]] for p in per])
            l = np.concatenate([p[1][i, :p[2][i]] for p in per])
            rk = np.concatenate([np.full(p[2][i], p[3]) for p in per])
            top = np.lexsort((rk, d))[:k]
            d, l = d[top], l[top]
            o = np.lexsort((l, d))
            res.append((d[o], l[o]))
        return res

    def close(self):
        close(self.one, *self.shards)


def assert_knn_equal(want, got, ctx):
    D0, L0, C0 = want
    for r, (D, L, C) in enumerate(got):
        assert (C == C0).all(), (ctx, r)
        for i in range(len(C0)):
            c = C0[i]
            assert (L[i, :c] == L0[i, :c]).all(), (ctx, r, i, L[i, :c][:8], L0[i, :c][:8])
            assert (bits(D[i, :c]) == bits(D0[i, :c])).all(), (ctx, r, i)


@pytest.fixture(scope="module")
def world():
    w = World(rx.L2, 3, 12000, 32, 64, 5)
    yield w
    w.close()


@pytest.mark.parametrize("k", [1, 10, 256, 257, 1000, 65535])
@pytest.mark.parametrize("nprobe", [1, 7, 64])
def test_knn_equals_one_index(world, k, nprobe):
    q = data(99, 40, world.dim)
    want = world.one.ivf_search_knn_large_k(q, k, nprobe)
    got = ok(world.knn(q, k, nprobe))
    assert_knn_equal(want, got, (k, nprobe))
    if k <= 1000:  # the (distance, rank, local row) model agrees where there are no ties
        for i, (d, l) in enumerate(world.model_knn(q, k, nprobe)):
            assert (got[0][1][i, :len(l)] == l).all() and (bits(got[0][0][i, :len(d)]) == bits(d)).all()


def test_one_query(world):
    """nq = 1: the coarse pass stages a single query alone"""
    q = data(94, 1, world.dim)
    for k, nprobe in ((10, 7), (1000, 64)):
        assert_knn_equal(world.one.ivf_search_knn_large_k(q, k, nprobe), ok(world.knn(q, k, nprobe)), (k, nprobe))
    d, _, _ = world.one.ivf_search_knn_large_k(q, 100, 64)
    for nprobe, max_out in ((7, 50), (64, 0)):
        want = world.one.ivf_search_range_batch(q, d[:, 99], nprobe, max_out)
        assert_range_equal(want, ok(world.range(q, d[:, 99], nprobe, max_out)), max_out, (nprobe, max_out))


def test_knn_single_rank_is_large_k_bit_for_bit():
    w = World(rx.IP, 1, 6000, 24, 32, 8)
    q = data(98, 300, 24)
    for k, nprobe in ((10, 3), (300, 32), (2000, 5)):
        assert_knn_equal(w.one.ivf_search_knn_large_k(q, k, nprobe), ok(w.knn(q, k, nprobe)), (k, nprobe))
        assert_knn_equal(w.shards[0].ivf_search_knn_large_k(q, k, nprobe), ok(w.knn(q, k, nprobe)), (k, nprobe))
    w.close()


def test_knn_past_one_query_chunk_and_k_above_all_rows():
    w = World(rx.COS, 2, 5000, 16, 16, 9)
    q = data(97, 300, 16)  # k = 65535: 256 queries per survivor chunk
    assert_knn_equal(w.one.ivf_search_knn_large_k(q, 65535, 16), ok(w.knn(q, 65535, 16)), "chunks")
    out = ok(w.knn(q[:3], 65535, 16))
    assert (out[0][2] == 5000).all()
    out = ok(w.knn(q[:0], 10, 4))
    assert all(len(c) == 0 for _, _, c in out)
    w.close()


def test_knn_after_removes_and_adds():
    w = World(rx.L2, 3, 9000, 24, 48, 11, empty=1)
    rng = np.random.default_rng(4)
    extra = data(12, 6000, 24)
    xl = (np.arange(6000, dtype=np.uint64) << np.uint64(20)) + np.uint64(7)
    for step in range(3):  # remove a third of a shard, then add more rows than it held: its slab relocates lists and compacts
        r = step % 3
        have = w.part(r, w.labels)
        if len(have):
            for lb in rng.choice(have, size=len(have) // 3, replace=False):
                w.shards[r].ivf_remove(int(lb))
                w.one.ivf_remove(int(lb))
        sl = slice(step * 2000, (step + 1) * 2000)
        w.shards[r].ivf_add_assign(xl[sl], extra[sl])
        w.one.ivf_add_assign(xl[sl], extra[sl])
    st = [s.ivf_list_stats() for s in w.shards]
    assert sum(s["relocations"] for s in st) > 0
    q = data(96, 50, 24)
    for k, nprobe in ((10, 5), (700, 48)):
        assert_knn_equal(w.one.ivf_search_knn_large_k(q, k, nprobe), ok(w.knn(q, k, nprobe)), (k, nprobe))
    w.close()


@pytest.mark.parametrize("k", [5, 300])
def test_knn_ties_across_ranks_follow_the_rank_model(k):
    """every rank holds a copy of the same rows: each distance appears R times, and the k-th place straddles copies"""
    R, dim = 3, 16
    base = data(21, 1500, dim)
    x = np.concatenate([base] * R)
    labels = (np.arange(len(x), dtype=np.uint64)[::-1].copy() << np.uint64(8)) + np.uint64(1)  # label order against rank order
    w = World(rx.L2, R, 0, dim, 24, 21, x=x, labels=labels, cuts=[0, 1500, 3000, 4500])
    q = base[:20] + np.float32(0.01)
    kk = k - 1 if k % R == 0 else k  # k not a multiple of R: the k-th place cuts a group of R copies
    got = ok(w.knn(q, kk, 24))
    for i, (d, l) in enumerate(w.model_knn(q, kk, 24)):
        for D, L, C in got:
            assert C[i] == kk and (L[i, :kk] == l).all() and (bits(D[i, :kk]) == bits(d)).all(), i
    w.close()


def assert_range_equal(want, got, max_out, ctx):
    D0, L0, N0 = want
    valid = np.arange(max_out)[None, :] < np.minimum(N0, max_out)[:, None]
    for r, (D, L, N) in enumerate(got):
        assert (N == N0).all(), (ctx, r, np.argwhere(N != N0)[:4])
        assert (~valid | (L == L0)).all(), (ctx, r)
        assert (~valid | (bits(D) == bits(D0))).all(), (ctx, r)


@pytest.mark.parametrize("nprobe", [1, 7, 64])
@pytest.mark.parametrize("max_out", [0, 1, 50, 4000])
def test_range_equals_one_index(world, nprobe, max_out):
    q = data(95, 30, world.dim)
    d, _, _ = world.one.ivf_search_knn_large_k(q, 200, 64)
    radii = d[np.arange(30), np.array([1, 20, 200])[np.arange(30) % 3] - 1].copy()
    radii[:6] = [np.nan, -np.inf, np.inf, 0.0, -1.0, 1e-30]
    want = world.one.ivf_search_range_batch(q, radii, nprobe, max_out)
    assert_range_equal(want, ok(world.range(q, radii, nprobe, max_out)), max_out, (nprobe, max_out))


def test_range_no_match_anywhere_and_on_one_shard_only(world):
    r = 2
    q = world.part(r, world.x)[:8].copy()  # each query is a row of rank 2: a radius just above its distance matches it there only
    d, _, _ = world.one.ivf_search_knn_large_k(q, 1, 3)
    for radii, n in ((np.nextafter(d[:, 0], np.float32(np.inf)), 1), (np.full(8, -5.0, np.float32), 0)):
        want = world.one.ivf_search_range_batch(q, radii, 3, 10)
        got = ok(world.range(q, radii, 3, 10))
        assert_range_equal(want, got, 10, n)
        assert (want[2] == n).all()


# ---------------------------------------------------------------------------------------------------------------- errors
def codes(res):
    out, err = res
    assert all(e is not None for e in err), err
    return [e.code for e in err]


def test_errors_are_agreed_and_leave_every_index_unchanged():
    dim, R = 16, 3
    x = data(31, 900, dim)
    cuts = cuts_of(900, R, 31)
    shards = shards_for(rx.L2, dim, R)
    bad = x.copy()
    bad[cuts[1] + 3, 5] = np.nan  # a NaN in rank 1's rows only
    assert codes(collective(R, lambda comm, r: comm.ivf_train(shards[r], 20, bad[cuts[r]:cuts[r + 1]]))) == [3] * R
    assert codes(collective(R, lambda comm, r: comm.ivf_train(shards[r], 901, x[cuts[r]:cuts[r + 1]]))) == [3] * R  # n < nlist
    assert codes(collective(R, lambda comm, r: comm.ivf_train(shards[r], 20 + (r == 2), x[cuts[r]:cuts[r + 1]]))) == [3] * R
    for s in shards:  # still empty, with no lists: the next training succeeds
        assert s.ivf_size() == 0
        with pytest.raises(rx.RxGpuError):
            s.ivf_list_stats()
    ok(collective(R, lambda comm, r: comm.ivf_train(shards[r], 20, x[cuts[r]:cuts[r + 1]], niter=2)))
    for r in range(R):
        shards[r].ivf_add_assign(np.arange(cuts[r], cuts[r + 1], dtype=np.uint64), x[cuts[r]:cuts[r + 1]])
    q = data(32, 4, dim)
    ok(collective(R, lambda comm, r: comm.ivf_search_knn(shards[r], q, 5, 3)))
    other = rx.GpuBruteforceSearch(rx.L2, dim, 1)  # rank 1 searches lists over other centroids
    other.ivf_train(20, x[::-1].copy(), niter=2)
    mixed = [shards[0], other, shards[2]]
    assert codes(collective(R, lambda comm, r: comm.ivf_search_knn(mixed[r], q, 5, 3))) == [4] * R
    assert codes(collective(R, lambda comm, r: comm.ivf_search_range_batch(mixed[r], q, 1.0, 3, 10))) == [4] * R
    assert codes(collective(R, lambda comm, r: comm.ivf_search_knn(shards[r], q, 5, 3 + r))) == [4] * R  # nprobe differs
    plain = [shards[0], rx.GpuBruteforceSearch(rx.L2, dim, 1), shards[2]]  # rank 1 has no lists: its error reaches everyone
    assert codes(collective(R, lambda comm, r: comm.ivf_search_knn(plain[r], q, 5, 3))) == [4] * R
    assert codes(collective(R, lambda comm, r: comm.ivf_search_range_batch(plain[r], q, 1.0, 3, 10))) == [4] * R
    ok(collective(R, lambda comm, r: comm.ivf_search_range_batch(shards[r], q, 1.0, 3, 10)))
    close(other, plain[1], *shards)


def test_two_ranks_nccl():
    if rx.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29623", os.path.join(ROOT, "tests", "mp_sharded_ivf_nccl.py")], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "mp_sharded_ivf_nccl ok" in r.stdout
