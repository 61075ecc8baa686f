"""GPU tests of the index's mutable state against a model of the index (tests/index_model.py) through sequences of upserts, removes,
resizes, clones, synthetic appends, IVF list updates and HNSW graph updates.

The library keeps derived state in step with every mutation: the int8 shadow of the rows and its per-row constants (brought up to
date from a log of rewritten ranges), the Cosine norms, the label dictionary, the filter's candidate lists that the tie replay
reuses, the IVF slab and its list bounds, and the device copy of an HNSW graph.  None of it can be checked by comparing the library
with itself, since every search path reads the same rows, norms and labels.  So every case applies one schedule of bursts to the GPU
index, to an IndexModel and, for integer-valued rows, to the C port of the reference's map (oracle.PortBF), and after every burst
checks the GPU against them:
  * every live label's row, bit for bit, and the size, capacity and device bytes;
  * float rows: every search path (exact scan, filter, staged thresholds, range batch on both, single-query range) against the fp64
    envelope of test_fp64_envelope_gpu.py over the model's rows in internal order, the filter bit-identical to the exact scan;
  * integer rows (values in {-2, ..., 2}: every summation order gives the same bits): labels, order and distance bits equal to the
    port on every path, with ties at the k-th place, and the filter's tie replay served from its candidate lists.
Queries are aimed at the rows the last burst wrote, so a row whose shadow, constants or norm went stale changes the answer."""
import ctypes as C
import threading

import numpy as np
import pytest
from hnsw_replay import search_knn as replay_knn
from index_model import HnswModel, IndexModel, IvfModel, LogicError, NotFound
from test_fp64_envelope_gpu import Envelope, assert_identical, check_knn, check_range, probed_rows, radii_at
from test_hnsw_exact_gpu import check_one, random_graph
from test_sq8_exact_gpu import params_for

import reindexer_b200 as rx
from oracle import oracle as O
from reindexer_b200 import binding as B

pytestmark = pytest.mark.gpu

F = np.float32
ERR_LOGIC, ERR_NOT_FOUND = 4, 13
METRICS = [rx.L2, rx.IP, rx.COS]
MNAME = {rx.L2: "l2", rx.IP: "ip", rx.COS: "cos"}
SLICE_768 = (64 << 20) // (768 * 4)  # rows per staging slice of rxgpu_index_upsert_batch at 768 dims


def lab(ids):
    return (np.asarray(ids, np.uint64) << np.uint64(32)) | np.uint64(5)


class Pool:
    """integer rows drawn from a pool of n // 8 distinct non-zero vectors: every distance is shared by several rows, so ties straddle
    the k-th place of most queries"""

    def __init__(self, rng, n, dim):
        self.v = rng.integers(-2, 3, size=(max(n // 8, 4), dim)).astype(F)
        self.v[~self.v.any(1), 0] = 1
        self.rng = rng

    def rows(self, n):
        return self.v[self.rng.integers(0, len(self.v), size=n)]


class Mirror:
    """one GPU index, its model and (integer rows) the port, mutated together"""

    def __init__(self, metric, dim, cap, integer, seed, host_mirror=False):
        self.metric, self.dim, self.integer = metric, dim, integer
        self.rng = np.random.default_rng(seed)
        self.gpu = rx.GpuBruteforceSearch(metric, dim, cap, host_mirror=host_mirror)
        self.model = IndexModel(metric, dim, cap)
        self.port = O.PortBF(metric, dim, cap) if integer else None
        self.pool = Pool(self.rng, 4096, dim) if integer else None
        self.touched = set()
        self.next_id = 1

    def fresh(self, n):
        ids = np.arange(self.next_id, self.next_id + n)
        self.next_id += n
        return lab(ids)

    def vecs(self, n, scale=0.25):
        if self.integer:
            return self.pool.rows(n)
        return (self.rng.standard_normal((n, self.dim)) * scale).astype(F)

    def upsert(self, labels, vecs):
        labels = np.ascontiguousarray(labels, np.uint64)
        vecs = np.ascontiguousarray(vecs, F).reshape(len(labels), self.dim)
        err = None
        try:
            self.gpu.add_points(labels, vecs)
        except rx.RxGpuError as e:
            err = e
        full = False
        try:
            self.model.upsert(labels, vecs)
        except LogicError:
            full = True
        if self.port is not None:
            assert (self.port.add_batch(labels, vecs) != 0) == full
        assert (err is not None) == full, err
        assert err is None or err.code == ERR_LOGIC, err
        pos = self.model.row_of(labels)
        self.touched.update(pos[pos >= 0].tolist())
        return full

    def remove(self, label):
        cur = int(self.model.row_of([label])[0])
        self.gpu.remove_point(int(label))
        self.model.remove(label)
        if self.port is not None:
            self.port.remove(int(label))
        if 0 <= cur < self.model.size:
            self.touched.add(cur)  # the hole now holds the former last row

    def resize(self, cap):
        err = None
        try:
            self.gpu.resize_index(cap)
        except rx.RxGpuError as e:
            err = e
        try:
            self.model.resize(cap)
            assert err is None, err
            if self.port is not None:
                assert self.port.resize(cap) == 0
        except LogicError:
            assert err is not None and err.code == ERR_LOGIC, err

    def live(self, n):
        return self.rng.choice(self.model.label_array(), size=n, replace=False)

    def queries(self, nq=24):
        """rows the last bursts wrote (a few nudged for float data) and a few others"""
        m = self.model
        touched = np.array(sorted(p for p in self.touched if p < m.size), np.int64)
        self.touched = set()
        pick = self.rng.choice(touched, size=min(len(touched), nq - 4), replace=False) if len(touched) else np.zeros(0, np.int64)
        pick = np.concatenate([pick, self.rng.integers(0, m.size, size=nq - len(pick))])
        q = m.rows[pick].astype(F)
        if not self.integer:
            q = (q + self.rng.standard_normal(q.shape) * 0.01 * (np.abs(q).mean() + 1e-3)).astype(F)
        return q


def device_bytes(metric, dim, cap):
    cap = max(cap, 1)
    return cap * ((dim + 3) // 4 * 4) * 4 + cap * 8 + (cap * 4 if metric == rx.COS else 0)


def check_rows(gpu, model, ctx=""):
    assert gpu.current_element_count() == model.size and gpu.max_elements() == model.capacity, ctx
    assert gpu.device_bytes() == device_bytes(model.metric, model.dim, model.capacity), ctx
    for i, label in enumerate(model.labels):
        got = gpu.float_ptr_by_external_label(label)
        assert (got.view(np.uint32) == model.rows[i].view(np.uint32)).all(), (ctx, "stored row differs", i, label)


def knn(gpu, queries, k, mode):
    gpu.set_tensor_core_filter(mode)
    out = gpu.search_knn(queries, k)
    return out, rx.last_search_stats()


def same_as_port(port, queries, out, k, ctx):
    d, l, c = out
    for q in range(len(queries)):
        dp, lp = port.search_knn(queries[q], k)
        assert c[q] == len(lp), (ctx, q, int(c[q]), len(lp))
        assert (l[q, :len(lp)] == lp).all(), (ctx, q, "labels differ from the port", l[q, :8], lp[:8])
        assert (d[q, :len(lp)].view(np.uint32) == dp.view(np.uint32)).all(), (ctx, q, "distance bits differ from the port")


def same_range_as_port(port, queries, radii, out, ctx):
    d, l, c = out
    for q in range(len(queries)):
        dp, lp = port.search_range(queries[q], float(radii[q]))
        assert c[q] == len(lp), (ctx, q, int(c[q]), len(lp))
        assert (l[q, :len(lp)] == lp).all() and (d[q, :len(lp)].view(np.uint32) == dp.view(np.uint32)).all(), (ctx, q)


def verify(mx, ctx="", ks=(10, 300), queries=None, rows=True):
    """every check of the module docstring on one Mirror"""
    gpu, m = mx.gpu, mx.model
    if rows:
        check_rows(gpu, m, ctx)
    if m.size == 0:
        return
    queries = mx.queries() if queries is None else queries
    env = None if mx.integer else Envelope(m.metric, m.rows, queries)
    ties = 0
    for k in ks:
        if k >= m.size and k > 10:
            continue
        ref, st = knn(gpu, queries, k, 2)
        assert st["tc_used"] == 0, st
        got, st = knn(gpu, queries, k, 1)
        assert st["tc_used"] == 1, (ctx, k, st)
        assert (st["passes"] == 1) if k + 1 <= 128 else (st["passes"] >= 2), (ctx, k, st)
        if mx.integer:
            assert st["tie_from_lists"] == st["tie_replays"], (ctx, k, st)
            ties += st["tie_replays"]
            same_as_port(mx.port, queries, ref, k, (ctx, k, "exact"))
        else:
            check_knn(env, *ref, k, ctx=(ctx, k), row_of=m.row_of)
        assert_identical(ref, got, ctx=(ctx, k, "filter"))
    if mx.integer:
        assert ties > 0, (ctx, "no tie was replayed")
        radii = np.array([np.sort(m.distances(q))[min(20, m.size - 1)] for q in queries], F)
    else:
        radii = radii_at(env)
    gpu.set_tensor_core_filter(2)
    exact = gpu.search_range_batch(queries, radii)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_range_batch(queries, radii)
    assert rx.last_search_stats()["tc_used"] == 1
    assert_identical(exact, got, ctx=(ctx, "range"))
    singles = [gpu.search_range(queries[q], float(radii[q])) for q in range(4)]
    if mx.integer:
        same_range_as_port(mx.port, queries, radii, exact, (ctx, "range"))
        for q, (d, l, n) in enumerate(singles):
            dp, lp = mx.port.search_range(queries[q], float(radii[q]))
            assert n == len(lp) and (l == lp).all() and (d.view(np.uint32) == dp.view(np.uint32)).all(), (ctx, "single range", q)
    else:
        check_range(env, radii, *exact, ctx=(ctx, "range"), row_of=m.row_of)
        for q, (d, l, n) in enumerate(singles):
            e1 = Envelope(m.metric, m.rows, queries[q])
            check_range(e1, radii[q], d[None], l[None], [n], ctx=(ctx, "single range", q), row_of=m.row_of)


# ---------------------------------------------------------------------------------------------------------------- a. shadow, then churn


@pytest.mark.parametrize("dim", [3, 97, 128, 768])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_shadow_built_then_churn(metric, dim):
    integer = dim in (3, 97)
    mx = Mirror(metric, dim, 2600, integer, seed=dim * 3 + metric, host_mirror=dim in (3, 128))
    mx.upsert(mx.fresh(1500), mx.vecs(1500))
    verify(mx, "built")  # the shadow exists from here on
    for burst in range(4):
        m = mx.model
        # scattered rewrites, moved onto (integer) or next to (float) other rows, which the queries then aim at
        targets = mx.live(60)
        near = m.rows[mx.rng.integers(0, m.size, size=60)]
        mx.upsert(targets, near if integer else near + mx.vecs(60, 0.01))
        mx.upsert(mx.fresh(40 + burst), mx.vecs(40 + burst))  # an appended run
        for label in mx.live(25):
            mx.remove(label)
        mx.remove(m.labels[-1])  # the last row
        gone = int(mx.live(1)[0])
        mx.remove(gone)
        mx.upsert([gone], mx.vecs(1))  # its label comes back, appended
        mx.remove(int(lab([10**6 + burst])[0]))  # unknown: nothing happens
        verify(mx, ("burst", burst))


# ---------------------------------------------------------------------------------------------------------------- b. the dirty log


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_dirty_log_at_its_edge(metric):
    """between two filter searches, 4095, 4096 and 4097 disjoint one-row rewrites (the log holds 4096 ranges and gives up beyond), then
    adjacent rewrites one call each (they coalesce into one range), then the same rows in descending order (which never coalesce)"""
    dim, n = 97, 9000
    mx = Mirror(metric, dim, n, False, seed=0xB0 + metric)
    mx.upsert(mx.fresh(n), mx.vecs(n))
    verify(mx, "built", ks=(10,))
    for count in (4095, 4096, 4097):
        pos = np.arange(0, 2 * count, 2)  # every other row: no two ranges touch
        labels = mx.model.label_array()[pos]
        src = mx.rng.integers(0, n, size=count)
        mx.upsert(labels, mx.model.rows[src] + mx.vecs(count, 0.01))
        mx.touched = {int(pos[-1]), int(pos[-2]), int(pos[0])} | set(mx.rng.choice(pos, 16).tolist())
        verify(mx, ("disjoint", count), ks=(10,), rows=count == 4097)
    for order in ("ascending", "descending"):
        pos = np.arange(100, 5300)
        if order == "descending":
            pos = pos[::-1]
        for p in pos:
            mx.upsert([mx.model.labels[p]], mx.model.rows[mx.rng.integers(0, n, size=1)] + mx.vecs(1, 0.01))
        mx.touched = {int(pos[-1]), int(pos[0])} | set(mx.rng.choice(pos, 20).tolist())
        verify(mx, order, ks=(10,), rows=False)


# ---------------------------------------------------------------------------------------------------------------- c. batch mechanics


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_batch_mechanics(metric):
    dim = 768
    mx = Mirror(metric, dim, SLICE_768 + 700, True, seed=0xC0 + metric)
    mx.upsert(mx.fresh(1000), mx.vecs(1000))
    verify(mx, "built", ks=(10,))
    # a label repeated inside one slice (rewrites and appends mixed): the last write wins
    labels = np.concatenate([mx.live(20), mx.fresh(20)])
    labels = np.concatenate([labels, labels[::3], labels[5:9]])
    mx.upsert(labels, mx.vecs(len(labels)))
    verify(mx, "repeat in a slice", ks=(10,))
    # a batch of more than one slice, with a label repeated on both sides of the slice boundary
    labels = np.concatenate([mx.live(500), mx.fresh(SLICE_768 - 500 + 100)])
    mx.rng.shuffle(labels)
    labels[SLICE_768 + 50] = labels[SLICE_768 - 50]
    labels[SLICE_768] = labels[SLICE_768 - 1]
    assert len(labels) > SLICE_768
    mx.upsert(labels, mx.vecs(len(labels)))
    verify(mx, "repeat across slices", ks=(10,))
    # a batch that reaches the capacity midway: LOGIC, its leading rows applied
    room = mx.model.capacity - mx.model.size
    labels = np.concatenate([mx.live(3), mx.fresh(room + 10)])
    assert mx.upsert(labels, mx.vecs(len(labels)))
    assert mx.model.size == mx.model.capacity
    verify(mx, "full", ks=(10,))


# ---------------------------------------------------------------------------------------------------------------- d. resize and clone


@pytest.mark.parametrize("dim", [97, 128])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_resize_and_clone(metric, dim):
    mx = Mirror(metric, dim, 1200, True, seed=0xD0 + metric + dim)
    mx.upsert(mx.fresh(1100), mx.vecs(1100))
    verify(mx, "built", ks=(10, 300))
    for step, cap in (("grow", 1800), ("to size", None), ("refused shrink", -1)):
        cap = mx.model.size if cap is None else mx.model.size - 1 if cap == -1 else cap
        mx.resize(cap)
        mx.touched = set(range(mx.model.size - 10, mx.model.size))
        verify(mx, step, ks=(10, 300))
        if step == "grow":
            mx.upsert(mx.fresh(300), mx.vecs(300))
            for label in mx.live(40):
                mx.remove(label)
            verify(mx, "churn after grow")
    # a clone taken after churn equals the model; then each side is mutated alone
    cm = Mirror.__new__(Mirror)
    cm.__dict__.update(mx.__dict__)
    cm.gpu = mx.gpu.clone(mx.model.capacity + 100)
    cm.model = mx.model.clone(mx.model.capacity + 100)
    cm.port = mx.port.clone(mx.model.capacity + 100)
    cm.touched = set()
    verify(cm, "clone")
    mx.upsert(mx.live(50), mx.vecs(50))
    mx.upsert(mx.fresh(60), mx.vecs(60))
    for label in mx.live(30):
        mx.remove(label)
    verify(mx, "source after its clone")
    verify(cm, "clone after the source changed", queries=mx.queries())
    cm.upsert(cm.live(50), cm.vecs(50))
    for label in cm.live(30):
        cm.remove(label)
    verify(cm, "clone changed")
    verify(mx, "source after the clone changed", queries=cm.queries())


# ---------------------------------------------------------------------------------------------------------------- e. Cosine norms


@pytest.mark.parametrize("dim", [3, 97, 128, 768])
def test_cosine_norms_follow_the_rows(dim):
    """rows rewritten between unit norm, the |1 - s| <= 1e-5 edge, norms far from 1 and zero, through the scatter path, the append
    fast path (pitch == dim) and swap-removes"""
    mx = Mirror(rx.COS, dim, 3000, False, seed=0xE0 + dim)
    rng = mx.rng

    def shaped(n):
        base = rng.standard_normal((n, dim))
        base /= np.linalg.norm(base, axis=1, keepdims=True)
        s = rng.choice([1.0, 1 + 2e-6, 1 - 2e-6, 1 + 1e-5, 1 - 1e-5, 1 + 4e-5, 1 - 4e-5, 100.0, 1e-4, 0.0], size=n)
        return (base * np.sqrt(s)[:, None]).astype(F)

    mx.upsert(mx.fresh(2000), shaped(2000))
    verify(mx, "built")
    for burst in range(3):
        m = mx.model
        targets = mx.live(200)
        # the same directions at other norms: a stale norm coefficient scales the distance of exactly these rows
        old = m.rows[m.row_of(targets)].astype(np.float64)
        nrm = np.linalg.norm(old, axis=1, keepdims=True)
        unit = np.where(nrm > 0, old / np.where(nrm > 0, nrm, 1), shaped(200))
        s = rng.choice([1.0, 1 + 1e-5, 1 - 1e-5, 100.0, 1e-4, 0.0], size=200)
        mx.upsert(targets, (unit * np.sqrt(s)[:, None]).astype(F))  # scattered rewrites
        mx.upsert(mx.fresh(100), shaped(100))  # an append: the fast path at 128 and 768 dims, the scatter path at 3 and 97
        for label in mx.live(60):
            mx.remove(label)
        verify(mx, ("burst", burst))


# ---------------------------------------------------------------------------------------------------------------- f. lists invalidated


@pytest.mark.parametrize("dim", [3, 97])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_tie_lists_invalidated_by_mutation(metric, dim):
    """filter KNN on tie-heavy rows builds the candidate lists; rows inside those lists are then rewritten, removed and re-added, and
    the next KNN with ties must equal the port again"""
    mx = Mirror(metric, dim, 3000, True, seed=0xF0 + metric + dim)
    mx.upsert(mx.fresh(2500), mx.vecs(2500))
    queries = mx.queries()
    for burst in range(3):
        (d, l, c), st = knn(mx.gpu, queries, 300, 1)
        assert st["tie_replays"] > 0 and st["tie_from_lists"] == st["tie_replays"], st
        same_as_port(mx.port, queries, (d, l, c), 300, ("before", burst))
        hit = np.unique(l[:, :300].ravel())
        hit = mx.rng.choice(hit, size=min(len(hit), 200), replace=False)
        mx.upsert(hit[:120], mx.vecs(120))
        for label in hit[120:]:
            mx.remove(int(label))
        mx.upsert(hit[150:], mx.vecs(len(hit) - 150))
        verify(mx, ("after", burst), queries=queries)


# ---------------------------------------------------------------------------------------------------------------- g. append_synth


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_append_synth_interleaved(metric):
    dim, seed = 128, 0x600 + metric
    mx = Mirror(metric, dim, 6000, False, seed=seed)
    first = 100
    for burst in range(4):
        n = 700 + 13 * burst
        mx.gpu.append_synth(seed, first, n)
        mx.model.append_synth(seed, first, n)
        mx.touched.update(range(mx.model.size - n, mx.model.size))
        mx.upsert(mx.live(40), mx.vecs(40))
        mx.upsert(lab(np.arange(first, first + 40)), mx.vecs(40))  # plain upserts beside the synthetic labels
        for label in mx.live(30):
            mx.remove(label)
        # a synthetic run whose labels are fresh at first and then reach a live one is refused and leaves the index as it was
        with pytest.raises(rx.RxGpuError) as e:
            mx.gpu.append_synth(seed, first - 30, 40)
        assert e.value.code == ERR_LOGIC
        with pytest.raises(LogicError):
            mx.model.append_synth(seed, first - 30, 40)
        first += n + 50
        verify(mx, ("burst", burst))
    more = mx.fresh(30)
    mx.upsert(more, mx.vecs(30))
    for label in more[:10]:
        mx.remove(int(label))
    verify(mx, "after")


def test_automatic_routing_after_churn_100k():
    dim, n, seed = 128, 100_000, 0x100
    mx = Mirror(rx.IP, dim, n + 1000, False, seed=seed)
    mx.gpu.append_synth(seed, 0, n)
    mx.model.append_synth(seed, 0, n)
    queries = mx.queries(64)
    mx.gpu.set_tensor_core_filter(0)
    mx.gpu.search_knn(queries, 10)  # 64 queries on 100 k rows: the filter builds its shadow
    assert rx.last_search_stats()["tc_used"] == 1
    mx.upsert(mx.fresh(400), mx.vecs(400))
    targets = mx.live(500)
    mx.upsert(targets, mx.model.rows[mx.rng.integers(0, n, size=500)] + mx.vecs(500, 0.01))
    for label in mx.live(200):
        mx.remove(label)
    queries = mx.queries(64)
    mx.gpu.set_tensor_core_filter(0)
    d, l, c = mx.gpu.search_knn(queries, 10)
    assert rx.last_search_stats()["tc_used"] == 1
    check_knn(Envelope(rx.IP, mx.model.rows, queries), d, l, c, 10, row_of=mx.model.row_of)
    check_rows(mx.gpu, mx.model)


# ---------------------------------------------------------------------------------------------------------------- h. sharded


def collective(shards, call):
    comms = B.ShardComm.local_group(len(shards))
    out, err = [None] * len(shards), [None] * len(shards)

    def work(r):
        try:
            out[r] = call(comms[r], shards[r])
        except Exception as e:  # noqa: BLE001 - reported by the main thread
            err[r] = e

    threads = [threading.Thread(target=work, args=(r,), daemon=True) for r in range(len(shards))]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    for c in comms:
        c.close()
    assert not any(t.is_alive() for t in threads)
    for e in err:
        if e is not None:
            raise e
    return out


def concat(mirrors, metric, dim):
    m = IndexModel(metric, dim, sum(x.model.capacity for x in mirrors))
    for x in mirrors:
        m.upsert(x.model.labels, x.model.rows)
    return m


@pytest.mark.parametrize("integer", [True, False], ids=["int", "float"])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_sharded_in_process(metric, integer):
    dim = 97 if integer else 768
    ms = [Mirror(metric, dim, 1500, integer, seed=0x700 + 10 * r + metric) for r in range(3)]
    for r, mx in enumerate(ms):
        mx.next_id = 1 + r * 10**6
        if integer:
            mx.pool = ms[0].pool
        mx.upsert(mx.fresh(900 + 50 * r), mx.vecs(900 + 50 * r))
    for burst in range(3):
        for r, mx in enumerate(ms):
            mx.upsert(mx.fresh(40), mx.vecs(40))
            if mx.model.size:
                mx.upsert(mx.live(30), mx.vecs(30))
                for label in mx.live(20):
                    mx.remove(label)
        if burst == 1:  # one shard emptied, then refilled
            for label in list(ms[1].model.labels):
                ms[1].remove(label)
            assert ms[1].model.size == 0
        if burst == 2:
            ms[1].upsert(ms[1].fresh(700), ms[1].vecs(700))
        for mx in ms:
            check_rows(mx.gpu, mx.model, ("shard", burst))
        whole = concat(ms, metric, dim)
        src = [mx for mx in ms if mx.model.size]
        queries = np.concatenate([x.queries(8) for x in src])
        for k in (10, 300):
            for mx in ms:
                mx.gpu.set_tensor_core_filter(1)
            out = collective(ms, lambda comm, mx, k=k: comm.search_knn(mx.gpu, queries, k))
            for d, l, c in out[1:]:
                assert_identical(out[0], (d, l, c), ctx=(burst, k, "ranks differ"))
            d, l, c = out[0]
            if integer:
                for q in range(len(queries)):
                    dm, lm = whole.knn(queries[q], k)
                    assert c[q] == len(lm) and (l[q, :len(lm)] == lm).all(), (burst, k, q, l[q, :8], lm[:8])
                    assert (d[q, :len(lm)].view(np.uint32) == dm.view(np.uint32)).all(), (burst, k, q)
            else:
                check_knn(Envelope(metric, whole.rows, queries), d, l, c, k, ctx=(burst, k), row_of=whole.row_of)
        if integer:
            radii = np.array([np.sort(whole.distances(q))[20] for q in queries], F)
        else:
            radii = radii_at(Envelope(metric, whole.rows, queries))
        out = collective(ms, lambda comm, mx: comm.search_range_batch(mx.gpu, queries, radii, whole.size))
        d, l, c = out[0]
        if integer:
            for q in range(len(queries)):
                dm, lm = whole.range_search(queries[q], radii[q])
                assert c[q] == len(lm) and (l[q, :len(lm)] == lm).all(), (burst, q)
                assert (d[q, :len(lm)].view(np.uint32) == dm.view(np.uint32)).all(), (burst, q)
        else:
            check_range(Envelope(metric, whole.rows, queries), radii, d, l, c, ctx=burst, row_of=whole.row_of)


# ---------------------------------------------------------------------------------------------------------------- IVF mutable lists


@pytest.mark.parametrize("metric", [rx.L2, rx.COS], ids=MNAME.get)
def test_ivf_lists_through_relocations_and_compaction(metric):
    dim, nlist = 16, 64
    rng = np.random.default_rng(0x1F + metric)
    cents = (rng.standard_normal((nlist, dim)) * 0.25).astype(F)
    gpu = rx.GpuBruteforceSearch(metric, dim, 16)
    gpu.ivf_create(cents)
    model = IvfModel(nlist, dim)
    next_id = [1]
    removed = []

    def add(lists):
        labels = lab(np.arange(next_id[0], next_id[0] + len(lists)))
        next_id[0] += len(lists)
        vecs = (rng.standard_normal((len(lists), dim)) * 0.25).astype(F)
        gpu.ivf_add(np.asarray(lists, np.uint32), labels, vecs)
        model.add(lists, labels, vecs)

    def remove(label):
        gpu.ivf_remove(int(label))
        model.remove(label)
        removed.append(int(label))

    def check(ctx):
        assert gpu.ivf_size() == model.size, ctx
        rows, labels, lists = model.flat()
        pos = {int(x): i for i, x in enumerate(labels)}

        def row_of(ls):
            return np.array([pos.get(int(x), -1) for x in np.asarray(ls).ravel()], np.int64)

        queries = (rows[rng.integers(0, len(rows), size=12)] + rng.standard_normal((12, dim)).astype(F) * 0.02).astype(F)
        env = Envelope(metric, rows, queries)
        for k in (10, 256):
            d, l, c = gpu.ivf_search_knn(queries, k, nlist)
            check_knn(env, d, l, c, k, ctx=(ctx, k), row_of=row_of)
        for q in range(3):
            e1 = Envelope(metric, rows, queries[q])
            radius = np.float32(np.sort(e1.mid[0])[min(30, len(rows) - 1)])
            rd, rl, total = gpu.ivf_search_range(queries[q], float(radius), nlist)
            check_range(e1, radius, rd[None], rl[None], [total], ctx=(ctx, "range", q), row_of=row_of)
        for nprobe in (1, 4):
            allowed, clear = probed_rows(metric, cents, queries, lists, nprobe)
            d, l, c = gpu.ivf_search_knn(queries, 10, nprobe)
            e = Envelope(metric, rows, queries[clear]).restrict(allowed[clear])
            check_knn(e, d[clear], l[clear], c[clear], 10, ctx=(ctx, nprobe), row_of=row_of)

    add(rng.integers(0, nlist, size=2000))
    check("built")
    st0 = gpu.ivf_list_stats()
    for burst in range(20):  # four lists grow by about 75 rows a burst: relocated again and again
        add(rng.integers(0, 4, size=300))
    st1 = gpu.ivf_list_stats()
    assert st1["relocations"] > st0["relocations"] and st1["dead_rows"] > 0, st1
    check("grown")
    lst0 = [l for l, _ in model.lists[0]]
    remove(lst0[-1])  # the last entry of a list
    for label in [l for l, _ in model.lists[5]]:  # a list emptied
        remove(label)
    assert not model.lists[5]
    live = np.array(list(model.where), np.uint64)
    for label in rng.choice(live, size=5000, replace=False):
        remove(label)
    with pytest.raises(rx.RxGpuError) as e:
        gpu.ivf_remove(removed[0])
    assert e.value.code == ERR_NOT_FOUND
    check("removed")
    st2 = gpu.ivf_list_stats()
    assert st2["dead_rows"] > model.size + 100 + 4096, st2
    add(rng.integers(0, nlist, size=100))  # more dead space than live rows: the slab is compacted first
    st3 = gpu.ivf_list_stats()
    assert st3["compactions"] == st2["compactions"] + 1 and st3["dead_rows"] == 0, st3
    check("compacted")
    back = removed[:50]  # removed labels come back, into other lists
    vecs = (rng.standard_normal((50, dim)) * 0.25).astype(F)
    lists = rng.integers(0, nlist, size=50)
    gpu.ivf_add(lists.astype(np.uint32), np.array(back, np.uint64), vecs)
    model.add(lists, back, vecs)
    with pytest.raises(rx.RxGpuError) as e:
        gpu.ivf_add(np.zeros(1, np.uint32), np.array(back[:1], np.uint64), vecs[:1])
    assert e.value.code == ERR_LOGIC
    check("re-added")


# ---------------------------------------------------------------------------------------------------------------- HNSW maintenance


def slot_labels(hm, lab_):
    """GPU labels -> slot << 32, the form check_one reads"""
    slots = hm.slot_of(lab_)
    assert (slots >= 0).all()
    return (slots.astype(np.uint64) << np.uint64(32)).reshape(np.shape(lab_))


def hnsw_table(gpu, hm, queries):
    gpu.set_tensor_core_filter(2)
    d, l, c = gpu.search_knn(queries, hm.n)
    assert (c == hm.n).all()
    t = np.zeros((len(queries), hm.n), F)
    for q in range(len(queries)):
        t[q, hm.slot_of(l[q])] = d[q]
    env = Envelope(gpu.metric, hm.rows, queries)
    assert ((env.lo <= t) & (t <= env.hi)).all()
    return t


def check_hnsw(gpu, hm, queries, ctx):
    assert gpu.hnsw_update_count() == hm.updates and gpu.hnsw_deleted_count() == len(hm.deleted), ctx
    assert gpu.current_element_count() == hm.n
    table = hnsw_table(gpu, hm, queries)
    fresh = rx.GpuBruteforceSearch(gpu.metric, gpu.dim, hm.n)
    fresh.add_points(np.array(hm.labels, np.uint64), hm.rows)
    fresh.hnsw_import(hm.graph())
    for v in sorted(hm.deleted):
        fresh.hnsw_mark_deleted(hm.labels[v])
    clean = 0
    for k, ef in ((10, 0), (10, 64), (40, 200)):
        d, l, c, st = gpu.hnsw_search_knn(queries, k, ef, with_stats=True)
        ref = fresh.hnsw_search_knn(queries, k, ef, with_stats=True)
        assert_identical((d, l, c), ref[:3], ctx=(ctx, k, ef, "fresh import"))
        assert (st == ref[3]).all(), (ctx, k, ef)
        for q in range(len(queries)):
            rep = replay_knn(hm.graph(), lambda ids, q=q: table[q][ids], k, ef, frozenset(hm.deleted))
            sl = slot_labels(hm, l[q, :c[q]])
            clean += check_one(d[q], sl, c[q], st[q], table[q], rep, hm.deleted, (ctx, k, ef, q))
    assert clean >= 0.75 * 3 * len(queries), (ctx, "too many tied queries")
    fresh.close()


def new_lists(g, rng, v, n_after, level):
    l0 = rng.choice(n_after, size=min(g["maxM0"], n_after - 1), replace=False)
    l0 = l0[l0 != v][: g["maxM0"]]
    ups = []
    for lv in range(1, level + 1):
        cand = [u for u in range(n_after) if u != v and (u >= len(g["levels"]) or g["levels"][u] >= lv)]
        ups.append(rng.choice(cand, size=min(g["M"], len(cand)), replace=False) if cand else [])
    return l0, ups


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_hnsw_maintenance(metric):
    dim, n, extra = 16, 2000, 24
    rng = np.random.default_rng(0x4E + metric)
    rows = (rng.standard_normal((n, dim)) * 0.5).astype(F)
    g = random_graph(0x4E + metric, n, 16, M=8, maxlevel=3)
    labels = O.row_labels(n)
    gpu = rx.GpuBruteforceSearch(metric, dim, n + extra)
    gpu.add_points(labels, rows)
    gpu.hnsw_import(g)
    hm = HnswModel(g, rows, labels)
    queries = (rng.standard_normal((16, dim)) * 0.5).astype(F)
    check_hnsw(gpu, hm, queries, "imported")

    def push(nodes, new_rows=None):
        gpu.hnsw_update(hm.graph(), nodes, new_rows, deleted=hm.deleted)
        hm.updates += len(set(nodes) | set(new_rows or {}))

    # appended nodes of levels 0-3, linked from existing nodes
    new_rows = {}
    for i, level in enumerate([0, 1, 2, 3, 0, 1]):
        v = hm.n
        l0, ups = new_lists(hm.g, rng, v, v + 1, level)
        vec = queries[i] + (rng.standard_normal(dim) * 0.01).astype(F)
        hm.append(int(lab([10**5 + i])[0]), vec, level, l0, ups)
        new_rows[v] = (hm.labels[v], vec)
    linked = rng.choice(n, size=40, replace=False)
    for u in linked:
        l0 = hm.g["level0"][u, 1:1 + hm.g["level0"][u, 0]].copy()
        l0[-1] = n + int(rng.integers(0, len(new_rows)))
        hm.set_lists(u, level0=np.unique(l0))
    push(list(linked), new_rows)
    check_hnsw(gpu, hm, queries, "appended")
    # rewritten neighbour lists, updatePoint of existing nodes
    nodes = rng.choice(hm.n, size=60, replace=False)
    for u in nodes[:30]:
        hm.set_lists(int(u), level0=new_lists(hm.g, rng, int(u), hm.n, 0)[0])
    moved = {}
    for u in nodes[30:]:
        vec = queries[int(rng.integers(0, len(queries)))] + (rng.standard_normal(dim) * 0.05).astype(F)
        hm.update_point(int(u), hm.labels[int(u)], vec)
        moved[int(u)] = (hm.labels[int(u)], vec)
    push(list(nodes[:30]), moved)
    check_hnsw(gpu, hm, queries, "lists and points")
    # tombstones set, then some cleared
    dead = rng.choice(hm.n, size=200, replace=False)
    hm.deleted |= set(int(x) for x in dead)
    push([int(x) for x in dead])
    check_hnsw(gpu, hm, queries, "tombstones")
    back = [int(x) for x in dead[:60]]
    hm.deleted -= set(back)
    push(back)
    check_hnsw(gpu, hm, queries, "tombstones cleared")
    # a tombstoned slot's label lives again: in an appended slot, and in an existing slot through updatePoint
    a, b, c_ = (int(x) for x in dead[100:103])
    v = hm.n
    l0, _ = new_lists(hm.g, rng, v, v + 1, 0)
    vec = queries[0] + (rng.standard_normal(dim) * 0.02).astype(F)
    label_a = hm.labels[a]
    hm.append(label_a, vec, 0, l0, [])
    other = int(rng.choice([u for u in range(n) if u not in hm.deleted]))
    label_b = hm.labels[b]
    vec_b = queries[1] + (rng.standard_normal(dim) * 0.02).astype(F)
    hm.update_point(other, label_b, vec_b)
    hm.labels[other] = label_b
    push([], {v: (label_a, vec), other: (label_b, vec_b)})
    assert hm.labels[a] == (1 << 63) | a and hm.labels[b] == (1 << 63) | b
    check_hnsw(gpu, hm, queries, "labels reborn")
    # hnsw_mark_deleted
    for u in rng.choice([u for u in range(hm.n) if u not in hm.deleted], size=30, replace=False):
        gpu.hnsw_mark_deleted(hm.labels[int(u)])
        hm.deleted.add(int(u))
    check_hnsw(gpu, hm, queries, "marked")
    del c_

    # staleness is refused: a stream opened before an update reports exhausted ...
    q = np.ascontiguousarray(queries[0], F)
    s = C.c_void_p()
    B._check(gpu._lib.rxgpu_hnsw_stream_begin(gpu._h, B._p(q, B._f32p), 32, C.byref(s)))
    try:
        u = int(rng.integers(0, n))
        hm.set_lists(u, level0=new_lists(hm.g, rng, u, hm.n, 0)[0])
        hm.update_point(u, hm.labels[u], hm.rows[u] + F(0.5))
        push([], {u: (hm.labels[u], hm.rows[u])})
        d = np.zeros(8, F)
        lab_ = np.zeros(8, np.uint64)
        cnt, ex = C.c_uint32(0), C.c_int(0)
        B._check(gpu._lib.rxgpu_hnsw_stream_next(s, 8, B._p(d, B._f32p), B._p(lab_, B._u64p), C.byref(cnt), C.byref(ex)))
        assert ex.value == 1 and cnt.value == 0
    finally:
        gpu._lib.rxgpu_hnsw_stream_end(s)
    check_hnsw(gpu, hm, queries, "after the stream")
    # ... and a brute-force upsert without hnsw_update leaves the graph stale
    gpu.add_point(hm.rows[3] + F(1), hm.labels[3])
    with pytest.raises(rx.RxGpuError) as e:
        gpu.hnsw_search_knn(queries, 10, 32)
    assert e.value.code == ERR_LOGIC
    gpu.close()


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_sq8_refuses_after_a_row_mutation(metric):
    dim, n = 16, 500
    rng = np.random.default_rng(0x58 + metric)
    rows = (rng.standard_normal((n, dim)) * 0.3).astype(F)
    queries = (rng.standard_normal((4, dim)) * 0.3).astype(F)
    norms = np.ones(len(queries), F) if metric == rx.COS else None
    for mutate in ("upsert", "append", "remove"):
        gpu = rx.GpuBruteforceSearch(metric, dim, n + 1)
        gpu.add_points(O.row_labels(n), rows)
        gpu.sq8_attach(params_for(metric, dim))
        gpu.sq8_search_knn(queries, 10, norms)
        if mutate == "upsert":
            gpu.add_point(rows[0] * 2, int(O.row_labels(1)[0]))
        elif mutate == "append":
            gpu.add_point(rows[0], int(O.row_labels(1, n)[0]))
        else:
            gpu.remove_point(int(O.row_labels(1, 7)[0]))
        with pytest.raises(rx.RxGpuError):
            gpu.sq8_search_knn(queries, 10, norms)
        gpu.close()
