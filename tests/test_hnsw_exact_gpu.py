"""GPU tests of the HNSW kernels (reindexer_b200/csrc/hnsw.cu) against an exact replay of the reference's traversal.

A row's fp32 distance on the HNSW path is computed with the per-row arithmetic of the exact scan, so the scan's full result
(search_knn with k = n) is a table of the very distances the HNSW kernels see.  Given that table, the reference's traversal
(tests/hnsw_replay.py) is a deterministic function of the graph, and every query must come back exactly as the replay says:
labels, distance bits, count, distance evaluations and hops.  For every case:
  (a) every returned distance is bit-equal to the table entry of its row;
  (b) every query whose replay took no decision between two equal distances matches the replay exactly;
  (c) the few tie-flagged queries still return sorted, duplicate-free, live rows with table-exact distances.
The table itself is held to the fp64 envelope of test_fp64_envelope_gpu.py.  SQ8 graphs use the bit-exact SQ8 formula of
test_sq8_exact_gpu.py as their table.  The graphs are generated here, so no test needs the reference build."""
import ctypes as C

import numpy as np
import pytest
from hnsw_replay import Stream, search_knn, search_range
from test_fp64_envelope_gpu import Envelope, check_knn
from test_sq8_exact_gpu import params_for, query_codes, quantize, sq8_table

import reindexer_b200 as rx
from oracle import oracle as O
from reindexer_b200 import binding as B

pytestmark = pytest.mark.gpu

F = np.float32
METRICS = [rx.L2, rx.IP, rx.COS]
MNAME = {rx.L2: "l2", rx.IP: "ip", rx.COS: "cos"}
MAX_TIE_SHARE = 0.25  # high dimensions concentrate distances, and a heap pop between equal distances is undefined

# ---------------------------------------------------------------------------------------------------------------- graphs


def distinct_ids(rng, own, size, m):
    """[len(own), m] ids in [0, size), distinct per row and never the row's own id: offsets are cumulative sums of positive gaps"""
    if m == 0 or size < 2:
        return np.zeros((len(own), 0), np.int64)
    m = min(m, size - 1)
    gap = max(1, (size - 1) // m)
    off = np.cumsum(rng.integers(1, gap + 1, size=(len(own), m)), axis=1)
    return rng.permuted((np.asarray(own)[:, None] + off) % size, axis=1)


def random_graph(seed, n, maxM0, M=16, maxlevel=2, fill="full", upper_fill="full", ep_empty_upper=False, split=None, isolated=False):
    """a valid hnsw_import dict: level-0 lists of random distinct neighbours ("full": maxM0 each, "mixed": 0..maxM0, some empty),
    `split` = first node of a second component that no level-0 list crosses, `isolated` = the last node has no list and is in none;
    levels geometric up to maxlevel, the enter point on the top level"""
    rng = np.random.default_rng(seed)
    level0 = np.zeros((n, 1 + maxM0), np.uint32)
    comps = [(0, n)]
    if split:
        comps = [(0, split), (split, n)]
    if isolated:
        last = comps[-1]
        comps[-1] = (last[0], n - 1)
        comps.append((n - 1, n))
    for lo, hi in comps:
        size = hi - lo
        ids = distinct_ids(rng, np.arange(size), size, maxM0) + lo
        m = ids.shape[1]
        cnt = np.full(size, m) if fill == "full" else rng.integers(0, m + 1, size=size)
        if fill != "full" and size > 4:
            cnt[rng.integers(0, size, size=max(1, size // 50))] = 0
            cnt[rng.integers(0, size, size=max(1, size // 10))] = m
        level0[lo:hi, 0] = cnt
        for j in range(m):
            level0[lo:hi, 1 + j] = np.where(j < cnt, ids[:, j], 0)
    levels = np.zeros(n, np.int32)
    if maxlevel:
        levels = np.minimum(rng.geometric(0.5, size=n) - 1, maxlevel).astype(np.int32)
        levels[n - 1] = 0 if isolated else levels[n - 1]
    ep = int(rng.integers(0, n - 1 if isolated else n))
    levels[ep] = maxlevel
    offs = np.zeros(n + 1, np.int64)
    offs[1:] = np.cumsum(levels)
    upper = np.zeros((int(offs[-1]), 1 + M), np.uint32)
    for lv in range(1, maxlevel + 1):
        nodes = np.nonzero(levels >= lv)[0]
        ids = nodes[distinct_ids(rng, np.arange(len(nodes)), len(nodes), M)]
        m = ids.shape[1]
        cnt = np.full(len(nodes), m) if upper_fill == "full" else rng.integers(0, m + 1, size=len(nodes))
        slot = offs[nodes] + lv - 1
        upper[slot, 0] = cnt
        for j in range(m):
            upper[slot, 1 + j] = np.where(j < cnt, ids[:, j], 0)
    if ep_empty_upper and maxlevel:
        upper[offs[ep]:offs[ep] + maxlevel, 0] = 0
    return dict(n=n, M=M, maxM0=maxM0, maxlevel=maxlevel, enterpoint=ep, level0=level0, levels=levels, upper_offsets=offs, upper=upper)


# ---------------------------------------------------------------------------------------------------------------- data


def unit64(x):
    x = np.asarray(x, np.float64)
    nrm = np.linalg.norm(x, axis=1, keepdims=True)
    return (x / np.where(nrm == 0, 1.0, nrm)).astype(F)


def rows_for(metric, seed, n, dim, zero_rows=0):
    x = (np.random.default_rng(seed).standard_normal((n, dim)) * 0.5).astype(F)
    if metric == rx.COS:
        x = unit64(x)
        x[1:1 + zero_rows] = 0
    return x


def make_index(metric, rows, g):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], len(rows))
    gpu.add_points(O.row_labels(len(rows)), rows)
    gpu.hnsw_import(g)
    return gpu


def fp32_table(gpu, metric, rows, queries, envelope=True):
    """every row's distance from the exact scan, indexed by row; checked against the certified fp64 envelope"""
    n = len(rows)
    gpu.set_tensor_core_filter(2)
    d, lab, cnt = gpu.search_knn(queries, n)
    assert (cnt == n).all()
    t = np.zeros((len(queries), n), F)
    for q in range(len(queries)):
        t[q, (lab[q] >> np.uint64(32)).astype(np.int64)] = d[q]
    if envelope:
        env = Envelope(metric, rows, queries)
        bad = np.argwhere(~((env.lo <= t) & (t <= env.hi)))
        assert len(bad) == 0, ("table outside the fp64 envelope", bad[:5])
    return t


def rows_of(lab):
    return (np.asarray(lab) >> np.uint64(32)).astype(np.int64)


# ---------------------------------------------------------------------------------------------------------------- checks


def check_one(d, lab, cnt, stats, table_q, rep, deleted=frozenset(), ctx=""):
    """(a), then (b) or (c) for one query; returns whether the replay was tie-free"""
    c = int(cnt)
    rows = rows_of(lab[:c])
    dq = d[:c]
    assert (dq.view(np.uint32) == table_q[rows].view(np.uint32)).all(), (ctx, "distance differs from the table", rows[:5])
    if not rep.tie:
        want = np.array([v for _, v in rep.top], np.int64)
        assert c == len(want), (ctx, c, len(want))
        assert (rows == want).all(), (ctx, rows[:8], want[:8])
        assert (dq.view(np.uint32) == np.array([x for x, _ in rep.top], F).view(np.uint32)).all(), ctx
        if stats is not None:
            assert (int(stats[0]), int(stats[1])) == (rep.n_dist, rep.hops), (ctx, tuple(stats), (rep.n_dist, rep.hops))
        return True
    assert c == len(rep.top), (ctx, c, len(rep.top))
    assert len(np.unique(rows)) == c and not (set(rows.tolist()) & set(deleted)), ctx
    assert all((dq[i], rows[i]) <= (dq[i + 1], rows[i + 1]) for i in range(c - 1)), (ctx, "not sorted")
    return False


def run_knn(gpu, g, table, queries, k, ef, deleted=frozenset(), ctx="", max_tie_share=MAX_TIE_SHARE):
    d, lab, cnt, st = gpu.hnsw_search_knn(queries, k, ef, with_stats=True)
    reps, clean = [], 0
    for q in range(len(queries)):
        rep = search_knn(g, lambda ids, q=q: table[q][ids], k, ef, deleted)
        clean += check_one(d[q], lab[q], cnt[q], st[q], table[q], rep, deleted, (ctx, q))
        reps.append(rep)
    assert len(queries) - clean <= max_tie_share * len(queries) + 1, (ctx, "too many tied queries", len(queries) - clean)
    return reps, (d, lab, cnt)


def slots_with_one_cta_per_sm(monkeypatch):
    import torch

    monkeypatch.setenv("RXGPU_HNSW_CTAS_PER_SM", "1")  # read by hnsw_import: slots = SMs x 1 CTA x 4 warps
    return 4 * torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------- dimensions


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("dim", [1, 3, 4, 5, 127, 128, 129, 257, 1000, 2048, 4096])
def test_dimensions(metric, dim):
    n = 1000 if dim >= 2048 else 2500
    rows = rows_for(metric, dim, n, dim, zero_rows=2)
    g = random_graph(dim + 10 * metric, n, 32, M=16, maxlevel=3)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, dim + 1, 24, dim)
    table = fp32_table(gpu, metric, rows, queries)
    # one-dimensional unit rows are +-1: every Cosine distance ties with half the rows, so only (a) and (c) can be asked there
    share = 1.0 if (metric == rx.COS and dim == 1) else MAX_TIE_SHARE
    for k, ef in ((10, 0), (10, 64), (1, 200)):
        run_knn(gpu, g, table, queries, k, ef, ctx=(dim, k, ef), max_tie_share=share)


# ---------------------------------------------------------------------------------------------------------------- graph shapes


@pytest.mark.parametrize("maxM0", [2, 31, 32, 33, 63, 64])
def test_graph_shapes(maxM0):
    """level-0 lists full, partly full and empty; an isolated node; two components; maxlevel 0, 1 and 6; upper lists of exactly M
    and partly full; an enter point whose upper lists are empty"""
    metric, dim, n = rx.L2, 24, 3000
    rows = rows_for(metric, maxM0, n, dim)
    queries = rows_for(metric, maxM0 + 1, 16, dim)
    variants = [
        dict(fill="full", maxlevel=0),
        dict(fill="mixed", maxlevel=1, isolated=True),
        dict(fill="mixed", maxlevel=6, split=n // 3, upper_fill="mixed"),
        dict(fill="full", maxlevel=6, ep_empty_upper=True),
    ]
    table = None
    for i, v in enumerate(variants):
        g = random_graph(100 * maxM0 + i, n, maxM0, M=max(2, maxM0 // 2), **v)
        gpu = make_index(metric, rows, g)
        if table is None:
            table = fp32_table(gpu, metric, rows, queries)
        for k, ef in ((10, 1), (10, 40), (50, 300)):
            run_knn(gpu, g, table, queries, k, ef, ctx=(maxM0, v, k, ef))


def test_upper_lists_of_33_to_64_neighbours():
    """M = 64: the upper-level descent reads lists of up to 64 neighbours (two 32-lane rounds)"""
    metric, dim, n = rx.IP, 20, 4000
    rows = rows_for(metric, 5, n, dim)
    queries = rows_for(metric, 6, 16, dim)
    for M, upper_fill in ((33, "full"), (64, "full"), (64, "mixed")):
        g = random_graph(M, n, 64, M=M, maxlevel=4, upper_fill=upper_fill)
        assert g["upper"][:, 0].max() == M or upper_fill == "mixed"
        gpu = make_index(metric, rows, g)
        table = fp32_table(gpu, metric, rows, queries)
        run_knn(gpu, g, table, queries, 10, 32, ctx=(M, upper_fill))
    with pytest.raises(rx.RxGpuError, match="must be <= 64"):
        make_index(metric, rows, random_graph(1, n, 64, M=65, maxlevel=1))


# ---------------------------------------------------------------------------------------------------------------- ef and k


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_ef_and_k(metric):
    dim, n = 16, 800
    rows = rows_for(metric, 77, n, dim)
    g = random_graph(77, n, 24, M=12, maxlevel=2)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 78, 16, dim)
    table = fp32_table(gpu, metric, rows, queries)
    for ef in (0, 1, 2, 3, 4, 5, 1023, 1024):
        for k in (1, 3, 10, 100):
            run_knn(gpu, g, table, queries, k, ef, ctx=(ef, k))
    for k in (n, n + 5):  # k = n and k > n: min(k, n) results
        reps, (d, lab, cnt) = run_knn(gpu, g, table, queries, k, 1024, ctx=k)
    # ef >= n on a connected graph visits every row: the result is the exact brute force, checked against the fp64 envelope too
    env = Envelope(metric, rows, queries)
    for k in (10, n):
        reps, (d, lab, cnt) = run_knn(gpu, g, table, queries, k, 1000, ctx=("ef>=n", k))
        assert all(r.visited == n for r in reps)
        check_knn(env, d, lab, cnt, k, ctx=("ef>=n", k))
    with pytest.raises(rx.RxGpuError, match="ef must be <= 1024"):
        gpu.hnsw_search_knn(queries, 10, 1025)


# ---------------------------------------------------------------------------------------------------------------- shared memory


def test_shared_memory_edges():
    """(nch * 512 + efp * 8 + 512) * 4 <= 200 KiB for the search, nch * 512 + 16896 <= 200 KiB for a streaming session"""
    metric, n = rx.L2, 48
    for dim, ef, served in ((10624, 1024, True), (10625, 1024, False), (12544, 1, True), (12545, 1, False)):
        rows = rows_for(metric, dim, n, dim)
        g = random_graph(dim, n, 8, M=4, maxlevel=1)
        gpu = make_index(metric, rows, g)
        queries = rows_for(metric, dim + 1, 3, dim)
        if served:
            table = fp32_table(gpu, metric, rows, queries)
            run_knn(gpu, g, table, queries, 5, ef, ctx=(dim, ef))
        else:
            with pytest.raises(rx.RxGpuError, match="dimension/ef combination"):
                gpu.hnsw_search_knn(queries, 5, ef)
    for dim, served in ((46976, True), (46977, False)):
        rows = rows_for(metric, dim, 16, dim)
        g = random_graph(dim, 16, 4, M=2, maxlevel=0)
        gpu = make_index(metric, rows, g)
        if served:
            batches = list(gpu.hnsw_stream(rows[3], 16, 8))
            d = np.concatenate([b[0] for b in batches]).astype(np.float64)
            got = rows_of(np.concatenate([b[1] for b in batches]))
            env = Envelope(metric, rows, rows[3:4])
            assert len(got) >= 1 and len(np.unique(got)) == len(got)
            assert ((env.lo[0, got] <= d) & (d <= env.hi[0, got])).all()
        else:
            with pytest.raises(rx.RxGpuError, match="shared-memory budget of the streaming"):
                list(gpu.hnsw_stream(rows[3], 16, 8))


# ---------------------------------------------------------------------------------------------------------------- slots


def test_slot_reuse(monkeypatch):
    """with one CTA per SM a batch larger than the slot count makes every warp serve several queries from one visited bitmap"""
    slots = slots_with_one_cta_per_sm(monkeypatch)
    metric, dim, n = rx.L2, 12, 5000
    rows = rows_for(metric, 3, n, dim)
    g = random_graph(3, n, 48, M=24, maxlevel=3)
    gpu = make_index(metric, rows, g)
    base = rows_for(metric, 4, 16, dim)
    table = fp32_table(gpu, metric, rows, base)
    reps, (d0, l0, c0) = run_knn(gpu, g, table, base, 10, 200, ctx="distinct")
    assert min(r.visited for r in reps) > 100
    for nq in (slots - 1, slots, slots + 1, 3 * slots + 7):
        d, lab, cnt, st = gpu.hnsw_search_knn(base[np.arange(nq) % 16], 10, 200, with_stats=True)
        for i in range(nq):
            j = i % 16
            assert cnt[i] == c0[j] and (lab[i, :cnt[i]] == l0[j, :c0[j]]).all(), (nq, i)
            assert (d[i, :cnt[i]].view(np.uint32) == d0[j, :c0[j]].view(np.uint32)).all(), (nq, i)
            check_one(d[i], lab[i], cnt[i], st[i], table[j], reps[j], ctx=(nq, i))


def test_visited_log_overflow_clears_the_whole_bitmap(monkeypatch):
    """queries that visit more than 2^15 nodes clear the whole bitmap instead of the logged words; later queries on the same slot
    must see a clean bitmap"""
    slots = slots_with_one_cta_per_sm(monkeypatch)
    metric, dim, n = rx.L2, 8, 50000
    rows = rows_for(metric, 11, n, dim)
    g = random_graph(11, n, 64, M=32, maxlevel=3)
    gpu = make_index(metric, rows, g)
    cands = rows_for(metric, 12, 12, dim)
    table = fp32_table(gpu, metric, rows, cands, envelope=False)
    # tens of thousands of visited distances make an equal pair in the heaps likely: keep the tie-free queries that overflow the log
    reps = [search_knn(g, lambda ids, q=q: table[q][ids], 10, 1024) for q in range(len(cands))]
    keep = [q for q, r in enumerate(reps) if not r.tie and r.visited > 1 << 15][:4]
    assert len(keep) >= 2, [(r.visited, r.tie) for r in reps]
    nq = 3 * slots
    pick = np.array(keep)[np.arange(nq) % len(keep)]
    d, lab, cnt, st = gpu.hnsw_search_knn(cands[pick], 10, 1024, with_stats=True)
    for i in range(nq):
        check_one(d[i], lab[i], cnt[i], st[i], table[pick[i]], reps[pick[i]], ctx=i)


# ---------------------------------------------------------------------------------------------------------------- tombstones


def delete(gpu, n, ids):
    lab = O.row_labels(n)
    for i in ids:
        gpu.hnsw_mark_deleted(int(lab[i]))
    return frozenset(int(i) for i in ids)


@pytest.mark.parametrize("share", [0.0, 0.5, 0.95])
def test_tombstones(share):
    metric, dim, n = rx.IP, 16, 4000
    rows = rows_for(metric, 21, n, dim)
    g = random_graph(21, n, 32, M=16, maxlevel=3)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 22, 16, dim)
    table = fp32_table(gpu, metric, rows, queries)
    rng = np.random.default_rng(23)
    deleted = delete(gpu, n, np.nonzero(rng.random(n) < share)[0]) if share else frozenset()
    for k, ef in ((10, 0), (10, 100), (30, 400)):
        run_knn(gpu, g, table, queries, k, ef, deleted, ctx=(share, k, ef))


def test_deleted_enter_point_and_its_neighbours():
    metric, dim, n = rx.L2, 16, 3000
    rows = rows_for(metric, 31, n, dim)
    queries = rows_for(metric, 32, 16, dim)
    for case in ("enter point", "its level-0 neighbours", "both"):
        g = random_graph(31, n, 16, M=8, maxlevel=0)
        gpu = make_index(metric, rows, g)
        table = fp32_table(gpu, metric, rows, queries, envelope=False)
        ep = int(g["enterpoint"])
        ids = set()
        if case != "its level-0 neighbours":
            ids.add(ep)
        if case != "enter point":
            ids |= set(g["level0"][ep, 1:1 + g["level0"][ep, 0]].tolist())
        deleted = delete(gpu, n, sorted(ids))
        for k, ef in ((10, 1), (10, 50)):
            run_knn(gpu, g, table, queries, k, ef, deleted, ctx=(case, k, ef))


def test_deleted_candidate_list_at_its_cap():
    """the device keeps at most 4096 deleted candidates per query: a query whose replay peaks just under the cap matches it exactly,
    one that peaks above it is refused"""
    metric, dim, n = rx.L2, 8, 40000
    rows = rows_for(metric, 41, n, dim)
    g = random_graph(41, n, 64, M=32, maxlevel=2)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 42, 8, dim)
    table = fp32_table(gpu, metric, rows, queries, envelope=False)
    deleted = delete(gpu, n, np.nonzero(np.random.default_rng(43).random(n) < 0.9)[0])
    under = over = None
    for ef in (96, 112, 120, 128, 136, 144):
        for q in range(len(queries)):
            rep = search_knn(g, lambda ids: table[q][ids], 10, ef, deleted)
            if 3800 <= rep.peak_deleted <= 4096 and not rep.tie and under is None:
                under = (q, ef, rep)
            if rep.peak_deleted > 4096 and over is None:
                over = (q, ef, rep)
    assert under is not None and over is not None
    q, ef, rep = under
    d, lab, cnt, st = gpu.hnsw_search_knn(queries[q:q + 1], 10, ef, with_stats=True)
    assert check_one(d[0], lab[0], cnt[0], st[0], table[q], rep, deleted, ctx=("under", ef, rep.peak_deleted))
    q, ef, rep = over
    with pytest.raises(rx.RxGpuError, match="too many deleted nodes"):
        gpu.hnsw_search_knn(queries[q:q + 1], 10, ef)


# ---------------------------------------------------------------------------------------------------------------- range


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("share", [0.0, 0.3])
def test_range_closure(metric, share):
    dim, n = 12, 2500
    rows = rows_for(metric, 51, n, dim)
    g = random_graph(51, n, 20, M=10, maxlevel=2, fill="mixed")
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 52, 6, dim)
    table = fp32_table(gpu, metric, rows, queries)
    deleted = delete(gpu, n, np.nonzero(np.random.default_rng(53).random(n) < share)[0]) if share else frozenset()
    for q in range(len(queries)):
        srt = np.unique(table[q])
        half = F((np.float64(srt[40]) + np.float64(srt[41])) / 2)
        assert srt[40] < half < srt[41]
        for radius in (-np.inf, 0.0, half, np.inf):
            for ef in (1, 32):
                rep = search_range(g, lambda ids: table[q][ids], radius, ef, deleted)
                total = len(rep.top)
                for max_out in sorted({0, 1, max(total - 1, 0), total}):
                    d, lab, got = gpu.hnsw_search_range(queries[q], radius, ef, max_out)
                    ctx = (q, radius, ef, max_out)
                    rows_q = rows_of(lab)
                    assert (d.view(np.uint32) == table[q, rows_q].view(np.uint32)).all(), ctx
                    assert not (set(rows_q.tolist()) & deleted), ctx
                    if rep.tie:
                        continue
                    assert got == total, (ctx, got, total)
                    want = rep.top[:max_out]
                    assert (rows_q == np.array([v for _, v in want], np.int64)).all(), ctx


# ---------------------------------------------------------------------------------------------------------------- streaming


def stream_session(gpu, query, ef):
    """rxgpu_hnsw_stream_begin / _next / _end with a batch size per call"""
    lib = gpu._lib
    q = np.ascontiguousarray(query, F)
    s = C.c_void_p()
    B._check(lib.rxgpu_hnsw_stream_begin(gpu._h, B._p(q, B._f32p), ef, C.byref(s)))

    def next_batch(batch):
        d = np.zeros(max(batch, 1), F)
        lab = np.zeros(max(batch, 1), np.uint64)
        cnt, ex = C.c_uint32(0), C.c_int(0)
        B._check(lib.rxgpu_hnsw_stream_next(s, batch, B._p(d, B._f32p), B._p(lab, B._u64p), C.byref(cnt), C.byref(ex)))
        return d[:cnt.value], lab[:cnt.value], bool(ex.value)

    return next_batch, lambda: lib.rxgpu_hnsw_stream_end(s)


def run_stream(gpu, g, table_q, query, ef, batches, deleted=frozenset(), max_calls=400, ctx=""):
    """both sessions call for batches[i % len(batches)] until exhausted; returns the replay (for its peak candidate count)"""
    rep = Stream(g, lambda ids: table_q[ids], ef, deleted)
    nxt, end = stream_session(gpu, query, ef)
    seen = set()
    try:
        for call in range(max_calls):
            b = batches[call % len(batches)]
            want, wex = rep.next(b)
            d, lab, ex = nxt(b)
            rows = rows_of(lab)
            assert (d.view(np.uint32) == table_q[rows].view(np.uint32)).all(), (ctx, call)
            assert not (set(rows.tolist()) & seen) and not (set(rows.tolist()) & deleted), (ctx, call, "row returned twice or deleted")
            seen |= set(rows.tolist())
            if rep.res.tie:
                return rep
            assert (rows == np.array([v for _, v in want], np.int64)).all(), (ctx, call, b, rows[:5], [v for _, v in want][:5])
            assert ex == wex, (ctx, call, ex, wex)
            if ex:
                return rep
        return rep
    finally:
        end()


@pytest.mark.parametrize("share", [0.0, 0.4])
def test_streaming(share):
    metric, dim, n = rx.L2, 10, 2500
    rows = rows_for(metric, 61, n, dim)
    g = random_graph(61, n, 64, M=16, maxlevel=2)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 62, 4, dim)
    table = fp32_table(gpu, metric, rows, queries)
    deleted = delete(gpu, n, np.nonzero(np.random.default_rng(63).random(n) < share)[0]) if share else frozenset()
    peak = 0
    ties = 0
    for i, (ef, batches) in enumerate([(0, [1]), (50, [31]), (50, [32]), (50, [33]), (100, [1024]), (64, [1, 300, 7, 1024]),
                                       (10, [300]), (1024, [64, 1024, 5])]):
        q = i % len(queries)
        rep = run_stream(gpu, g, table[q], queries[q], ef, batches, deleted, ctx=(share, ef, batches))
        peak = max(peak, rep.res.peak_candidates)
        ties += rep.res.tie
    assert peak > 1024, peak  # candidates spilled out of the shared list and came back
    assert ties <= 2, ties
    nxt, end = stream_session(gpu, queries[0], 0)
    try:
        with pytest.raises(rx.RxGpuError, match="batch size must be <= 1024"):
            nxt(1025)
    finally:
        end()


# ---------------------------------------------------------------------------------------------------------------- SQ8


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("dim", [1, 15, 16, 17, 100, 2048])
def test_sq8_hnsw(metric, dim):
    # quantised distances collide more often than fp32 ones; 600 rows keep equal pairs in the heaps rare even when ef covers the graph
    n = 600
    rows = rows_for(metric, 71 + dim, n, dim)
    g = random_graph(71 + dim, n, 64, M=16, maxlevel=3)
    gpu = make_index(metric, rows, g)
    params = params_for(metric, dim)
    gpu.sq8_attach(params)
    queries = rows_for(metric, 72 + dim, 16, dim)
    norms = np.linspace(0.6, 1.6, len(queries)).astype(F) if metric == rx.COS else None
    rcodes, rcorr = quantize(params, metric, rows)
    qc, qcorr, qcoef = query_codes(params, metric, queries, norms if norms is not None else np.ones(len(queries), F))
    # normalised rows: the fp32 sum of squares lies within 1e-5 of 1, so the device's row coefficient is exactly 1
    table = sq8_table(params, metric, qc, qcorr, qcoef, rcodes, rcorr)
    # SQ8 distances carry the coarse integer part, so equal distances meet in the heaps far more often than with fp32 rows; every
    # query is held to (a) and (c), the tie-free ones to (b), and some queries of every shape must be tie-free
    clean = 0
    for k, ef in ((10, 1), (10, 1024)):
        d, lab, cnt, st = gpu.hnsw_search_knn_sq8(queries, k, ef, norms, with_stats=True)
        for q in range(len(queries)):
            rep = search_knn(g, lambda ids, q=q: table[q][ids], k, ef)
            clean += check_one(d[q], lab[q], cnt[q], st[q], table[q], rep, ctx=(dim, k, ef, q))
    assert clean >= (1 if dim == 1 and metric == rx.COS else 4), clean
