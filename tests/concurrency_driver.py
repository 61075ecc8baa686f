"""Child process of tests/test_concurrency_gpu.py: concurrent searches must return exactly what the same call returns alone.

include/rxgpu.h promises that searches are re-entrant and may run concurrently from many host threads (the reference runs selects
under a namespace *shared* lock).  Every scenario here first computes a serial baseline of each call on the handle it races on, checks
that baseline once against an independent reference (the fp64 envelope, the HNSW replay, the reference merger), then starts T threads
together on a barrier.  Each thread works through its own seeded, shuffled schedule of the calls, and every answer -- distance bits,
labels, counts, totals, the thread's own search statistics and error text -- must equal its baseline bit for bit.  ctypes releases the
GIL inside library calls, so the calls really overlap.

It runs in a fresh process so that process-wide first-use state (shared-memory ceilings, workspace pools, the int8 shadow, the streams
created by the first lease) is really used for the first time, and so that a stuck scenario is killed by the parent's timeout.  One line
per scenario: "<name> OK <detail>" or "<name> FAIL <reason>".

    python tests/concurrency_driver.py [scenario ...]      (default: all, in order a..h)"""
import ctypes as C
import os
import sys
import threading
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import reindexer_b200 as rx  # noqa: E402
from oracle import oracle as O  # noqa: E402
from reindexer_b200 import binding as B  # noqa: E402

T = 8  # racing threads
F = np.float32
STAT_KEYS = ("tc_used", "tc_fallbacks", "tie_replays", "tie_from_lists")


# ---------------------------------------------------------------------------------------------------------------- race machinery


def same(a, b, ctx):
    """bit equality of nested tuples / lists / dicts of numpy arrays and scalars"""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), ctx
        for key in a:
            same(a[key], b[key], (ctx, key))
    elif isinstance(a, (tuple, list)):
        assert len(a) == len(b), (ctx, len(a), len(b))
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, (ctx, i))
    elif isinstance(a, np.ndarray) and a.dtype.names:  # field by field: padding bytes are not part of the answer
        assert a.shape == b.shape and a.dtype == b.dtype, (ctx, a.shape, b.shape)
        for f in a.dtype.names:
            same(np.ascontiguousarray(a[f]), np.ascontiguousarray(b[f]), (ctx, f))
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and a.dtype == b.dtype, (ctx, a.shape, b.shape, a.dtype, b.dtype)
        assert a.tobytes() == b.tobytes(), (ctx, "differs", a.ravel()[:6], b.ravel()[:6])
    else:
        assert a == b, (ctx, a, b)


def stats():
    s = rx.last_search_stats()
    return {k: s[k] for k in STAT_KEYS}


def ft_stats(ft):
    s = ft.last_stats()
    s.pop("device_ms")  # a timing
    return s


def race(calls, rounds=3, seed=0, per_thread=None):
    """calls: {name: fn() -> result}.  Serial baselines first (unless given), then T threads on a barrier, each running every call
    `rounds` times in its own shuffled order (or per_thread[t]: the names thread t runs).  Returns the baselines."""
    base = {name: fn() for name, fn in calls.items()}
    race_against(calls, base, rounds, seed, per_thread)
    return base


def race_against(calls, base, rounds=3, seed=0, per_thread=None):
    barrier = threading.Barrier(T)
    errors = []

    def work(t):
        rng = np.random.default_rng(seed * 1000 + t)
        names = list(per_thread[t] if per_thread else calls) * rounds
        order = rng.permutation(len(names))
        try:
            barrier.wait()
            for i in order:
                got = calls[names[i]]()
                same(got, base[names[i]], (t, names[i]))
        except Exception:  # noqa: BLE001
            errors.append(f"thread {t}: {traceback.format_exc(limit=4)}")
            barrier.abort()

    threads = [threading.Thread(target=work, args=(t,)) for t in range(T)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors[0]


# ---------------------------------------------------------------------------------------------------------------- brute-force calls


def integer_rows(seed, n, dim):
    """small integers: many bit-equal distances, so ties straddle the k-th place"""
    return np.random.default_rng(seed).integers(-2, 3, size=(n, dim)).astype(F)


def queries_for(metric, rows, seed, nq):
    rng = np.random.default_rng(seed)
    q = rows[rng.integers(0, len(rows), nq)] + rng.integers(-1, 2, size=(nq, rows.shape[1])).astype(F)
    if metric == rx.COS:
        from test_fp64_envelope_gpu import unit

        q = unit(q)
    return np.ascontiguousarray(q, F)


def knn_call(gpu, q, k):
    def f():
        out = gpu.search_knn(q, k)
        return out, stats()

    return f


def range_call(gpu, q, radius, max_out):
    """rxgpu_search_range with a small max_out, then rxgpu_last_range_results for this thread's tail"""
    lib = gpu._lib

    def f():
        qq = np.ascontiguousarray(q, F)
        d = np.zeros(max(max_out, 1), F)
        lab = np.zeros(max(max_out, 1), np.uint64)
        n = C.c_uint64(0)
        B._check(lib.rxgpu_search_range(gpu._h, B._p(qq, B._f32p), radius, max_out, B._p(d, B._f32p), B._p(lab, B._u64p), C.byref(n)))
        total = n.value
        tail = max(total - max_out, 0)
        td = np.zeros(max(tail, 1), F)
        tl = np.zeros(max(tail, 1), np.uint64)
        B._check(lib.rxgpu_last_range_results(max_out, tail, B._p(td, B._f32p), B._p(tl, B._u64p)))
        m = min(total, max_out)
        return total, np.concatenate([d[:m], td[:tail]]), np.concatenate([lab[:m], tl[:tail]])

    return f


def range_batch_call(gpu, q, radii, max_out):
    def f():
        return gpu.search_range_batch(q, radii, max_out), stats()

    return f


def select_call(gpu, q, **kw):
    return lambda: gpu.select(q, **kw)


def device_calls(gpu, q, k, dstar, own_stream):
    """rxgpu_search_knn_device and rxgpu_search_tie_rows_device; own_stream: a torch stream per thread, else the NULL stream"""
    import torch

    local = threading.local()
    nq = len(q)

    def bufs():
        if not hasattr(local, "b"):
            dev = torch.device("cuda", 0)
            local.b = dict(q=torch.from_numpy(q).to(dev), d=torch.zeros((nq, k), dtype=torch.float32, device=dev),
                           i=torch.zeros((nq, k), dtype=torch.int32, device=dev), l=torch.zeros((nq, k), dtype=torch.int64, device=dev),
                           c=torch.zeros(nq, dtype=torch.int32, device=dev), s=torch.cuda.Stream(dev) if own_stream else None)
            torch.cuda.synchronize()
        return local.b

    def knn():
        b = bufs()
        st = b["s"].cuda_stream if b["s"] is not None else 0
        gpu.search_knn_device(nq, b["q"].data_ptr(), k, b["d"].data_ptr(), b["i"].data_ptr(), b["l"].data_ptr(), b["c"].data_ptr(), st)
        return b["d"].cpu().numpy(), b["i"].cpu().numpy(), b["l"].cpu().numpy(), b["c"].cpu().numpy(), stats()

    def tie():
        b = bufs()
        st = b["s"].cuda_stream if b["s"] is not None else 0
        gpu.search_tie_rows_device(b["q"].data_ptr(), float(dstar), k, b["d"].data_ptr(), b["i"].data_ptr(), b["l"].data_ptr(),
                                   b["c"].data_ptr(), st)
        c = int(b["c"][0])
        return c, b["d"][0, :c].cpu().numpy(), b["l"][0, :c].cpu().numpy()

    return knn, tie


def label_rows(lab):
    from test_fp64_envelope_gpu import label_rows as rows_of_labels

    return rows_of_labels(lab)


def check_knn_baseline(env, out, k, ctx, row_of=None):
    from test_fp64_envelope_gpu import check_knn, label_rows

    d, lab, cnt = out
    check_knn(env, d, lab, cnt, k, ctx=ctx, row_of=row_of or label_rows)


def brute_force_calls(gpu, metric, rows, seed, mode):
    """scenario a's call mix on one index; every baseline is checked against the fp64 envelope here"""
    from test_fp64_envelope_gpu import Envelope, check_range

    dim = rows.shape[1]
    qb = queries_for(metric, rows, seed, 96)
    env = Envelope(metric, rows, qb)
    calls = {}
    for k in (10, 300, 1500):
        calls[f"knn96_k{k}"] = knn_call(gpu, qb, k)
    calls["knn1"] = knn_call(gpu, qb[:1], 10)
    srt = np.sort(env.mid, 1)
    radii = np.float32(srt[:, 40])
    radii[0] = np.float32(srt[0, len(rows) // 2])  # half the rows match query 0: its candidate list overflows, the exact scan answers
    calls["range_batch"] = range_batch_call(gpu, qb, radii, 100)
    calls["range"] = range_call(gpu, qb[1], float(radii[1]), 7)
    calls["select"] = select_call(gpu, qb[2], k=25, need_sort=True, is_array=False)
    calls["select_array"] = select_call(gpu, qb[3], k=25, need_sort=False, is_array=True)
    base = {name: fn() for name, fn in calls.items()}
    for k in (10, 300, 1500):
        check_knn_baseline(env, base[f"knn96_k{k}"][0], k, ("knn", k))
        assert base[f"knn96_k{k}"][1]["tc_used"] == (k <= 1023), ("filter", k, base[f"knn96_k{k}"][1])
    check_knn_baseline(Envelope(metric, rows, qb[:1]), base["knn1"][0], 10, "knn1")
    (bd, bl, bn), bst = base["range_batch"]
    assert bst["tc_used"] == 1 and bst["tc_fallbacks"] >= 1, bst
    assert bn[0] > 4096, bn[0]  # more matches than the candidate list of max_out = 100 holds
    kept = np.minimum(bn, 100)
    sub = Envelope(metric, rows, qb[1:])
    check_range(sub, radii[1:], bd[1:], bl[1:], kept[1:], ctx="range batch")
    total, rd, rl = base["range"]
    assert total == bn[1] and rd[:kept[1]].tobytes() == bd[1, :kept[1]].tobytes(), ("range vs batch", total, bn[1])
    check_range(Envelope(metric, rows, qb[1:2]), radii[1:2], rd[None], rl[None], [total], ctx="range + tail")
    for name, qi in (("select", 2), ("select_array", 3)):  # FloatVectorIndex::Select: the rows of the same query's top 25
        ids, _ = base[name]
        _, lab25, _ = gpu.search_knn(qb[qi:qi + 1], 25)
        check_knn_baseline(Envelope(metric, rows, qb[qi:qi + 1]), gpu.search_knn(qb[qi:qi + 1], 25), 25, name)
        assert sorted(ids.tolist()) == sorted(label_rows(lab25[0]).tolist()), (name, ids[:5], label_rows(lab25[0])[:5])
    # device entry points: per-thread torch streams and the NULL stream
    dstar = base["knn96_k10"][0][0][4, 9]
    for own in (True, False):
        kn, tie = device_calls(gpu, qb[4:36] if own else qb[36:40], 10, dstar, own)
        calls[f"dev_knn_{own}"] = kn
        calls[f"dev_tie_{own}"] = tie
        base[f"dev_knn_{own}"] = kn()
        base[f"dev_tie_{own}"] = tie()
    for own, qs in ((True, qb[4:36]), (False, qb[36:40])):
        dd, di, dl, dc, _ = base[f"dev_knn_{own}"]
        check_knn_baseline(Envelope(metric, rows, qs), (dd, dl.view(np.uint64), dc), 10, ("device knn", own))
        # the first 10 rows in internal (= insertion) order with dist <= d*: every returned row's distance is in the envelope and not
        # above d*, and no row before the last one returned is missing although the envelope puts it surely at or below d*
        c, td, tl = base[f"dev_tie_{own}"]
        e1 = Envelope(metric, rows, qs[:1])
        got = label_rows(tl.view(np.uint64))
        assert 1 <= c <= 10 and (td <= dstar).all() and (np.diff(got) > 0).all(), (own, c, td, dstar)
        assert ((e1.lo[0, got] <= td) & (td <= e1.hi[0, got])).all(), (own, "tie distances outside the envelope")
        must = np.nonzero(e1.hi[0] <= dstar)[0]
        must = must[must < (got[-1] if c == 10 else len(rows))]
        assert set(must.tolist()) <= set(got.tolist()), (own, "tie rows missing", sorted(set(must.tolist()) - set(got.tolist()))[:5])
    return calls, base


# ---------------------------------------------------------------------------------------------------------------- scenarios


def scenario_b():
    """first use in a fresh process, then serial mutations with every thread racing on the first filter search of each round"""
    from test_fp64_envelope_gpu import Envelope

    metric, dim, n = rx.IP, 768, 40000  # a full conversion of the shadow takes long enough to overlap the other threads' filters
    rng = np.random.default_rng(0xB1)
    cap = n + 4096
    vecs = np.zeros((cap + 8192, dim), F)  # by label id
    vecs[:n] = integer_rows(0xB2, n, dim)
    live = set(range(n))
    gpu = rx.GpuBruteforceSearch(metric, dim, cap)
    gpu.add_points(O.row_labels(n), vecs[:n])
    qb = queries_for(metric, vecs[:n], 0xB3, 64)
    rounds = []

    def first_search_race(g, ctx):
        ids = np.array(sorted(live), np.int64)
        pos = np.full(len(vecs), -1, np.int64)
        pos[ids] = np.arange(len(ids))
        env = Envelope(metric, vecs[ids], qb)
        # the expected answer comes from the exact scan, which touches neither the shadow nor the filter's kernels
        g.set_tensor_core_filter(2)
        want = {k: g.search_knn(qb, k) for k in (10, 300)}
        for k in want:
            check_knn_baseline(env, want[k], k, (ctx, k), row_of=lambda lab: pos[(np.asarray(lab, np.uint64) >> np.uint64(32)).astype(np.int64)])
        g.set_tensor_core_filter(3)
        ks = [10 if t % 2 == 0 else 300 for t in range(T)]
        calls = {f"k{k}": (lambda k=k: (g.search_knn(qb, k), rx.last_search_stats()["tc_used"])) for k in (10, 300)}
        base = {f"k{k}": (want[k], 1) for k in (10, 300)}
        race_against(calls, base, rounds=1, per_thread=[[f"k{ks[t]}"] for t in range(T)])  # the first call of every thread races
        race_against(calls, base, rounds=2, seed=len(rounds))
        rounds.append(ctx)

    first_search_race(gpu, "fresh")
    next_id = n
    # upserts of live labels (rewrites) and new ones (appends), then swap-removes: a short shadow log
    for step in range(3):
        ids = rng.choice(sorted(live), 300, replace=False)
        vecs[ids] = integer_rows(0xB4 + step, len(ids), dim)
        gpu.add_points(O.row_labels(len(vecs))[ids], vecs[ids])
        new = np.arange(next_id, next_id + 200)
        vecs[new] = integer_rows(0xB8 + step, len(new), dim)
        gpu.add_points(O.row_labels(len(vecs))[new], vecs[new])
        live |= set(new.tolist())
        next_id += 200
        for i in rng.choice(sorted(live), 150, replace=False):
            gpu.remove_point(int(O.row_labels(len(vecs))[i]))
            live.discard(int(i))
        first_search_race(gpu, ("short log", step))
    # more than 4096 disjoint one-row rewrites: the log gives up and the shadow is rebuilt whole
    order = np.array(sorted(live), np.int64)[::2][:5000]
    vecs[order] = integer_rows(0xBC, len(order), dim)
    for i in order:
        gpu.add_point(vecs[i], int(O.row_labels(len(vecs))[i]))
    first_search_race(gpu, "log overflow")
    gpu.resize_index(cap + 8192)
    first_search_race(gpu, "resize")
    clone = gpu.clone(cap + 8192)
    first_search_race(clone, "clone")
    clone.close()
    gpu.close()
    return f"{len(rounds)} rounds"


def scenario_a():
    cases = []
    for i, (metric, dim) in enumerate([(m, d) for m in (rx.L2, rx.IP, rx.COS) for d in (96, 768)]):
        cases.append((metric, dim, 20000, 3 + i % 3))
    cases.append((rx.IP, 96, 100000, 0))  # automatic routing on 100 000 rows
    for ci, (metric, dim, n, mode) in enumerate(cases):
        rows = integer_rows(0xA0 + ci, n, dim)
        gpu = rx.GpuBruteforceSearch(metric, dim, n)
        gpu.add_points(O.row_labels(n), rows)
        gpu.set_tensor_core_filter(mode)
        calls, base = brute_force_calls(gpu, metric, rows, 0xA10 + ci, mode)
        race_against(calls, base, rounds=2, seed=ci)
        gpu.close()
    return f"{len(cases)} indexes"


def scenario_c():
    from test_fp64_envelope_gpu import Envelope

    metric, dim = rx.L2, 32
    out = []
    gpus = []
    for nlist, n in ((1000, 30000), (20000, 40000)):
        rng = np.random.default_rng(0xC0 + nlist)
        cents = (rng.standard_normal((nlist, dim)) * 0.5).astype(F)
        vecs = (rng.standard_normal((n + 4000, dim)) * 0.5).astype(F)
        lists = rng.integers(0, nlist, len(vecs)).astype(np.uint32)
        labels = O.row_labels(len(vecs))
        gpu = rx.GpuBruteforceSearch(metric, dim, 16)
        gpu.ivf_create(cents)
        gpu.ivf_add(lists[:n], labels[:n], vecs[:n])
        gpus.append(dict(gpu=gpu, nlist=nlist, vecs=vecs, lists=lists, labels=labels, live=set(range(n)), next=n, rng=rng))
    qs = [np.ascontiguousarray(g["vecs"][g["rng"].integers(0, 1000, 24)] + 0.05, F) for g in gpus]

    def calls_of(gi):
        g, q = gpus[gi], qs[gi]
        gpu = g["gpu"]
        ids = np.array(sorted(g["live"]), np.int64)
        pos = np.full(len(g["vecs"]), -1, np.int64)
        pos[ids] = np.arange(len(ids))

        def row_of(lab):
            return pos[(np.asarray(lab, np.uint64) >> np.uint64(32)).astype(np.int64)]

        env = Envelope(metric, g["vecs"][ids], q)
        full = gpu.ivf_search_knn_large_k(q, 10, g["nlist"])  # every list probed: the exact answer
        check_knn_baseline(env, full, 10, ("ivf full probe", g["nlist"]), row_of=row_of)
        radii = np.float32(np.sort(env.mid, 1)[:, 30])
        p = 16
        return {f"{gi}knn": lambda: gpu.ivf_search_knn(q, 10, p),
                f"{gi}knn256": lambda: gpu.ivf_search_knn(q[:4], 256, p),
                f"{gi}large_k": lambda: gpu.ivf_search_knn_large_k(q, 700, p),
                f"{gi}range": lambda: gpu.ivf_search_range(q[5], float(radii[5]), p, 12),
                f"{gi}range_batch": lambda: gpu.ivf_search_range_batch(q, radii, p, 20)}

    for rnd in range(3):
        calls = {}
        for gi in range(len(gpus)):
            calls.update(calls_of(gi))
        base = race(calls, rounds=2, seed=rnd)
        out.append(len(base))
        for g in gpus:  # serial add and remove round
            new = np.arange(g["next"], g["next"] + 1000)
            g["gpu"].ivf_add(g["lists"][new], g["labels"][new], g["vecs"][new])
            g["live"] |= set(new.tolist())
            g["next"] += 1000
            for i in g["rng"].choice(sorted(g["live"]), 500, replace=False):
                g["gpu"].ivf_remove(int(g["labels"][i]))
                g["live"].discard(int(i))
    for g in gpus:
        g["gpu"].close()
    return f"{len(out)} rounds, 2 indexes"


def scenario_d():
    from hnsw_replay import search_knn as replay_knn
    from hnsw_replay import search_range as replay_range
    from test_hnsw_exact_gpu import check_one, delete, fp32_table, make_index, random_graph, rows_for, rows_of, run_knn, run_stream
    from test_sq8_exact_gpu import params_for, query_codes, quantize, sq8_table

    metric, dim, n = rx.L2, 16, 4000
    rows = rows_for(metric, 0xD1, n, dim)
    g = random_graph(0xD1, n, 32, M=16, maxlevel=3)
    gpu = make_index(metric, rows, g)
    queries = rows_for(metric, 0xD2, 24, dim)
    table = fp32_table(gpu, metric, rows, queries)
    deleted = delete(gpu, n, np.nonzero(np.random.default_rng(0xD3).random(n) < 0.2)[0])
    params = params_for(metric, dim)
    gpu.sq8_attach(params)
    run_knn(gpu, g, table, queries, 10, 64, deleted, ctx="hnsw knn")
    radius = F(np.sort(table[0])[60])
    rep = replay_range(g, lambda ids: table[0][ids], radius, 32, deleted)
    d, lab, tot = gpu.hnsw_search_range(queries[0], float(radius), 32, 25)
    if not rep.tie:
        assert tot == len(rep.top) and (rows_of(lab) == np.array([v for _, v in rep.top[:25]])).all(), "hnsw range vs replay"
    rcodes, rcorr = quantize(params, metric, rows)
    qc, qcorr, qcoef = query_codes(params, metric, queries, np.ones(len(queries), F))
    stable = sq8_table(params, metric, qc, qcorr, qcoef, rcodes, rcorr)
    sd, sl, sc, sst = gpu.hnsw_search_knn_sq8(queries, 10, 64, with_stats=True)
    clean = sum(check_one(sd[q], sl[q], sc[q], sst[q], stable[q], replay_knn(g, lambda ids, q=q: stable[q][ids], 10, 64, deleted), deleted,
                          ("sq8 hnsw", q)) for q in range(len(queries)))
    assert clean >= 4, clean
    radii = np.array([np.sort(table[q])[50] for q in range(len(queries))], F)
    calls = {"knn": lambda: gpu.hnsw_search_knn(queries, 10, 64, with_stats=True),
             "knn_ef0": lambda: gpu.hnsw_search_knn(queries[:3], 5, 0),
             "range": lambda: gpu.hnsw_search_range(queries[0], float(radius), 32, 25),
             "range_batch": lambda: gpu.hnsw_search_range_batch(queries, radii, 32, 40),
             "sq8_hnsw": lambda: gpu.hnsw_search_knn_sq8(queries, 10, 64),
             "sq8_scan": lambda: gpu.sq8_search_knn(queries, 10)}
    hbase = race(calls, rounds=3, seed=0xD)
    # streaming sessions: each one's batches replayed alone, then T sessions advanced in turn by different threads
    from test_hnsw_exact_gpu import stream_session

    batches = [1, 31, 64, 7]
    nsess = 2 * T
    alone = []
    for s in range(nsess):
        nxt, end = stream_session(gpu, queries[s % len(queries)], 40 + s)
        seq = [nxt(batches[i % len(batches)]) for i in range(12)]
        end()
        alone.append(seq)
    run_stream(gpu, g, table[0], queries[0], 40, batches, deleted, ctx="stream replay")
    sessions = [stream_session(gpu, queries[s % len(queries)], 40 + s) for s in range(nsess)]
    locks = [threading.Lock() for _ in range(nsess)]
    progress = [0] * nsess
    errors = []
    barrier = threading.Barrier(T)

    def work(t):
        rng = np.random.default_rng(0xD5 + t)
        try:
            barrier.wait()
            for _ in range(nsess * 12):
                s = int(rng.integers(0, nsess))
                with locks[s]:  # a session is advanced by one thread at a time, by whichever thread holds it now
                    i = progress[s]
                    if i >= 12:
                        continue
                    got = sessions[s][0](batches[i % len(batches)])
                    progress[s] = i + 1
                same(got, alone[s][i], ("session", s, i))
                if t < 2:  # searches on the same maintenance stream, under the graph mutex, between the sessions' steps
                    name = ("knn", "range")[t]
                    same(calls[name](), hbase[name], ("search beside sessions", name))
        except Exception:  # noqa: BLE001
            errors.append(f"thread {t}: {traceback.format_exc(limit=4)}")

    threads = [threading.Thread(target=work, args=(t,)) for t in range(T)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    for nxt, end in sessions:
        end()
    assert not errors, errors[0]
    assert sum(progress) > nsess * 6, progress
    gpu.close()
    return f"{len(calls)} calls, {nsess} sessions"


def scenario_e():
    from ft_helpers import add_random_synonyms, assert_same_merge, random_problem
    from test_ft_sharded_gpu import upload

    from oracle import ft_oracle as Fo

    calls = {}
    fts = []
    for pi, seed in enumerate((0xE1, 0xE2)):
        prob = add_random_synonyms(random_problem(seed, total_docs=3000, nfields=2, nterms=3, density=0.3), seed, nsyn=1) \
            if Fo.ref_available() else random_problem(seed, total_docs=3000, nfields=2, nterms=3, density=0.3)
        ft, ids = upload(prob)
        fts.append(ft)
        terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]], synonym_ids=np.zeros(0, np.uint32)) for t in prob.terms]
        sterms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in prob.terms]
        syns = [[dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in syn] for syn in prob.synonyms] or None
        plain = ft.merge(prob.cfg, prob.field_cfg, terms, excluded=prob.excluded)
        assert_same_merge(Fo.best_merge(random_problem(seed, total_docs=3000, nfields=2, nterms=3, density=0.3))[0], plain, Fo.RANK_AND_ID,
                          ctx=("ft merge", seed))
        if syns:
            assert_same_merge(Fo.ref_merge(prob)[0], ft.merge(prob.cfg, prob.field_cfg, sterms, excluded=prob.excluded, synonyms=syns),
                              Fo.RANK_AND_ID, ctx=("ft merge with synonyms", seed))

        def merge(ft=ft, prob=prob, terms=terms):
            return ft.merge(prob.cfg, prob.field_cfg, terms, excluded=prob.excluded), ft_stats(ft)

        calls[f"{pi}merge"] = merge
        calls[f"{pi}merge_syn"] = lambda ft=ft, prob=prob, terms=sterms, syns=syns: (
            ft.merge(prob.cfg, prob.field_cfg, terms, excluded=prob.excluded, synonyms=syns), ft_stats(ft))
        calls[f"{pi}merge_areas"] = lambda ft=ft, prob=prob, terms=terms: (
            ft.merge_areas(prob.cfg, prob.field_cfg, terms, max_areas_in_doc=3), ft_stats(ft))
        calls[f"{pi}select"] = lambda ft=ft, prob=prob, terms=terms: (ft.select(prob.cfg, prob.field_cfg, terms, 200), ft_stats(ft))
        calls[f"{pi}select_syn"] = lambda ft=ft, prob=prob, terms=sterms, syns=syns: (
            ft.select(prob.cfg, prob.field_cfg, terms, 200, synonyms=syns), ft_stats(ft))
    race(calls, rounds=2, seed=0xE)
    for ft in fts:
        ft.close()
    return f"{len(calls)} calls on 2 indexes"


def scenario_f():
    metric, dim = rx.IP, 64
    rng = np.random.default_rng(0xF0)
    groups = []
    for gi in range(2):
        rows_per = 12000
        allv = rng.integers(-2, 3, size=(2 * rows_per, dim)).astype(F)
        labels = O.row_labels(2 * rows_per)
        shards = []
        for r in range(2):
            s = rx.GpuBruteforceSearch(metric, dim, rows_per)
            s.add_points(labels[r * rows_per:(r + 1) * rows_per], allv[r * rows_per:(r + 1) * rows_per])
            s.set_tensor_core_filter(1 if gi else 2)
            shards.append(s)
        whole = rx.GpuBruteforceSearch(metric, dim, 2 * rows_per)
        whole.add_points(labels, allv)
        whole.set_tensor_core_filter(2)
        q = np.ascontiguousarray(rng.integers(-2, 3, size=(48, dim)), F)
        groups.append(dict(comms=rx.ShardComm.local_group(2), shards=shards, whole=whole, q=q))
    plain = rx.GpuBruteforceSearch(rx.L2, 48, 20000)
    plain.add_points(O.row_labels(20000), integer_rows(0xF5, 20000, 48))
    plain.set_tensor_core_filter(3)
    pq = queries_for(rx.L2, integer_rows(0xF5, 20000, 48), 0xF6, 64)

    def group_call(gi):
        g = groups[gi]
        radius = -40.0

        def run():
            res, errs = [None, None], []

            def rank(r):
                try:
                    res[r] = (g["comms"][r].search_knn(g["shards"][r], g["q"], 10),
                              g["comms"][r].search_range_batch(g["shards"][r], g["q"], radius, 50))
                except Exception as e:  # noqa: BLE001
                    errs.append(e)

            ths = [threading.Thread(target=rank, args=(r,)) for r in range(2)]
            for th in ths:
                th.start()
            for th in ths:
                th.join()
            if errs:
                raise errs[0]
            return res

        return run

    calls = {"g0": group_call(0), "g1": group_call(1), "plain": lambda: plain.search_knn(pq, 10), "plain_range":
             lambda: plain.search_range_batch(pq, 30.0, 64)}
    base = {name: fn() for name, fn in calls.items()}
    for gi, g in enumerate(groups):
        want = g["whole"].search_knn(g["q"], 10)
        wr = g["whole"].search_range_batch(g["q"], -40.0, 50)
        for r in range(2):
            same(base[f"g{gi}"][r][0], want, ("sharded knn vs one index", gi, r))
            same(base[f"g{gi}"][r][1][2], wr[2], ("sharded range totals", gi, r))
    # a group's two ranks meet in a rendezvous, so each group is driven by one thread at a time; the other threads search plain indexes
    per_thread = [["g0"] if t == 0 else ["g1"] if t == 1 else ["plain", "plain_range"] for t in range(T)]
    race_against(calls, base, rounds=3, seed=0xF, per_thread=per_thread)
    for g in groups:
        for c in g["comms"]:
            c.close()
        for s in g["shards"]:
            s.close()
        g["whole"].close()
    plain.close()
    return "2 shard groups beside plain searches"


def scenario_g():
    """thread-local error text and retained range results"""
    metric, dim, n = rx.L2, 32, 20000
    rows = integer_rows(0x61, n, dim)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    gpu.set_tensor_core_filter(3)
    hn = rx.GpuBruteforceSearch(metric, dim, 3000)
    hn.add_points(O.row_labels(3000), rows[:3000])
    from test_hnsw_exact_gpu import random_graph

    hn.hnsw_import(random_graph(0x62, 3000, 16, M=8, maxlevel=2))
    from ft_helpers import random_problem
    from test_ft_sharded_gpu import upload

    prob = random_problem(0x63, total_docs=500, nfields=1, nterms=2)
    ft, ids = upload(prob)
    terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in prob.terms]
    q = queries_for(metric, rows, 0x64, 8)
    lib = gpu._lib
    import torch

    # real device buffers for the k = 0 call, so that nothing but its argument check can tell it apart from a valid one
    dq = torch.from_numpy(q[:1]).cuda()
    dd, dc = torch.zeros((1, 1), dtype=torch.float32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    di, dl = torch.zeros((1, 1), dtype=torch.int32, device="cuda"), torch.zeros((1, 1), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()

    def failing(name, fn):
        def f():
            try:
                fn()
            except rx.RxGpuError as e:
                return e.code, str(e), lib.rxgpu_last_error().decode()
            raise AssertionError(("the call did not fail", name))

        return f

    bad_calls = {"bad_k": lambda: hn.hnsw_search_knn(q, 0, 0),
                 "bad_dev_k": lambda: gpu.search_knn_device(1, dq.data_ptr(), 0, dd.data_ptr(), di.data_ptr(), dl.data_ptr(), dc.data_ptr()),
                 "bad_ef": lambda: hn.hnsw_search_knn(q, 5, 1025),
                 "bad_areas": lambda: ft.merge_areas(prob.cfg, prob.field_cfg, terms, max_areas_in_doc=0),
                 "bad_ivf": lambda: gpu.ivf_search_knn(q, 10, 4)}
    calls = {name: failing(name, fn) for name, fn in bad_calls.items()}
    for r in range(4):
        calls[f"range{r}"] = range_call(gpu, q[r], float(np.sort(((rows - q[r]) ** 2).sum(1))[200 + 50 * r]), 10 + r)
        calls[f"knn{r}"] = knn_call(gpu, q, 10 + 290 * r)
    base = {name: fn() for name, fn in calls.items()}
    texts = {base[nm][2] for nm in calls if nm.startswith("bad")}
    assert len(texts) >= 4, texts  # different messages: one that leaks into another thread is visible
    bad = [nm for nm in calls if nm.startswith("bad")]
    good = [nm for nm in calls if not nm.startswith("bad")]
    per_thread = [bad if t % 2 else good for t in range(T)]
    race_against(calls, base, rounds=40, seed=0x6, per_thread=per_thread)
    # mixed within a thread: a failure between a range search and its tail, and a range search between a failure and its text
    lib2 = lib

    def mixed():
        total, d, lab = calls["range1"]()
        code, msg, _ = calls["bad_ef"]()
        tail = max(total - 11, 0)
        td, tl = np.zeros(max(tail, 1), F), np.zeros(max(tail, 1), np.uint64)
        B._check(lib2.rxgpu_last_range_results(11, tail, B._p(td, B._f32p), B._p(tl, B._u64p)))
        return total, d, lab, td[:tail], tl[:tail], msg

    calls["mixed"] = mixed
    base["mixed"] = mixed()
    race_against(calls, base, rounds=20, seed=0x66, per_thread=[["mixed", "bad_k", "range2"]] * T)
    ft.close()
    hn.close()
    gpu.close()
    return f"{len(bad)} failing and {len(good)} succeeding calls"


def scenario_h():
    """indexes, full-text indexes and communicators created, searched and destroyed beside searches on an index that lives on"""
    metric, dim, n = rx.COS, 64, 20000
    rows = integer_rows(0x81, n, dim)
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    gpu.set_tensor_core_filter(4)
    q = queries_for(metric, rows, 0x82, 64)
    calls = {"knn": knn_call(gpu, q, 10), "knn300": knn_call(gpu, q, 300), "range_batch": range_batch_call(gpu, q, -0.6, 50)}
    base = {name: fn() for name, fn in calls.items()}
    from test_fp64_envelope_gpu import Envelope

    check_knn_baseline(Envelope(metric, rows, q), base["knn"][0], 10, "h knn")
    from ft_helpers import random_problem
    from test_ft_sharded_gpu import upload

    prob = random_problem(0x83, total_docs=800, nfields=1, nterms=2)

    def churn(t):
        def f():
            tmp = rx.GpuBruteforceSearch(rx.IP, 32, 6000)
            tmp.add_points(O.row_labels(6000), integer_rows(0x84 + t, 6000, 32))
            tmp.set_tensor_core_filter(1)
            a = tmp.search_knn(integer_rows(0x90 + t, 40, 32), 10)
            tmp.close()
            ft, ids = upload(prob)
            terms = [dict(tt, postings=[ids[int(x)] for x in tt["postings"]]) for tt in prob.terms]
            m = ft.merge(prob.cfg, prob.field_cfg, terms)
            ft.close()
            comms = rx.ShardComm.local_group(1)
            for c in comms:
                c.close()
            return a, m

        return f

    for t in range(T):
        calls[f"churn{t}"] = churn(t)
        base[f"churn{t}"] = calls[f"churn{t}"]()
    per_thread = [["knn", "knn300", "range_batch"] if t % 2 == 0 else [f"churn{t}", "knn"] for t in range(T)]
    race_against(calls, base, rounds=4, seed=0x8, per_thread=per_thread)
    gpu.close()
    return "searches beside create / destroy"


SCENARIOS = {"b": scenario_b, "a": scenario_a, "c": scenario_c, "d": scenario_d, "e": scenario_e, "f": scenario_f, "g": scenario_g,
             "h": scenario_h}


def main():
    # b goes first: its first filter batch is this process's first use of the filter, the pool and the shared-memory ceilings
    names = sys.argv[1:] or list(SCENARIOS)
    failed = 0
    for name in names:
        t0 = time.time()
        try:
            detail = SCENARIOS[name]()
            print(f"{name} OK {detail} ({time.time() - t0:.1f} s)", flush=True)
        except Exception:  # noqa: BLE001
            failed += 1
            print(f"{name} FAIL " + traceback.format_exc().replace("\n", " | "), flush=True)
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
