#!/usr/bin/env python
"""Batched HNSW range search (rxgpu_hnsw_search_range_batch) against one rxgpu_hnsw_search_range call per query.

  python bench_hnsw_range.py [--rows 500000] [--queries 1024] [--runs 10] [--ef 128] [--max-out 1024]

The graph is BASELINE configs[2]'s shape at --rows rows, as `bench_extra.py hnsw` builds it: 768-dim low-rank vectors, Cosine,
M=16 efC=200, inserted by the reference's CPU code (oracle/_ref).  Every query gets its own radius: its 10th-best exact map distance
in one setting and its 100th-best in the other, both from one exact KNN batch with k = 100.  For each setting the script times the
batched call (one warm-up, then --runs timed calls with output buffers allocated once; the call returns its results on the host, so
each ends after the device finished), then one single call per query, and checks that every query of the batch is bit-identical to
its single call.  It prints one JSON line with the card, its power limit and SM clocks.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only: importing bench.py leaves nothing behind

from bench import ClockSampler  # noqa: E402
from bench_extra import lowrank  # noqa: E402
from bench_range import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--ef", type=int, default=128)
    ap.add_argument("--max-out", type=int, default=1024)
    args = ap.parse_args()
    if args.runs < 10:
        raise SystemExit("bench_hnsw_range.py: --runs must be at least 10")

    import reindexer_b200 as rx
    from oracle import oracle as O
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_hnsw_range.py: no CUDA device -- librxgpu has no CPU fallback")
    if not O.ref_knn_available():
        raise SystemExit("bench_hnsw_range.py: the graph is built by the reference's inserter (oracle/_ref); run build() first")
    n, dim, nq = args.rows, 768, args.queries
    threads = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    vecs, labels = lowrank(1, n, dim), O.row_labels(n)
    t0 = time.perf_counter()
    ref = O.RefHnsw(O.COS, dim, n, M=16, ef_construction=200, seed=100, multithread=True)
    ref.add_batch(labels, vecs, threads=threads)
    build_s = time.perf_counter() - t0
    g = ref.export(with_vectors=False)
    del ref
    idx = rx.GpuBruteforceSearch(rx.COS, dim, n)  # multithreaded insert: internal id != insertion order, so rows follow the graph
    idx.add_points(g["labels"], vecs[(g["labels"] >> np.uint64(32)).astype(np.int64)])
    idx.hnsw_import(g)
    queries = np.ascontiguousarray(np.stack([O.normalize_copy(q)[0] for q in lowrank(2, nq, dim)]))
    kd, _, kc = idx.search_knn(queries, 100)
    assert (kc == 100).all()

    D = np.zeros((nq, args.max_out), np.float32)
    L = np.zeros((nq, args.max_out), np.uint64)
    N = np.zeros(nq, np.uint64)
    records = []
    for rank in (10, 100):
        radii = np.ascontiguousarray(kd[:, rank - 1])
        ptrs = [B._p(a, t) for a, t in ((queries, B._f32p), (radii, B._f32p), (D, B._f32p), (L, B._u64p), (N, B._u64p))]

        def batch():
            B._check(B.lib().rxgpu_hnsw_search_range_batch(idx._h, nq, ptrs[0], ptrs[1], args.ef, args.max_out, *ptrs[2:]))

        sampler = ClockSampler(0)
        sampler.start()
        batch()  # warm-up
        t_begin = time.perf_counter()
        times = []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            batch()
            times.append(time.perf_counter() - t0)
        st = rx.last_search_stats()
        d1 = np.zeros(args.max_out, np.float32)
        l1 = np.zeros(args.max_out, np.uint64)
        n1 = ctypes.c_uint64(0)
        single = [B._p(d1, B._f32p), B._p(l1, B._u64p), ctypes.byref(n1)]
        identical = 0
        single_s = 0.0
        for q in range(nq):
            t0 = time.perf_counter()
            B._check(B.lib().rxgpu_hnsw_search_range(idx._h, B._p(queries[q], B._f32p), float(radii[q]), args.ef, args.max_out, *single))
            single_s += time.perf_counter() - t0
            m = min(n1.value, args.max_out)
            identical += int(N[q] == n1.value and (L[q, :m] == l1[:m]).all() and (D[q, :m].view(np.uint32) == d1[:m].view(np.uint32)).all())
        clocks = sampler.stop(t_begin, time.perf_counter())
        best = min(times)
        records.append({
            "radius": f"{rank}th-best exact map distance per query",
            "batch_qps": nq / best, "batch_qps_median": nq / float(np.median(times)), "batch_s": [round(t, 5) for t in times],
            "spread": (max(times) - best) / best,
            "single_qps": nq / single_s, "single_ms_per_query": single_s / nq * 1e3, "speedup_best": single_s / best,
            "matches_per_query": float(N.astype(np.float64).mean()), "max_matches": int(N.max()),
            "bfs_levels": st["passes"], "launches": st["launches"], "fallbacks": st["tc_fallbacks"],
            "identical": identical == nq, "identical_queries": identical, "clocks": clocks,
        })
    print(json.dumps({
        "workload": f"HNSW range search, {n} x {dim} fp32, cosine, M=16 efC=200 (graph by the reference's CPU inserter), ef={args.ef}, "
                    f"batch of {nq} queries, max_out {args.max_out}",
        "card": card(), "graph_build_s_reference_cpu": build_s, "build_threads": threads, "results": records,
    }))
    idx.close()


if __name__ == "__main__":
    main()
