#!/usr/bin/env python
"""Batched KNN at growing k on the config-1 index (10M x 768 fp32, inner product), through the int8 tensor-core filter.

  python bench_knn_k.py [--rows N] [--queries 1024] [--runs 10] [--ks 10,127,128,300,1000,1023]

The rows and the 1024 queries come from bench.py's generator, the rows produced directly in HBM.  k + 1 <= 128 runs on the filter's
bound list, larger k on staged exact thresholds (DESIGN 3.2).  For each k the script times rxgpu_search_knn through the C ABI with
output buffers allocated once (one warm-up call, then --runs timed calls; the call returns its results on the host, so each ends after
the device finished), then the exact scan (filter mode 2) on --exact-queries of the queries, and checks that those answers are
bit-identical.  `passes` counts the filter launches plus, on the staged path, the exact seed scan's passes over its prefix.  It
prints one JSON line with the card, its power limit and SM clocks.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only: importing bench.py leaves nothing behind

from bench import DIM, ROWS_FULL, SEED, ClockSampler, bench_queries  # noqa: E402
from bench_range import card  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_FULL)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--ks", default="10,127,128,300,1000,1023")
    ap.add_argument("--exact-queries", type=int, default=16)
    args = ap.parse_args(argv)
    if args.runs < 3:
        raise SystemExit("bench_knn_k.py: --runs must be at least 3")

    import reindexer_b200 as rx
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_knn_k.py: no CUDA device -- librxgpu has no CPU fallback")
    idx = rx.GpuBruteforceSearch(rx.IP, DIM, args.rows)
    idx.append_synth(SEED, 0, args.rows)
    queries = bench_queries(args.queries)
    sel = np.linspace(0, args.queries - 1, args.exact_queries).astype(int)
    sample = np.ascontiguousarray(queries[sel])

    records = []
    for k in (int(x) for x in args.ks.split(",")):
        # the C call with output buffers allocated once, as a C++ caller holds them
        D = np.zeros((args.queries, k), np.float32)
        L = np.zeros((args.queries, k), np.uint64)
        N = np.zeros(args.queries, np.uint32)
        ptrs = [B._p(queries, B._f32p), B._p(D, B._f32p), B._p(L, B._u64p), B._p(N, B._u32p)]

        def batch():
            B._check(B.lib().rxgpu_search_knn(idx._h, args.queries, ptrs[0], k, *ptrs[1:]))

        idx.set_tensor_core_filter(0)
        batch()  # warm-up
        sampler = ClockSampler(0)
        sampler.start()
        t_begin = time.perf_counter()
        times = []
        for _ in range(args.runs):
            t0 = time.perf_counter()
            batch()
            times.append(time.perf_counter() - t0)
        st = rx.last_search_stats()
        clocks = sampler.stop(t_begin, time.perf_counter())
        idx.set_tensor_core_filter(2)
        t0 = time.perf_counter()
        d0, l0, c0 = idx.search_knn(sample, k)
        exact_s = time.perf_counter() - t0
        idx.set_tensor_core_filter(0)
        identical = bool((c0 == N[sel]).all() and (l0 == L[sel]).all() and (d0.view(np.uint32) == D[sel].view(np.uint32)).all())
        best = min(times)
        records.append({
            "k": k, "qps": args.queries / best, "qps_median": args.queries / float(np.median(times)),
            "batch_s": [round(t, 5) for t in times], "spread": (max(times) - best) / best,
            "candidates_per_query": st["tc_candidates"] / args.queries, "passes": st["passes"],
            "tc_used": st["tc_used"], "tc_fallbacks": st["tc_fallbacks"],
            "exact_qps": len(sel) / exact_s, "identical": identical, "checked_queries": len(sel), "clocks": clocks,
        })
        print(json.dumps(records[-1]), file=sys.stderr, flush=True)
    print(json.dumps({
        "workload": f"KNN, {args.rows} x {DIM} fp32, inner product, batch of {args.queries} queries",
        "card": card(), "results": records,
    }))


if __name__ == "__main__":
    main()
