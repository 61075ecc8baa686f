#!/usr/bin/env python
"""Batched range search on the config-1 index (10M x 768 fp32, inner product), through the int8 tensor-core filter.

  python bench_range.py [--rows N] [--queries 1024] [--runs 10] [--max-out 4096]

The rows and the 1024 queries come from bench.py's generator, the rows produced directly in HBM.  Every query gets its own radius:
its 10th-best map distance in one setting and its 100th-best in the other, both taken from one KNN batch with k = 100 (k1 = 101
fits the filter).  For each setting the script times the batched call (one warm-up, then --runs timed calls; the call returns its
results on the host, so each ends after the device finished), then the exact single-query path on --exact-queries of the queries,
and checks that those answers are bit-identical.  It prints one JSON line with the card, its power limit and SM clocks.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only: importing bench.py leaves nothing behind

from bench import DIM, ROWS_FULL, SEED, ClockSampler, bench_queries  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                                       "-i", "0"], text=True).strip().split(", ")
        return {"name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError):
        return {"name": None, "power_limit_w": None, "sm_max_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_FULL)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--max-out", type=int, default=4096, help="results kept per query; the filter's lists hold 2x as many candidates")
    ap.add_argument("--exact-queries", type=int, default=16)
    args = ap.parse_args()
    if args.runs < 3:
        raise SystemExit("bench_range.py: --runs must be at least 3")

    import reindexer_b200 as rx
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_range.py: no CUDA device -- librxgpu has no CPU fallback")
    idx = rx.GpuBruteforceSearch(rx.IP, DIM, args.rows)
    idx.append_synth(SEED, 0, args.rows)
    queries = bench_queries(args.queries)
    kd, _, kc = idx.search_knn(queries, 100)
    assert (kc == 100).all()
    knn_stats = rx.last_search_stats()

    records = []
    for rank in (10, 100):
        radii = np.ascontiguousarray(kd[:, rank - 1])
        # the C call with output buffers allocated once, as a C++ caller holds them: the binding's per-call allocation of
        # nq x max_out results would be timed otherwise
        D = np.zeros((args.queries, args.max_out), np.float32)
        L = np.zeros((args.queries, args.max_out), np.uint64)
        N = np.zeros(args.queries, np.uint64)
        ptrs = [B._p(a, t) for a, t in ((queries, B._f32p), (radii, B._f32p), (D, B._f32p), (L, B._u64p), (N, B._u64p))]

        def batch():
            B._check(B.lib().rxgpu_search_range_batch(idx._h, args.queries, ptrs[0], ptrs[1], args.max_out, *ptrs[2:]))

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
        sel = np.linspace(0, args.queries - 1, args.exact_queries).astype(int)
        identical = True
        t0 = time.perf_counter()
        singles = [idx.search_range(queries[q], float(radii[q]), args.max_out) for q in sel]
        exact_s = time.perf_counter() - t0
        for q, (d, l, n) in zip(sel, singles):
            m = min(n, args.max_out)
            identical &= bool(N[q] == n and (L[q, :m] == l).all() and (D[q, :m].view(np.uint32) == d.view(np.uint32)).all())
        best = min(times)
        records.append({
            "radius": f"{rank}th-best map distance per query",
            "batch_qps": args.queries / best, "batch_qps_median": args.queries / float(np.median(times)),
            "batch_s": [round(t, 5) for t in times],
            "spread": (max(times) - best) / best,
            "exact_qps": len(sel) / exact_s, "exact_ms_per_query": exact_s / len(sel) * 1e3,
            "matches_per_query": float(N.mean()), "candidates_per_query": st["tc_candidates"] / args.queries,
            "tc_used": st["tc_used"], "tc_fallbacks": st["tc_fallbacks"], "filter_launches": st["passes"],
            "identical": identical, "checked_queries": len(sel), "clocks": clocks,
        })
    print(json.dumps({
        "workload": f"range search, {args.rows} x {DIM} fp32, inner product, batch of {args.queries} queries, max_out {args.max_out}",
        "card": card(), "knn_k100_tc_used": knn_stats["tc_used"], "results": records,
    }))


if __name__ == "__main__":
    main()
