#!/usr/bin/env python
"""HNSW graph construction on the device (rxgpu_hnsw_build) at BASELINE config 2's parameters: Cosine, dim 768, M = 16, efC = 200.

  python bench_hnsw_build.py [--n 1000000] [--full-n 10000000] [--no-ref] [--queries 1024]

  * data: bench_extra's low-rank vectors (latent 32, as bench_extra's HNSW workload; i.i.d. 768-d rows have no meaningful
    neighbours and no graph recalls them);
  * --n rows (at most 1M): the device build (host clock around the call, which ends synchronised, and the build's own
    CUDA-event phases and counts) against the reference's multithreaded inserter (oracle/_ref, AddPointConcurrent on every core) over
    the same rows; recall@10 against the exact scan of --queries queries at ef 64 / 128 / 256, both graphs searched by
    rxgpu_hnsw_search_knn;
  * --full-n rows (0: skipped): the device build alone, then the device search's QPS at ef 128 (k 10) on that graph;
  * --no-ref skips the reference's build (it takes far longer than the device's).
Prints one JSON line with the card and its power limit.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only

from bench_extra import lowrank  # noqa: E402
from bench_range import card  # noqa: E402

import reindexer_b200 as rx  # noqa: E402
from oracle import oracle as O  # noqa: E402

SEED, M, EFC, DIM = 0xB1D0, 16, 200, 768


def labels(n):
    return np.arange(n, dtype=np.uint64) << np.uint64(32)


CHUNK = 1_000_000


def rows_chunk(c, n):
    """rows [c * CHUNK, c * CHUNK + n): bench_extra's low-rank vectors (latent 32), one generator seed per million rows"""
    return lowrank(SEED + c, n, DIM)


def queries(nq):
    q = lowrank(SEED - 1, nq, DIM)
    return np.stack([O.normalize_copy(x, False)[0] for x in q])


def recall(found, truth):
    return float(np.mean([len(set(f.tolist()) & set(t.tolist())) / len(t) for f, t in zip(found, truth)]))


def device_build(n):
    g = rx.GpuBruteforceSearch(rx.COS, DIM, n)
    for c in range(0, (n + CHUNK - 1) // CHUNK):
        m = min(CHUNK, n - c * CHUNK)
        g.add_points(labels(n)[c * CHUNK:c * CHUNK + m], rows_chunk(c, m))
        print(f"rows uploaded: {c * CHUNK + m}", file=sys.stderr, flush=True)
    t0 = time.perf_counter()
    st = g.hnsw_build(M, EFC)
    return g, time.perf_counter() - t0, st


def compare(n, nq, with_ref):
    q = queries(nq)
    g, build_s, st = device_build(n)
    g.set_tensor_core_filter(2)
    _, truth, _ = g.search_knn(q, 10)
    out = {"rows": n, "device_build_s": build_s, "device_stats": st,
           "device_recall": {ef: recall(g.hnsw_search_knn(q, 10, ef)[1], truth) for ef in (64, 128, 256)}}
    if with_ref:
        assert n <= CHUNK
        rows = rows_chunk(0, n)
        ref = O.RefHnsw(O.COS, DIM, n, M=M, ef_construction=EFC, seed=100, multithread=True)
        build_s = 0.0
        for r0 in range(0, n, 50_000):  # in slices, with a line on stderr after each: the whole build takes minutes
            r1 = min(n, r0 + 50_000)
            t0 = time.perf_counter()
            ref.add_batch(labels(n)[r0:r1], rows[r0:r1], threads=os.cpu_count())
            build_s += time.perf_counter() - t0
            print(f"reference build: {r1} rows, {build_s:.1f} s", file=sys.stderr, flush=True)
        out["reference_build_s"] = build_s
        out["reference_threads"] = os.cpu_count()
        rg = rx.GpuBruteforceSearch(rx.COS, DIM, n)
        rg.add_points(labels(n), rows)
        rg.hnsw_import(ref.export(with_vectors=False))
        del ref, rows
        out["reference_recall"] = {ef: recall(rg.hnsw_search_knn(q, 10, ef)[1], truth) for ef in (64, 128, 256)}
        out["speedup_vs_reference"] = out["reference_build_s"] / out["device_build_s"]
        rg.close()
    g.close()
    return out


def full_shape(n, nq):
    g, build_s, st = device_build(n)
    print(f"device build: {n} rows, {build_s:.1f} s", file=sys.stderr, flush=True)
    q = queries(nq)
    g.hnsw_search_knn(q[:256], 10, 128)  # warm-up
    t0 = time.perf_counter()
    reps = 5
    for _ in range(reps):
        g.hnsw_search_knn(q, 10, 128)
    qps = reps * nq / (time.perf_counter() - t0)
    g.close()
    return {"rows": n, "device_build_s": build_s, "device_stats": st, "search_qps_ef128_k10": qps, "search_queries": nq}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--full-n", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    if rx.device_count() < 1:
        raise SystemExit("bench_hnsw_build.py needs a CUDA device")
    res = {"metric": "Cosine", "dim": DIM, "M": M, "efConstruction": EFC, "card": card(), "compare": compare(a.n, a.queries, not a.no_ref)}
    if a.full_n:
        res["full_shape"] = full_shape(a.full_n, 10_000)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
