#!/usr/bin/env python
"""IVF KNN at large k (rxgpu_ivf_search_knn_large_k) on two shapes, at batch 1 and batch 256.

  python bench_ivf_large_k.py [--runs 10] [--large-rows 1000000] [--large-dim 256] [--no-cpu-baseline]

  * fixture: the reference's own KNN benchmark shape for IVF (100 000 x 32, nlist 1000, nprobe 16, K = 1000, L2);
  * large:   --large-rows x --large-dim Cosine, nlist 1024, nprobe 32, k = 100, 256, 257, 1000, 10000.  k = 256 and 257 are the two
             sides of the routing choice: k <= 256 (at nprobe <= 1024) runs the fused per-list top-k, larger k the key pass + radix select.
             The default 1M x 256 keeps the FAISS build (k-means over 262 144 sampled rows and the list assignment of every row, through
             the oracle's plain-loop sgemm: about 1e12 multiply-adds) to a minute on a many-core host; 2M x 768 costs about 4e12.

The index is trained and filled by the reference's FAISS (oracle/_ref, built by __graft_entry__.build()) and imported, as the tests do.
Each configuration is timed through the C ABI with output buffers allocated once: one warm-up call, then --runs calls, each ending
after the results are on the host; the median is reported.  Probed bytes = rows in the probed lists x dim x 4 (+ 4 per row for the
Cosine norm coefficients), from the lists' sizes and the nprobe nearest centroids; their rate is set against the H100 SXM's 3.35 TB/s.
Every timed answer is checked against FAISS on a 16-query sample.  The CPU arm runs FAISS' batched search on the same lists with
OpenMP threads from the CPU affinity.  Prints one JSON line with the card, its power limit and SM clocks.
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
os.environ.setdefault("OMP_NUM_THREADS", str(len(os.sched_getaffinity(0))))  # before the reference's FAISS (OpenMP) is loaded

from bench import ClockSampler  # noqa: E402
from bench_range import card  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def probed_rows(metric, centroids, list_sizes, queries, nprobe):
    c, q = centroids.astype(np.float64), queries.astype(np.float64)
    if metric == 0:
        d = (q * q).sum(1)[:, None] - 2 * q @ c.T + (c * c).sum(1)[None, :]
    else:
        d = -(q @ c.T) / (np.sqrt((c * c).sum(1))[None, :] if metric == 2 else 1.0)
    near = np.argsort(d, axis=1, kind="stable")[:, :nprobe]
    return list_sizes.astype(np.int64)[near].sum(1)


def check(ref, metric, queries, k, nprobe, d, l, c):
    for i, q in enumerate(queries):
        dr, lr = ref.search(q, k, nprobe)
        dr_map = dr if metric == 0 else -dr
        if c[i] != len(lr) or not np.allclose(d[i, :c[i]], dr_map, rtol=1e-4, atol=2e-6):
            return False
        if not (l[i, :c[i]] == lr).all():
            bad = np.nonzero(l[i, :c[i]] != lr)[0]
            if not (set(l[i, :c[i]]) == set(lr) or np.allclose(d[i, bad], dr_map[bad], rtol=1e-5)):
                return False
    return True


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--large-rows", type=int, default=1_000_000)
    ap.add_argument("--large-dim", type=int, default=256)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    args = ap.parse_args(argv)
    if args.runs < 3:
        raise SystemExit("bench_ivf_large_k.py: --runs must be at least 3")

    import reindexer_b200 as rx
    from oracle import oracle as O
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_ivf_large_k.py: no CUDA device -- librxgpu has no CPU fallback")
    if not O.ref_ivf_available():
        raise SystemExit("bench_ivf_large_k.py: needs oracle/_ref (the reference's FAISS, built by __graft_entry__.build())")

    shapes = [
        dict(name="fixture", metric=rx.L2, rows=100_000, dim=32, nlist=1000, nprobe=16, ks=[1000], seed=0x1F0000),
        dict(name="large", metric=rx.COS, rows=args.large_rows, dim=args.large_dim, nlist=1024, nprobe=32, ks=[100, 256, 257, 1000, 10000],
             seed=0x1F1000),
    ]
    records = []
    for sh in shapes:
        metric, dim, nprobe = sh["metric"], sh["dim"], sh["nprobe"]
        t0 = time.perf_counter()
        # N(0, 0.25) rows like oracle.synth_matrix, from numpy's generator (synth_matrix hashes element by element: minutes at 1e9 values)
        vecs = np.random.default_rng(sh["seed"]).standard_normal((sh["rows"], dim), dtype=np.float32) * np.float32(0.25)
        labels = O.row_labels(sh["rows"])
        ref = O.RefIvf(metric, dim, sh["nlist"])
        ref.train_add(labels, vecs)
        del vecs
        st = ref.export()
        idx = rx.GpuBruteforceSearch(metric, dim, sh["rows"])
        idx.add_points(st["labels"], st["vecs"])
        idx.ivf_import(st["centroids"], st["list_sizes"])
        del st["vecs"]
        build_s = time.perf_counter() - t0
        raw = np.random.default_rng(sh["seed"] + 1).standard_normal((256, dim), dtype=np.float32) * np.float32(0.25)
        queries = np.ascontiguousarray(np.stack([O.normalize_copy(q)[0] for q in raw]) if metric == rx.COS else raw, np.float32)
        rows = probed_rows(metric, st["centroids"], st["list_sizes"], queries, nprobe)
        per_row = dim * 4 + (4 if metric == rx.COS else 0)
        sample = np.linspace(0, 255, 16).astype(int)
        for batch in (1, 256):
            qs = np.ascontiguousarray(queries[:batch])
            probed_bytes = int(rows[:batch].sum()) * per_row
            for k in sh["ks"]:
                D = np.zeros((batch, k), np.float32)
                L = np.zeros((batch, k), np.uint64)
                N = np.zeros(batch, np.uint32)
                ptrs = [B._p(qs, B._f32p), B._p(D, B._f32p), B._p(L, B._u64p), B._p(N, B._u32p)]

                def call():
                    B._check(B.lib().rxgpu_ivf_search_knn_large_k(idx._h, batch, ptrs[0], k, nprobe, *ptrs[1:]))

                sampler = ClockSampler(0)
                sampler.start()
                call()  # warm-up
                t_begin = time.perf_counter()
                times = []
                for _ in range(args.runs):
                    t1 = time.perf_counter()
                    call()
                    times.append(time.perf_counter() - t1)
                stats = rx.last_search_stats()
                clocks = sampler.stop(t_begin, time.perf_counter())
                # the answers of the timed calls, checked against FAISS (batch 256: a 16-query sample; batch 1: its query)
                chk = sample if batch == 256 else np.array([0])
                ok = check(ref, metric, queries[chk], k, nprobe, D[chk], L[chk], N[chk])
                med = float(np.median(times))
                rec = {"shape": sh["name"], "batch": batch, "k": k, "nprobe": nprobe, "path": "fused" if k <= 256 else "select",
                       "median_s": med, "spread": (max(times) - min(times)) / med, "qps": batch / med,
                       "probed_rows_per_query": float(rows[:batch].mean()), "probed_bytes": probed_bytes,
                       "probed_bytes_per_s": probed_bytes / med, "share_of_3_35_TBps": probed_bytes / med / HBM_BPS,
                       "launches": stats["launches"], "faiss_agrees": bool(ok), "clocks": clocks}
                if not args.no_cpu_baseline:
                    ref.search_batch(qs, k, nprobe)  # warm-up
                    ct = []
                    for _ in range(3):
                        t1 = time.perf_counter()
                        ref.search_batch(qs, k, nprobe)
                        ct.append(time.perf_counter() - t1)
                    rec["cpu_faiss_median_s"] = float(np.median(ct))
                    rec["cpu_threads"] = int(os.environ["OMP_NUM_THREADS"])
                    rec["speedup_vs_cpu"] = rec["cpu_faiss_median_s"] / med
                records.append(rec)
                print(json.dumps(rec), file=sys.stderr, flush=True)
        idx.close()
        records.append({"shape": sh["name"], "rows": sh["rows"], "dim": dim, "metric": ["L2", "IP", "Cosine"][metric],
                        "nlist": sh["nlist"], "build_s": build_s})
    print(json.dumps({"workload": "IVF KNN at large k (rxgpu_ivf_search_knn_large_k)", "card": card(),
                      "all_agree_with_faiss": all(r.get("faiss_agrees", True) for r in records), "results": records}))


if __name__ == "__main__":
    main()
