#!/usr/bin/env python
"""IVF range search over a batch (rxgpu_ivf_search_range_batch) against one rxgpu_ivf_search_range call per query.

  python bench_ivf_range.py [--runs 5] [--large-rows 1000000] [--large-dim 256]

  * fixture: the reference's own KNN benchmark shape for IVF (100 000 x 32 L2, nlist 1000, nprobe 16);
  * large:   --large-rows x --large-dim Cosine, nlist 1024, nprobe 32 (the two shapes of bench_ivf_large_k.py).
Batches of 256 and 1024 queries; each query's radius sits at its 10th, 100th or 1000th best probed distance (map space, from one
rxgpu_ivf_search_knn_large_k call at k = 1000), max_out = 1024, so every match of every query comes back.

The index is trained and filled by the reference's FAISS (oracle/_ref, built by __graft_entry__.build()) and imported, as the tests do.
Both arms run through the C ABI with output buffers allocated once: one warm-up, then --runs timed repetitions, each ending after the
results are on the host; the median is reported.  The batch arm is one call; the loop arm is one call per query.  Every query of every
timed batch is checked bit for bit against its single call.  Probed bytes = rows in the probed lists x dim x 4 (+ 4 per row for the
Cosine norm coefficients); their rate is set against the H100 SXM's 3.35 TB/s.  Prints one JSON line with the card, its power limit
and SM clocks.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only: importing the other bench scripts leaves nothing behind

from bench import ClockSampler  # noqa: E402
from bench_ivf_large_k import HBM_BPS, probed_rows  # noqa: E402
from bench_range import card  # noqa: E402

MAX_OUT = 1024


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--large-rows", type=int, default=1_000_000)
    ap.add_argument("--large-dim", type=int, default=256)
    args = ap.parse_args(argv)
    if args.runs < 3:
        raise SystemExit("bench_ivf_range.py: --runs must be at least 3")

    import reindexer_b200 as rx
    from oracle import oracle as O
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_ivf_range.py: no CUDA device -- librxgpu has no CPU fallback")
    if not O.ref_ivf_available():
        raise SystemExit("bench_ivf_range.py: needs oracle/_ref (the reference's FAISS, built by __graft_entry__.build())")

    shapes = [
        dict(name="fixture", metric=rx.L2, rows=100_000, dim=32, nlist=1000, nprobe=16, seed=0x1F0000),
        dict(name="large", metric=rx.COS, rows=args.large_rows, dim=args.large_dim, nlist=1024, nprobe=32, seed=0x1F1000),
    ]
    lib = B.lib()
    records = []
    for sh in shapes:
        metric, dim, nprobe = sh["metric"], sh["dim"], sh["nprobe"]
        t0 = time.perf_counter()
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
        raw = np.random.default_rng(sh["seed"] + 2).standard_normal((1024, dim), dtype=np.float32) * np.float32(0.25)
        queries = np.ascontiguousarray(np.stack([O.normalize_copy(q)[0] for q in raw]) if metric == rx.COS else raw, np.float32)
        rows = probed_rows(metric, st["centroids"], st["list_sizes"], queries, nprobe)
        per_row = dim * 4 + (4 if metric == rx.COS else 0)
        kd, _, kc = idx.ivf_search_knn_large_k(queries, 1000, nprobe)
        for batch in (256, 1024):
            qs = np.ascontiguousarray(queries[:batch])
            probed_bytes = int(rows[:batch].sum()) * per_row
            for rank in (10, 100, 1000):
                radii = np.ascontiguousarray([kd[q, min(rank, int(kc[q])) - 1] for q in range(batch)], np.float32)
                D = np.zeros((batch, MAX_OUT), np.float32)
                L = np.zeros((batch, MAX_OUT), np.uint64)
                N = np.zeros(batch, np.uint64)
                SD, SL, SN = np.zeros_like(D), np.zeros_like(L), np.zeros_like(N)
                bp = [B._p(qs, B._f32p), B._p(radii, B._f32p), nprobe, MAX_OUT, B._p(D, B._f32p), B._p(L, B._u64p), B._p(N, B._u64p)]
                sp = [(B._p(qs[q], B._f32p), float(radii[q]), nprobe, MAX_OUT, B._p(SD[q], B._f32p), B._p(SL[q], B._u64p),
                       B._p(SN[q:q + 1], B._u64p)) for q in range(batch)]

                def call_batch():
                    B._check(lib.rxgpu_ivf_search_range_batch(idx._h, batch, *bp))

                def call_loop():
                    for p in sp:
                        B._check(lib.rxgpu_ivf_search_range(idx._h, *p))

                sampler = ClockSampler(0)
                sampler.start()
                call_batch()  # warm-up
                call_loop()
                t_begin = time.perf_counter()
                tb, tl = [], []
                for _ in range(args.runs):  # the two arms alternate, so drift in the card's clocks hits both alike
                    t1 = time.perf_counter()
                    call_batch()
                    tb.append(time.perf_counter() - t1)
                    if _ == 0:
                        stats = rx.last_search_stats()
                    t1 = time.perf_counter()
                    call_loop()
                    tl.append(time.perf_counter() - t1)
                clocks = sampler.stop(t_begin, time.perf_counter())
                same = bool((N == SN).all())
                for q in range(batch):
                    m = int(min(N[q], MAX_OUT))
                    same = same and (L[q, :m] == SL[q, :m]).all() and (D[q, :m].view(np.uint32) == SD[q, :m].view(np.uint32)).all()
                mb, ml = float(np.median(tb)), float(np.median(tl))
                rec = {"shape": sh["name"], "batch": batch, "radius_at_rank": rank, "nprobe": nprobe, "mean_matches": float(N.mean()),
                       "batch_median_s": mb, "batch_spread": (max(tb) - min(tb)) / mb, "loop_median_s": ml,
                       "loop_spread": (max(tl) - min(tl)) / ml, "batch_speedup_vs_loop": ml / mb,
                       "probed_rows_per_query": float(rows[:batch].mean()), "probed_bytes": probed_bytes,
                       "batch_probed_bytes_per_s": probed_bytes / mb, "batch_share_of_3_35_TBps": probed_bytes / mb / HBM_BPS,
                       "loop_probed_bytes_per_s": probed_bytes / ml, "launches": stats["launches"], "identical_to_single_calls": bool(same),
                       "clocks": clocks}
                records.append(rec)
                print(json.dumps(rec), file=sys.stderr, flush=True)
        idx.close()
        records.append({"shape": sh["name"], "rows": sh["rows"], "dim": dim, "metric": ["L2", "IP", "Cosine"][metric],
                        "nlist": sh["nlist"], "build_s": build_s})
    print(json.dumps({"workload": "IVF range batch (rxgpu_ivf_search_range_batch) vs one rxgpu_ivf_search_range per query", "card": card(),
                      "all_identical_to_single_calls": all(r.get("identical_to_single_calls", True) for r in records),
                      "results": records}))


if __name__ == "__main__":
    main()
