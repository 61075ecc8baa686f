#!/usr/bin/env python
"""Sharded IVF (rxgpu_sharded_ivf_train, rxgpu_sharded_ivf_search_knn, rxgpu_sharded_ivf_search_range_batch) against one index over the
same rows (rxgpu_ivf_train, rxgpu_ivf_search_knn_large_k, rxgpu_ivf_search_range_batch) in the same run.

  python bench_sharded_ivf.py [--shards 2] [--shapes default|large] [--runs 5]

Shapes: default = 1M x 256 Cosine at nlist 16 384; large = 10M x 768 inner product at nlist 131 072 (about 31 GB of host rows per copy).
The rows are seeded normals; shard r holds an uneven contiguous share of them, and the shards are in-process ranks
(rxgpu_comm_create_local, one thread per rank) over the visible GPUs, round-robin.  A sharded call's time is the slowest rank's.
Training: FAISS's defaults (10 iterations, 256 points per centroid), the whole call and the per-iteration assignment and update.
Search: 1024 queries at nprobe 32, KNN at k = 10 and k = 1000, and a range batch whose radius per query is its 100th-best distance.
Every centroid and every answer is checked for bit-identity with the single index.  With every shard on one GPU the figures are the
cost of the exchanges, not a multi-GPU speed-up; the JSON line says which case it is, with the card and power limit of every GPU used.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only

import reindexer_b200 as rx  # noqa: E402
from reindexer_b200 import binding as B  # noqa: E402

SHAPES = {"default": (1_000_000, 256, rx.COS, 16384), "large": (10_000_000, 768, rx.IP, 131072)}


def card(i):
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", str(i)],
                                      text=True).strip().split(", ")
        return {"index": i, "name": out[0], "power_limit_w": float(out[1])}
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError):
        return {"index": i, "name": None, "power_limit_w": None}


def collective(comms, call):
    """call(comm, r) on every rank from its own thread; returns (results by rank, the slowest rank's seconds)"""
    R = len(comms)
    out, err, secs = [None] * R, [None] * R, [0.0] * R
    go = threading.Barrier(R)

    def work(r):
        try:
            go.wait()
            t0 = time.perf_counter()
            out[r] = call(comms[r], r)
            secs[r] = time.perf_counter() - t0
        except Exception as e:  # noqa: BLE001 - re-raised below
            err[r] = e

    threads = [threading.Thread(target=work, args=(r,)) for r in range(R)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for e in err:
        if e is not None:
            raise e
    return out, max(secs)


def median_time(fn, runs):
    fn()  # warm-up
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=2)
    ap.add_argument("--shapes", choices=sorted(SHAPES), default="default")
    ap.add_argument("--runs", type=int, default=5)
    args = ap.parse_args()
    if rx.device_count() < 1:
        raise SystemExit("bench_sharded_ivf.py needs a CUDA device (librxgpu has no CPU fallback)")
    n, dim, metric, nlist = SHAPES[args.shapes]
    R, ngpu = args.shards, rx.device_count()
    devices = [r % ngpu for r in range(R)]
    rng = np.random.default_rng(7)
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x[: n // 4] += np.float32(0.5)
    labels = np.arange(n, dtype=np.uint64)
    queries = rng.standard_normal((1024, dim), dtype=np.float32)
    w = rng.uniform(0.6, 1.4, R)
    cuts = [0] + [int(c) for c in np.round(np.cumsum(w) / w.sum() * n)[:-1]] + [n]
    rec = {"bench": "sharded_ivf", "shape": args.shapes, "rows": n, "dim": dim, "metric": {rx.L2: "L2", rx.IP: "IP", rx.COS: "Cosine"}[metric],
           "nlist": nlist, "shards": R, "devices": devices, "cards": [card(i) for i in sorted(set(devices))],
           "case": "exchange overhead (every shard on one GPU)" if len(set(devices)) == 1 else "several GPUs", "bit_identical": True}

    # ---- one index
    one = rx.GpuBruteforceSearch(metric, dim, 1, device=0)
    t0 = time.perf_counter()
    c0, s0 = one.ivf_train(nlist, x)
    rec["train_ms_single"] = (time.perf_counter() - t0) * 1e3
    rec["assign_ms_per_iter_single"] = float(np.mean([s["assign_ms"] for s in s0]))
    rec["update_ms_per_iter_single"] = float(np.mean([s["update_ms"] + s["host_ms"] for s in s0]))
    one.ivf_add_assign(labels, x)

    # ---- the shards
    comms = B.ShardComm.local_group(R, devices)
    shards = [rx.GpuBruteforceSearch(metric, dim, 1, device=devices[r]) for r in range(R)]
    out, secs = collective(comms, lambda comm, r: comm.ivf_train(shards[r], nlist, x[cuts[r]:cuts[r + 1]]))
    rec["train_ms_sharded"] = secs * 1e3
    rec["assign_ms_per_iter_sharded"] = float(max(np.mean([s["assign_ms"] for s in st]) for _, st in out))
    rec["update_ms_per_iter_sharded"] = float(max(np.mean([s["update_ms"] + s["host_ms"] for s in st]) for _, st in out))
    for c, st in out:
        rec["bit_identical"] &= same_bits(c, c0) and [(s["obj"], s["nsplit"]) for s in st] == [(s["obj"], s["nsplit"]) for s in s0]
    for r in range(R):
        shards[r].ivf_add_assign(labels[cuts[r]:cuts[r + 1]], x[cuts[r]:cuts[r + 1]])

    # ---- search
    nprobe = 32
    d100, _, _ = one.ivf_search_knn_large_k(queries, 100, nprobe)
    radii = np.ascontiguousarray(d100[:, 99])
    for k in (10, 1000):
        want = one.ivf_search_knn_large_k(queries, k, nprobe)
        got, _ = collective(comms, lambda comm, r: comm.ivf_search_knn(shards[r], queries, k, nprobe))
        rec["bit_identical"] &= all(all(same_bits(a, b) for a, b in zip(g, want)) for g in got)
        rec[f"knn_k{k}_ms_single"] = median_time(lambda: one.ivf_search_knn_large_k(queries, k, nprobe), args.runs)
        rec[f"knn_k{k}_ms_sharded"] = median_time(
            lambda: collective(comms, lambda comm, r: comm.ivf_search_knn(shards[r], queries, k, nprobe)), args.runs)
    max_out = 1000
    want = one.ivf_search_range_batch(queries, radii, nprobe, max_out)
    got, _ = collective(comms, lambda comm, r: comm.ivf_search_range_batch(shards[r], queries, radii, nprobe, max_out))
    valid = np.arange(max_out)[None, :] < np.minimum(want[2], max_out)[:, None]
    for D, L, N in got:
        rec["bit_identical"] &= bool((N == want[2]).all() and (~valid | (L == want[1])).all()
                                     and (~valid | (D.view(np.uint32) == want[0].view(np.uint32))).all())
    rec["range_ms_single"] = median_time(lambda: one.ivf_search_range_batch(queries, radii, nprobe, max_out), args.runs)
    rec["range_ms_sharded"] = median_time(
        lambda: collective(comms, lambda comm, r: comm.ivf_search_range_batch(shards[r], queries, radii, nprobe, max_out)), args.runs)
    rec["range_matches_per_query"] = float(want[2].mean())
    for o in (one, *shards, *comms):
        o.close()
    print(json.dumps(rec))
    if not rec["bit_identical"]:
        raise SystemExit("sharded IVF answers differ from the single index")


if __name__ == "__main__":
    main()
