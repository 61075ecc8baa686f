#!/usr/bin/env python
"""Sharded batched range search on the config-1 rows (10M x 768 fp32, inner product), against the same batch on one index.

  python bench_sharded_range.py [--shards 2] [--rows N] [--queries 1024] [--runs 10] [--max-out 4096]

The rows and the 1024 queries come from bench.py's generator, the rows produced directly in HBM.  Every query gets its own radius: its
10th-best map distance in one setting and its 100th-best in the other, both taken from one KNN batch with k = 100, as bench_range.py
takes them.  The whole index is built and timed first (rxgpu_search_range_batch) and its outputs kept; it is freed before the shards
are built, because one 80 GB card does not hold the whole index and the shards at once.  Shard r holds rows [base_r, base_r + n_r) of
the whole index with the same labels (append_synth), and the shards are in-process ranks (rxgpu_comm_create_local, one thread per rank)
over the visible GPUs, round-robin.  Each timed sharded call is one rxgpu_sharded_search_range_batch on every rank, started together;
its time is the slowest rank's.  Output buffers are allocated once, as a C++ caller holds them.  The whole batch output of every rank
is checked for bit-identity with the single index.  With every shard on one GPU the figure is the cost of the exchange and merge, not a
multi-GPU speed-up; the JSON line says which case it is, with the card, power limit and SM clocks of every GPU used.
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
sys.dont_write_bytecode = True  # the tree may be read-only: importing bench.py leaves nothing behind

from bench import DIM, ROWS_FULL, SEED, ClockSampler, bench_queries  # noqa: E402


def card(i):
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                                       "-i", str(i)], text=True).strip().split(", ")
        return {"index": i, "name": out[0], "power_limit_w": float(out[1]), "sm_max_mhz": float(out[2])}
    except (OSError, subprocess.CalledProcessError, ValueError, IndexError):
        return {"index": i, "name": None, "power_limit_w": None, "sm_max_mhz": None}


def timed(run_once, runs, gpus):
    """one warm-up, then `runs` timed calls; nvidia-smi samples every GPU used during the timed region"""
    run_once()
    samplers = [ClockSampler(g) for g in gpus]
    for s in samplers:
        s.start()
    t_begin = time.perf_counter()
    times = [run_once() for _ in range(runs)]
    t_end = time.perf_counter()
    return times, {str(g): s.stop(t_begin, t_end) for g, s in zip(gpus, samplers)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=2)
    ap.add_argument("--rows", type=int, default=ROWS_FULL)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--max-out", type=int, default=4096)
    args = ap.parse_args()
    if args.runs < 3:
        raise SystemExit("bench_sharded_range.py: --runs must be at least 3")

    import reindexer_b200 as rx
    from reindexer_b200 import binding as B

    ngpu = rx.device_count()
    if ngpu < 1:
        raise SystemExit("bench_sharded_range.py: no CUDA device -- librxgpu has no CPU fallback")
    R, nq, mo = args.shards, args.queries, args.max_out
    devices = [r % ngpu for r in range(R)]
    gpus = sorted(set(devices))
    lib = B.lib()
    queries = bench_queries(nq)
    settings = (10, 100)

    # ---- the whole index: radii, timing, and the outputs every rank must reproduce
    whole = rx.GpuBruteforceSearch(rx.IP, DIM, args.rows, device=0)
    whole.append_synth(SEED, 0, args.rows)
    kd, _, kc = whole.search_knn(queries, 100)
    assert (kc == 100).all()
    radii = {s: np.ascontiguousarray(kd[:, s - 1]) for s in settings}
    single = {}
    for s in settings:
        D, L, N = np.zeros((nq, mo), np.float32), np.zeros((nq, mo), np.uint64), np.zeros(nq, np.uint64)
        ptrs = [B._p(queries, B._f32p), B._p(radii[s], B._f32p), B._p(D, B._f32p), B._p(L, B._u64p), B._p(N, B._u64p)]

        def batch():
            t0 = time.perf_counter()
            B._check(lib.rxgpu_search_range_batch(whole._h, nq, ptrs[0], ptrs[1], mo, *ptrs[2:]))
            return time.perf_counter() - t0

        times, clocks = timed(batch, args.runs, [0])
        st = rx.last_search_stats()
        single[s] = {"out": (D, L, N), "times": times, "clocks": clocks, "tc_used": st["tc_used"], "tc_fallbacks": st["tc_fallbacks"]}
    whole.close()
    del whole

    # ---- the shards: in-process ranks, round-robin over the visible GPUs
    cuts = [args.rows * r // R for r in range(R + 1)]
    comms = B.ShardComm.local_group(R, devices)
    shards = []
    for r in range(R):
        sh = rx.GpuBruteforceSearch(rx.IP, DIM, cuts[r + 1] - cuts[r], device=devices[r])
        sh.append_synth(SEED, cuts[r], cuts[r + 1] - cuts[r])
        shards.append(sh)
    records = []
    for s in settings:
        outs = [(np.zeros((nq, mo), np.float32), np.zeros((nq, mo), np.uint64), np.zeros(nq, np.uint64)) for _ in range(R)]
        ptrs = [[B._p(D, B._f32p), B._p(L, B._u64p), B._p(N, B._u64p)] for D, L, N in outs]
        qp, rp = B._p(queries, B._f32p), B._p(radii[s], B._f32p)
        start = threading.Barrier(R)
        took, stats, errs = [0.0] * R, [None] * R, [None] * R

        def rank_call(r):
            try:
                start.wait()
                t0 = time.perf_counter()
                B._check(lib.rxgpu_sharded_search_range_batch(comms[r]._h, shards[r]._h, nq, qp, 0, rp, mo, *ptrs[r]))
                took[r] = time.perf_counter() - t0
                stats[r] = rx.last_search_stats()
            except Exception as e:  # noqa: BLE001 - reported by the main thread
                errs[r] = e

        def sharded():
            threads = [threading.Thread(target=rank_call, args=(r,), daemon=True) for r in range(R)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
            for e in errs:
                if e is not None:
                    raise e
            return max(took)

        times, clocks = timed(sharded, args.runs, gpus)
        D0, L0, N0 = single[s]["out"]
        valid = np.arange(mo)[None, :] < np.minimum(N0, mo)[:, None]
        identical = all(bool((N == N0).all() and (~valid | (L == L0)).all() and (~valid | (D.view(np.uint32) == D0.view(np.uint32))).all())
                        for D, L, N in outs)
        st_single = single[s]
        records.append({
            "radius": f"{s}th-best map distance per query",
            "single_qps": nq / float(np.median(st_single["times"])), "single_s": [round(t, 5) for t in st_single["times"]],
            "sharded_qps": nq / float(np.median(times)), "sharded_s": [round(t, 5) for t in times],
            "overhead_ms": (float(np.median(times)) - float(np.median(st_single["times"]))) * 1e3,
            "matches_per_query": float(N0.mean()), "max_matches_per_query": int(N0.max()),
            "identical": identical, "checked_queries": nq,
            "single_tc_used": st_single["tc_used"], "single_tc_fallbacks": st_single["tc_fallbacks"],
            "per_rank": [{"rank": r, "gpu": devices[r], "rows": cuts[r + 1] - cuts[r], "tc_used": stats[r]["tc_used"],
                          "tc_fallbacks": stats[r]["tc_fallbacks"], "tc_candidates": stats[r]["tc_candidates"]} for r in range(R)],
            "clocks_single": st_single["clocks"], "clocks_sharded": clocks,
        })
    for sh in shards:
        sh.close()
    for c in comms:
        c.close()
    case = ("all shards on one GPU: sharded_qps measures the exchange and merge overhead, not a multi-GPU speed-up" if len(gpus) == 1
            else f"shards spread over {len(gpus)} GPUs")
    print(json.dumps({
        "workload": f"sharded range search, {args.rows} x {DIM} fp32, inner product, {R} shards, batch of {nq} queries, max_out {mo}",
        "case": case, "gpus": [card(g) for g in gpus], "results": records,
    }))


if __name__ == "__main__":
    main()
