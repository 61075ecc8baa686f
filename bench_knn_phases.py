#!/usr/bin/env python
"""Where one config-1 KNN step goes (10M x 768 fp32, inner product, k = 10, batch of 1024 queries), kernel by kernel.

  python bench_knn_phases.py [--rows N] [--queries 1024] [--steps 10] [--warmup 3] [--trace-dir DIR]

Runs bench.py's device-resident step (search_knn_device, queries and results in HBM) and prints one JSON line with
  * step_ms       the step time from CUDA events around --steps steps, with the profiler off;
  * kernels       device time per step of every kernel, memset and copy of the step, from one torch.profiler run of its own
                  (CUDA activities, --steps steps), grouped by kernel name (tc_prepare_queries, tc_seed_slices, tc_seed_merge,
                  knn_tc_filter, knn_rerank, knn_merge_lists, ...), with the launches per step;
  * candidates    candidates per query in the lists from the search statistics, and the exact-scan fallbacks;
  * gathered      rows per query knn_rerank gathered (the candidates under the query's final threshold), from the stamped run;
  * bookkeepers   the counters of one run of the stamped diagnostic instantiation (knn_tc.cuh: kTcDiagStamps, selected with
                  rxgpu_tc_diag): hits, rows rescored by the bookkeepers, bound-list inserts, the bookkeepers' cycles spent rescoring
                  against the consumer warpgroups' cycles, and the enqueues that found a candidate queue full.
The card, its power limit and the SM clock samples of the timed run are in the line.
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

from bench import DIM, K, ROWS_FULL, SEED, ClockSampler  # noqa: E402
from bench_range import card  # noqa: E402

# knn_tc.cuh: the diagnostic counters (per-CTA slots, per consumer warpgroup and bookkeeper)
SLOTS, WALK, MARK_EVERY = 32, 8192, 64
TILE, BLOCKS, HITS, QWAIT, PER_WG = 8, 9, 10, 11, 12
RESCORED, INSERTS, RESCORE_CYC = 2 * PER_WG + 4, 2 * PER_WG + 5, 2 * PER_WG + 6  # summed over the two bookkeeper warps
GATHERED = 41  # knn_tc.cuh: kTcDgGathered, in CTA 0's slots
MAX_CTAS = 1024
GROUPS = ["tc_prepare_queries", "tc_seed_slices", "tc_seed_merge", "tc_init_tau", "knn_tc_filter", "knn_rerank", "knn_merge_lists", "knn_select_topk", "knn_scan_warp"]


def group_of(name):
    for g in GROUPS:
        if g in name:
            return g
    low = name.lower()
    if "memset" in low:
        return "memset"
    if "memcpy" in low:
        return "memcpy " + ("DtoH" if "dtoh" in low else "HtoD" if "htod" in low else "DtoD" if "dtod" in low else "other")
    return name[:80]


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_FULL)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--trace-dir", default=None, help="also export the profiler's chrome trace here")
    args = ap.parse_args(argv)

    os.environ["RXGPU_TC_DIAG"] = "1"  # rxgpu_tc_diag refuses the diagnostic instantiations without it
    import torch
    from torch.profiler import ProfilerActivity, profile

    import reindexer_b200 as rx
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_knn_phases.py: no CUDA device -- librxgpu has no CPU fallback")
    lib = B.lib()
    nq, k1 = args.queries, K + 1
    idx = rx.GpuBruteforceSearch(rx.IP, DIM, args.rows)
    idx.append_synth(SEED, 0, args.rows)
    stream = torch.cuda.current_stream()
    dq = torch.empty((nq, DIM), dtype=torch.float32, device="cuda")
    B._check(lib.rxgpu_synth_fill_device(dq.data_ptr(), SEED + 1, 0, nq * DIM, 0, stream.cuda_stream))
    od = torch.zeros((nq, k1), dtype=torch.float32, device="cuda")
    oi = torch.zeros((nq, k1), dtype=torch.int32, device="cuda")
    ol = torch.zeros((nq, k1), dtype=torch.int64, device="cuda")
    oc = torch.zeros((nq,), dtype=torch.int32, device="cuda")

    def step():
        idx.search_knn_device(nq, dq.data_ptr(), k1, od.data_ptr(), oi.data_ptr(), ol.data_ptr(), oc.data_ptr(), stream.cuda_stream)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()

    # events only
    sampler = ClockSampler(0)
    sampler.start()
    t_begin = time.perf_counter()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        step()
    ev1.record(stream)
    torch.cuda.synchronize()
    clocks = sampler.stop(t_begin, time.perf_counter())
    step_ms = ev0.elapsed_time(ev1) / args.steps
    st = rx.last_search_stats()
    if st["tc_used"] != 1:
        raise SystemExit(f"bench_knn_phases.py: the filter did not answer: {st}")

    # profiler, a run of its own
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    if args.trace_dir:
        os.makedirs(args.trace_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(args.trace_dir, "knn_phases.pt.trace.json"))
    kernels = {}
    for ev in prof.key_averages():
        us = getattr(ev, "device_time_total", None)
        if us is None:
            us = getattr(ev, "cuda_time_total", 0.0)
        if not us:
            continue
        g = kernels.setdefault(group_of(ev.key), {"ms_per_step": 0.0, "launches_per_step": 0.0})
        g["ms_per_step"] += us / 1e3 / args.steps
        g["launches_per_step"] += ev.count / args.steps
    kernels = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["ms_per_step"]))
    device_sum = sum(v["ms_per_step"] for v in kernels.values())

    # one stamped diagnostic run: the bookkeepers' counters
    counters = torch.zeros(MAX_CTAS * SLOTS + WALK + MAX_CTAS * (WALK // MARK_EVERY), dtype=torch.int64, device="cuda:0")
    B._check(lib.rxgpu_tc_diag(1, ctypes.c_void_p(counters.data_ptr())))
    torch.cuda.synchronize()
    step()
    torch.cuda.synchronize()
    dst = rx.last_search_stats()
    B._check(lib.rxgpu_tc_diag(0, None))
    if dst["tc_kernel"] != 2:
        raise SystemExit(f"bench_knn_phases.py: expected the stamped instantiation, got {dst}")
    c = counters.cpu().numpy().astype(np.uint64).astype(np.float64)
    ntiles = (args.rows + 127) // 128
    groups = (nq + 127) // 128
    grid = groups * min(torch.cuda.get_device_properties(0).multi_processor_count // groups, ntiles)
    cta = c[:grid * SLOTS].reshape(grid, SLOTS)
    consumer_cycles = sum(cta[:, wg * PER_WG + TILE].sum() / 4 for wg in range(2))  # per warp, summed over both warpgroups
    book = {
        "hits": float(sum(cta[:, wg * PER_WG + HITS].sum() for wg in range(2))),
        "rescored_rows": float(cta[:, RESCORED].sum()),
        "bound_list_inserts": float(cta[:, INSERTS].sum()),
        "queue_full_waits": float(sum(cta[:, wg * PER_WG + QWAIT].sum() for wg in range(2))),
        # a bookkeeper warp's cycles spent rescoring over its consumer warpgroup's cycles walking the tiles
        "rescore_share_of_walk": float(cta[:, RESCORE_CYC].sum() / consumer_cycles) if consumer_cycles else None,
    }
    book["rescored_per_query"] = book["rescored_rows"] / nq
    book["inserts_per_query"] = book["bound_list_inserts"] / nq

    line = {
        "workload": f"KNN step (search_knn_device), {args.rows} x {DIM} fp32, inner product, k = {K}, batch of {nq}",
        "card": card(), "clocks": clocks,
        "step_ms": step_ms, "qps": nq / (step_ms * 1e-3),
        "device_ms_per_step_profiled": device_sum, "kernels": kernels,
        "candidates_per_query": st["tc_candidates"] / nq, "fallbacks": st["tc_fallbacks"],
        "gathered_per_query": float(c[GATHERED]) / nq,
        "bookkeepers": book,
    }
    print(json.dumps(line, default=float))


if __name__ == "__main__":
    main()
