#!/usr/bin/env python
"""Where the int8 filter launch spends its time at config 1 (10M x 768 fp32, inner product, k = 10, batch of 1024 queries).

  python bench_tc_phases.py [--rows N] [--queries 1024] [--runs 5] [--cluster 1|2|4] [--metric ip|l2|cosine] [--out FILE]

Runs the batch through the diagnostic instantiations of knn_tc_filter (knn_tc.cuh: kTcDiag*, selected with rxgpu_tc_diag; the
searches themselves never take them) and prints one JSON line with
  * phases      per consumer warpgroup, the share of its clock64 cycles in each phase of a 64-row block (wait on `full`, the rest of
                the K loop, the wgmma_wait<0> drain, the two bar.syncs, the block test (the loop that builds the hit mask), the append
                (the vote and the enqueues of the hits, their waits on a full candidate queue included), the wait for the
                warpgroup's turn to issue its MMAs),
                the cycles per block, the enqueues that found the queue full, and the producer's share of time waiting on `empty`;
  * hits        (query, row) pairs that passed the block test per 64-row block, against the walk position (the walker's i-th tile);
  * drift       how far apart the CTAs of one walker are: the spread of the walk positions they have reached at fixed times;
  * launches    the filter launch time (CUDA events, median of --runs) of the production kernel, of the stamped kernel, and of the three
                ablations: (a) the rare path compiled out (block test kept, hits only counted), (b) the producer not fetching
                (the consumers multiply zeroed stages; the barriers still cycle) and (c) the block test and the rare path compiled
                out (ring, MMAs, turns, drain and bar.syncs kept): the MMA path's own floor.
--cluster C runs every instantiation in clusters of C CTAs that share each row stage by TMA multicast (rxgpu_set_tensor_core_filter
3 / 4 / 5); the default is single CTAs.  --metric runs the same rows and queries as an L2 or a Cosine index instead.  Clock stamps are cycles of the SM clock; the card, its power limit and the SM clock samples of the timed runs are in the line.
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

from bench import DIM, K, ROWS_FULL, SEED, ClockSampler, bench_queries  # noqa: E402
from bench_range import card  # noqa: E402

# knn_tc.cuh: the diagnostic counters
SLOTS, WALK, MARK_EVERY = 64, 8192, 64
PHASES = ["full_wait", "k_loop", "drain", "bar1", "block_test", "append", "turn_wait", "bar2"]
TILE, BLOCKS, HITS, QWAIT, PER_WG = 8, 9, 10, 11, 12
CONSUMERS = 3  # consumer warpgroups, each followed by PER_WG counters; then the producer's
EMPTY, PROD = CONSUMERS * PER_WG, CONSUMERS * PER_WG + 1
MODES = {"production": 0, "stamped": 1, "no_rare_path": 2, "no_fetch": 3, "mma_only": 4}
METRICS = {"ip": ("IP", "inner product"), "l2": ("L2", "L2"), "cosine": ("COS", "cosine")}
MAX_CTAS = 1024


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_FULL)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--cluster", type=int, default=1, choices=[1, 2, 4], help="CTAs per cluster sharing every row stage")
    ap.add_argument("--metric", default="ip", choices=list(METRICS))
    ap.add_argument("--out", default=None, help="also write the JSON line (with the full hit histogram and marks) here")
    args = ap.parse_args(argv)

    os.environ["RXGPU_TC_DIAG"] = "1"  # rxgpu_tc_diag refuses the diagnostic instantiations without it
    import torch

    import reindexer_b200 as rx
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_tc_phases.py: no CUDA device -- librxgpu has no CPU fallback")
    lib = B.lib()
    idx = rx.GpuBruteforceSearch(getattr(rx, METRICS[args.metric][0]), DIM, args.rows)
    idx.append_synth(SEED, 0, args.rows)
    idx.set_tensor_core_filter({1: 3, 2: 4, 4: 5}[args.cluster])
    queries = bench_queries(args.queries)
    counters = torch.zeros(MAX_CTAS * SLOTS + WALK + MAX_CTAS * (WALK // MARK_EVERY), dtype=torch.int64, device="cuda:0")

    def run(mode):
        B._check(lib.rxgpu_tc_diag(mode, ctypes.c_void_p(counters.data_ptr()) if mode else None))
        counters.zero_()
        torch.cuda.synchronize()
        lib.rxgpu_set_profile(1)
        idx.search_knn(queries, K)
        st = rx.last_search_stats()
        lib.rxgpu_set_profile(0)
        B._check(lib.rxgpu_tc_diag(0, None))
        if st["tc_used"] != 1 or st["scan_launches"] != 1 or st["tc_kernel"] != 1 + mode or st["tc_cluster"] != args.cluster:
            raise SystemExit(f"bench_tc_phases.py: expected one filter launch, got {st}")
        return st["scan_kernel_ms"], st

    for mode in MODES.values():  # warm every instantiation
        run(mode)
    launches, clocks = {}, {}
    stamped = None
    for name, mode in MODES.items():
        sampler = ClockSampler(0)
        sampler.start()
        t0 = time.perf_counter()
        ms = []
        for _ in range(args.runs):
            t, st = run(mode)
            ms.append(t)
            if mode == MODES["stamped"]:
                stamped = counters.cpu().numpy().astype(np.uint64).astype(np.float64), st
            if mode == MODES["production"]:
                prod_stats = st
        clocks[name] = sampler.stop(t0, time.perf_counter())
        launches[name] = {"median_ms": float(np.median(ms)), "runs_ms": [round(x, 3) for x in ms]}
        print(json.dumps({name: launches[name], "clocks": clocks[name]}), file=sys.stderr, flush=True)

    c, st = stamped
    # the launch shape of index.cu's tcLaunch: G query groups (C query blocks each) x W walkers x C CTAs.  The G C CTAs of a walker
    # walk its 2 (its tiles) blocks each, so over the whole grid the blocks add up to 2 ntiles G C: the grid is the first multiple of
    # G C whose CTAs' block counters (per warp, four warps per warpgroup) reach that sum
    ntiles = (args.rows + 127) // 128
    C = args.cluster
    groups = ((args.queries + 127) // 128 + C - 1) // C
    per_cta = c[:MAX_CTAS * SLOTS].reshape(MAX_CTAS, SLOTS)[:, [wg * PER_WG + BLOCKS for wg in range(CONSUMERS)]].sum(axis=1) / 4
    grid = next(g for g in range(groups * C, MAX_CTAS + 1, groups * C) if per_cta[:g].sum() >= 2 * ntiles * groups * C)
    walkers = grid // (groups * C)
    cta = c[:grid * SLOTS].reshape(grid, SLOTS)
    phases = {}
    for wg in range(CONSUMERS):
        v = cta[:, wg * PER_WG:(wg + 1) * PER_WG].sum(axis=0)
        tile, blocks = v[TILE], v[BLOCKS]  # cycles and blocks summed over the warpgroup's four warps
        phases[f"warpgroup{wg}"] = {
            "share": {p: v[i] / tile for i, p in enumerate(PHASES)},
            "cycles_per_block": tile / blocks,
            "cycles_per_block_by_phase": {p: v[i] / blocks for i, p in enumerate(PHASES)},
            "blocks": blocks / 4, "hits": v[HITS], "hits_per_block": v[HITS] / (blocks / 4), "queue_full_waits": v[QWAIT],
        }
    phases["producer_empty_wait_share"] = cta[:, EMPTY].sum() / cta[:, PROD].sum()

    hist = c[grid * SLOTS:grid * SLOTS + WALK]
    walk_len = min(WALK, ntiles // walkers)  # positions every CTA reaches
    per_block = hist / (2 * grid)  # two 64-row blocks per tile, every CTA walks every position below its walk length
    edges = [0, 1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096, WALK]
    hits = [{"walk_from": a, "walk_to": b - 1, "hits_per_block": float(per_block[a:min(b, walk_len)].mean())} for a, b in zip(edges, edges[1:])
            if a < walk_len]

    marks = c[grid * SLOTS + WALK:grid * SLOTS + WALK + grid * (WALK // MARK_EVERY)].reshape(grid, WALK // MARK_EVERY)
    tiles_per_cta = ntiles / walkers
    spreads = []
    for w in range(walkers):
        m = marks[w * groups * C:(w + 1) * groups * C]  # CTA (walker * G + group) * C + rank in the cluster
        n = int(min(np.count_nonzero(row) for row in m))
        if n < 2:
            continue
        pos = np.arange(n) * MARK_EVERY
        for t in np.linspace(m[:, 0].max(), m[:, n - 1].min(), 16):
            reached = [np.interp(t, row[:n], pos) for row in m]
            spreads.append(max(reached) - min(reached))
    drift = {"walkers": walkers, "ctas_per_walker": groups * C, "tiles_per_cta": tiles_per_cta,
             "spread_tiles_median": float(np.median(spreads)) if spreads else None,
             "spread_tiles_p90": float(np.percentile(spreads, 90)) if spreads else None,
             "spread_tiles_max": float(np.max(spreads)) if spreads else None}

    sm_mhz = clocks["production"]["sm_mhz"]
    prod_ms = launches["production"]["median_ms"]
    ops = 2.0 * args.rows * DIM * args.queries
    line = {
        "workload": f"int8 filter launch, {args.rows} x {DIM}, {METRICS[args.metric][1]}, k = {K}, batch of {args.queries}",
        "card": card(), "cluster": C, "grid": grid,
        "launches": launches,
        "ablation_ceiling_no_rare_path_speedup": prod_ms / launches["no_rare_path"]["median_ms"],
        "ablation_floor_no_fetch_speedup": prod_ms / launches["no_fetch"]["median_ms"],
        "ablation_floor_mma_only_speedup": prod_ms / launches["mma_only"]["median_ms"],
        "int8_ops_per_clk_per_sm": (ops / (prod_ms * 1e-3) / (sm_mhz * 1e6) / grid) if sm_mhz else None,
        "candidates_per_batch": prod_stats["tc_candidates"], "fallbacks": prod_stats["tc_fallbacks"],
        "phases": phases, "hits_by_walk_position": hits, "drift": drift, "clocks": clocks,
    }
    print(json.dumps(line, default=float))
    if args.out:
        line["hits_histogram"] = hist[:walk_len].tolist()
        line["raw_counters"] = c[:grid * SLOTS].tolist()
        line["marks"] = marks.tolist()
        with open(args.out, "w") as f:
            json.dump(line, f, default=float)


if __name__ == "__main__":
    main()
