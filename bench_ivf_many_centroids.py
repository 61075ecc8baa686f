#!/usr/bin/env python
"""IVF search at large nlist (up to the reference's 131 072 centroids): the whole call and the coarse pass alone.

  python bench_ivf_many_centroids.py [--runs 5] [--shapes small,large] [--nlists 4096,16384,32768,65536,131072] [--no-cpu-baseline]

  * shapes: small = 1M x 256 Cosine, large = 10M x 768 inner product (30.7 GB of rows on the device);
  * nlist 4 096 ... 131 072, nprobe 32 and 256, batch 1, 256 and 1024;
  * per configuration: k = 10 (rxgpu_ivf_search_knn: the fused per-list top-k), k = 1000 (rxgpu_ivf_search_knn_large_k: key pass +
    radix select) and rxgpu_ivf_search_range_batch at each query's 100th-best probed distance.

The index: rows from the device generator (rxgpu_index_append_synth, the same values as oracle.synth_matrix), lists = contiguous
blocks of rows with multinomial sizes, each centroid a row sampled from its own block.  The answer is defined by the stored lists, and
the cost of a search by the list sizes it probes; a nearest-centroid assignment of 10M x 768 rows to 131 072 centroids would cost
2e15 FLOPs per nlist.  Timing through the C ABI with output buffers allocated once: one warm-up call, then --runs calls, each ending
after the results are on the host; the median is reported.  The coarse pass alone: a torch.profiler run of its own per (shape, nlist,
nprobe, batch) at k = 10, summing the kernels of the coarse pass (ivf_coarse_*, and the segmented sort between them), against its
floor: max(2 nq nlist dim / 67 TFLOP/s, centroid bytes / 3.35 TB/s) with centroid bytes = nlist x dim x 4 per query tile of 16 (one
tile at batch 1).  Probed bytes = rows in the probed lists x dim x 4 (+ 4 per row for the Cosine norm coefficients).

Correctness: every timed answer of the first 16 queries (query 0 at batch 1) is checked bit for bit against a device model: the
nprobe nearest centroids by an exact brute-force search over a centroid index (the same per-row arithmetic and tie rule as the coarse
pass), then an exact brute-force search over an index holding only the probed lists' rows, in row order.  The CPU arm runs FAISS
(tests/ivf_lists_oracle.py: the reference's FAISS over the same centroids and lists) on the 16 sample queries with OpenMP threads from the CPU affinity, on the
small shape only (the large one would need 61 GB of host memory for the rows and FAISS' copy).  Prints one JSON line with the card,
its power limit and SM clocks.
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
FP32_FLOPS = 67e12
COARSE_TILE = 16  # queries per tile of the coarse pass in a batch (kCoarseTile)
SHAPES = {
    "small": dict(metric=2, rows=1_000_000, dim=256, seed=0x1C0000),
    "large": dict(metric=1, rows=10_000_000, dim=768, seed=0x1C1000),
}


def coarse_kernel(name):
    return "ivf_coarse" in name or "DeviceSegmentedSort" in name


def time_calls(fn, runs):
    sampler = ClockSampler(0)
    sampler.start()
    fn()  # warm-up
    t_begin = time.perf_counter()
    times = []
    for _ in range(runs):
        t1 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t1)
    clocks = sampler.stop(t_begin, time.perf_counter())
    med = float(np.median(times))
    return med, (max(times) - min(times)) / med, clocks


def same_bits(d0, l0, n0, d1, l1, n1):
    return n0 == n1 and (l0[:n0] == l1[:n1]).all() and (d0[:n0].view(np.uint32) == d1[:n1].view(np.uint32)).all()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--shapes", default="small,large")
    ap.add_argument("--nlists", default="4096,16384,32768,65536,131072")
    ap.add_argument("--nprobes", default="32,256")
    ap.add_argument("--batches", default="1,256,1024")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args(argv)
    if args.runs < 3:
        raise SystemExit("bench_ivf_many_centroids.py: --runs must be at least 3")

    import reindexer_b200 as rx
    from oracle import oracle as O
    from reindexer_b200 import binding as B

    if rx.device_count() < 1:
        raise SystemExit("bench_ivf_many_centroids.py: no CUDA device -- librxgpu has no CPU fallback")
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import ivf_lists_oracle as LO

    cpu_arm = not args.no_cpu_baseline and LO.available()
    nlists = [int(x) for x in args.nlists.split(",")]
    nprobes = [int(x) for x in args.nprobes.split(",")]
    batches = [int(x) for x in args.batches.split(",")]
    nq_max = max(batches)
    lib = B.lib()
    records = []
    for shape in args.shapes.split(","):
        sh = SHAPES[shape]
        metric, n, dim, seed = sh["metric"], sh["rows"], sh["dim"], sh["seed"]
        per_row = dim * 4 + (4 if metric == rx.COS else 0)
        t0 = time.perf_counter()
        idx = rx.GpuBruteforceSearch(metric, dim, n)
        for r0 in range(0, n, 1 << 20):
            idx.append_synth(seed, r0, min(1 << 20, n - r0))
        raw = O.synth_matrix(seed + 1, nq_max, dim)
        queries = np.ascontiguousarray(np.stack([O.normalize_copy(q)[0] for q in raw]) if metric == rx.COS else raw, np.float32)
        host_rows = O.synth_matrix(seed, n, dim) if cpu_arm and shape == "small" else None
        build_s = time.perf_counter() - t0
        for nlist in nlists:
            rng = np.random.default_rng(seed + nlist)
            sizes = rng.multinomial(n, np.ones(nlist) / nlist).astype(np.int64)
            begin = np.concatenate([[0], np.cumsum(sizes)])
            pick = begin[:-1] + (rng.random(nlist) * np.maximum(sizes, 1)).astype(np.int64)
            pick = np.minimum(pick, n - 1)
            cents = np.stack([O.synth_matrix(seed, 1, dim, int(p))[0] for p in pick])
            idx.ivf_import(cents, sizes.astype(np.uint64))
            cidx = rx.GpuBruteforceSearch(metric, dim, nlist)  # the coarse model: same arithmetic and tie rule
            cidx.add_points(O.row_labels(nlist), cents)
            ref = None
            if host_rows is not None:
                list_nos = np.repeat(np.arange(nlist, dtype=np.int64), sizes)
                ref = LO.ListsIvf(metric, cents, list_nos, O.row_labels(n), host_rows)
            for nprobe in nprobes:
                sample = np.arange(min(16, nq_max))  # in every batch (query 0 alone at batch 1)
                # the device model of each sample query: its probed lists, then an exact search over those rows only
                model = {}
                probed = np.zeros(nq_max, np.int64)
                _, near, _ = cidx.search_knn(queries, nprobe)
                lists_of = (near >> np.uint64(32)).astype(np.int64)
                probed[:] = sizes[lists_of].sum(1)
                for qi in sample:
                    ls = np.sort(lists_of[qi])
                    m = rx.GpuBruteforceSearch(metric, dim, int(probed[qi]))
                    for l in ls:
                        if sizes[l]:
                            m.append_synth(seed, int(begin[l]), int(sizes[l]))
                    k10 = m.search_knn(queries[qi:qi + 1], 10)
                    k1000 = m.search_knn(queries[qi:qi + 1], 1000)
                    radius = float(k1000[0][0, min(int(k1000[2][0]), 100) - 1])
                    rd, rl, rn = m.search_range(queries[qi], radius)
                    best = np.lexsort((rl, rd))[:64]  # the range batch keeps the best 64 by (distance, label)
                    model[qi] = dict(k10=k10, k1000=k1000, radius=radius, range=(rd[best], rl[best], rn))
                    m.close()
                for batch in batches:
                    qs = np.ascontiguousarray(queries[:batch])
                    chk = sample[sample < batch]
                    probed_bytes = int(probed[:batch].sum()) * per_row
                    base = {"shape": shape, "metric": ["L2", "IP", "Cosine"][metric], "rows": n, "dim": dim, "nlist": nlist,
                            "nprobe": nprobe, "batch": batch, "probed_rows_per_query": float(probed[:batch].mean())}
                    tiles = 1 if batch == 1 else -(-batch // COARSE_TILE)
                    cflops = 2.0 * batch * nlist * dim
                    cbytes = float(tiles) * nlist * dim * 4
                    radii = np.zeros(batch, np.float32)
                    for mode, width in (("k10", 10), ("k1000", 1000), ("range", 64)):
                        D = np.zeros((batch, width), np.float32)
                        L = np.zeros((batch, width), np.uint64)
                        C32 = np.zeros(batch, np.uint32)
                        C64 = np.zeros(batch, np.uint64)
                        pq, pd, pl = B._p(qs, B._f32p), B._p(D, B._f32p), B._p(L, B._u64p)
                        if mode == "k10":
                            def call():
                                B._check(lib.rxgpu_ivf_search_knn(idx._h, batch, pq, 10, nprobe, pd, pl, B._p(C32, B._u32p)))
                        elif mode == "k1000":
                            def call():
                                B._check(lib.rxgpu_ivf_search_knn_large_k(idx._h, batch, pq, 1000, nprobe, pd, pl, B._p(C32, B._u32p)))
                        else:
                            # each query's 100th-best probed distance (its last one when it probes fewer rows); the model's for the sample
                            radii[:] = D_1000[np.arange(batch), np.clip(N_1000.astype(np.int64) - 1, 0, 99)]
                            for qi in chk:
                                radii[qi] = model[qi]["radius"]

                            def call():
                                B._check(lib.rxgpu_ivf_search_range_batch(idx._h, batch, pq, B._p(radii, B._f32p), nprobe, 64, pd, pl,
                                                                          B._p(C64, B._u64p)))
                        med, spread, clocks = time_calls(call, args.runs)
                        stats = rx.last_search_stats()
                        ok = True
                        for qi in chk:
                            if mode == "range":
                                rd, rl, rn = model[qi]["range"]
                                ok = ok and C64[qi] == rn and same_bits(D[qi], L[qi], min(int(rn), 64), rd, rl, len(rd))
                            else:
                                md, ml, mc = model[qi][mode]
                                ok = ok and same_bits(D[qi], L[qi], int(C32[qi]), md[0], ml[0], int(mc[0]))
                        if mode == "k1000":
                            D_1000, N_1000 = D.copy(), C32.copy()
                        rec = dict(base, mode=mode, path={"k10": "fused", "k1000": "select", "range": "range batch"}[mode],
                                   median_s=med, spread=spread, qps=batch / med, probed_bytes=probed_bytes,
                                   probed_bytes_per_s=probed_bytes / med, probed_share_of_3_35_TBps=probed_bytes / med / HBM_BPS,
                                   coarse_flops=cflops, coarse_centroid_bytes=cbytes, launches=stats["launches"],
                                   algorithmic_bytes=stats["algorithmic_bytes"], exact_on_sample=bool(ok), clocks=clocks)
                        if mode == "k10" and not args.no_profile:
                            rec.update(profile_coarse(call, cflops, cbytes))
                        if ref is not None and mode == "k1000" and batch == batches[-1]:
                            sq = np.ascontiguousarray(queries[chk])
                            ref.search_batch(sq, 1000, nprobe)  # warm-up
                            ct = []
                            for _ in range(3):
                                t1 = time.perf_counter()
                                ref.search_batch(sq, 1000, nprobe)
                                ct.append(time.perf_counter() - t1)
                            rec["cpu_faiss_s_per_query"] = float(np.median(ct)) / len(chk)
                            rec["cpu_threads"] = int(os.environ["OMP_NUM_THREADS"])
                            rec["speedup_vs_cpu_per_query"] = rec["cpu_faiss_s_per_query"] / (med / batch)
                        records.append(rec)
                        print(json.dumps(rec), file=sys.stderr, flush=True)
            cidx.close()
            del ref
        idx.close()
        records.append({"shape": shape, "rows": n, "dim": dim, "metric": ["L2", "IP", "Cosine"][metric], "build_s": build_s})
    print(json.dumps({"workload": "IVF search at large nlist (coarse pass over the whole GPU)", "card": card(),
                      "all_exact_on_sample": all(r.get("exact_on_sample", True) for r in records), "results": records}))


def profile_coarse(call, flops, nbytes, reps=3):
    """kernel time of the coarse pass per call, from a torch.profiler run of its own"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call()
            torch.cuda.synchronize()
    except RuntimeError as e:  # reported, not hidden: the record then has no coarse time
        return {"coarse_kernel_s": None, "profile_error": str(e)[:200]}
    coarse_us = total_us = 0.0
    names = set()
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total_us += t
        if coarse_kernel(ev.name):
            coarse_us += t
            names.add(ev.name.split("<")[0].split("(")[0][-40:])
    coarse_s = coarse_us * 1e-6 / reps
    floor_c, floor_b = flops / FP32_FLOPS, nbytes / HBM_BPS
    return {"coarse_kernel_s": coarse_s, "kernels_s": total_us * 1e-6 / reps,
            "coarse_bound": "fp32 FLOPs" if floor_c >= floor_b else "centroid bytes",
            "coarse_share_of_floor": (max(floor_c, floor_b) / coarse_s) if coarse_s > 0 else None,
            "coarse_kernels": sorted(names)}


if __name__ == "__main__":
    main()
