#!/usr/bin/env python
"""IVF training and list assignment on the device (rxgpu_ivf_train, rxgpu_ivf_assign).

  python bench_ivf_train.py [--shapes small,large] [--niter 10] [--cpu-baseline]

  * small = 1M x 256 Cosine at nlist 1 024 and 16 384; large = 10M x 768 inner product at nlist 131 072 (the training set only:
    39 x nlist = 5.1M rows of the synthetic generator, 15.7 GB on the host);
  * each trains on the full 39 x nlist training set (IvfIndex trains when a namespace passes 39 x centroids rows) with --niter Lloyd
    iterations, then assigns every row (the fill: small shape only, all 1M rows; large: the training rows);
  * reported: the whole rxgpu_ivf_train call (host clock, it ends synchronised), per iteration the assignment kernel (CUDA events
    inside the call) as FLOP / time against the H100 SXM data sheet's 67 TFLOP/s FP32, with FLOP = 2 x points x nlist x dim, and the
    update's device work (sort, sums, splits, renormalisation; CUDA events) and its host work (keys back, objective, histogram, split
    choices); the fill's whole call.
  * --cpu-baseline: the reference's FAISS k-means (tests/ivf_train_oracle.py) at the smallest shape.  That build's sgemm is a
    triple-loop stub, so its time says nothing about FAISS with a real BLAS, which is not measured here.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.dont_write_bytecode = True  # the tree may be read-only

from bench_range import card  # noqa: E402

import reindexer_b200 as rx  # noqa: E402
from oracle import oracle as O  # noqa: E402

SHAPES = {"small": [(1_000_000, 256, rx.COS, 1024), (1_000_000, 256, rx.COS, 16384)], "large": [(10_000_000, 768, rx.IP, 131072)]}
FP32_PEAK = 67e12


def run(n, dim, metric, nlist, niter):
    ntrain = 39 * nlist
    rows = min(n, ntrain)
    x = np.empty((rows, dim), np.float32)
    for r0 in range(0, rows, 1 << 18):  # generated in slices: the large shape's training set alone is 15.7 GB
        r1 = min(rows, r0 + (1 << 18))
        x[r0:r1] = O.synth_matrix(0x7E1A + dim, r1 - r0, dim, r0)
    g = rx.GpuBruteforceSearch(metric, dim, 1)
    t0 = time.perf_counter()
    cent, st = g.ivf_train(nlist, x, niter=niter)
    train_s = time.perf_counter() - t0
    flop = 2.0 * ntrain * nlist * dim
    it = [{"assign_ms": s["assign_ms"], "assign_tflops": flop / (s["assign_ms"] * 1e-3) / 1e12, "assign_share_of_fp32_peak":
           flop / (s["assign_ms"] * 1e-3) / FP32_PEAK, "update_ms": s["update_ms"], "update_host_ms": s["host_ms"], "nsplit": s["nsplit"], "obj": s["obj"]} for s in st]
    fill = O.synth_matrix(0x7E1B + dim, n, dim) if n <= 1_000_000 else x
    g.ivf_assign(fill[:1024])  # warm-up
    t0 = time.perf_counter()
    g.ivf_assign(fill)
    fill_s = time.perf_counter() - t0
    g.close()
    return {"rows": n, "dim": dim, "metric": {rx.L2: "L2", rx.IP: "IP", rx.COS: "Cosine"}[metric], "nlist": nlist, "train_points": ntrain,
            "niter": niter, "train_s": train_s, "iterations": it, "fill_rows": len(fill), "fill_s": fill_s,
            "fill_tflops": 2.0 * len(fill) * nlist * dim / fill_s / 1e12}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="small")
    ap.add_argument("--niter", type=int, default=10)
    ap.add_argument("--cpu-baseline", action="store_true")
    a = ap.parse_args()
    if rx.device_count() < 1:
        raise SystemExit("bench_ivf_train.py needs a CUDA device")
    out = []
    for s in a.shapes.split(","):
        for shape in SHAPES[s]:
            out.append(run(*shape, a.niter))
    cpu = None
    if a.cpu_baseline:
        import ivf_train_oracle as TO
        n, dim, metric, nlist = SHAPES["small"][0]
        x = O.synth_matrix(0x7E1A + dim, 39 * nlist, dim)
        t0 = time.perf_counter()
        TO.train(2, x, nlist, niter=a.niter)
        cpu = {"train_s": time.perf_counter() - t0, "nlist": nlist, "note": "reference FAISS built with a triple-loop sgemm stub, not a real BLAS"}
    print(json.dumps({"workload": "IVF k-means training and list assignment on the device", "card": card(), "results": out,
                      "cpu_faiss_stub_sgemm": cpu}))


if __name__ == "__main__":
    main()
