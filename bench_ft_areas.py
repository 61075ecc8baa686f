#!/usr/bin/env python
"""What highlight areas cost on the device: BASELINE configs[3] (ft_fast BM25, 50 M documents, 3-term OR with df 10% / 1% / 0.1%,
merge_limit 20000, built like bench_extra.ft_record) merged by rxgpu_ft_merge_query and by rxgpu_ft_merge_query_areas
(maxAreasInDoc = 5), alternating, five timed calls each; and the reference's Merger<..., MergeDataAreas<Area>> on one thread.  Checks
that the areas call returns the plain merge's bits and the reference's areas, and prints one JSON line.

  python bench_ft_areas.py [--docs 50000000] [--areas 5] [--reps 5]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card_state():
    """the card's name, power limit and SM clocks, read in the same run as the measurement"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # noqa: BLE001 -- the measurement stands without it, but says so
        return {"gpu": "unknown", "error": str(e)}


def problem(ndocs):
    from oracle import ft_oracle as F

    total = ndocs + 1
    rng = np.random.default_rng(7)
    words = (rng.poisson(100, size=total).astype(np.uint32) + 1).reshape(-1, 1)
    words[0] = 0
    p = F.FtProblem(total, words)
    npost = 0
    for df in (0.10, 0.01, 0.001):
        nd = int(df * ndocs)
        docs = np.unique(rng.integers(1, total, size=int(nd * 1.06), dtype=np.int64))[:nd].astype(np.uint32)
        npos = rng.integers(1, 4, size=len(docs)).astype(np.uint32)
        begin = np.concatenate([[0], np.cumsum(npos, dtype=np.int64)]).astype(np.uint32)
        first = (rng.random(len(docs)) * np.minimum(words[docs, 0], 60)).astype(np.uint32)
        pos = np.repeat(first, npos) + (np.arange(begin[-1], dtype=np.uint32) - np.repeat(begin[:-1], npos)) * 2
        p.add_term([(p.add_list_arrays(docs, begin, pos), 100.0)], op=F.OP_OR)
        npost += len(docs)
    return p, npost


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=50_000_000)
    ap.add_argument("--areas", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()

    import reindexer_b200 as rx
    from oracle import ft_areas_oracle as FA

    if rx.device_count() < 1:
        raise SystemExit("bench_ft_areas.py needs a CUDA device")
    p, npost = problem(args.docs)
    max_out = min(p.cfg["merge_limit"], npost) + 1
    ft = rx.GpuFtIndex(p.total_docs, p.words, p.avg)
    ids = [ft.add_postings(d, b, q) for d, b, q in p.lists]
    terms = [dict(t, postings=[ids[int(x)] for x in t["postings"]]) for t in p.terms]

    def plain():
        t0 = time.perf_counter()
        r = ft.merge(p.cfg, p.field_cfg, terms, max_out=max_out)
        return r, time.perf_counter() - t0, ft.last_stats()["device_ms"]

    def areas():
        t0 = time.perf_counter()
        r = ft.merge_areas(p.cfg, p.field_cfg, terms, max_areas_in_doc=args.areas, max_out=max_out)
        return r, time.perf_counter() - t0, ft.last_stats()["device_ms"]

    plain()  # warm-up: both paths allocate their scratch on the first call
    areas()
    t = {"plain": [], "areas": []}
    for _ in range(args.reps):  # alternating, so that both see the same state of the shared machine
        res_plain, wall, dev = plain()
        t["plain"].append((wall * 1e3, dev))
        res_areas, wall, dev = areas()
        t["areas"].append((wall * 1e3, dev))
    st = ft.last_stats()
    ft.close()
    infos, begin, got_areas, raw = res_areas

    def same_bits(a, b):
        return len(a) == len(b) and all((a[f] == b[f]).all() for f in ("id", "field", "normalized_proc")) and \
            (a["proc"].view(np.uint32) == b["proc"].view(np.uint32)).all()

    same_plain = bool(same_bits(infos, res_plain))
    ref_infos, ref_begin, ref_areas, ref_raw, ref_ns = FA.ref_merge_areas(p, args.areas, max_out=max_out)
    same_ref = bool(same_bits(ref_infos, infos) and (ref_begin == begin).all() and (ref_areas == got_areas).all() and (ref_raw == raw).all())
    med = {k: {"host_ms": float(np.median([w for w, _ in v])), "device_ms": float(np.median([d for _, d in v]))} for k, v in t.items()}
    print(json.dumps({
        "workload": f"ft_fast BM25 merge with highlight areas, {args.docs} docs, 3-term OR (df 10% / 1% / 0.1% = {npost} postings), "
                    f"merge_limit {p.cfg['merge_limit']}, maxAreasInDoc {args.areas} (BASELINE configs[3])",
        "card": card_state(),
        "reps": args.reps,
        "merge_query": {"median": med["plain"], "runs": t["plain"], "call": "rxgpu_ft_merge (the query path of rxgpu_ft_merge_query without synonyms)"},
        "merge_query_areas": {"median": med["areas"], "runs": t["areas"], "call": "rxgpu_ft_merge_query_areas"},
        "areas_overhead_device_ms": med["areas"]["device_ms"] - med["plain"]["device_ms"],
        "areas_overhead_host_ms": med["areas"]["host_ms"] - med["plain"]["host_ms"],
        "reference_cpu_ms": ref_ns / 1e6, "reference": "ft::Merger<IdRelVec, MergeDataAreas<Area>, uint32_t>::Merge, one thread",
        "merged_docs": int(len(infos)), "preselected": st["preselected"], "launches_areas": st["launches"],
        "areas_committed_total": int(begin[-1]), "areas_raw_total": int(raw.sum()),
        "identical_to_plain_merge": bool(same_plain),
        "identical_to_reference": bool(same_plain and same_ref)}))


if __name__ == "__main__":
    main()
