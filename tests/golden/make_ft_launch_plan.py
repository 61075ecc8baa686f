#!/usr/bin/env python
"""Generates tests/golden/ft_launch_plan.npz: what rxgpu_ft_last_stats reports after every call of the sequence that
tests/test_ft_launch_plan_gpu.py replays (kernel launches, preselect decision, postings scanned, algorithmic bytes), and the rows of
the selects that read their row total back first.  Needs a CUDA device; run it at the commit whose launch plan the test should pin:
    python tests/golden/make_ft_launch_plan.py [out.npz]"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_ft_launch_plan_gpu import run_plan  # noqa: E402

plan, rows = run_plan()
out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ft_launch_plan.npz")
pinned = {f"{name}/{k}": v for name, (ids, ranks, n) in rows.items() for k, v in (("ids", ids), ("ranks", ranks), ("n", np.int64(n)))}
np.savez_compressed(out, names=np.array([n for n, _ in plan]), stats=np.array([s for _, s in plan], np.int64), **pinned)
for name, stats in plan:
    print(f"{name:28s} {stats}")
print("wrote", out)
