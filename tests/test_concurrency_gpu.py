"""GPU tests of the threading promise of include/rxgpu.h: searches are re-entrant and may run concurrently from many host threads, and a
concurrent answer is bit-identical to the answer the same call gives alone (distance bits, labels, counts, totals, the thread's own
statistics and error text).  The scenarios run in one child process, tests/concurrency_driver.py, so that process-wide first-use state
is really first used there and a stuck scenario ends at a timeout instead of hanging the session:
  a  brute force: every search path on one index (exact scan, bound list, staged thresholds, exact rounds, range, range batch with an
     overflowing candidate list, select, device entry points on per-thread and NULL streams, tie rows), filter modes 3, 4 and 5 and
     automatic routing on 100 000 rows;
  b  the first filter batch of a fresh process raced by every thread, then after each serial round of upserts, swap-removes (a short
     shadow log, then more than 4096 ranges), a resize and a clone;
  c  IVF: fused KNN, large k, range and range batch on two mutable indexes (1 000 and 20 000 lists) between add / remove rounds;
  d  HNSW KNN, range, range batch and SQ8 on a graph with tombstones, and streaming sessions advanced in turn by different threads;
  e  full-text merge (plain, synonyms, areas) and select on two indexes, with each thread's rxgpu_ft_last_stats;
  f  two in-process shard groups beside plain searches;
  g  thread-local error text and retained range results, half the threads failing their argument checks;
  h  indexes, full-text indexes and communicators created and destroyed beside searches on an index that lives on."""
import os
import subprocess
import sys

import pytest

import reindexer_b200 as rx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCENARIOS = "bacdefgh"


@pytest.fixture(scope="module")
def driver_lines():
    if rx.device_count() < 1:
        pytest.skip("needs a CUDA device")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "concurrency_driver.py")], capture_output=True, text=True, timeout=1500)
    lines = {ln.split(" ", 1)[0]: ln for ln in r.stdout.splitlines() if ln[:1] in SCENARIOS and ln[1:2] == " "}
    return r, lines


@pytest.mark.parametrize("scenario", list(SCENARIOS))
def test_concurrent_answers_equal_serial_answers(driver_lines, scenario):
    r, lines = driver_lines
    assert scenario in lines, ("no line for scenario", scenario, r.returncode, r.stdout[-2000:], r.stderr[-3000:])
    assert lines[scenario].startswith(f"{scenario} OK"), lines[scenario].replace(" | ", "\n")
