"""GPU tests of the int8 tensor-core filter's certified bound on rows built to stress the quantiser: a single huge coordinate over
tiny noise, integer rows, constant rows, row and query magnitudes from 1e-15 to 1e15 in one index, and all-zero rows and queries.
The filter only selects candidates; the answers must stay bit-identical to the exact scan for all three metrics (a query whose
candidate list overflows is answered by the exact scan, which keeps it identical too)."""
import numpy as np
import pytest
from helpers import prep_query

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def adversarial_rows(rng, n, dim):
    parts = []
    v = O.synth_matrix(0x1A7 + dim, n // 4, dim)
    parts.append(v * (10.0 ** rng.uniform(-15, 15, size=(len(v), 1))))  # every magnitude from 1e-15 to 1e15
    spike = rng.normal(0, 1e-6, size=(n // 8, dim))
    spike[np.arange(len(spike)), rng.integers(0, dim, size=len(spike))] = rng.choice([-1e3, 1e3], size=len(spike))
    parts.append(spike)  # one huge coordinate over tiny noise
    parts.append(rng.integers(-300, 301, size=(n // 8, dim)).astype(np.float64))  # integer rows
    parts.append(np.repeat(rng.uniform(-1, 1, size=(n // 64, 1)), dim, axis=1))  # constant rows: every code is +-127
    parts.append(np.zeros((n // 64, dim)))  # all-zero rows
    rest = n - sum(len(p) for p in parts)
    parts.append(O.synth_matrix(0x1A8 + dim, rest, dim))
    rows = np.concatenate(parts).astype(np.float32)
    return rows[rng.permutation(n)]


def adversarial_queries(rng, rows, nq, dim):
    q = O.synth_matrix(0x1A9 + dim, nq, dim).astype(np.float64)
    q[: nq // 4] *= 10.0 ** rng.uniform(-15, 15, size=(nq // 4, 1))
    near = rows[rng.integers(0, len(rows), size=nq // 4)].astype(np.float64)
    q[nq // 4: nq // 2] = near * (1 + rng.normal(0, 1e-3, size=near.shape))  # close to a row of any shape above
    q[nq // 2] = 0.0  # an all-zero query
    q[nq // 2 + 1] = 0.0
    q[nq // 2 + 1, 0] = 1e3  # a one-hot query
    return q.astype(np.float32)


@pytest.mark.parametrize("metric", [rx.L2, rx.IP, rx.COS])
@pytest.mark.parametrize("n,dim,nq,k", [(24000, 96, 160, 10), (12000, 300, 100, 5)])
def test_tc_int8_filter_is_exact_on_adversarial_rows(metric, n, dim, nq, k):
    rng = np.random.default_rng(dim * 7 + metric)
    rows = adversarial_rows(rng, n, dim)
    queries = adversarial_queries(rng, rows, nq, dim)
    if metric == rx.COS:
        queries = np.stack([prep_query(metric, q) if np.any(q) else q for q in queries])
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.add_points(O.row_labels(n), rows)
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    assert rx.last_search_stats()["tc_used"] == 0
    gpu.set_tensor_core_filter(1)
    d1, l1, c1 = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1, st
    # the filter itself must decide most queries: only the few whose rows all tie (the zero query) or crowd the bound's window may
    # overflow their candidate lists to the exact scan
    assert st["tc_fallbacks"] < nq // 4, st
    assert (c0 == c1).all()
    assert (l0 == l1).all(), np.argwhere(l0 != l1)[:5]
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all()
    gpu.close()
