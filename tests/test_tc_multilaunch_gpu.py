"""A query batch with more query blocks than the GPU holds CTAs at once is split into several filter launches, each serving as many
blocks as are resident together; the answers must still be bit-identical to the exact scan."""
import numpy as np
import pytest

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", [1, 4])  # single CTAs, clusters of two (313 blocks: the last cluster is padded)
@pytest.mark.parametrize("metric", [rx.L2, rx.IP])
def test_tc_batch_larger_than_one_launch(metric, mode):
    n, dim, nq, k = 20000, 64, 40000, 10
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0xD1CE + metric, 0, n)
    queries = O.synth_matrix(0xD1CF + metric, nq, dim)
    gpu.set_tensor_core_filter(2)
    d0, l0, c0 = gpu.search_knn(queries, k)
    gpu.set_tensor_core_filter(mode)
    d1, l1, c1 = gpu.search_knn(queries, k)
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
    assert st["passes"] >= 2, st  # 128 queries per block: 313 blocks cannot be resident in one launch
    assert st["tc_cluster"] == (2 if mode == 4 else 1), st
    assert (c0 == c1).all() and (c1 == k).all()
    assert (l0 == l1).all(), np.argwhere(l0 != l1)[:5]
    assert (d0.view(np.uint32) == d1.view(np.uint32)).all()
    gpu.close()
