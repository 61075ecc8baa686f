"""CPU pins of rxgpu_hnsw_build_plan: the drawn levels against the reference's own inserter, and the batch rules on hand-made levels."""
import numpy as np
import pytest

import reindexer_b200 as rx
from oracle import oracle as O

import hnsw_build_model as model


@pytest.mark.parametrize("M", [2, 16, 32])
def test_drawn_levels_are_the_reference_inserters(M):
    if not O.ref_knn_available():
        pytest.skip("the reference's HNSW is not built")
    n, dim = 100_000, 2
    rows = O.synth_matrix(0xB11D + M, n, dim)
    ref = O.RefHnsw(O.L2, dim, n, M=M, ef_construction=4, seed=100)
    ref.add_batch(O.row_labels(n), rows)
    want = ref.export(with_vectors=False)["levels"]
    levels, ends = rx.hnsw_build_plan(M, n, seed=100)
    assert (levels == want).all()
    assert ends[-1] == n and (np.diff(ends.astype(np.int64)) > 0).all()
    # the same draws continue a graph: rows [first, n) with the same seed repeat the first rows' levels
    lv2, _ = rx.hnsw_build_plan(M, n, first=1000, maxlevel=int(want[:1000].max()), seed=100)
    assert (lv2 == want[:n - 1000]).all()


def sizes(ends, first):
    return np.diff(np.concatenate([[first], ends.astype(np.int64)])).tolist()


def test_first_row_alone_then_the_cap():
    n = 5000
    lv = np.zeros(n, np.int32)
    _, ends = rx.hnsw_build_plan(16, n, levels=lv)
    s = sizes(ends, 0)
    assert s[0] == 1  # row 0 alone
    start = 1
    for size in s[1:]:  # a batch from graph size start holds max(1, start // 64) rows, the last one what is left
        assert size == min(max(1, start // 64), n - start), (start, size)
        start += size
    assert ends.tolist() == model.plan(16, 0, n, -1, lv)


def test_batch_cap_is_65536_rows():
    first, n = 10_000_000, 10_200_000
    lv = np.zeros(n - first, np.int32)
    _, ends = rx.hnsw_build_plan(16, n, first=first, maxlevel=3, levels=lv)
    s = sizes(ends, first)
    assert s[:3] == [65536, 65536, 65536] and sum(s) == n - first


def test_a_new_top_level_ends_its_batch():
    first, n = 6400, 6700  # batches of 100 rows
    lv = np.zeros(n - first, np.int32)
    lv[[10, 150, 151, 260]] = [3, 4, 2, 5]  # above the graph's top level 2, then above 3, not above 4, above 4
    _, ends = rx.hnsw_build_plan(16, n, first=first, maxlevel=2, levels=lv)
    e = ends.tolist()
    assert e[:2] == [first + 11, first + 111]  # the row of level 3 is the last of its batch; the next batch starts fresh
    assert first + 151 in e and first + 261 in e  # levels 4 and 5 end theirs, level 2 (below the running 4) does not
    assert first + 152 not in e
    assert e == model.plan(16, first, n, 2, lv)


def test_random_levels_match_the_model():
    rng = np.random.default_rng(5)
    for first, maxlevel in ((0, -1), (300, 1), (70_000, 4)):
        n = first + 20_000
        lv = np.minimum(rng.geometric(0.7, n - first) - 1, 9).astype(np.int32)
        _, ends = rx.hnsw_build_plan(8, n, first=first, maxlevel=maxlevel, levels=lv)
        assert ends.tolist() == model.plan(8, first, n, maxlevel, lv)


def test_plan_rejects_bad_arguments():
    for kw in (dict(M=1, n=10), dict(M=33, n=10), dict(M=16, n=10, levels=np.array([0, 1, -1] + [0] * 7, np.int32)),
               dict(M=16, n=10, first=5), dict(M=16, n=10, maxlevel=2)):
        with pytest.raises(rx.RxGpuError) as e:
            rx.hnsw_build_plan(**kw)
        assert e.value.code == 3, kw
