"""CPU pin of tests/index_model.py: IndexModel and the C port of the reference's brute-force map (oracle.PortBF) go through the same
seeded random sequences of upserts, removes, resizes, clones and synthetic appends on integer-valued rows, and after every step must
hold the same rows in the same internal order.  The order is read back twice: through get() for every label, and through KNN and
range results, which are exact on integer data and reveal the internal order through the heap's tie rule (a query at the origin
under IP puts every row at distance 0, so the result of k is the first k rows in internal order)."""
import numpy as np
import pytest
from index_model import COS, IP, L2, IndexModel, IvfModel, LogicError, NotFound

from oracle import oracle as O

MNAME = {L2: "l2", IP: "ip", COS: "cos"}


def ints(rng, n, dim):
    return rng.integers(-2, 3, size=(n, dim)).astype(np.float32)


def port_upsert(port, labels, vecs):
    """the port's sequential adds; returns whether a row reached the capacity"""
    return port.add_batch(np.asarray(labels, np.uint64), vecs) != 0


def assert_same(model, port, rng, ctx):
    assert model.size == port.size() and model.capacity == port.capacity(), ctx
    for lab in model.labels:
        got = port.get(lab)
        assert got is not None and (got.view(np.uint32) == model.get(lab).view(np.uint32)).all(), (ctx, lab)
    dim = model.dim
    queries = np.concatenate([np.zeros((1, dim), np.float32), ints(rng, 3, dim)])
    for q in queries:
        for k in sorted({1, 2, max(1, model.size // 2), model.size, model.size + 3}):
            dm, lm = model.knn(q, k)
            dp, lp = port.search_knn(q, k)
            assert (lm == lp).all() and (dm.view(np.uint32) == dp.view(np.uint32)).all(), (ctx, k, lm[:6], lp[:6])
        if model.metric == IP and not q.any():
            # every distance is 0: k = j returns the first j rows of the internal order
            for j in range(1, model.size + 1, max(1, model.size // 7)):
                assert set(port.search_knn(q, j)[1].tolist()) == set(model.labels[:j]), (ctx, j)
        radius = float(np.median(model.distances(q))) if model.size else 1.0
        dm, lm = model.range_search(q, radius)
        dp, lp = port.search_range(q, radius)
        assert (lm == lp).all() and (dm.view(np.uint32) == dp.view(np.uint32)).all(), (ctx, "range")


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("metric", [L2, IP, COS], ids=MNAME.get)
def test_model_follows_the_port(metric, seed):
    rng = np.random.default_rng(1000 * metric + seed)
    dim = int(rng.choice([1, 3, 8, 17]))
    cap = int(rng.integers(20, 60))
    model, port = IndexModel(metric, dim, cap), O.PortBF(metric, dim, cap)
    next_label = 1
    for step in range(60):
        op = rng.choice(["append", "rewrite", "mixed", "dup", "remove", "remove_last", "remove_unknown", "resize", "clone", "synth"])
        ctx = (seed, step, op)
        if op in ("append", "rewrite", "mixed", "dup"):
            n = int(rng.integers(1, 12))
            live = model.labels
            if op == "append" or not live:
                labels = list(range(next_label, next_label + n))
            elif op == "rewrite":
                labels = [int(x) for x in rng.choice(live, size=n)]
            else:
                labels = [int(x) if rng.random() < 0.5 else next_label + i for i, x in enumerate(rng.choice(live, size=n))]
                if op == "dup":
                    labels += labels[: max(1, n // 2)]
            next_label += n + 1
            vecs = ints(rng, len(labels), dim)
            full = port_upsert(port, labels, vecs)
            try:
                model.upsert(labels, vecs)
                assert not full, ctx
            except LogicError:
                assert full, ctx
        elif op == "remove" and model.size:
            lab = int(rng.choice(model.labels))
            model.remove(lab)
            port.remove(lab)
        elif op == "remove_last" and model.size:
            lab = model.labels[-1]
            model.remove(lab)
            port.remove(lab)
        elif op == "remove_unknown":
            model.remove(10**9 + step)
            port.remove(10**9 + step)
        elif op == "resize":
            cap = int(rng.integers(max(0, model.size - 3), model.size + 30))
            refused = port.resize(cap) != 0
            try:
                model.resize(cap)
                assert not refused, ctx
            except LogicError:
                assert refused and cap < model.size, ctx
        elif op == "clone":
            cap = int(rng.integers(0, model.capacity + 20))
            model, port = model.clone(cap), port.clone(cap)
        elif op == "synth":
            n = int(rng.integers(1, 6))
            first = int(rng.integers(0, 40))
            labels = [(first + r) << 32 for r in range(n)]
            try:
                model.append_synth(seed, first, n)
            except LogicError:
                assert model.size + n > model.capacity or any(lab in model.pos for lab in labels), ctx
                continue
            # the port appends the same synthetic rows through plain adds: equal bits under the same labels ...
            assert not port_upsert(port, labels, O.synth(seed, first * dim, n * dim).reshape(n, dim)), ctx
            for lab in labels:
                assert (port.get(lab).view(np.uint32) == model.get(lab).view(np.uint32)).all(), ctx
            # ... then both rewrite them onto the integer grid, where the KNN comparison below is exact
            vecs = ints(rng, n, dim)
            model.upsert(labels, vecs)
            assert not port_upsert(port, labels, vecs), ctx
        assert_same(model, port, rng, ctx)


def test_model_refusals():
    m = IndexModel(L2, 2, 3)
    with pytest.raises(LogicError):
        m.upsert([1, 2, 1, 3, 4, 5], np.arange(12, dtype=np.float32).reshape(6, 2))
    assert m.labels == [1, 2, 3] and (m.get(1) == [4, 5]).all()  # leading rows applied, the repeat of label 1 rewrote row 0
    with pytest.raises(LogicError):
        m.resize(2)
    m.remove(99)
    assert m.size == 3
    m.remove(3)  # the last row
    assert m.labels == [1, 2]
    m.resize(5)
    m.append_synth(7, 4, 2)
    assert m.labels[2:] == [4 << 32, 5 << 32] and (m.rows[2:] == O.synth_matrix(7, 2, 2, first_row=4)).all()
    with pytest.raises(LogicError):
        m.append_synth(7, 5, 1)  # label 5 << 32 is live: nothing applied
    assert m.size == 4
    c = m.clone(2)
    c.remove(1)
    assert m.labels[0] == 1 and c.capacity == 5 and c.labels[0] == 5 << 32


def test_ivf_model_swap_remove():
    m = IvfModel(3, 2)
    m.add([0, 0, 0, 1], [10, 11, 12, 13], np.arange(8, dtype=np.float32).reshape(4, 2))
    m.remove(10)
    assert [lab for lab, _ in m.lists[0]] == [12, 11]
    m.remove(11)  # the last entry of its list
    assert [lab for lab, _ in m.lists[0]] == [12]
    with pytest.raises(NotFound):
        m.remove(11)
    with pytest.raises(LogicError):
        m.add([2], [13], np.zeros((1, 2), np.float32))
    rows, labels, lists = m.flat()
    assert labels.tolist() == [12, 13] and lists.tolist() == [0, 1] and (rows[0] == [4, 5]).all()
