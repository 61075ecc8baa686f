"""CPU pin of the host halves of the KNN tie rule: rx.tie_replay (the closed form of the reference's heap, knn_select.h tieReplay) and
rx.merge_shards (the host k-way merge and its tie flag), against the reference's heap applied literally (bruteforce.cc:103-127): the
first k rows in internal order fill a max-heap on (dist, label), every later row replaces the top only when its distance is strictly
smaller, and the heap drains best first.

Every configuration is tiny (at most 40 rows) and checked at every k from 1 to n + 2, so all the places a tie run can straddle are
covered: the run before the strictly closer rows (evictions), after them, longer than k, one row too long, every row equal, and zero
distances of both signs, which compare equal (-0 == +0) but keep their own bits in the answer.  No device is involved."""
import heapq

import numpy as np
import pytest

import reindexer_b200 as rx

F = np.float32


def literal_heap(d, labels, k):
    """bruteforce.cc:103-127 on distances `d` (fp32, internal order) and `labels`: returns the row indices of the answer best first.
    Rows are looked at in internal order; a block's rows that are not below the heap's top when the block starts can never enter,
    because the top only decreases, so they are skipped without changing the outcome."""
    d = np.asarray(d, F)
    n = len(d)
    k = min(k, n)
    if k == 0:
        return np.zeros(0, np.int64)
    heap = [(-float(d[i]), -int(labels[i]), i) for i in range(k)]  # max-heap on (dist, label) with a float compare: -0 == +0
    heapq.heapify(heap)
    top = -heap[0][0]
    for start in range(k, n, 4096):
        for j in np.nonzero(d[start:start + 4096] < top)[0]:
            i = start + int(j)
            if float(d[i]) < top:
                heapq.heapreplace(heap, (-float(d[i]), -int(labels[i]), i))
                top = -heap[0][0]
    return np.array([i for _, _, i in sorted(heap, key=lambda t: (-t[0], -t[1]))], np.int64)


def replay_inputs(d, gidx, labels, k):
    """what the library hands tie_replay: d* = the k-th distance under (dist, internal row), `lower` = the rows strictly below it,
    `first` = the first min(k, #) rows in internal order with dist <= d* (float compares)"""
    order = sorted(range(len(d)), key=lambda i: (float(d[i]), int(gidx[i])))
    dstar = d[order[k - 1]]
    lower = [i for i in order[:k] if d[i] < dstar]
    first = [i for i in sorted(range(len(d)), key=lambda i: int(gidx[i])) if d[i] <= dstar][:k]
    return dstar, lower, first


def call_replay(k, dstar, d, gidx, labels, lower, first):
    pick = lambda ix: (d[ix], gidx[ix], labels[ix])  # noqa: E731
    return rx.tie_replay(k, dstar, pick(np.array(lower, np.int64)), pick(np.array(first, np.int64)))


def assert_same(want_idx, d, labels, got_d, got_l, ctx):
    assert len(got_l) == len(want_idx), (ctx, len(got_l), len(want_idx))
    assert (got_l == labels[want_idx]).all(), (ctx, got_l, labels[want_idx])
    assert (got_d.view(np.uint32) == d[want_idx].view(np.uint32)).all(), (ctx, got_d, d[want_idx])


VALUES = F([-2.0, -1.0, -0.0, 0.0, 0.5, 1.0, 3.0])


def random_config(rng, n, nvals):
    vals = rng.choice(VALUES, nvals, replace=False)
    d = rng.choice(vals, n).astype(F)
    labels = rng.choice(1 << 40, n, replace=False).astype(np.uint64) << np.uint64(8)  # label order is not internal order
    return d, labels


def shaped(shape, k, rng):
    """(d, labels) in internal order: `m` strictly closer rows (0.5) and `t` rows tied at 1.0 around the k-th place, plus farther rows"""
    m = k // 2
    if shape == "a":      # the tie run first, then the closer rows: every closer row after the run evicts a tie (E > 0)
        d = [1.0] * (k - m + 2) + [0.5] * m
    elif shape == "b":    # the closer rows first (E = 0)
        d = [0.5] * m + [1.0] * (k - m + 2)
    elif shape == "c":    # more tied rows than k
        d = [1.0] * (2 * k + 1) + [0.5] * (k // 3)
    elif shape == "d":    # exactly one tied row too many
        d = [1.0] * (k + 1 - m) + [0.5] * m
    elif shape == "e":    # every row at the same distance
        d = [1.0] * (k + 3)
    else:                 # "f": d* = 0 with zeros of both signs, the closer rows negative
        d = [0.0, -0.0] * (k - m + 1) + [-1.0] * m
    d = F(d + [3.0] * 3)
    if shape != "f":
        perm = rng.permutation(len(d)) if shape in ("c", "e") else np.arange(len(d))
        d = d[perm]
    labels = rng.choice(1 << 40, len(d), replace=False).astype(np.uint64) << np.uint64(8)
    return d, labels


def check_single(d, labels, ctx):
    """tie_replay on one index at every k"""
    n = len(d)
    gidx = np.arange(n, dtype=np.uint64)
    straddled = 0
    for k in range(1, n + 3):
        want = literal_heap(d, labels, k)
        kk = min(k, n)
        dstar, lower, first = replay_inputs(d, gidx, labels, kk)
        gd, gl = call_replay(kk, dstar, d, gidx, labels, lower, first)
        assert_same(want, d, labels, gd, gl, (ctx, k))
        srt = np.sort(d, kind="stable")
        straddled += kk < n and not (srt[kk - 1] < srt[kk])
    return straddled


@pytest.mark.parametrize("shape", list("abcdef"))
def test_tie_replay_shapes(shape):
    rng = np.random.default_rng(ord(shape))
    evict = 0
    for k in range(1, 25):
        d, labels = shaped(shape, k, rng)
        kk = min(k, len(d))
        dstar, lower, first = replay_inputs(d, np.arange(len(d)), labels, kk)
        evict += len(set(lower) - set(first))
        gd, gl = call_replay(kk, dstar, d, np.arange(len(d), dtype=np.uint64), labels, lower, first)
        assert_same(literal_heap(d, labels, k), d, labels, gd, gl, (shape, k))
        assert check_single(d, labels, (shape, k)) > 0
    assert (evict == 0) == (shape in "be"), (shape, evict)  # (a) evicts by construction, (b) and (e) never


def test_tie_replay_random_exhaustive_k():
    rng = np.random.default_rng(7)
    straddled = 0
    for it in range(1500):
        n = int(rng.integers(1, 41))
        d, labels = random_config(rng, n, int(rng.integers(1, 5)))
        straddled += check_single(d, labels, it)
    assert straddled > 5000


def test_tie_replay_signed_zero_bits():
    """a tie at d* = 0 whose members carry both signs: the survivors keep the bits of their own rows"""
    d = F([0.0, -0.0, -0.0, 0.0, -1.0, 0.0, -0.0])
    labels = np.array([70, 10, 60, 20, 90, 30, 5], np.uint64)
    for k in range(1, 8):
        dstar, lower, first = replay_inputs(d, np.arange(7), labels, k)
        gd, gl = call_replay(k, dstar, d, np.arange(7, dtype=np.uint64), labels, lower, first)
        want = literal_heap(d, labels, k)
        assert_same(want, d, labels, gd, gl, k)
    assert list(gl) == [90, 5, 10, 20, 30, 60, 70] and list(np.signbit(gd)) == [True, True, True, False, False, True, False]


def shard_lists(d, labels, cuts, k1):
    """every shard's top-min(k1, size) under (dist, local row), padded to k1: what rxgpu_search_knn_device returns per shard"""
    R = len(cuts) - 1
    dist = np.zeros((R, 1, k1), F)
    idx = np.zeros((R, 1, k1), np.uint32)
    lab = np.zeros((R, 1, k1), np.uint64)
    cnt = np.zeros((R, 1), np.uint32)
    for s in range(R):
        a, b = cuts[s], cuts[s + 1]
        order = sorted(range(b - a), key=lambda i: (float(d[a + i]), i))[:k1]
        cnt[s, 0] = len(order)
        dist[s, 0, :len(order)] = d[a + np.array(order, np.int64)] if order else []
        idx[s, 0, :len(order)] = order
        lab[s, 0, :len(order)] = labels[a + np.array(order, np.int64)] if order else []
    return dist, idx, lab, cnt


def test_merge_shards_and_replay_random():
    """rx.merge_shards over random cuts (empty shards, shards shorter than k + 1), then the replay fed shard by shard in rank order as
    rxgpu_sharded_search_knn does it: equal to the literal heap over the concatenated rows"""
    rng = np.random.default_rng(11)
    flagged = 0
    for it in range(500):
        n = int(rng.integers(1, 41))
        d, labels = random_config(rng, n, int(rng.integers(1, 5)))
        R = int(rng.integers(1, 7))
        cuts = [0] + sorted(int(x) for x in rng.integers(0, n + 1, R - 1)) + [n]
        base = np.array(cuts[:-1], np.uint64)
        for k in range(1, n + 3):
            k1 = k + 1
            dist, idx, lab, cnt = shard_lists(d, labels, cuts, k1)
            od, og, ol, oc, nt = rx.merge_shards(k, dist, idx, lab, cnt, base)
            srt = sorted(range(n), key=lambda i: (float(d[i]), i))
            top = srt[:k]
            assert oc[0] == len(top), (it, k)
            assert nt[0] == (n > k and not (d[srt[k - 1]] < d[srt[k]])), (it, k)
            want_top = sorted(top, key=lambda i: (float(d[i]), int(labels[i])))  # runs of equal distances ordered by label
            assert (og[0, :len(top)] == np.array(want_top, np.uint64)).all(), (it, k)
            assert (ol[0, :len(top)] == labels[want_top]).all() and (od[0, :len(top)].view(np.uint32) == d[want_top].view(np.uint32)).all()
            want = literal_heap(d, labels, k)
            if not nt[0]:
                assert_same(want, d, labels, od[0, :oc[0]], ol[0, :oc[0]], (it, k))
                continue
            flagged += 1
            dstar = od[0, k - 1]
            lower = [int(g) for g in og[0, :k] if d[int(g)] < dstar]
            first = []
            for s in range(R):  # each shard's first min(k, #) rows with dist <= d*, concatenated in rank order
                first += [i for i in range(cuts[s], cuts[s + 1]) if d[i] <= dstar][:k]
            gd, gl = call_replay(k, dstar, d, np.arange(n, dtype=np.uint64), labels, lower, first[:k])
            assert_same(want, d, labels, gd, gl, (it, k, cuts))
    assert flagged > 1000
