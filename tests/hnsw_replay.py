"""A plain replay of the reference's HNSW traversal (test infrastructure).

The functions below follow the algorithm as cpp_src/core/index/float_vector/hnswlib/hnswalg.h states it, with its two heaps:
  getLayer0EntryPoint         :799-827   greedy descent through levels maxlevel..1 (strict <, first minimum wins)
  initLayer0SearchState       :829-858   the entry point seeds candidate_set (and top_candidates unless streaming)
  layer0ShouldStopBeforePop   :860-869   bare-bone: stop when the closest candidate is worse than lowerBound; otherwise also
                                         require top_candidates to hold ef entries
  runLayer0Step               :871-966   pop the closest candidate, expand its level-0 list in list order
  SearchKnn                   :1988-2012 trim top_candidates to k
  SearchRange                 :2015-2070 breadth-first closure over level-0 lists from the ef-search's top_candidates
  Begin/ContinueStreamingSearch :1864-1975 (mergeExtrasIntoTopCandidates :1894-1925, emitStreamingBatch :1927-1945)
It does not know how the device organises its lists; the device must reproduce what this computes.

`dist(ids)` returns the float32 distances of one query to the rows `ids` (an int64 array).  The heaps of the reference compare the
distance only (CompareByFirst), so which of two equal distances a heap yields first is not defined.  Whenever the traversal takes
such a decision the result carries tie=True: the device may then legitimately differ."""
import heapq
from collections import Counter

import numpy as np

FLT_MAX = float(np.finfo(np.float32).max)


def _level0(g, v):
    row = g["level0"][v]
    return row[1:1 + int(row[0])]


def _upper(g, v, level):
    row = g["upper"][int(g["upper_offsets"][v]) + level - 1]
    return row[1:1 + int(row[0])]


def _dists(dist, ids):
    return [float(x) for x in np.asarray(dist(np.asarray(ids, np.int64)), np.float32)] if len(ids) else []


class Result:
    """top: [(dist, id)] sorted by (dist, label); n_dist / hops: the reference's metric_distance_computations / metric_hops;
    visited: nodes marked in the level-0 visited list; peak_deleted: most deleted nodes waiting in candidate_set at once;
    peak_candidates: largest candidate_set; tie: a decision compared two equal distances"""

    def __init__(self):
        self.top, self.n_dist, self.hops, self.visited, self.peak_deleted, self.peak_candidates, self.tie = [], 0, 0, 0, 0, 0, False


def entry_point(g, dist, res):
    """getLayer0EntryPoint (:799-827): every listed neighbour is one distance evaluation, every list read one hop"""
    cur = int(g["enterpoint"])
    curdist = _dists(dist, [cur])[0]
    for level in range(int(g["maxlevel"]), 0, -1):
        changed = True
        while changed:
            changed = False
            nb = _upper(g, cur, level)
            res.hops += 1
            res.n_dist += len(nb)
            for u, d in zip(nb.tolist(), _dists(dist, nb)):
                if d < curdist:
                    curdist, cur, changed = d, u, True
    return cur, curdist


class _Heaps:
    """candidate_set (min-heap on distance) and top_candidates (max-heap on distance) with the distance multiset of each, so that a
    pop or replace_top among equal distances is seen"""

    def __init__(self, deleted):
        self.cand, self.top, self.ccount, self.tcount = [], [], Counter(), Counter()
        self.deleted = deleted
        self.waiting_deleted = 0
        self.tie = False

    def push_cand(self, d, v):
        heapq.heappush(self.cand, (d, v))
        self.ccount[d] += 1
        if v in self.deleted:
            self.waiting_deleted += 1

    def pop_cand(self):
        d, v = heapq.heappop(self.cand)
        if self.ccount[d] > 1:
            self.tie = True
        self.ccount[d] -= 1
        if v in self.deleted:
            self.waiting_deleted -= 1
        return d, v

    def push_top(self, d, v):
        heapq.heappush(self.top, (-d, v))
        self.tcount[d] += 1

    def replace_top(self, d, v):
        """replace_top: the worst entry leaves; returns it"""
        wd = -self.top[0][0]
        if self.tcount[wd] > 1:
            self.tie = True
        self.tcount[wd] -= 1
        _, wv = heapq.heapreplace(self.top, (-d, v))
        self.tcount[d] += 1
        return wd, wv

    def top_max(self):
        return -self.top[0][0]


def _take_best(entries, m, res):
    """the m best of entries under the distance alone; a tie across the cut is a tie of the heap that makes the cut"""
    s = sorted(entries)
    if 0 < m < len(s) and s[m - 1][0] == s[m][0]:
        res.tie = True
    return s[:m], s[m:]


def _sorted_out(pairs, labels):
    return sorted(pairs, key=lambda p: (p[0], int(labels[p[1]]) if labels is not None else p[1]))


def search_top(g, dist, ef, deleted=frozenset()):
    """searchBaseLayerST after getLayer0EntryPoint (search(), :1979-1986): returns (Result with the whole top_candidates)"""
    res = Result()
    ep, epd = entry_point(g, dist, res)
    bare = not deleted
    h = _Heaps(deleted)
    visited = np.zeros(int(g["n"]), bool)
    if bare or ep not in deleted:  # initLayer0SearchState :844-855
        lower = epd
        h.push_top(epd, ep)
        h.push_cand(epd, ep)
    else:
        lower = FLT_MAX
        h.push_cand(FLT_MAX, ep)
    visited[ep] = True
    nvis = 1
    res.peak_deleted = h.waiting_deleted
    res.peak_candidates = len(h.cand)
    while h.cand:  # layer0ShouldStopBeforePop
        cd = h.cand[0][0]
        if cd > lower and (bare or len(h.top) >= ef):
            break
        _, v = h.pop_cand()  # runLayer0Step
        nb = _level0(g, v)
        res.hops += 1
        res.n_dist += len(nb)
        fresh = [u for u in nb.tolist() if not visited[u]]
        visited[fresh] = True
        nvis += len(fresh)
        for u, d in zip(fresh, _dists(dist, fresh)):
            if len(h.top) < ef or lower > d:  # flag_consider_candidate
                h.push_cand(d, u)
                if bare or u not in deleted:
                    if len(h.top) < ef:
                        h.push_top(d, u)
                    else:
                        h.replace_top(d, u)
                if h.top:
                    lower = h.top_max()
        res.peak_deleted = max(res.peak_deleted, h.waiting_deleted)
        res.peak_candidates = max(res.peak_candidates, len(h.cand))
    res.visited = nvis
    res.tie = h.tie
    res.top = [(-nd, v) for nd, v in h.top]
    return res


def search_knn(g, dist, k, ef=0, deleted=frozenset(), labels=None):
    """SearchKnn (:1988-2012): k = min(k, n), ef = ef or 3k/2; top-k as [(dist, id)] sorted by (dist, label)"""
    k = min(int(k), int(g["n"]))
    ef = max(int(ef) if ef else k * 3 // 2, 1)
    res = search_top(g, dist, ef, deleted)
    best, _ = _take_best(res.top, k, res)  # while (top_candidates.size() > k) pop()
    res.top = _sorted_out(best, labels)
    return res


def search_range(g, dist, radius, ef, deleted=frozenset(), labels=None):
    """SearchRange (:2015-2070): the ef-search's top_candidates seed a breadth-first expansion over level-0 lists; deleted neighbours
    are skipped without being marked.  Returns a Result whose top holds every match, sorted by (dist, label)"""
    res = search_top(g, dist, max(int(ef), 1), deleted)
    radius = float(np.float32(radius))
    visited = np.zeros(int(g["n"]), bool)
    queue, out = [], []
    for d, v in res.top:
        if d < radius:
            queue.append(v)
            out.append((d, v))
        visited[v] = True
    head = 0
    while head < len(queue):
        v = queue[head]
        head += 1
        fresh = []
        for u in _level0(g, v).tolist():
            if u in deleted or visited[u]:
                continue
            visited[u] = True
            fresh.append(u)
        for u, d in zip(fresh, _dists(dist, fresh)):
            if d < radius:
                queue.append(u)
                out.append((d, u))
    res.top = _sorted_out(out, labels)
    return res


class Stream:
    """BeginStreamingSearch (:1864-1892) and ContinueStreamingSearch (:1947-1975) of one query"""

    def __init__(self, g, dist, ef=0, deleted=frozenset(), labels=None):
        self.g, self.dist, self.deleted, self.labels = g, dist, deleted, labels
        self.ef = int(ef) if ef else 100  # kDefaultStreamingEf
        self.res = Result()
        ep, epd = entry_point(g, dist, self.res)
        self.bare = not deleted
        self.h = _Heaps(deleted)
        self.extras = []  # top_candidates_extras: (dist, id)
        self.visited = np.zeros(int(g["n"]), bool)
        # initLayer0SearchState in streaming mode: the entry point is a candidate only
        self.lower = epd if (self.bare or ep not in deleted) else FLT_MAX
        self.h.push_cand(self.lower, ep)
        self.visited[ep] = True
        self.res.peak_candidates = 1
        self.exhausted = False

    def next(self, batch):
        """one ContinueStreamingSearch call: the batch as [(dist, id)] sorted by (dist, label), and the exhausted flag"""
        if batch == 0:
            return [], self.exhausted
        h, res = self.h, self.res
        ef = max(self.ef, int(batch))  # state.ef = max(state.ef, batchSize), restored before the call returns (:1961-1970)
        if len(h.top) < ef and self.extras:  # mergeExtrasIntoTopCandidates: the best extras fill top_candidates up to ef
            take, self.extras = _take_best(self.extras, ef - len(h.top), res)
            for d, v in take:
                h.push_top(d, v)
            self.lower = h.top_max()
        while h.cand:
            cd = h.cand[0][0]
            if cd > self.lower and len(h.top) >= ef:
                break
            d0, v = h.pop_cand()
            if self.bare or v not in self.deleted:  # the streaming branch of runLayer0Step (:880-893)
                if len(h.top) < ef:
                    h.push_top(d0, v)
                elif self.lower > d0:
                    self.extras.append(h.replace_top(d0, v))
                self.lower = h.top_max()
            nb = _level0(self.g, v)
            res.hops += 1
            res.n_dist += len(nb)
            fresh = [u for u in nb.tolist() if not self.visited[u]]
            self.visited[fresh] = True
            for u, d in zip(fresh, _dists(self.dist, fresh)):
                h.push_cand(d, u)
            res.peak_candidates = max(res.peak_candidates, len(h.cand))
        # emitStreamingBatch: the batch best leave top_candidates
        out, rest = _take_best([(-nd, v) for nd, v in h.top], int(batch), res)
        h.top, h.tcount = [], Counter()
        for d, v in rest:
            h.push_top(d, v)
        res.tie = res.tie or h.tie
        self.exhausted = not h.cand and not h.top and not self.extras
        return _sorted_out(out, self.labels), self.exhausted
