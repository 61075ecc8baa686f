"""A plain model of the device HNSW builder (test infrastructure): the rules of rxgpu_hnsw_build (DESIGN.md §3.8) written out one
row and one list at a time, over a table of float32 distances.

D[a, b] is the builder's distance with row a as the query: the exact scan's distance of row b to row a staged as a query (for Cosine
normalised as NormalizeCopyVector normalises it, times b's norm coefficient).  `distance_table` obtains every entry from
rxgpu_search_knn, so the model and the device share nothing but the rows.  Equal distances are ordered by row id everywhere."""
import bisect
import heapq

import numpy as np

import reindexer_b200 as rx


def staged_rows(metric, rows):
    """rows as the builder stages them as queries: for Cosine x * k with k = 1 / sqrt(sum x^2) summed in row order in float32
    (tools/normalize.cc:10-23), left alone when the sum is 0 or within 1e-5 of 1"""
    rows = np.ascontiguousarray(rows, np.float32)
    if metric != rx.COS:
        return rows
    s = np.add.accumulate(rows * rows, axis=1, dtype=np.float32)[:, -1]
    k = np.ones(len(rows), np.float32)
    use = (s > 0) & (np.abs(np.float32(1.0) - s) > np.float32(1e-5))
    k[use] = (1.0 / np.sqrt(s[use]).astype(np.float64)).astype(np.float32)
    return (rows * k[:, None]).astype(np.float32)


def distance_table(gpu, metric, rows):
    """D[a, b] for every pair, from the exact scan of the index `gpu` (which holds `rows` as rows 0..n-1, labels row << 32)"""
    n = len(rows)
    gpu.set_tensor_core_filter(2)
    d, lab, cnt = gpu.search_knn(staged_rows(metric, rows), n)
    assert (cnt == n).all()
    t = np.zeros((n, n), np.float32)
    for q in range(n):
        t[q, (lab[q] >> np.uint64(32)).astype(np.int64)] = d[q]
    return t


def plan(M, first, n, maxlevel, levels):
    """the batch ends: row 0 alone on an empty graph; then at most min(2^16, max(1, s // 64)) rows from graph size s, and a row above
    the running top level ends its batch"""
    ends, s, ml = [], first, maxlevel
    if first == 0 and n > 0:
        ends.append(1)
        s, ml = 1, int(levels[0])
    while s < n:
        cap = min(1 << 16, max(1, s >> 6))
        e = s
        while e < n and e - s < cap:
            lv = int(levels[e - first])
            e += 1
            if lv > ml:
                ml = lv
                break
        ends.append(e)
        s = e
    return ends


class Graph:
    """lists[l][v] = neighbour ids in list order; levels[v]; maxlevel / enterpoint"""

    def __init__(self, M):
        self.M, self.lists, self.levels, self.maxlevel, self.enterpoint = M, [{}], [], -1, 0

    @classmethod
    def from_dict(cls, g):
        out = cls(int(g["M"]))
        for v in range(int(g["n"])):
            out.add_node(int(g["levels"][v]))
            row = g["level0"][v]
            out.lists[0][v] = [int(x) for x in row[1:1 + int(row[0])]]
            for l in range(1, int(g["levels"][v]) + 1):
                r = g["upper"][int(g["upper_offsets"][v]) + l - 1]
                out.lists[l][v] = [int(x) for x in r[1:1 + int(r[0])]]
        out.maxlevel, out.enterpoint = int(g["maxlevel"]), int(g["enterpoint"])
        return out

    def add_node(self, level):
        v = len(self.levels)
        self.levels.append(level)
        while len(self.lists) <= level:
            self.lists.append({})
        for l in range(level + 1):
            self.lists[l][v] = []


def search_layer(D, q, ep, level, ef, g):
    """searchBaseLayer as one list of the <= ef best visited nodes ascending by (distance, id): the first unexpanded entry is expanded
    next, the search ends when every entry is expanded.  An entry pushed out of the list is worse than every entry from then on, so
    the unexpanded entries are a heap whose smallest key is past the list's end exactly when none is left."""
    dq = D[q].tolist()
    lst = [(dq[ep], ep)]
    heap = [(dq[ep], ep)]
    visited = {ep}
    lists = g.lists[level]
    while heap:
        k = heapq.heappop(heap)
        if k > lst[-1]:
            break
        fresh = [nid for nid in lists[k[1]] if nid not in visited]
        visited.update(fresh)
        for nid in fresh:
            key = (dq[nid], nid)
            if len(lst) >= ef and not key < lst[-1]:
                continue
            bisect.insort(lst, key)
            del lst[ef:]
            heapq.heappush(heap, key)
    return lst


def heuristic(D, cands, m):
    """getNeighborsByHeuristic2 over (distance, id) candidates in ascending order: fewer than m are all kept; x is dropped when a
    selected s has D[x, s] < its distance"""
    if len(cands) < m:
        return [x for _, x in cands]
    sel = []
    for d, x in cands:
        if len(sel) >= m:
            break
        if all(not (float(D[x, s]) < d) for s in sel):
            sel.append(x)
    return sel


def build(D, M, efc, levels, graph=None):
    """inserts len(levels) rows after the graph's (levels: theirs).  Returns (graph, stats); longest_segment = the most links one list
    received in one batch"""
    g = graph or Graph(M)
    first, n = len(g.levels), len(g.levels) + len(levels)
    links = pruned = longest = 0
    b0 = first
    for e in plan(M, first, n, g.maxlevel, levels):
        ml, ep = g.maxlevel, g.enterpoint
        for u in range(b0, e):
            g.add_node(int(levels[u - first]))
        keys = []
        if ml >= 0:
            for u in range(b0, e):
                lvl = g.levels[u]
                cur = ep
                if lvl < ml:
                    curdist = float(D[u, cur])
                    for level in range(ml, lvl, -1):
                        changed = True
                        while changed:
                            changed = False
                            for nid in list(g.lists[level][cur]):
                                if float(D[u, nid]) < curdist:
                                    curdist, cur, changed = float(D[u, nid]), nid, True
                for l in range(min(lvl, ml), -1, -1):
                    sel = heuristic(D, search_layer(D, u, cur, l, efc, g), M)
                    g.lists[l][u] = sel[::-1]
                    keys += [(l, v, u) for v in sel]
                    cur = sel[0]
            keys.sort()
            links += len(keys)
            i = 0
            while i < len(keys):
                l, v = keys[i][:2]
                j = i
                while j < len(keys) and keys[j][:2] == (l, v):
                    j += 1
                inc = [k[2] for k in keys[i:j]]
                longest = max(longest, len(inc))
                old = g.lists[l][v]
                mc = M if l else 2 * M
                if len(old) + len(inc) <= mc:
                    g.lists[l][v] = old + inc
                else:
                    union = sorted((float(D[v, x]) + 0.0, x) for x in old + inc)
                    g.lists[l][v] = heuristic(D, union, mc)[::-1]
                    pruned += 1
                i = j
        last = e - 1
        if ml < 0 or g.levels[last] > ml:
            g.maxlevel, g.enterpoint = g.levels[last], last
        b0 = e
    return g, dict(reverse_links=links, lists_pruned=pruned, longest_segment=longest)


def assert_same_graph(exported, g, ctx=""):
    """every list in order, the levels, the enter point and the top level of the device's export equal the model's"""
    n = len(g.levels)
    assert int(exported["n"]) == n, ctx
    assert [int(x) for x in exported["levels"]] == g.levels, ctx
    assert (int(exported["maxlevel"]), int(exported["enterpoint"])) == (g.maxlevel, g.enterpoint), ctx
    for v in range(n):
        row = exported["level0"][v]
        got = [int(x) for x in row[1:1 + int(row[0])]]
        assert got == g.lists[0][v], (ctx, "level 0", v, got, g.lists[0][v])
        for l in range(1, g.levels[v] + 1):
            r = exported["upper"][int(exported["upper_offsets"][v]) + l - 1]
            got = [int(x) for x in r[1:1 + int(r[0])]]
            assert got == g.lists[l][v], (ctx, "level", l, v, got, g.lists[l][v])
