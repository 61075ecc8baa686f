"""A plain NumPy model of the mutable index state (test infrastructure).

`IndexModel` mirrors one brute-force shard: its capacity and its live rows in internal order, as the reference's
BruteforceSearch keeps them (SURVEY.md §8a rules 3-5, bruteforce.cc:44-101):
  * upserting a label that exists rewrites its row in place; a new label appends;
  * labels repeated inside one batch apply in order, so the last write wins;
  * a batch that reaches capacity applies its leading rows and then fails (LogicError);
  * remove moves the last row into the hole; removing an unknown label does nothing;
  * resize refuses a capacity below the size; clone is a deep copy with capacity max(old, new);
  * append_synth(seed, first_row, n) appends rows O.synth_matrix(seed, n, dim, first_row) under labels (first_row + r) << 32, and
    refuses (applying nothing) when it would pass the capacity or reuse a live label.
`knn` / `range_search` restate the reference's heap on the model's rows (bruteforce.cc:103-143) for integer-valued rows, where every
summation order gives the same fp32 distance, so the result (labels, order and distance bits) is fully determined.

`IvfModel` holds IVF lists in per-list order, with the FAISS swap-remove inside a list (DirectMap::remove_ids, Hashtable flavour).
`HnswModel` holds a host HNSW graph in the dict layout of hnsw_import / hnsw_update, the row and label of every slot and the set of
tombstoned slots."""
import copy
import heapq

import numpy as np

from oracle import oracle as O

L2, IP, COS = 0, 1, 2
F = np.float32
TOMB = np.uint64(1) << np.uint64(63)


class LogicError(Exception):
    """the operation the reference refuses with errLogic"""


class NotFound(Exception):
    """the operation the reference refuses with errNotFound"""


def norm_coef(v):
    """calculateL2Module (normalize.cc:10-23) on fp32 sums that are exact for integer-valued rows"""
    s = F(np.dot(v.astype(np.float64), v.astype(np.float64)))
    if s > 0 and abs(F(1) - s) > F(1e-5):
        return F(1.0 / np.float64(np.sqrt(s)))
    return F(1)


class IndexModel:
    def __init__(self, metric, dim, capacity):
        self.metric, self.dim, self.capacity = metric, dim, capacity
        self._buf = np.zeros((16, dim), F)  # grows by doubling; rows = its first `size` rows
        self.labels = []
        self.pos = {}

    @property
    def size(self):
        return len(self.labels)

    @property
    def rows(self):
        return self._buf[:self.size]

    def _set(self, idx, label, vec):
        if idx == self.size:
            if idx == len(self._buf):
                self._buf = np.concatenate([self._buf, np.zeros_like(self._buf)])
            self.labels.append(label)
        self._buf[idx] = vec
        self.pos[label] = idx

    def upsert(self, labels, vecs):
        vecs = np.asarray(vecs, F).reshape(-1, self.dim)
        for lab, v in zip((int(x) for x in labels), vecs):
            idx = self.pos.get(lab, self.size)
            if idx == self.size and self.size >= self.capacity:
                raise LogicError("The number of elements exceeds the specified limit")
            self._set(idx, lab, v.copy())

    def remove(self, label):
        label = int(label)
        cur = self.pos.pop(label, None)
        if cur is None:
            return
        last = self.size - 1
        if cur != last:
            moved = self.labels[last]
            self._buf[cur] = self._buf[last]
            self.labels[cur] = moved
            self.pos[moved] = cur
        self.labels.pop()

    def resize(self, capacity):
        if capacity < self.size:
            raise LogicError("Cannot resize, max element is less than the current number of elements")
        self.capacity = capacity

    def clone(self, capacity):
        c = copy.deepcopy(self)
        c.capacity = max(self.capacity, capacity)
        return c

    def append_synth(self, seed, first_row, n):
        labels = [(first_row + r) << 32 for r in range(n)]
        if self.size + n > self.capacity or any(lab in self.pos for lab in labels):
            raise LogicError("append_synth refused")
        rows = O.synth_matrix(seed, n, self.dim, first_row=first_row)
        for lab, v in zip(labels, rows):
            self._set(self.size, lab, v)

    def get(self, label):
        return self.rows[self.pos[int(label)]]

    def row_of(self, labels):
        """internal positions of `labels` (-1 for a label the model does not hold)"""
        return np.array([self.pos.get(int(x), -1) for x in np.asarray(labels).ravel()], np.int64).reshape(np.shape(labels))

    def label_array(self):
        return np.array(self.labels, np.uint64)

    # ---- exact answers on integer-valued rows
    def distances(self, q):
        """fp32 distance of query q to every row in internal order (exact on integer-valued rows and queries)"""
        q64, v64 = np.asarray(q, np.float64), self.rows.astype(np.float64)
        if self.metric == L2:
            return F(1) * ((v64 - q64) ** 2).sum(1).astype(F)
        d = -(v64 @ q64).astype(F)
        if self.metric == COS:
            s = (v64 * v64).sum(1).astype(F)
            long = (s > 0) & (np.abs(F(1) - s) > F(1e-5))
            with np.errstate(divide="ignore"):
                coef = np.where(long, (1.0 / np.sqrt(np.where(long, s, F(1))).astype(np.float64)).astype(F), F(1))
            d = d * coef.astype(F)
        return d.astype(F)

    def knn(self, q, k):
        """bruteforce.cc:103-127: the first k rows enter the max-heap on (dist, label), later rows replace its top only when strictly
        closer; returned best first"""
        d = self.distances(q)
        k = min(k, self.size)
        if k == 0:
            return np.zeros(0, F), np.zeros(0, np.uint64)
        heap = [(-float(d[i]), -self.labels[i]) for i in range(k)]
        heapq.heapify(heap)
        for i in range(k, self.size):
            if d[i] < -heap[0][0]:
                heapq.heapreplace(heap, (-float(d[i]), -self.labels[i]))
        out = sorted((-a, -b) for a, b in heap)
        return np.array([a for a, _ in out], F), np.array([b for _, b in out], np.uint64)

    def range_search(self, q, radius):
        d = self.distances(q)
        hit = sorted((float(d[i]), self.labels[i]) for i in np.nonzero(d < F(radius))[0])
        return np.array([a for a, _ in hit], F), np.array([b for _, b in hit], np.uint64)


class IvfModel:
    """IVF lists in per-list order"""

    def __init__(self, nlist, dim):
        self.dim = dim
        self.lists = [[] for _ in range(nlist)]  # [(label, row)]
        self.where = {}

    @property
    def size(self):
        return len(self.where)

    def add(self, list_nos, labels, vecs):
        labels = [int(x) for x in labels]
        if any(lab in self.where for lab in labels) or len(set(labels)) != len(labels):
            raise LogicError("the id is already in the IVF lists")
        for l, lab, v in zip(list_nos, labels, np.asarray(vecs, F).reshape(-1, self.dim)):
            self.lists[int(l)].append((lab, v.copy()))
            self.where[lab] = int(l)

    def remove(self, label):
        label = int(label)
        if label not in self.where:
            raise NotFound("the id is not in the IVF lists")
        lst = self.lists[self.where.pop(label)]
        pos = next(i for i, (lab, _) in enumerate(lst) if lab == label)
        lst[pos] = lst[-1]
        lst.pop()

    def flat(self):
        """(rows, labels, list of each row) over the lists in list order"""
        ent = [(lab, v, l) for l, lst in enumerate(self.lists) for lab, v in lst]
        rows = np.array([v for _, v, _ in ent], F).reshape(-1, self.dim)
        return rows, np.array([lab for lab, _, _ in ent], np.uint64), np.array([l for _, _, l in ent], np.int64)


class HnswModel:
    """a host HNSW graph (hnsw_import layout), the row and label of every slot, and the tombstoned slots"""

    def __init__(self, graph, rows, labels):
        self.g = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in graph.items()}
        self.g["upper"] = self.g["upper"].reshape(-1, 1 + self.g["M"])
        self.rows = np.asarray(rows, F).copy()
        self.labels = [int(x) for x in labels]
        self.deleted = set()
        self.updates = 0

    @property
    def n(self):
        return self.g["n"]

    def slot_of(self, labels):
        pos = {lab: i for i, lab in enumerate(self.labels)}
        return np.array([pos.get(int(x), -1) for x in np.asarray(labels).ravel()], np.int64)

    def _retire_label(self, label, slot):
        """a label that lives again in `slot`: its tombstoned former slot takes the label (1 << 63) | slot of its own"""
        for i, lab in enumerate(self.labels):
            if lab == label and i != slot and i in self.deleted:
                self.labels[i] = int(TOMB) | i

    def append(self, label, vec, level, level0, upper_lists):
        g, v = self.g, self.n
        self._retire_label(int(label), v)
        row = np.zeros(1 + g["maxM0"], np.uint32)
        row[0], row[1:1 + len(level0)] = len(level0), level0
        g["level0"] = np.concatenate([g["level0"], row[None]])
        g["levels"] = np.append(g["levels"], np.int32(level)).astype(np.int32)
        g["upper_offsets"] = np.append(g["upper_offsets"], g["upper_offsets"][-1] + level).astype(np.int64)
        up = np.zeros((level, 1 + g["M"]), np.uint32)
        for lv, lst in enumerate(upper_lists):
            up[lv, 0], up[lv, 1:1 + len(lst)] = len(lst), lst
        g["upper"] = np.concatenate([g["upper"], up])
        g["n"] = v + 1
        self.rows = np.concatenate([self.rows, np.asarray(vec, F)[None]])
        self.labels.append(int(label))
        return v

    def set_lists(self, v, level0=None, upper_lists=None):
        g = self.g
        if level0 is not None:
            g["level0"][v] = 0
            g["level0"][v, 0], g["level0"][v, 1:1 + len(level0)] = len(level0), level0
        for lv, lst in enumerate(upper_lists or ()):
            slot = int(g["upper_offsets"][v]) + lv
            g["upper"][slot] = 0
            g["upper"][slot, 0], g["upper"][slot, 1:1 + len(lst)] = len(lst), lst

    def update_point(self, v, label, vec):
        self._retire_label(int(label), v)
        self.rows[v] = vec
        self.labels[v] = int(label)

    def graph(self):
        return self.g
