"""The reference's FAISS IndexIVFFlat over GIVEN centroids and list assignments, without k-means (test infrastructure: ctypes over
tests/cpp/_build/libivf_lists_oracle.so, built from tests/cpp/ivf_lists_oracle.cc by __graft_entry__.build() where the reference
tree exists).  The search surface matches oracle.RefIvf: search / range_search / search_batch in FAISS' distance convention, and add /
remove / list_of as IvfIndex::upsert / del drive the index."""
import ctypes as C
import os

import numpy as np

LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "_build", "libivf_lists_oracle.so")
_f32p, _i64p, _u32p = C.POINTER(C.c_float), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
_lib = None


def available():
    return os.path.exists(LIB)


def _p(a, t):
    return a.ctypes.data_as(t)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        L.ivf_lists_last_error.restype = C.c_char_p
        L.ivf_lists_create.restype = C.c_void_p
        L.ivf_lists_create.argtypes = [C.c_int, C.c_size_t, C.c_size_t, _f32p, C.c_size_t, _i64p, _i64p, _f32p]
        L.ivf_lists_destroy.argtypes = [C.c_void_p]
        L.ivf_lists_add.argtypes = [C.c_void_p, C.c_size_t, _f32p, _i64p]
        L.ivf_lists_remove.argtypes = [C.c_void_p, C.c_int64]
        L.ivf_lists_list_of.argtypes = [C.c_void_p, C.c_size_t, _i64p, _u32p]
        L.ivf_lists_search.argtypes = [C.c_void_p, C.c_size_t, _f32p, C.c_size_t, C.c_size_t, _f32p, _i64p]
        L.ivf_lists_range_search.restype = C.c_int64
        L.ivf_lists_range_search.argtypes = [C.c_void_p, _f32p, C.c_float, C.c_size_t, C.c_size_t, _f32p, _i64p]
        _lib = L
    return _lib


class ListsIvf:
    """metric: 0 = L2, 1 = IP, 2 = Cosine; row i of vecs goes to list list_nos[i] with id labels[i]"""

    def __init__(self, metric, centroids, list_nos, labels, vecs):
        self.lib = lib()
        cent = np.ascontiguousarray(centroids, np.float32)
        vecs = np.ascontiguousarray(vecs, np.float32)
        ln = np.ascontiguousarray(list_nos).astype(np.int64)
        ids = np.ascontiguousarray(labels).astype(np.int64)
        self.metric, self.dim, self.nlist = metric, cent.shape[1], len(cent)
        self.h = self.lib.ivf_lists_create(metric, self.dim, self.nlist, _p(cent, _f32p), len(ids), _p(ln, _i64p), _p(ids, _i64p),
                                           _p(vecs, _f32p))
        assert self.h, self.lib.ivf_lists_last_error().decode()

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.ivf_lists_destroy(self.h)
            self.h = None

    def _ok(self, rc):
        assert rc == 0, self.lib.ivf_lists_last_error().decode()

    def add(self, labels, vecs):
        """IvfIndex::upsert on the trained index, one add_with_ids per row (FAISS' quantizer picks the list)"""
        vecs = np.ascontiguousarray(vecs, np.float32)
        ids = np.ascontiguousarray(labels).astype(np.int64)
        self._ok(self.lib.ivf_lists_add(self.h, len(ids), _p(vecs, _f32p), _p(ids, _i64p)))

    def remove(self, label):
        self._ok(self.lib.ivf_lists_remove(self.h, int(label)))

    def list_of(self, labels):
        ids = np.ascontiguousarray(labels).astype(np.int64)
        out = np.zeros(len(ids), np.uint32)
        self._ok(self.lib.ivf_lists_list_of(self.h, len(ids), _p(ids, _i64p), _p(out, _u32p)))
        return out

    def search_batch(self, queries, k, nprobe):
        q = np.ascontiguousarray(queries, np.float32).reshape(-1, self.dim)
        d = np.zeros((len(q), k), np.float32)
        i = np.zeros((len(q), k), np.int64)
        self._ok(self.lib.ivf_lists_search(self.h, len(q), _p(q, _f32p), k, nprobe, _p(d, _f32p), _p(i, _i64p)))
        return d, i

    def search(self, q, k, nprobe):
        """(dist, label) best first; dist in FAISS' convention (L2: squared distance, IP / Cosine: +similarity)"""
        d, i = self.search_batch(q, k, nprobe)
        n = int((i[0] >= 0).sum())
        return d[0, :n].copy(), i[0, :n].astype(np.uint64)

    def range_search(self, q, radius, nprobe, max_out=100000):
        """(dist, label) unsorted; radius and dist in FAISS' convention"""
        q = np.ascontiguousarray(q, np.float32)
        d = np.zeros(max_out, np.float32)
        i = np.zeros(max_out, np.int64)
        n = self.lib.ivf_lists_range_search(self.h, _p(q, _f32p), float(radius), nprobe, max_out, _p(d, _f32p), _p(i, _i64p))
        assert 0 <= n <= max_out, (n, self.lib.ivf_lists_last_error().decode())
        return d[:n].copy(), i[:n].astype(np.uint64)
