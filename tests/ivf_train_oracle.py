"""FAISS's IVF k-means as reindexer::IvfIndex trains it, with the Clustering's iteration statistics, and faiss::rand_perm (test
infrastructure: ctypes over tests/cpp/_build/libivf_train_oracle.so, built from tests/cpp/ivf_train_oracle.cc by __graft_entry__.build()
where the reference tree exists).  Its sgemm is a triple loop, so keep the shapes small."""
import ctypes as C
import os

import numpy as np

LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "_build", "libivf_train_oracle.so")
_f32p, _f64p, _i32p = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int32)
_lib = None


def available():
    return os.path.exists(LIB)


def _p(a, t):
    return a.ctypes.data_as(t)


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        L.ivf_train_last_error.restype = C.c_char_p
        L.ivf_train_rand_perm.argtypes = [_i32p, C.c_size_t, C.c_int64]
        L.ivf_train_faiss.argtypes = [C.c_int, C.c_size_t, C.c_size_t, C.c_size_t, _f32p, _f32p, C.c_int, C.c_int, C.c_int, _f32p, _f64p,
                                      _i32p, _i32p]
        _lib = L
    return _lib


def rand_perm(n, seed):
    out = np.zeros(max(n, 1), np.int32)
    lib().ivf_train_rand_perm(_p(out, _i32p), n, seed)
    return out[:n]


def train(metric, vecs, nlist, niter=10, seed=1234, max_points_per_centroid=256, norms=None):
    """IndexIVFFlat::train(n, vecs, norms) with cp.niter / seed / max_points_per_centroid: (centroids [nlist, dim], obj, nsplit) with
    one obj / nsplit entry per iteration (one zero entry when the sample size equals nlist)"""
    x = np.ascontiguousarray(vecs, np.float32)
    n, dim = x.shape
    nm = None if norms is None else np.ascontiguousarray(norms, np.float32)
    cent = np.zeros((nlist, dim), np.float32)
    obj = np.zeros(niter + 1, np.float64)
    nsplit = np.zeros(niter + 1, np.int32)
    ns = C.c_int32(0)
    rc = lib().ivf_train_faiss(metric, dim, nlist, n, _p(x, _f32p), None if nm is None else _p(nm, _f32p), niter, seed,
                               max_points_per_centroid, _p(cent, _f32p), _p(obj, _f64p), _p(nsplit, _i32p), C.byref(ns))
    assert rc == 0, lib().ivf_train_last_error().decode()
    return cent, obj[:ns.value], nsplit[:ns.value]
