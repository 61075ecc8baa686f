"""ORACLE / TEST INFRASTRUCTURE ONLY: ctypes access to the reference merger with highlight areas.

  oracle/_ref/liboracle_ref_ft_areas.so: ft::Merger<IdCont, ft::MergeDataAreas<Area>, OffsetT> compiled in place
  (oracle/ref_ft_areas_facade.cc, built by oracle/areas.mk)
Problems are the FtProblem objects of ft_oracle.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import ft_oracle as F

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def ref_available():
    return os.path.exists(os.path.join(HERE, "_ref", "liboracle_ref_ft_areas.so"))


def ref_lib():
    global _lib
    if _lib is None:
        lib = C.CDLL(os.path.join(HERE, "_ref", "liboracle_ref_ft_areas.so"))
        lib.ref_ft_last_error.restype = C.c_char_p
        u32p = C.POINTER(C.c_uint32)
        lib.ref_ft_merge_query_areas.restype = C.c_int
        lib.ref_ft_merge_query_areas.argtypes = [
            C.c_uint32, C.c_uint32, u32p, C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), C.c_uint32,
            C.POINTER(F.Postings), C.POINTER(F.Config), C.c_uint32, C.POINTER(F.Term), C.c_uint32, C.POINTER(F.Synonym), C.c_int, C.c_int,
            C.c_int32, C.c_uint64, C.c_void_p, u32p, u32p, C.c_uint64, u32p, C.POINTER(C.c_uint64), C.POINTER(C.c_int64)]
        _lib = lib
    return _lib


def ref_merge_areas(prob: F.FtProblem, max_areas_in_doc, rank_sort_type=F.RANK_AND_ID, packed=False, max_out=None):
    """Returns (infos, begin, areas, raw, merge_ns) for at most max_out entries (default: total_docs): infos as ft_oracle.ref_merge;
    begin[len(infos) * nfields + 1] offsets into areas[:, 2] = the committed (start, end) of entry i, field f at begin[i * nfields + f] ..;
    raw[i] = GetAreasCount() before the commit; merge_ns = the Merge call's wall time."""
    p = F._p
    lists, cfg, terms, syns = prob.c_lists(), prob.c_config(), prob.c_terms(), prob.c_synonyms()
    n_max = max(prob.total_docs if max_out is None else max_out, 1)
    cap = n_max * prob.nfields * max(int(max_areas_in_doc), 1)
    out = np.zeros(n_max, F.MERGE_INFO_DTYPE)
    begin = np.zeros(n_max * prob.nfields + 1, np.uint32)
    areas = np.zeros((cap, 2), np.uint32)
    raw = np.zeros(n_max, np.uint32)
    n, ns = C.c_uint64(0), C.c_int64(0)
    u32p = C.POINTER(C.c_uint32)
    rc = ref_lib().ref_ft_merge_query_areas(
        prob.total_docs, prob.nfields, p(prob.words, u32p), p(prob.avg, C.POINTER(C.c_float)),
        None if prob.removed is None else p(prob.removed, C.POINTER(C.c_uint8)),
        None if prob.excluded is None else p(prob.excluded, C.POINTER(C.c_uint8)), len(prob.lists), lists, C.byref(cfg), len(prob.terms), terms,
        len(prob.synonyms), syns, rank_sort_type, int(packed), int(max_areas_in_doc), n_max, out.ctypes.data, p(begin, u32p),
        p(areas, u32p), cap, p(raw, u32p), C.byref(n), C.byref(ns))
    assert rc == 0, ref_lib().ref_ft_last_error().decode()
    m = min(n.value, n_max)
    begin = begin[:m * prob.nfields + 1].copy()
    return out[:m].copy(), begin, areas[:int(begin[-1])].copy(), raw[:m].copy(), ns.value
