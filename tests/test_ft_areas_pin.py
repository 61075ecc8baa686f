"""CPU tests: the reference merger with highlight areas (oracle/_ref/liboracle_ref_ft_areas.so, MergeDataAreas<Area>) pinned against a
restatement of core/ft/areaholder.h and Merger::addAreas (ft_fast/merger.h:196-205) in a few lines of Python, on hand-made edge cases
and on random OR problems.  For OR terms with non-zero field boosts every posting of every term reaches its document, term by term,
subterms by descending proc, so the model only needs calcTermRank, which the reference's own function supplies."""
import numpy as np
import pytest
from ft_helpers import random_problem

from oracle import ft_areas_oracle as FA
from oracle import ft_oracle as F

pytestmark = pytest.mark.skipif(not (FA.ref_available() and F.ref_available()), reason="needs oracle/_ref (the reference's own merger)")


# ---- areaholder.h restated ------------------------------------------------------------------------------------------------------------
def concat(a, b):
    """Area::Concat: a (a mutable [start, end]) absorbs b when b touches it (note the asymmetric containment test)"""
    if a[0] <= b[0] <= a[1] or a[0] <= b[1] <= a[1] or (a[0] > b[0] and a[1] < b[1]):
        a[0], a[1] = min(a[0], b[0]), max(a[1], b[1])
        return True
    return False


class Doc:
    """AreasInDocument<Area>: one AreasInField ring (data, index_) per field and maxTermRank_"""

    def __init__(self, nfields):
        self.data = [[] for _ in range(nfields)]
        self.index = [0] * nfields
        self.max_rank = 0.0

    def insert(self, f, area, rank, A):  # AreasInField::Insert
        data, idx = self.data[f], self.index[f]
        if idx > 0 and concat(data[(idx - 1) % A], area):
            return True
        if len(data) == A:
            if rank > self.max_rank:
                data[idx % A] = list(area)
                self.index[f] += 1
                return True
            return False
        data.append(list(area))
        self.index[f] += 1
        return True

    def add_areas(self, positions, rank, A):  # Merger::addAreas: the first refused word ends the walk, later fields included
        for q in positions:
            p = int(q) & 0xFFFFFF
            if not self.insert(int(q) >> 24, (p, p + 1), rank, A):
                break
        self.max_rank = max(self.max_rank, rank)  # UpdateRank

    def raw(self):
        return sum(len(d) for d in self.data)

    def committed(self, f):  # AreasInField::Commit: sort by start, fold each area into its left neighbour when they touch
        out = sorted((list(a) for a in self.data[f]), key=lambda a: a[0])
        i = 1
        while i < len(out):
            if concat(out[i], out[i - 1]):
                del out[i - 1]
            else:
                i += 1
        return [tuple(a) for a in out]


def model(prob, A):
    """the areas of every document an OR-only problem merges: {doc id: Doc}"""
    import ctypes as C

    lib, cfg, terms = F.ref_lib(), prob.c_config(), prob.c_terms()
    out = [C.c_float() for _ in range(4)] + [C.c_int()]
    u32p, f32p = C.POINTER(C.c_uint32), C.POINTER(C.c_float)

    def calc_term_rank(ti, proc, matched, pp, words):  # ft_oracle.ref_calc_term_rank without rebuilding the ctypes views per posting
        assert lib.ref_ft_calc_term_rank(prob.nfields, C.byref(cfg), C.byref(terms[ti]), proc, prob.total_docs - 1, matched, len(pp),
                                         pp.ctypes.data_as(u32p), words.ctypes.data_as(u32p), prob.avg.ctypes.data_as(f32p),
                                         *[C.byref(o) for o in out]) == 0
        return out[0].value

    docs = {}
    for ti, t in enumerate(prob.terms):
        assert t["op"] == F.OP_OR and (np.asarray(t["field_boosts"]) != 0).all()
        subs = sorted(zip(t["postings"], t["procs"]), key=lambda s: -s[1])  # SortSubterms (procs are distinct)
        for li, proc in subs:
            d_ids, begin, pos = prob.lists[int(li)]
            for i, d in enumerate(d_ids):
                pp = pos[begin[i]:begin[i + 1]]
                rank = calc_term_rank(ti, float(proc), len(d_ids), np.ascontiguousarray(pp), np.ascontiguousarray(prob.words[d]))
                if rank == 0.0:
                    continue
                docs.setdefault(int(d), Doc(prob.nfields)).add_areas(pp, rank, A)
    return docs


def split(prob, begin, areas, i):
    nf = prob.nfields
    return [[tuple(int(x) for x in a) for a in areas[begin[i * nf + f]:begin[i * nf + f + 1]]] for f in range(nf)]


def check(prob, A, ctx=""):
    infos, begin, areas, raw, _ = FA.ref_merge_areas(prob, A)
    ref_plain, _ = F.ref_merge(prob)
    assert (infos == ref_plain).all(), ctx  # MergeDataAreas merges the same documents with the same ranks as MergeData
    docs = model(prob, A)
    assert sorted(docs) == sorted(int(x) for x in infos["id"]), ctx
    for i, d in enumerate(infos["id"]):
        doc = docs[int(d)]
        assert raw[i] == doc.raw(), (ctx, int(d))
        assert split(prob, begin, areas, i) == [doc.committed(f) for f in range(prob.nfields)], (ctx, int(d))
    return infos, begin, areas, raw


# ---- hand-made edge cases -------------------------------------------------------------------------------------------------------------
def one_doc(nfields, terms):
    """document 1 only; terms: list of (boost, [subterm positions as [(pos, field)], ...]) -- every subterm its own list"""
    words = np.full((3, nfields), 40, np.uint32)
    words[0] = 0
    p = F.FtProblem(3, words)
    procs = [100.0, 90.0, 80.0, 70.0]
    for boost, subs in terms:
        p.add_term([(p.add_list([1], [pp]), procs[s]) for s, pp in enumerate(subs)], boost=boost, field_boosts=np.ones(nfields, np.float32))
    return p


def areas_of(prob, A):
    infos, begin, areas, raw = check(prob, A)
    assert len(infos) == 1
    return split(prob, begin, areas, 0), int(raw[0])


def test_ring_of_one():
    # (3,4) is appended, (4,5) widens it to (3,5), (9,10) overwrites the full ring: the first term's rank beats maxTermRank_ = 0
    assert areas_of(one_doc(1, [(1.0, [[(3, 0), (4, 0), (9, 0)]])]), 1) == ([[(9, 10)]], 1)


def test_overwrite_after_full_needs_a_higher_rank():
    # term 2 ranks higher than term 1: it overwrites slot index_ % A = 0; ranked lower it is refused
    assert areas_of(one_doc(1, [(1.0, [[(0, 0), (5, 0)]]), (3.0, [[(10, 0)]])]), 2) == ([[(5, 6), (10, 11)]], 2)
    assert areas_of(one_doc(1, [(1.0, [[(0, 0), (5, 0)]]), (0.3, [[(10, 0)]])]), 2) == ([[(0, 1), (5, 6)]], 2)


def test_concat_while_full():
    # the ring is full and term 2 ranks lower, but (6,7) touches the last written area (5,6): widened, not refused
    assert areas_of(one_doc(1, [(1.0, [[(0, 0), (5, 0)]]), (0.3, [[(6, 0)]])]), 2) == ([[(0, 1), (5, 7)]], 2)


def test_duplicate_positions_from_two_subterms():
    # both variants of one term hold word 3: the second (3,4) merges into the first
    assert areas_of(one_doc(1, [(1.0, [[(3, 0)], [(3, 0), (7, 0)]])]), 5) == ([[(3, 4), (7, 8)]], 2)


def test_break_skips_later_fields():
    # term 2 (lower rank) is refused in field 0, whose ring is full: its position in field 1 is never offered
    assert areas_of(one_doc(2, [(1.0, [[(0, 0)]]), (0.3, [[(5, 0), (2, 1)]])]), 1) == ([[(0, 1)], []], 1)
    # ranked higher it overwrites field 0 and goes on to field 1
    assert areas_of(one_doc(2, [(1.0, [[(0, 0)]]), (3.0, [[(5, 0), (2, 1)]])]), 1) == ([[(5, 6)], [(2, 3)]], 2)


def test_commit_unites_touching_areas_after_overwrites():
    # each term ranks higher than the one before, so each overwrites the oldest slot: the ring ends as (11,12) (2,3) (12,13), unsorted,
    # and the commit sorts it by start and unites (11,12) with (12,13)
    p = one_doc(1, [(1.0, [[(10, 0), (20, 0), (30, 0)]]), (2.0, [[(11, 0)]]), (3.0, [[(2, 0), (12, 0)]])])
    assert areas_of(p, 3) == ([[(2, 3), (11, 13)]], 3)


# ---- random problems ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("A", [1, 2, 3, 5, 64])
@pytest.mark.parametrize("nfields", [1, 3])
def test_random_problems_match_the_model(A, nfields):
    for seed in range(20):
        p = random_problem(1000 * A + 100 * nfields + seed, total_docs=60, nfields=nfields, nterms=int(1 + seed % 3), max_sub=3, density=0.3,
                           ops=[F.OP_OR] * 3, max_pos=12, doc_len=(2, 14))
        for t in p.terms:
            t["field_boosts"] = np.maximum(t["field_boosts"], np.float32(0.5))
        check(p, A, ctx=f"A={A} nfields={nfields} seed={seed}")
