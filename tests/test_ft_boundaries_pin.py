"""CPU tests: the C port (oracle/ft_port.c) against the reference's own merger on the boundary problems of
tests/test_ft_boundaries_gpu.py at small and medium sizes, and the numpy restatement of the preselect (ft_helpers.preselect_plan)
against both: the documents it keeps are exactly the ones the mergers return."""
import numpy as np
import pytest
from ft_helpers import assert_same_merge, cut_limit, planted_scores, preselect_plan, random_problem, ref_u16, score_problem

from oracle import ft_oracle as F

needs_ref = pytest.mark.skipif(not F.ref_available(), reason="oracle/_ref not built (needs the reference sources)")


def test_ref_u16_is_the_x86_conversion():
    # cvttss2si: truncation to int32, out of range and NaN give INT32_MIN (low 16 bits 0), then the low 16 bits
    got = ref_u16([70000.5, 65536.0, -5.0, 2147488512.0, 2.0 ** 32, float("nan"), -1e9, 16384.0, 100.9, -0.5])
    assert got.tolist() == [4464, 0, 65531, 0, 0, 0, 13824, 16384, 100, 0]


def threshold_cases(n=20000, seed=0):
    """designed preselect scores: (name, problem) pairs with the threshold below the top by more than one 1024-bin round, on a round
    edge, at score 1, inside the saturated top bin and at the 8192 bin"""
    out = []
    for name, top, thr in (("deep", 30000, 9000), ("edge1023", 65535, 65535 - 1023), ("edge1024", 20000, 20000 - 1024),
                           ("at8192", 12000, 8192), ("below8192", 8192, 8191), ("top", 65535, 65535)):
        s = planted_scores(n, seed, top, thr, run_start=n // 3, run_len=200)
        p = score_problem(s, seed=seed, merge_limit=cut_limit(s, thr, n // 3 + 77))
        p.cfg["min_rank"] = 0
        out.append((name, p))
    s = planted_scores(n, seed, 40, 1, run_start=100, run_len=50, frac=0.01)
    p = score_problem(s, seed=seed, merge_limit=int((s > 0).sum()) + 300)
    p.cfg["min_rank"] = 0
    out.append(("to_one", p))
    return out


@pytest.mark.parametrize("seed", [0, 1])
def test_preselect_restatement_matches_the_port(seed):
    for name, p in threshold_cases(seed=seed):
        plan = preselect_plan(p)
        assert plan["preselect"], name
        if name == "to_one":
            assert plan["min_score"] == 1 and plan["positive"] < p.cfg["merge_limit"] < plan["popcount"]
        else:
            assert plan["top"] >= 8192 and plan["budget"] < len(plan["eq"]), name
        got, _ = F.port_merge(p)
        kept = np.nonzero(plan["score"] > plan["min_score"])[0].tolist() + plan["eq"][:plan["budget"]].tolist()
        assert sorted(got["id"].tolist()) == sorted(kept), name
    sat = np.zeros(3000, bool)
    sat[1:200] = True
    p = score_problem(np.zeros(3000, np.int64), saturated=sat, merge_limit=100)
    plan = preselect_plan(p)
    assert plan["top"] == 65535 and plan["min_score"] == 65535 and plan["budget"] == 100  # five capped terms saturate the u16 score
    assert F.port_merge(p)[0]["id"].tolist() == list(range(1, 101))


@needs_ref
@pytest.mark.parametrize("seed", [0, 1])
def test_port_matches_reference_on_threshold_cases(seed):
    for name, p in threshold_cases(seed=seed):
        for rst in (F.RANK_AND_ID, F.RANK_ONLY, F.ID_ONLY):
            assert_same_merge(F.ref_merge(p, rst)[0], F.port_merge(p, rst)[0], rst, ctx=f"{name} rst {rst}")


def boost_problem(seed, boost, n=3000):
    """random OR / AND terms under the preselect with one term of an out-of-range boost: negative, wrapping past 65536, >= 2^31"""
    p = random_problem(seed, total_docs=n, nfields=1, nterms=4, density=0.3, merge_limit=150, ops=[F.OP_OR, F.OP_OR, F.OP_OR, F.OP_AND])
    p.terms[1]["boost"] = boost
    p.terms[1]["procs"] = np.asarray([100.0, 90.0, 85.0][:len(p.terms[1]["procs"])], np.float32)
    p.cfg["min_rank"] = 0
    return p


# negative, wrapping past 65536 (both sides agree there), in [2^31, 2^32) (max proc 100 x 2.2e7), >= 2^32, infinite
BOOSTS = [-1.0, -5.0, -1e7, 700.005, 2.2e7, 4.3e7, 1e9, float("inf")]


def saturating_u16(proc):
    """a float -> u32 conversion that saturates (NaN -> 0), then the low 16 bits: what a plain uint16_t(float) gives on the device"""
    x = np.nan_to_num(np.asarray(proc, np.float64), nan=0.0, posinf=2.0 ** 32, neginf=0.0)
    return (np.trunc(np.clip(x, 0, 2.0 ** 32 - 1)).astype(np.int64)) & 0xFFFF


def test_out_of_range_boosts_reach_the_conversion():
    """every boost but the wrapping one gives a preselect score that a saturating conversion would not give"""
    for i, b in enumerate(BOOSTS):
        p = boost_problem(i, b)
        plan = preselect_plan(p)
        assert plan["preselect"] and plan["popcount"] > p.cfg["merge_limit"]
        proc = (np.asarray(p.terms[1]["procs"], np.float32) * np.float32(b)).astype(np.float32)
        differs = np.minimum(ref_u16(proc), 16383) != np.minimum(saturating_u16(proc), 16383)
        assert differs.any() == (b != 700.005), (b, proc)


@needs_ref
def test_port_matches_reference_with_out_of_range_boosts():
    for i, b in enumerate(BOOSTS):
        p = boost_problem(i, b)
        for rst in (F.RANK_AND_ID, F.RANK_ONLY):
            a, _ = F.ref_merge(p, rst)
            c, _ = F.port_merge(p, rst)
            assert_same_merge(a, c, rst, ctx=f"boost {b} rst {rst}")
