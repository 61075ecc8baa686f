"""CPU tests of the int8 filter's certificate, independent of any kernel: the restated quantiser (tests/tc_certificate.py) against exact
Fractions, and the derivation of tc_block_threshold (knn_tc.cuh) -- its float32 evaluation, every operation rounded once from the
exact value, never admits less than the real block threshold T_B(q) <= T(q, v) on random and adversarial factors."""
import math
from fractions import Fraction as F

import numpy as np
import pytest

import tc_certificate as TC


def test_f32_rounding_is_correct_and_single():
    # a value just above a float32 tie: rounding through float64 first lands on the tie and then rounds to even (down)
    x = F(1) + F(1, 2 ** 24) + F(1, 2 ** 60)
    assert np.float32(float(x)) == np.float32(1.0)
    assert TC.f32(x) == np.nextafter(np.float32(1.0), np.float32(2.0))
    assert TC.f32(F(1) + F(1, 2 ** 24)) == np.float32(1.0)                       # tie to even
    assert TC.fr(TC.f32(F(-3, 10), "rd")) < F(-3, 10) < TC.fr(TC.f32(F(-3, 10), "ru"))
    assert TC.f32(F(2) ** 200) == np.inf and TC.f32(F(2) ** 200, "rd") == np.finfo(np.float32).max
    assert TC.f32(F(1, 2 ** 150) * 3) == np.float32(2.0 ** -148)                   # subnormal, tie to even
    assert TC.f32(F(1, 2 ** 151), "ru") == np.float32(2.0 ** -149) and TC.f32(F(1, 2 ** 151)) == 0.0
    rng = np.random.default_rng(1)
    for a in rng.standard_normal(200).astype(np.float32) * np.float32(1e3):
        for b in rng.standard_normal(3).astype(np.float32):
            assert TC.f32(TC.fr(a) * TC.fr(b)) == a * b      # IEEE float32 products are correctly rounded


@pytest.mark.parametrize("dim", [1, 127, 128, 129, 768, 2048])
def test_quantiser_bounds_exact(dim):
    rng = np.random.default_rng(dim)
    rows = [rng.standard_normal((24, dim)) * 10.0 ** rng.uniform(-30, 30, (24, 1)),
            np.concatenate([np.full((4, 1), 127), rng.integers(-127, 128, (4, dim - 1))], 1) * 2.0 ** rng.integers(-10, 10, (4, 1)),
            np.full((2, dim), 127.0) * np.array([[1.0], [-1.0]])]
    rows = np.concatenate(rows).astype(np.float32)                # rows 24..29: max |v| = 127 2^j, so r = 0 exactly
    rows[0, 0] = 1e-39                                          # a subnormal-scale row
    s, codes, rho = TC.quantize(rows)
    for i, v in enumerate(rows):
        # s = max |v| / 127 rounded once; the codes round v / s, clamped; rho = v - s c is exact in fp64
        assert s[i] == TC.f32(F(float(np.max(np.abs(v)))) / 127)
        if s[i] > 0:
            assert np.all(np.abs(codes[i].astype(np.int32)) <= 127)
            assert np.all(codes[i] == np.clip(np.rint(v / s[i]), -127, 127))
        for j in rng.integers(0, dim, 4):
            assert F(float(rho[i, j])) == TC.fr(v[j]) - TC.fr(s[i]) * int(codes[i, j])
        # r and n, rounded up from the fp64 sums as tc_quantize does, bound ||rho|| and ||v|| within 2^-20
        r = np.float32(TC.f32(F(math.sqrt(float(np.dot(rho[i], rho[i])))) * (1 + F(1, 2 ** 40)), "ru"))
        n = np.float32(TC.f32(F(math.sqrt(float(np.dot(v.astype(np.float64), v.astype(np.float64))))) * (1 + F(1, 2 ** 40)), "ru"))
        assert TC.check_norm_bound(r, rho[i]) or (r == 0 and not rho[i].any())
        assert TC.check_norm_bound(n, v.astype(np.float64))
    assert not rho[24:30].any()                                 # integer rows with max |v| = 127 2^j quantise exactly


def random_case(rng, kind):
    """(R, P, Z, ka, kb, b0, b1) of one (query, block) pair and a few rows inside the block's ranges (u, rho, nu, w)"""
    e = lambda lo, hi: np.float32(10.0 ** rng.uniform(lo, hi))
    u_hi = e(-3, 3)
    u_lo = np.float32(u_hi * (10.0 ** -rng.uniform(0, 0.01)))
    rho_hi, nu_hi = e(-4, -1), e(0, 2)
    ka, kb = np.float32(1.0 + rng.uniform(0, 0.2)), np.float32(rng.uniform(1e-6, 0.2))
    P, Z = e(-2, 4), np.float32(0.0)
    w_lo = w_hi = np.float32(0.0)
    R = np.float32(rng.choice([-1, 1]) * 10.0 ** rng.uniform(-4, 4))
    if kind in ("l2", "zw", "spread", "mag"):
        Z = e(-2, 4)
        w_hi = e(-2, 6)
        w_lo = np.float32(w_hi * (10.0 ** -rng.uniform(0, 0.01)))
    if kind == "spread":                      # u_lo far below u_hi (a block holding 1e-30 and 1e30 scales)
        u_lo = np.float32(u_hi * 2.0 ** -rng.uniform(20, 60))
        w_lo = np.float32(w_hi * 2.0 ** -rng.uniform(20, 60))
    if kind == "mag":                         # mag near 2^30: the integer clamp and the slack at their largest
        R = np.float32(rng.choice([-1, 1]) * 2.0 ** rng.uniform(28, 31) / float(u_hi))
    if kind == "zw":                          # Z w near fp32's overflow
        w_hi = np.float32(min(3.0e38 / float(Z) * rng.uniform(0.5, 1.2), 3.4e38))
        w_lo = np.float32(w_hi * 0.999)
    if kind == "near":                        # T_B near an integer: the floor and the +1 decide
        R = np.float32(rng.uniform(-3000, 3000))
        u_lo = u_hi = np.float32(1.0)
        P = np.float32(rng.uniform(0, 2))
    if kind == "inf":
        R = np.float32(rng.choice([np.inf, -np.inf, np.nan]))
    b0 = np.array([u_lo, u_hi, rho_hi, nu_hi], np.float32)
    b1 = np.array([w_lo, w_hi, 0.0, 0.0], np.float32)
    rows = [(u_lo, rho_hi, nu_hi, w_lo), (u_hi, rho_hi, nu_hi, w_lo)]
    for _ in range(3):
        t = rng.uniform(0, 1)
        rows.append((np.float32(u_lo + t * (u_hi - u_lo)), np.float32(rho_hi * rng.uniform(0, 1)), np.float32(nu_hi * rng.uniform(0, 1)),
                     np.float32(w_lo + rng.uniform(0, 1) * (w_hi - w_lo))))
    return (R, P, Z, ka, kb, b0, b1), rows


@pytest.mark.parametrize("kind", ["ip", "l2", "spread", "mag", "zw", "near", "inf"])
def test_block_threshold_never_above_row_thresholds(kind):
    rng = np.random.default_rng(hash(kind) % 2 ** 32)
    for _ in range(300):
        (R, P, Z, ka, kb, b0, b1), rows = random_case(rng, kind)
        thr = TC.block_threshold(R, P, Z, ka, kb, b0, b1)
        if not np.isfinite(R):
            assert thr == (TC.PASS_NONE if R == -np.inf else TC.PASS_ALL), (R, thr)
            continue
        if not np.isfinite(TC.mul(Z, b1[1])) and thr == TC.PASS_NONE:
            continue                          # Z w_hi beyond fp32 while the others stay finite: T_B is beyond 2^25 too
        tb = TC.block_threshold_exact(R, P, Z, ka, kb, b0, b1)
        assert TC.sound(thr, tb), (kind, R, P, Z, ka, kb, b0, b1, thr, float(tb))
        for (u, rho, nu, w) in rows:
            t = TC.row_threshold(R, P, Z, ka, kb, u, rho, nu, w)
            assert tb <= t
            assert TC.sound(thr, t), (kind, thr, float(t))
        # the threshold is not vacuous: within the slack of T_B
        if abs(tb) < 2 ** 29:
            mag = abs(TC.fr(R)) * TC.fr(b0[1]) + TC.fr(P) * (TC.fr(ka) * TC.fr(b0[2]) + TC.fr(kb) * TC.fr(b0[3])) + TC.fr(Z) * TC.fr(b1[1])
            assert thr >= math.floor(tb - mag * F(1, 2 ** 17) - 2), (kind, thr, float(tb))


def test_block_threshold_flags():
    b0 = np.zeros(4, np.float32)
    assert TC.block_threshold(1.0, 1.0, 0.0, 1.0, 1.0, b0, np.array([0, 0, 1, 0], np.float32)) == TC.PASS_ALL
    assert TC.block_threshold(-1e30, 1.0, 0.0, 1.0, 1.0, b0, np.array([0, 0, -1, 0], np.float32)) == TC.PASS_NONE

