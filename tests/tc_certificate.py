"""An exact host restatement of the int8 filter's certificate (reindexer_b200/csrc/knn_tc.cuh, header comment and tc_block_threshold).

numpy for what is exact in fp32 / fp64 as written, fractions.Fraction where exactness matters: the quantiser of tc_quantize (s, codes,
r, n), the exact code dot product I, the per-row threshold T(q, v) and the block threshold T_B(q) in real arithmetic, and a float32
emulation of tc_block_threshold in which every operation is rounded once, correctly, from its exact value.  f32() rounds a Fraction to
float32 directly: going through float64 first would round twice."""
from __future__ import annotations

import math
from fractions import Fraction as F

import numpy as np

PASS_ALL, PASS_NONE = -(1 << 30), 1 << 30
I_MAX = 2048 * 127 * 127        # |I| at every dimension the filter accepts
L2, IP, COS = 0, 1, 2
F32_MAX = F(float(np.finfo(np.float32).max))
TINY_NORM = np.float32(2.0 ** -48)  # kTcTinyNorm: a row with a smaller norm passes the block test (fp32 underflow)


def f32(x, mode: str = "rn") -> np.float32:
    """x (a Fraction or anything Fraction takes) rounded to float32: to nearest even ("rn"), down ("rd") or up ("ru")"""
    x = F(x)
    if x == 0:
        return np.float32(0.0)
    neg = x < 0
    a = -x if neg else x
    if mode == "rd" and neg:
        mode = "ru_mag"
    elif mode == "ru" and neg:
        mode = "rd_mag"
    elif mode == "rd":
        mode = "rd_mag"
    elif mode == "ru":
        mode = "ru_mag"
    e = a.numerator.bit_length() - a.denominator.bit_length()  # within one of floor(log2 a)
    while F(2) ** e > a:
        e -= 1
    while F(2) ** (e + 1) <= a:
        e += 1
    if e >= 128:
        r = np.float32(F32_MAX) if mode == "rd_mag" else np.float32(np.inf)
        return -r if neg else r
    q = max(e - 23, -149)           # the unit in the last place (subnormals: 2^-149)
    m = a / F(2) ** q               # a = m ulp
    lo = m.numerator // m.denominator
    rem = m - lo
    if mode == "rd_mag":
        mi = lo
    elif mode == "ru_mag":
        mi = lo + (1 if rem else 0)
    else:
        mi = lo + (1 if rem > F(1, 2) or (rem == F(1, 2) and lo % 2) else 0)
    v = F(mi) * F(2) ** q
    r = np.float32(np.inf) if v > F32_MAX else np.float32(float(v))  # float(v) is exact: v has at most 24 significant bits
    return -r if neg else r


def fr(x) -> F:
    return F(float(x))


def _finite(*xs) -> bool:
    return all(np.isfinite(np.float32(x)) for x in xs)


def mul(a, b):
    if _finite(a, b):
        return f32(fr(a) * fr(b))
    with np.errstate(all="ignore"):
        return np.float32(np.float32(a) * np.float32(b))


def sub(a, b):
    if _finite(a, b):
        return f32(fr(a) - fr(b))
    with np.errstate(all="ignore"):
        return np.float32(np.float32(a) - np.float32(b))


def fma(a, b, c):
    if _finite(a, b, c):
        return f32(fr(a) * fr(b) + fr(c))
    with np.errstate(all="ignore"):
        return np.float32(np.float64(a) * np.float64(b) + np.float64(c))


def block_threshold(R, P, Z, ka, kb, b0, b1, contract: bool = True) -> int:
    """tc_block_threshold in float32, each operation rounded once.  contract: `t - m + Z w_lo` is evaluated as the compiler contracts
    it, fma(Z, w_lo, t - m); otherwise as a product and a sum."""
    if b1[2] != 0:
        return PASS_ALL if b1[2] > 0 else PASS_NONE
    m = mul(P, fma(ka, b0[2], mul(kb, b0[3])))
    nR = np.float32(-np.float32(R))
    t = np.fmin(mul(nR, b0[0]), mul(nR, b0[1]))
    t = fma(Z, b1[0], sub(t, m)) if contract else sub(t, m) + mul(Z, b1[0])
    t = np.float32(t)
    if t == np.inf:
        return PASS_NONE
    mag = fma(abs(np.float32(R)), b0[1], fma(Z, b1[1], m))
    f = sub(t, fma(mag, np.float32(2.0 ** -18), np.float32(1.0)))
    if not f >= -2.0 ** 30:
        return PASS_ALL
    return PASS_NONE if f > 2.0 ** 30 else int(math.floor(float(f)))


def row_threshold(R, P, Z, ka, kb, u, rho, nu, w) -> F:
    """T(q, v) = -R u - P (ka rho + kb nu) + Z w in real arithmetic (finite arguments)"""
    return -fr(R) * fr(u) - fr(P) * (fr(ka) * fr(rho) + fr(kb) * fr(nu)) + fr(Z) * fr(w)


def block_threshold_exact(R, P, Z, ka, kb, b0, b1) -> F:
    """T_B(q) = min(-R u_lo, -R u_hi) - P (ka rho_hi + kb nu_hi) + Z w_lo in real arithmetic (finite arguments)"""
    return min(-fr(R) * fr(b0[0]), -fr(R) * fr(b0[1])) - fr(P) * (fr(ka) * fr(b0[2]) + fr(kb) * fr(b0[3])) + fr(Z) * fr(b1[0])


def sound(thr: int, t_exact) -> bool:
    """whether every integer I in [-I_MAX, I_MAX] with I >= t_exact passes I >= thr"""
    if isinstance(t_exact, float) and math.isnan(t_exact):
        return thr <= -I_MAX
    if t_exact == math.inf:
        return True
    if t_exact == -math.inf:
        return thr <= -I_MAX
    c = math.ceil(t_exact)
    return thr <= max(c, -I_MAX) or c > I_MAX


# ---- the quantiser -----------------------------------------------------------------------------------------------------------
def quantize(v: np.ndarray):
    """tc_quantize of fp32 rows [n, dim]: (s [n] fp32, codes [n, dim] int8, rho [n, dim] fp64, exact as a difference)"""
    v = np.ascontiguousarray(v, np.float32)
    with np.errstate(all="ignore"):
        mx = np.max(np.abs(v), axis=1) if v.shape[1] else np.zeros(len(v), np.float32)
        s = (mx / np.float32(127.0)).astype(np.float32)
        c = np.where(s[:, None] > 0, np.clip(np.rint(v / s[:, None]), -127, 127), 0).astype(np.float32)
        rho = v.astype(np.float64) - s[:, None].astype(np.float64) * c.astype(np.float64)
        return s, c.astype(np.int8), rho


def exact_sumsq(x: np.ndarray) -> F:
    return sum((F(float(t)) ** 2 for t in x), F(0))


def check_norm_bound(bound: np.float32, x: np.ndarray, rel: float = 2.0 ** -20) -> bool:
    """||x|| <= bound <= ||x|| (1 + rel) + 2^-149 (one subnormal step: a bound rounded up to fp32), decided exactly (fp64 first,
    Fractions where fp64 cannot tell)"""
    b2 = float(bound) ** 2                           # exact: 24-bit significand
    t2 = max(float(bound) - 2.0 ** -149, 0.0) ** 2   # exact as well
    s64 = float(np.dot(x, x))
    err = (len(x) + 2) * 2.0 ** -52 * s64 + 1e-300
    if b2 >= s64 + err and t2 <= (s64 - err) * (1 + rel) ** 2:
        return True
    s = exact_sumsq(x)
    return fr(bound) ** 2 >= s and max(fr(bound) - F(1, 2 ** 149), F(0)) ** 2 <= s * F(1 + rel) ** 2


def check_norm_bounds(bounds: np.ndarray, X: np.ndarray, rel: float = 2.0 ** -20) -> bool:
    """check_norm_bound for every row of X, fp64 first for all of them at once"""
    b = bounds.astype(np.float64)
    s64 = np.einsum("ij,ij->i", X, X)
    err = (X.shape[1] + 2) * 2.0 ** -52 * s64 + 1e-300
    t = np.maximum(b - 2.0 ** -149, 0.0)
    ok = (b * b >= s64 + err) & (t * t <= (s64 - err) * (1 + rel) ** 2)
    return all(check_norm_bound(bounds[i], X[i], rel) for i in np.nonzero(~ok)[0])


def integer_dots(qcodes: np.ndarray, rcodes: np.ndarray) -> np.ndarray:
    """I = codes of the queries x codes of the rows, exact: fp64 products and sums of integers below 2^53"""
    return (qcodes.astype(np.float64) @ rcodes.astype(np.float64).T).astype(np.int64)


def l2eps(dim: int) -> np.float32:
    return np.float32(np.float32(1e-5) + np.float32(dim + 1) * np.float32(2.0 ** -23))


def make_pr(metric, tau, qc, eps):
    """tc_make_pr in numpy float32 (products and differences correctly rounded, contracted as the device does not matter here: this
    only ranks rows by margin)"""
    with np.errstate(all="ignore"):
        p = np.float32(qc[2] * qc[3])
        if metric != L2:
            return p, np.float32(np.float32(tau) * qc[3])
        return p, np.float32(np.float32(0.5) * (np.float32(tau) - (np.float32(1) - eps) * qc[2] * qc[2]) * qc[3])


def row_factors(rowc: np.ndarray, metric: int, one_minus_eps: np.float32):
    """(u, rho, nu, w) of every row in fp64 (ranking only; block_consts_exact decides exactly)"""
    s, r, n, c = (rowc[:, i].astype(np.float64) for i in range(4))
    with np.errstate(all="ignore"):
        S = s * c
        u, rho, nu = 1.0 / S, r / s, n / s
        w = (n * n) * float(one_minus_eps) / (2.0 * S) if metric == L2 else np.zeros_like(S)
    return u, rho, nu, w


def block_consts_exact(rc, metric: int, one_minus_eps: np.float32):
    """one live row's exact factors and whether it forces pass-all (tc_block_consts: S <= 0, a non-finite factor or quotient, or a
    norm below TINY_NORM): (bad, u, rho, nu, w) as Fractions"""
    s, r, n, c = (np.float32(x) for x in rc)
    if not (np.isfinite(s) and np.isfinite(c) and np.isfinite(r) and np.isfinite(n)):
        return True, None, None, None, None
    S = fr(s) * fr(c)
    if not S > 0 or n < TINY_NORM:
        return True, None, None, None, None
    u, rho, nu = 1 / S, fr(r) / fr(s), fr(n) / fr(s)
    w = fr(n) ** 2 * fr(one_minus_eps) / (2 * S) if metric == L2 else F(0)
    bad = (not np.isfinite(f32(u, "ru")) or not np.isfinite(f32(rho, "ru")) or not np.isfinite(f32(nu, "ru"))
           or not np.isfinite(f32(w, "ru")) or f32(u, "rd") == 0)
    return bad, u, rho, nu, w
