"""GPU tests of the int8 filter's certificate, pair by pair (rxgpu_tc_audit: the shipped __device__ functions, read back).

For every metric the per-row constants are checked against the host restatement of tc_quantize (tests/tc_certificate.py), the slot
map and every block's constants against exact Fractions over its live rows, and the two tests a row must pass -- the consumers'
integer block test I >= block_thr and the bookkeeper's !(d~ - err > tau) -- for every live (query, row) pair whose exact-scan distance
is at or below tau, with tau put exactly on a chosen row's distance: near and far neighbours, the rows whose certificate is tightest,
random rows and the special thresholds.  The same thresholds then go through real range batches in every cluster shape, which must
equal the exact scan byte for byte.  All of it again after swap-removes, an in-place rewrite, unsorted appends, a dead block and the
re-sort they trigger."""

import numpy as np
import pytest

import reindexer_b200 as rx
import tc_certificate as TC
from oracle import oracle as O

pytestmark = pytest.mark.gpu

METRICS = [rx.L2, rx.IP, rx.COS]
DEAD = 0xFFFFFFFF
F32_MAX = np.float32(np.finfo(np.float32).max)
SPECIAL_TAUS = [np.inf, -np.inf, np.nan, 0.0, -0.0, F32_MAX]


class Index:
    """a brute-force index and the row order it keeps (swap-removes move the last row into the hole)"""

    def __init__(self, metric, rows, extra=8192):
        self.metric, self.dim = metric, rows.shape[1]
        self.gpu = rx.GpuBruteforceSearch(metric, self.dim, len(rows) + extra)
        self.rows = np.array(rows, np.float32)
        self.labels = O.row_labels(len(rows))
        self.next = len(rows)
        self.gpu.add_points(self.labels, self.rows)

    def remove(self, labels):
        for lab in labels:
            i = int(np.nonzero(self.labels == lab)[0][0])
            self.gpu.remove_point(int(lab))
            self.rows[i], self.labels[i] = self.rows[-1], self.labels[-1]
            self.rows, self.labels = self.rows[:-1], self.labels[:-1]

    def rewrite(self, i, vec):
        self.gpu.add_points(self.labels[i:i + 1], vec[None].astype(np.float32))
        self.rows[i] = vec

    def append(self, vecs):
        labs = O.row_labels(len(vecs), self.next)
        self.next += len(vecs)
        self.gpu.add_points(labs, vecs.astype(np.float32))
        self.rows = np.concatenate([self.rows, vecs.astype(np.float32)])
        self.labels = np.concatenate([self.labels, labs])
        return labs

    def exact_dists(self, queries):
        """the exact scan's fp32 distance of every (query, row) pair (filter off, radius +inf); NaN where it reports none"""
        self.gpu.set_tensor_core_filter(2)
        d, l, c = self.gpu.search_range_batch(queries, np.inf, len(self.rows))
        order = np.argsort(self.labels)
        out = np.full((len(queries), len(self.rows)), np.nan, np.float32)
        for q in range(len(queries)):
            rows = order[np.searchsorted(self.labels[order], l[q, :c[q]])]
            out[q, rows] = d[q, :c[q]]
        return out


def base_queries(metric, rows, dim, seed, extra=()):
    q = O.synth_matrix(seed, 6, dim)
    q[1] = rows[len(rows) // 3]                      # a row itself
    q[2] = 0.0                                       # a zero query (s_q = 0)
    q[3] = q[0] * np.float32(1e-40)                  # subnormal s_q: 1 / s_q = inf
    q[4, 0] = np.float32(50.0) * np.abs(q[4]).max()  # one large component: a high residual that inflates (a*, b*) of its block
    q = np.concatenate([q, np.asarray(extra, np.float32).reshape(-1, dim)]).astype(np.float32)
    if metric == rx.COS:
        q = np.stack([O.normalize_copy(x)[0] if np.abs(x).max() > 1e-30 else x for x in q])  # the zero and subnormal queries stay
    return q


def check_constants(ix, au):
    """s_v, codes, r_v, n_v and c_v of every live slot against the restatement; the slot map; dead slots"""
    slot_row, rowc = au["slot_row"], au["rowc"]
    live = slot_row != DEAD
    assert np.array_equal(np.sort(slot_row[live]), np.arange(len(ix.rows))), "live slots are a bijection onto the rows"
    assert not rowc[~live].any(), "dead slots have zero constants"
    rows = ix.rows[slot_row[live]]
    s, codes, rho = TC.quantize(rows)
    rc = rowc[live]
    fin = np.isfinite(rows).all(axis=1)
    assert np.array_equal(rc[fin, 0].view(np.uint32), s[fin].view(np.uint32)), "s_v"
    assert np.array_equal(au["row_codes"][live][fin], codes[fin]), "codes"
    assert TC.check_norm_bounds(rc[fin, 1], rho[fin]), "r_v"
    assert TC.check_norm_bounds(rc[fin, 2], rows[fin].astype(np.float64)), "n_v"
    if ix.metric != rx.COS:
        assert (rc[:, 3] == 1.0).all(), "c_v = 1"
    else:  # the exact scan's coefficient: 1 / ||v|| (to its fp32 sum), or 1 in the 1e-5 shortcut window and for a row whose fp32
        # sum of squares underflows or overflows
        nn = np.einsum("ij,ij->i", rows[fin].astype(np.float64), rows[fin].astype(np.float64))
        c = rc[fin, 3].astype(np.float64)
        ok = (np.abs(c * np.sqrt(nn) - 1.0) <= 2.0 ** -18) | ((c == 1.0) & (np.abs(nn - 1.0) <= 1.1e-5))
        ok |= (nn < 1e-36) | ((nn > 3e38) & ((c == 0.0) | (c == 1.0)))  # the fp32 sum of squares is subnormal or overflows
        assert ok.all(), np.nonzero(~ok)[0][:5]


def check_sorted(ix, au):
    """after a full build: S_v = s_v c_v (fp32) non-increasing within each sort bucket (L2: the top mantissa bits of n_v^2)"""
    rc = au["rowc"][: len(ix.rows)]
    with np.errstate(invalid="ignore"):
        S = (rc[:, 0] * rc[:, 3]).astype(np.float32)
    ok = np.isfinite(S)
    S = S[ok]
    if ix.metric != rx.L2:
        assert (np.diff(S.astype(np.float64)) <= 0).all()
        return
    nn = rc[ok, 2].astype(np.float64) ** 2
    bucket = lambda x: np.asarray(x, np.float32).view(np.uint32) >> 13
    b_lo, b_hi = bucket(nn * (1 - 2.0 ** -16)), bucket(nn * (1 + 2.0 ** -16))
    up = np.nonzero(np.diff(S.astype(np.float64)) > 0)[0]
    assert all(b_hi[i] < b_lo[i + 1] or b_lo[i] != b_hi[i] or b_lo[i + 1] != b_hi[i + 1] for i in up), up[:5]


def check_blocks(ix, au):
    """every block's constants against exact Fractions over its live rows: bounds, one-ulp tightness and the flags (fp64 screens the
    rows; Fractions decide every row fp64 cannot, and the extreme row of every bound)"""
    slot_row, rowc, blockc = au["slot_row"], au["rowc"], au["blockc"]
    ome = np.float32(1) - TC.l2eps(ix.dim) if ix.metric == rx.L2 else np.float32(1)
    up = lambda x: TC.fr(np.nextafter(np.float32(x), np.float32(np.inf)))
    dn = lambda x: TC.fr(np.nextafter(np.float32(x), np.float32(-np.inf)))
    for b in range(len(blockc)):
        slots = np.array([s for s in range(64 * b, min(64 * b + 64, len(slot_row))) if slot_row[s] != DEAD], np.int64)
        b0, b1 = blockc[b, :4], blockc[b, 4:]
        if len(slots) == 0:
            assert b1[2] == -1 and not b0.any(), ("a block with no live slot passes none", b)
            continue
        rc = rowc[slots].astype(np.float64)
        with np.errstate(all="ignore"):
            S = rc[:, 0] * rc[:, 3]
            vals = np.stack(TC.row_factors(rowc[slots], ix.metric, ome), 1)
        maybe = ~np.isfinite(rc).all(1) | ~(S > 0) | ~np.isfinite(vals).all(1) | (vals.max(1) > 1e37) | (vals[:, 0] < 1e-43) | (rc[:, 2] < 2.0 ** -40)
        facts = {i: TC.block_consts_exact(rowc[slots[i]], ix.metric, ome) for i in np.nonzero(maybe)[0]}
        bad = any(f[0] for f in facts.values())
        assert b1[2] == (1 if bad else 0), ("flag", b, b1[2], bad)
        if bad:
            continue
        exact = lambda i, k: (facts.get(i) or facts.setdefault(i, TC.block_consts_exact(rowc[slots[i]], ix.metric, ome)))[1 + k]
        if ix.metric != rx.L2:
            assert b1[0] == 0 and b1[1] == 0, ("w = 0 for IP and Cosine", b)
        for k, bound, lower in ((0, b0[0], True), (3, b1[0], True), (0, b0[1], False), (1, b0[2], False), (2, b0[3], False),
                                (3, b1[1], False)):
            if k == 3 and ix.metric != rx.L2:
                continue
            v = vals[:, k]
            ext = int(np.argmin(v) if lower else np.argmax(v))
            close = np.nonzero(v <= float(bound) * (1 + 2.0 ** -40) if lower else v >= float(bound) * (1 - 2.0 ** -40))[0]
            assert (v >= float(bound) * (1 - 2.0 ** -40) if lower else v <= float(bound) * (1 + 2.0 ** -40)).all(), (b, k, bound)
            for i in set(close.tolist()) | {ext}:
                e = exact(i, k)
                assert (TC.fr(bound) <= e) if lower else (e <= TC.fr(bound)), ("bound", b, k, bound, float(e))
            e = exact(ext, k)
            assert (e <= up(bound)) if lower else (dn(bound) <= e), ("one ulp of the extreme row", b, k, bound, float(e))


def choose_taus(ix, au, qb, d, I):
    """(base query, tau) pairs: tau = the exact distance of the 1st, 2nd, 10th, 100th and 1000th neighbour, of the 20 rows whose
    certificate is tightest at their own distance, of a few random rows, and the special thresholds"""
    rng = np.random.default_rng(len(ix.rows))
    slot_row, rowc = au["slot_row"], au["rowc"]
    live = np.nonzero(slot_row != DEAD)[0]
    ome = np.float32(1) - TC.l2eps(ix.dim)
    u, rho, nu, w = TC.row_factors(rowc[live], ix.metric, ome)
    ka, kb = (float(x) for x in au["kab"].max(axis=0))
    out = []
    for q in range(len(qb)):
        dq = d[q, slot_row[live]]
        fin = np.nonzero(np.isfinite(dq))[0]
        if len(fin) == 0:
            out += [(q, t) for t in SPECIAL_TAUS]
            continue
        order = fin[np.argsort(dq[fin], kind="stable")]
        picks = [order[r] for r in (0, 1, 9, 99, 999) if r < len(order)]
        qc = au["qc"][q]
        with np.errstate(all="ignore"):
            P, R = (np.float64(x) for x in TC.make_pr(ix.metric, dq[fin], qc, TC.l2eps(ix.dim)))
            Z = float(qc[3]) if ix.metric == rx.L2 else 0.0
            T = -R * u[fin] - P * (ka * rho[fin] + kb * nu[fin]) + Z * w[fin]
            mag = np.abs(R) * u[fin] + P * (ka * rho[fin] + kb * nu[fin]) + Z * w[fin] + 1.0
            margin = (I[q, live[fin]] - T) / mag
        margin = np.where(np.isfinite(margin), margin, np.inf)
        picks += list(fin[np.argsort(margin, kind="stable")[:20]])
        picks += list(rng.choice(fin, size=min(5, len(fin)), replace=False))
        out += [(q, dq[i]) for i in picks] + [(q, t) for t in SPECIAL_TAUS]
    return out


def is_special(t):
    return not np.isfinite(t) or t == 0 or t == F32_MAX


def check_soundness(ix, qb, taus, d, I, query_block):
    """every live pair with d_scan <= tau passes both tests, with the hook's fp32 values"""
    qs = np.stack([qb[q] for q, _ in taus])
    tv = np.array([t for _, t in taus], np.float32)
    au = ix.gpu.tc_audit(qs, tv, query_block)
    slot_row = au["slot_row"]
    live = np.nonzero(slot_row != DEAD)[0]
    rows = slot_row[live]
    for j, (q, t) in enumerate(taus):
        assert np.array_equal(au["query_codes"][j], au["query_codes"][[k for k, (p, _) in enumerate(taus) if p == q][0]])
        with np.errstate(invalid="ignore"):
            need = d[q, rows] <= tv[j]
        Ij = I[q, live]
        thr = au["block_thr"][j, live // 64]
        bad = need & (Ij < thr)
        assert not bad.any(), ("block test", j, float(tv[j]), live[bad][:5], Ij[bad][:5], thr[bad][:5])
        de = au["row_bound"][j, live]
        with np.errstate(invalid="ignore", over="ignore"):
            rej = (de[:, 0] - de[:, 1]) > tv[j]
        assert not (need & rej).any(), ("row bound", j, float(tv[j]), live[need & rej][:5])
    check_threshold_arithmetic(ix, au, tv, query_block)
    return au


def check_threshold_arithmetic(ix, au, tv, query_block, pairs=300):
    """block_thr is bit for bit the float32 arithmetic whose soundness test_tc_certificate_pin.py proves (tc_make_pr, then
    tc_block_threshold with every operation rounded once), on random (query, block) pairs and every query's first block"""
    rng = np.random.default_rng(len(tv))
    nb = au["block_thr"].shape[1]
    eps = TC.l2eps(ix.dim)
    js = np.concatenate([np.arange(len(tv)), rng.integers(0, len(tv), pairs)])
    bs = np.concatenate([np.zeros(len(tv), np.int64), rng.integers(0, nb, pairs)])
    for j, b in zip(js, bs):
        qc, (ka, kb) = au["qc"][j], au["kab"][j // query_block]
        b0, b1 = au["blockc"][b, :4], au["blockc"][b, 4:]
        P = TC.mul(qc[2], qc[3])
        if ix.metric != rx.L2:
            Rs, Z = [TC.mul(tv[j], qc[3])], np.float32(0)
        else:  # tau - (1 - eps) n_q n_q, contracted into one fma or not
            ome, Z = np.float32(np.float32(1) - eps), qc[3]
            a = TC.mul(ome, qc[2])
            Rs = [TC.mul(TC.mul(np.float32(0.5), d), qc[3]) for d in (TC.fma(-a, qc[2], tv[j]), TC.sub(tv[j], TC.mul(a, qc[2])))]
        want = [TC.block_threshold(R, P, Z, ka, kb, b0, b1) for R in Rs]
        assert au["block_thr"][j, b] in want, (j, b, au["block_thr"][j, b], want)


def range_sweep(ix, qb, taus, d):
    """the chosen thresholds through real range batches: radius = nextafter(d*, +inf) and d*; modes 1, 3, 4, 5 give the exact scan's
    bytes, and the chosen row is present exactly when d_scan < radius"""
    picks = [(q, t) for q, t in taus if not is_special(t)]
    qs = np.stack([qb[q] for q, _ in picks] * 2)
    rad = np.array([np.nextafter(np.float32(t), np.float32(np.inf)) for _, t in picks] + [t for _, t in picks], np.float32)
    max_out = 1536
    ix.gpu.set_tensor_core_filter(2)
    ref = ix.gpu.search_range_batch(qs, rad, max_out)
    for mode in (1, 3, 4, 5):
        ix.gpu.set_tensor_core_filter(mode)
        got = ix.gpu.search_range_batch(qs, rad, max_out)
        assert rx.last_search_stats()["tc_used"] == 1
        for a, b in zip(ref, got):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), mode
    dl, ll, cl = ref
    order = np.argsort(ix.labels)
    for j, (q, t) in enumerate(picks * 2):
        if cl[j] > max_out:
            continue
        members = set(order[np.searchsorted(ix.labels[order], ll[j, :cl[j]])].tolist())
        want = set(np.nonzero(d[q] < rad[j])[0].tolist())
        assert members == want, (j, float(rad[j]), len(members), len(want))


def check_state(ix, qb, sorted_=False, query_block=128, sweep=True):
    au = ix.gpu.tc_audit(qb, np.zeros(len(qb), np.float32), query_block)
    check_constants(ix, au)
    if sorted_:
        check_sorted(ix, au)
    check_blocks(ix, au)
    d = ix.exact_dists(qb)
    codes = au["row_codes"].copy()
    codes[au["slot_row"] == DEAD] = 0
    I = TC.integer_dots(au["query_codes"], codes)
    taus = choose_taus(ix, au, qb, d, I)
    check_soundness(ix, qb, taus, d, I, query_block)
    if sweep:
        range_sweep(ix, qb, taus, d)


@pytest.mark.parametrize("metric", METRICS)
def test_certificate_through_mutations(metric):
    """synth rows at 768 dims: the full build, then each incremental state, then the re-sort they trigger"""
    rng = np.random.default_rng(7 + metric)
    n, dim = 16000, 768
    rows = O.synth_matrix(0xCE70, n, dim)
    ix = Index(metric, rows)
    qb = base_queries(metric, rows, dim, 0xCE71)
    check_state(ix, qb, sorted_=True)
    ix.remove(rng.choice(ix.labels[: n // 2], 30, replace=False))                  # swap-removes
    check_state(ix, qb)
    big = ix.rows[n // 4] * np.float32(1e6)                                         # a row 1e6x larger, rewritten in a sorted block
    ix.rewrite(n // 4, big)
    check_state(ix, qb, sweep=False)
    labs = ix.append(O.synth_matrix(0xCE72, 320, dim) * np.float32(10.0) ** rng.uniform(-3, 3, (320, 1)).astype(np.float32))
    check_state(ix, qb, sweep=False)                                                # unsorted appends
    ix.remove(labs[::-1][:200])                                                     # the last rows: their slots die, whole blocks too
    au = ix.gpu.tc_audit(qb, np.zeros(len(qb), np.float32))
    assert (au["blockc"][:, 6] == -1).any(), "a block with every slot dead"
    check_state(ix, qb)
    ix.remove(rng.choice(ix.labels[:-1], 2500, replace=False))                      # beyond 1 / kShadowResortDiv: the re-sort
    check_state(ix, qb, sorted_=True)
    ix.gpu.close()


@pytest.mark.parametrize("dim", [1, 127, 128, 129, 2047, 2048])
@pytest.mark.parametrize("metric", METRICS)
def test_certificate_at_every_dim_edge(metric, dim):
    n = 3000 if dim >= 2047 else 6000
    rows = O.synth_matrix(0xCE73 + dim, n, dim)
    ix = Index(metric, rows)
    check_state(ix, base_queries(metric, rows, dim, 0xCE74 + dim), sorted_=True, query_block=64 if dim % 2 else 128)
    ix.gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_certificate_exact_codes_and_full_scale(metric):
    """integer rows with max |v| = 127 2^j (r_v = 0: the bound is only the fp32 budget) at 256 dims, and all-+-127 rows with queries
    of matching sign at 2048 dims (|I| = 2048 127^2 > 2^24: float(I) rounds)"""
    rng = np.random.default_rng(3 + metric)
    n, dim = 4000, 256
    ints = rng.integers(-127, 128, (n, dim)).astype(np.float32)
    ints[:, 0] = 127.0
    rows = ints * np.float32(2.0) ** rng.integers(-6, 6, (n, 1)).astype(np.float32)
    ix = Index(metric, rows)
    check_state(ix, base_queries(metric, rows, dim, 0xCE75, extra=rows[:3] * np.float32(3.0)), sorted_=True)
    ix.gpu.close()
    n, dim = 1500, 2048
    sign = np.where(rng.random((n, 1)) < 0.5, -1.0, 1.0)
    rows = (np.where(rng.random((n, dim)) < 0.97, 127.0, -127.0) * sign * rng.integers(1, 4, (n, 1))).astype(np.float32)
    ix = Index(metric, rows)
    extra = np.stack([np.full(dim, 127.0), np.full(dim, -127.0), rows[0], -rows[1]]).astype(np.float32)
    check_state(ix, base_queries(metric, rows, dim, 0xCE76, extra=extra), sorted_=True)
    ix.gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_certificate_on_extreme_rows(metric):
    """scales from 1e-30 to 1e30 in one (appended, unsorted) block; zero, non-finite and subnormal-scale rows; L2 rows with a common
    offset and squared norms near fp32's maximum; Cosine rows at the 1e-5 edge of the norm shortcut"""
    rng = np.random.default_rng(13 + metric)
    n, dim = 6000, 96
    rows = O.synth_matrix(0xCE77, n, dim)
    rows[rng.choice(n, 40, replace=False)] = 0.0
    rows[rng.choice(n, 8, replace=False), rng.integers(0, dim, 8)] = np.inf
    rows[rng.choice(n, 8, replace=False), rng.integers(0, dim, 8)] = np.nan
    rows[rng.choice(n, 16, replace=False)] *= np.float32(1e-42)                 # s = 0: below 127 subnormal steps
    if metric == rx.L2:
        rows[:500] += np.float32(1000.0)
        rows[500:520] = (rows[500:520] / np.abs(rows[500:520]).max() * np.float32(1.7e18)).astype(np.float32)
    if metric == rx.COS:
        r = rows[600:1200].astype(np.float64)
        r /= np.maximum(np.linalg.norm(r, axis=1, keepdims=True), 1e-300)  # the zero rows among them stay zero
        rows[600:1200] = (r * np.sqrt(1.0 + rng.choice([-1.2e-5, -0.9e-5, 0.9e-5, 1.2e-5], (600, 1)))).astype(np.float32)
    ix = Index(metric, rows)
    qb = base_queries(metric, rows, dim, 0xCE78)
    check_state(ix, qb, sorted_=True)
    spread = O.synth_matrix(0xCE79, 128, dim) * np.float32(10.0) ** np.linspace(-30, 30, 128).astype(np.float32)[:, None]
    ix.append(spread.astype(np.float32))
    check_state(ix, qb)
    ix.gpu.close()


@pytest.mark.parametrize("metric", METRICS)
def test_block_test_is_not_vacuous(metric):
    """synth rows at 768 dims, 2^17 of them so that a sorted block is as narrow as in a real index: with tau on the 1st, 2nd, 10th,
    100th and 1000th neighbour, the block test rejects at least 90 % of the pairs above tau.  A threshold stuck at pass-all would
    make every soundness check above trivially true, and the filter slow."""
    n, dim = 1 << 17, 768
    gpu = rx.GpuBruteforceSearch(metric, dim, n)
    gpu.append_synth(0xCE7A, 0, n)                                  # row r has the label r << 32
    qb = O.synth_matrix(0xCE7B, 2, dim)
    if metric == rx.COS:
        qb = np.stack([O.normalize_copy(x)[0] for x in qb])
    gpu.set_tensor_core_filter(2)
    dl, ll, cl = gpu.search_range_batch(qb, np.inf, n)
    d = np.full((len(qb), n), np.nan, np.float32)
    taus = []
    for q in range(len(qb)):
        d[q, (ll[q, :cl[q]] >> np.uint64(32)).astype(np.int64)] = dl[q, :cl[q]]
        srt = np.sort(d[q][np.isfinite(d[q])])
        taus += [(q, srt[r]) for r in (0, 1, 9, 99, 999)]
    au = gpu.tc_audit(np.stack([qb[q] for q, _ in taus]), np.array([t for _, t in taus], np.float32), 128, row_bound=False)
    live = np.nonzero(au["slot_row"] != DEAD)[0]
    rows = au["slot_row"][live]
    # fp32 sums of 768 products of codes (each at most 127^2 in magnitude) stay below 2^24: exact
    qcodes = au["query_codes"].astype(np.float32)
    I = np.concatenate([qcodes @ au["row_codes"][live[i:i + 16384]].astype(np.float32).T for i in range(0, len(live), 16384)], 1)
    far = rejected = 0
    for j, (q, t) in enumerate(taus):
        with np.errstate(invalid="ignore"):
            above = d[q, rows] > t
        far += int(above.sum())
        rejected += int((above & (I[j] < au["block_thr"][j, live // 64])).sum())
    assert far and rejected >= 0.9 * far, (rejected, far)
    gpu.close()
