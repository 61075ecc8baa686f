"""GPU tests of brute-force KNN, range and IVF search against a plain fp64 reference with a certified per-distance error bound, at the
shape boundaries the kernels define.

The exact scan computes every distance the same way (knn_scan.cuh): lane l of a warp runs one sequential fmaf chain over the 4 nch
elements it owns (nch = ceil(dim / 128)), then five xor-butterfly adds combine the lanes.  Each of those 4 nch + 5 roundings is at
most 2^-24 of a partial sum, and every partial sum is at most S = sum |q_i v_i| (IP) or sum (q_i - v_i)^2 (L2; 2 more roundings per
term for q_i - v_i and its square), so the fp32 distance lies within

    b = 2 (4 nch + 8) 2^-24 S      (the factor 2 is slack for the higher-order terms)

of the fp64 one, plus an absolute term for subnormal products.  Cosine multiplies the IP sum by the row's coefficient 1 / ||v||, a
lane-strided sum of ceil(dim / 32) + 5 roundings, __fsqrt_rn, 1 / double and a final fp32 rounding; the coefficient is exactly 1 when
the fp32 sum of squares s has |1 - s| <= 1e-5f (the reference's normalize.cc rule), and where s lies within its own error of that
edge both coefficients are accepted.  The filter (modes 1, 3, 4), the staged thresholds and the IVF list scans re-use this arithmetic,
so every path is held to the same envelope; the filter paths must also stay bit-identical to the exact scan (mode 2).

A dropped, duplicated or mis-padded element of any real size moves a distance far outside b, and a row that a correct fp32 scan
would have ranked ahead of the k-th result (hi < d_k) shows up as missing."""
import math

import numpy as np
import pytest
from test_tc_int8_bound_gpu import adversarial_queries, adversarial_rows

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24      # unit roundoff of fp32
U64 = 2.0 ** -53    # unit roundoff of fp64 (the reference's own error)
TINY = 2.0 ** -149  # smallest fp32 subnormal: the absolute error of an fmaf whose result underflows
NORM_EDGE = float(np.float32(1e-5))  # norm_coef_kernel: |1 - s| <= 1e-5f keeps the coefficient at exactly 1
ERR_PARAMS = 3

# ---------------------------------------------------------------------------------------------------------------- fp64 reference


def _nch(dim):
    return (dim + 127) // 128


def _scan_bound(dim, s):
    """the certified error of the exact scan's fp32 sum over the magnitude sum s (module docstring)"""
    m = 4 * _nch(dim) + 8
    return 2.0 * m * U * s + 2.0 * m * TINY


def norm_coefs(rows):
    """per row: (coefficient allowed by the shortcut, coefficient 1 / ||v|| and its relative error, which ones are allowed)"""
    dim = rows.shape[1]
    s = (rows.astype(np.float64) ** 2).sum(1)
    m = math.ceil(dim / 32) + 5
    s_err = 2.0 * m * U * s + 2.0 * m * TINY + 4.0 * (dim + 2) * U64 * s
    dev = np.abs(1.0 - s)
    zero = s == 0.0
    short_ok = zero | (dev - s_err <= NORM_EDGE)  # the fp32 sum may fall inside the edge
    long_ok = ~zero & (dev + s_err > NORM_EDGE)   # ... or outside it
    with np.errstate(divide="ignore"):
        inv = np.where(zero, 1.0, 1.0 / np.sqrt(np.where(zero, 1.0, s)))
    rel = (m + 4) * U
    return short_ok, long_ok, inv, rel


class Envelope:
    """lo[q, r] <= the library's fp32 distance of (query q, row r) <= hi[q, r], certified; mid = the fp64 distance"""

    def __init__(self, metric, rows, queries, coefs=None, chunk=8192):
        rows = np.asarray(rows, np.float32)
        queries = np.asarray(queries, np.float32).reshape(-1, rows.shape[1])
        # L2: a common shift (the coordinate-wise median, robust to a few huge rows) keeps q.q + v.v - 2 q.v free of cancellation
        mu = np.median(rows, 0).astype(np.float64) if metric == rx.L2 else None
        if metric == rx.COS and coefs is None:
            coefs = norm_coefs(rows)
        parts = []
        for i in range(0, len(rows), chunk):
            part = None if coefs is None else tuple(c[i:i + chunk] if np.ndim(c) else c for c in coefs)
            parts.append(self._block(metric, rows[i:i + chunk], queries, mu, part))
        self.lo, self.hi, self.mid = (np.concatenate([p[j] for p in parts], axis=1) for j in range(3))

    @staticmethod
    def _block(metric, rows, queries, mu, coefs):
        dim = rows.shape[1]
        v64, q64 = rows.astype(np.float64), queries.astype(np.float64)
        if metric == rx.L2:
            v64, q64 = v64 - mu, q64 - mu
            qn, vn = (q64 ** 2).sum(1), (v64 ** 2).sum(1)
            mid = qn[:, None] + vn[None, :] - 2.0 * (q64 @ v64.T)
            ref_err = 8.0 * (dim + 4) * U64 * (qn[:, None] + vn[None, :])
            b = _scan_bound(dim, np.maximum(mid, 0.0) + ref_err) + ref_err
            return mid - b, mid + b, mid
        p = q64 @ v64.T
        s = np.abs(q64) @ np.abs(v64).T
        b_ip = _scan_bound(dim, s) + 4.0 * (dim + 2) * U64 * s
        if metric == rx.IP:
            return -p - b_ip, -p + b_ip, -p
        short_ok, long_ok, inv, rel = coefs
        lo = np.full(p.shape, np.inf)
        hi = np.full(p.shape, -np.inf)
        for ok, c, r in ((short_ok, np.ones_like(inv), 0.0), (long_ok, inv, rel)):
            mid_c = -p * c[None, :]
            bc = c[None, :] * (1 + r) * (b_ip * (1 + U) + np.abs(p) * U) + np.abs(p) * c[None, :] * r
            lo = np.where(ok[None, :], np.minimum(lo, mid_c - bc), lo)
            hi = np.where(ok[None, :], np.maximum(hi, mid_c + bc), hi)
        return lo, hi, np.where(long_ok[None, :], -p * inv[None, :], -p)

    def restrict(self, allowed):
        """only the rows allowed[q, r] exist for query q (IVF: the rows of the probed lists)"""
        self.lo = np.where(allowed, self.lo, np.inf)
        self.hi = np.where(allowed, self.hi, np.inf)
        self.mid = np.where(allowed, self.mid, np.inf)
        self.allowed = allowed
        return self


def label_rows(lab):
    """the envelope row a label names when row r was inserted as O.row_labels: its row id"""
    return (np.asarray(lab, np.uint64) >> np.uint64(32)).astype(np.int64)


def check_knn(env, d, lab, cnt, k, ctx="", row_of=label_rows):
    """distances inside the envelope of the rows their labels name, sorted, min(k, n) results, and no missing row with hi < d_k;
    row_of maps labels to envelope rows (-1: no such row)"""
    nq, n = env.lo.shape
    avail = getattr(env, "allowed", np.ones((nq, n), bool)).sum(1)
    for q in range(nq):
        want = min(k, int(avail[q]))
        assert cnt[q] == want, (ctx, q, int(cnt[q]), want)
        if want == 0:
            continue
        dq = d[q, :want].astype(np.float64)
        rows = row_of(lab[q, :want])
        assert len(np.unique(rows)) == want, (ctx, q, "a row returned twice")
        assert ((rows >= 0) & (rows < n)).all(), (ctx, q, rows)
        assert (np.diff(dq) >= 0).all(), (ctx, q, "not sorted", dq)
        lo, hi = env.lo[q, rows], env.hi[q, rows]
        bad = np.nonzero(~((lo <= dq) & (dq <= hi)))[0]
        assert len(bad) == 0, (ctx, q, "distance outside the fp64 envelope", bad[:5], dq[bad[:5]], env.mid[q, rows[bad[:5]]],
                               hi[bad[:5]] - env.mid[q, rows[bad[:5]]])
        if want < avail[q]:
            missing = np.ones(n, bool)
            missing[rows] = False
            ahead = np.nonzero(missing & (env.hi[q] < dq[-1]))[0]
            assert len(ahead) == 0, (ctx, q, "rows missing from the result", ahead[:5], env.mid[q, ahead[:5]], dq[-1])


def check_range(env, radius, d, lab, cnt, ctx="", row_of=label_rows):
    """every row with hi < radius returned, every returned row lo < radius, distances in the envelope and sorted, totals exact"""
    nq, n = env.lo.shape
    radius = np.broadcast_to(np.asarray(radius, np.float32), (nq,)).astype(np.float64)
    for q in range(nq):
        c = int(cnt[q])
        assert c <= d.shape[1], (ctx, q, c)
        dq = d[q, :c].astype(np.float64)
        rows = row_of(lab[q, :c])
        assert len(np.unique(rows)) == c, (ctx, q, "a row returned twice")
        assert ((rows >= 0) & (rows < n)).all(), (ctx, q, rows)
        assert (np.diff(dq) >= 0).all(), (ctx, q, "not sorted")
        assert ((env.lo[q, rows] <= dq) & (dq <= env.hi[q, rows])).all(), (ctx, q, "distance outside the fp64 envelope")
        assert (dq < radius[q]).all() and (env.lo[q, rows] < radius[q]).all(), (ctx, q, "a row at or above the radius")
        got = np.zeros(n, bool)
        got[rows] = True
        must = np.nonzero((env.hi[q] < radius[q]) & ~got)[0]
        assert len(must) == 0, (ctx, q, "matches missing", must[:5], env.mid[q, must[:5]], radius[q])


def radii_at(env, ranks=(1, 10, 100)):
    """per query: the fp32 value of its j-th best fp64 distance and one ulp above, cycling over the queries"""
    nq, n = env.mid.shape
    srt = np.sort(env.mid, axis=1)
    opts = []
    for j in ranks:
        r = np.float32(srt[:, min(j, n) - 1])
        opts += [r, np.nextafter(r, np.float32(np.inf))]
    return np.array([opts[i % len(opts)][i] for i in range(nq)], np.float32)


# ---------------------------------------------------------------------------------------------------------------- data and searches


def gaussian(seed, n, dim):
    return (np.random.default_rng(seed).standard_normal((n, dim)) * 0.25).astype(np.float32)


def unit(x):
    x = np.asarray(x, np.float64)
    nrm = np.linalg.norm(x, axis=1, keepdims=True)
    return (x / np.where(nrm == 0, 1.0, nrm)).astype(np.float32)


def queries_for(metric, seed, nq, dim):
    q = gaussian(seed, nq, dim)
    return unit(q) if metric == rx.COS else q


def make_index(metric, rows):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], max(len(rows), 1))
    if len(rows):
        gpu.add_points(O.row_labels(len(rows)), rows)
    return gpu


def knn(gpu, queries, k, mode):
    gpu.set_tensor_core_filter(mode)
    out = gpu.search_knn(queries, k)
    return out, rx.last_search_stats()


def assert_identical(a, b, ctx=""):
    (d0, l0, c0), (d1, l1, c1) = a, b
    assert (c0 == c1).all(), ctx
    for q in range(len(c0)):
        m = int(min(c0[q], d0.shape[1]))
        assert (l0[q, :m] == l1[q, :m]).all(), (ctx, q)
        assert (d0[q, :m].view(np.uint32) == d1[q, :m].view(np.uint32)).all(), (ctx, q)


def tc_query_block(nq, dim):
    """the query block tcQueryBlock picks (index.cu), from tc_smem_bytes (knn_tc.cuh)"""
    kchunks = (dim + 127) // 128

    def smem(nqb):
        return 1024 + nqb * kchunks * 128 + 12 * 8192 + 256 + nqb * 40 + 64

    nqb = min(128, (nq + 31) // 32 * 32)
    while nqb >= 32 and smem(nqb) > 227 * 1024:
        nqb -= 32
    blocks = (nq + nqb - 1) // nqb
    return min(nqb, ((nq + blocks - 1) // blocks + 31) // 32 * 32)


def scan_smem_bytes(qt, dim, k1):
    """knn_scan.cuh: staged queries + per-warp key lists, candidate buffers, thresholds and counts"""
    dp = (dim + 127) // 128 * 128
    return qt * dp * 4 + 8 * qt * (k1 + 32) * 8 + 8 * qt * 8 + 8 * qt * 4


METRICS = [rx.L2, rx.IP, rx.COS]
MNAME = {rx.L2: "l2", rx.IP: "ip", rx.COS: "cos"}

# ---------------------------------------------------------------------------------------------------------------- exact scan (mode 2)

# every (RW, CG) variant of launchScanQ at both ends of its nch band where cheap: nch = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 16, 17
SCAN_DIMS = [1, 2, 3, 127, 128, 129, 257, 385, 513, 640, 641, 769, 897, 1025, 1153, 1409, 1536, 2048, 2049]


@pytest.mark.parametrize("dim", SCAN_DIMS)
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_exact_scan_every_variant(metric, dim):
    n, nq, k = 3001, 7, 10  # 3001 rows: not a multiple of RW = 2, 4 or 8
    rows = gaussian(dim * 10 + metric, n, dim)
    queries = queries_for(metric, dim * 10 + metric + 5, nq, dim)
    env = Envelope(metric, rows, queries)
    gpu = make_index(metric, rows)
    outs = []
    for qt in (1, 2, 4):
        gpu.set_query_tile(qt)
        out, st = knn(gpu, queries, k, 2)
        assert st["tc_used"] == 0, st
        assert st["query_tile"] == qt or st["tie_replays"] > 0, st  # a tie replay (one query per scan) reports its own tile
        check_knn(env, *out, k, ctx=(dim, qt))
        outs.append(out)
    for out in outs[1:]:
        assert_identical(outs[0], out, ctx=dim)  # every query tile runs the same per-row arithmetic
    gpu.close()


@pytest.mark.parametrize("dim", [3, 640, 1409, 2049])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_exact_scan_k_rounds(metric, dim):
    # k + 1 > 256 runs ceil((k + 1) / 256) rounds over the rows, each admitting only keys above the previous round's last one
    n, nq = 3001, 5
    rows = gaussian(dim * 11 + metric, n, dim)
    queries = queries_for(metric, dim * 11 + metric + 5, nq, dim)
    env = Envelope(metric, rows, queries)
    gpu = make_index(metric, rows)
    for k in (1, 255, 256, 257, 1000):
        out, st = knn(gpu, queries, k, 2)
        rounds = -(-(k + 1) // 256)
        qt = 4  # scanTopKExact halves the query tile until the shared memory of one round fits
        while qt > 1 and scan_smem_bytes(qt, dim, min(k + 1, 256)) > 100 * 1024:
            qt //= 2
        assert st["tc_used"] == 0 and st["query_tile"] == qt and st["passes"] == -(-nq // qt) * rounds, (k, qt, st)
        check_knn(env, *out, k, ctx=(dim, k))
    gpu.close()


@pytest.mark.parametrize("n", [1, 7, 8, 9])
@pytest.mark.parametrize("dim", [1, 129, 640, 2049])
def test_exact_scan_row_counts(dim, n):
    # fewer rows than one warp step of RW = 8, 4 or 2 rows, and a step exactly filled
    for metric in METRICS:
        rows = gaussian(n * 7 + dim + metric, n, dim)
        queries = queries_for(metric, n * 7 + dim + metric + 1, 6, dim)
        env = Envelope(metric, rows, queries)
        gpu = make_index(metric, rows)
        for qt in (1, 4):
            gpu.set_query_tile(qt)
            for k in (1, 10, 257):
                out, _ = knn(gpu, queries, k, 2)
                check_knn(env, *out, k, ctx=(metric, qt, k))
        gpu.close()


def test_exact_scan_dimension_ceiling():
    """scanTopKExact serves a search while scan_smem_bytes(1, dim, k + 1) <= 100 KB: at k = 10 the largest such dimension must give
    certified results, and one padded step above it must be refused, never answered wrongly"""
    k = 10
    top = max(d for d in range(128, 65537, 128) if scan_smem_bytes(1, d, k + 1) <= 100 * 1024)
    assert scan_smem_bytes(1, top + 1, k + 1) > 100 * 1024
    for metric in METRICS:
        rows = gaussian(top + metric, 300, top)
        queries = queries_for(metric, top + metric + 1, 3, top)
        gpu = make_index(metric, rows)
        out, st = knn(gpu, queries, k, 0)
        assert st["tc_used"] == 0 and st["query_tile"] == 1, st  # 3 queries: the tile shrinks to fit
        check_knn(Envelope(metric, rows, queries), *out, k, ctx=(metric, top))
        gpu.close()
        big = make_index(metric, gaussian(top + 7, 20, top + 1))
        with pytest.raises(rx.RxGpuError) as e:
            big.search_knn(queries_for(metric, 1, 1, top + 1), k)
        assert e.value.code == ERR_PARAMS and "exceeds the fused top-k shared-memory budget" in e.value.what, e.value.what
        big.close()
    assert top == 24832  # the ceiling rxgpu.h documents


# ---------------------------------------------------------------------------------------------------------------- filter, staged, range batch

FILTER_DIMS = [1, 3, 64, 896, 897, 1280, 1281, 1536, 1920, 1921, 2047, 2048]


@pytest.mark.parametrize("dim", FILTER_DIMS)
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_filter_every_query_block(metric, dim):
    """384 queries, a multiple of every query block, so the block tcQueryBlock keeps is the largest that fits: 128 up to 896 dims,
    96 up to 1280, 64 up to 1920 and 32 up to 2048, each run at its largest K"""
    n, nq = 3000, 384
    rows = gaussian(dim * 13 + metric, n, dim)
    queries = queries_for(metric, dim * 13 + metric + 1, nq, dim)
    env = Envelope(metric, rows, queries)
    expect = 128 if dim <= 896 else 96 if dim <= 1280 else 64 if dim <= 1920 else 32
    assert tc_query_block(nq, dim) == expect
    gpu = make_index(metric, rows)
    for k in (10, 300):
        ref, st = knn(gpu, queries, k, 2)
        assert st["tc_used"] == 0
        check_knn(env, *ref, k, ctx=(dim, k, "exact"))
        for mode in (3, 4):
            got, st = knn(gpu, queries, k, mode)
            assert st["tc_used"] == 1, (k, mode, st)
            if mode == 3 and k == 10:
                assert st["query_tile"] == expect, st
            assert_identical(ref, got, ctx=(dim, k, mode))
    gpu.close()


def test_filter_leaves_2049_dims_to_the_exact_scan():
    n, nq, dim, k = 2000, 128, 2049, 10
    for metric in METRICS:
        rows = gaussian(0x2049 + metric, n, dim)
        queries = queries_for(metric, 0x2050 + metric, nq, dim)
        gpu = make_index(metric, rows)
        out, st = knn(gpu, queries, k, 1)
        assert st["tc_used"] == 0, st
        check_knn(Envelope(metric, rows, queries), *out, k, ctx=metric)
        gpu.set_tensor_core_filter(1)
        r = np.full(nq, np.inf, np.float32)
        d, l, c = gpu.search_range_batch(queries, r, max_out=5)
        assert rx.last_search_stats()["tc_used"] == 0 and (c == n).all()
        gpu.close()


@pytest.mark.parametrize("dim", [200, 1000])
@pytest.mark.parametrize("nq", [1, 31, 32, 33, 95, 97, 127, 128, 129, 257])
def test_filter_query_counts(nq, dim):
    n, k, metric = 3000, 10, rx.IP
    rows = gaussian(nq + dim, n, dim)
    queries = queries_for(metric, nq + dim + 1, nq, dim)
    env = Envelope(metric, rows, queries)
    gpu = make_index(metric, rows)
    ref, _ = knn(gpu, queries, k, 2)
    check_knn(env, *ref, k, ctx=nq)
    got, st = knn(gpu, queries, k, 3)
    assert st["tc_used"] == 1 and st["query_tile"] == tc_query_block(nq, dim), (st, tc_query_block(nq, dim))
    assert_identical(ref, got, ctx=nq)
    got, st = knn(gpu, queries, k, 4)
    assert st["tc_used"] == 1
    assert_identical(ref, got, ctx=(nq, 4))
    gpu.close()


@pytest.mark.parametrize("n", [1, 2, 127, 128, 129, 1023, 1025, 5000])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_filter_row_counts(metric, n):
    """fewer rows than one 128-row tile, than tc_init_tau's 1024 rows, and (5000 rows = 40 tiles, 33 queries = one query group) fewer
    tiles than the walkers one query group could use"""
    dim, nq = 96, 33
    rows = gaussian(n * 3 + metric, n, dim)
    queries = queries_for(metric, n * 3 + metric + 1, nq, dim)
    env = Envelope(metric, rows, queries)
    gpu = make_index(metric, rows)
    for k in (1, 10, 300):
        ref, _ = knn(gpu, queries, k, 2)
        check_knn(env, *ref, k, ctx=(n, k))
        got, st = knn(gpu, queries, k, 1)
        assert st["tc_used"] == 1, st
        assert_identical(ref, got, ctx=(n, k))
    radius = radii_at(env)
    gpu.set_tensor_core_filter(2)
    exact = gpu.search_range_batch(queries, radius)
    check_range(env, radius, *exact, ctx=n)
    gpu.set_tensor_core_filter(1)
    got = gpu.search_range_batch(queries, radius)
    assert rx.last_search_stats()["tc_used"] == 1
    assert_identical(exact, got, ctx=(n, "range"))
    gpu.close()


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_filter_k_boundaries(metric):
    """k + 1 = 128 is the last k on the in-kernel bound list (one filter launch), 129 the first on staged thresholds (a seed scan and
    at least one stage), 1024 the last staged, 1025 the exact scan"""
    n, dim, nq = 4000, 96, 64
    rows = gaussian(0x4B + metric, n, dim)
    queries = queries_for(metric, 0x4C + metric, nq, dim)
    env = Envelope(metric, rows, queries)
    gpu = make_index(metric, rows)
    for k in (1, 10, 126, 127, 128, 1022, 1023, 1024):
        ref, _ = knn(gpu, queries, k, 2)
        check_knn(env, *ref, k, ctx=k)
        got, st = knn(gpu, queries, k, 1)
        if k + 1 <= 128:
            assert st["tc_used"] == 1 and st["passes"] == 1 and st["tc_fallbacks"] == 0, (k, st)
        elif k + 1 <= 1024:
            assert st["tc_used"] == 1 and st["passes"] >= 2 and st["tc_fallbacks"] == 0, (k, st)
        else:
            assert st["tc_used"] == 0, (k, st)
        assert_identical(ref, got, ctx=k)
    gpu.close()


@pytest.mark.parametrize("dim", [1536, 2048])
@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_filter_range_batch_large_dims(metric, dim):
    n, nq = 3000, 96
    rows = gaussian(dim * 17 + metric, n, dim)
    queries = queries_for(metric, dim * 17 + metric + 1, nq, dim)
    env = Envelope(metric, rows, queries)
    radius = radii_at(env)
    gpu = make_index(metric, rows)
    gpu.set_tensor_core_filter(2)
    exact = gpu.search_range_batch(queries, radius)
    check_range(env, radius, *exact, ctx=dim)
    for mode in (3, 4):
        gpu.set_tensor_core_filter(mode)
        got = gpu.search_range_batch(queries, radius)
        st = rx.last_search_stats()
        assert st["tc_used"] == 1 and st["tc_fallbacks"] == 0, st
        assert_identical(exact, got, ctx=(dim, mode))
    gpu.close()


@pytest.mark.parametrize("dim", [768, 1536])
def test_cosine_unit_norm_rows(dim):
    """Unit-norm rows take norm_coef_kernel's shortcut (coefficient exactly 1).  Rows scaled to |v|^2 = 1 +- 2e-6 keep it,
    1 +- 4e-5 do not, and 1 +- 1e-5 sit on the edge; queries next to those rows make |q.v| about 1, so a coefficient on the wrong
    side of the rule moves the distance by 2e-5, several times the envelope"""
    n, nq, k = 4000, 128, 10
    rng = np.random.default_rng(dim)
    base = unit(rng.standard_normal((n, dim)))
    scale = np.ones(n)
    scale[: n // 2] = np.sqrt(1.0 + np.resize([2e-6, -2e-6, 4e-5, -4e-5, 1e-5, -1e-5], n // 2))
    rows = (base.astype(np.float64) * scale[:, None]).astype(np.float32)
    near = rows[rng.integers(0, n // 2, size=nq // 2)].astype(np.float64)
    queries = np.concatenate([unit(near + rng.normal(0, 0.003, near.shape)), unit(rng.standard_normal((nq - nq // 2, dim)))])
    short_ok, long_ok, _, _ = coefs = norm_coefs(rows)
    assert short_ok[n // 2:].all() and not long_ok[n // 2:].any()  # the unit rows: the shortcut
    assert (short_ok & ~long_ok).sum() > n // 2 and (long_ok & ~short_ok).sum() > n // 8
    env = Envelope(rx.COS, rows, queries, coefs)
    gpu = make_index(rx.COS, rows)
    ref, _ = knn(gpu, queries, k, 2)
    check_knn(env, *ref, k, ctx=dim)
    got, st = knn(gpu, queries, k, 1)
    assert st["tc_used"] == 1
    assert_identical(ref, got)
    radius = radii_at(env)
    gpu.set_tensor_core_filter(2)
    exact = gpu.search_range_batch(queries, radius)
    check_range(env, radius, *exact, ctx=dim)
    gpu.set_tensor_core_filter(1)
    assert_identical(exact, gpu.search_range_batch(queries, radius))
    gpu.close()


def test_l2_rows_with_a_large_common_offset():
    """rows and queries near 1000 * 1: the filter's eps (|q|^2 + |v|^2) term dwarfs every gap, every row is a candidate, the lists
    overflow, and those queries must come back from the exact scan with exact answers"""
    n, dim, nq, k = 10000, 768, 64, 10
    rows = (1000.0 + gaussian(0x0FF, n, dim)).astype(np.float32)
    queries = (1000.0 + gaussian(0x100, nq, dim)).astype(np.float32)
    env = Envelope(rx.L2, rows, queries)
    gpu = make_index(rx.L2, rows)
    ref, _ = knn(gpu, queries, k, 2)
    check_knn(env, *ref, k)
    got, st = knn(gpu, queries, k, 1)
    assert st["tc_used"] == 1 and st["tc_fallbacks"] > 0, st
    assert_identical(ref, got)
    radius = radii_at(env)
    gpu.set_tensor_core_filter(1)
    rng_out = gpu.search_range_batch(queries, radius)
    check_range(env, radius, *rng_out)
    gpu.close()


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_int8_stress_rows_at_2048_dims(metric):
    n, dim, nq, k = 6000, 2048, 160, 10
    rng = np.random.default_rng(0x800 + metric)
    rows = adversarial_rows(rng, n, dim)
    queries = adversarial_queries(rng, rows, nq, dim)
    if metric == rx.COS:
        queries = np.stack([unit(q[None])[0] if np.any(q) else q for q in queries])
    env = Envelope(metric, rows, queries)
    gpu = make_index(metric, rows)
    ref, _ = knn(gpu, queries, k, 2)
    check_knn(env, *ref, k)
    got, st = knn(gpu, queries, k, 1)
    assert st["tc_used"] == 1, st
    assert_identical(ref, got)
    gpu.close()


def test_automatic_routing_100k_rows_1536_dims():
    n, dim, nq, k, seed = 100_000, 1536, 128, 10, 0x1536
    gpu = rx.GpuBruteforceSearch(rx.IP, dim, n)
    gpu.append_synth(seed, 0, n)
    queries = gaussian(seed + 1, nq, dim)
    d, l, c = gpu.search_knn(queries, k)  # mode 0: 128 queries on 100 k rows take the filter
    st = rx.last_search_stats()
    assert st["tc_used"] == 1 and st["query_tile"] == 64, st
    sample = np.arange(0, nq, 8)
    rows = O.synth_matrix(seed, n, dim)
    env = Envelope(rx.IP, rows, queries[sample])
    check_knn(env, d[sample], l[sample], c[sample], k)
    gpu.close()


# ---------------------------------------------------------------------------------------------------------------- IVF


def ivf_index(metric, dim, nlist, n, seed, empty_every=7):
    """centroids and list assignments chosen here (no k-means): rows go to random lists, every `empty_every`-th list stays empty"""
    rng = np.random.default_rng(seed)
    cents = gaussian(seed + 1, nlist, dim)
    rows = gaussian(seed + 2, n, dim)
    usable = np.array([l for l in range(nlist) if l % empty_every != 0], np.uint32)
    lists = usable[rng.integers(0, len(usable), size=n)]
    gpu = rx.GpuBruteforceSearch(metric, dim, 16)
    gpu.ivf_create(cents)
    gpu.ivf_add(lists, O.row_labels(n), rows)
    assert gpu.ivf_size() == n
    return gpu, cents, rows, lists


def probed_rows(metric, cents, queries, lists, nprobe):
    """the rows of the nprobe nearest lists of each query, and which queries have an unambiguous probed set in fp64"""
    cenv = Envelope(metric, cents, queries)
    nlist = len(cents)
    order = np.argsort(cenv.mid, axis=1, kind="stable")
    inside = order[:, :nprobe]
    clear = np.ones(len(queries), bool)
    if nprobe < nlist:
        hi_in = np.take_along_axis(cenv.hi, inside, 1).max(1)
        lo_out = np.take_along_axis(cenv.lo, order[:, nprobe:], 1).min(1)
        clear = hi_in < lo_out
    probed = np.zeros((len(queries), nlist), bool)
    np.put_along_axis(probed, inside, True, 1)
    return probed[:, lists], clear


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_ivf_at_its_documented_limits(metric):
    """k = 256, nprobe = 1024 (a full merge fan-in: knn_merge_lists merges 1024 lists per query) over 16384 centroids, with empty
    lists and lists far shorter than k"""
    dim, nlist, n, nq, k, nprobe = 64, 16384, 40000, 24, 256, 1024
    gpu, cents, rows, lists = ivf_index(metric, dim, nlist, n, 0x1F0 + metric)
    queries = queries_for(metric, 0x1F5 + metric, nq, dim)
    allowed, clear = probed_rows(metric, cents, queries, lists, nprobe)
    assert clear.sum() >= nq // 2, clear.sum()
    d, l, c = gpu.ivf_search_knn(queries, k, nprobe)
    env = Envelope(metric, rows, queries[clear]).restrict(allowed[clear])
    check_knn(env, d[clear], l[clear], c[clear], k)
    # range search over the same 1024 probed lists, at the 10th and 100th best probed distance
    for q in np.nonzero(clear)[0][:6]:
        e1 = Envelope(metric, rows, queries[q]).restrict(allowed[q][None])
        for j in (10, 100):
            radius = np.float32(np.sort(e1.mid[0])[j - 1])
            rd, rl, total = gpu.ivf_search_range(queries[q], float(radius), nprobe)
            check_range(e1, radius, rd[None], rl[None], [total], ctx=(q, j))
    gpu.close()


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_ivf_every_list_probed_and_fan_in_refusal(metric):
    dim, n, nq, k = 48, 20000, 16, 256
    gpu, cents, rows, lists = ivf_index(metric, dim, 1024, n, 0x2F0 + metric)
    queries = queries_for(metric, 0x2F5 + metric, nq, dim)
    d, l, c = gpu.ivf_search_knn(queries, k, 1024)  # nprobe = nlist: the exact answer over all rows
    check_knn(Envelope(metric, rows, queries), d, l, c, k)
    d2, l2, c2 = gpu.ivf_search_knn(queries, k, 1025)  # clamped to nlist first, like faiss::IndexIVF::search
    assert_identical((d, l, c), (d2, l2, c2))
    gpu.close()
    big, _, _, _ = ivf_index(metric, dim, 2048, 4000, 0x3F0 + metric)
    with pytest.raises(rx.RxGpuError) as e:
        big.ivf_search_knn(queries, 10, 1025)
    assert e.value.code == ERR_PARAMS and "merge fan-in (1024)" in e.value.what, e.value.what
    d, l, c = big.ivf_search_knn(queries, 10, 1024)
    assert (c == 10).all()
    big.close()
