"""GPU tests of the SQ8 quantiser and the dp4a scan (reindexer_b200/csrc/sq8.cu) against a NumPy replay, bit for bit.

The quantiser (sq8_quantize_rows on the device, sq8QuantizeHost for queries) is a fixed chain of float32 operations without FMA; NumPy
float32 operations round the same way, so the replay below reproduces codes and corrective offsets exactly.  The scan's integer
distance is exact, and its float epilogue is

    dist = float32(alpha_2 * float32(int_dist)) + qcorr + corr,  negated for IP / Cosine, then * norm_coef, then * qcoef

in that order, so every returned distance is known to the bit and the top-k under (dist, label) is known exactly.  No test here
needs the reference build."""
import numpy as np
import pytest

import reindexer_b200 as rx
from oracle import oracle as O

pytestmark = pytest.mark.gpu

F = np.float32
METRICS = [rx.L2, rx.IP, rx.COS]
MNAME = {rx.L2: "l2", rx.IP: "ip", rx.COS: "cos"}


# ---------------------------------------------------------------------------------------------------------------- replay


def sq8_params(min_q, max_q, dim):
    alpha = F((F(max_q) - F(min_q)) / F(255))
    return dict(min_q=float(F(min_q)), max_q=float(F(max_q)), alpha=float(alpha), alpha_2=float(F(alpha * alpha)),
                delta=float(F(F(dim) * F(min_q) * F(min_q))))


def quantize(params, metric, vals):
    """Quantizer::quantize of every row of vals [n, dim] as sq8_quantize_rows / sq8QuantizeHost write it: (codes, offsets)"""
    v = np.ascontiguousarray(vals, F)
    min_q, alpha, delta = F(params["min_q"]), F(params["alpha"]), F(params["delta"])
    with np.errstate(invalid="ignore", over="ignore"):
        qf = np.minimum(np.maximum((v - min_q) / alpha, F(0)), F(255))
    u = qf.astype(np.uint8)  # float -> uint8 truncates
    uf = u.astype(F)
    err = v - (alpha * uf + min_q)
    if metric == rx.L2:
        terms_res = ((F(2) * alpha) * uf + err) * err
        terms_shift = -(((F(2) * alpha) * err) * uf)  # shift - t == shift + (-t) exactly
    else:
        terms_res = alpha * uf + err
        terms_shift = (alpha * err) * uf
    # the sums are sequential over the elements: a float32 accumulate adds strictly left to right
    res = np.add.accumulate(terms_res, axis=1, dtype=F)[:, -1]
    shift = np.add.accumulate(terms_shift, axis=1, dtype=F)[:, -1]
    if metric != rx.L2:
        res = res * min_q
        res = res + delta
    return u, (res + shift).astype(F)


def query_codes(params, metric, queries, norms):
    """the host quantisation of a query batch (rxgpu_sq8_search_knn): Cosine restores the length first, val = (1 / (1 / norm)) * q"""
    queries = np.asarray(queries, F)
    coef = np.ones(len(queries), F)
    if metric == rx.COS:
        coef = (F(1) / np.asarray(norms, F)).astype(F)
        queries = (F(1) / coef)[:, None] * queries
    codes, corr = quantize(params, metric, queries)
    return codes, corr, coef


def int_dists(metric, qcodes, rcodes):
    q, r = qcodes.astype(np.int64), rcodes.astype(np.int64)
    if metric == rx.L2:
        return (q * q).sum(1)[:, None] + (r * r).sum(1)[None, :] - 2 * (q @ r.T)
    return q @ r.T


def sq8_table(params, metric, qcodes, qcorr, qcoef, rcodes, rcorr, norm_coefs=None):
    """[nq, n] float32 distances in the device's operation order"""
    idist = int_dists(metric, qcodes, rcodes)
    assert idist.max(initial=0) < 2 ** 32
    d = F(params["alpha_2"]) * idist.astype(np.uint32).astype(F)  # __uint2float_rn
    d = (d + qcorr[:, None].astype(F)) + rcorr[None, :].astype(F)
    if metric != rx.L2:
        d = -d
        if norm_coefs is not None:
            d = d * norm_coefs[None, :].astype(F)
    return (qcoef[:, None].astype(F) * d).astype(F)


def topk(table, k):
    """per query: rows of the k best under (dist, row) -- labels grow with the row, so this is the (dist, label) order"""
    n = table.shape[1]
    out = []
    for q in range(len(table)):
        order = np.lexsort((np.arange(n), table[q]))[:min(k, n)]
        out.append(order)
    return out


# ---------------------------------------------------------------------------------------------------------------- data


def unit64(x):
    x = np.asarray(x, np.float64)
    nrm = np.linalg.norm(x, axis=1, keepdims=True)
    return (x / np.where(nrm == 0, 1.0, nrm)).astype(F)


def rows_for(metric, seed, n, dim):
    x = np.random.default_rng(seed).standard_normal((n, dim)).astype(F)
    return unit64(x) if metric == rx.COS else x * F(0.5)


def make(metric, rows, params):
    gpu = rx.GpuBruteforceSearch(metric, rows.shape[1], len(rows))
    gpu.add_points(O.row_labels(len(rows)), rows)
    gpu.sq8_attach(params)
    return gpu


def params_for(metric, dim):
    return sq8_params(-1.0, 1.0, dim) if metric == rx.COS else sq8_params(-1.25, 1.5, dim)


def check_scan(gpu, params, metric, rows, queries, norms, k, ctx=""):
    d, lab, cnt = gpu.sq8_search_knn(queries, k, norms)
    rcodes, rcorr = quantize(params, metric, rows)
    qc, qcorr, qcoef = query_codes(params, metric, queries, norms if norms is not None else np.ones(len(queries), F))
    table = sq8_table(params, metric, qc, qcorr, qcoef, rcodes, rcorr)
    want = topk(table, k)
    for q in range(len(queries)):
        w = want[q]
        assert cnt[q] == len(w), (ctx, q, int(cnt[q]), len(w))
        assert (lab[q, :len(w)] == O.row_labels(len(rows))[w]).all(), (ctx, q, lab[q, :5], w[:5])
        assert (d[q, :len(w)].view(np.uint32) == table[q, w].view(np.uint32)).all(), (ctx, q)
    return d, lab, cnt


# ---------------------------------------------------------------------------------------------------------------- quantiser


def boundary_values(params, dim, rng):
    """values exactly on a code boundary ((v - min_q) / alpha an integer in float32), below min_q, above max_q and min_q itself"""
    min_q, alpha = F(params["min_q"]), F(params["alpha"])
    c = np.arange(256, dtype=F)
    v = (min_q + alpha * c).astype(F)
    exact = v[((v - min_q) / alpha) == c]
    assert len(exact) > 100
    special = np.array([min_q, np.nextafter(min_q, F(-np.inf)), min_q - F(3), F(params["max_q"]), F(params["max_q"]) + F(2),
                        np.nextafter(F(params["max_q"]), F(np.inf))], F)
    pool = np.concatenate([exact, special])
    return pool[rng.integers(0, len(pool), size=dim)]


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("dim", [1, 15, 16, 17, 2048, 65536])
def test_quantiser_bit_exact(metric, dim):
    rng = np.random.default_rng(dim * 3 + metric)
    n = 5 if dim == 65536 else 37
    params = params_for(metric, dim)
    rows = rng.uniform(-1.6, 1.8, size=(n, dim)).astype(F)
    rows[0] = boundary_values(params, dim, rng)
    rows[1] = F(params["min_q"])
    if metric == rx.COS:
        rows[2:] = unit64(rows[2:])
    gpu = make(metric, rows, params)
    codes, offs = gpu.sq8_export()
    want_codes, want_offs = quantize(params, metric, rows)
    assert (codes == want_codes).all(), np.argwhere(codes != want_codes)[:5]
    assert (offs.view(np.uint32) == want_offs.view(np.uint32)).all(), np.argwhere(offs.view(np.uint32) != want_offs.view(np.uint32))[:5]
    # the whole code range is used: the boundary row hits codes 0 and 255 and values in between
    if dim >= 2048:
        assert codes[0].min() == 0 and codes[0].max() == 255
    # queries through sq8_prepare_query: the same arithmetic on the host (Cosine: scaled by 1 / (1 / norm) first)
    for i, norm in ((0, 1.0), (3 % n, 1.0), (n - 1, 0.75)):
        qc, qo = gpu.sq8_prepare_query(rows[i], norm)
        wc, wo, _ = query_codes(params, metric, rows[i:i + 1], np.array([norm], F))
        assert (qc == wc[0]).all()
        assert F(qo).view(np.uint32) == wo[0].view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- scan


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
@pytest.mark.parametrize("dim", [1, 15, 16, 17, 100])
def test_scan_query_tiles_and_k(metric, dim):
    """nq in {1, 2, 3, 4, 5, 7, 9}: every query tile and a partial last tile; k = 1, 255, 256; 257 refused"""
    n = 700
    params = params_for(metric, dim)
    rows = rows_for(metric, 40 + dim, n, dim)
    gpu = make(metric, rows, params)
    queries = rows_for(metric, 90 + dim, 9, dim)
    norms = np.linspace(0.5, 2.0, 9).astype(F) if metric == rx.COS else None
    for nq in (1, 2, 3, 4, 5, 7, 9):
        for k in (1, 255, 256):
            check_scan(gpu, params, metric, rows, queries[:nq], None if norms is None else norms[:nq], k, (nq, k))
            assert rx.last_search_stats()["query_tile"] == (4 if nq >= 4 else 2 if nq >= 2 else 1)
    with pytest.raises(rx.RxGpuError, match="k <= 256"):
        gpu.sq8_search_knn(queries[:2], 257, None if norms is None else norms[:2])


@pytest.mark.parametrize("metric", METRICS, ids=MNAME.get)
def test_scan_row_counts(metric):
    """n = 1, 2, 15, 16, 17 with k > n, and the row count at which the grid reaches 2 x SMs (one row more too)"""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    dim = 33
    params = params_for(metric, dim)
    queries = rows_for(metric, 7, 5, dim)
    norms = np.full(5, 1.0, F) if metric == rx.COS else None
    for n in (1, 2, 15, 16, 17, 32 * sms, 32 * sms + 1, 32 * sms + 17):
        rows = rows_for(metric, n, n, dim)
        gpu = make(metric, rows, params)
        for k in (1, 16, 256):
            check_scan(gpu, params, metric, rows, queries, norms, k, (n, k))


@pytest.mark.parametrize("metric", [rx.L2, rx.IP], ids=MNAME.get)
def test_scan_integer_sums_above_2_24(metric):
    """dim 2048 with codes near 255 against codes 0 (L2) or near 255 (IP): the integer sums exceed 2^24 and their float32 rounding
    (__uint2float_rn) decides the low bits of the distance"""
    dim, n = 2048, 300
    params = sq8_params(0.0, 255.0, dim)  # alpha = 1: value v -> code floor(v)
    rng = np.random.default_rng(5 + metric)
    rows = rng.integers(240, 256, size=(n, dim)).astype(F)
    queries = np.zeros((3, dim), F) if metric == rx.L2 else rng.integers(240, 256, size=(3, dim)).astype(F)
    gpu = make(metric, rows, params)
    rcodes, _ = quantize(params, metric, rows)
    qc, _, _ = query_codes(params, metric, queries, None)
    idist = int_dists(metric, qc, rcodes)
    assert idist.min() > 2 ** 24
    assert (idist.astype(np.uint32).astype(F).astype(np.int64) != idist).mean() > 0.5  # most sums are not representable
    check_scan(gpu, params, metric, rows, queries, None, 256)


def test_scan_cosine_unnormalised_rows():
    """Cosine rows of any length: the row coefficient comes from norm_coef_kernel, held to 2e-6 relative here"""
    dim, n = 64, 500
    params = params_for(rx.COS, dim)
    rows = rows_for(rx.L2, 3, n, dim) * F(1.7)
    gpu = make(rx.COS, rows, params)
    queries = rows_for(rx.COS, 4, 4, dim)
    norms = np.ones(4, F)
    d, lab, cnt = gpu.sq8_search_knn(queries, 20, norms)
    rcodes, rcorr = quantize(params, rx.COS, rows)
    qc, qcorr, qcoef = query_codes(params, rx.COS, queries, norms)
    coef = (1.0 / np.linalg.norm(rows.astype(np.float64), axis=1)).astype(F)
    table = sq8_table(params, rx.COS, qc, qcorr, qcoef, rcodes, rcorr, coef)
    for q in range(4):
        rows_q = (lab[q, :cnt[q]] >> np.uint64(32)).astype(np.int64)
        assert cnt[q] == 20 and (np.diff(d[q, :20]) >= 0).all()
        assert np.allclose(d[q, :20], table[q, rows_q], rtol=2e-6, atol=0)
        missing = np.setdiff1d(np.arange(n), rows_q)
        assert (table[q, missing] >= d[q, 19] - 4e-6 * np.abs(table[q, missing]).max()).all()


# ---------------------------------------------------------------------------------------------------------------- tile fallback


@pytest.mark.parametrize("dim,tile", [(7056, 4), (7057, 2), (32656, 2), (32657, 1)])
def test_query_tile_falls_back_to_the_shared_memory_budget(dim, tile):
    """k = 256: a tile of 4 queries fits 100 KiB up to 7056 dims, a tile of 2 up to 32656; past that the scan takes the next smaller
    tile instead of refusing, and a batch of 9 equals the 9 single-query calls bit for bit"""
    metric, n, k = rx.L2, 260, 256
    params = params_for(metric, dim)
    rows = rows_for(metric, dim, n, dim)
    gpu = make(metric, rows, params)
    queries = rows_for(metric, dim + 1, 9, dim)
    d, lab, cnt = check_scan(gpu, params, metric, rows, queries, None, k, dim)
    assert rx.last_search_stats()["query_tile"] == tile
    for q in range(9):
        d1, l1, c1 = gpu.sq8_search_knn(queries[q:q + 1], k)
        assert c1[0] == cnt[q] == k
        assert (l1[0] == lab[q]).all() and (d1[0].view(np.uint32) == d[q].view(np.uint32)).all(), q
