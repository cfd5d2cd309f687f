"""PolyGamma, GammaIncInv, GammaIncCInv and BetaIncInv on the device against the reference C linker (which evaluates
them through SciPy: scalar/math.py has no C code for any of the four), their gradients with respect to the probability
argument, a fused map+row-reduce over gammaincinv, and inverse-CDF sampling of a truncated Gamma distribution.

Bars: float64 rtol 1e-9 on the regular domain and 1e-8 in the extreme regimes, atol 0 (exact zeros must be exact);
float32 rtol 2e-7 (one float32 ulp), except betaincinv, whose float32 C-linker values come from SciPy's single-precision
loop and carry up to 3e-4 of its own error (DESIGN.md section 9).  Edge cases are planted in the vector tail."""

import os

import numpy as np
import pytest
import scipy.special as sp
import scipy.stats as st

from helpers import compare_cuda_and_cvm, pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu

DRY = os.environ.get("PTK_DRY") == "1"


def _regular(n, seed):
    rng = np.random.default_rng(seed)
    a = np.exp(rng.uniform(np.log(0.05), np.log(50), n))
    b = np.exp(rng.uniform(np.log(0.05), np.log(50), n))
    p = np.exp(rng.uniform(np.log(1e-12), 0, n))
    p = np.clip(np.where(rng.random(n) < 0.5, p, 1 - p), 1e-12, 1 - 1e-12)
    k = rng.integers(0, 13, n)
    x = rng.uniform(-40, 40, n)
    x[np.abs(x - np.round(x)) < 1e-2] += 0.05
    return a, b, p, x, k


GAMMA_EDGES = [(np.nan, 0.5), (0.0, 0.5), (-1.0, 0.5), (np.inf, 0.5), (2.0, np.nan), (2.0, -0.1), (2.0, 1.5),
               (2.0, 0.0), (2.0, 1.0), (1e-3, 0.5), (1e-3, 1e-10)]
BETA_EDGES = [(0.0, 1.0, 0.5), (-1.0, 1.0, 0.5), (1.0, -2.0, 0.5), (2.0, 3.0, -0.1), (2.0, 3.0, 1.5),
              (np.nan, 1.0, 0.5), (2.0, 3.0, 0.0), (2.0, 3.0, 1.0), (1e-3, 5.0, 0.3), (np.inf, 1.0, 0.5)]
POLYGAMMA_EDGES = [(0, 0.0), (0, -2.0), (1, 0.0), (2, 0.0), (1, -3.0), (2, -3.0), (1, -1.5), (171, 2.0), (200, 50.0),
                   (-1, 2.0), (1, np.inf), (2, -np.inf)]


def _edge_layouts(values, edges):
    """One input set per edge case: `values` (one array per argument), then every edge case (inside full vectors), then
    the case itself as the last element of a length = 1 (mod 4) array, so that it is the whole scalar tail for both the
    4-wide float32 and the 2-wide float64 vectors."""
    body = [np.concatenate([v, np.array(e, dtype=v.dtype)]) for v, e in zip(values, zip(*edges))]
    n = len(body[0]) - (len(body[0]) % 4)
    for case in edges:
        yield [np.concatenate([v[:n], np.array([c], dtype=v.dtype)]) for v, c in zip(body, case)]


def _compare_with_edges(ins, outs, values, edges, **kw):
    for layout in _edge_layouts(values, edges):
        compare_cuda_and_cvm(ins, outs, layout, **kw)


def _rtol(dtype, fp64):
    return fp64 if dtype == "float64" else 2e-7


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_regular_domain_and_edges(gpu, dtype):
    pytensor.config.floatX = dtype
    av, bv, pv, xv, kv = _regular(20001, 51)
    a, b, p, x = (pt.vector(nm, dtype=dtype) for nm in "abpx")
    k = pt.vector("k", dtype="int64")
    _compare_with_edges([a, p], [pt.gammaincinv(a, p), pt.gammainccinv(a, p)], [av.astype(dtype), pv.astype(dtype)],
                        GAMMA_EDGES, rtol=_rtol(dtype, 1e-9), atol=0)
    _compare_with_edges([k, x], [pt.polygamma(k, x)], [kv.astype("int64"), xv.astype(dtype)], POLYGAMMA_EDGES,
                        rtol=_rtol(dtype, 1e-9), atol=0)
    beta = [pt.betaincinv(a, b, p)]
    vals = [av.astype(dtype), bv.astype(dtype), pv.astype(dtype)]
    if dtype == "float64":
        _compare_with_edges([a, b, p], beta, vals, BETA_EDGES, rtol=1e-9, atol=0)
    else:
        for layout in _edge_layouts(vals, BETA_EDGES):
            _, got = compare_cuda_and_cvm([a, b, p], beta, layout, rtol=5e-4, atol=1e-37)
            if got is not None:       # ... and one rounding of SciPy's float64 quantile
                ref64 = sp.betaincinv(*[v.astype("float64") for v in layout]).astype(np.float32)
                np.testing.assert_allclose(got[0], ref64, rtol=2e-7, atol=0)


EXTREME_P = np.array([1e-300, 1e-200, 1e-100, 1e-30, 1e-12, 1e-5, 0.01, 0.3, 0.5, 0.7, 0.99, 1 - 1e-5, 1 - 1e-12])


def _grid(*axes):
    return [g.ravel() for g in np.meshgrid(*axes, indexing="ij")]


def test_extreme_regimes_float64(gpu):
    """a or b in {1e-3, 1e4}, p down to 1e-300 and up to 1 - 1e-12, x next to the poles.  Excluded and pinned in the
    CPU suite (DESIGN.md section 9): a = 1e6 for gammaincinv, and the betaincinv points where SciPy returns 0 / NaN."""
    pytensor.config.floatX = "float64"
    a, b, p = pt.dvectors("a", "b", "p")
    av, pv = _grid(np.array([1e-3, 0.05, 1.0, 50.0, 1e4]), EXTREME_P)
    compare_cuda_and_cvm([a, p], [pt.gammaincinv(a, p), pt.gammainccinv(a, p)], [av, pv], rtol=1e-8, atol=0)
    par = np.array([1e-3, 0.5, 2.0, 1e4])
    av, bv, pv = _grid(par, par, EXTREME_P)
    ref = sp.betaincinv(av, bv, pv)
    keep = ~(((av == 0.5) & (bv == 0.5) & (pv < 1e-100)) | np.isnan(ref))
    compare_cuda_and_cvm([a, b, p], [pt.betaincinv(a, b, p)], [av[keep], bv[keep], pv[keep]], rtol=1e-8, atol=0)
    near = np.array([1e-4, 0.3, 0.5])
    xs = np.concatenate([(np.array([-12.0, -3.0, -1.0])[:, None] + np.concatenate([near, -near])).ravel(),
                         [1e-12, 1e-8, -1e-12, -1e-8, 1 + 1e-12, 1 - 1e-8, 1e-300, 1e3, 1e8, 1e15]])
    kv, xv = _grid(np.arange(0, 13), xs)
    k, x = pt.vector("k", dtype="int64"), pt.dvector("x")
    f = pytensor.function([k, x], pt.polygamma(k, x), mode="CUDA")
    if DRY:
        return
    got = np.asarray(f(kv.astype("int64"), xv))
    ref = pytensor.function([k, x], pt.polygamma(k, x), mode="CVM")(kv.astype("int64"), xv)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    np.testing.assert_array_equal(got[~fin], ref[~fin])
    # where the shifted terms of a negative x cancel (e.g. n = 10 at x = -2.5: +-2048 down to 4 / 10!), both sides keep
    # 1e-13 of the sum of the terms' magnitudes (their summation rounding), not of the result
    tol = 1e-8 * np.abs(ref) + 1e-13 * _polygamma_term_scale(kv, xv)
    np.testing.assert_array_less(np.abs(got[fin] - ref[fin]), tol[fin] + 1e-300)


def _polygamma_term_scale(n, x):
    """n! sum_k |x + k|^-(n+1) (bounded by the two Hurwitz zetas about the fractional part of x), 0 where n = 0."""
    fr = x - np.floor(x)
    with np.errstate(all="ignore"):
        s = sp.gamma(n + 1.0) * (sp.zeta(n + 1.0, np.where(fr > 0, fr, 1.0)) + sp.zeta(n + 1.0, 1.0 - fr + (fr == 0)))
    return np.where((n > 0) & (x < 0) & np.isfinite(s), s, 0.0)


BETA_POINTS = [(0.0013417, 171.37, 0.8867), (0.00246589, 170.764, 0.9779), (170.623, 0.00181, 0.3618),
               (0.00118779, 4497.18, 0.993142), (0.00158509, 9343.59, 0.990772), (0.00293188, 3110.69, 0.985293)]


def test_betaincinv_small_shape_next_to_a_large_one(gpu):
    """Random (a, b, p): a in [1e-3, 0.1], b in [10, 1e4], p in (0, 1), half mirrored to (b, a, p), a quarter with
    a + b in [168, 171.6]; plus fixed points where the root lies between the mean and (a+1)/(a+b+2), or where BetaInc's
    linear branch would overflow tgamma(a) tgamma(b)."""
    pytensor.config.floatX = "float64"
    rng = np.random.default_rng(56)
    n = 20000
    av = np.exp(rng.uniform(np.log(1e-3), np.log(0.1), n))
    bv = np.exp(rng.uniform(np.log(10), np.log(1e4), n))
    q = rng.random(n) < 0.25
    bv[q] = rng.uniform(168, 171.6, q.sum()) - av[q]
    pv = rng.uniform(0, 1, n)
    m = rng.random(n) < 0.5
    av, bv = np.where(m, bv, av), np.where(m, av, bv)
    pa, pb, pp = (np.array(c) for c in zip(*BETA_POINTS))
    av, bv, pv = np.concatenate([av, pa]), np.concatenate([bv, pb]), np.concatenate([pv, pp])
    # (quantiles in the denormal range: SciPy returns 0 for some, the device the largest denormal; DESIGN.md section 9,
    # pinned in the CPU suite)
    keep = sp.betaincinv(av, bv, pv) > 0
    a, b, p = pt.dvectors("a", "b", "p")
    compare_cuda_and_cvm([a, b, p], [pt.betaincinv(a, b, p)], [av[keep], bv[keep], pv[keep]], rtol=1e-8, atol=0)


def test_gradients(gpu):
    """d tri_gamma / dx is polygamma(2, x); a symbolic order reaches PolyGamma itself (a constant 0 or 1 is rewritten
    to psi / tri_gamma); the inverses' gradients w.r.t. the probability are Elemwise graphs around the inverse."""
    pytensor.config.floatX = "float64"
    rng = np.random.default_rng(52)
    x, p = pt.dvectors("x", "p")
    n = pt.lscalar("n")
    av, bv = pt.dscalars("a", "b")
    xv = rng.uniform(0.1, 30, 4097)
    pv = rng.uniform(0.01, 0.99, 4097)
    g_tri = pytensor.grad(pt.tri_gamma(x).sum(), x)
    compare_cuda_and_cvm([x], [g_tri], [xv], rtol=1e-9, atol=0)
    pg = pt.polygamma(n, x)
    compare_cuda_and_cvm([n, x], [pg, pytensor.grad(pg.sum(), x)], [3, xv], rtol=1e-9, atol=0)
    outs = [pytensor.grad(pt.gammaincinv(av, p).sum(), p), pytensor.grad(pt.gammainccinv(av, p).sum(), p),
            pytensor.grad(pt.betaincinv(av, bv, p).sum(), p)]
    compare_cuda_and_cvm([av, bv, p], outs, [2.5, 3.5, pv], rtol=1e-8, atol=0)


def test_fused_map_row_reduce(gpu):
    from pytensor_b200.vm.nodes_elemwise import ElemwiseReduceNode

    pytensor.config.floatX = "float64"
    rng = np.random.default_rng(53)
    a, u = pt.dvector("a"), pt.dmatrix("u")
    av = rng.uniform(0.5, 20, 4099)
    uv = rng.uniform(0.0, 1.0, (257, 4099))
    f, _ = compare_cuda_and_cvm([a, u], [pt.gammaincinv(a[None, :], u).sum(axis=1)], [av, uv], rtol=1e-10, atol=0)
    assert any(isinstance(st_.impl, ElemwiseReduceNode) for st_ in f.vm.executor.program.steps)


def test_truncated_gamma_by_inverse_cdf(gpu):
    """u ~ Uniform(P(alpha, lo beta), P(alpha, hi beta)), x = gammaincinv(alpha, u) / beta: one compiled function, draws
    from Gamma(alpha, rate beta) truncated to [lo, hi]."""
    pytensor.config.floatX = "float64"
    alpha, beta, lo, hi = 2.5, 1.5, 0.4, 3.0
    rng = pytensor.shared(np.random.default_rng(54), name="rng")
    pl, ph = pt.gammainc(alpha, lo * beta), pt.gammainc(alpha, hi * beta)
    nr, uu = pt.random.uniform(pl, ph, size=(200_000,), rng=rng).owner.outputs
    xs = pt.gammaincinv(alpha, uu) / beta
    f = pytensor.function([], xs, updates={rng: nr}, mode="CUDA")
    if DRY:
        return
    x = np.asarray(f())
    assert x.shape == (200_000,) and np.all((x >= lo) & (x <= hi))
    d = st.gamma(alpha, scale=1 / beta)
    c0, c1 = d.cdf(lo), d.cdf(hi)
    ks = st.kstest(x, lambda t: (d.cdf(t) - c0) / (c1 - c0))
    assert ks.pvalue > 1e-4, ks
