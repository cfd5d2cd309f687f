"""Discrete-count and row samplers on the device (ptk_random_count / ptk_random_rows in csrc/ptk_random.cu, vm/nodes_random.py)
against the reference's RandomVariables (pytensor/tensor/random/basic.py: PoissonRV, BinomialRV, NegBinomialRV, GeometricRV,
BetaBinomialRV, CategoricalRV, MultinomialRV, DirichletRV).  Values come from counter-based Philox streams, so they differ
from the C linker's; what must agree is the distribution (chi-squared against scipy's pmf, moments within 5 standard
errors, KS for Dirichlet marginals; fixed seeds, so a failure reproduces), the shapes / dtypes / broadcasting and the
parameter errors of the C linker, and the generator protocol."""

import numpy as np
import pytest
import scipy.stats as st

from discrete_fit import chi2_counts, chi2_pvalue, moments_ok
from helpers import pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu

N = 200_000
R = pt.random


def _draw(build, seed=123, n_calls=1, mode="CUDA"):
    rng = pytensor.shared(np.random.default_rng(seed), name="rng")
    nr, x = build(rng).owner.outputs
    f = pytensor.function([], x, updates={rng: nr}, mode=mode)
    return [np.asarray(f()) for _ in range(n_calls)], f


COUNT_CASES = [(f"poisson-{lam:g}", lambda r, lam=lam: R.poisson(lam, size=(N,), rng=r), st.poisson(lam))
               for lam in (1e-3, 0.5, 9.99, 10.0, 37.5, 1e4, 1e12)]
COUNT_CASES += [(f"binomial-{n}-{p:g}", lambda r, n=n, p=p: R.binomial(n, p, size=(N,), rng=r), st.binom(n, p))
                for n, p in ((10, 0.3), (1000, 0.5), (1000, 0.97), (40, 0.249), (40, 0.251), (2 ** 40, 1e-9))]
COUNT_CASES += [
    ("negative_binomial-2.5-0.3", lambda r: R.negative_binomial(2.5, 0.3, size=(N,), rng=r), st.nbinom(2.5, 0.3)),
    ("geometric-0.5", lambda r: R.geometric(0.5, size=(N,), rng=r), st.geom(0.5)),
    ("geometric-1e-4", lambda r: R.geometric(1e-4, size=(N,), rng=r), st.geom(1e-4)),
    ("beta_binomial-10-2-3", lambda r: R.betabinom(10, 2.0, 3.0, size=(N,), rng=r), st.betabinom(10, 2.0, 3.0)),
    ("beta_binomial-100-.5-.5", lambda r: R.betabinom(100, 0.5, 0.5, size=(N,), rng=r), st.betabinom(100, 0.5, 0.5)),
]


class _NormalLimit:
    """N(m, s^2) as the distribution of an integer variable (continuity-corrected cdf) for chi2_pvalue."""

    def __init__(self, m, s):
        self.d = st.norm(m, s)

    def ppf(self, q):
        return self.d.ppf(q)

    def cdf(self, c):
        return self.d.cdf(np.asarray(c) + 0.5)


@pytest.mark.parametrize("name,build,dist", COUNT_CASES, ids=[c[0] for c in COUNT_CASES])
def test_count_samplers_fit_the_reference_distribution(gpu, name, build, dist):
    pytensor.config.floatX = "float64"
    (x,), _ = _draw(build)
    assert x.shape == (N,) and x.dtype == np.int64
    # scipy's Poisson ppf / cdf lose their precision at lam = 1e12: fit the normal limit there (skewness 1e-6)
    fit = _NormalLimit(dist.mean(), dist.std()) if name == "poisson-1e+12" else dist
    p = chi2_pvalue(x, fit)
    assert p > 1e-4, (name, p)
    ok, info = moments_ok(x, dist.mean(), dist.var())
    assert ok, (name, info)
    if name == "poisson-1e+12":
        assert x.min() > 2 ** 31


def test_per_element_parameters_mixing_regimes(gpu):
    pytensor.config.floatX = "float64"
    lams = [0.3, 9.9, 10.1, 500.0]
    (x,), _ = _draw(lambda r: R.poisson(np.repeat(lams, 50_000), rng=r))
    for j, lam in enumerate(lams):
        blk = x[j * 50_000:(j + 1) * 50_000]
        assert chi2_pvalue(blk, st.poisson(lam)) > 1e-4, lam
        assert moments_ok(blk, lam, lam)[0], lam
    ns = np.repeat([10, 40, 1000, 5], 50_000)
    ps = np.repeat([0.3, 0.251, 0.97, 0.5], 50_000)
    (y,), _ = _draw(lambda r: R.binomial(ns, ps, rng=r))
    for j in range(4):
        blk = y[j * 50_000:(j + 1) * 50_000]
        assert chi2_pvalue(blk, st.binom(ns[j * 50_000], ps[j * 50_000])) > 1e-4, j


@pytest.mark.parametrize("k", [1, 2, 5, 31, 32, 33, 1000, 70_000])
def test_categorical_fits_p_and_never_draws_a_zero_category(gpu, k):
    pytensor.config.floatX = "float64"
    p = np.random.default_rng(k).dirichlet(np.ones(k))
    if k >= 2:
        p[1] = 0.0
        p /= p.sum()
    (x,), _ = _draw(lambda r: R.categorical(p, size=(N,), rng=r), seed=k)
    assert x.shape == (N,) and x.dtype == np.int64 and x.min() >= 0 and x.max() < k
    counts = np.bincount(x, minlength=k)
    if k >= 2:
        assert counts[1] == 0
    nz = p > 0
    assert chi2_counts(counts[nz], N * p[nz]) > 1e-4


def test_categorical_batches_and_mass_beyond_the_total(gpu):
    pytensor.config.floatX = "float64"
    P = np.random.default_rng(4).dirichlet(np.ones(5), size=4)
    (x,), _ = _draw(lambda r: R.categorical(P, size=(50_000, 4), rng=r))
    assert x.shape == (50_000, 4)
    for i in range(4):
        assert chi2_counts(np.bincount(x[:, i], minlength=5), 50_000 * P[i]) > 1e-4, i
    (h,), _ = _draw(lambda r: R.categorical(np.full(4, 0.125), size=(N,), rng=r))
    assert abs(np.mean(h == 4) - 0.5) < 5 * np.sqrt(0.25 / N)


@pytest.mark.parametrize("k", [2, 5, 31, 32, 33])
def test_multinomial_rows_sum_to_n_with_binomial_marginals(gpu, k):
    pytensor.config.floatX = "float64"
    n = 20
    p = np.random.default_rng(k).dirichlet(np.ones(k))
    p[0] = 0.0
    p /= p.sum()
    rows = 100_000
    (x,), _ = _draw(lambda r: R.multinomial(n, p, size=(rows,), rng=r))
    assert x.shape == (rows, k) and x.dtype == np.int64
    assert np.all(x.sum(axis=1) == n) and np.all(x[:, 0] == 0) and x.min() >= 0
    for i in range(1, min(k, 6)):
        assert moments_ok(x[:, i], n * p[i], n * p[i] * (1 - p[i]))[0], i
        for j in range(i + 1, min(k, 6)):
            prod = (x[:, i] - n * p[i]) * (x[:, j] - n * p[j])
            assert abs(prod.mean() + n * p[i] * p[j]) < 5 * prod.std() / np.sqrt(rows), (i, j)
    (z,), _ = _draw(lambda r: R.multinomial(0, p, size=(10,), rng=r))
    assert np.all(z == 0)


def test_dirichlet_rows_sum_to_one_with_beta_marginals(gpu):
    pytensor.config.floatX = "float64"
    a = np.array([0.5, 2.0, 3.5, 1.0, 0.2, 7.0])
    (x,), _ = _draw(lambda r: R.dirichlet(a, size=(N,), rng=r))
    assert x.shape == (N, a.size) and x.dtype == np.float64
    assert np.max(np.abs(x.sum(axis=1) - 1.0)) < 1e-12
    for j in range(a.size):
        assert st.kstest(x[:, j], st.beta(a[j], a.sum() - a[j]).cdf).pvalue > 1e-4, j
    (t,), _ = _draw(lambda r: R.dirichlet(np.full(50, 1e-3), size=(1000,), rng=r))
    assert np.all(np.isfinite(t)) and np.max(np.abs(t.sum(axis=1) - 1.0)) < 1e-12
    pytensor.config.floatX = "float32"
    (f,), _ = _draw(lambda r: R.dirichlet(np.ones(3, dtype="float32"), size=(100,), rng=r))
    assert f.dtype == np.float32 and np.max(np.abs(f.sum(axis=1) - 1.0)) < 1e-5


# ---- shapes / dtypes / parameter errors: the C linker's ---------------------------------------------------------------------
SHAPE_CASES = {
    "poisson": [lambda r: R.poisson(np.ones((2, 1)) * 3, size=None, rng=r), lambda r: R.poisson(np.ones(3), size=(4, 3), rng=r),
                lambda r: R.poisson(2.0, size=(0, 3), rng=r), lambda r: R.poisson(2.0, rng=r),
                lambda r: R.poisson(2.0, size=(5,), dtype="int32", rng=r)],
    "binomial": [lambda r: R.binomial(np.arange(3).reshape(3, 1), np.full(4, 0.5), rng=r),
                 lambda r: R.binomial(10, np.full(2, 0.5), size=(3, 2), rng=r), lambda r: R.binomial(10, 0.5, size=(0,), rng=r),
                 lambda r: R.binomial(10, 0.5, rng=r), lambda r: R.binomial(10, 0.5, size=(4,), dtype="int16", rng=r)],
    "negative_binomial": [lambda r: R.negative_binomial(np.full((2, 1), 3.0), np.full(3, 0.5), rng=r),
                          lambda r: R.negative_binomial(3.0, 0.5, size=(2, 2), rng=r),
                          lambda r: R.negative_binomial(3.0, 0.5, size=(0,), rng=r), lambda r: R.negative_binomial(3.0, 0.5, rng=r),
                          lambda r: R.negative_binomial(3.0, 0.5, size=(3,), dtype="int32", rng=r)],
    "geometric": [lambda r: R.geometric(np.full((2, 3), 0.3), rng=r), lambda r: R.geometric(np.full(3, 0.3), size=(2, 3), rng=r),
                  lambda r: R.geometric(0.3, size=(3, 0), rng=r), lambda r: R.geometric(0.3, rng=r),
                  lambda r: R.geometric(0.3, size=(3,), dtype="int32", rng=r)],
    "beta_binomial": [lambda r: R.betabinom(np.arange(2).reshape(2, 1), 2.0, np.ones(3), rng=r),
                      lambda r: R.betabinom(5, 2.0, 3.0, size=(2, 3), rng=r), lambda r: R.betabinom(5, 2.0, 3.0, size=(0,), rng=r),
                      lambda r: R.betabinom(5, 2.0, 3.0, rng=r), lambda r: R.betabinom(5, 2.0, 3.0, size=(2,), dtype="int32", rng=r)],
    "categorical": [lambda r: R.categorical(np.full((2, 3, 4), 0.25), rng=r), lambda r: R.categorical(np.full((3, 4), 0.25), size=(5, 3), rng=r),
                    lambda r: R.categorical(np.full(4, 0.25), size=(0,), rng=r), lambda r: R.categorical(np.full(4, 0.25), rng=r),
                    lambda r: R.categorical(np.full(4, 0.25), size=(6,), dtype="int32", rng=r)],
    "multinomial": [lambda r: R.multinomial(np.arange(1, 4).reshape(3, 1), np.full((2, 4), 0.25), rng=r),
                    lambda r: R.multinomial(np.arange(1, 4), np.full(4, 0.25), size=(2, 3), rng=r),
                    lambda r: R.multinomial(5, np.full(4, 0.25), size=(0,), rng=r), lambda r: R.multinomial(5, np.full(4, 0.25), rng=r),
                    lambda r: R.multinomial(5, np.full(4, 0.25), size=(3,), dtype="int32", rng=r)],
    "dirichlet": [lambda r: R.dirichlet(np.ones((2, 3, 4)), rng=r), lambda r: R.dirichlet(np.ones((3, 4)), size=(5, 3), rng=r),
                  lambda r: R.dirichlet(np.ones(4), size=(0, 2), rng=r), lambda r: R.dirichlet(np.ones(4), rng=r),
                  lambda r: R.dirichlet(np.ones(4), size=(3,), dtype="float32", rng=r)],
}


@pytest.mark.parametrize("name", list(SHAPE_CASES))
def test_shapes_and_dtypes_match_the_c_linker(gpu, name):
    pytensor.config.floatX = "float64"
    for i, build in enumerate(SHAPE_CASES[name]):
        (got,), _ = _draw(build)
        (exp,), _ = _draw(build, mode="CVM")
        assert got.shape == exp.shape and got.dtype == exp.dtype, (name, i, got.shape, exp.shape, got.dtype, exp.dtype)


EDGE_CASES = {
    "pois-neg": lambda r: R.poisson(-1.0, size=(3,), rng=r), "pois-nan": lambda r: R.poisson(np.nan, size=(3,), rng=r),
    "pois-big": lambda r: R.poisson(9.3e18, size=(3,), rng=r), "pois-0": lambda r: R.poisson(0.0, size=(3,), rng=r),
    "binom-n": lambda r: R.binomial(-1, 0.5, size=(3,), rng=r), "binom-p<0": lambda r: R.binomial(3, -0.1, size=(3,), rng=r),
    "binom-p>1": lambda r: R.binomial(3, 1.1, size=(3,), rng=r), "binom-pnan": lambda r: R.binomial(3, np.nan, size=(3,), rng=r),
    "binom-n0": lambda r: R.binomial(0, 0.5, size=(3,), rng=r), "binom-p0": lambda r: R.binomial(5, 0.0, size=(3,), rng=r),
    "binom-p1": lambda r: R.binomial(5, 1.0, size=(3,), rng=r),
    "binom-float-n": lambda r: R.binomial(np.array([5.0, 3.0]), 0.5, rng=r),
    "nb-n0": lambda r: R.negative_binomial(0.0, 0.5, size=(3,), rng=r), "nb-p0": lambda r: R.negative_binomial(2.0, 0.0, size=(3,), rng=r),
    "nb-p>1": lambda r: R.negative_binomial(2.0, 1.1, size=(3,), rng=r),
    "nb-too-large": lambda r: R.negative_binomial(2.5, 1e-300, size=(3,), rng=r),
    "nb-p1": lambda r: R.negative_binomial(2.5, 1.0, size=(3,), rng=r),
    "geo-0": lambda r: R.geometric(0.0, size=(3,), rng=r), "geo>1": lambda r: R.geometric(1.1, size=(3,), rng=r),
    "geo-nan": lambda r: R.geometric(np.nan, size=(3,), rng=r), "geo-1": lambda r: R.geometric(1.0, size=(3,), rng=r),
    "geo-tiny": lambda r: R.geometric(1e-300, size=(3,), rng=r),
    "bb-n": lambda r: R.betabinom(-1, 2.0, 3.0, size=(3,), rng=r), "bb-nonint": lambda r: R.betabinom(2.5, 2.0, 3.0, size=(3,), rng=r),
    "bb-a0": lambda r: R.betabinom(3, 0.0, 3.0, size=(3,), rng=r), "bb-b0": lambda r: R.betabinom(3, 2.0, 0.0, size=(3,), rng=r),
    "bb-float-n": lambda r: R.betabinom(np.array([3.0, 0.0]), 2.0, 3.0, rng=r),
    "mn-n": lambda r: R.multinomial(-1, [0.5, 0.5], rng=r), "mn-p": lambda r: R.multinomial(3, [-0.1, 1.1], rng=r),
    "mn-nan": lambda r: R.multinomial(3, [np.nan, 0.5], rng=r), "mn-sum": lambda r: R.multinomial(3, [0.7, 0.7, 0.1], rng=r),
    "mn-float-n": lambda r: R.multinomial(np.array([3.5]), [0.5, 0.5], rng=r),
    "mn-float-n-0d": lambda r: R.multinomial(np.array(3.0), [0.5, 0.5], rng=r),
    "mn-float-n-0d-size": lambda r: R.multinomial(np.array(3.0), [0.5, 0.5], size=(4,), rng=r),
    "mn-0.2-0.2": lambda r: R.multinomial(10, [0.2, 0.2], size=(5,), rng=r),
    "dir-neg": lambda r: R.dirichlet([-1.0, 1.0], rng=r), "dir-00": lambda r: R.dirichlet([0.0, 0.0], rng=r),
    "dir-nan": lambda r: R.dirichlet([np.nan, 1.0], rng=r), "dir-0-1": lambda r: R.dirichlet([0.0, 1.0], rng=r),
    "cat-size": lambda r: R.categorical(np.ones((3, 2)) / 2, size=(1,), rng=r),
    "cat-short-size": lambda r: R.categorical(np.ones((2, 3, 2)) / 2, size=(3,), rng=r),
}
DEGENERATE = {"pois-0", "binom-n0", "binom-p0", "binom-p1", "nb-p1", "geo-1", "geo-tiny", "dir-00", "dir-nan", "dir-0-1"}


def _outcome(build, mode):
    try:
        (x,), _ = _draw(build, mode=mode)
        return "ok", x
    except Exception as e:   # noqa: BLE001 — the exception TYPE is what is compared
        return type(e), None


@pytest.mark.parametrize("case", list(EDGE_CASES))
def test_parameter_edge_cases_match_the_c_linker(gpu, case):
    pytensor.config.floatX = "float64"
    got, gx = _outcome(EDGE_CASES[case], "CUDA")
    exp, ex = _outcome(EDGE_CASES[case], "CVM")
    assert got == exp, (case, got, exp)
    if case in DEGENERATE:
        np.testing.assert_array_equal(gx, ex)
    elif case == "mn-0.2-0.2":
        assert np.all(gx.sum(axis=1) == 10)
    elif case in ("mn-float-n", "mn-float-n-0d-size"):   # a float n of batched rows is truncated, as NumPy converts it
        assert np.all(gx.sum(axis=-1) == 3)


def test_invalid_parameters_raise_on_device_outputs_at_the_next_check(gpu):
    pytensor.config.floatX = "float64"
    from pytensor_b200.link.cuda import cuda_mode

    lam = pt.dvector("lam")
    rng = pytensor.shared(np.random.default_rng(1))
    f = pytensor.function([lam], R.poisson(lam, rng=rng), mode=cuda_mode(device_outputs=True))
    f(np.ones(4))
    f.vm.check_errors()
    f(np.array([1.0, -1.0]))
    with pytest.raises(ValueError, match="outside the distribution's domain"):
        f.vm.check_errors()
    f(np.ones(4))
    f.vm.check_errors()


def test_integer_n_beyond_float64_precision_is_refused(gpu):
    pytensor.config.floatX = "float64"
    with pytest.raises(ValueError, match="2\\*\\*53"):
        _draw(lambda r: R.binomial(2 ** 60, 0.5, size=(3,), rng=r))


def test_generator_protocol(gpu):
    pytensor.config.floatX = "float64"
    rng = pytensor.shared(np.random.default_rng(7))
    for x in (R.poisson(4.0, size=(1000,), rng=rng), R.categorical(np.full(5, 0.2), size=(1000,), rng=rng),
              R.dirichlet(np.ones(3), size=(100,), rng=rng)):
        f_same = pytensor.function([], x, mode="CUDA")
        np.testing.assert_array_equal(f_same(), f_same())
    for build in (lambda r: R.binomial(100, 0.3, size=(1000,), rng=r), lambda r: R.multinomial(30, np.full(4, 0.25), size=(300,), rng=r)):
        (a1, a2), _ = _draw(build, seed=5, n_calls=2)
        (b1, b2), _ = _draw(build, seed=5, n_calls=2)
        assert not np.array_equal(a1, a2)
        np.testing.assert_array_equal(a1, b1)
        np.testing.assert_array_equal(a2, b2)


def test_mixture_prior_predictive_end_to_end(gpu):
    """Dirichlet weights -> categorical assignments -> Poisson counts with the assigned rate, in one compiled function."""
    pytensor.config.floatX = "float64"
    rates = np.array([1.0, 8.0, 30.0])
    rng = pytensor.shared(np.random.default_rng(21))
    r1, w = R.dirichlet(np.array([50.0, 30.0, 20.0]) * 100, rng=rng).owner.outputs   # each draw takes the generator the
    r2, z = R.categorical(w, size=(N,), rng=r1).owner.outputs                       # previous one advanced, as in the
    y = R.poisson(pt.as_tensor(rates)[z], rng=r2)                                    # reference
    f = pytensor.function([], [w, z, y], mode="CUDA")
    names = [type(s.impl).__name__ for s in f.vm.executor.program.steps]
    assert names.count("RandomRowsNode") == 2 and names.count("RandomVariableNode") == 1, names
    assert not any("Host" in n or "Fallback" in n for n in names), names
    wv, zv, yv = f()
    assert abs(wv.sum() - 1.0) < 1e-12 and zv.shape == (N,) and yv.shape == (N,)
    for j in range(3):
        assert chi2_pvalue(yv[zv == j], st.poisson(rates[j])) > 1e-4, j
    hi = int(yv.max()) + 1
    pmf = sum(np.mean(zv == j) * st.poisson(rates[j]).pmf(np.arange(hi)) for j in range(3))
    pmf[-1] += 1.0 - pmf.sum()
    assert chi2_counts(np.bincount(yv, minlength=hi), N * pmf) > 1e-4
