"""CPU suite: PolyGamma, GammaIncInv, GammaIncCInv and BetaIncInv (codegen/scalar.py SPECIAL_HELPERS "polygamma",
"gammaincinv", "betaincinv") compiled for the host and run against the reference C linker, which evaluates these ops
through SciPy (scalar/math.py: none of the four has C code).

Regular domain: a, b in [0.05, 50], p in [1e-12, 1 - 1e-12], n in 0..12, x in [-40, 40] off the poles: float64 to rtol
1e-10, float32 within one float32 ulp.  Extreme regimes (a or b in {1e-3, 1e4}, p down to 1e-300, p near 1, x near the
poles): float64 to rtol 1e-8, and SciPy's forward function at the device's quantile gives back the smaller tail to 1e-10.
The documented differences (DESIGN.md section 9) are pinned as such."""

import subprocess
import sys

import numpy as np
import pytest
import scipy.special as sp

import test_scalar_table_cpu as tbl
from helpers import pytensor

import pytensor.tensor as pt

# sinpi / cospi (CUDA math functions) with the exact argument reduction the device versions have
SHIM_EXTRA = r"""
using std::signbit;
static inline double sinpi(double x) {
  const double n = std::nearbyint(2.0 * x), r = x - 0.5 * n;
  long long k = (long long)std::fmod(n, 4.0);
  if (k < 0) k += 4;
  const double s = std::sin(3.14159265358979323846 * r), c = std::cos(3.14159265358979323846 * r);
  return k == 0 ? s : k == 1 ? c : k == 2 ? -s : -c;
}
static inline double cospi(double x) { return sinpi(x + 0.5); }
"""


@pytest.fixture(autouse=True)
def _shim(monkeypatch):
    monkeypatch.setattr(tbl, "SHIM", tbl.SHIM + SHIM_EXTRA)


def _emulate(inputs, outputs, values, path):
    path.mkdir(exist_ok=True)  # a fresh directory per graph: dlopen caches handles by path
    return tbl._emulate(inputs, outputs, values, path)


def _within_one_ulp32(got, ref):
    got, ref = np.asarray(got, np.float32), np.asarray(ref, np.float32)
    same = (got == ref) | (np.isnan(got) & np.isnan(ref))
    fin = np.isfinite(ref) & np.isfinite(got)
    ulp = np.spacing(np.abs(ref[fin]))
    ok = same.copy()
    ok[fin] |= np.abs(got[fin].astype(np.float64) - ref[fin]) <= ulp
    assert ok.all(), list(zip(got[~ok][:5], ref[~ok][:5]))


def _regular(dtype, n=3000, seed=41):
    rng = np.random.default_rng(seed)
    a = np.exp(rng.uniform(np.log(0.05), np.log(50), n))
    b = np.exp(rng.uniform(np.log(0.05), np.log(50), n))
    p = np.exp(rng.uniform(np.log(1e-12), 0, n))
    p = np.clip(np.where(rng.random(n) < 0.5, p, 1 - p), 1e-12, 1 - 1e-12)
    k = rng.integers(0, 13, n)
    x = rng.uniform(-40, 40, n)
    x[np.abs(x - np.round(x)) < 1e-2] += 0.05
    return [v.astype(dtype) for v in (a, b, p, x)] + [k.astype("int64")]


def _check_regular(got, ref, dtype):
    if dtype == "float64":
        tbl._check(got, ref, rtol=1e-10)
    else:
        for g, r in zip(got, ref):
            assert g.dtype == np.float32 and np.asarray(r).dtype == np.float32
            _within_one_ulp32(g, r)


def _check_betaincinv_float32(got, ref32, av, bv, pv):
    """DESIGN.md section 9: SciPy's float32 betaincinv loop iterates in single precision and is accurate to about 3e-4
    relative only; the device computes in double and rounds once.  So the device must equal SciPy's float64 quantile
    rounded to float32 (to 1 ulp), and SciPy's float32 loop to 5e-4 where the quantile is a normal float32."""
    ref64 = sp.betaincinv(av.astype("float64"), bv.astype("float64"), pv.astype("float64"))
    _within_one_ulp32(got, ref64.astype(np.float32))
    normal = ref64 >= np.finfo(np.float32).tiny
    np.testing.assert_allclose(got[normal], ref32[normal], rtol=5e-4)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_regular_domain(tmp_path, dtype):
    pytensor.config.floatX = dtype
    av, bv, pv, xv, kv = _regular(dtype)
    a, b, p, x = (pt.vector(nm, dtype=dtype) for nm in "abpx")
    k = pt.vector("k", dtype="int64")
    got, ref = _emulate([a, p], [pt.gammaincinv(a, p), pt.gammainccinv(a, p)], [av, pv], tmp_path / "g")
    _check_regular(got, ref, dtype)
    got, ref = _emulate([a, b, p], [pt.betaincinv(a, b, p)], [av, bv, pv], tmp_path / "b")
    if dtype == "float64":
        _check_regular(got, ref, dtype)
    else:
        _check_betaincinv_float32(got[0], ref[0], av, bv, pv)
    got, ref = _emulate([k, x], [pt.polygamma(k, x)], [kv, xv], tmp_path / "p")
    _check_regular(got, ref, dtype)


EXTREME_P = np.array([1e-300, 1e-200, 1e-100, 1e-30, 1e-12, 1e-5, 0.01, 0.3, 0.5, 0.7, 0.99, 1 - 1e-5, 1 - 1e-12])


def _grid(*axes):
    return [g.ravel() for g in np.meshgrid(*axes, indexing="ij")]


def _smaller_tail_roundtrip(fwd_lower, fwd_upper, xhat, p, rtol):
    lower = p <= 0.5
    t = np.where(lower, p, 1 - p)
    back = np.where(lower, fwd_lower(xhat), fwd_upper(xhat))
    ok = (xhat == 0) | (np.abs(back - t) <= rtol * t)          # (x = 0: the quantile underflows, see edges)
    assert ok.all(), list(zip(xhat[~ok][:5], p[~ok][:5], back[~ok][:5]))


def test_gammaincinv_extreme_regimes(tmp_path):
    pytensor.config.floatX = "float64"
    av, pv = _grid(np.array([1e-3, 0.05, 1.0, 50.0, 1e4]), EXTREME_P)
    a, p = pt.dvectors("a", "p")
    (gi, gci), ref = _emulate([a, p], [pt.gammaincinv(a, p), pt.gammainccinv(a, p)], [av, pv], tmp_path / "g")
    tbl._check([gi, gci], ref, rtol=1e-8)
    _smaller_tail_roundtrip(lambda x: sp.gammainc(av, x), lambda x: sp.gammaincc(av, x), gi, pv, 1e-10)
    _smaller_tail_roundtrip(lambda x: sp.gammaincc(av, x), lambda x: sp.gammainc(av, x), gci, pv, 1e-10)


def test_gammaincinv_large_shape_is_limited_by_the_forward_series(tmp_path):
    """DESIGN.md section 9: at a = 1e6 the forward series and continued fraction (1024 terms) do not converge near
    x = a, so the device quantile is off by up to 3e-4 relative, where SciPy uses Temme's asymptotic expansion."""
    pytensor.config.floatX = "float64"
    pv = EXTREME_P
    av = np.full_like(pv, 1e6)
    a, p = pt.dvectors("a", "p")
    (gi, gci), (ri, rci) = _emulate([a, p], [pt.gammaincinv(a, p), pt.gammainccinv(a, p)], [av, pv], tmp_path / "g")
    np.testing.assert_allclose(gi, ri, rtol=1e-3)
    np.testing.assert_allclose(gci, rci, rtol=1e-3)
    assert np.max(np.abs(gi / ri - 1)) > 1e-8     # the difference is real: drop this test when it is fixed


def test_betaincinv_extreme_regimes(tmp_path):
    pytensor.config.floatX = "float64"
    par = np.array([1e-3, 0.5, 2.0, 1e4])
    av, bv, pv = _grid(par, par, EXTREME_P)
    a, b, p = pt.dvectors("a", "b", "p")
    (got,), (ref,) = _emulate([a, b, p], [pt.betaincinv(a, b, p)], [av, bv, pv], tmp_path / "b")
    # documented differences (DESIGN.md section 9): SciPy returns 0 for a = b = 1/2 and NaN for a = 2, b = 1e4 where
    # the quantile is below 1e-150
    scipy_quirk = ((av == 0.5) & (bv == 0.5) & (pv < 1e-100)) | np.isnan(ref)
    keep = ~scipy_quirk
    tbl._check([got[keep]], [ref[keep]], rtol=1e-8)
    assert np.isfinite(got[scipy_quirk]).all() and (got[scipy_quirk] > 0).all()
    # (round trip where x itself resolves the tail: not at the underflow floor, and not where 1 - x is quantised)
    rt = keep & (got > 2.3e-308) & (got < 0.5)
    _smaller_tail_roundtrip(lambda x: sp.betainc(av[rt], bv[rt], x), lambda x: sp.betaincc(av[rt], bv[rt], x),
                            got[rt], pv[rt], 1e-10)


# A small shape next to a large one (p > 1/2 puts the root within 1e-6 of x = 0 and between the mean and
# (a+1)/(a+b+2)), and a + b just below 171.62, where BetaInc's linear branch overflows tgamma(a) tgamma(b)
BETA_POINTS = [(0.0013417, 171.37, 0.8867), (0.00246589, 170.764, 0.9779), (170.623, 0.00181, 0.3618),
               (0.00118779, 4497.18, 0.993142), (0.00158509, 9343.59, 0.990772), (0.00293188, 3110.69, 0.985293)]


def _beta_sweep(n, seed):
    """Random (a, b, p) with a in [1e-3, 0.1], b in [10, 1e4], p in (0, 1); half of them mirrored to (b, a, p), and a
    quarter moved to a + b in [168, 171.6]; the fixed points above appended."""
    rng = np.random.default_rng(seed)
    a = np.exp(rng.uniform(np.log(1e-3), np.log(0.1), n))
    b = np.exp(rng.uniform(np.log(10), np.log(1e4), n))
    q = rng.random(n) < 0.25
    b[q] = rng.uniform(168, 171.6, q.sum()) - a[q]
    p = rng.uniform(0, 1, n)
    m = rng.random(n) < 0.5
    a, b = np.where(m, b, a), np.where(m, a, b)
    pa, pb, pp = (np.array(c) for c in zip(*BETA_POINTS))
    return np.concatenate([a, pa]), np.concatenate([b, pb]), np.concatenate([p, pp])


def test_betaincinv_small_shape_next_to_a_large_one(tmp_path):
    pytensor.config.floatX = "float64"
    av, bv, pv = _beta_sweep(4000, 43)
    a, b, p = pt.dvectors("a", "b", "p")
    (got,), (ref,) = _emulate([a, b, p], [pt.betaincinv(a, b, p)], [av, bv, pv], tmp_path / "b")
    rounds_to_one = ref == 1.0       # (x within 1e-16 of 1: both sides return 1)
    np.testing.assert_array_equal(got[rounds_to_one], 1.0)
    under = ref == 0.0               # (a denormal quantile: see test_documented_differences)
    np.testing.assert_array_equal(got[under], np.nextafter(np.finfo(np.float64).tiny, 0))
    rest = ~rounds_to_one & ~under
    tbl._check([got[rest]], [ref[rest]], rtol=1e-8)


def test_polygamma_near_poles_and_far_arguments(tmp_path):
    pytensor.config.floatX = "float64"
    # (SciPy's digamma reflects through tan(pi x) without an exact argument reduction, which costs it |x| eps / d of
    # relative accuracy at a distance d from a negative pole: the negative poles are approached to 1e-4 only)
    near = np.array([1e-4, 0.3, 0.5])
    xs = np.concatenate([(np.array([-12.0, -3.0, -1.0])[:, None] + np.concatenate([near, -near])).ravel(),
                         [1e-12, 1e-8, -1e-12, -1e-8, 1 + 1e-12, 1 - 1e-8, 1e-300, 1e3, 1e8, 1e15]])
    kv, xv = _grid(np.arange(0, 13), xs)
    k, x = pt.vector("k", dtype="int64"), pt.dvector("x")
    (got,), (ref,) = _emulate([k, x], [pt.polygamma(k, x)], [kv.astype("int64"), xv], tmp_path / "p")
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    # (where the shifted terms of a negative x cancel, both sides keep 1e-13 of the sum of their magnitudes)
    fr = xv - np.floor(xv)
    with np.errstate(all="ignore"):
        scale = sp.gamma(kv + 1.0) * (sp.zeta(kv + 1.0, np.where(fr > 0, fr, 1.0)) + sp.zeta(kv + 1.0, 1.0 - fr + (fr == 0)))
    scale = np.where((kv > 0) & (xv < 0) & np.isfinite(scale), scale, 0.0)
    fin = np.isfinite(ref)
    np.testing.assert_array_equal(got[~fin], ref[~fin])
    np.testing.assert_array_less(np.abs(got - ref)[fin], (1e-8 * np.abs(ref) + 1e-13 * scale)[fin] + 1e-300)


EDGES = {
    "gammaincinv": [(np.nan, 0.5), (0.0, 0.5), (-1.0, 0.5), (np.inf, 0.5), (2.0, np.nan), (2.0, -0.1), (2.0, 1.5),
                    (2.0, 0.0), (2.0, 1.0), (1e-3, 0.5), (1e-3, 1e-10)],
    "betaincinv": [(0.0, 1.0, 0.5), (-1.0, 1.0, 0.5), (1.0, 0.0, 0.5), (1.0, -2.0, 0.5), (2.0, 3.0, -0.1),
                   (2.0, 3.0, 1.5), (np.nan, 1.0, 0.5), (1.0, 1.0, np.nan), (2.0, 3.0, 0.0), (2.0, 3.0, 1.0),
                   (1e-3, 5.0, 0.3), (np.inf, 1.0, 0.5), (1.0, np.inf, 0.5)],
    "polygamma": [(0, 0.0), (0, -2.0), (1, 0.0), (2, 0.0), (1, -3.0), (2, -3.0), (3, -1.0), (1, -1.5), (171, 2.0),
                  (200, 50.0), (-1, 2.0), (0, np.nan), (1, np.inf), (2, np.inf), (1, -np.inf), (2, -np.inf)],
}


def test_edge_rows_match_the_c_linker_exactly(tmp_path):
    pytensor.config.floatX = "float64"
    a, b, p, x = pt.dvectors("a", "b", "p", "x")
    k = pt.vector("k", dtype="int64")
    av, pv = (np.array(c) for c in zip(*EDGES["gammaincinv"]))
    (gi, gci), (ri, rci) = _emulate([a, p], [pt.gammaincinv(a, p), pt.gammainccinv(a, p)], [av, pv], tmp_path / "g")
    for g, r in ((gi, ri), (gci, rci)):
        np.testing.assert_array_equal(np.isnan(g), np.isnan(r))
        np.testing.assert_allclose(g, r, rtol=1e-12)
    assert gi[9] != 0 and gi[10] == 0.0 and gi[8] == np.inf and gci[8] == 0.0 and gci[7] == np.inf
    av, bv, pv = (np.array(c) for c in zip(*EDGES["betaincinv"]))
    (g,), (r,) = _emulate([a, b, p], [pt.betaincinv(a, b, p)], [av, bv, pv], tmp_path / "b")
    np.testing.assert_array_equal(g, r)
    assert g[10] == np.nextafter(np.finfo(np.float64).tiny, 0)
    kv, xv = (np.array(c) for c in zip(*EDGES["polygamma"]))
    (g,), (r,) = _emulate([k, x], [pt.polygamma(k, x)], [kv.astype("int64"), xv], tmp_path / "p")
    np.testing.assert_allclose(g, r, rtol=1e-12)
    np.testing.assert_array_equal(np.signbit(g[np.isinf(g)]), np.signbit(r[np.isinf(r)]))


def test_documented_differences(tmp_path):
    """DESIGN.md section 9: for n >= 1 the Hurwitz zeta sums at most 256 shifted terms, so a non-integer x below about
    10 + n - 256 gives NaN where SciPy keeps summing; and SciPy's betaincinv returns 0 for a = b = 1/2 where the
    quantile underflows, the device the largest denormal, like SciPy for other shapes."""
    pytensor.config.floatX = "float64"
    k, x = pt.vector("k", dtype="int64"), pt.dvector("x")
    (g,), (r,) = _emulate([k, x], [pt.polygamma(k, x)], [np.array([1, 2, 0], "int64"), np.array([-300.5, -1000.5, -1000.5])],
                          tmp_path / "p")
    assert np.isnan(g[:2]).all() and np.isfinite(r[:2]).all()
    np.testing.assert_allclose(g[2], r[2], rtol=1e-12)           # (digamma reflects: no limit)
    a, b, p = pt.dvectors("a", "b", "p")
    # a = b = 1/2 (deep underflow), and a quantile just below DBL_MIN
    (g,), (r,) = _emulate([a, b, p], [pt.betaincinv(a, b, p)],
                          [np.array([0.5, 0.0022247066922887414]), np.array([0.5, 7830.642055829537]),
                           np.array([1e-300, 0.21121651625148097])], tmp_path / "b")
    assert (g == np.nextafter(np.finfo(np.float64).tiny, 0)).all() and (r == 0.0).all()


TRIP_VALUES = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, 1e-310, 1e300, -1e300, 0.5, 1.0, 2.0])

RUNNER = r"""
import ctypes, sys
import numpy as np
lib = ctypes.CDLL(sys.argv[1])
ins = [np.ascontiguousarray(np.load(f)) for f in sys.argv[3:]]
out = np.empty(len(ins[0]))
lib.run(ctypes.c_longlong(len(out)), *[a.ctypes.data_as(ctypes.c_void_p) for a in ins], out.ctypes.data_as(ctypes.c_void_p))
np.save(sys.argv[2], out)
"""


@pytest.mark.parametrize("op", ["gammaincinv", "gammainccinv", "betaincinv", "polygamma"])
def test_every_loop_ends_on_non_finite_tiny_and_huge_arguments(tmp_path, op):
    """NaN, +-inf, +-0, denormals and 1e300 in every argument position, in a separate process under a timeout: every
    loop of the helpers has a constant trip cap."""
    from pytensor_b200.codegen.scalar import single_op_program

    nin = 3 if op == "betaincinv" else 2
    in_dtypes = ["int64", "float64"] if op == "polygamma" else ["float64"] * nin
    op_name = {"gammaincinv": "GammaIncInv", "gammainccinv": "GammaIncCInv", "betaincinv": "BetaIncInv",
               "polygamma": "PolyGamma"}[op]
    lib = tbl._compile_body(single_op_program(op_name, in_dtypes, "float64"), tmp_path, op)
    orders = np.array([0, 1, 2, 5, 12, 170, 171, 1000, -1, -(1 << 62), 1 << 62])
    cols = _grid(orders, TRIP_VALUES) if op == "polygamma" else _grid(*[TRIP_VALUES] * nin)
    files = []
    for j, c in enumerate(cols):
        f = tmp_path / f"in{j}.npy"
        np.save(f, c.astype(in_dtypes[j]))
        files.append(str(f))
    out = tmp_path / "out.npy"
    subprocess.run([sys.executable, "-c", RUNNER, lib._name, str(out), *files], check=True, timeout=120)
    res = np.load(out)
    assert res.shape == cols[0].shape
