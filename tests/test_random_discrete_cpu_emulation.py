"""CPU suite: the discrete-count kernel and the row samplers of csrc/ptk_random.cu (count_kernel, multinomial_kernel,
categorical_kernel, dirichlet_kernel) run on the host through kernel_emulator, the warp kernels with one OS thread per
simulated lane.  Checked: distributions against scipy (chi-squared / KS, 20000 draws per case), draws independent of the
grid and block shape, and the error word set exactly for the parameters the reference rejects."""

import ctypes
import os
from ctypes import c_int, c_longlong, c_void_p

import numpy as np
import pytest
import scipy.stats as st

from discrete_fit import chi2_pvalue
from kernel_emulator import EmulatedKernel
from test_kernels_cpu_emulation import RNG_SHIM

CSRC = os.path.join(os.path.dirname(__file__), "..", "pytensor_b200", "csrc")
N = 20000
KEY, SEED = 0x0123456789abcdef, 0xfedcba9876543210

# warp votes and broadcasts for the threaded emulator (it already has __shfl_up/xor_sync and __popc)
WARP_RNG_SHIM = r"""
static unsigned emu_vote[32];
static inline unsigned __ballot_sync(unsigned, int pred) {
  const int w = threadIdx.x >> 5;
  pthread_barrier_wait(&emu_warp_bar[w]);
  if ((threadIdx.x & 31) == 0) emu_vote[w] = 0;
  pthread_barrier_wait(&emu_warp_bar[w]);
  if (pred) __atomic_fetch_or(&emu_vote[w], 1u << (threadIdx.x & 31), __ATOMIC_SEQ_CST);
  pthread_barrier_wait(&emu_warp_bar[w]);
  const unsigned r = __atomic_load_n(&emu_vote[w], __ATOMIC_SEQ_CST);
  pthread_barrier_wait(&emu_warp_bar[w]);
  return r;
}
template <typename T> static inline T __shfl_sync(unsigned, T v, int src) { return emu_exchange(v, (int)(threadIdx.x & ~31u) + src); }
"""


def _spans():
    text = open(os.path.join(CSRC, "ptk_random.cu")).read()
    a = text.index("struct Philox")
    b = text.index("}  // namespace")
    c = text.index("namespace {", b) + len("namespace {")
    d = text.index("}  // namespace", c)
    return text[a:b], text[c:d]


def _ptr(a):
    return c_void_p(a.ctypes.data)


@pytest.fixture(scope="module")
def kernels(tmp_path_factory):
    scalar, warp = _spans()
    ks = {}
    for name, out in (("count_kernel", "int64_t"), ("multinomial_kernel", "int64_t")):
        d = tmp_path_factory.mktemp(name)
        ks[name] = EmulatedKernel(RNG_SHIM + scalar, name, d, template_args=out, type_subst={"OUT": out})
    for name, out in (("categorical_kernel", "int64_t"), ("dirichlet_kernel", "double")):
        d = tmp_path_factory.mktemp(name)
        ks[name] = EmulatedKernel(RNG_SHIM + scalar + WARP_RNG_SHIM + warp, name, d, threaded=True, template_args=out,
                                  type_subst={"OUT": out})
    return ks


def _count(k, dist, n, params, grid=3, block=256, key=KEY, seed=SEED):
    out = np.full(n, -12345, dtype=np.int64)
    err = np.zeros(1, dtype=np.int32)
    ps, keep = [], []
    for p in list(params) + [None] * (3 - len(params)):
        if p is None:
            ps += [c_void_p(None), c_longlong(0)]
        else:
            p = np.ascontiguousarray(p, dtype=np.float64).reshape(-1)
            ps += [_ptr(p), c_longlong(0 if p.size == 1 else 1)]
            keep.append(p)
    k.launch(grid, block, [c_int(dist), _ptr(out), c_longlong(n), ctypes.c_uint64(key), ctypes.c_uint64(seed), *ps, _ptr(err)])
    return out, int(err[0])


def _rows(k, name, p, nv=None, grid=3, block=256, dtype=np.int64):
    p = np.ascontiguousarray(p, dtype=np.float64)
    rows, kk = p.shape
    err = np.zeros(1, dtype=np.int32)
    out = np.full((rows,) if name == "categorical_kernel" else (rows, kk), -7, dtype=dtype)
    args = [_ptr(out), c_longlong(rows), c_longlong(kk), ctypes.c_uint64(KEY), ctypes.c_uint64(SEED), _ptr(p), c_longlong(kk)]
    if name == "multinomial_kernel":
        nv = np.ascontiguousarray(np.broadcast_to(np.asarray(nv, dtype=np.float64), (rows,)))
        args += [_ptr(nv), c_longlong(1)]
    if name != "categorical_kernel":
        args.append(_ptr(err))
    k.launch(grid, block, args)
    return out, int(err[0])


COUNT_CASES = [
    (0, (0.5,), st.poisson(0.5)),
    (0, (9.99,), st.poisson(9.99)),
    (0, (10.0,), st.poisson(10.0)),
    (0, (37.5,), st.poisson(37.5)),
    (0, (1e4,), st.poisson(1e4)),
    (1, (10, 0.3), st.binom(10, 0.3)),
    (1, (1000, 0.5), st.binom(1000, 0.5)),
    (1, (1000, 0.97), st.binom(1000, 0.97)),
    (1, (40, 0.249), st.binom(40, 0.249)),
    (1, (40, 0.251), st.binom(40, 0.251)),
    (2, (2.5, 0.3), st.nbinom(2.5, 0.3)),
    (3, (0.5,), st.geom(0.5)),
    (3, (1e-4,), st.geom(1e-4)),
    (4, (10, 2.0, 3.0), st.betabinom(10, 2.0, 3.0)),
    (4, (100, 0.5, 0.5), st.betabinom(100, 0.5, 0.5)),
]


@pytest.mark.parametrize("dist,params,ref", COUNT_CASES, ids=[f"{c[0]}-{c[1]}" for c in COUNT_CASES])
def test_count_kernel_distributions(kernels, dist, params, ref):
    x, err = _count(kernels["count_kernel"], dist, N, [np.array([p]) for p in params])
    assert err == 0
    p = chi2_pvalue(x, ref)
    assert p > 1e-3, (params, p, x.mean(), ref.mean())


def test_count_kernel_per_element_parameters_and_launch_independence(kernels):
    k = kernels["count_kernel"]
    lam = np.repeat([0.3, 9.9, 10.1, 500.0], 5000)
    a, err = _count(k, 0, lam.size, [lam], grid=1)
    assert err == 0
    for j, l in enumerate([0.3, 9.9, 10.1, 500.0]):
        assert chi2_pvalue(a[j * 5000:(j + 1) * 5000], st.poisson(l)) > 1e-3, l
    np.testing.assert_array_equal(a, _count(k, 0, lam.size, [lam], grid=7)[0])
    np.testing.assert_array_equal(a, _count(k, 0, lam.size, [lam], grid=5, block=64)[0])
    b = _count(k, 1, 3000, [np.array([1000.0]), np.array([0.5])], grid=1)[0]
    np.testing.assert_array_equal(b, _count(k, 1, 3000, [np.array([1000.0]), np.array([0.5])], grid=7, block=64)[0])
    assert not np.array_equal(b, _count(k, 1, 3000, [np.array([1000.0]), np.array([0.5])], key=KEY ^ 1)[0])


INVALID = [
    (0, (-1.0,)), (0, (np.nan,)), (0, (9.3e18,)),
    (1, (-1.0, 0.5)), (1, (3.0, -0.1)), (1, (3.0, 1.1)), (1, (3.0, np.nan)), (1, (2.0 ** 60, 0.5)),
    (2, (0.0, 0.5)), (2, (2.0, 0.0)), (2, (2.0, 1.1)), (2, (2.5, 1e-300)), (2, (2.5, np.nan)),
    (3, (0.0,)), (3, (1.1,)), (3, (np.nan,)),
    (4, (-1.0, 2.0, 3.0)), (4, (2.5, 2.0, 3.0)), (4, (3.0, 0.0, 3.0)), (4, (3.0, 2.0, 0.0)), (4, (3.0, np.nan, 3.0)),
]
VALID = [
    (0, (0.0,), 0), (1, (0.0, 0.5), 0), (1, (5.0, 0.0), 0), (1, (5.0, 1.0), 5), (2, (2.5, 1.0), 0), (3, (1.0,), 1),
    (3, (1e-300,), 2 ** 63 - 1),
]


@pytest.mark.parametrize("dist,params", INVALID, ids=[f"{c[0]}-{c[1]}" for c in INVALID])
def test_count_kernel_flags_the_parameters_the_reference_rejects(kernels, dist, params):
    _, err = _count(kernels["count_kernel"], dist, 40, [np.array([p]) for p in params])
    assert err == 1


@pytest.mark.parametrize("dist,params,want", VALID, ids=[f"{c[0]}-{c[1]}" for c in VALID])
def test_count_kernel_boundary_values(kernels, dist, params, want):
    x, err = _count(kernels["count_kernel"], dist, 40, [np.array([p]) for p in params])
    assert err == 0 and np.all(x == want), x[:5]


def test_categorical_kernel(kernels):
    k = kernels["categorical_kernel"]
    # k = 5 with a zero-probability category, one uniform per row
    p = np.array([0.1, 0.0, 0.4, 0.3, 0.2])
    x, _ = _rows(k, "categorical_kernel", np.tile(p, (N, 1)), grid=1)
    assert not np.any(x == 1)
    counts = np.bincount(x, minlength=5)
    assert counts[5:].sum() == 0 and st.chisquare(counts[[0, 2, 3, 4]], N * p[[0, 2, 3, 4]]).pvalue > 1e-3
    np.testing.assert_array_equal(x[:2000], _rows(k, "categorical_kernel", np.tile(p, (2000, 1)), grid=7, block=64)[0])
    # k = 33 crosses a 32-wide chunk; p summing to 0.5 yields k half the time
    p33 = np.full(33, 1.0 / 66)
    y, _ = _rows(k, "categorical_kernel", np.tile(p33, (4000, 1)))
    assert abs(np.mean(y == 33) - 0.5) < 5 * np.sqrt(0.25 / 4000)
    assert st.chisquare(np.bincount(y, minlength=34)[:33]).pvalue > 1e-3


def test_multinomial_kernel(kernels):
    k = kernels["multinomial_kernel"]
    p = np.array([0.2, 0.0, 0.5, 0.3])
    x, err = _rows(k, "multinomial_kernel", np.tile(p, (5000, 1)), nv=np.full(5000, 40.0), grid=1)
    assert err == 0 and np.all(x.sum(axis=1) == 40) and np.all(x[:, 1] == 0)
    for j in (0, 2, 3):
        assert chi2_pvalue(x[:, j], st.binom(40, p[j])) > 1e-3
    np.testing.assert_array_equal(x[:1000], _rows(k, "multinomial_kernel", np.tile(p, (1000, 1)), nv=40.0, grid=7,
                                                  block=64)[0])
    # NumPy's algorithm: the last category takes the remainder whatever p[-1] is
    y, err = _rows(k, "multinomial_kernel", np.tile([0.2, 0.2], (4000, 1)), nv=10.0)
    assert err == 0 and np.all(y.sum(axis=1) == 10) and chi2_pvalue(y[:, 0], st.binom(10, 0.2)) > 1e-3
    assert _rows(k, "multinomial_kernel", np.zeros((3, 2)), nv=0.0)[0].sum() == 0
    for bad_p, bad_n in (([0.5, 0.5], -1.0), ([-0.1, 1.1], 3.0), ([np.nan, 0.5], 3.0), ([0.7, 0.7, 0.1], 3.0),
                         ([0.5, 1.5], 3.0)):
        assert _rows(k, "multinomial_kernel", np.array([bad_p]), nv=bad_n)[1] == 1, (bad_p, bad_n)


def test_dirichlet_kernel(kernels):
    k = kernels["dirichlet_kernel"]
    a = np.array([0.5, 2.0, 3.5, 1.0, 0.2])
    rows = N // a.size
    x, err = _rows(k, "dirichlet_kernel", np.tile(a, (rows, 1)), grid=1, dtype=np.float64)
    assert err == 0 and np.all(np.isfinite(x)) and np.max(np.abs(x.sum(axis=1) - 1.0)) < 1e-12
    for j in range(a.size):
        assert st.kstest(x[:, j], st.beta(a[j], a.sum() - a[j]).cdf).pvalue > 1e-3, j
    np.testing.assert_array_equal(x[:500], _rows(k, "dirichlet_kernel", np.tile(a, (500, 1)), grid=7, block=64,
                                                 dtype=np.float64)[0])
    # k = 40 spans two chunks per lane; alpha = 1e-3 underflows as direct gammas but not in log space
    t, _ = _rows(k, "dirichlet_kernel", np.full((64, 40), 1e-3), dtype=np.float64)
    assert np.all(np.isfinite(t)) and np.max(np.abs(t.sum(axis=1) - 1.0)) < 1e-12
    z, err = _rows(k, "dirichlet_kernel", np.array([[0.0, 0.0], [0.0, 1.0], [np.nan, 1.0]]), dtype=np.float64)
    assert err == 0 and z[0].tolist() == [0.0, 0.0] and z[1].tolist() == [0.0, 1.0] and np.all(np.isnan(z[2]))
    assert _rows(k, "dirichlet_kernel", np.array([[-1.0, 1.0]]), dtype=np.float64)[1] == 1
