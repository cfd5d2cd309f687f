"""Glue ops (views, alloc, basic/advanced indexing) — bit-exact against the C linker (BASELINE.json north_star:
"bit-exact for Subtensor/indexing ops")."""

import numpy as np
import pytest

from helpers import compare_cuda_and_cvm, pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu


def test_subtensor_views_bit_exact(gpu):
    rng = np.random.default_rng(31)
    x = pt.dtensor3("x")
    i = pt.lscalar("i")
    xv = rng.standard_normal((9, 10, 11))
    outs = [x[1], x[:, 2], x[..., -1], x[1:7:2, ::-1, 3:], x[i], x[i:, :i], x[::-2, 1, ::3], x[-3:, -2:, 5]]
    compare_cuda_and_cvm([x, i], outs, [xv, np.int64(4)], exact=True)


def test_set_and_inc_subtensor(gpu):
    rng = np.random.default_rng(32)
    x = pt.dmatrix("x")
    y = pt.dvector("y")
    xv, yv = rng.standard_normal((12, 7)), rng.standard_normal(7)
    outs = [pt.set_subtensor(x[2], y), pt.inc_subtensor(x[3:9:2], y), pt.set_subtensor(x[:, 1:3], 5.0),
            pt.inc_subtensor(x[::-1][0], y)]
    compare_cuda_and_cvm([x, y], outs, [xv, yv], exact=True)


def test_take_and_scatter_add(gpu):
    rng = np.random.default_rng(33)
    theta = pt.dvector("theta")
    th2 = pt.dmatrix("th2")
    g = pt.lvector("g")
    tv = rng.standard_normal(64)
    t2 = rng.standard_normal((32, 64))
    gv = rng.integers(0, 64, size=5000)
    r = pt.dvector("r")
    rv = rng.standard_normal(5000)
    # gathers are bit-exact
    compare_cuda_and_cvm([theta, th2, g], [theta[g], th2[:, g], th2.T[g[:10]]], [tv, t2, gv], exact=True)
    # scatter-add with duplicates: fp add order differs (atomics) -> tolerance, not bit-exact
    outs = [pt.inc_subtensor(pt.zeros_like(theta)[g], r), pt.set_subtensor(theta[g[:3]], r[:3])]
    compare_cuda_and_cvm([theta, g, r], outs, [tv, gv, rv], rtol=1e-9, atol=1e-9)


def test_take_negative_and_oob(gpu):
    x = pt.dvector("x")
    g = pt.lvector("g")
    f = pytensor.function([x, g], x[g], mode="CUDA")
    np.testing.assert_array_equal(f(np.arange(5.0), np.array([-1, 0, -5])), [4.0, 0.0, 0.0])
    with pytest.raises(IndexError):
        f(np.arange(5.0), np.array([0, 5]))


def test_alloc_shape_reshape_join(gpu):
    rng = np.random.default_rng(34)
    x = pt.dmatrix("x")
    v = pt.dvector("v")
    xv, vv = rng.standard_normal((6, 8)), rng.standard_normal(8)
    outs = [pt.alloc(v, 3, 8), pt.zeros((x.shape[0], 4)) + 1.5, x.reshape((8, 6)), x.T.reshape((-1,)),
            pt.concatenate([x, x * 2], axis=0), pt.concatenate([x, v[None, :]], axis=0), x.shape[0] * x.shape[1],
            pt.ones_like(x), x.dimshuffle(1, "x", 0), x.flatten()]
    compare_cuda_and_cvm([x, v], outs, [xv, vv], exact=True)


def test_shared_variable_and_updates(gpu):
    w = pytensor.shared(np.arange(6.0).reshape(2, 3), name="w")
    x = pt.dmatrix("x")
    f = pytensor.function([x], (w * x).sum(), updates={w: w + x}, mode="CUDA")
    xv = np.ones((2, 3))
    assert f(xv) == 15.0
    np.testing.assert_array_equal(w.get_value(), np.arange(6.0).reshape(2, 3) + 1)
    assert f(xv) == 21.0


def test_device_io(gpu):
    import torch

    from pytensor_b200.link.cuda import cuda_mode

    x = pt.fmatrix("x")
    f = pytensor.function([x], pt.tanh(x) * 2, mode=cuda_mode(device_outputs=True), trust_input=True)
    xv = torch.arange(12, dtype=torch.float32, device="cuda").reshape(3, 4) / 10
    out = f(xv)
    assert isinstance(out, torch.Tensor) and out.is_cuda
    np.testing.assert_allclose(out.cpu().numpy(), np.tanh(xv.cpu().numpy()) * 2, rtol=1e-6)


def test_unsupported_op_is_a_compile_time_error(gpu):
    x = pt.dmatrix("x")
    with pytest.raises(NotImplementedError):
        pytensor.function([x], pt.linalg.inv(x), mode="CUDA")


def test_cholesky_and_solve_triangular(gpu):
    import scipy.linalg

    rng = np.random.default_rng(35)
    A = pt.dmatrix("A")
    b = pt.dmatrix("b")
    Av = rng.standard_normal((48, 48))
    Av = Av @ Av.T + 48 * np.eye(48)
    bv = rng.standard_normal((48, 5))
    L = pt.linalg.cholesky(A)
    outs = [L, pt.linalg.cholesky(A, lower=False), pt.linalg.solve_triangular(L, b, lower=True),
            pt.linalg.solve_triangular(L.T, b, lower=False), pt.linalg.solve_triangular(L, b[:, 0], lower=True,
                                                                                         unit_diagonal=True)]
    compare_cuda_and_cvm([A, b], outs, [Av, bv], rtol=1e-8, atol=1e-8)
    # indefinite -> all-NaN (tests/tensor/linalg/test_decomposition/test_cholesky.py:57-69)
    f = pytensor.function([A], L, mode="CUDA")
    assert np.all(np.isnan(f(-np.eye(4))))
    del scipy


@pytest.mark.parametrize("n,nrhs", [(129, 3), (300, 70), (512, 1)])
def test_blocked_cholesky_and_solve_triangular(gpu, n, nrhs):
    # n > 128 takes the blocked (64-wide panel + GEMM trailing update) path
    rng = np.random.default_rng(36)
    A = pt.dmatrix("A")
    b = pt.dmatrix("b")
    Av = rng.standard_normal((n, n))
    Av = Av @ Av.T / n + np.eye(n)
    bv = rng.standard_normal((n, nrhs))
    L = pt.linalg.cholesky(A)
    U = pt.linalg.cholesky(A, lower=False)
    outs = [L, U, pt.linalg.solve_triangular(L, b, lower=True), pt.linalg.solve_triangular(U, b, lower=False),
            pt.linalg.solve_triangular(L.T, b, lower=False), pt.linalg.solve_triangular(L, b, lower=True,
                                                                                         unit_diagonal=True)]
    compare_cuda_and_cvm([A, b], outs, [Av, bv], rtol=1e-7, atol=1e-8)
    f = pytensor.function([A], L, mode="CUDA")
    bad = Av.copy()
    bad[n // 2, n // 2] = -5.0
    assert np.all(np.isnan(f(bad)))


def test_batched_cholesky_blockwise(gpu):
    rng = np.random.default_rng(37)
    A = pt.dtensor3("A")
    Av = rng.standard_normal((6, 9, 9))
    Av = Av @ Av.transpose(0, 2, 1) + 9 * np.eye(9)
    compare_cuda_and_cvm([A], [pt.linalg.cholesky(A)], [Av], rtol=1e-9, atol=1e-10)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_row_batched_gather_and_deterministic_scatter_add(gpu, dtype):
    # cfg-5 pattern: theta[:, g] (B,J)->(B,n) and its transpose, zeros(B,J)[:, g] += r(B,n); the scatter-add is a
    # segmented reduction in ascending-index order => equal to np.add.at up to the last bit for float64
    rng = np.random.default_rng(38)
    theta = pt.tensor("theta", dtype=dtype, shape=(None, None))
    r = pt.tensor("r", dtype=dtype, shape=(None, None))
    g = pt.lvector("g")
    tv = rng.standard_normal((300, 64)).astype(dtype)
    rv = rng.standard_normal((300, 1024)).astype(dtype)
    gv = rng.integers(0, 64, size=1024)
    compare_cuda_and_cvm([theta, g], [theta[:, g]], [tv, gv], exact=True)
    out = pt.inc_subtensor(pt.zeros_like(theta)[:, g], r)
    f, got = compare_cuda_and_cvm([theta, r, g], [out], [tv, rv, gv], rtol=1e-6 if dtype == "float32" else 1e-13,
                                  atol=1e-5 if dtype == "float32" else 1e-12)
    # the scatter-add runs inside a row-fused region (codegen/rowfuse.py), so the bit-exact check below covers its
    # lane-ordered accumulation
    assert any(type(s.impl).__name__ == "RowRegionNode" for s in f.vm.executor.program.steps)
    ref = np.zeros_like(tv)
    np.add.at(ref, (slice(None), gv), rv)
    np.testing.assert_array_equal(got[0], ref)  # deterministic: same accumulation order as np.add.at
