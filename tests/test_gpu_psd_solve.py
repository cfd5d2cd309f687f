"""CholeskySolve, positive-definite Solve and Blockwise(AllocDiag) on the device against the reference C linker.

Bars are the reference's own linalg-test tolerances: float64 rtol 1e-8, float32 rtol 1e-4 (absolute: the same fraction of
the largest expected magnitude); integer-grid systems, whose every partial sum is exact, must match bit for bit.  n = 128 is
the last size of the one-launch warp-per-column kernel; larger systems take the blocked triangular solves.  Every function
is called three times on two alternating input sets (eager, CUDA-graph capture, replay), and each call must return its own
input set's result."""

import os

import numpy as np
import pytest

import psd_cases
import psd_port
from helpers import pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu

DRY = os.environ.get("PTK_DRY") == "1"


def _tol(dtype):
    return 1e-4 if np.dtype(dtype) == np.float32 else 1e-8


def _check(ins, outs, sets, rtol=None, exact=False, node=None):
    """Compile with mode="CUDA" and "CVM"; call the CUDA function on sets[0], sets[1], sets[0] and compare each call with the
    C linker's result for its set.  Under PTK_DRY the lowered program is interpreted by the NumPy port instead."""
    f = pytensor.function(ins, outs, mode="CUDA")
    steps = {type(st.impl).__name__ for st in f.vm.executor.program.steps}
    if node is not None:
        assert node in steps, steps
    f_ref = pytensor.function(ins, outs, mode="CVM")
    exp = [f_ref(*[np.array(x, copy=True) for x in s]) for s in sets]
    order = [0, 1, 0] if len(sets) > 1 else [0, 0, 0]
    for call, k in enumerate(order):
        if DRY:
            got = psd_port.evaluate_program(f.vm.executor.program, [np.array(x, copy=True) for x in sets[k]])
        else:
            got = [np.array(g, copy=True) for g in f(*[np.array(x, copy=True) for x in sets[k]])]
        for g, e in zip(got, exp[k]):
            assert g.dtype == e.dtype and g.shape == e.shape, (g.dtype, e.dtype, g.shape, e.shape)
            if exact:
                np.testing.assert_array_equal(g, e)
            else:
                r = rtol if rtol is not None else _tol(e.dtype)
                fin = np.isfinite(e)
                scale = float(np.max(np.abs(e[fin]))) if fin.any() else 1.0
                np.testing.assert_allclose(g, e, rtol=r, atol=r * scale, equal_nan=True)
    if not DRY and "AssertNode" not in steps:
        assert f.vm.executor.last_from_graph, "the third call did not replay a captured CUDA graph"
    return f


def _factor(A, lower, dtype):
    L = np.linalg.cholesky(A)
    return np.ascontiguousarray(L if lower else np.swapaxes(L, -1, -2)).astype(dtype)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
@pytest.mark.parametrize("lower", [True, False])
@pytest.mark.parametrize("n", [1, 7, 32, 128, 129, 300, 1024])
def test_cho_solve_matches_the_c_linker(gpu, n, lower, dtype):
    C = pt.matrix("C", dtype=dtype)
    for b, shape in ((pt.vector("b", dtype=dtype), (n,)), (pt.matrix("b", dtype=dtype), (n, 5)),
                     (pt.matrix("b", dtype=dtype), (n, 64))):
        sets = []
        for seed in (0, 1):
            rng = np.random.default_rng(1000 * n + seed)
            sets.append([_factor(psd_cases.spd(rng, n), lower, dtype), rng.standard_normal(shape).astype(dtype)])
        _check([C, b], [pt.linalg.cho_solve((C, lower), b)], sets, node="CholeskySolveNode")


def _int_system(rng, n, lower, dtype, xmax=2):
    L = np.tril(rng.integers(-1, 2, (n, n)), -1) + np.diag(2.0 ** rng.integers(0, 3, n))
    X = rng.integers(-xmax, xmax + 1, (n, 3)).astype(np.float64)
    F = np.where(np.tril(np.ones((n, n), bool)), L, np.nan)          # NaN in the unreferenced triangle: never read
    return np.ascontiguousarray(F if lower else F.T).astype(dtype), (L @ (L.T @ X)).astype(dtype), X.astype(dtype)


@pytest.mark.parametrize("lower", [True, False])
@pytest.mark.parametrize("n,dtype", [(100, "float64"), (128, "float64"), (129, "float64"), (500, "float64"),
                                     (1000, "float64"), (128, "float32"), (129, "float32")])
def test_integer_grid_is_bit_exact(gpu, n, dtype, lower):
    C, b = pt.matrix("C", dtype=dtype), pt.matrix("b", dtype=dtype)
    xmax = 1 if dtype == "float32" else 2       # float32: every partial sum below 2^24
    systems = [_int_system(np.random.default_rng(n + s), n, lower, dtype, xmax) for s in (0, 1)]
    f = _check([C, b], [pt.linalg.cho_solve((C, lower), b)], [s[:2] for s in systems], exact=True)
    if not DRY:
        np.testing.assert_array_equal(f(*systems[1][:2])[0], systems[1][2])


def test_batches_broadcast_like_the_c_linker(gpu):
    rng = np.random.default_rng(5)
    G, B, n, k = 3, 4, 20, 6
    # factor (G, 1, n, n) against b (G, B, n, k)
    C4 = pt.tensor("C4", dtype="float64", shape=(None, 1, None, None))
    b4 = pt.tensor("b4", dtype="float64", shape=(None, None, None, None))
    sets = [[_factor(psd_cases.spd(np.random.default_rng(s), n, (G, 1)), True, "float64"), rng.standard_normal((G, B, n, k))]
            for s in (1, 2)]
    _check([C4, b4], [pt.linalg.cho_solve((C4, True), b4)], sets, node="CholeskySolveNode")
    # one factor for a batch of right-hand sides
    C, b3 = pt.dmatrix("C"), pt.dtensor3("b3")
    sets = [[_factor(psd_cases.spd(np.random.default_rng(s), n), False, "float64"), rng.standard_normal((B, n, k))]
            for s in (3, 4)]
    _check([C, b3], [pt.linalg.cho_solve((C, False), b3)], sets)
    # 70 000 small systems: more than a grid's y dimension holds
    Cb, bb = pt.dtensor3("Cb"), pt.dmatrix("bb")
    sets = [[_factor(psd_cases.spd(np.random.default_rng(s), 8, (70000,)), True, "float64"), rng.standard_normal((70000, 8))]
            for s in (5, 6)]
    _check([Cb, bb], [pt.linalg.cho_solve((Cb, True), bb, b_ndim=1)], sets)
    # a length-1 batch dimension that is not marked broadcastable is an error, as in the C linker
    Cr = pt.dtensor3("Cr")
    f = pytensor.function([Cr, bb], pt.linalg.cho_solve((Cr, True), bb, b_ndim=1), mode="CUDA")
    bad = [_factor(psd_cases.spd(rng, 8, (1,)), True, "float64"), rng.standard_normal((3, 8))]
    with pytest.raises(ValueError):
        pytensor.function([Cr, bb], pt.linalg.cho_solve((Cr, True), bb, b_ndim=1), mode="CVM")(*bad)
    if not DRY:
        with pytest.raises(ValueError):
            f(*bad)


@pytest.mark.parametrize("cdt,bdt", [("float32", "float64"), ("float64", "int64"), ("float32", "int64"), ("float32", "float32")])
def test_mixed_dtypes(gpu, cdt, bdt):
    C, b = pt.matrix("C", dtype=cdt), pt.matrix("b", dtype=bdt)
    sets = []
    for s in (7, 8):
        rng = np.random.default_rng(s)
        bv = rng.integers(-9, 10, (40, 3)) if bdt == "int64" else rng.standard_normal((40, 3))
        sets.append([_factor(psd_cases.spd(rng, 40), True, cdt), bv.astype(bdt)])
    out = pt.linalg.cho_solve((C, True), b)
    _check([C, b], [out], sets, rtol=_tol(out.dtype))


@pytest.mark.parametrize("n", [2, 40, 200])
def test_zero_pivot_and_non_finite_b_give_the_c_linker_inf_nan(gpu, n):
    C, b = pt.dmatrix("C"), pt.dmatrix("b")
    rng = np.random.default_rng(n)
    if n == 2:
        Cz = np.array([[0.0, 0.0], [1.0, 1.0]])
        sets = [[Cz, np.ones((2, 1))], [Cz, np.array([[1.0], [0.0]])]]
    else:
        L = _factor(psd_cases.spd(rng, n), True, "float64")
        Lz = L.copy()
        Lz[n // 3, n // 3] = 0.0
        bb = rng.standard_normal((n, 3))
        bb[5, 0], bb[n - 7, 1], bb[n // 2, 2] = np.inf, -np.inf, np.nan
        sets = [[Lz, rng.standard_normal((n, 2))], [L, bb]]
    f = _check([C, b], [pt.linalg.cho_solve((C, True), b)], sets)
    if not DRY:
        got = f(*sets[0])[0]
        ref = pytensor.function([C, b], pt.linalg.cho_solve((C, True), b), mode="CVM")(*sets[0])
        np.testing.assert_array_equal(np.isposinf(got), np.isposinf(ref))
        np.testing.assert_array_equal(np.isneginf(got), np.isneginf(ref))
        if n == 2:
            np.testing.assert_array_equal(got[:, 0], [np.inf, -np.inf])


@pytest.mark.parametrize("n", [9, 150])
@pytest.mark.parametrize("lower", [False, True])
def test_positive_definite_solve(gpu, n, lower):
    A, y = pt.dmatrix("A"), pt.dvector("y")
    x = pt.linalg.solve(A, y, assume_a="pos", lower=lower)
    sets = []
    for s in (10, 11):
        rng = np.random.default_rng(s)
        Av = psd_cases.spd(rng, n)
        Av[np.triu_indices(n, 1) if lower else np.tril_indices(n, -1)] = 7.0    # only the triangle `lower` names is read
        sets.append([Av, rng.standard_normal(n)])
    f = _check([A, y], [x], sets, node="PosSolveNode")
    # gradient (CholeskySolve after PyTensor's rewrites)
    _check([A, y], pt.grad(pt.sum(x**2), [A, y]), sets)
    # batched, one vector per matrix
    A3, y2 = pt.dtensor3("A3"), pt.dmatrix("y2")
    xb = pt.linalg.solve(A3, y2, assume_a="pos", lower=lower, b_ndim=1)
    bsets = [[psd_cases.spd(np.random.default_rng(s), n, (5,)), np.random.default_rng(s).standard_normal((5, n))] for s in (12, 13)]
    fb = _check([A3, y2], [xb], bsets, node="PosSolveNode")
    if DRY:
        return
    # not positive definite: the device gives NaN of b's shape where the C linker gives NaN of A's shape (DESIGN.md §9)
    bad = sets[0][0].copy()
    bad[n // 2, n // 2] = -50.0
    got = f(bad, sets[0][1])[0]
    assert got.shape == (n,) and np.all(np.isnan(got))
    ref = pytensor.function([A, y], x, mode="CVM")(bad, sets[0][1])
    assert ref.shape == (n, n) and np.all(np.isnan(ref))
    badb = bsets[0][0].copy()
    badb[2, n // 2, n // 2] = -50.0
    gotb = fb(badb, bsets[0][1])[0]
    assert np.all(np.isnan(gotb[2])) and np.all(np.isfinite(np.delete(gotb, 2, axis=0)))
    np.testing.assert_allclose(np.delete(gotb, 2, axis=0), np.linalg.solve(np.delete(bsets[0][0], 2, axis=0),
                                                                           np.delete(bsets[0][1], 2, axis=0)[..., None])[..., 0],
                               rtol=1e-8, atol=1e-10)


@pytest.mark.parametrize("n", [50, 400])
def test_gp_marginal_likelihood_gradient_and_prediction(gpu, n):
    ins, outs = psd_cases.gp_graph()
    _check(ins, outs, [psd_cases.gp_inputs(n, 12, s) for s in (20, 21)], rtol=1e-7, node="CholeskySolveNode")


def test_batched_mvnormal_logp_and_gradient(gpu):
    ins, outs = psd_cases.mvn_graph()
    _check(ins, outs, [psd_cases.mvn_inputs(64, 6, s) for s in (30, 31)], node="AllocDiagNode")


@pytest.mark.parametrize("offset", [0, 3, -2])
def test_blockwise_alloc_diag(gpu, offset):
    from pytensor.graph.replace import vectorize_graph

    v, x = pt.fvector("v"), pt.fmatrix("x")
    out = vectorize_graph(pt.diag(v, k=offset), {v: x})
    sets = [[np.random.default_rng(s).standard_normal((5, 9)).astype("float32")] for s in (40, 41)]
    _check([x], [out], sets, exact=True, node="AllocDiagNode")
