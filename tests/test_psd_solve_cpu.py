"""CholeskySolve, positive-definite Solve and Blockwise(AllocDiag) without a GPU.

a. Lowering: the Gaussian-process and batched-MvNormal graphs and their gradients compile under mode="CUDA" into programs
   holding CholeskySolveNode / PosSolveNode / AllocDiagNode, and their launch logic runs in trace-only mode; every other
   Solve variant stays a compile-time error.
b. Port oracle: those lowered programs, interpreted node by node in NumPy (tests/psd_port.py), match the C linker.
c. Emulator: `potrs_small_kernel` (csrc/ptk_linalg.cu) runs on the host with real warp shuffles and shared memory and is
   compared with scipy.linalg.lapack.?potrs: bit-exactly on integer-grid factors (every partial sum an integer below 2^24,
   power-of-two pivots), to 1e-12 on random SPD float64, with NaN in the unreferenced triangle, with ?potrs's inf / NaN
   pattern for a zero pivot or non-finite b, with broadcast factor strides, and bit-identically across launch shapes."""

import ctypes
import os
import re
from ctypes import c_int, c_longlong, c_void_p

import numpy as np
import pytest
import scipy.linalg.lapack as lapack

import psd_cases
import psd_port
from helpers import pytensor
from kernel_emulator import EmulatedKernel, extract_static_kernel

import pytensor.tensor as pt
from pytensor_b200.precompile import trace_function

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytensor_b200", "csrc")


# ---- lowering and port oracle ---------------------------------------------------------------------------------------------
def _steps(f):
    return {type(st.impl).__name__ for st in f.vm.executor.program.steps}


def _trace(f, vals):
    """trace_function with shape assertions waived: in trace-only mode every device-computed value is a placeholder, and
    these graphs fuse their broadcast checks into device kernels."""
    from pytensor_b200.vm.nodes_basic import AssertNode
    from pytensor_b200.vm.values import Val

    old = AssertNode.run
    AssertNode.run = lambda self, v: [Val(h=v[0].h, d=v[0].d)]
    try:
        return trace_function(f, [np.array(x, copy=True) for x in vals])
    finally:
        AssertNode.run = old


def _lower_and_port(ins, outs, vals, node, rtol=1e-9):
    f = pytensor.function(ins, outs, mode="CUDA")
    assert node in _steps(f), _steps(f)
    _trace(f, vals)
    exp = pytensor.function(ins, outs, mode="CVM")(*[np.array(x, copy=True) for x in vals])
    got = psd_port.evaluate_program(f.vm.executor.program, [np.array(x, copy=True) for x in vals])
    for g, e in zip(got, exp):
        assert g.dtype == e.dtype and g.shape == e.shape
        np.testing.assert_allclose(g, e, rtol=rtol, atol=rtol * max(1.0, float(np.max(np.abs(e)))))
    return f


def test_gp_likelihood_gradient_and_prediction_lower():
    ins, outs = psd_cases.gp_graph()
    f = _lower_and_port(ins, outs, psd_cases.gp_inputs(40, 6, 1), "CholeskySolveNode")
    forms = {(st.impl.lower, st.impl.b_ndim, st.impl.overwrite_b) for st in f.vm.executor.program.steps
             if type(st.impl).__name__ == "CholeskySolveNode"}
    assert forms == {(True, 1, False), (True, 1, True)}


def test_batched_mvnormal_gradient_lowers_alloc_diag():
    ins, outs = psd_cases.mvn_graph()
    _lower_and_port(ins, outs, psd_cases.mvn_inputs(8, 5, 2), "AllocDiagNode")


def test_cho_solve_and_pos_solve_lower():
    rng = np.random.default_rng(3)
    A, y = pt.dmatrix("A"), pt.dvector("y")
    Av, yv = psd_cases.spd(rng, 9), rng.standard_normal(9)
    _lower_and_port([A, y], [pt.linalg.cho_solve((A, True), y)], [np.linalg.cholesky(Av), yv], "CholeskySolveNode")
    x = pt.linalg.solve(A, y, assume_a="pos")
    f = _lower_and_port([A, y], [x], [Av, yv], "PosSolveNode")
    assert "CholeskyNode" not in _steps(f)
    _lower_and_port([A, y], [pt.grad(pt.sum(x**2), y), pt.grad(pt.sum(x**2), A)], [Av, yv], "CholeskySolveNode")
    A3, y2 = pt.dtensor3("A3"), pt.dmatrix("y2")
    _lower_and_port([A3, y2], [pt.linalg.solve(A3, y2, assume_a="pos", b_ndim=1)],
                    [psd_cases.spd(rng, 7, (4,)), rng.standard_normal((4, 7))], "PosSolveNode")


@pytest.mark.parametrize("offset", [0, 2, -1])
def test_blockwise_alloc_diag_any_offset(offset):
    from pytensor.graph.replace import vectorize_graph

    v, x = pt.dvector("v"), pt.dmatrix("x")
    out = vectorize_graph(pt.diag(v, k=offset), {v: x})      # Blockwise(AllocDiag) over the rows of x
    _lower_and_port([x], [out * 1.5], [np.arange(12.0).reshape(3, 4) + 1], "AllocDiagNode", rtol=0)


def test_mixed_dtypes_follow_the_op_output_dtype():
    rng = np.random.default_rng(4)
    C, b = pt.fmatrix("C"), pt.lvector("b")
    out = pt.linalg.cho_solve((C, True), b)
    assert out.dtype == "float64"
    Cv = np.linalg.cholesky(psd_cases.spd(rng, 6)).astype("float32")
    _lower_and_port([C, b], [out], [Cv, rng.integers(-5, 5, 6)], "CholeskySolveNode", rtol=1e-6)


@pytest.mark.parametrize("assume_a", ["gen", "sym"])
def test_other_solves_stay_unsupported(assume_a):
    from pytensor_b200.link.cuda.lower import UnsupportedOp

    A, y = pt.dmatrix("A"), pt.dvector("y")
    with pytest.raises(UnsupportedOp):
        pytensor.function([A, y], pt.linalg.solve(A, y, assume_a=assume_a), mode="CUDA")


# ---- the small-system kernel on the emulator ------------------------------------------------------------------------------
POTRS_SHIM = r"""
template <typename T> static inline T __shfl_sync(unsigned, T v, int src) { return emu_exchange(v, (int)((threadIdx.x & ~31u) + src)); }
"""


class _Batch(ctypes.Structure):
    _fields_ = [("nd", c_int), ("shape", c_longlong * 8), ("stride", c_longlong * 8)]


@pytest.fixture(scope="module")
def potrs_kernels(tmp_path_factory):
    path = os.path.join(CSRC, "ptk_linalg.cu")
    text = open(path).read()
    head = text[text.index("constexpr int POTRS_MAX_DIMS"):text.index("// small path: A = C C^T")]
    src = POTRS_SHIM + head + extract_static_kernel(path, "potrs_small_kernel")
    ks = {}
    for ctype in ("float", "double"):
        d = tmp_path_factory.mktemp(ctype)
        ks[ctype] = EmulatedKernel(src, "potrs_small_kernel", d, threaded=True, template_args=ctype,
                                   type_subst={"T": ctype}, warp_shim=True)
    return ks


def _run(k, C, B, lower, shape, strides, grid=2, block=64):
    """Solve B (batch..., n, nrhs) in place with factors C (strides in elements) on the emulated kernel."""
    n, nrhs = B.shape[-2], B.shape[-1]
    bat = _Batch(len(shape), (c_longlong * 8)(*shape), (c_longlong * 8)(*strides))
    pairs = int(np.prod(shape, dtype=np.int64)) * nrhs
    k.launch(grid, block, [c_void_p(C.ctypes.data), c_void_p(B.ctypes.data), c_longlong(n), c_longlong(nrhs), c_int(lower), bat,
                           c_longlong(pairs)])
    return B


def _potrs(C, b, lower):
    f = lapack.spotrs if C.dtype == np.float32 else lapack.dpotrs
    x, info = f(C, b, lower=lower)
    assert info == 0
    return x


def _int_factor(rng, n, lower, dtype):
    """Integer entries in {-1, 0, 1}, pivots in {1, 2, 4}, NaN in the other triangle."""
    L = np.tril(rng.integers(-1, 2, (n, n)), -1) + np.diag(2.0 ** rng.integers(0, 3, n))
    F = np.where(np.tril(np.ones((n, n), bool)), L, np.nan)
    return np.ascontiguousarray(F if lower else F.T).astype(dtype), L


@pytest.mark.parametrize("ctype", ["float", "double"])
@pytest.mark.parametrize("lower", [1, 0])
@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 64, 127, 128])
def test_integer_grid_is_bit_exact(potrs_kernels, ctype, lower, n):
    dtype = np.float32 if ctype == "float" else np.float64
    rng = np.random.default_rng(100 + n + 7 * lower)
    for nrhs in (1, 3, 33):
        F, L = _int_factor(rng, n, lower, dtype)
        X = rng.integers(-2, 3, (n, nrhs)).astype(np.float64)
        Bm = (L @ (L.T @ X)).astype(dtype)        # every partial sum of both sweeps is an integer below 2^24
        got = _run(potrs_kernels[ctype], F, Bm[None].copy(), lower, [1], [0])[0]
        np.testing.assert_array_equal(got, X.astype(dtype))
        np.testing.assert_array_equal(got, _potrs(F, Bm, lower))


@pytest.mark.parametrize("lower", [1, 0])
def test_random_spd_float64_and_broadcast_factor_strides(potrs_kernels, lower):
    rng = np.random.default_rng(7)
    n, nrhs = 45, 5
    A = psd_cases.spd(rng, n, (3,))
    Lf = np.linalg.cholesky(A)
    F = np.ascontiguousarray(Lf if lower else np.swapaxes(Lf, -1, -2))
    F[:, ~(np.tril if lower else np.triu)(np.ones((n, n), bool))] = np.nan   # the unreferenced triangle is never read
    # output batch (3, 2): system (i, j) uses factor i (stride n*n along the first axis, 0 along the second)
    B = rng.standard_normal((3, 2, n, nrhs))
    got = _run(potrs_kernels["double"], F, B.copy(), lower, [3, 2], [n * n, 0])
    for i in range(3):
        for j in range(2):
            want = _potrs(F[i], B[i, j], lower)
            np.testing.assert_allclose(got[i, j], want, rtol=1e-12, atol=1e-12 * np.abs(want).max())
            np.testing.assert_allclose(got[i, j], np.linalg.solve(A[i], B[i, j]), rtol=1e-12,
                                       atol=1e-12 * np.abs(want).max())
    # the transposed broadcast: factor j along the second axis
    got2 = _run(potrs_kernels["double"], F[:2].copy(), B.copy(), lower, [3, 2], [0, n * n])
    for i in range(3):
        for j in range(2):
            np.testing.assert_allclose(got2[i, j], _potrs(F[j], B[i, j], lower), rtol=1e-12, atol=1e-12)


def test_results_do_not_depend_on_the_launch_shape(potrs_kernels):
    rng = np.random.default_rng(8)
    n, nrhs = 70, 3
    A = psd_cases.spd(rng, n, (5,))
    F = np.linalg.cholesky(A)
    B = rng.standard_normal((5, n, nrhs))
    runs = [_run(potrs_kernels["double"], F, B.copy(), 1, [5], [n * n], grid=g, block=bl) for g, bl in ((1, 32), (2, 64), (7, 256))]
    for r in runs[1:]:
        np.testing.assert_array_equal(r, runs[0])


@pytest.mark.parametrize("lower", [1, 0])
def test_zero_pivot_and_non_finite_b_follow_potrs(potrs_kernels, lower):
    C = np.array([[0.0, 0.0], [1.0, 1.0]])
    F = np.ascontiguousarray(C if lower else C.T)
    got = _run(potrs_kernels["double"], F, np.ones((1, 2, 1)), lower, [1], [0])[0]
    np.testing.assert_array_equal(got, _potrs(F, np.ones((2, 1)), lower))
    if lower:
        np.testing.assert_array_equal(got[:, 0], [np.inf, -np.inf])
    rng = np.random.default_rng(9)
    n = 40
    L = np.linalg.cholesky(psd_cases.spd(rng, n))
    cases = []
    Lz = L.copy()
    Lz[17, 17] = 0.0
    cases.append((Lz, rng.standard_normal((n, 2))))
    b = rng.standard_normal((n, 3))
    b[5, 0], b[30, 1], b[12, 2] = np.inf, -np.inf, np.nan
    cases.append((L, b))
    for Lc, bc in cases:
        F = np.ascontiguousarray(Lc if lower else Lc.T)
        with np.errstate(all="ignore"):
            want = _potrs(F, bc, lower)
        got = _run(potrs_kernels["double"], F, bc[None].copy(), lower, [1], [0])[0]
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        np.testing.assert_array_equal(np.isposinf(got), np.isposinf(want))
        np.testing.assert_array_equal(np.isneginf(got), np.isneginf(want))
        fin = np.isfinite(want)
        np.testing.assert_allclose(got[fin], want[fin], rtol=1e-10, atol=1e-10)


def test_kernel_signature_matches_the_launch():
    """The emulator passes the batch descriptor by value: its layout must be the kernel's."""
    text = open(os.path.join(CSRC, "ptk_linalg.cu")).read()
    body = re.search(r"struct PotrsBatch \{(.*?)\};", text, re.S).group(1)
    assert [ln.split()[0] for ln in body.strip().splitlines()] == ["int", "int64_t", "int64_t"]
    assert "POTRS_MAX_DIMS = 8" in text
