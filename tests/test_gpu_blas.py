"""Parity of the native-precision BLAS family (K4/K6 fp32/fp64 paths) vs the C linker — alpha/beta grid and
layouts after the reference's TestGemm (tests/tensor/test_blas.py:94-191, :286-404) and BaseGemv (:1412-1620)."""

import numpy as np
import pytest

from helpers import compare_cuda_and_cvm, pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu


def test_readme_graph(gpu):
    # BASELINE.json configs[0]: a/a + (M+a).dot(v), fp64 (README.rst:38-61)
    a = pt.dscalar("a")
    v = pt.dvector("v")
    M = pt.dmatrix("M")
    d = a / a + (M + a).dot(v)
    rng = np.random.default_rng(0)
    f, _ = compare_cuda_and_cvm([a, v, M], [d], [1.5, np.ones(1024), rng.standard_normal((1024, 1024))])
    names = [type(n.op).__name__ for n in f.maker.fgraph.toposort()]
    assert "Gemv" in names


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("shapes", [((4, 5), (5, 3)), ((64, 64), (64, 64)), ((130, 70), (70, 257)), ((1, 9), (9, 1)),
                                    ((300, 1), (1, 200)), ((0, 4), (4, 5)), ((3, 0), (0, 5))])
def test_dot22(gpu, dtype, shapes):
    rng = np.random.default_rng(21)
    x = pt.tensor("x", dtype=dtype, shape=(None, None))
    y = pt.tensor("y", dtype=dtype, shape=(None, None))
    xv = rng.standard_normal(shapes[0]).astype(dtype)
    yv = rng.standard_normal(shapes[1]).astype(dtype)
    tol = dict(rtol=1e-5, atol_scale=1e-5) if dtype == "float32" else {}   # 1e-5 of the output scale (DESIGN.md §6)
    compare_cuda_and_cvm([x, y], [pt.dot(x, y), pt.dot(x, y) * 0.6], [xv, yv], **tol)


@pytest.mark.parametrize("a,b", [(1.0, 1.0), (0.6, 0.0), (-1.0, 0.6), (0.0, 1.0), (0.6, -1.0)])
def test_gemm_alpha_beta(gpu, a, b):
    rng = np.random.default_rng(22)
    z = pt.dmatrix("z")
    x = pt.dmatrix("x")
    y = pt.dmatrix("y")
    zv, xv, yv = rng.standard_normal((33, 47)), rng.standard_normal((33, 29)), rng.standard_normal((29, 47))
    f, _ = compare_cuda_and_cvm([z, x, y], [b * z + a * pt.dot(x, y)], [zv, xv, yv])


def test_gemm_transposed_operands(gpu):
    rng = np.random.default_rng(23)
    x = pt.fmatrix("x")
    y = pt.fmatrix("y")
    xv = rng.standard_normal((65, 129)).astype("float32")
    yv = rng.standard_normal((65, 77)).astype("float32")
    compare_cuda_and_cvm([x, y], [pt.dot(x.T, y), pt.dot(y.T, x), pt.dot(x.T[::2], y[:, ::3])], [xv, yv], rtol=1e-5,
                         atol_scale=1e-5)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_gemv_variants(gpu, dtype):
    rng = np.random.default_rng(24)
    A = pt.tensor("A", dtype=dtype, shape=(None, None))
    x = pt.tensor("x", dtype=dtype, shape=(None,))
    y = pt.tensor("y", dtype=dtype, shape=(None,))
    Av = rng.standard_normal((70, 1300)).astype(dtype)
    xv = rng.standard_normal(1300).astype(dtype)
    yv = rng.standard_normal(70).astype(dtype)
    tol = dict(rtol=1e-5, atol_scale=1e-5) if dtype == "float32" else {}
    compare_cuda_and_cvm([A, x, y], [pt.dot(A, x), y + 0.5 * pt.dot(A, x), pt.dot(A.T, y), pt.dot(x, A.T),
                                     pt.dot(x, x)], [Av, xv, yv], **tol)


def test_tall_skinny_gemv_transposed(gpu):
    # cfg-5 secondary shape: X (N,8)^T @ r
    rng = np.random.default_rng(25)
    X = pt.dmatrix("X")
    r = pt.dvector("r")
    Xv = rng.standard_normal((1 << 16, 8))
    rv = rng.standard_normal(1 << 16)
    compare_cuda_and_cvm([X, r], [pt.dot(X.T, r), pt.dot(X, X.T[:, 0])], [Xv, rv], rtol=1e-9)


def test_ger(gpu):
    rng = np.random.default_rng(26)
    A = pt.dmatrix("A")
    x = pt.dvector("x")
    y = pt.dvector("y")
    compare_cuda_and_cvm([A, x, y], [A + 0.3 * pt.outer(x, y)],
                         [rng.standard_normal((40, 50)), rng.standard_normal(40), rng.standard_normal(50)])


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_skinny_gemm_shapes(gpu, dtype):
    # cfg-5 regression shapes: (B x K)(K x n) with K = 8 and (B x n)(n x K) with N = 8 take the HBM-bound skinny kernels
    rng = np.random.default_rng(27)
    beta = pt.tensor("beta", dtype=dtype, shape=(None, None))
    X = pt.tensor("X", dtype=dtype, shape=(None, None))
    R = pt.tensor("R", dtype=dtype, shape=(None, None))
    bv = rng.standard_normal((1500, 8)).astype(dtype)
    Xv = rng.standard_normal((1030, 8)).astype(dtype)
    Rv = rng.standard_normal((1500, 1030)).astype(dtype)
    tol = dict(rtol=1e-5, atol_scale=1e-5) if dtype == "float32" else dict(rtol=1e-9, atol=1e-9)
    compare_cuda_and_cvm([beta, X, R], [pt.dot(beta, X.T), pt.dot(R, X), 0.5 * R + 2.0 * pt.dot(beta, X.T)], [bv, Xv, Rv], **tol)


def test_gemm_zero_sized_and_broadcast_z(gpu):
    # zero-size operands (tests/tensor/test_blas.py:185-191) and a row-broadcast Z (gemm.py:194-198)
    rng = np.random.default_rng(28)
    x, y = pt.dmatrix("x"), pt.dmatrix("y")
    zrow = pt.drow("zrow")
    compare_cuda_and_cvm([x, y], [pt.dot(x, y)], [np.zeros((0, 5)), rng.standard_normal((5, 7))])
    compare_cuda_and_cvm([x, y], [pt.dot(x, y)], [rng.standard_normal((4, 0)), np.zeros((0, 7))])
    compare_cuda_and_cvm([zrow, x, y], [zrow + 2.0 * pt.dot(x, y)],
                         [rng.standard_normal((1, 7)), rng.standard_normal((4, 5)), rng.standard_normal((5, 7))])
    # an empty contraction leaves b * z (gemm.py: z *= b; z += a * dot): inf, NaN and values whose products overflow stay
    # in their own elements, in Gemm and in Gemv
    for dtype, huge in (("float64", 1e200), ("float32", 1e20)):
        z, a, b = pt.matrix("z", dtype=dtype), pt.matrix("a", dtype=dtype), pt.matrix("b", dtype=dtype)
        yv, A, v = pt.vector("yv", dtype=dtype), pt.matrix("A", dtype=dtype), pt.vector("v", dtype=dtype)
        zv = rng.standard_normal((4, 7)).astype(dtype)
        zv[0, 0], zv[1, 2], zv[2, 3], zv[3, :], zv[:, 6] = np.inf, np.nan, -np.inf, huge, huge
        yvv = rng.standard_normal(6).astype(dtype)
        yvv[0], yvv[2], yvv[4] = np.inf, np.nan, huge
        f, _ = compare_cuda_and_cvm([z, a, b, yv, A, v], [0.5 * z + 2.0 * pt.dot(a, b), 0.5 * yv + 2.0 * pt.dot(A, v)],
                                    [zv, np.zeros((4, 0), dtype), np.zeros((0, 7), dtype), yvv, np.zeros((6, 0), dtype),
                                     np.zeros(0, dtype)])
        names = [type(n.op).__name__ for n in f.maker.fgraph.toposort()]
        assert "Gemm" in names and "Gemv" in names, names


def test_gemv_beta_zero_ignores_nan_y(gpu):
    # contract: beta == 0 => y's contents (possibly NaN from AllocEmpty) are never read (gemv.py:79-86)
    rng = np.random.default_rng(29)
    A, x = pt.dmatrix("A"), pt.dvector("x")
    Av, xv = rng.standard_normal((33, 17)), rng.standard_normal(17)
    f, got = compare_cuda_and_cvm([A, x], [pt.dot(A, x)], [Av, xv])
    assert np.all(np.isfinite(got[0]))
    for _ in range(3):  # repeated calls reuse NaN-poisoned allocator blocks; result must stay finite
        assert np.all(np.isfinite(f(Av, xv)[0]))


def _chain_graph(widths, acts, bias=True):
    x = pt.fmatrix("x")
    Ws = [pt.fmatrix(f"W{i}") for i in range(len(widths) - 1)]
    bs = [pt.fvector(f"b{i}") for i in range(len(widths) - 1)]
    h = x
    for W, b, a in zip(Ws, bs, acts):
        h = pt.dot(h, W) + b if bias else pt.dot(h, W)
        if a:
            h = pt.tanh(h)
    return x, Ws, bs, h


@pytest.mark.parametrize("M,widths,acts,bias", [
    (64, [64] * 9, [1] * 8, True),                         # the metric graph's layer shape
    (37, [20, 128, 4, 68, 128, 12], [1, 1, 1, 1, 1], True),  # ragged widths, rows not a multiple of 16
    (130, [32, 32, 32, 32, 32], [1, 1, 1, 1], False),       # tanh(A @ B) layers without bias
])
def test_small_mlp_chain_is_one_launch_and_matches_the_c_linker(gpu, M, widths, acts, bias):
    """>= 4 dense layers of at most 128 columns run as ONE kernel (MlpChainNode / ptk_mlp_chain); same 1e-5 bar as the
    layer-by-layer path."""
    pytensor.config.floatX = "float32"
    rng = np.random.default_rng(71)
    x, Ws, bs, h = _chain_graph(widths, acts, bias)
    ins = [x, *Ws, *(bs if bias else [])]
    vals = [rng.standard_normal((M, widths[0])).astype("float32")]
    vals += [(rng.standard_normal((widths[i], widths[i + 1])) / np.sqrt(widths[i])).astype("float32") for i in range(len(widths) - 1)]
    if bias:
        vals += [(rng.standard_normal(widths[i + 1]) * 0.1).astype("float32") for i in range(len(widths) - 1)]
    f, _ = compare_cuda_and_cvm(ins, [h, h.sum(axis=0)], vals, rtol=1e-5, atol=1e-5)
    chain = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "MlpChainNode"]
    assert len(chain) == 1 and chain[0].fused_calls >= 1 and chain[0].unfused_calls == 0


def test_mlp_chain_with_a_wide_layer_runs_layer_by_layer(gpu):
    pytensor.config.floatX = "float32"
    rng = np.random.default_rng(72)
    widths = [64, 300, 64, 64, 64]
    x, Ws, bs, h = _chain_graph(widths, [1, 1, 1, 1])
    vals = [rng.standard_normal((40, 64)).astype("float32")]
    vals += [(rng.standard_normal((widths[i], widths[i + 1])) / np.sqrt(widths[i])).astype("float32") for i in range(4)]
    vals += [(rng.standard_normal(widths[i + 1]) * 0.1).astype("float32") for i in range(4)]
    f, _ = compare_cuda_and_cvm([x, *Ws, *bs], [h], vals, rtol=1e-5, atol=1e-5)
    chain = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "MlpChainNode"]
    assert len(chain) == 1 and chain[0].fused_calls == 0 and chain[0].unfused_calls >= 1
