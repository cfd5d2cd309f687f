"""The native-precision BLAS family (ptk_blas.cu: the SIMT GEMM, the small-K / small-N skinny GEMMs, GEMV, GER and the
one-launch small-MLP chain) at its routing edges, against fp64 references of the same operation.

a. Integer-grid operands x = n * 2^e (small |n|, one exponent per row of A / column of B): while every partial sum,
   alpha * acc + beta * C and the bias fit in 24 (fp32) / 53 (fp64) bits of their finest unit, every summation order is
   exact, so each route must reproduce the fp64 product bit for bit.  beta == 0 runs against a NaN-poisoned output, and
   every output view sits in a sentinel-filled buffer that must not change outside [M, N].
b. Random normals, rows of A / columns of B scaled over 2^+-20: every element within (K + 8) * u * (|A| @ |B|)_ij.
c. ±inf / NaN in A, B and C, also where they meet the zero padding of a partial tile: the C linker's inf / NaN pattern.
d. The small-MLP chain: exact on integer chains up to and across the 96-layer launch split, and bit-identical to the
   layer-by-layer program on random data with tanh.
e. PTK_BLAS_V2=1 (the pipelined skinny kernels, read once per process) gives v1's bits.
f. Empty contractions (K = 0) and products taller than 65535 m-tiles of the SIMT kernel.

Which kernel runs is not observable from Python: `gemm_route` / `gemv_route` restate launch_gemm / launch_smalln /
launch_gemv, every case names the route it is meant to take, and the tables hold a shape on both sides of every
threshold, so coverage does not rest on the restatement alone.  The C-ABI tests skip in the dry run (PTK_DRY=1); the graph
tests go through compare_cuda_and_cvm, which traces them there."""

import os
import subprocess
import sys

import numpy as np
import pytest

from helpers import compare_cuda_and_cvm, pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SENTINEL = 12345.0
BITS = {"float32": 24, "float64": 53}
NP = {"float32": np.float32, "float64": np.float64}


def _abi(gpu):
    if not gpu:
        pytest.skip("calls the C ABI on the device")
    import torch

    from pytensor_b200.runtime import lib as _lib

    return _lib.lib(), torch


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cdiv(a, b):
    return -(-a // b)


# ---- the routing of launch_gemm / launch_smalln / launch_gemv, restated ---------------------------------------------------
def _sn_width(N):
    return 1 if N <= 1 else 2 if N <= 2 else 4 if N <= 4 else 8 if N <= 8 else 16


def smalln_kchunk(dtype, N, K):
    """K elements of B staged per CTA pass of the small-N kernel (launch_smalln)."""
    isz = np.dtype(dtype).itemsize
    V = 16 // isz
    unit = 32 * V * 4
    kchunk = _cdiv(K, unit) * unit
    max_elems = (96 * 1024) // (isz * _sn_width(N)) - V
    if kchunk > max_elems:
        kchunk = max(unit, max_elems // unit * unit)
    return kchunk


def gemm_route(dtype, A, B, C, sms, bias=False, act=0):
    M, K = A.shape
    N = B.shape[1]
    (sa0, sa1), (sb0, sb1), (sc0, sc1) = A.stride(), B.stride(), C.stride()
    plain = not bias and not act
    if plain and 1 <= K <= 16 and sc1 == 1 and M >= 256 and N >= 64:
        gx = _cdiv(N, 256)
        gy = min(_cdiv(M, 64), max(1, sms * 12 // gx))
        return f"smallk{4 if K <= 4 else 8 if K <= 8 else 16}" + ("/loop" if _cdiv(M, 64) > gy else "")
    if plain and N <= 16 and sa1 == 1 and M >= 256 and K >= 64:
        V = 16 // np.dtype(dtype).itemsize
        vec = sa0 % V == 0 and A.data_ptr() % 16 == 0
        return f"smalln{_sn_width(N)}/{_cdiv(K, smalln_kchunk(dtype, N, K))}ch/{'vec' if vec else 'scalar'}"
    akf, bnf = sa1 == 1 or K == 1, sb1 == 1 or N == 1
    if sa0 == 1 and sa1 != 1:
        akf = False
    if sb0 == 1 and sb1 != 1:
        bnf = False
    return f"simt{int(akf)}{int(bnf)}"


def gemv_route(A, sms):
    M, N = A.shape
    sa0, sa1 = A.stride()
    if sa0 == 1 and sa1 != 1 and N > 1:
        want = max(1, sms * 4 // _cdiv(M, 32))
        return f"gemv_col/{max(1, min(want, _cdiv(N, 64), 65535))}"
    nchunks = 1
    if M < sms * 32 and N > 4096:
        nchunks = min(_cdiv(sms * 32, M), _cdiv(N, 1024))
    return f"gemv_row/{nchunks}"


# ---- operands on the device in a given layout ------------------------------------------------------------------------------
def _strides(layout, R, C):
    """(row stride, column stride, element offset) of an R x C view in a flat buffer.  Offset 64 keeps a view 256-byte
    aligned; 'shift' moves it by one element."""
    if layout == "row":
        return C, 1, 64
    if layout == "pad":                           # row pitch a multiple of 8: the small-N kernel's vector loads
        return _cdiv(C, 8) * 8, 1, 64
    if layout == "odd":                           # odd row pitch: rows alternate between vector and scalar paths
        return C + 1 if C % 2 == 0 else C + 2, 1, 64
    if layout == "shift":
        return C, 1, 65
    if layout == "col":
        return 1, R, 64
    if layout == "every_other":                  # both strides non-unit
        return 2 * C, 2, 64
    raise ValueError(layout)


def _place(torch, x, layout, fill=SENTINEL):
    """(view holding x in `layout`, the flat sentinel-filled buffer behind it)."""
    R, C = x.shape
    s0, s1, off = _strides(layout, R, C)
    size = off + (R - 1) * s0 + (C - 1) * s1 + 1 + 64 if R and C else off + 64
    big = torch.full((size,), fill, dtype=getattr(torch, str(x.dtype)), device="cuda")
    v = torch.as_strided(big, (R, C), (s0, s1), off)
    v.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    return v, big


def _untouched(view, big):
    view.fill_(SENTINEL)   # what is left is what the kernel wrote outside its view
    assert bool((big == SENTINEL).all()), "written outside the [M, N] view"


def _gemm(L, torch, dtype, A, B, C, alpha, beta, bias=None, act=0):
    from pytensor_b200.runtime import device as dev
    from pytensor_b200.runtime import lib as _lib

    M, K = A.shape
    N = B.shape[1]
    code = _lib.DTYPE_CODE[dtype]
    if bias is not None or act:
        _lib.check(L.ptk_gemm_bias_act(code, M, N, K, A.data_ptr(), A.stride(0), A.stride(1), B.data_ptr(), B.stride(0),
                                       B.stride(1), bias.data_ptr() if bias is not None else None, act, C.data_ptr(),
                                       C.stride(0), C.stride(1), 0, None, 0, dev.stream_ptr()), "ptk_gemm_bias_act")
    else:
        _lib.check(L.ptk_gemm(code, M, N, K, alpha, A.data_ptr(), A.stride(0), A.stride(1), B.data_ptr(), B.stride(0),
                              B.stride(1), beta, C.data_ptr(), C.stride(0), C.stride(1), 0, None, 0, dev.stream_ptr()),
                   "ptk_gemm")
    torch.cuda.synchronize()


def _gemv(L, torch, dtype, A, x, y, alpha, beta):
    from pytensor_b200.runtime import device as dev
    from pytensor_b200.runtime import lib as _lib

    M, N = A.shape
    _lib.check(L.ptk_gemv(_lib.DTYPE_CODE[dtype], M, N, alpha, A.data_ptr(), A.stride(0), A.stride(1), x.data_ptr(),
                          x.stride(0), beta, y.data_ptr(), y.stride(0), dev.stream_ptr()), "ptk_gemv")
    torch.cuda.synchronize()


# ---- a. integer grid, exact --------------------------------------------------------------------------------------------
def _grid(rng, rows, cols, nmax, emin, emax, axis):
    """n * 2^e, |n| <= nmax, one exponent per row (axis 0) or per column (axis 1); returns (values, exponents)."""
    n = rng.integers(-nmax, nmax + 1, size=(rows, cols)).astype(np.float64)
    e = rng.integers(emin, emax + 1, size=rows if axis == 0 else cols)
    x = n * np.exp2(e)[:, None] if axis == 0 else n * np.exp2(e)[None, :]
    return x, e


# (alpha, beta): beta == 0 runs against a NaN-poisoned C, alpha == 0 leaves beta * C
EPILOGUES = [(1.0, 0.0), (-2.0, 1.0), (0.5, -0.5), (0.0, 0.75)]


def _grid_case(rng, M, N, K, alpha, beta, with_bias, dtype):
    """A [M, K], B [K, N], C0 [M, N], bias [N] on the integer grid and the exact fp64 result; asserts the exactness
    precondition: every partial sum and epilogue term fits in BITS[dtype] bits of its finest unit."""
    bits = BITS[dtype]
    plain = beta == 0.0 and not with_bias
    if plain:
        nmax, (emin, emax) = max(1, min(127, int(np.sqrt(2.0 ** (bits - 1) / max(K, 1))))), (-10, 10)
    else:
        nmax, (emin, emax) = max(1, min(7, int(np.sqrt(2.0 ** (bits - 9) / max(K, 1))))), (-1, 1)
    A, ea = _grid(rng, M, K, nmax, emin, emax, 0)
    B, eb = _grid(rng, K, N, nmax, emin, emax, 1)
    C0, ec = _grid(rng, M, N, 1023, -2, -2, 0)
    bias = rng.integers(-255, 256, N) * 2.0 ** -2 if with_bias else None
    ref = alpha * (A @ B) + (beta * C0 if beta else 0.0) + (bias if with_bias else 0.0)
    unit = np.full((M, N), np.inf)
    bound = np.zeros((M, N))
    if alpha:
        unit = abs(alpha) * np.exp2(ea[:, None] + eb[None, :]) * np.ones((M, N))
        bound = abs(alpha) * (np.abs(A) @ np.abs(B))
    if beta:
        unit = np.minimum(unit, abs(beta) * np.exp2(ec)[:, None])
        bound = bound + np.abs(beta * C0)
    if with_bias:
        unit = np.minimum(unit, 2.0 ** -2)
        bound = bound + np.abs(bias)[None, :]
    assert np.all(bound < 2.0 ** bits * unit), "test operands break the exactness precondition"
    t = NP[dtype]
    assert np.array_equal(ref.astype(t).astype(np.float64), ref)
    return A.astype(t), B.astype(t), C0.astype(t), None if bias is None else bias.astype(t), ref


def _grid_gemm(gpu, dtype, M, N, K, alay, blay, clay, route, seed, epilogues=EPILOGUES):
    L, torch = _abi(gpu)
    if callable(M):
        M = M(_sms(torch))
    rng = np.random.default_rng(seed)
    for alpha, beta in epilogues:
        A, B, C0, _, ref = _grid_case(rng, M, N, K, alpha, beta, False, dtype)
        Ad, _ = _place(torch, A, alay)
        Bd, _ = _place(torch, B, blay)
        Cd, big = _place(torch, C0 if beta else np.full((M, N), np.nan, NP[dtype]), clay)
        assert gemm_route(dtype, Ad, Bd, Cd, _sms(torch)) == route
        _gemm(L, torch, dtype, Ad, Bd, Cd, alpha, beta)
        got = Cd.cpu().numpy().astype(np.float64)
        np.testing.assert_array_equal(got, ref, err_msg=f"{route} alpha={alpha} beta={beta}")
        _untouched(Cd, big)
    return Ad, Bd


f32, f64 = "float32", "float64"
# (id, dtype, M, N, K, A layout, B layout, C layout, intended route); M may depend on the SM count
SMALLK = [
    ("k1", f32, 256, 64, 1, "row", "row", "row", "smallk4"),
    ("k4", f64, 257, 65, 4, "row", "row", "row", "smallk4"),
    ("k5_n66", f32, 300, 66, 5, "row", "row", "row", "smallk8"),            # N not a multiple of 4
    ("k8_n255", f64, 256, 255, 8, "row", "row", "row", "smallk8"),
    ("k9_n257", f32, 257, 257, 9, "row", "row", "row", "smallk16"),
    ("k16_n513", f64, 300, 513, 16, "row", "row", "row", "smallk16"),
    ("k16_n511_transposed", f32, 300, 511, 16, "col", "col", "row", "smallk16"),
    ("k17", f32, 300, 100, 17, "row", "row", "row", "simt11"),
    ("m255", f32, 255, 64, 8, "row", "row", "row", "simt11"),
    ("n63", f64, 256, 63, 8, "row", "row", "row", "simt11"),
    ("odd_pitch_c_f32", f32, 301, 130, 7, "row", "row", "odd", "smallk8"),
    ("odd_pitch_c_f64", f64, 301, 130, 7, "row", "row", "odd", "smallk8"),   # the 32-byte vector store on every 4th row
    ("shifted_c", f32, 260, 67, 3, "row", "row", "shift", "smallk4"),
    ("c_colmajor", f32, 300, 70, 8, "row", "row", "col", "simt11"),
    ("row_loop_f32", f32, lambda s: s * 12 * 64 + 77, 64, 3, "row", "row", "row", "smallk4/loop"),
    ("row_loop_f64", f64, lambda s: s * 12 * 64 + 77, 200, 12, "every_other", "row", "row", "smallk16/loop"),
]
SMALLN = [
    ("n1", f32, 256, 1, 64, "pad", "row", "row", "smalln1/1ch/vec"),
    ("n2", f64, 257, 2, 64, "pad", "row", "row", "smalln2/1ch/vec"),
    ("n3", f32, 300, 3, 100, "row", "row", "row", "smalln4/1ch/vec"),
    ("n4_odd_k", f64, 300, 4, 65, "row", "row", "row", "smalln4/1ch/scalar"),
    ("n5_many_rows", f32, 5000, 5, 200, "row", "row", "row", "smalln8/1ch/vec"),
    ("n8_f32_2ch", f32, 300, 8, 2561, "pad", "row", "row", "smalln8/2ch/vec"),
    ("n8_f64_1ch", f64, 300, 8, 1280, "pad", "row", "row", "smalln8/1ch/vec"),
    ("n8_f64_2ch", f64, 300, 8, 1281, "pad", "row", "row", "smalln8/2ch/vec"),
    ("n7_f64_3ch", f64, 260, 7, 2600, "pad", "row", "row", "smalln8/3ch/vec"),
    ("n9_1ch", f32, 300, 9, 1024, "pad", "row", "row", "smalln16/1ch/vec"),
    ("n16_2ch", f32, 300, 16, 1025, "pad", "row", "row", "smalln16/2ch/vec"),
    ("n12_3ch_shifted", f32, 300, 12, 2100, "shift", "row", "row", "smalln16/3ch/scalar"),
    ("n16_f64_1ch", f64, 300, 16, 512, "pad", "row", "row", "smalln16/1ch/vec"),
    ("n16_f64_2ch_odd", f64, 300, 16, 513, "odd", "row", "row", "smalln16/2ch/scalar"),
    ("n10_f64_4ch", f64, 300, 10, 1600, "pad", "row", "every_other", "smalln16/4ch/vec"),
    ("n5_c_colmajor", f64, 300, 5, 100, "pad", "row", "col", "smalln8/1ch/vec"),
    ("n3_b_colmajor", f32, 300, 3, 300, "row", "col", "odd", "smalln4/1ch/vec"),
    ("n17", f32, 300, 17, 100, "row", "row", "row", "simt11"),
    ("k63", f64, 300, 8, 63, "row", "row", "row", "simt11"),
    ("m255", f32, 255, 8, 100, "row", "row", "row", "simt11"),
    ("a_colmajor", f32, 300, 8, 100, "col", "row", "row", "simt01"),         # sa1 != 1
]
SIMT = [
    ("kfast_nfast", f32, 65, 130, 33, "row", "row", "row", "simt11"),
    ("mfast_nfast", f64, 64, 64, 16, "col", "row", "row", "simt01"),
    ("kfast_kfast", f32, 70, 47, 29, "row", "col", "col", "simt10"),
    ("mfast_kfast", f64, 5, 200, 3, "col", "col", "every_other", "simt00"),
    ("k1_strided_a", f32, 70, 50, 1, "every_other", "row", "row", "simt11"),  # K == 1 makes A k-fast
    ("k2_strided_a", f32, 70, 50, 2, "every_other", "row", "row", "simt01"),
    ("n1_strided_b", f64, 70, 1, 40, "row", "every_other", "row", "simt11"),  # N == 1 makes B n-fast
    ("k1_colmajor_a", f32, 65, 70, 1, "col", "row", "row", "simt01"),       # sa0 == 1 overrides K == 1
    ("ragged_odd_c", f64, 129, 65, 47, "row", "row", "odd", "simt11"),
]


@pytest.mark.parametrize("case", SMALLK, ids=[c[0] for c in SMALLK])
def test_small_k_integer_grid_is_exact(gpu, case):
    _grid_gemm(gpu, *case[1:], seed=SMALLK.index(case))


@pytest.mark.parametrize("case", SMALLN, ids=[c[0] for c in SMALLN])
def test_small_n_integer_grid_is_exact(gpu, case):
    _grid_gemm(gpu, *case[1:], seed=100 + SMALLN.index(case))


@pytest.mark.parametrize("case", SIMT, ids=[c[0] for c in SIMT])
def test_simt_integer_grid_is_exact(gpu, case):
    _grid_gemm(gpu, *case[1:], seed=200 + SIMT.index(case))


def _tanh_ulps(dtype):
    """CUDA's documented bounds: tanhf within 2 ulp, tanh within 1 ulp; +0.5 ulp for rounding the exact tanh."""
    return 2.5 if dtype == "float32" else 1.5


@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("case", SIMT, ids=[c[0] for c in SIMT])
def test_simt_bias_epilogue(gpu, case, act):
    """act(A @ B + bias) through ptk_gemm_bias_act: exact without tanh; tanh within its ulp bound of the exact input."""
    L, torch = _abi(gpu)
    _, dtype, M, N, K, alay, blay, clay, route = case
    rng = np.random.default_rng(300 + SIMT.index(case))
    A, B, _, bias, pre = _grid_case(rng, M, N, K, 1.0, 0.0, True, dtype)
    Ad, _ = _place(torch, A, alay)
    Bd, _ = _place(torch, B, blay)
    Cd, big = _place(torch, np.full((M, N), np.nan, NP[dtype]), clay)
    assert gemm_route(dtype, Ad, Bd, Cd, _sms(torch), bias=True, act=act) == route
    _gemm(L, torch, dtype, Ad, Bd, Cd, 1.0, 0.0, bias=torch.from_numpy(bias).cuda(), act=act)
    got = Cd.cpu().numpy().astype(np.float64)
    if act:
        exp = np.tanh(pre)
        tol = _tanh_ulps(dtype) * np.spacing(np.abs(exp).astype(NP[dtype])).astype(np.float64)
        assert np.all(np.abs(got - exp) <= tol), f"worst {np.max(np.abs(got - exp) / tol):.2f} x the ulp bound"
    else:
        np.testing.assert_array_equal(got, pre)
    _untouched(Cd, big)


@pytest.mark.parametrize("dtype", [f32, f64])
def test_simt_empty_contraction_through_the_abi(gpu, dtype):
    """K = 0: alpha * 0 + beta * C, with C's inf / NaN / largest finite values scaled alone; bias + tanh gives tanh(bias)."""
    L, torch = _abi(gpu)
    M, N = 300, 70   # (skinny-sized: K = 0 is below every skinny kernel's K range)
    t = NP[dtype]
    big_v = np.finfo(t).max / 2
    C0 = np.random.default_rng(1).integers(-50, 50, (M, N)).astype(t)
    C0[3, 4], C0[5, 6], C0[M - 1, N - 1], C0[0, :] = np.inf, -np.inf, np.nan, big_v
    A = torch.empty((M, 0), dtype=getattr(torch, dtype), device="cuda")
    B = torch.empty((0, N), dtype=getattr(torch, dtype), device="cuda")
    for alpha, beta in [(1.0, 0.0), (-2.0, 1.0), (0.5, -0.5)]:
        Cd, big = _place(torch, C0 if beta else np.full((M, N), np.nan, t), "odd")
        assert gemm_route(dtype, A, B, Cd, _sms(torch)) == "simt11"
        _gemm(L, torch, dtype, A, B, Cd, alpha, beta)
        exp = (beta * C0.astype(np.float64)).astype(t) if beta else np.zeros((M, N), t)
        np.testing.assert_array_equal(Cd.cpu().numpy(), exp)
        _untouched(Cd, big)
    bias = np.linspace(-3, 3, N).astype(t)
    Cd, big = _place(torch, np.full((M, N), np.nan, t), "row")
    _gemm(L, torch, dtype, A, B, Cd, 1.0, 0.0, bias=torch.from_numpy(bias).cuda(), act=1)
    got = Cd.cpu().numpy().astype(np.float64)
    exp = np.broadcast_to(np.tanh(bias.astype(np.float64)), (M, N))
    assert np.all(np.abs(got - exp) <= _tanh_ulps(dtype) * np.spacing(np.abs(exp).astype(t)))
    _untouched(Cd, big)


# GEMV: (id, dtype, M, N, A layout, x stride, y stride, intended route); "col" = an A.T view (sa0 == 1)
GEMV = [
    ("row", f32, 70, 1300, "row", 1, 1, "gemv_row/1"),
    ("row_n4096", f64, 100, 4096, "row", 3, 2, "gemv_row/1"),
    ("row_split_n4097", f64, 100, 4097, "row", 1, 1, "gemv_row/5"),
    ("row_split_m1", f32, 1, 5000, "odd", 2, 1, "gemv_row/5"),
    ("row_m_below_target", f32, lambda s: s * 32 - 1, 4097, "row", 1, 3, "gemv_row/2"),
    ("row_m_at_target", f32, lambda s: s * 32, 4097, "row", 1, 1, "gemv_row/1"),
    ("col_one_chunk", f32, 600, 64, "col", 1, 1, "gemv_col/1"),
    ("col_chunks", f64, 600, 1000, "col", 3, 2, lambda s: f"gemv_col/{min(s * 4 // 19, 16)}"),
    ("col_tall", f32, 20000, 300, "col", 1, 1, "gemv_col/1"),
    ("n1_colmajor", f64, 500, 1, "col", 1, 1, "gemv_row/1"),
    ("strided_a", f64, 97, 333, "every_other", 2, 3, "gemv_row/1"),
]


def _gemv_case(gpu, case, alpha, beta, seed, y_nan=True):
    L, torch = _abi(gpu)
    sms = _sms(torch)
    _, dtype, M, N, alay, sx, sy, route = case
    M = M(sms) if callable(M) else M
    route = route(sms) if callable(route) else route
    rng = np.random.default_rng(seed)
    A, x, y0, _, ref = _grid_case(rng, M, 1, N, alpha, beta, False, dtype)
    Ad, _ = _place(torch, A, alay)
    xd, _ = _place(torch, x.reshape(1, N).repeat(sx, 0).T.copy(), "row")   # x in column 0 of an [N, sx] matrix
    xd = xd[:, 0]
    yv, ybig = _place(torch, (y0 if beta else np.full((M, 1), np.nan, NP[dtype])).repeat(sy, 1), "row")
    yv[:, 1:] = SENTINEL   # (y is column 0: the elements between y's are sentinels too)
    yd = yv[:, 0]
    assert gemv_route(Ad, sms) == route
    _gemv(L, torch, dtype, Ad, xd, yd, alpha, beta)
    np.testing.assert_array_equal(yd.cpu().numpy().astype(np.float64), ref[:, 0], err_msg=f"{route} {alpha} {beta}")
    yd.fill_(SENTINEL)
    assert bool((ybig == SENTINEL).all()), "gemv wrote outside y"


@pytest.mark.parametrize("case", GEMV, ids=[c[0] for c in GEMV])
def test_gemv_integer_grid_is_exact(gpu, case):
    for i, (alpha, beta) in enumerate(EPILOGUES):
        _gemv_case(gpu, case, alpha, beta, seed=400 + 10 * GEMV.index(case) + i)


@pytest.mark.parametrize("dtype", [f32, f64])
@pytest.mark.parametrize("alay", ["row", "every_other", "col"])
def test_ger_integer_grid_is_exact(gpu, dtype, alay):
    """A += alpha * x y^T on a strided A with strided x and y; nothing between A's elements changes."""
    L, torch = _abi(gpu)
    from pytensor_b200.runtime import device as dev
    from pytensor_b200.runtime import lib as _lib

    M, N = 130, 77
    rng = np.random.default_rng(500)
    A0 = _grid(rng, M, N, 1023, -3, -3, 0)[0].astype(NP[dtype])
    x = _grid(rng, M, 1, 31, 0, 4, 0)[0][:, 0]
    y = _grid(rng, 1, N, 31, -4, 0, 1)[0][0]
    for alpha in (1.0, -0.5, 0.0):
        Ad, big = _place(torch, A0, alay)
        xd = _place(torch, x.astype(NP[dtype]).reshape(1, M), "every_other")[0][0]
        yd = _place(torch, y.astype(NP[dtype]).reshape(N, 1), "odd")[0][:, 0]
        _lib.check(L.ptk_ger(_lib.DTYPE_CODE[dtype], M, N, alpha, xd.data_ptr(), xd.stride(0), yd.data_ptr(), yd.stride(0),
                             Ad.data_ptr(), Ad.stride(0), Ad.stride(1), dev.stream_ptr()), "ptk_ger")
        torch.cuda.synchronize()
        ref = A0.astype(np.float64) + alpha * np.outer(x, y)
        np.testing.assert_array_equal(Ad.cpu().numpy().astype(np.float64), ref)
        _untouched(Ad, big)


@pytest.mark.parametrize("dtype", [f32, f64])
def test_ger_graph_in_place_and_cloned(gpu, dtype):
    rng = np.random.default_rng(501)
    A, x, y = pt.matrix("A", dtype=dtype), pt.vector("x", dtype=dtype), pt.vector("y", dtype=dtype)
    Av = rng.integers(-9, 10, (40, 50)).astype(dtype)
    xv, yv = rng.integers(-9, 10, 40).astype(dtype), rng.integers(-9, 10, 50).astype(dtype)
    # the first output keeps A alive, so the second Ger works on a copy; the third may update its own temporary in place
    compare_cuda_and_cvm([A, x, y], [A + 0.5 * pt.outer(x, y), A - 2.0 * pt.outer(x[::-1], y),
                                     (A * 2.0) + pt.outer(x, y[::-1])], [Av, xv, yv], exact=True)


@pytest.mark.parametrize("dtype", [f32, f64])
def test_dot_node_vector_forms_are_exact(gpu, dtype):
    """Dot's 1-d . 1-d and 1-d . 2-d forms (gemv over a one-row view, gemv over B.T), with strided vectors."""
    rng = np.random.default_rng(502)
    v, w, B = pt.vector("v", dtype=dtype), pt.vector("w", dtype=dtype), pt.matrix("B", dtype=dtype)
    vv, wv = rng.integers(-9, 10, 6001).astype(dtype), rng.integers(-9, 10, 6001).astype(dtype)
    Bv = rng.integers(-9, 10, (3000, 70)).astype(dtype)
    compare_cuda_and_cvm([v, w, B], [pt.dot(v, w), pt.dot(v[:6000:2], w[1::2]), pt.dot(v[:3000], B), pt.dot(w[:6000:2], B[::-1])],
                         [vv, wv, Bv], exact=True)


# ---- b. random data within a bound -------------------------------------------------------------------------------------
def _scaled_normal(rng, M, N, K, dtype):
    A = rng.standard_normal((M, K)) * np.exp2(rng.uniform(-20, 20, (M, 1)))
    B = rng.standard_normal((K, N)) * np.exp2(rng.uniform(-20, 20, (1, N)))
    return A.astype(dtype), B.astype(dtype)


def _random_bound(dtype, K):
    """Every route sums each output as a tree of fused multiply-adds and adds no deeper than K + 8 (a lane's serial
    k-loop, at most five shuffle levels, the per-chunk and per-group adds, one epilogue add), so with u the unit roundoff
    the classic bound gamma_(K+8) (|A| @ |B|) holds; gamma_n = n u / (1 - n u) <= 1.01 n u here."""
    u = 2.0 ** -24 if dtype == "float32" else 2.0 ** -53
    return 1.01 * (K + 8) * u


RANDOM = [   # (id, dtype, M, N, K, A layout, intended route)
    ("smallk", f32, 1000, 300, 12, "row", "smallk16"),
    ("smalln_vec_3ch", f32, 2000, 12, 3000, "pad", "smalln16/3ch/vec"),
    ("smalln_scalar_2ch", f64, 600, 8, 1500, "odd", "smalln8/2ch/scalar"),
    ("simt", f32, 300, 200, 100, "col", "simt01"),
    ("simt_f64", f64, 257, 130, 1000, "row", "simt11"),
]


@pytest.mark.parametrize("case", RANDOM, ids=[c[0] for c in RANDOM])
def test_random_gemm_meets_the_elementwise_bound(gpu, case):
    L, torch = _abi(gpu)
    _, dtype, M, N, K, alay, route = case
    A, B = _scaled_normal(np.random.default_rng(600 + RANDOM.index(case)), M, N, K, dtype)
    Ad, _ = _place(torch, A, alay)
    Bd, _ = _place(torch, B, "row")
    Cd, _ = _place(torch, np.full((M, N), np.nan, dtype), "row")
    assert gemm_route(dtype, Ad, Bd, Cd, _sms(torch)) == route
    _gemm(L, torch, dtype, Ad, Bd, Cd, 1.0, 0.0)
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    err = np.abs(Cd.cpu().numpy() - A64 @ B64) / (np.abs(A64) @ np.abs(B64))
    assert err.max() <= _random_bound(dtype, K), f"{err.max():.2e} of (|A| @ |B|)_ij"


RANDOM_GEMV = [   # (id, dtype, M, N, A layout, intended route); the first is the README graph's 1024^2 fp64 Gemv
    ("readme_1024", f64, 1024, 1024, "row", "gemv_row/1"),
    ("row_split", f32, 64, 20000, "row", lambda s: f"gemv_row/{min(_cdiv(s * 32, 64), 20)}"),
    ("col_chunks", f32, 300, 3000, "col", lambda s: f"gemv_col/{min(s * 4 // 10, 47)}"),
]


@pytest.mark.parametrize("case", RANDOM_GEMV, ids=[c[0] for c in RANDOM_GEMV])
def test_random_gemv_meets_the_elementwise_bound(gpu, case):
    L, torch = _abi(gpu)
    _, dtype, M, N, alay, route = case
    route = route(_sms(torch)) if callable(route) else route
    A, x = _scaled_normal(np.random.default_rng(700 + RANDOM_GEMV.index(case)), M, 1, N, dtype)
    Ad, _ = _place(torch, A, alay)
    xd = torch.from_numpy(x[:, 0].copy()).cuda()
    yd = torch.full((M,), float("nan"), dtype=getattr(torch, dtype), device="cuda")
    assert gemv_route(Ad, _sms(torch)) == route
    _gemv(L, torch, dtype, Ad, xd, yd, 1.0, 0.0)
    A64, x64 = A.astype(np.float64), x[:, 0].astype(np.float64)
    err = np.abs(yd.cpu().numpy() - A64 @ x64) / (np.abs(A64) @ np.abs(x64))
    assert err.max() <= _random_bound(dtype, N), f"{err.max():.2e} of (|A| @ |x|)_i"


# ---- c. special values against the C linker ----------------------------------------------------------------------------
def _plant(rng, M, N, K, dtype):
    """Normal operands with ±inf / NaN: in row 2 of A (meeting an exact zero of B: NaN), in A's last row and last column
    (the partial tiles, where the padding zeros sit), in B's last column and in C."""
    A = rng.standard_normal((M, K)).astype(dtype)
    B = rng.standard_normal((K, N)).astype(dtype)
    C = rng.standard_normal((M, N)).astype(dtype)
    A[2, min(3, K - 1)] = np.inf
    B[min(3, K - 1), min(5, N - 1)] = 0.0
    A[M - 1, K - 1] = -np.inf
    B[0, N - 1] = np.nan
    C[min(4, M - 1), 0], C[M - 1, N - 1], C[0, N // 2] = np.inf, np.nan, -np.inf
    return A, B, C


SPECIAL_GEMM = [   # (dtype, M, N, K): the route follows from the shape of a row-major Gemm
    (f32, 300, 70, 8),      # small K
    (f64, 300, 5, 100),     # small N
    (f32, 70, 65, 33),      # SIMT
]


@pytest.mark.parametrize("dtype,M,N,K", SPECIAL_GEMM)
def test_special_values_gemm_graph(gpu, dtype, M, N, K):
    A, B, C = _plant(np.random.default_rng(800 + M + N + K), M, N, K, dtype)
    z, x, y = (pt.matrix(n, dtype=dtype) for n in "zxy")
    compare_cuda_and_cvm([z, x, y], [0.5 * z + 2.0 * pt.dot(x, y), pt.dot(x, y)], [C, A, B], rtol=1e-5,
                         atol_scale=1e-5)


@pytest.mark.parametrize("dtype,M,N,transposed", [(f64, 70, 130, False), (f32, 50, 5000, False), (f64, 600, 1000, True)])
def test_special_values_gemv_graph(gpu, dtype, M, N, transposed):
    """The row kernel, the split row kernel (pre-scaled y, atomic chunks) and the column kernel."""
    A, x, y = _plant(np.random.default_rng(900 + M), M, 1, N, dtype)
    x, y = x[:, 0], y[:, 0]
    x[0], A[7, 10] = 1.0, np.nan   # (a NaN in x would make every output NaN)
    Am, xv, yv = pt.matrix("A", dtype=dtype), pt.vector("x", dtype=dtype), pt.vector("y", dtype=dtype)
    Aop = Am.T if transposed else Am
    compare_cuda_and_cvm([Am, xv, yv], [0.5 * yv + 2.0 * pt.dot(Aop, xv)], [A.T.copy() if transposed else A, x, y],
                         rtol=1e-5, atol_scale=1e-5)


def test_special_values_ger_graph(gpu):
    rng = np.random.default_rng(950)
    A, x, y = rng.standard_normal((40, 50)), rng.standard_normal(40), rng.standard_normal(50)
    x[3], y[7], y[8], A[5, 5], A[0, 9] = np.inf, 0.0, np.nan, -np.inf, np.inf
    Am, xv, yv = pt.dmatrix("A"), pt.dvector("x"), pt.dvector("y")
    compare_cuda_and_cvm([Am, xv, yv], [Am + 0.3 * pt.outer(xv, yv)], [A, x, y])


# ---- d. the small-MLP chain --------------------------------------------------------------------------------------------
def _chain_graph(widths, acts, with_bias):
    pytensor.config.floatX = "float32"
    x = pt.fmatrix("x")
    Ws = [pt.fmatrix(f"W{i}") for i in range(len(widths) - 1)]
    bs = [pt.fvector(f"b{i}") if with_bias[i] else None for i in range(len(widths) - 1)]
    h = x
    for W, b, a in zip(Ws, bs, acts):
        h = pt.dot(h, W) if b is None else pt.dot(h, W) + b
        if a:
            h = pt.tanh(h)
    return [x, *Ws, *[b for b in bs if b is not None]], h


def _chain_node(f):
    chain = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "MlpChainNode"]
    assert len(chain) == 1
    return chain[0]


def _signed_selection(rng, K, N):
    """K x N in {-1, 0, 1} with one ±1 per column: every output is ±(one input) — integer chains stay bounded."""
    W = np.zeros((K, N), np.float32)
    W[rng.integers(0, K, N), np.arange(N)] = rng.choice([-1.0, 1.0], N)
    return W


CHAINS = [   # (M, widths of the activations, layers with a bias: every "all" / alternate "alt" / "none")
    (1, [1, 64, 64, 64, 64], "all"),
    (15, [3, 68, 4, 128, 64], "alt"),
    (16, [128, 128, 128, 68, 4], "all"),
    (17, [64, 4, 64, 128, 128, 68], "none"),
    (1000, [3] + [64] * 96, "alt"),          # 96 layers: one launch, 63 CTAs
    (37, [64] * 98, "all"),                   # 97 layers: 96 + 1
    (300, [128] + [68] * 100, "alt"),         # 100 layers: 96 + 4
]


@pytest.mark.parametrize("M,widths,bias", CHAINS, ids=[f"M{c[0]}_L{len(c[1]) - 1}" for c in CHAINS])
def test_integer_chain_is_exact(gpu, M, widths, bias):
    L = len(widths) - 1
    with_bias = [bias == "all" or (bias == "alt" and i % 2 == 0) for i in range(L)]
    ins, h = _chain_graph(widths, [0] * L, with_bias)
    rng = np.random.default_rng(1000 + M + L)
    vals = [rng.integers(-20, 21, (M, widths[0])).astype(np.float32)]
    vals += [_signed_selection(rng, widths[i], widths[i + 1]) for i in range(L)]
    vals += [rng.integers(-3, 4, widths[i + 1]).astype(np.float32) for i in range(L) if with_bias[i]]
    f, got = compare_cuda_and_cvm(ins, [h], vals, exact=True)
    node = _chain_node(f)
    if gpu:
        assert node.fused_calls == 1 and node.unfused_calls == 0
        ref = vals[0].astype(np.float64)
        wi, bi = 1, 1 + L
        for i in range(L):
            ref = ref @ vals[wi].astype(np.float64)
            wi += 1
            if with_bias[i]:
                ref = ref + vals[bi]
                bi += 1
        np.testing.assert_array_equal(got[0], ref)


@pytest.mark.parametrize("M,widths,bias", [(300, [128] + [68] * 100, "alt"), (33, [20, 128, 4, 68, 128, 12], "all"),
                                           (17, [64] * 9, "all")], ids=["L100", "ragged", "metric_layer"])
def test_fused_chain_equals_the_layer_by_layer_program(gpu, monkeypatch, M, widths, bias):
    """Every layer has a bias or tanh, so unfused each takes the SIMT kernel, whose arithmetic the chain kernel copies
    (fp32 FMA, k ascending, then + bias, then tanhf): the two must agree bit for bit."""
    if not gpu:
        pytest.skip("runs the chain on the device")
    L = len(widths) - 1
    with_bias = [bias == "all" or i % 2 == 0 for i in range(L)]
    acts = [1 if (not with_bias[i] or i % 3 == 0) else 0 for i in range(L)]
    ins, h = _chain_graph(widths, acts, with_bias)
    rng = np.random.default_rng(1100 + M)
    vals = [rng.standard_normal((M, widths[0])).astype(np.float32)]
    vals += [(rng.standard_normal((widths[i], widths[i + 1])) / np.sqrt(widths[i])).astype(np.float32) for i in range(L)]
    vals += [(rng.standard_normal(widths[i + 1]) * 0.1).astype(np.float32) for i in range(L) if with_bias[i]]
    f, fused = compare_cuda_and_cvm(ins, [h], vals, rtol=1e-5, atol=1e-5)
    node = _chain_node(f)
    assert node.fused_calls == 1 and node.unfused_calls == 0
    monkeypatch.setenv("PTK_MLP_CHAIN", "0")
    unfused = f(*vals)
    assert node.fused_calls == 1 and node.unfused_calls >= 1
    np.testing.assert_array_equal(unfused[0].view(np.uint32), fused[0].view(np.uint32))


# ---- e. PTK_BLAS_V2 gives v1's bits --------------------------------------------------------------------------------------
V2_GRID = [c for c in SMALLK + SMALLN if c[-1].startswith(("smallk", "smalln"))]
V2_RANDOM = [c for c in RANDOM if c[-1].startswith(("smallk", "smalln"))]


def skinny_outputs(gpu):
    """Every skinny integer-grid case of (a) under every epilogue and the skinny random cases of (b): name -> output."""
    L, torch = _abi(gpu)
    out = {}
    for case in V2_GRID:
        _, dtype, M, N, K, alay, blay, clay, route = case
        M = M(_sms(torch)) if callable(M) else M
        rng = np.random.default_rng(SMALLK.index(case) if case in SMALLK else 100 + SMALLN.index(case))
        for i, (alpha, beta) in enumerate(EPILOGUES):
            A, B, C0, _, _ = _grid_case(rng, M, N, K, alpha, beta, False, dtype)
            Cd = _place(torch, C0 if beta else np.full((M, N), np.nan, NP[dtype]), clay)[0]
            _gemm(L, torch, dtype, _place(torch, A, alay)[0], _place(torch, B, blay)[0], Cd, alpha, beta)
            out[f"{case[0]}/{i}"] = np.ascontiguousarray(Cd.cpu().numpy())
    for case in V2_RANDOM:
        _, dtype, M, N, K, alay, route = case
        A, B = _scaled_normal(np.random.default_rng(600 + RANDOM.index(case)), M, N, K, dtype)
        Cd = _place(torch, np.full((M, N), np.nan, dtype), "row")[0]
        _gemm(L, torch, dtype, _place(torch, A, alay)[0], _place(torch, B, "row")[0], Cd, 1.0, 0.0)
        out[case[0]] = np.ascontiguousarray(Cd.cpu().numpy())
    return out


V2_CHILD = r"""
import sys
import numpy as np
sys.path[:0] = [{repo!r}, {tests!r}]
from oracle import cvm
cvm.configure()
import pytensor_b200
from pytensor_b200.runtime import device
device.device()
import test_gpu_blas_edges as t
np.savez({out!r}, **t.skinny_outputs(True))
"""


def test_blas_v2_skinny_kernels_give_v1_bits(gpu, tmp_path):
    if not gpu:
        pytest.skip("runs the skinny kernels on the device")
    out = tmp_path / "v2.npz"
    script = tmp_path / "child.py"
    script.write_text(V2_CHILD.format(repo=os.path.dirname(HERE), tests=HERE, out=str(out)))
    p = subprocess.run([sys.executable, str(script)], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, PTK_BLAS_V2="1"))
    assert p.returncode == 0, (p.stdout[-3000:], p.stderr[-3000:])
    v1 = skinny_outputs(gpu)
    v2 = np.load(out)
    assert sorted(v2.files) == sorted(v1)
    for k, a in v1.items():
        np.testing.assert_array_equal(v2[k].view(np.uint8), a.view(np.uint8), err_msg=k)


# ---- f. empty contractions and products taller than 65535 m-tiles ------------------------------------------------------
TALL_M = 65535 * 64 + 1


@pytest.mark.parametrize("dtype", [f32, f64])
def test_simt_taller_than_the_y_grid_abi(gpu, dtype):
    """M = 65535 * 64 + 1 and a few rows more, K = N = 17 (no skinny kernel): the m-tiles past grid.y's limit come from
    the grid-stride loop.  Integer operands: every output is exact, checked against an fp64 product on the device."""
    L, torch = _abi(gpu)
    tdt = getattr(torch, dtype)
    g = torch.Generator(device="cuda").manual_seed(5)
    for M in (TALL_M, TALL_M + 200):
        A = torch.randint(-7, 8, (M, 17), generator=g, device="cuda").to(tdt)
        B = torch.randint(-7, 8, (17, 17), generator=g, device="cuda").to(tdt)
        C = torch.full((M, 17), float("nan"), dtype=tdt, device="cuda")
        assert gemm_route(dtype, A, B, C, _sms(torch)) == "simt11" and _cdiv(M, 64) > 65535
        _gemm(L, torch, dtype, A, B, C, 1.0, 0.0)
        ref = A.double() @ B.double()
        assert bool((C.double() == ref).all()), f"{int((C.double() != ref).any(dim=1).sum())} rows differ"
        del A, C, ref


@pytest.mark.parametrize("dtype", [f32, f64])
def test_tall_gemm_graph(gpu, dtype):
    """X (4.2M x 17) @ W (17 x 17): the C linker computes it; so must the device."""
    if not gpu:
        pytest.skip("a 0.3-0.6 GB product")
    rng = np.random.default_rng(11)
    X = rng.integers(-7, 8, (TALL_M + 5, 17)).astype(dtype)
    W = rng.integers(-7, 8, (17, 17)).astype(dtype)
    x, w = pt.matrix("x", dtype=dtype), pt.matrix("w", dtype=dtype)
    compare_cuda_and_cvm([x, w], [pt.dot(x, w)], [X, W], exact=True)


def test_empty_contraction_bias_tanh_graph(gpu):
    """tanh(x @ W + b) with x of 0 columns at run time: tanh(b) in every row (the fused bias epilogue at K = 0)."""
    pytensor.config.floatX = "float32"
    x, W, b = pt.fmatrix("x"), pt.fmatrix("W"), pt.fvector("b")
    bv = np.linspace(-2, 2, 7).astype(np.float32)
    f, got = compare_cuda_and_cvm([x, W, b], [pt.tanh(pt.dot(x, W) + b)], [np.zeros((5, 0), np.float32),
                                                                           np.zeros((0, 7), np.float32), bv],
                                  rtol=1e-6, atol=1e-6)
    assert any(type(st.impl).__name__ == "GemmBiasActNode" for st in f.vm.executor.program.steps)
