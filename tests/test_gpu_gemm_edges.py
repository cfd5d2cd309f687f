"""The tensor-core GEMM (ptk_gemm_tc.cu) at its edges, against fp64 references of the same operation.

a. Integer-grid operands x = n * 2^e (|n| <= 127, e per row of A / column of B) are exact in bf16, so every correction
   piece is 0 and every product is an integer on one unit: while each exact output, alpha * acc + beta * C + bias included,
   fits in 24 bits of its finest unit, EVERY tensor-core mode must reproduce the fp64 product bit for bit — ragged M / N /
   K, more tiles than SMs, K-chunked accumulation with beta, every C layout the epilogue handles.
b. Random operands whose rows of A / columns of B span 2^+-20: every element within c * (|A| @ |B|)_ij of fp64.
c. The staged output pieces an epilogue writes for the next product, bit for bit, and nothing outside [M, N] touched.
d. Workspace rows past M / N hold garbage that must never reach an output.
e. ±inf / NaN operands give the C linker's inf / NaN pattern (an infinite x staged as (x, 0, 0) meets zero pieces of the
   other operand: inf * 0 = NaN piece products, which the epilogue must not let through).

The C-ABI tests skip in the dry run (PTK_DRY=1); the graph tests go through compare_cuda_and_cvm, which traces them there."""

import numpy as np
import pytest

from helpers import compare_cuda_and_cvm, pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu

MODES = ["bf16", "split6", "split3", "staged1", "staged3", "staged6", "staged6_plain"]
LAYOUTS = ["dense", "slice_odd", "colmajor", "every_other"]
SENTINEL = 12345.0


def _abi(gpu):
    if not gpu:
        pytest.skip("calls the C ABI on the device")
    import torch

    from pytensor_b200.runtime import lib as _lib

    return _lib.lib(), torch


def _c_view(torch, M, N, layout):
    """(view [M, N] with the layout's strides, the whole buffer behind it) — the buffer is filled with SENTINEL."""
    if layout == "dense":
        big = torch.full((M, N), SENTINEL, device="cuda")
        return big, big
    if layout == "slice_odd":   # odd element offset, odd row pitch: the float2 path is misaligned on every other row
        big = torch.full((M, N + 3), SENTINEL, device="cuda")
        return big[:, 1:N + 1], big
    if layout == "colmajor":    # sc0 = 1, sc1 = M
        big = torch.full((N, M), SENTINEL, device="cuda")
        return big.t(), big
    big = torch.full((M, 2 * N), SENTINEL, device="cuda")   # both strides non-unit
    return big[:, ::2], big


def _run(mode, torch, A, B, C, alpha, beta, bias=None, act=0):
    """C = act(alpha * A @ B + beta * C + bias) through the tensor-core entry point `mode` (torch device tensors)."""
    from pytensor_b200.runtime import device as dev
    from pytensor_b200.runtime import lib as _lib
    from pytensor_b200.vm import nodes_blas as nb

    L = _lib.lib()
    M, K = A.shape
    N = B.shape[1]
    st = dev.stream_ptr()
    bp = bias.data_ptr() if bias is not None else None
    if mode == "bf16":
        wsb = int(L.ptk_gemm_workspace_bytes(M, N, K, 1))
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
        _lib.check(L.ptk_gemm_tc_ex(M, N, K, alpha, A.data_ptr(), A.stride(0), A.stride(1), None, 0, B.data_ptr(), B.stride(0),
                                    B.stride(1), beta, C.data_ptr(), C.stride(0), C.stride(1), bp, act, None, 0, ws.data_ptr(),
                                    wsb, st), "ptk_gemm_tc_ex")
    elif mode in ("split6", "split3"):
        wsb = int(L.ptk_gemm_split_workspace_bytes(M, N, K))
        ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
        _lib.check(L.ptk_gemm_tc_split(M, N, K, alpha, A.data_ptr(), A.stride(0), A.stride(1), B.data_ptr(), B.stride(0),
                                       B.stride(1), beta, C.data_ptr(), C.stride(0), C.stride(1), bp, act,
                                       6 if mode == "split6" else 3, ws.data_ptr(), wsb, st), "ptk_gemm_tc_split")
    else:
        pieces, terms, aligned = {"staged1": (1, 1, False), "staged3": (3, 3, False), "staged6": (3, 6, True),
                                  "staged6_plain": (3, 6, False)}[mode]
        Ast = nb.stage_operand(A, pieces, aligned=aligned)
        Bst = nb.stage_operand(B, pieces, transposed=True, aligned=aligned)
        nb.gemm_staged(Ast, Bst, terms, alpha, beta, C, bias=bias, act=act)
    torch.cuda.synchronize()


def _grid(rng, rows, cols, nmax, emin, emax, axis):
    """n * 2^e, |n| <= nmax, one exponent per row (axis 0) or per column (axis 1); returns (values, exponents)."""
    n = rng.integers(-nmax, nmax + 1, size=(rows, cols)).astype(np.float64)
    e = rng.integers(emin, emax + 1, size=rows if axis == 0 else cols)
    x = n * np.exp2(e)[:, None] if axis == 0 else n * np.exp2(e)[None, :]
    return x, e


# alpha, beta, integer-grid bias; with beta != 0 or a bias the operands stay small and their exponents narrow
EPILOGUES = [(1.0, 0.0, False), (-2.0, 1.0, False), (0.5, -0.5, True)]


def _grid_case(rng, M, N, K, alpha, beta, with_bias):
    plain = beta == 0.0 and not with_bias
    nmax, (emin, emax) = (127, (-10, 10)) if plain else (7, (-1, 1))
    A, ea = _grid(rng, M, K, nmax, emin, emax, 0)
    B, eb = _grid(rng, K, N, nmax, emin, emax, 1)
    C0, ec = _grid(rng, M, N, 1023, -2, -2, 0)
    bias = (rng.integers(-255, 256, N) * 2.0 ** -2) if with_bias else None
    ref = alpha * (A @ B) + (beta * C0 if beta else 0.0) + (bias if with_bias else 0.0)
    # precondition: every exact output, its partial sums included, fits in 24 bits of its finest unit, so the tensor
    # core's fp32 accumulation and the epilogue's fp32 adds are exact
    unit = abs(alpha) * np.exp2(ea[:, None] + eb[None, :])
    bound = abs(alpha) * (np.abs(A) @ np.abs(B))
    if beta:
        unit = np.minimum(unit, abs(beta) * np.exp2(ec)[:, None])
        bound = bound + np.abs(beta * C0)
    if with_bias:
        unit = np.minimum(unit, 2.0 ** -2)
        bound = bound + np.abs(bias)[None, :]
    assert np.all(bound < 2.0 ** 24 * unit), "test operands break the exactness precondition"
    assert np.array_equal(ref.astype(np.float32).astype(np.float64), ref)
    return A.astype(np.float32), B.astype(np.float32), C0.astype(np.float32), bias, ref


def _check_grid(gpu, mode, M, N, K, alpha, beta, with_bias, layout, seed):
    L, torch = _abi(gpu)
    rng = np.random.default_rng(seed)
    A, B, C0, bias, ref = _grid_case(rng, M, N, K, alpha, beta, with_bias)
    Cv, big = _c_view(torch, M, N, layout)
    Cv.copy_(torch.from_numpy(C0) if beta else torch.full((M, N), float("nan")))   # beta == 0: C must not be read
    bt = torch.from_numpy(bias.astype(np.float32)).cuda() if with_bias else None
    _run(mode, torch, torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), Cv, alpha, beta, bias=bt)
    got = Cv.cpu().numpy().astype(np.float64)
    np.testing.assert_array_equal(got, ref)
    Cv.fill_(SENTINEL)   # what is left of the write is what the epilogue wrote outside its [M, N] view
    assert bool((big == SENTINEL).all()), "the epilogue wrote outside its [M, N] view"


# 319 rows leave the second consumer warpgroup of the last tile partly masked; K = 1000 gives the 3-term mode two
# accumulation chunks (8 k-blocks each); (2049, 2051, 520) has more 128 x 128 tiles than the H100's 132 SMs
SHAPES = [(256, 256, 256), (257, 257, 257), (319, 263, 300), (383, 511, 1000), (256, 257, 1024), (2049, 2051, 520)]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("mode", MODES)
def test_integer_grid_is_bit_exact(gpu, mode, M, N, K):
    i = SHAPES.index((M, N, K))
    alpha, beta, with_bias = EPILOGUES[i % 3]
    _check_grid(gpu, mode, M, N, K, alpha, beta, with_bias, LAYOUTS[i % 4], seed=100 + i)


@pytest.mark.parametrize("epi", range(len(EPILOGUES)))
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("mode", MODES)
def test_integer_grid_every_layout_and_epilogue(gpu, mode, layout, epi):
    alpha, beta, with_bias = EPILOGUES[epi]
    _check_grid(gpu, mode, 257, 263, 1000, alpha, beta, with_bias, layout, seed=200 + epi)


# ---- b. accuracy, element by element -------------------------------------------------------------------------------------
def _scaled_normal(rng, M, N, K):
    A = rng.standard_normal((M, K)) * np.exp2(rng.uniform(-20, 20, (M, 1)))
    B = rng.standard_normal((K, N)) * np.exp2(rng.uniform(-20, 20, (1, N)))
    return A.astype(np.float32), B.astype(np.float32)


def _bf16(torch, x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).bfloat16().double().numpy()


def _split6_c(K):
    """Per-element bound of the default fp32-accurate mode, as a fraction of (|A| @ |B|)_ij.  Error model
    (test_gemm_split_model_cpu.py): the error-free leading products are exact; what is left is (i) the dropped piece
    products and the split's own 2^-23-of-the-row-maximum residue, (ii) the final round-to-nearest adds, both below 2^-22,
    and (iii) the truncation of the correction accumulator, which grows linearly with the accumulation chain: about 3e-7
    for a chain of 4096.  Chunks (split_kchunk) hold at most 16384: up to 4x that — so c = 1e-6 up to a chain of 4096 and
    1e-6 * chain / 4096 beyond."""
    chain = min(K, 16384)
    return 1e-6 * max(1.0, chain / 4096)


def _bf16_c(K):
    """bf16 mode against its model (fp64 product of the bf16-rounded operands): only the fp32 accumulation errs; one
    truncating add per 16-deep wgmma step, each off by at most 2^-23 of a partial sum <= (|Ab| @ |Bb|)."""
    return (K / 16 + 2) * 2.0 ** -23


ACC_SHAPES = [(257, 263, 300), (383, 511, 1000), (256, 256, 4096), (300, 260, 4097)]


@pytest.mark.parametrize("M,N,K", ACC_SHAPES)
@pytest.mark.parametrize("mode", ["split6", "bf16"])
def test_rows_and_columns_of_different_scales_meet_an_elementwise_bound(gpu, mode, M, N, K):
    L, torch = _abi(gpu)
    rng = np.random.default_rng(M + N + K)
    A, B = _scaled_normal(rng, M, N, K)
    C = torch.full((M, N), float("nan"), device="cuda")
    _run(mode, torch, torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), C, 1.0, 0.0)
    got = C.cpu().numpy().astype(np.float64)
    if mode == "bf16":
        A64, B64, c = _bf16(torch, A), _bf16(torch, B), _bf16_c(K)
    else:
        A64, B64, c = A.astype(np.float64), B.astype(np.float64), _split6_c(K)
    err = np.abs(got - A64 @ B64) / (np.abs(A64) @ np.abs(B64))
    assert err.max() <= c, f"max error {err.max():.2e} of (|A| @ |B|)_ij, bound {c:.1e}"


@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("mode", ["split6", "bf16"])
def test_two_accumulation_chunks_with_beta_and_bias(gpu, mode, act):
    """K = 16448 = 257 k-blocks: the exact mode accumulates 256 k-blocks, then one partial k-block (chunk 0 applies beta,
    chunk 1 adds onto C), then bias and tanh.  A tanh output lies within c * (|A| @ |B|)_ij + 2^-23 of fp64 tanh of the fp64
    pre-activation (tanh is 1-Lipschitz; 2^-23: its own rounding)."""
    L, torch = _abi(gpu)
    M = N = 256
    K = 16448
    rng = np.random.default_rng(7 + act)
    A = (rng.standard_normal((M, K)) * np.exp2(rng.uniform(-6, 6, (M, 1)))).astype(np.float32)
    B = (rng.standard_normal((K, N)) * np.exp2(rng.uniform(-6, 6, (1, N)))).astype(np.float32)
    if act:
        A = (A / np.abs(A).max(axis=1, keepdims=True) / 64).astype(np.float32)   # pre-activations of order 1
    C0 = rng.standard_normal((M, N)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    alpha, beta = 0.75, -1.25
    C = torch.from_numpy(C0).cuda()
    _run(mode, torch, torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), C, alpha, beta,
         bias=torch.from_numpy(bias).cuda(), act=act)
    got = C.cpu().numpy().astype(np.float64)
    if mode == "bf16":
        A64, B64, c = _bf16(torch, A), _bf16(torch, B), _bf16_c(K)
    else:
        A64, B64, c = A.astype(np.float64), B.astype(np.float64), _split6_c(K)
    pre = alpha * (A64 @ B64) + beta * C0.astype(np.float64) + bias.astype(np.float64)
    # the epilogue's own fp32 operations on alpha * acc, beta * C and bias: a few roundings of their magnitudes
    tol = c * abs(alpha) * (np.abs(A64) @ np.abs(B64)) + 2.0 ** -22 * (abs(alpha) * np.abs(A64 @ B64) + np.abs(beta * C0)
                                                                        + np.abs(bias))
    exp = np.tanh(pre) if act else pre
    if act:
        tol = tol + 2.0 ** -23
    bad = np.abs(got - exp) > tol
    assert not bad.any(), f"{bad.sum()} elements off; worst excess {(np.abs(got - exp) - tol).max():.2e}"


# ---- c. staged output pieces, bit for bit --------------------------------------------------------------------------------
def _bf16_bits(x):
    """float32 -> bf16 bits, round to nearest even (finite inputs)."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _bits_to_f32(h):
    return (h.astype(np.uint32) << 16).view(np.float32)


@pytest.mark.parametrize("kind", ["bf16_copy", "three_pieces", "three_pieces_aligned_tanh"])
def test_staged_output_pieces_bitwise(gpu, kind):
    L, torch = _abi(gpu)
    from pytensor_b200.runtime import device as dev
    from pytensor_b200.runtime import lib as _lib
    from pytensor_b200.vm import nodes_blas as nb

    M, N, K = 257, 263, 300     # rows M .. c_rows and the pad column N of every piece must stay untouched
    rng = np.random.default_rng({"bf16_copy": 1, "three_pieces": 2, "three_pieces_aligned_tanh": 3}[kind])
    A = (rng.standard_normal((M, K)) / 4).astype(np.float32)
    B = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    bias = (rng.standard_normal(N) * 0.1).astype(np.float32)
    pieces, terms, aligned, act = {"bf16_copy": (1, 1, False, 0), "three_pieces": (3, 3, False, 0),
                                   "three_pieces_aligned_tanh": (3, 6, True, 1)}[kind]
    At, Bt = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    Ast = nb.stage_operand(At, pieces, aligned=aligned)
    Bst = nb.stage_operand(Bt, pieces, transposed=True, aligned=aligned)
    ld, c_rows = (N + 7) // 8 * 8, (M + 255) // 256 * 256
    stage = torch.full((pieces * c_rows, ld), 0x2BCD, dtype=torch.int16, device="cuda")   # sentinel bits
    C = torch.empty((M, N), device="cuda")
    out_exp = int(L.ptk_gemm_lead_bits(N)) - 1 if aligned else nb.NO_EXP
    _lib.check(L.ptk_gemm_tc_staged(M, N, K, 1.0, Ast.ptr, Ast.ld, Ast.piece_rows, Bst.ptr, Bst.ld, Bst.piece_rows, terms, 0.0,
                                    C.data_ptr(), C.stride(0), C.stride(1), torch.from_numpy(bias).cuda().data_ptr(), act,
                                    stage.data_ptr(), ld, c_rows, pieces, 1 if aligned else 0, out_exp,
                                    Ast.flags_ptr if Ast.flagged else None, Bst.flags_ptr if Bst.flagged else None, None,
                                    dev.stream_ptr()), "ptk_gemm_tc_staged")
    torch.cuda.synchronize()
    x = C.cpu().numpy()
    st = stage.cpu().numpy().view(np.uint16).reshape(pieces, c_rows, ld)
    rem = x.astype(np.float32)
    for pc in range(pieces):
        if pc == 0 and aligned:
            lead = (np.rint(rem.astype(np.float64) * 2.0 ** out_exp) * 2.0 ** -out_exp).astype(np.float32)
            want = _bf16_bits(lead)
        else:
            want = _bf16_bits(rem)
        np.testing.assert_array_equal(st[pc, :M, :N], want, err_msg=f"piece {pc}")
        rem = (rem - _bits_to_f32(want)).astype(np.float32)   # exact in fp32
        assert np.all(st[pc, M:, :] == 0x2BCD) and np.all(st[pc, :, N:] == 0x2BCD), f"piece {pc} written outside [M, N]"


# ---- d. staging rows past M / N never reach an output --------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["bf16", "split6", "split3"])
def test_workspace_garbage_never_reaches_the_result(gpu, mode):
    L, torch = _abi(gpu)
    from pytensor_b200.runtime import lib as _lib

    M, N, K = 259, 263, 300
    rng = np.random.default_rng(5)
    A, B = (rng.standard_normal((M, K)).astype(np.float32), rng.standard_normal((K, N)).astype(np.float32))
    At, Bt = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    outs = []
    for fill in (0, 0xFF):      # 0xFFFF is a bf16 NaN
        if mode == "bf16":
            wsb = int(L.ptk_gemm_workspace_bytes(M, N, K, 1))
        else:
            wsb = int(L.ptk_gemm_split_workspace_bytes(M, N, K))
        ws = torch.full((wsb,), fill, dtype=torch.uint8, device="cuda")
        C = torch.empty((M, N), device="cuda")
        if mode == "bf16":
            _lib.check(L.ptk_gemm_tc_ex(M, N, K, 1.0, At.data_ptr(), K, 1, None, 0, Bt.data_ptr(), N, 1, 0.0, C.data_ptr(), N, 1,
                                        None, 0, None, 0, ws.data_ptr(), wsb, 0), "ptk_gemm_tc_ex")
        else:
            _lib.check(L.ptk_gemm_tc_split(M, N, K, 1.0, At.data_ptr(), K, 1, Bt.data_ptr(), N, 1, 0.0, C.data_ptr(), N, 1, None,
                                           0, 6 if mode == "split6" else 3, ws.data_ptr(), wsb, 0), "ptk_gemm_tc_split")
        torch.cuda.synchronize()
        outs.append(C.cpu().numpy())
    assert np.isfinite(outs[1]).all()
    np.testing.assert_array_equal(outs[1].view(np.uint32), outs[0].view(np.uint32))


def test_staging_buffer_garbage_never_reaches_the_result(gpu):
    L, torch = _abi(gpu)
    from pytensor_b200.vm import nodes_blas as nb

    M, N, K = 259, 263, 300
    rng = np.random.default_rng(6)
    A, B = rng.standard_normal((M, K)).astype(np.float32), rng.standard_normal((K, N)).astype(np.float32)
    At, Bt = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    outs = []
    for fill in (0, 0xFF):
        Ast, Bst = nb.Staged(M, K, 3, aligned=True), nb.Staged(N, K, 3, aligned=True)
        Ast.buf.fill_(fill)
        Bst.buf.fill_(fill)
        from pytensor_b200.runtime import device as dev
        from pytensor_b200.runtime import lib as _lib

        for st, t, tr in ((Ast, At, False), (Bst, Bt, True)):
            R, Cc = st.rows, st.cols
            sr, sc = (t.stride(1), t.stride(0)) if tr else (t.stride(0), t.stride(1))
            _lib.check(L.ptk_stage_operand(t.data_ptr(), sr, sc, R, Cc, 3, 1, st.ptr, st.ld, st.piece_rows, dev.stream_ptr()),
                       "ptk_stage_operand")
            st.flagged = True
        C = torch.empty((M, N), device="cuda")
        nb.gemm_staged(Ast, Bst, 6, 1.0, 0.0, C)
        torch.cuda.synchronize()
        outs.append(C.cpu().numpy())
    assert np.isfinite(outs[1]).all()
    np.testing.assert_array_equal(outs[1].view(np.uint32), outs[0].view(np.uint32))


# ---- e. ±inf / NaN operands ----------------------------------------------------------------------------------------------
BIG_ROW, BIG_KS = 12, list(range(100, 108))


def _non_finite_operands(M, N, K, seed=9):
    """Finite normal A [M, K], B [K, N] except: A[3] holds +inf and -inf, paired with B rows that mix exact zeros (-> NaN),
    ±1e-3 in columns whose largest value is ~1 (leading piece 0 -> ±inf), normal values; column 30 of B holds -inf and +inf,
    paired with A columns that hold zeros and ±1e-3; NaN in A[9]; A[BIG_ROW] is zero except values near FLT_MAX (one in the
    top binade, >= 127.5 * 2^121, and beyond the largest bf16), whose B partners are <= 1e-30: a finite result of about 1e9.
    (Partners much nearer FLT_MIN would put their bf16 correction pieces below 2^-126, which the tensor core flushes.)"""
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = rng.standard_normal((K, N)).astype(np.float32)
    A[3, 10], A[3, 20] = np.inf, -np.inf
    B[10, 0:4] = 0.0
    B[10, 4:6], B[10, 6:8] = 1e-3, -1e-3
    B[20, 0:2], B[20, 4:6] = 0.0, -1e-3
    B[7, 30], B[50, 30] = -np.inf, np.inf
    A[0:4, 7], A[4:6, 7], A[6:8, 7] = 0.0, 1e-3, -1e-3
    A[0:2, 50], A[8:10, 50] = 0.0, 1e-3
    A[9, 40] = np.nan
    A[BIG_ROW, :] = 0.0
    A[BIG_ROW, BIG_KS] = np.array([3.40e38, -3.39e38, 3.0e38, -3.2e38, 3.3e38, 1e38, -2e38, 3.39e38], np.float32)
    B[BIG_KS, :] = (rng.uniform(-1, 1, (len(BIG_KS), N)) * 1e-30).astype(np.float32)
    return A, B


def _reference_with_non_finite(A, B):
    """fp64 A @ B and |A| @ |B| without BLAS on the non-finite rows / columns: products broadcast, then summed."""
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    rows = np.flatnonzero(~np.isfinite(A64).all(axis=1))
    cols = np.flatnonzero(~np.isfinite(B64).all(axis=0))
    Af, Bf = np.where(np.isfinite(A64), A64, 0.0), np.where(np.isfinite(B64), B64, 0.0)
    ref, mag = Af @ Bf, np.abs(Af) @ np.abs(Bf)
    with np.errstate(invalid="ignore"):
        ref[rows, :] = (A64[rows, :, None] * B64[None, :, :]).sum(axis=1)
        ref[:, cols] = (A64[:, :, None] * B64[None, :, cols]).sum(axis=1)
    return ref, mag


def _assert_same_non_finite(got, ref):
    for f in (np.isnan, np.isposinf, np.isneginf):
        bad = np.argwhere(f(got) != f(ref))
        assert not len(bad), f"{f.__name__} differs at {len(bad)} outputs, first {bad[:4].tolist()}: " \
                             f"got {[got[tuple(i)] for i in bad[:4]]}, want {[ref[tuple(i)] for i in bad[:4]]}"


def _check_non_finite(got, ref, mag, c, big_row_c):
    _assert_same_non_finite(got, ref)
    assert np.isnan(ref).any() and np.isposinf(ref).any() and np.isneginf(ref).any()
    fin = np.isfinite(ref)
    assert np.isfinite(ref[BIG_ROW]).sum() > ref.shape[1] // 2
    err = np.where(fin, np.abs(got - np.where(fin, ref, 0.0)), 0.0)
    cc = np.full(ref.shape[0], c)
    cc[BIG_ROW] = big_row_c
    rel = err / np.maximum(cc[:, None] * mag, 1e-300)
    w = np.unravel_index(np.argmax(rel), rel.shape)
    assert rel.max() <= 1.0, f"finite error {rel.max():.2e} x its bound at {w}: got {got[w]!r}, want {ref[w]!r}, |A|@|B| {mag[w]:.3e}"


def test_the_oracle_gives_the_fp64_non_finite_pattern(gpu):
    """The C linker's sgemm (mode="CVM") on the same operands: the fp64 reference's inf / NaN pattern is its pattern."""
    A, B = _non_finite_operands(300, 264, 320)
    x, y = pt.fmatrix("x"), pt.fmatrix("y")
    got = pytensor.function([x, y], pt.dot(x, y), mode="CVM")(A, B).astype(np.float64)
    ref, _ = _reference_with_non_finite(A, B)
    _assert_same_non_finite(got, ref)


# the leading piece of a B partner ~2^100 below its column's largest value is 0: the two correction pieces carry 16 bits
BIG_ROW_C = 2.0 ** -15


@pytest.mark.parametrize("mode", ["split6", "split3", "staged6", "staged3", "staged6_plain"])
def test_non_finite_operands_fp32_accurate_modes(gpu, mode):
    L, torch = _abi(gpu)
    M, N, K = 300, 264, 320
    A, B = _non_finite_operands(M, N, K)
    C = torch.full((M, N), float("nan"), device="cuda")
    _run(mode, torch, torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), C, 1.0, 0.0)
    ref, mag = _reference_with_non_finite(A, B)
    c = _split6_c(K) if mode in ("split6", "staged6") else 1e-5
    _check_non_finite(C.cpu().numpy().astype(np.float64), ref, mag, c, BIG_ROW_C)


def test_non_finite_operands_tanh_epilogue_abi(gpu):
    """tanh(A @ B + bias) through the default mode: ±1 where the reference has tanh(±inf), NaN where it has NaN."""
    L, torch = _abi(gpu)
    M, N, K = 300, 264, 320
    A, B = _non_finite_operands(M, N, K)
    bias = np.linspace(-1, 1, N).astype(np.float32)
    C = torch.empty((M, N), device="cuda")
    _run("split6", torch, torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), C, 1.0, 0.0,
         bias=torch.from_numpy(bias).cuda(), act=1)
    ref, mag = _reference_with_non_finite(A, B)
    with np.errstate(invalid="ignore"):
        exp = np.tanh(ref + bias)
    got = C.cpu().numpy().astype(np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(exp))
    assert (np.abs(exp[~np.isfinite(ref)]) == 1.0).any()
    fin = ~np.isnan(exp)
    tol = np.where(np.isfinite(ref), _split6_c(K) * mag, 0.0) + 2.0 ** -23
    tol[BIG_ROW] = np.where(np.isfinite(ref[BIG_ROW]), BIG_ROW_C * mag[BIG_ROW], 0.0) + 2.0 ** -23
    bad = np.argwhere(fin & (np.abs(got - exp) > tol))
    assert not len(bad), f"{len(bad)} outputs off, first {bad[:4].tolist()}: got {got[tuple(bad[0])]!r} want {exp[tuple(bad[0])]!r}"


def test_non_finite_operands_bf16_mode_follows_its_model(gpu):
    """bf16 operands: the model is the fp64 product of the bf16-rounded operands, where a value above the largest bf16
    rounds to inf and inf * 0 is NaN."""
    L, torch = _abi(gpu)
    M, N, K = 300, 264, 320
    A, B = _non_finite_operands(M, N, K)
    C = torch.full((M, N), float("nan"), device="cuda")
    _run("bf16", torch, torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), C, 1.0, 0.0)
    Ab, Bb = _bf16(torch, A), _bf16(torch, B)
    assert np.isposinf(Ab[BIG_ROW]).any()   # 3.40e38 rounds to bf16 inf
    ref, mag = _reference_with_non_finite(Ab.astype(np.float32), Bb.astype(np.float32))
    got = C.cpu().numpy().astype(np.float64)
    _assert_same_non_finite(got, ref)
    fin = np.isfinite(ref)
    bad = np.argwhere(fin & (np.abs(got - np.where(fin, ref, 0.0)) > _bf16_c(K) * mag))
    assert not len(bad), f"{len(bad)} outputs off, first {bad[:4].tolist()}: got {got[tuple(bad[0])]!r} want {ref[tuple(bad[0])]!r}"


# graph tests: compare_cuda_and_cvm compares inf / NaN positions exactly (assert_allclose, equal_nan)
def _graph_operands():
    return _non_finite_operands(300, 264, 320)


def test_non_finite_dot_graph(gpu):
    A, B = _graph_operands()
    x, y = pt.fmatrix("x"), pt.fmatrix("y")
    A[BIG_ROW] = 0.0   # (the 2^-16 leading-piece-0 case is checked against fp64 above; CVM parity is 1e-5 here)
    compare_cuda_and_cvm([x, y], pt.dot(x, y), [A, B], rtol=1e-5, atol_scale=1e-5)


def test_non_finite_tanh_layer_and_chain_graph(gpu):
    pytensor.config.floatX = "float32"
    A, W1 = _graph_operands()
    A[BIG_ROW] = 0.0
    W1 = (W1 / 16).astype(np.float32)          # pre-activations of order 1
    rng = np.random.default_rng(3)
    W2 = (rng.standard_normal((264, 256)) / 16).astype(np.float32)
    b1 = np.linspace(-1, 1, 264).astype(np.float32)
    b2 = np.linspace(1, -1, 256).astype(np.float32)
    x, w1, w2, c1, c2 = pt.fmatrix("x"), pt.fmatrix("w1"), pt.fmatrix("w2"), pt.fvector("c1"), pt.fvector("c2")
    h1 = pt.tanh(pt.dot(x, w1) + c1)
    h2 = pt.tanh(pt.dot(h1, w2) + c2)          # the chained three-piece operand of the tanh layer
    compare_cuda_and_cvm([x, w1, w2, c1, c2], [h1, h2], [A, W1, W2, b1, b2], rtol=1e-5, atol=1e-5)


def test_non_finite_constant_weight_graph(gpu):
    """A constant weight is staged once and stays resident: its ±inf column flags must travel with it."""
    A, B = _graph_operands()
    A[BIG_ROW] = 0.0
    x = pt.fmatrix("x")
    out = pt.dot(x, pt.constant(B))
    f, _ = compare_cuda_and_cvm([x], out, [A], rtol=1e-5, atol_scale=1e-5)
    if gpu:
        ref = pytensor.function([x], out, mode="CVM")(A)
        np.testing.assert_allclose(f(A)[0], ref, rtol=1e-5, atol=1e-5 * np.abs(ref[np.isfinite(ref)]).max())   # a resident call


def test_non_finite_matmul_recurrence_graph(gpu):
    from pytensor.scan import scan

    pytensor.config.floatX = "float32"
    rng = np.random.default_rng(4)
    h0v = rng.standard_normal((260, 256)).astype(np.float32)
    h0v[5, 17] = np.inf
    Wv = (rng.standard_normal((256, 256)) * 0.05).astype(np.float32)
    Wv[17, :3] = 0.0                          # inf * 0: NaN in row 5 of the first state
    h0, Wm = pt.fmatrix("h0"), pt.fmatrix("W")
    hs = scan(lambda h, W: pt.tanh(pt.dot(h, W)), outputs_info=[h0], non_sequences=[Wm], n_steps=3, return_updates=False)
    f, got = compare_cuda_and_cvm([h0, Wm], [hs], [h0v, Wv], rtol=1e-5, atol=1e-5)
    assert any(type(st.impl).__name__ == "ScanMatmulRecurrenceNode" for st in f.vm.executor.program.steps)
    if got is not None:
        assert np.isnan(got[0][0, 5]).any() and (np.abs(got[0][0, 5]) == 1.0).any()


@pytest.mark.parametrize("dtype,size", [("float32", 200), ("float64", 300)])
def test_non_finite_operands_fma_path(gpu, dtype, size):
    """Below 256 (and for fp64) the product takes the FMA kernel."""
    A, B = _non_finite_operands(size, size, size)
    A[BIG_ROW] = 0.0
    x, y = pt.matrix("x", dtype=dtype), pt.matrix("y", dtype=dtype)
    compare_cuda_and_cvm([x, y], pt.dot(x, y), [A.astype(dtype), B.astype(dtype)], rtol=1e-5, atol_scale=1e-5)
