"""BLAS-family nodes (reference: pytensor/tensor/blas/gemm.py:76 Gemm, :248 Dot22, :298 Dot22Scalar,
gemv.py:16 Gemv, ger.py:8 Ger, and the generic Dot of pytensor/tensor/math.py).  All arithmetic runs in
ptk_gemm / ptk_gemv / ptk_ger; `precision` selects the bf16 wgmma tensor-core path for fp32 matrices."""

from __future__ import annotations

import numpy as np
import torch

from ..runtime import device as dev
from ..runtime import lib as _lib
from .nodes_basic import _broadcast_view
from .nodes_elemwise import Node
from .values import Val

# Linker-level knob: 0 = fp32-accurate (<= 1e-5 vs BLAS); 1 = bf16 operands / fp32 accumulation
TC_MIN_DIM = 256
# How precision 0 multiplies large fp32 matrices: "tc6" / "tc3" = wgmma with every operand split into three bf16 pieces
# and 6 / 3 piece products per k-block (include/ptk.h ptk_gemm_tc_split; 6 terms is more accurate than sgemm itself,
# 3 terms ~4e-6 of the output scale), "simt" = the fp32 FMA kernel.  fp64 and small / skinny products always take FMA.
import os as _os

FP32_MODE = _os.environ.get("PTK_GEMM_FP32", "tc6")

_workspace = {"buf": None}


def _get_workspace(nbytes: int):
    buf = _workspace["buf"]
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty((max(nbytes, 1),), dtype=torch.uint8, device=dev.device())
        _workspace["buf"] = buf
    return buf


def _scalar(v: Val) -> float:
    return float(np.asarray(v.host()).reshape(-1)[0])


def gemm(dtype, alpha, A, B, beta, C, precision=0, bias=None, act=0, a_bf16=None, want_bf16=False, b_key=None):
    """C = alpha*A@B + beta*C (or act(A@B + bias) when bias/act given) through the C-ABI.
    Tensor-core path extras: `a_bf16` = an already staged bf16 copy of A (skips the staging pass); `want_bf16` returns a
    bf16 copy of C (torch.bfloat16 container) for the next layer, else None."""
    M, K = A.shape
    K2, N = B.shape
    if K != K2 or tuple(C.shape) != (M, N):
        raise ValueError(f"gemm: shape mismatch {tuple(A.shape)} @ {tuple(B.shape)} -> {tuple(C.shape)}")
    L = _lib.lib()
    use_tc = precision == 1 and dtype == "float32" and min(M, N, K) >= TC_MIN_DIM
    code = _lib.DTYPE_CODE[dtype]
    st = dev.stream_ptr()
    plan = tc_plan(dtype, precision, M, N, K) if b_key is not None else None
    if plan is not None:
        # resident weights: B comes from the staged-operand cache, only A is staged per call (or chained from the
        # previous layer's epilogue in the bf16 mode)
        pieces, terms = plan
        Bst = staged_weight(b_key, B, pieces)
        if Bst is not None:
            if isinstance(a_bf16, Staged):
                ok = (a_bf16.pieces, a_bf16.rows, a_bf16.cols, a_bf16.aligned) == (pieces, M, K, Bst.aligned)
                Ast = a_bf16 if ok else stage_operand(A, pieces, aligned=Bst.aligned)
            elif pieces == 1 and a_bf16 is not None and a_bf16.shape[0] == M and a_bf16.shape[1] >= K \
                    and a_bf16.stride(1) == 1 and a_bf16.stride(0) % 8 == 0 and dev.ptr(a_bf16) % 16 == 0:
                Ast = Staged.wrap(a_bf16, M, K)
            else:
                Ast = stage_operand(A, pieces, aligned=Bst.aligned)
            ret = cst = None
            if want_bf16 and pieces == 1:
                ret = dev.empty_t((M, (N + 7) // 8 * 8), torch.bfloat16)
                cst = Staged.wrap(ret, M, N)
            elif want_bf16 and can_chain_pieces(act):
                ret = cst = Staged(M, N, pieces, aligned=Bst.aligned)   # the three-piece operand of the next product
            gemm_staged(Ast, Bst, terms, alpha, beta, C, bias=bias, act=act, out=cst)
            return ret
    if isinstance(a_bf16, Staged):
        a_bf16 = None   # (a chained three-piece operand is only usable together with a resident B)
    if use_tc:
        ws_bytes = int(L.ptk_gemm_workspace_bytes(M, N, K, 1))
        if dev.alloc_state.arena is not None or dev.alloc_state.measuring:
            # inside a captured graph GEMMs may run concurrently on different streams: each gets its own staging area
            ws = dev.empty_t((ws_bytes,), torch.uint8)
        else:
            ws = _get_workspace(ws_bytes)
        cbf = None
        if want_bf16:
            Np = (N + 7) // 8 * 8
            cbf = dev.empty_t((M, Np), torch.bfloat16)
        abf_ptr, lda = None, 0
        if a_bf16 is not None and a_bf16.shape[0] == M and a_bf16.shape[1] >= K and a_bf16.stride(1) == 1:
            abf_ptr, lda = dev.ptr(a_bf16), a_bf16.stride(0)
        _lib.check(L.ptk_gemm_tc_ex(M, N, K, float(alpha), dev.ptr(A), A.stride(0), A.stride(1), abf_ptr, lda, dev.ptr(B),
                                    B.stride(0), B.stride(1), float(beta), dev.ptr(C), C.stride(0), C.stride(1),
                                    dev.ptr(bias) if bias is not None else None, act,
                                    dev.ptr(cbf) if cbf is not None else None, cbf.stride(0) if cbf is not None else 0,
                                    dev.ptr(ws), ws_bytes, st), "ptk_gemm_tc_ex")
        return cbf
    if precision == 0 and dtype == "float32" and FP32_MODE in ("tc6", "tc3") and min(M, N, K) >= TC_MIN_DIM:
        ws_bytes = int(L.ptk_gemm_split_workspace_bytes(M, N, K))
        if dev.alloc_state.arena is not None or dev.alloc_state.measuring:
            ws = dev.empty_t((ws_bytes,), torch.uint8)
        else:
            ws = _get_workspace(ws_bytes)
        _lib.check(L.ptk_gemm_tc_split(M, N, K, float(alpha), dev.ptr(A), A.stride(0), A.stride(1), dev.ptr(B), B.stride(0),
                                       B.stride(1), float(beta), dev.ptr(C), C.stride(0), C.stride(1),
                                       dev.ptr(bias) if bias is not None else None, act, 6 if FP32_MODE == "tc6" else 3,
                                       dev.ptr(ws), ws_bytes, st), "ptk_gemm_tc_split")
        return None
    if bias is not None or act:
        _lib.check(L.ptk_gemm_bias_act(code, M, N, K, dev.ptr(A), A.stride(0), A.stride(1), dev.ptr(B), B.stride(0),
                                       B.stride(1), dev.ptr(bias) if bias is not None else None, act, dev.ptr(C),
                                       C.stride(0), C.stride(1), 0, None, 0, st), "ptk_gemm_bias_act")
    else:
        _lib.check(L.ptk_gemm(code, M, N, K, float(alpha), dev.ptr(A), A.stride(0), A.stride(1), dev.ptr(B),
                              B.stride(0), B.stride(1), float(beta), dev.ptr(C), C.stride(0), C.stride(1),
                              0, None, 0, st), "ptk_gemm")
    return None


def gemv(dtype, alpha, A, x, beta, y):
    M, N = A.shape
    if x.shape[0] != N or y.shape[0] != M:
        raise ValueError(f"gemv: shape mismatch {tuple(A.shape)} @ {tuple(x.shape)} -> {tuple(y.shape)}")
    _lib.check(_lib.lib().ptk_gemv(_lib.DTYPE_CODE[dtype], M, N, float(alpha), dev.ptr(A), A.stride(0), A.stride(1),
                                   dev.ptr(x), x.stride(0), float(beta), dev.ptr(y), y.stride(0), dev.stream_ptr()),
               "ptk_gemv")


# ---- operands staged once, products chained (include/ptk.h: ptk_stage_operand / ptk_gemm_tc_staged) -----------------------
class Staged:
    """A matrix in the tensor-core kernel's operand layout: `pieces` (1 = bf16, 3 = bf16x3 split) K-major matrices
    [rows, cols] stacked with a pitch of `piece_rows` rows in one device buffer."""

    __slots__ = ("buf", "rows", "cols", "ld", "piece_rows", "pieces", "in_graph", "aligned")

    @classmethod
    def wrap(cls, t: torch.Tensor, rows, cols):
        """A caller-provided row-major bf16 matrix (pitch multiple of 8, 16-byte aligned) as a one-piece operand."""
        st = cls.__new__(cls)
        st.rows, st.cols, st.pieces, st.ld, st.piece_rows, st.buf, st.in_graph = int(rows), int(cols), 1, int(t.stride(0)), 0, t, False
        st.aligned = False
        return st

    def __init__(self, rows, cols, pieces, aligned=False):
        self.in_graph = False
        self.aligned = bool(aligned) and int(pieces) == 3   # leading piece on a per-row power-of-two grid (exact main term)
        self.rows, self.cols, self.pieces = int(rows), int(cols), int(pieces)
        self.ld = (self.cols + 7) // 8 * 8
        self.piece_rows = (self.rows + 255) // 256 * 256
        nbytes = int(_lib.lib().ptk_stage_bytes(self.rows, self.cols, self.pieces))
        self.buf = dev.empty_t((nbytes,), torch.uint8)

    @property
    def ptr(self):
        if self.buf.dtype != torch.uint8:   # a caller-provided bf16 matrix used as is (already 16-byte aligned)
            return dev.ptr(self.buf)
        return (dev.ptr(self.buf) + 255) & ~255


def exact_main() -> bool:
    """fp32-accurate products use error-free leading pieces (include/ptk.h) unless PTK_GEMM_EXACT=0."""
    return bool(_lib.lib().ptk_gemm_exact_main_default())


def stage_operand(t: torch.Tensor, pieces: int, transposed: bool = False, aligned: bool | None = None) -> Staged:
    """fp32 matrix -> Staged.  `transposed`: stage t^T — the B operand of A @ B is staged as B^T [N, K].  `aligned`
    (default: whatever the fp32-accurate mode uses): 3-piece split with the leading piece on a per-row power-of-two grid."""
    R, C = (t.shape[1], t.shape[0]) if transposed else (t.shape[0], t.shape[1])
    sr, sc = (t.stride(1), t.stride(0)) if transposed else (t.stride(0), t.stride(1))
    if aligned is None:
        aligned = pieces == 3 and exact_main() and FP32_MODE == "tc6"   # (the 3-term variant needs 8-bit leading pieces)
    st = Staged(R, C, pieces, aligned)
    _lib.check(_lib.lib().ptk_stage_operand(dev.ptr(t), sr, sc, R, C, pieces, 1 if st.aligned else 0, st.ptr, st.ld,
                                            st.piece_rows, dev.stream_ptr()), "ptk_stage_operand")
    return st


def tc_plan(dtype, precision, M, N, K):
    """(pieces, terms) of the tensor-core path this product takes, or None for the FMA kernels."""
    if dtype != "float32" or min(M, N, K) < TC_MIN_DIM:
        return None
    if precision == 1:
        return 1, 1
    if FP32_MODE in ("tc6", "tc3"):
        return 3, 6 if FP32_MODE == "tc6" else 3
    return None


NO_EXP = -100000   # PTK_STAGE_NO_EXP


def can_chain_pieces(act) -> bool:
    """May a product's epilogue write the three-piece operand of the next fp32-accurate product?  With error-free leading
    pieces only when the result is known to lie in [-1, 1] (tanh): the leading piece then sits on the fixed grid 2^-6."""
    return (not exact_main()) or FP32_MODE != "tc6" or act == 1


def gemm_staged(A: Staged, B: Staged, terms, alpha, beta, C, bias=None, act=0, out: Staged | None = None):
    """C = act(alpha * A @ B + beta * C + bias) from staged operands; `out` receives the staged pieces of the result."""
    M, K, N = A.rows, A.cols, B.rows
    if B.cols != K or tuple(C.shape) != (M, N):
        raise ValueError(f"gemm_staged: shape mismatch ({M},{K}) @ ({B.cols},{N}) -> {tuple(C.shape)}")
    exact = 1 if (terms != 1 and A.aligned and B.aligned) else 0
    out_exp = NO_EXP
    if out is not None and out.pieces == 3 and out.aligned:
        if act != 1:
            raise ValueError("gemm_staged: an aligned three-piece output needs a bounded activation (tanh)")
        out_exp = int(_lib.lib().ptk_gemm_lead_bits(N)) - 1   # the result is the A operand of a contraction over N
    _lib.check(_lib.lib().ptk_gemm_tc_staged(M, N, K, float(alpha), A.ptr, A.ld, A.piece_rows, B.ptr, B.ld, B.piece_rows,
                                             int(terms), float(beta), dev.ptr(C), C.stride(0), C.stride(1),
                                             dev.ptr(bias) if bias is not None else None, int(act),
                                             out.ptr if out is not None else None, out.ld if out is not None else 0,
                                             out.piece_rows if out is not None else 0, out.pieces if out is not None else 1,
                                             exact, out_exp, dev.stream_ptr()), "ptk_gemm_tc_staged")


# ---- staged weights stay resident ---------------------------------------------------------------------------------------
# A B operand whose content the VM knows to be unchanged (Val.key: graph constants, caller-owned device tensors that are the
# same object at the same torch version as in the previous calls, device-resident shared variables between updates) is
# staged ONCE and the staged copy is reused by every later call / graph capture; PTK_STAGE_CACHE=0 turns this off.
STAGE_CACHE_ON = _os.environ.get("PTK_STAGE_CACHE", "1") != "0"
STAGE_CACHE_BYTES = int(_os.environ.get("PTK_STAGE_CACHE_MB", "32768")) << 20
_stage_cache: dict = {}   # (key, pieces, shape, strides) -> Staged   (insertion order = LRU order)
_stage_cache_stats = {"hits": 0, "misses": 0, "bytes": 0}


def forget_weights(kind, serial) -> None:
    """Drop every resident staged copy whose content key starts with (kind, serial): the VM calls this when the tensor
    behind a key is replaced or changes version, and when an Executor (with its captured graphs) dies."""
    for ck in [c for c in _stage_cache if c[0][0] == kind and c[0][1] == serial]:
        _stage_cache_stats["bytes"] -= _stage_cache.pop(ck).buf.numel()


def staged_weight(key, t: torch.Tensor, pieces: int) -> Staged | None:
    """The resident staged copy of B (as B^T) for content identity `key`, staging it on first sight; None = not cacheable.
    Keys are ("const", executor serial, slot) or ("in", tracking serial, torch version): process-unique numbers handed out
    by the VM (never id(): ids recycle), so a hit can only be the content it was staged from."""
    if key is None or not STAGE_CACHE_ON or _lib.TRACE_ONLY:
        return None
    ck = (key, pieces, tuple(t.shape), tuple(t.stride()))
    st = _stage_cache.get(ck)
    if st is not None:
        _stage_cache[ck] = _stage_cache.pop(ck)  # most recently used last
        _stage_cache_stats["hits"] += 1
        st.in_graph = st.in_graph or dev.alloc_state.capturing
        return st
    _stage_cache_stats["misses"] += 1
    with dev.unmanaged():          # persistent: outlives the call, never part of a capture arena
        if dev.alloc_state.capturing:
            # stage NOW on a side stream (the operand was complete before the capture began), not as a node of the graph
            side = dev._side_stream()
            with torch.cuda.stream(side):
                st = stage_operand(t, pieces, transposed=True)
            _lib.check(_lib.lib().ptk_sync_stream(side.cuda_stream), "sync")
        else:
            st = stage_operand(t, pieces, transposed=True)
    st.in_graph = dev.alloc_state.capturing
    _stage_cache[ck] = st
    _stage_cache_stats["bytes"] += st.buf.numel()
    if _stage_cache_stats["bytes"] > STAGE_CACHE_BYTES:   # oldest first; buffers a live captured graph reads are kept
        for old in [k for k, v in _stage_cache.items() if k != ck and not v.in_graph]:
            _stage_cache_stats["bytes"] -= _stage_cache.pop(old).buf.numel()
            if _stage_cache_stats["bytes"] <= STAGE_CACHE_BYTES:
                break
    return st


class Dot22Node(Node):
    emit_bf16 = False  # set by the fusion pass when the only consumer is another tensor-core GEMM taking this as A

    def __init__(self, dtype, precision=0, scalar=False, name="Dot22"):
        self.dtype, self.precision, self.scalar, self.name = dtype, precision, scalar, name

    def run(self, vals):
        A, B = vals[0].dev(), vals[1].dev()
        alpha = _scalar(vals[2]) if self.scalar else 1.0
        out = dev.empty((A.shape[0], B.shape[1]), self.dtype)
        aux = None
        if out.numel():
            if A.shape[1] == 0:
                _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(),
                                                       dev.stream_ptr()), "memset")
            else:
                aux = gemm(self.dtype, alpha, A, B, 0.0, out, self.precision, a_bf16=vals[0].aux,
                           want_bf16=self.emit_bf16, b_key=vals[1].key)
        return [Val(d=out, aux=aux)]


class GemmNode(Node):
    """z_out = b*z + a*x@y; in place on z when `inplace` (gemm.py:111-114), z broadcast otherwise (:194-198)."""

    def __init__(self, dtype, inplace, precision=0, name="Gemm"):
        self.dtype, self.inplace, self.precision, self.name = dtype, inplace, precision, name
        self.destroy = {0: 0} if inplace else {}

    def run(self, vals):
        z, a, x, y, b = vals
        X, Y = x.dev(), y.dev()
        alpha, beta = _scalar(a), _scalar(b)
        Z = z.dev()
        M, N = X.shape[0], Y.shape[1]
        if self.inplace and tuple(Z.shape) == (M, N):
            out = Z
        else:
            out = dev.empty((M, N), self.dtype)
            if out.numel() and beta != 0.0:
                dev.copy_strided(out, _broadcast_view(Z, (M, N)))
        if out.numel():
            if X.shape[1] == 0:
                if beta == 0.0:
                    _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(),
                                                           dev.stream_ptr()), "memset")
                else:
                    gemm(self.dtype, 0.0, out[:, :1], out[:1, :], beta, out, 0)
            else:
                gemm(self.dtype, alpha, X, Y, beta, out, self.precision, b_key=y.key)
        return [Val(d=out)]


class GemvNode(Node):
    """y_out = beta*y + alpha*A@x; beta == 0 never reads y (gemv.py:79-86)."""

    def __init__(self, dtype, inplace, name="Gemv"):
        self.dtype, self.inplace, self.name = dtype, inplace, name
        self.destroy = {0: 0} if inplace else {}

    def run(self, vals):
        y, alpha, A, x, beta = vals
        Y, Am, X = y.dev(), A.dev(), x.dev()
        al, be = _scalar(alpha), _scalar(beta)
        out = Y if self.inplace else (dev.clone(Y) if be != 0.0 else dev.empty(tuple(Y.shape), self.dtype))
        if out.numel():
            if Am.shape[1] == 0:
                al = 0.0
                Am = out.as_strided((out.shape[0], 1), (out.stride(0), 1), out.storage_offset())
                X = out[:1]
                if be == 0.0:
                    _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(),
                                                           dev.stream_ptr()), "memset")
                    return [Val(d=out)]
            gemv(self.dtype, al, Am, X, be, out)
        return [Val(d=out)]


class GerNode(Node):
    """A_out = A + alpha * outer(x, y) (ger.py:8)."""

    def __init__(self, dtype, inplace, name="Ger"):
        self.dtype, self.inplace, self.name = dtype, inplace, name
        self.destroy = {0: 0} if inplace else {}

    def run(self, vals):
        A, alpha, x, y = vals
        Am = A.dev() if self.inplace else dev.clone(A.dev())
        X, Y = x.dev(), y.dev()
        if Am.numel():
            _lib.check(_lib.lib().ptk_ger(_lib.DTYPE_CODE[self.dtype], Am.shape[0], Am.shape[1], _scalar(alpha),
                                          dev.ptr(X), X.stride(0), dev.ptr(Y), Y.stride(0), dev.ptr(Am), Am.stride(0),
                                          Am.stride(1), dev.stream_ptr()), "ptk_ger")
        return [Val(d=Am)]


class DotNode(Node):
    """Generic Dot for float vectors/matrices that the BLAS rewrites left alone (1-d x 1-d, etc.)."""

    def __init__(self, dtype, precision=0, name="Dot"):
        self.dtype, self.precision, self.name = dtype, precision, name

    def run(self, vals):
        A, B = vals[0].dev(), vals[1].dev()
        if A.dim() == 2 and B.dim() == 2:
            return Dot22Node(self.dtype, self.precision).run(vals)
        if A.dim() == 2 and B.dim() == 1:
            out = dev.empty((A.shape[0],), self.dtype)
            if out.numel():
                if A.shape[1] == 0:
                    _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(), dev.stream_ptr()), "memset")
                else:
                    gemv(self.dtype, 1.0, A, B, 0.0, out)
            return [Val(d=out)]
        if A.dim() == 1 and B.dim() == 2:
            out = dev.empty((B.shape[1],), self.dtype)
            if out.numel():
                if B.shape[0] == 0:
                    _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(), dev.stream_ptr()), "memset")
                else:
                    gemv(self.dtype, 1.0, B.t(), A, 0.0, out)
            return [Val(d=out)]
        if A.dim() == 1 and B.dim() == 1:
            out = dev.empty((1,), self.dtype)
            if A.shape[0] == 0:
                _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.element_size(), dev.stream_ptr()), "memset")
            else:
                Am = A.as_strided((1, A.shape[0]), (A.shape[0] * max(1, A.stride(0)), A.stride(0)), A.storage_offset())
                gemv(self.dtype, 1.0, Am, B, 0.0, out)
            return [Val(d=out.view(()))]
        raise NotImplementedError(f"Dot with ndims {A.dim()},{B.dim()}")


class GemmBiasActNode(Node):
    """K5: Dot22 followed by Elemwise{act(x + bias_row)} as ONE launch (epilogue of the GEMM kernel).  The reference
    leaves these as two nodes (`Dot22` then `Composite{tanh(i0 + i1)}`, SURVEY.md §2.3 K5); fused by the linker-level
    peephole in link/cuda/fusion_passes.py.  Inputs: A, B, bias (1, N) row; act: 0 none, 1 tanh."""

    emit_bf16 = False

    def __init__(self, dtype, precision, act, name="Dot22+bias+act"):
        self.dtype, self.precision, self.act, self.name = dtype, precision, act, name

    def run(self, vals):
        A, B = vals[0].dev(), vals[1].dev()
        bias = vals[2].dev() if len(vals) > 2 else None  # (two inputs: act(A @ B), no bias)
        M, N = A.shape[0], B.shape[1]
        b1 = None
        if bias is not None:
            if bias.shape[-1] != N:
                raise ValueError(f"{self.name}: bias of shape {tuple(bias.shape)} does not match N={N}")
            b1 = bias.reshape(-1) if bias.is_contiguous() else dev.contiguous(bias).reshape(-1)
        out = dev.empty((M, N), self.dtype)
        if out.numel():
            if A.shape[1] == 0:
                raise NotImplementedError("fused bias epilogue with K == 0")
            aux = gemm(self.dtype, 1.0, A, B, 0.0, out, self.precision, bias=b1, act=self.act, a_bf16=vals[0].aux,
                       want_bf16=self.emit_bf16, b_key=vals[1].key)
            return [Val(d=out, aux=aux)]
        return [Val(d=out)]


class BatchedDotNode(Node):
    """out[i] = dot(a[i], b[i]) over the leading batch axis (reference: BatchedDot, pytensor/tensor/blas/batched.py:18).
    One GEMM launch per batch element on the current stream (strided views, no copies)."""

    def __init__(self, dtype, precision=0, name="BatchedDot"):
        self.dtype, self.precision, self.name = dtype, precision, name

    def run(self, vals):
        A, B = vals[0].dev(), vals[1].dev()
        if A.shape[0] != B.shape[0] or A.shape[2] != B.shape[1]:
            raise ValueError(f"{self.name}: shape mismatch {tuple(A.shape)} x {tuple(B.shape)}")
        nb, M, K = A.shape
        N = B.shape[2]
        out = dev.empty((nb, M, N), self.dtype)
        if out.numel():
            if K == 0:
                _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(),
                                                       dev.stream_ptr()), "memset")
            else:
                for i in range(nb):
                    gemm(self.dtype, 1.0, A[i], B[i], 0.0, out[i], self.precision)
        return [Val(d=out)]


class MlpChainNode(Node):
    """A run of >= 4 dense layers h <- act(h @ W_l + b_l) in which every product feeds only the next one (found by
    link/cuda/fusion_passes.py::fuse_small_mlp_chains).  When every layer is at most 128 wide — the BASELINE metric graph at
    n = 64: 84 layers of 64x64 — the whole chain is ONE launch (`ptk_mlp_chain`: activations stay in shared memory, weights
    stream in behind the arithmetic) instead of one launch per layer at ~3 us each; otherwise the constituent nodes run one
    after the other exactly as they would have in the program (tensor cores, resident weights, chained operands).
    Inputs: [A0, W_0, (b_0), W_1, (b_1), ...]; `layers` = [(node, has_bias), ...]."""

    MAX_W = 128

    def __init__(self, layers, name="MlpChain"):
        self.layers = list(layers)
        self.name = name
        self.fused_calls = self.unfused_calls = 0
        pos, wpos = 1, []
        for _, has_bias in self.layers:
            wpos.append(pos)
            pos += 2 if has_bias else 1
        self.weight_in_positions = wpos   # (Program.weight_inputs: the B operands this node reads directly)

    def _small(self, vals):
        if vals[0].ndim != 2 or vals[0].dtype != "float32" or vals[0].shape[0] == 0 or not 1 <= vals[0].shape[1] <= self.MAX_W:
            return None
        pos = 1
        for node, has_bias in self.layers:   # shapes first (metadata only): nothing is uploaded for a chain that stays unfused
            w = vals[pos]
            if node.dtype != "float32" or w.ndim != 2 or w.dtype != "float32" or not 4 <= w.shape[1] <= self.MAX_W or w.shape[1] % 4:
                return None
            pos += 2 if has_bias else 1
        A = vals[0].dev()
        if A.shape[1] > 1 and A.stride(1) != 1:
            return None
        width, pos, spec = A.shape[1], 1, []
        if not 1 <= width <= self.MAX_W:
            return None
        for node, has_bias in self.layers:
            W = vals[pos].dev()
            b = vals[pos + 1].dev() if has_bias else None
            if (W.dim() != 2 or W.shape[0] != width or not 4 <= W.shape[1] <= self.MAX_W or W.shape[1] % 4 or not W.is_contiguous()
                    or dev.ptr(W) % 16 or W.dtype != torch.float32):
                return None
            if has_bias and (b is None or b.numel() != W.shape[1] or not b.is_contiguous() or b.dtype != torch.float32):
                return None
            spec.append((W, b, int(getattr(node, "act", 0))))
            width = W.shape[1]
            pos += 2 if has_bias else 1
        return A, spec

    def run(self, vals):
        small = self._small(vals) if _os.environ.get("PTK_MLP_CHAIN", "1") != "0" else None
        if small is None:
            self.unfused_calls += 1
            h, pos = vals[0], 1
            for node, has_bias in self.layers:
                n = 2 if has_bias else 1
                h = node.run([h, *vals[pos:pos + n]])[0]   # the previous activation dies with this rebinding
                pos += n
            return [h]
        self.fused_calls += 1
        A, spec = small
        import ctypes

        L = _lib.lib()
        cur, M = A, A.shape[0]
        for s0 in range(0, len(spec), 96):                  # (ptk_mlp_chain takes up to 96 layers per launch)
            seg = spec[s0:s0 + 96]
            n = len(seg)
            out = dev.empty((M, seg[-1][0].shape[1]), "float32")
            Wp = (ctypes.c_void_p * n)(*[dev.ptr(w) for w, _, _ in seg])
            Bp = (ctypes.c_void_p * n)(*[(dev.ptr(b) if b is not None else None) for _, b, _ in seg])
            Ks = (ctypes.c_int * n)(*[w.shape[0] for w, _, _ in seg])
            Ns = (ctypes.c_int * n)(*[w.shape[1] for w, _, _ in seg])
            acts = (ctypes.c_int * n)(*[a for _, _, a in seg])
            _lib.check(L.ptk_mlp_chain(dev.ptr(cur), cur.stride(0), dev.ptr(out), out.stride(0), M, n, Wp, Bp, Ks, Ns, acts,
                                       dev.stream_ptr()), "ptk_mlp_chain")
            cur = out
        return [Val(d=cur)]
