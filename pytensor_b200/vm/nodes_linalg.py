"""Cholesky / SolveTriangular / CholeskySolve / positive-definite Solve / AllocDiag nodes (reference:
pytensor/tensor/linalg/decomposition/cholesky.py:18, solvers/triangular.py:13, solvers/psd.py:14, solvers/general.py:17,
tensor/basic.py:3887; batched through Blockwise, tensor/blockwise.py:153)."""

from __future__ import annotations

import numpy as np

from ..runtime import device as dev
from ..runtime import lib as _lib
from .nodes_cast import cast_to
from .nodes_elemwise import Node
from .values import Val


class CholeskyNode(Node):
    serial_group = "linalg"  # the blocked kernels share one device status word: never overlap two of them

    def __init__(self, dtype, lower=True, name="Cholesky"):
        self.dtype, self.lower, self.name = dtype, lower, name

    def run(self, vals):
        a = vals[0].dev()
        if a.shape[-1] != a.shape[-2]:
            raise ValueError("Cholesky: last two dims must be square")
        out = dev.clone(a) if a.numel() else dev.empty(tuple(a.shape), self.dtype)
        n = a.shape[-1]
        batch = out.numel() // (n * n) if n else 0
        if n and batch:
            _lib.check(_lib.lib().ptk_potrf(_lib.DTYPE_CODE[self.dtype], dev.ptr(out), n, batch, 1 if self.lower else 0,
                                            dev.stream_ptr()), "ptk_potrf")
        return [Val(d=out)]


class SolveTriangularNode(Node):
    """x = solve(op(A), b): lower/upper, trans, unit_diagonal, b_ndim 1|2 (triangular.py:16-21)."""

    serial_group = "linalg"

    def __init__(self, dtype, lower, unit_diagonal, b_ndim, trans=0, name="SolveTriangular"):
        self.dtype, self.lower, self.unit_diagonal, self.b_ndim, self.trans, self.name = (
            dtype, lower, unit_diagonal, b_ndim, trans, name)

    def run(self, vals):
        A = dev.contiguous(vals[0].dev())
        b = vals[1].dev()
        n = A.shape[-1]
        if self.b_ndim == 1:
            bb = b.unsqueeze(-1)
        else:
            bb = b
        if bb.shape[-2] != n:
            raise ValueError("SolveTriangular: A and b have incompatible shapes")
        out = dev.clone(bb) if bb.numel() else dev.empty(tuple(bb.shape), self.dtype)
        nrhs = bb.shape[-1]
        batchA = A.numel() // (n * n) if n else 0
        batchB = out.numel() // (n * nrhs) if (n and nrhs) else 0
        if n and nrhs and batchB:
            if batchA != batchB:
                raise NotImplementedError("SolveTriangular: broadcasting between batched A and b")
            _lib.check(_lib.lib().ptk_trsm(_lib.DTYPE_CODE[self.dtype], dev.ptr(A), dev.ptr(out), n, nrhs, batchB,
                                           1 if self.lower else 0, 1 if self.trans else 0,
                                           1 if self.unit_diagonal else 0, dev.stream_ptr()), "ptk_trsm")
        if self.b_ndim == 1:
            out = out.squeeze(-1)
        return [Val(d=out)]


def _batch_shape(shapes, bcast):
    """Output batch shape of a Blockwise over inputs with batch shapes `shapes` and static batch broadcast patterns `bcast`,
    raising what the reference's vectorised perform raises (tensor/blockwise.py:84-93): ValueError for a length-1 dimension
    that was not marked broadcastable beside a longer one, and for lengths that do not broadcast."""
    for dims in zip(*[tuple(zip(s, b)) for s, b in zip(shapes, bcast)]):
        if any(d != 1 for d, _ in dims) and (1, False) in dims:
            raise ValueError("Runtime broadcasting not allowed. At least one input has a distinct batch dimension length of 1, "
                             "but was not marked as broadcastable.")
    return tuple(np.broadcast_shapes(*shapes))


def _solve_with_factor(dtype, factor, b, b_ndim, lower, bcast):
    """x = A^-1 b with A given by its Cholesky factor (?potrs): the (batch..., n, n) `factor` is contiguous in `dtype`,
    `b` has b_ndim core dimensions.  b is broadcast into a fresh output buffer and solved there in place."""
    n = factor.shape[-1]
    fb, bb = tuple(factor.shape[:-2]), tuple(b.shape[:b.dim() - b_ndim])
    if b.shape[b.dim() - b_ndim] != n:
        raise ValueError(f"incompatible dimensions ({tuple(factor.shape[-2:])} and {tuple(b.shape[b.dim() - b_ndim:])})")
    batch = _batch_shape([fb, bb], bcast)
    core = (n,) if b_ndim == 1 else (n, b.shape[-1])
    out = dev.empty(batch + core, dtype)
    if out.numel() == 0:
        return out
    dev.copy_strided(out, cast_to(b, dtype).expand(batch + core))
    shape, strides = [], []
    for d, size in enumerate(batch):      # drop length-1 dimensions, merge dimensions the factor walks contiguously
        if size == 1:
            continue
        st = factor.stride(d) if fb[d] != 1 else 0
        if shape and strides[-1] == st * size:
            shape[-1] *= size
            strides[-1] = st
        else:
            shape.append(size)
            strides.append(st)
    if len(shape) > 8:
        raise NotImplementedError("CholeskySolve: more than 8 batch dimensions that do not collapse")
    nrhs = 1 if b_ndim == 1 else b.shape[-1]
    _lib.check(_lib.lib().ptk_potrs(_lib.DTYPE_CODE[dtype], dev.ptr(factor), dev.ptr(out), n, nrhs, 1 if lower else 0,
                                    len(shape), dev.i64_array(shape), dev.i64_array(strides), dev.stream_ptr()), "ptk_potrs")
    return out


class CholeskySolveNode(Node):
    """x = cho_solve((C, lower), b) (solvers/psd.py:14, perform :35-54 = LAPACK ?potrs), plain or through Blockwise: factor
    and b are cast to the op's output dtype, the batch dimensions broadcast.  Unlike SolveTriangular there is no singularity
    check: a zero pivot gives IEEE inf / NaN, as ?potrs does.  Always writes a fresh buffer (overwrite_b is a permission)."""

    serial_group = "linalg"

    def __init__(self, dtype, lower, b_ndim, overwrite_b=False, bcast=((), ()), name="CholeskySolve"):
        self.dtype, self.lower, self.b_ndim, self.overwrite_b, self.bcast, self.name = (
            dtype, lower, b_ndim, overwrite_b, bcast, name)

    def run(self, vals):
        c, b = vals[0].dev(), vals[1].dev()
        if c.shape[-1] != c.shape[-2]:
            raise ValueError("The factored matrix c is not square.")
        factor = dev.contiguous(cast_to(c, self.dtype))
        return [Val(d=_solve_with_factor(self.dtype, factor, b, self.b_ndim, self.lower, self.bcast))]


class PosSolveNode(Node):
    """x = solve(A, b, assume_a="pos") (solvers/general.py:17, perform :60-75), plain or through Blockwise: A is copied in the
    output dtype, factored in place (ptk_potrf reads the triangle `lower` names) and the factor solved (ptk_potrs).  A matrix
    that is not positive definite NaN-fills its factor, so its solution is all NaN with b's shape; the reference returns
    NaN with A's shape there (DESIGN.md §9)."""

    serial_group = "linalg"

    def __init__(self, dtype, lower, b_ndim, bcast=((), ()), name="Solve"):
        self.dtype, self.lower, self.b_ndim, self.bcast, self.name = dtype, lower, b_ndim, bcast, name

    def run(self, vals):
        A, b = vals[0].dev(), vals[1].dev()
        if A.shape[-1] != A.shape[-2]:
            raise ValueError("Input a needs to be a square matrix.")
        a = cast_to(A, self.dtype)
        a = dev.clone(a) if a is A else dev.contiguous(a)       # a private contiguous copy: factored in place
        n = a.shape[-1]
        nmat = a.numel() // (n * n) if n else 0
        if nmat:
            _lib.check(_lib.lib().ptk_potrf(_lib.DTYPE_CODE[self.dtype], dev.ptr(a), n, nmat, 1 if self.lower else 0,
                                            dev.stream_ptr()), "ptk_potrf")
        return [Val(d=_solve_with_factor(self.dtype, a, b, self.b_ndim, self.lower, self.bcast))]


class AllocDiagNode(Node):
    """Blockwise(AllocDiag) (tensor/basic.py:3887, inner graph :3903-3922): x (batch..., k) -> (batch..., m, m), m = k + |offset|,
    zero everywhere but diagonal `offset`, which holds x.  A memset and a strided copy into the diagonal view."""

    def __init__(self, offset, name="AllocDiag"):
        self.offset, self.name = int(offset), name

    def run(self, vals):
        x = vals[0].dev()
        m = x.shape[-1] + abs(self.offset)
        out = dev.empty_t(tuple(x.shape[:-1]) + (m, m), x.dtype)
        if out.numel():
            _lib.check(_lib.lib().ptk_memset_async(dev.ptr(out), 0, out.numel() * out.element_size(), dev.stream_ptr()),
                       "memset")
            dev.copy_strided(out.diagonal(self.offset, -2, -1), x)
        return [Val(d=out)]
