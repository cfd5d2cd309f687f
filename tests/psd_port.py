"""NumPy restatement of the Cholesky-solve nodes (vm/nodes_linalg.py CholeskySolveNode, PosSolveNode, AllocDiagNode) for the
port-oracle check of lowered programs: `evaluate_program` interprets a program like oracle/numpy_port.evaluate_program,
taking these three nodes from here and every other node from the port oracle.

  CholeskySolve   pytensor/tensor/linalg/solvers/psd.py:35-54 (?potrs on the factor)
  Solve, "pos"    pytensor/tensor/linalg/solvers/general.py:60-75 (?potrf, then ?potrs)
  AllocDiag       pytensor/tensor/basic.py:3903-3922 (zeros, then the diagonal set)
Batches loop over the broadcast batch shape like Blockwise (tensor/blockwise.py:84-120)."""

import numpy as np
import scipy.linalg

from oracle import numpy_port


def _psd_solve(node, a, b, factored):
    """A matrix that is not positive definite gives NaN of b's core shape, as the device does (DESIGN.md §9)."""
    dt = np.dtype(node.dtype)
    cb = b.ndim - node.b_ndim
    batch = np.broadcast_shapes(a.shape[:-2], b.shape[:cb])
    a = np.broadcast_to(a, batch + a.shape[-2:]).astype(dt)
    b = np.broadcast_to(b, batch + b.shape[cb:]).astype(dt)
    potrf, potrs = scipy.linalg.lapack.get_lapack_funcs(("potrf", "potrs"), (np.empty(0, dt),))
    out = np.empty(b.shape, dtype=dt)
    for i in np.ndindex(*batch):
        c = a[i]
        if not factored:
            c, info = potrf(c, lower=node.lower)
            if info != 0:
                out[i] = np.nan
                continue
        out[i] = potrs(c, b[i], lower=node.lower)[0] if b[i].size else b[i]
    return out


def _alloc_diag(node, x):
    k, off = x.shape[-1], node.offset
    out = np.zeros(x.shape[:-1] + (k + abs(off),) * 2, dtype=x.dtype)
    idx = np.arange(k)
    out[..., idx + max(0, -off), idx + max(0, off)] = x
    return out


def eval_node(node, vals):
    name = type(node).__name__
    if name in ("CholeskySolveNode", "PosSolveNode"):
        return [_psd_solve(node, np.asarray(vals[0]), np.asarray(vals[1]), factored=name == "CholeskySolveNode")]
    if name == "AllocDiagNode":
        return [_alloc_diag(node, np.asarray(vals[0]))]
    if name == "SolveTriangularNode" and node.b_ndim == 1 and np.ndim(vals[1]) > 1:
        # a batch of vectors: SciPy's batched solve_triangular would read b's batch axis as its core one
        x = scipy.linalg.solve_triangular(vals[0], np.asarray(vals[1])[..., None], lower=node.lower,
                                          unit_diagonal=node.unit_diagonal)
        return [x[..., 0]]
    return numpy_port.eval_node(node, vals)


def evaluate_program(program, inputs):
    vals = [None] * program.n_slots
    for s, a in program.constants.items():
        vals[s] = np.asarray(a)
    for s, x in zip(program.inputs, inputs):
        vals[s] = np.asarray(x)
    for st in program.steps:
        for j, r in zip(st.outs, eval_node(st.impl, [vals[j] for j in st.ins])):
            vals[j] = r
    return [np.asarray(vals[s]) for s in program.outputs]
