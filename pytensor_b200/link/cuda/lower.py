"""Lowering: PyTensor `Apply` node -> executable CUDA node (pytensor_b200.vm.*).

This is the backend's analogue of `Op.make_thunk` (pytensor/graph/op.py:610-659) / `COp.make_c_thunk`
(pytensor/link/c/op.py:38-106): it is called once per node at link time, and raises `NotImplementedError` for any
op without an sm_90a implementation — compile-time, never a CPU fallback (SURVEY.md §7 step 1).
"""

from __future__ import annotations

import numpy as np

from pytensor.compile.ops import DeepCopyOp, ViewOp
from pytensor.graph.basic import Constant
from pytensor.raise_op import CheckAndRaise
from pytensor.scalar import basic as ps
from pytensor.tensor.basic import (
    Alloc,
    AllocEmpty,
    Join,
    MakeVector,
    ScalarFromTensor,
    TensorFromScalar,
)
from pytensor.tensor.blas import Dot22, Dot22Scalar, Gemm, Gemv, Ger
from pytensor.tensor.blockwise import Blockwise
from pytensor.tensor.elemwise import CAReduce, DimShuffle, Elemwise
from pytensor.tensor.math import Dot
from pytensor.tensor.shape import Reshape, Shape, Shape_i, SpecifyShape
from pytensor.tensor.subtensor import (
    AdvancedIncSubtensor,
    AdvancedSubtensor,
    IncSubtensor,
    Subtensor,
)

from pytensor_b200.codegen.scalar import ScalarInst, ScalarProgram, UnsupportedScalarOp, OPS, simplify
from pytensor_b200.vm import nodes_basic as nb
from pytensor_b200.vm import nodes_blas as nblas
from pytensor_b200.vm import nodes_linalg as nlin
from pytensor_b200.vm.nodes_elemwise import CAReduceNode, ElemwiseNode


class UnsupportedOp(NotImplementedError):
    pass


# ---- scalar graphs ------------------------------------------------------------------------------------------------
def scalar_program(scalar_op, in_dtypes, out_dtypes) -> ScalarProgram:
    """ScalarOp (possibly a nested Composite) -> ScalarProgram."""
    prog = ScalarProgram(in_dtypes=list(in_dtypes), out_dtypes=list(out_dtypes))

    def emit(op, arg_refs, arg_dtypes, out_types):
        """Append instructions for `op`; returns refs of its outputs."""
        if isinstance(op, ps.Composite):
            fg = op.fgraph
            env = dict(zip(fg.inputs, arg_refs))
            dts = dict(zip(fg.inputs, arg_dtypes))

            def ref_of(v):
                if v in env:
                    return env[v], dts[v]
                if isinstance(v, Constant):
                    d = v.type.dtype
                    prog.consts.append((d, np.asarray(v.data).item()))
                    env[v] = ("c", len(prog.consts) - 1)
                    dts[v] = d
                    return env[v], d
                raise UnsupportedOp(f"Composite inner variable {v} has no value")

            for n in fg.toposort():
                refs, rdts = [], []
                for i in n.inputs:
                    r, d = ref_of(i)
                    refs.append(r)
                    rdts.append(d)
                outs = emit(n.op, refs, rdts, [o.type.dtype for o in n.outputs])
                for o, r in zip(n.outputs, outs):
                    env[o] = r
                    dts[o] = o.type.dtype
            return [ref_of(o)[0] for o in fg.outputs]
        name = type(op).__name__
        if name not in OPS:
            raise UnsupportedOp(f"scalar op {name} ({op}) has no sm_90a device expression")
        if len(out_types) != 1:
            raise UnsupportedOp(f"multi-output scalar op {name}")
        prog.insts.append(ScalarInst(name, list(arg_refs), list(arg_dtypes), out_types[0]))
        return [("t", len(prog.insts) - 1)]

    outs = emit(scalar_op, [("i", k) for k in range(len(in_dtypes))], list(in_dtypes), list(out_dtypes))
    prog.outputs = list(outs)
    return simplify(prog)


_RED_NAMES = {"Add": "add", "Mul": "mul", "Maximum": "maximum", "Minimum": "minimum", "AND": "and", "OR": "or",
              "XOR": "xor"}


def _reduce_identity(red, acc_dtype):
    dt = np.dtype(acc_dtype)
    if red == "add" or red == "or" or red == "xor":
        return 0
    if red == "mul":
        return 1
    if red == "and":
        if dt.kind == "b":
            return 1
        return int(np.iinfo(dt).max) if dt.kind == "u" else -1
    if red == "maximum":
        if dt.kind == "f":
            return float("-inf")
        return 0 if dt.kind == "b" else int(np.iinfo(dt).min)
    if red == "minimum":
        if dt.kind == "f":
            return float("inf")
        return 1 if dt.kind == "b" else int(np.iinfo(dt).max)
    raise UnsupportedOp(red)


def _idx_template(idx_list):
    out = []
    for e in idx_list:
        if isinstance(e, slice):
            out.append((e.start, e.stop, e.step))
        else:
            out.append(int(e))
    return out


def _take_axis(idx_list, ndim):
    """(first axis, k) when the index arrays sit on k consecutive axes and every other axis is taken in full
    (NumPy then leaves the broadcast index shape in place of the block); None for any other pattern."""
    int_axes = [i for i, e in enumerate(idx_list) if isinstance(e, int)]
    if not 1 <= len(int_axes) <= 8 or int_axes != list(range(int_axes[0], int_axes[0] + len(int_axes))):
        return None
    if any(e != slice(None) for i, e in enumerate(idx_list) if i not in int_axes):
        return None
    return int_axes[0], len(int_axes)


def _adv_template(idx_list, index_inputs, op):
    """(template, kinds) for vm/nodes_advidx.py: per index entry ("s", start, stop, step) with positions into the node's
    index inputs (or None), or ("a", position); kinds[position] = ("bool" | "int", ndim) for array entries."""
    tmpl, kinds = [], {}
    for e in idx_list:
        if isinstance(e, slice):
            tmpl.append(("s", e.start, e.stop, e.step))
        else:
            t = index_inputs[int(e)].type
            if t.dtype == "bool":
                if t.ndim == 0:
                    raise UnsupportedOp(f"{op}: indexing with scalar booleans")
                kinds[int(e)] = ("bool", t.ndim)
            elif t.dtype.startswith(("int", "uint")):
                kinds[int(e)] = ("int", t.ndim)
            else:
                raise UnsupportedOp(f"{op}: index of dtype {t.dtype}")
            tmpl.append(("a", int(e)))
    if not kinds:
        raise UnsupportedOp(f"{op}: advanced indexing without an index array")
    return tmpl, kinds


def lower_node(node, opts):
    """Apply -> Node.  `opts`: dict(gemm_precision=0|1)."""
    op = node.op
    prec = opts.get("gemm_precision", 0)

    if isinstance(op, Elemwise):
        in_dt = [i.type.dtype for i in node.inputs]
        out_dt = [o.type.dtype for o in node.outputs]
        try:
            prog = scalar_program(op.scalar_op, in_dt, out_dt)
            from pytensor_b200.codegen.scalar import emit_body

            emit_body(prog)  # surface unsupported dtypes/ops at compile time
        except UnsupportedScalarOp as e:
            raise UnsupportedOp(str(e)) from e
        nd = node.outputs[0].type.ndim
        bc = [tuple(i.type.broadcastable) for i in node.inputs]
        return ElemwiseNode(prog, nd, bc, dict(op.inplace_pattern), name=str(op))

    if isinstance(op, ps.ScalarOp):
        # A scalar op applied to 0-d SCALAR-typed values (the reference's shape / index arithmetic between
        # ScalarFromTensor and TensorFromScalar, e.g. maximum(shape_i, shape_j) of a broadcast; C code from
        # ScalarOp.c_code, scalar/basic.py:1411-3861): the same scalar program as a 0-d Elemwise.
        in_dt = [i.type.dtype for i in node.inputs]
        out_dt = [o.type.dtype for o in node.outputs]
        try:
            prog = scalar_program(op, in_dt, out_dt)
            from pytensor_b200.codegen.scalar import emit_body

            emit_body(prog)
        except UnsupportedScalarOp as e:
            raise UnsupportedOp(str(e)) from e
        return ElemwiseNode(prog, 0, [() for _ in node.inputs], {}, name=str(op))

    if isinstance(op, CAReduce):
        sname = type(op.scalar_op).__name__
        if sname not in _RED_NAMES:
            raise UnsupportedOp(f"CAReduce over scalar op {sname}")
        red = _RED_NAMES[sname]
        x = node.inputs[0]
        in_dt = x.type.dtype
        out_dt = node.outputs[0].type.dtype
        acc_dt = getattr(op, "acc_dtype", None) or op._acc_dtype(in_dt)
        if in_dt == "bool" and red in ("add", "mul"):
            pass
        for d in (in_dt, out_dt, acc_dt):
            if d not in ("bool", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32",
                         "float64"):
                raise UnsupportedOp(f"CAReduce dtype {d}")
        if getattr(op, "no_zeros_in_input", False):
            pass
        return CAReduceNode(red, op.axis, x.type.ndim, in_dt, acc_dt, out_dt, _reduce_identity(red, acc_dt),
                            name=str(op))

    if isinstance(op, DimShuffle):
        return nb.DimShuffleNode(op.new_order, op.input_ndim, name=str(op))

    if isinstance(op, Gemm):
        return nblas.GemmNode(node.outputs[0].type.dtype, bool(op.inplace), prec, name=str(op))
    if isinstance(op, Dot22Scalar):
        return nblas.Dot22Node(node.outputs[0].type.dtype, prec, scalar=True, name=str(op))
    if isinstance(op, Dot22):
        return nblas.Dot22Node(node.outputs[0].type.dtype, prec, name=str(op))
    if isinstance(op, Gemv):  # also CGemv (subclass, pytensor/tensor/blas/blas_c.py:59)
        return nblas.GemvNode(node.outputs[0].type.dtype, bool(op.inplace), name=str(op))
    if isinstance(op, Ger):  # also CGer
        return nblas.GerNode(node.outputs[0].type.dtype, bool(op.destructive), name=str(op))
    if isinstance(op, Dot):
        dt = node.outputs[0].type.dtype
        if dt not in ("float32", "float64") or any(i.type.dtype != dt for i in node.inputs):
            raise UnsupportedOp(f"Dot with dtypes {[i.type.dtype for i in node.inputs]}")
        return nblas.DotNode(dt, prec, name=str(op))

    if isinstance(op, Shape_i):
        return nb.ShapeINode(op.i)
    if isinstance(op, Shape):
        return nb.ShapeNode()
    if isinstance(op, MakeVector):
        return nb.MakeVectorNode(op.dtype)
    if isinstance(op, AllocEmpty):
        return nb.AllocEmptyNode(op.dtype)
    if isinstance(op, Alloc):
        return nb.AllocNode(node.outputs[0].type.dtype)
    if isinstance(op, Reshape):
        return nb.ReshapeNode(op.ndim)
    if isinstance(op, ScalarFromTensor | TensorFromScalar | ViewOp | SpecifyShape):
        return nb.ViewNode(name=str(op))
    if isinstance(op, DeepCopyOp):
        return nb.DeepCopyNode()
    if isinstance(op, CheckAndRaise):
        et = op.exc_type
        return nb.AssertNode(op.msg, getattr(et, "__qualname__", "AssertionError"), getattr(et, "__module__", "builtins"))
    if isinstance(op, Join):
        return nb.JoinNode(node.outputs[0].type.dtype, op.axis)

    if isinstance(op, Subtensor):
        return nb.SubtensorNode(_idx_template(op.idx_list), name=str(op))
    if isinstance(op, IncSubtensor):
        return nb.IncSubtensorNode(_idx_template(op.idx_list), bool(op.inplace), bool(op.set_instead_of_inc),
                                   node.outputs[0].type.dtype, name=str(op))
    if isinstance(op, AdvancedSubtensor):
        blk = _take_axis(op.idx_list, node.inputs[0].type.ndim)
        if (blk is None or len(node.inputs) != 1 + blk[1]
                or any(i.type.dtype == "bool" or i.type.dtype.startswith("float") for i in node.inputs[1:])):
            from pytensor_b200.vm.nodes_advidx import AdvIndexNode

            return AdvIndexNode(*_adv_template(op.idx_list, node.inputs[1:], op), name=str(op))
        return nb.TakeNode(blk[0], name=str(op), naxes=blk[1])
    if isinstance(op, AdvancedIncSubtensor):
        blk = _take_axis(op.idx_list, node.inputs[0].type.ndim)
        if (blk is None or len(node.inputs) != 2 + blk[1]
                or any(i.type.dtype == "bool" or i.type.dtype.startswith("float") for i in node.inputs[2:])
                or (op.ignore_duplicates and not op.set_instead_of_inc)):
            from pytensor_b200.vm.nodes_advidx import AdvIndexPutNode

            tmpl, kinds = _adv_template(op.idx_list, node.inputs[2:], op)
            return AdvIndexPutNode(tmpl, kinds, bool(op.inplace), bool(op.set_instead_of_inc), bool(op.ignore_duplicates),
                                   node.outputs[0].type.dtype, name=str(op))
        return nb.PutNode(blk[0], bool(op.inplace), bool(op.set_instead_of_inc), node.outputs[0].type.dtype,
                          name=str(op), naxes=blk[1])

    # linear algebra (possibly wrapped in Blockwise for batches)
    core = op.core_op if isinstance(op, Blockwise) else op
    cname = type(core).__name__
    if cname == "Cholesky":
        return nlin.CholeskyNode(node.outputs[0].type.dtype, bool(core.lower), name=str(op))
    if cname == "SolveTriangular":
        return nlin.SolveTriangularNode(node.outputs[0].type.dtype, bool(core.lower), bool(core.unit_diagonal),
                                        int(core.b_ndim), name=str(op))

    # more of the Op library (SURVEY.md §8(f).3)
    if cname in ("ARange", "Eye", "ExtractDiag", "Split", "Argmax", "CumOp") and not isinstance(op, Blockwise):
        from pytensor_b200.vm import nodes_extra as nx

        if cname == "ARange":
            return nx.ARangeNode(op.dtype)
        if cname == "Eye":
            return nx.EyeNode(op.dtype)
        if cname == "ExtractDiag":
            return nx.ExtractDiagNode(op.offset, op.axis1, op.axis2, op.view, name=str(op))
        if cname == "Split":
            return nx.SplitNode(op.len_splits, op.axis, name=str(op))
        x = node.inputs[0]
        if cname == "Argmax":
            if x.type.dtype not in ("bool", "int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64",
                                    "float32", "float64"):
                raise UnsupportedOp(f"Argmax of dtype {x.type.dtype}")
            return nx.ArgmaxNode(op.axis, x.type.ndim, x.type.dtype, name=str(op))
        if x.type.dtype not in nx.CumOpNode.SUPPORTED:
            raise UnsupportedOp(f"{op}: np.cumsum/cumprod widen dtype {x.type.dtype}; only "
                                f"{nx.CumOpNode.SUPPORTED} keep the declared output type")
        return nx.CumOpNode(op.axis, op.mode, x.type.dtype, name=str(op))

    from pytensor.tensor.random.op import RandomVariable

    if isinstance(op, RandomVariable):
        from pytensor_b200.vm.nodes_random import DIST, RandomVariableNode
        from pytensor.tensor.type_other import NoneTypeT

        if op.name not in DIST or op.ndim_supp != 0 or len(node.inputs) - 2 != DIST[op.name][1]:
            raise UnsupportedOp(f"{op}: random variable '{op.name}' has no device sampler (supported: {sorted(DIST)})")
        if op.dtype not in ("float32", "float64", "int64", "int32", "int16", "int8", "uint8", "bool"):
            raise UnsupportedOp(f"{op}: draws of dtype {op.dtype}")
        return RandomVariableNode(op.name, op.dtype, bool(op.inplace), isinstance(node.inputs[1].type, NoneTypeT), name=str(op))

    if cname == "BatchedDot":
        dt = node.outputs[0].type.dtype
        if dt not in ("float32", "float64"):
            raise UnsupportedOp(f"BatchedDot with dtype {dt}")
        return nblas.BatchedDotNode(dt, prec, name=str(op))

    from pytensor.compile.builders import OpFromGraph

    if isinstance(op, OpFromGraph):
        from pytensor_b200.link.cuda.linker import build_program
        from pytensor_b200.vm.nodes_inner import InnerProgramNode

        inner = op.fgraph
        program, _ = build_program(inner, list(inner.toposort()), dict(opts), storage_map=None)
        return InnerProgramNode(program, len(node.outputs), name=str(op))

    if cname == "Scan":
        from pytensor_b200.link.cuda.lower_scan import lower_scan

        return lower_scan(node, opts)

    raise UnsupportedOp(
        f"CUDALinker: op {op} ({type(op).__module__}.{type(op).__name__}) has no sm_90a implementation; "
        "the CUDA backend never falls back to the CPU"
    )
