"""Executable nodes for the Elemwise / CAReduce family (reference: pytensor/tensor/elemwise.py:375 Elemwise,
:1233 CAReduce).  Plain data + launch logic; no pytensor import, so a lowered program can be pickled and run on a box
that only has torch + libptk.
"""

from __future__ import annotations

import ctypes
import os
from ctypes import c_int, c_longlong, c_uint, c_void_p

import numpy as np

from ..codegen import careduce as cg_red
from ..codegen import elemwise as cg_ew
from ..codegen.scalar import ITEMSIZE, ScalarProgram, is_float
from ..runtime import device as dev
from ..runtime import jit
from ..runtime import lib as _lib
from .values import Val



class Node:
    """Base of all executable nodes. `run(vals) -> list[Val]`."""

    n_out = 1
    name = "node"
    destroy = {}  # out_idx -> in_idx (the output reuses that input's buffer)

    def run(self, vals):
        raise NotImplementedError

    def __repr__(self):
        return f"<{type(self).__name__} {self.name}>"

    # Nodes are plain data + caches of device handles; only the data is pickled (a lowered Program can be shipped to a
    # box that has torch + libptk but no host framework).
    _TRANSIENT = ("_kernels", "_fn", "_const_cache", "_flag", "_plans", "_occupancy")

    def __getstate__(self):
        d = dict(self.__dict__)
        for k in self._TRANSIENT:
            if k in d:
                d[k] = {} if isinstance(d[k], dict) else None
        return d


def _collapse(shape, strides_list):
    """Merge adjacent dims that are mergeable for EVERY operand. Returns (shape, strides_list)."""
    nd = len(shape)
    keep = [i for i in range(nd) if shape[i] != 1]
    if not keep:
        return [1], [[0] for _ in strides_list]
    shp = [shape[keep[0]]]
    sts = [[st[keep[0]]] for st in strides_list]
    for i in keep[1:]:
        ok = all(st_acc[-1] == st[i] * shape[i] for st_acc, st in zip(sts, strides_list))
        if ok:
            shp[-1] *= shape[i]
            for st_acc, st in zip(sts, strides_list):
                st_acc[-1] = st[i]
        else:
            shp.append(shape[i])
            for st_acc, st in zip(sts, strides_list):
                st_acc.append(st[i])
    return shp, sts


def _dense_order(t):
    """Permutation (slowest dim first) if `t` is a dense permuted buffer, else None."""
    nd = t.dim()
    if nd <= 1:
        return None
    order = sorted(range(nd), key=lambda i: (-t.stride(i), i))
    expect = 1
    for i in reversed(order):
        if t.shape[i] != 1 and t.stride(i) != expect:
            return None
        expect *= t.shape[i]
    return order


def host_eval_program(prog: ScalarProgram, inputs):
    """Evaluate an integer/bool ScalarProgram on host arrays (shape arithmetic only — see vm/values.py)."""
    def ref(r):
        k, i = r
        if k == "i":
            return inputs[i]
        if k == "c":
            d, v = prog.consts[i]
            return np.asarray(v, dtype=d)
        return tmp[i]

    def c_differs_from_numpy(a):
        """NumPy promotes a signed/unsigned pair to a wider signed type (or float64); the C expressions the reference
        generates — and the device kernels, which compile the same expressions — convert the signed operand to the unsigned
        type when that is at least as wide (and at least `int`): int32(-1) * uint32(3) is 4294967293 there.  Such programs
        are left to the device path (they never occur in shape arithmetic, which is all int64)."""
        kinds = [x.dtype for x in a if x.dtype.kind in "iu"]
        signed = [d.itemsize for d in kinds if d.kind == "i"]
        unsigned = [d.itemsize for d in kinds if d.kind == "u"]
        return any(u >= 4 and u >= s_ for u in unsigned for s_ in signed)

    tmp = []
    for inst in prog.insts:
        a = [np.asarray(ref(r)) for r in inst.args]
        op, od = inst.op, inst.out_dtype
        if len(a) > 1 and c_differs_from_numpy(a if op != "Switch" else a[1:]):
            return None
        if op == "Add":
            r = a[0]
            for x in a[1:]:
                r = r + x
        elif op == "Mul":
            r = a[0]
            for x in a[1:]:
                r = r * x
        elif op == "Sub":
            r = a[0] - a[1]
        elif op == "Neg":
            r = -a[0]
        elif op == "Abs":
            r = np.abs(a[0])
        elif op in ("IntDiv", "Mod"):
            if not is_float(od) and np.any(a[1] == 0):
                # the reference's C code fails the thunk (scalar/basic.py:2058-2066 for IntDiv, the Mod twin below it)
                raise ZeroDivisionError("integer division by zero" if op == "IntDiv" else "integer modulo by zero")
            r = np.floor_divide(a[0], a[1]) if op == "IntDiv" else np.mod(a[0], a[1])
        elif op == "Maximum":
            r = np.maximum(a[0], a[1])
        elif op == "Minimum":
            r = np.minimum(a[0], a[1])
        elif op in ("Cast", "Identity"):
            r = a[0]
        elif op == "Second":
            r = np.broadcast_to(a[1], np.broadcast(a[0], a[1]).shape)
        elif op == "Switch":
            r = np.where(a[0], a[1], a[2])
        elif op == "Sqr":
            r = a[0] * a[0]
        elif op == "Sign":
            r = np.sign(a[0])
        elif op in ("LT", "GT", "LE", "GE", "EQ", "NEQ"):
            r = {"LT": np.less, "GT": np.greater, "LE": np.less_equal, "GE": np.greater_equal, "EQ": np.equal,
                 "NEQ": np.not_equal}[op](a[0], a[1])
        elif op in ("AND", "OR", "XOR"):
            r = {"AND": np.bitwise_and, "OR": np.bitwise_or, "XOR": np.bitwise_xor}[op](a[0], a[1])
        elif op == "Invert":
            r = np.invert(a[0])
        elif op == "TrueDiv" and is_float(od):
            r = np.true_divide(a[0], a[1])
        elif op in ("Ceil", "Floor", "Trunc", "RoundHalfToEven"):
            r = {"Ceil": np.ceil, "Floor": np.floor, "Trunc": np.trunc, "RoundHalfToEven": np.rint}[op](a[0])
        else:
            return None
        tmp.append(np.asarray(r).astype(od))
    return [np.asarray(ref(r)).astype(d) for r, d in zip(prog.outputs, prog.out_dtypes)]


class ElemwiseNode(Node):
    """One fused elementwise kernel: n_in broadcast operands -> n_out results (Elemwise with a Composite or a
    single ScalarOp; pytensor/tensor/elemwise.py:375).  `in_bcast[k][d]` is the STATIC broadcast pattern: a runtime
    length-1 dim that is not typed broadcastable is an error (elemwise.py:825-840)."""

    HOST_MAX = 64

    def __init__(self, prog: ScalarProgram, ndim: int, in_bcast, inplace: dict, name="Elemwise"):
        self.prog = prog
        self.ndim = ndim
        self.in_bcast = [tuple(b) for b in in_bcast]
        self.inplace = dict(inplace)
        self.destroy = dict(inplace)
        self.n_in = len(prog.in_dtypes)
        self.n_out = len(prog.out_dtypes)
        self.name = name
        self._kernels = {}
        self._plans = {}
        self._host_ok = all((not is_float(d)) for d in list(prog.in_dtypes) + list(prog.out_dtypes))

    # -- shape logic -------------------------------------------------------------------------------------------------
    def _out_shape(self, shapes):
        out = []
        for d in range(self.ndim):
            s = None
            for k, shp in enumerate(shapes):
                if self.in_bcast[k][d]:
                    if shp[d] != 1:
                        raise ValueError(f"{self.name}: input {k} is typed broadcastable in dim {d} but has length {shp[d]}")
                    continue
                if s is None:
                    s = shp[d]
                elif shp[d] != s:
                    raise ValueError(
                        f"{self.name}: input dimension mismatch in dim {d}: {s} vs {shp[d]} (input {k}); "
                        "runtime broadcasting of a non-broadcastable dim is not allowed"
                    )
            out.append(1 if s is None else int(s))
        return out

    def run(self, vals):
        if self._host_ok and all(v.d is None for v in vals):
            shapes = [v.shape for v in vals]
            oshape = self._out_shape(shapes)
            if int(np.prod(oshape, dtype=np.int64)) <= self.HOST_MAX:
                res = host_eval_program(self.prog, [np.asarray(v.h) for v in vals])
                if res is not None:
                    return [Val(h=np.broadcast_to(r, oshape).copy() if tuple(np.shape(r)) != tuple(oshape) else r)
                            for r in res]
        if any(v.d is None for v in vals):
            self._out_shape([v.shape for v in vals])  # shape errors surface before any host->device transfer
        ins = [v.dev() for v in vals]
        # launch-plan cache: same operand layouts (shape, strides, 16-byte alignment class) => same kernel, grid and
        # argument block; only the pointers change.  Keeps the eager per-node host cost at allocation + one ctypes call.
        pkey = tuple((tuple(t.shape), t.stride(), t.data_ptr() & 31) for t in ins)
        plan = self._plans.get(pkey)
        if plan is None:
            oshape = self._out_shape([tuple(t.shape) for t in ins])  # raises on runtime broadcasting
            order = None
            for k, t in enumerate(ins):
                if tuple(t.shape) == tuple(oshape) and not any(self.in_bcast[k]):
                    order = _dense_order(t)
                    break
            total = 1
            for s_ in oshape:
                total *= s_
            plan = [oshape, order, total, None]
            if len(self._plans) > 64:
                self._plans.clear()
            self._plans[pkey] = plan
        oshape, order, total, launch = plan
        outs = []
        for k, dt in enumerate(self.prog.out_dtypes):
            if k in self.inplace:
                outs.append(ins[self.inplace[k]])
            else:
                outs.append(dev.empty_like_layout(oshape, dt, order))
        if total == 0:
            return [Val(d=o) for o in outs]
        if launch is None or (outs and (outs[0].data_ptr() & 31)):
            launch = self._plan_launch(ins, outs, oshape)
            plan[3] = launch
            fn, grid, kargs, nptr = launch
        else:
            fn, grid, kargs, nptr = launch
            ptrs = kargs._vals
            for j, t in enumerate(ins):
                ptrs[j].value = t.data_ptr()
            for j, t in enumerate(outs):
                ptrs[len(ins) + j].value = t.data_ptr()
        jit.launch(fn, (grid,), (256,), kargs, 0, dev.stream_ptr())
        return [Val(d=o) for o in outs]

    # -- launch --------------------------------------------------------------------------------------------------------
    def _plan_launch(self, ins, outs, oshape):
        """Kernel selection + argument block for these operand layouts: (fn, grid, KernelArgs, n_pointer_slots)."""
        nd = self.ndim
        ops = ins + outs
        strides = []
        for k, t in enumerate(ins):
            strides.append([0 if (self.in_bcast[k][d] or t.shape[d] == 1 and oshape[d] != 1) else t.stride(d)
                            for d in range(nd)])
        for t in outs:
            strides.append([t.stride(d) for d in range(nd)])
        # iterate in the memory order of the first output
        perm = sorted(range(nd), key=lambda i: (-outs[0].stride(i), i)) if nd > 1 else list(range(nd))
        shp = [oshape[i] for i in perm]
        sts = [[st[i] for i in perm] for st in strides]
        cshape, csts = _collapse(shp, sts)
        stream = dev.stream_ptr()
        total = 1
        for s in cshape:
            total *= s
        dtypes = list(self.prog.in_dtypes) + list(self.prog.out_dtypes)
        vw = cg_ew.vec_width(dtypes)
        if len(cshape) <= 2 and self._vec_ok(ops, dtypes, cshape, csts, vw):
            rows = cshape[0] if len(cshape) == 2 else 1
            cols = cshape[-1]
            col_modes = tuple(1 if st[-1] == 1 else 0 for st in csts)
            flat = rows == 1
            key = ("vec", col_modes, vw, flat)
            fn = self._kernels.get(key)
            if fn is None:
                fn, _ = jit.get_function_gen(
                    lambda kn: cg_ew.gen_vec_kernel(self.prog, kn, col_modes, self.inplace, vw, flat=flat),
                    "ptk_ew_vec")
                self._kernels[key] = fn
            cpr_chunks = cols // vw
            nchunks = rows * cpr_chunks
            tail_start = cpr_chunks * vw if rows == 1 else cols
            n_total = cols if rows == 1 else cols  # tail loop is a no-op for rows > 1 (cols % vw == 0 enforced)
            args = [c_void_p(dev.ptr(t)) for t in ops]
            args += [c_longlong(st[0] if len(cshape) == 2 else 0) for st in csts]
            args += [c_longlong(nchunks), c_uint(cpr_chunks if rows > 1 else 0), c_longlong(tail_start),
                     c_longlong(n_total)]
            per_block = 256 * cg_ew.VEC_UNROLL
            want = max(1, (max(nchunks, n_total - tail_start) + per_block - 1) // per_block)
            grid = min(want, _lib.sm_count() * 8)
            return fn, grid, jit.KernelArgs(args), len(ops)
        if len(cshape) > cg_ew.MAX_DIMS:
            raise NotImplementedError(f"{self.name}: more than {cg_ew.MAX_DIMS} non-collapsible dims")
        key = ("gen",)
        fn = self._kernels.get(key)
        nops = len(ops)
        if fn is None:
            if nops > 48:
                raise NotImplementedError(f"{self.name}: {nops} strided operands exceed the by-value descriptor")
            fn, _ = jit.get_function_gen(lambda kn: cg_ew.gen_generic_kernel(self.prog, kn, self.inplace), "ptk_ew_gen")
            self._kernels[key] = fn

        class EwDims(ctypes.Structure):
            _fields_ = [("ndim", c_int), ("shape", c_longlong * cg_ew.MAX_DIMS),
                        ("st", (c_longlong * cg_ew.MAX_DIMS) * nops)]

        d = EwDims()
        d.ndim = len(cshape)
        for i, s in enumerate(cshape):
            d.shape[i] = s
        for j, st in enumerate(csts):
            for i, s in enumerate(st):
                d.st[j][i] = s
        args = [c_void_p(dev.ptr(t)) for t in ops] + [d, c_longlong(total)]
        grid = min(max(1, (total + 255) // 256), _lib.sm_count() * 16)
        return fn, grid, jit.KernelArgs(args), len(ops)

    @staticmethod
    def _vec_ok(ops, dtypes, cshape, csts, vw):
        two_d = len(cshape) == 2
        cols = cshape[-1]
        if two_d and cols % vw != 0:
            return False
        for t, dt, st in zip(ops, dtypes, csts):
            inner = st[-1]
            if inner not in (0, 1):
                return False
            if inner == 1:
                if dev.ptr(t) % (ITEMSIZE[dt] * vw) != 0:
                    return False
                if two_d and st[0] % vw != 0:
                    return False
        if not two_d and cols < vw:
            return True  # pure tail loop
        return True


# ---------------------------------------------------------------------------------------------------------------------
class CAReduceNode(Node):
    """Reduction over `axes` with a commutative-associative scalar op (pytensor/tensor/elemwise.py:1233).
    acc_dtype / out_dtype follow `_acc_dtype` / `_output_dtype` (:1352-1417)."""

    def __init__(self, red_op: str, axes, ndim: int, in_dtype: str, acc_dtype: str, out_dtype: str, identity,
                 name="CAReduce"):
        self.red_op = red_op
        self.axes = tuple(sorted(range(ndim) if axes is None else [a % ndim for a in axes])) if ndim else ()
        self.ndim = ndim
        self.in_dtype = in_dtype
        self.acc_dtype = acc_dtype
        self.out_dtype = out_dtype
        self.identity = identity
        self.name = name
        self._kernels = {}

    def _fn(self, key, gen):
        fn = self._kernels.get(key)
        if fn is None:
            fn, _ = jit.get_function_gen(gen, "ptk_red_" + key[0])
            self._kernels[key] = fn
        return fn

    def _fill_identity(self, out):
        src = dev.to_device(np.asarray(self.identity, dtype=self.out_dtype).reshape(()))
        dev.copy_strided(out, src.as_strided(tuple(out.shape), (0,) * out.dim()))

    HOST_MAX = 64
    _HOST_RED = {"add": np.add, "mul": np.multiply, "maximum": np.maximum, "minimum": np.minimum, "and": np.bitwise_and,
                 "or": np.bitwise_or, "xor": np.bitwise_xor}

    def _run_host(self, x):
        """Integer / bool reduction of a small HOST value (shape plumbing: `All(MakeVector(eq(shape_i, shape_j), ...))` in
        front of the reference's "could not broadcast" Assert): NumPy in the declared accumulator / output types, so that
        the check never leaves the host — no upload, no device round trip for the Assert, and the program stays
        capturable into a CUDA graph."""
        x = np.asarray(x)
        kept = [i for i in range(self.ndim) if i not in self.axes]
        if not self.axes:
            return x.astype(self.out_dtype)
        if x.size == 0 or any(x.shape[a] == 0 for a in self.axes):
            return np.full([x.shape[i] for i in kept], self.identity, dtype=self.out_dtype)
        return np.asarray(self._HOST_RED[self.red_op].reduce(x.astype(self.acc_dtype), axis=self.axes)).astype(self.out_dtype)

    def run(self, vals):
        v = vals[0]
        if (v.d is None and v.h is not None and np.size(v.h) <= self.HOST_MAX and self.red_op in self._HOST_RED
                and not any(is_float(d) for d in (self.in_dtype, self.acc_dtype, self.out_dtype))):
            return [Val(h=self._run_host(v.h))]
        t = vals[0].dev()
        shape = tuple(t.shape)
        kept = [i for i in range(self.ndim) if i not in self.axes]
        oshape = [shape[i] for i in kept]
        out = dev.empty(oshape, self.out_dtype)
        n_out = 1
        for s in oshape:
            n_out *= s
        n_red = 1
        for a in self.axes:
            n_red *= shape[a]
        if n_out == 0:
            return [Val(d=out)]
        if n_red == 0:
            self._fill_identity(out)
            return [Val(d=out)]
        if not self.axes:  # nothing to reduce: a dtype-casting copy
            self._generic(t, out, kept, n_out, 1)
            return [Val(d=out)]
        tc = dev.contiguous(t)
        # group dims of the contiguous input into alternating kept / reduced runs
        groups = []  # (is_red, size)
        for i in range(self.ndim):
            if shape[i] == 1:
                continue
            r = i in self.axes
            if groups and groups[-1][0] == r:
                groups[-1] = (r, groups[-1][1] * shape[i])
            else:
                groups.append((r, shape[i]))
        pattern = tuple(g[0] for g in groups)
        sizes = [g[1] for g in groups]
        if pattern in ((True,), ()):
            self._row(tc, out, 1, n_red)
        elif pattern == (False, True):
            self._row(tc, out, sizes[0], sizes[1])
        elif pattern == (True, False):
            self._col(tc, out, 1, sizes[0], sizes[1])
        elif pattern == (False, True, False):
            self._col(tc, out, sizes[0], sizes[1], sizes[2])
        elif pattern == (False,):
            self._generic(t, out, kept, n_out, 1)
        else:
            self._generic(t, out, kept, n_out, n_red)
        return [Val(d=out)]

    # -- kernels -------------------------------------------------------------------------------------------------------
    def _row(self, tc, out, rows, cols):
        stream = dev.stream_ptr()
        sms = _lib.sm_count()
        isz = ITEMSIZE[self.in_dtype]
        vw = 4 if isz >= 4 else (8 if isz == 2 else 16)
        if dev.ptr(tc) % (isz * vw) != 0 or (rows > 1 and cols % vw != 0):
            vw = 1
        tpr = 256 if cols >= 2048 else 32
        rows_per_block = 256 // tpr
        row_blocks = (rows + rows_per_block - 1) // rows_per_block
        nsplit = 1
        ncv = cols // vw
        if row_blocks < sms * 2 and ncv >= tpr * 16:
            nsplit = int(min((sms * 4 + row_blocks - 1) // row_blocks, max(1, ncv // (tpr * 8)), 1024))
        prog = cg_red.identity_program(self.in_dtype)
        key = ("row", vw, tpr)
        fn = self._fn(key, lambda kn: cg_red.gen_row_kernel(prog, kn, (1,), (False,), self.red_op, self.acc_dtype,
                                                              self.out_dtype, self.identity, vw, tpr))
        gx = min(row_blocks, sms * 32)
        if nsplit == 1:
            args = [c_void_p(dev.ptr(tc)), c_void_p(dev.ptr(out)), c_longlong(cols), c_longlong(rows),
                    c_longlong(cols), c_int(1)]
            jit.launch(fn, (gx, 1), (256,), jit.KernelArgs(args), 0, stream)
            return
        part = dev.empty((rows, nsplit), self.acc_dtype)
        args = [c_void_p(dev.ptr(tc)), c_void_p(dev.ptr(part)), c_longlong(cols), c_longlong(rows), c_longlong(cols),
                c_int(nsplit)]
        jit.launch(fn, (gx, nsplit), (256,), jit.KernelArgs(args), 0, stream)
        self._finish(part, out, rows, nsplit, nsplit, 1)

    def _finish(self, part, out, n_out, nsplit, stride_o, stride_s):
        fn = self._fn(("finish",), lambda kn: cg_red.gen_finish_kernel(kn, self.red_op, self.acc_dtype,
                                                                        self.out_dtype, self.identity))
        args = [c_void_p(dev.ptr(part)), c_void_p(dev.ptr(out)), c_longlong(n_out), c_int(nsplit),
                c_longlong(stride_o), c_longlong(stride_s)]
        grid = min(max(1, (n_out + 7) // 8), _lib.sm_count() * 16)
        jit.launch(fn, (grid,), (256,), jit.KernelArgs(args), 0, dev.stream_ptr())

    def _col(self, tc, out, outer, red, inner):
        stream = dev.stream_ptr()
        sms = _lib.sm_count()
        fn = self._fn(("col",), lambda kn: cg_red.gen_col_kernel(kn, self.in_dtype, self.red_op, self.acc_dtype,
                                                                  self.out_dtype, self.identity))
        gx = (inner + 255) // 256
        gy = min(outer, 65535)
        nsplit = 1
        if gx * gy < sms * 2 and red >= 64:
            nsplit = int(min((sms * 4 + gx * gy - 1) // (gx * gy), red // 16, 65535))
            nsplit = max(nsplit, 1)
        if nsplit == 1:
            args = [c_void_p(dev.ptr(tc)), c_void_p(dev.ptr(out)), c_longlong(outer), c_longlong(red),
                    c_longlong(inner), c_int(1)]
            jit.launch(fn, (gx, gy, 1), (256,), jit.KernelArgs(args), 0, stream)
            return
        part = dev.empty((nsplit, outer, inner), self.acc_dtype)
        args = [c_void_p(dev.ptr(tc)), c_void_p(dev.ptr(part)), c_longlong(outer), c_longlong(red), c_longlong(inner),
                c_int(nsplit)]
        jit.launch(fn, (gx, gy, nsplit), (256,), jit.KernelArgs(args), 0, stream)
        self._finish(part, out, outer * inner, nsplit, 1, outer * inner)

    def _generic(self, t, out, kept, n_out, n_red):
        MAXD = cg_ew.MAX_DIMS

        class RdDims(ctypes.Structure):
            _fields_ = [("nk", c_int), ("nr", c_int), ("kshape", c_longlong * MAXD), ("kst", c_longlong * MAXD),
                        ("rshape", c_longlong * MAXD), ("rst", c_longlong * MAXD)]

        red_axes = [a for a in self.axes]
        if len(kept) > MAXD or len(red_axes) > MAXD:
            raise NotImplementedError("CAReduce over more than 8 kept or reduced dims")
        d = RdDims()
        d.nk, d.nr = len(kept), len(red_axes)
        for i, a in enumerate(kept):
            d.kshape[i], d.kst[i] = t.shape[a], t.stride(a)
        for i, a in enumerate(red_axes):
            d.rshape[i], d.rst[i] = t.shape[a], t.stride(a)
        fn = self._fn(("generic",), lambda kn: cg_red.gen_generic_kernel(kn, self.in_dtype, self.red_op,
                                                                          self.acc_dtype, self.out_dtype,
                                                                          self.identity))
        args = [c_void_p(dev.ptr(t)), c_void_p(dev.ptr(out)), d, c_longlong(n_out), c_longlong(n_red)]
        grid = min(max(1, (n_out + 255) // 256), _lib.sm_count() * 16)
        jit.launch(fn, (grid,), (256,), jit.KernelArgs(args), 0, dev.stream_ptr())


# ---------------------------------------------------------------------------------------------------------------------
class ElemwiseReduceNode(Node):
    """K3: Elemwise(Composite) whose output feeds a CAReduce over its trailing axes, as ONE kernel — the map result
    stays in registers for the reduction and is written to memory only if something else needs it.

    The reference cannot fuse a multi-input Elemwise into a CAReduce (pytensor/tensor/rewriting/elemwise.py:1119-1121),
    so its C linker materialises the elementwise result and re-reads it.  Outputs of this node: the Elemwise outputs
    (in the Elemwise's order) followed by the reduction result.  Falls back to running the two constituent nodes
    back-to-back (still on the device) whenever the runtime layout does not fit the fused row kernel.
    """

    def __init__(self, ew: ElemwiseNode, red: CAReduceNode, which: int, store_reduced_input: bool):
        self.ew, self.red, self.which = ew, red, which
        self.store_reduced_input = store_reduced_input
        self.n_out = ew.n_out + 1
        self.destroy = dict(ew.destroy)
        self.name = f"{ew.name}->{red.name}[fused]"
        # program with the reduced output first (the row kernel accumulates map output 0)
        p = ew.prog
        order = [which] + [k for k in range(ew.n_out) if k != which]
        self.order = order
        self.prog = ScalarProgram(list(p.in_dtypes), [p.out_dtypes[k] for k in order], list(p.consts), list(p.insts),
                                  [p.outputs[k] for k in order])
        self._kernels = {}
        self._occupancy = {}

    def _unfused(self, vals):
        outs = self.ew.run(vals)
        return outs + self.red.run([outs[self.which]])

    def run(self, vals):
        ew, red = self.ew, self.red
        nd = ew.ndim
        n_red = len(red.axes)
        if nd == 0 or n_red == 0 or tuple(red.axes) != tuple(range(nd - n_red, nd)):
            return self._unfused(vals)
        oshape = ew._out_shape([v.shape for v in vals])
        rows = 1
        for s in oshape[: nd - n_red]:
            rows *= s
        cols = 1
        for s in oshape[nd - n_red:]:
            cols *= s
        if rows == 0 or cols == 0:
            return self._unfused(vals)
        ins = [v.dev() for v in vals]
        # the reduced map output is never materialised unless something else reads it: no buffer for it (ADVICE r1)
        skip = None if self.store_reduced_input else self.which
        cstr = []  # C-contiguous strides of `oshape` (layout of every freshly allocated output)
        acc = 1
        for s_ in reversed(oshape):
            cstr.insert(0, acc)
            acc *= s_
        outs = []
        for k, dt in enumerate(ew.prog.out_dtypes):
            if k == skip and k not in ew.inplace:
                outs.append(None)
            else:
                outs.append(ins[ew.inplace[k]] if k in ew.inplace else dev.empty(oshape, dt))
        # collapse kept dims -> rows and reduced dims -> cols for every operand
        ops = ins + outs
        strides = []
        for k, t in enumerate(ins):
            strides.append([0 if (ew.in_bcast[k][d] or (t.shape[d] == 1 and oshape[d] != 1)) else t.stride(d)
                            for d in range(nd)])
        for t in outs:
            strides.append(list(cstr) if t is None else [t.stride(d) for d in range(nd)])
        kshape, ksts = _collapse(oshape[: nd - n_red], [st[: nd - n_red] for st in strides])
        cshape, csts = _collapse(oshape[nd - n_red:], [st[nd - n_red:] for st in strides])
        if len(kshape) != 1 or len(cshape) != 1:
            return self._unfused_given(vals, ins, outs)
        dtypes = list(ew.prog.in_dtypes) + list(ew.prog.out_dtypes)
        vw = cg_ew.vec_width(dtypes)
        col_modes = []
        for t, dt, cst, kst in zip(ops, dtypes, csts, ksts):
            inner = cst[0]
            if inner not in (0, 1):
                return self._unfused_given(vals, ins, outs)
            if t is not None and inner == 1 and (dev.ptr(t) % (ITEMSIZE[dt] * vw) != 0 or kst[0] % vw != 0):
                vw = 1
            col_modes.append(inner)
        if any(m != 1 for m in col_modes[len(ins):]):
            return self._unfused_given(vals, ins, outs)
        sms = _lib.sm_count()
        if cols >= (1 << 31):
            return self._unfused_given(vals, ins, outs)   # the fused kernel walks a row with 32-bit vector indices
        # threads per row: more elements per thread amortise the per-row reduction (shuffles, shared memory, barriers)
        # — 128 when that still leaves at least 4 row blocks per SM, the full CTA for long rows of short matrices
        tpr = 32 if cols < 1024 else (128 if (cols < 16384 and rows >= sms * 8) else 256)
        if os.environ.get("PTK_K3_TPR"):   # developer A/B switch
            tpr = int(os.environ["PTK_K3_TPR"])
        rows_per_block = 256 // tpr
        row_blocks = (rows + rows_per_block - 1) // rows_per_block
        if row_blocks < sms:  # too few rows to fill the GPU with one CTA-row mapping: keep the two-kernel path
            return self._unfused_given(vals, ins, outs)
        store = tuple((k != 0 or self.store_reduced_input) for k in range(ew.n_out))  # in self.order numbering
        in_modes = tuple(col_modes[: len(ins)])
        # TMA staging (cp.async.bulk through shared memory) needs 16-byte vectors on every streamed input and a staging
        # ring that fits the static shared memory
        tma = (cg_red._k3_pipeline() == "tma" and tpr >= 64
               and all(vw * ITEMSIZE[dt] == 16 for dt, m in zip(ew.prog.in_dtypes, in_modes) if m == 1)
               and cg_red.tma_smem_bytes(in_modes.count(1)) <= cg_red.STATIC_SMEM_LIMIT)
        key = (in_modes, vw, tpr, store, tma)
        fn = self._kernels.get(key)
        if fn is None:
            gen = cg_red.gen_row_kernel_tma if tma else cg_red.gen_row_kernel
            fn, _ = jit.get_function_gen(
                lambda kn: gen(self.prog, kn, in_modes, store, red.red_op, red.acc_dtype,
                               red.out_dtype, red.identity, vw, tpr, inplace=ew.inplace),
                "ptk_ew_red_row")
            self._kernels[key] = fn
        rout = dev.empty(oshape[: nd - n_red], red.out_dtype)
        stored = [k for k in range(ew.n_out) if store[k]]
        args = [c_void_p(dev.ptr(t)) for t in ins]
        args += [c_void_p(dev.ptr(outs[self.order[k]])) for k in stored]
        args += [c_void_p(dev.ptr(rout))]
        args += [c_longlong(ksts[j][0]) for j in range(len(ins))]
        args += [c_longlong(ksts[len(ins) + self.order[k]][0]) for k in stored]
        args += [c_longlong(rows), c_longlong(cols), c_int(1)]
        # persistent CTAs: exactly as many as are resident at once, each striding over the row blocks — the prologue is
        # paid once per CTA, and with the blocks dealt round-robin every SM ends up within one row block of the average
        if getattr(self, "_occupancy", None) is None:   # (unpickled programs)
            self._occupancy = {}
        occ = self._occupancy.get(key)
        if occ is None:
            nb = ctypes.c_int(0)
            if _lib.TRACE_ONLY:
                nb.value = 4
            else:
                _lib.check(_lib.lib().ptk_func_max_active_blocks(fn, 256, 0, ctypes.byref(nb)), "occupancy")
            occ = self._occupancy[key] = max(1, nb.value)
        gx = min(row_blocks, sms * occ)
        jit.launch(fn, (gx, 1), (256,), jit.KernelArgs(args), 0, dev.stream_ptr())
        res = [Val(d=o) if o is not None else None for o in outs]
        if not self.store_reduced_input:
            res[self.which] = None  # never materialised: the fusion pass guarantees nothing reads it
        return res + [Val(d=rout)]

    def _unfused_given(self, vals, ins, outs):
        del ins, outs
        return self._unfused(vals)
