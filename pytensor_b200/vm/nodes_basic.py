"""Glue nodes: views, shape plumbing, allocation, copies, basic and advanced indexing (SURVEY.md §8a rows G1-G4).

Views (DimShuffle, Subtensor, Reshape of a contiguous buffer) are metadata only — no kernel, exactly like the
reference (`DimShuffle` is pure stride arithmetic, pytensor/tensor/elemwise.py:186-256).  Every byte that moves does
so in a libptk kernel (ptk_copy_strided / ptk_inc_strided / ptk_take / ptk_put), which keeps gather/slicing
bit-exact by construction.
"""

from __future__ import annotations

import ctypes

import numpy as np
import torch

from ..runtime import device as dev
from ..runtime import lib as _lib
from .nodes_elemwise import Node
from .values import Val


def _host_int(v: Val) -> int:
    return int(np.asarray(v.host()).reshape(-1)[0]) if np.ndim(v.host()) else int(v.host())


class DimShuffleNode(Node):
    """Reference: DimShuffle, pytensor/tensor/elemwise.py:41 (view_map {0:[0]} :115; dropped dims must be 1 :195-203)."""

    def __init__(self, new_order, input_ndim, name="DimShuffle"):
        self.new_order = tuple(new_order)
        self.input_ndim = input_ndim
        self.drop = [i for i in range(input_ndim) if i not in self.new_order]
        self.name = name

    def run(self, vals):
        v = vals[0]
        shape = v.shape
        for i in self.drop:
            if shape[i] != 1:
                raise ValueError(f"{self.name}: cannot drop dim {i} of length {shape[i]} (must be 1)")
        out = Val()
        if v.d is not None:
            t = v.d
            oshape, ostride = [], []
            for o in self.new_order:
                if o == "x":
                    oshape.append(1)
                    ostride.append(1)
                else:
                    oshape.append(t.shape[o])
                    ostride.append(t.stride(o))
            out.d = t.as_strided(oshape, ostride, t.storage_offset())
        if v.h is not None:
            h = np.asarray(v.h)
            perm = [o for o in self.new_order if o != "x"]
            hh = h.transpose(perm + self.drop).reshape([h.shape[p] for p in perm]) if h.ndim else h
            oshape = [1 if o == "x" else h.shape[o] for o in self.new_order]
            out.h = hh.reshape(oshape)
        return [out]


class ViewNode(Node):
    """Identity-like ops whose output is the input value (ViewOp, SpecifyShape, ScalarFromTensor, TensorFromScalar,
    Rebroadcast...)."""

    def __init__(self, name="View"):
        self.name = name

    def run(self, vals):
        v = vals[0]
        return [Val(h=v.h, d=v.d)]


class DeepCopyNode(Node):
    """Reference: DeepCopyOp, pytensor/compile/ops.py:121."""

    name = "DeepCopyOp"

    def run(self, vals):
        v = vals[0]
        if v.d is not None:
            return [Val(d=dev.clone(v.d))]
        return [Val(h=np.array(v.h, copy=True))]


class ShapeINode(Node):
    """Reference: Shape_i, pytensor/tensor/shape.py:201 — host-side int64 scalar, never a device value."""

    def __init__(self, i):
        self.i = i
        self.name = f"Shape_i{{{i}}}"

    def run(self, vals):
        return [Val(h=np.asarray(vals[0].shape[self.i], dtype="int64"))]


class ShapeNode(Node):
    name = "Shape"

    def run(self, vals):
        return [Val(h=np.asarray(vals[0].shape, dtype="int64"))]


class MakeVectorNode(Node):
    """Reference: MakeVector, pytensor/tensor/basic.py:1900."""

    def __init__(self, dtype):
        self.dtype = dtype
        self.name = "MakeVector"

    def run(self, vals):
        return [Val(h=np.asarray([np.asarray(v.host()).reshape(()) for v in vals], dtype=self.dtype).reshape(len(vals)))]


class AllocEmptyNode(Node):
    """Reference: AllocEmpty, pytensor/tensor/basic.py:4197 — contents undefined."""

    def __init__(self, dtype):
        self.dtype = dtype
        self.name = "AllocEmpty"

    def run(self, vals):
        shape = [_host_int(v) for v in vals]
        return [Val(d=dev.empty(shape, self.dtype))]


def _broadcast_view(t: torch.Tensor, shape) -> torch.Tensor:
    """View of `t` broadcast (0 strides) to `shape`, left-padding dims like NumPy."""
    nd = len(shape)
    pad = nd - t.dim()
    if pad < 0:
        raise ValueError("cannot broadcast to fewer dims")
    strides = []
    for i in range(nd):
        if i < pad:
            strides.append(0)
        else:
            ts = t.shape[i - pad]
            if ts == shape[i]:
                strides.append(t.stride(i - pad))
            elif ts == 1:
                strides.append(0)
            else:
                raise ValueError(f"cannot broadcast shape {tuple(t.shape)} to {tuple(shape)}")
    return t.as_strided(tuple(shape), tuple(strides), t.storage_offset())


class AllocNode(Node):
    """Reference: Alloc, pytensor/tensor/basic.py:1545 — value broadcast into a fresh buffer."""

    def __init__(self, dtype):
        self.dtype = dtype
        self.name = "Alloc"

    def run(self, vals):
        val = vals[0].dev()
        shape = [_host_int(v) for v in vals[1:]]
        out = dev.empty(shape, self.dtype)
        if out.numel():
            dev.copy_strided(out, _broadcast_view(val, shape))
        return [Val(d=out)]


class ReshapeNode(Node):
    """Reference: Reshape, pytensor/tensor/shape.py:613 (view of a contiguous buffer, copy otherwise)."""

    def __init__(self, ndim):
        self.ndim = ndim
        self.name = "Reshape"

    def run(self, vals):
        v = vals[0]
        shp = [int(s) for s in np.asarray(vals[1].host()).reshape(-1)]
        total = v.size
        if -1 in shp:
            known = 1
            for s in shp:
                if s != -1:
                    known *= s
            shp[shp.index(-1)] = total // known if known else 0
        n = 1
        for s in shp:
            n *= s
        if n != total:
            raise ValueError(f"Reshape: cannot reshape array of size {total} into shape {tuple(shp)}")
        if v.d is None:
            return [Val(h=np.asarray(v.h).reshape(shp))]
        t = dev.contiguous(v.d)
        return [Val(d=t.view(shp))]


# ---- basic indexing ---------------------------------------------------------------------------------------------------
def _build_index(idx_template, index_vals):
    """idx_template entries: int position | (start, stop, step) of None/int positions -> python index tuple."""
    def get(p):
        return None if p is None else _host_int(index_vals[p])

    out = []
    for e in idx_template:
        if isinstance(e, tuple):
            out.append(slice(get(e[0]), get(e[1]), get(e[2])))
        else:
            out.append(get(e))
    return tuple(out)


def _probe(shape, strides, index):
    """NumPy-exact basic indexing on metadata only: returns (shape, strides, element offset) of x[index]."""
    base = np.empty(1, dtype=np.int8)
    index = tuple(index) + (Ellipsis,)  # keeps an all-integer index a 0-d VIEW (a NumPy scalar would be a copy)
    if any(s == 0 for s in shape):
        v = np.lib.stride_tricks.as_strided(base, shape=tuple(shape), strides=tuple(0 for _ in shape))
        w = v[index]
        return tuple(w.shape), tuple(0 for _ in w.shape), 0
    v = np.lib.stride_tricks.as_strided(base, shape=tuple(shape), strides=tuple(int(s) for s in strides))
    w = v[index]
    off = w.__array_interface__["data"][0] - v.__array_interface__["data"][0]
    return tuple(w.shape), tuple(w.strides), int(off)


class _Region:
    """A strided window into a device buffer that may carry negative strides (torch cannot express those)."""

    def __init__(self, base: torch.Tensor, shape, strides, offset):
        self.base, self.shape, self.strides, self.offset = base, tuple(shape), tuple(strides), offset

    def as_tensor(self):
        if all(s >= 0 for s in self.strides):
            return self.base.as_strided(self.shape, self.strides, self.base.storage_offset() + self.offset)
        return None

    @property
    def ptr(self):
        return self.base.data_ptr() + self.offset * self.base.element_size()


def _copy_region_out(reg: _Region, dtype) -> torch.Tensor:
    out = dev.empty_t(reg.shape, reg.base.dtype)
    if out.numel():
        L = _lib.lib()
        _lib.check(L.ptk_copy_strided(dev.ptr(out), dev.i64_array(out.stride()), reg.ptr, dev.i64_array(reg.strides),
                                      dev.i64_array(reg.shape), len(reg.shape), out.element_size(), dev.stream_ptr()),
                   "ptk_copy_strided")
    return out


class SubtensorNode(Node):
    """Reference: Subtensor, pytensor/tensor/subtensor.py:868 (a view; bit-exact by construction)."""

    def __init__(self, idx_template, name="Subtensor"):
        self.idx_template = idx_template
        self.name = name

    def run(self, vals):
        v = vals[0]
        index = _build_index(self.idx_template, vals[1:])
        if v.d is None:
            return [Val(h=np.asarray(v.h)[index])]
        t = v.d
        shape, strides, off = _probe(t.shape, t.stride(), index)
        reg = _Region(t, shape, strides, off)
        view = reg.as_tensor()
        if view is None:
            view = _copy_region_out(reg, t.dtype)
        return [Val(d=view)]


class IncSubtensorNode(Node):
    """Reference: IncSubtensor, pytensor/tensor/subtensor.py:1441 (x[idx] += y or x[idx] = y; optional in place)."""

    def __init__(self, idx_template, inplace, set_instead_of_inc, dtype, name="IncSubtensor"):
        self.idx_template = idx_template
        self.inplace = inplace
        self.set_instead_of_inc = set_instead_of_inc
        self.dtype = dtype
        self.destroy = {0: 0} if inplace else {}
        self.name = name

    def run(self, vals):
        x = vals[0].dev()
        y = vals[1].dev()
        if dev.TORCH_TO_NP[y.dtype] != self.dtype:  # y may be a narrower dtype than x (subtensor.py IncSubtensor.make_node)
            from .nodes_cast import cast_to

            y = cast_to(y, self.dtype)
        index = _build_index(self.idx_template, vals[2:])
        if not self.inplace:
            x = dev.clone(x)
        shape, strides, off = _probe(x.shape, x.stride(), index)
        n = 1
        for s in shape:
            n *= s
        if n:
            yb = _broadcast_view(y, shape)
            L = _lib.lib()
            ptr = x.data_ptr() + off * x.element_size()
            _lib.check(L.ptk_inc_strided(ptr, dev.i64_array(strides), dev.ptr(yb), dev.i64_array(yb.stride()),
                                         dev.i64_array(shape), len(shape), _lib.DTYPE_CODE[self.dtype],
                                         0 if self.set_instead_of_inc else 1, dev.stream_ptr()), "ptk_inc_strided")
        return [Val(d=x)]


# ---- advanced indexing: integer index arrays on one axis or on k consecutive axes, all other axes taken in full ---------
def _as_int64(t):
    if dev.TORCH_TO_NP[t.dtype] != "int64":
        from .nodes_cast import cast_to  # local import to avoid a cycle

        t = cast_to(t, "int64")
    return t


def _index_block(index_vals, dims, name):
    """k index arrays (NumPy broadcasting among them) -> ONE int64 device array of positions inside the row-major block
    of the k indexed axes (`ptk_linearize_index`: per-axis negative wrap + bounds check), shaped like the broadcast."""
    its = [_as_int64(v.dev()) for v in index_vals]
    if len(its) == 1:
        return dev.contiguous(its[0])  # ptk_take / ptk_put wrap and bounds-check a single axis themselves
    shape = tuple(torch.broadcast_shapes(*[tuple(t.shape) for t in its]))
    its = [dev.contiguous(_broadcast_view(t, shape)) for t in its]
    n = 1
    for s in shape:
        n *= s
    lin = dev.empty(shape, "int64")
    if n:
        ptrs = (ctypes.c_void_p * len(its))(*[dev.ptr(t) for t in its])
        flag = _err_flag(f"{name}: index out of bounds")
        _lib.check(_lib.lib().ptk_linearize_index(len(its), ptrs, dev.i64_array(dims), n, dev.ptr(lin), flag,
                                                  dev.stream_ptr()), "ptk_linearize_index")
    return lin


class TakeNode(Node):
    """AdvancedSubtensor (pytensor/tensor/subtensor.py:1932; NumPy semantics, perform :2164): `naxes` integer index arrays
    on the consecutive axes [axis, axis + naxes), every other axis taken in full.  The indexed block is treated as one
    axis of length prod(dims) addressed by a linearised index, so a single gather kernel serves every case."""

    def __init__(self, axis, name="AdvancedSubtensor", naxes=1):
        self.axis = axis
        self.naxes = naxes
        self.name = name
        self._flag = None

    def run(self, vals):
        x = dev.contiguous(vals[0].dev())
        ax, k = self.axis, self.naxes
        it = _index_block(vals[1:1 + k], x.shape[ax:ax + k], self.name)
        outer = 1
        for s in x.shape[:ax]:
            outer *= s
        inner = 1
        for s in x.shape[ax + k:]:
            inner *= s
        n_src = 1
        for s in x.shape[ax:ax + k]:
            n_src *= s
        oshape = list(x.shape[:ax]) + list(it.shape) + list(x.shape[ax + k:])
        out = dev.empty_t(oshape, x.dtype)
        if out.numel():
            if n_src == 0:
                raise IndexError("index out of bounds (taking from an empty axis)")
            flag = _err_flag(f"{self.name}: index out of bounds")
            _lib.check(_lib.lib().ptk_take(dev.ptr(out), dev.ptr(x), dev.ptr(it), outer, n_src, it.numel(), inner,
                                           x.element_size(), flag, dev.stream_ptr()), "ptk_take")
        return [Val(d=out)]


class PutNode(Node):
    """AdvancedIncSubtensor with the same single-axis pattern (pytensor/tensor/subtensor.py:2275): x[.., idx, ..] += y
    (duplicates accumulate, np.add.at semantics :2513-2531) or = y."""

    def __init__(self, axis, inplace, set_instead_of_inc, dtype, name="AdvancedIncSubtensor", naxes=1):
        self.axis = axis
        self.naxes = naxes
        self.inplace = inplace
        self.set_instead_of_inc = set_instead_of_inc
        self.dtype = dtype
        self.destroy = {0: 0} if inplace else {}
        self.name = name

    def run(self, vals):
        x = vals[0].dev()
        if not self.inplace:
            x = dev.clone(x)
        elif not x.is_contiguous():
            raise NotImplementedError(f"{self.name}: in-place scatter into a non-contiguous buffer")
        x = x if x.is_contiguous() else dev.contiguous(x)
        ax, k = self.axis, self.naxes
        it = _index_block(vals[2:2 + k], x.shape[ax:ax + k], self.name)
        outer = 1
        for s in x.shape[:ax]:
            outer *= s
        inner = 1
        for s in x.shape[ax + k:]:
            inner *= s
        n_dst = 1
        for s in x.shape[ax:ax + k]:
            n_dst *= s
        yshape = list(x.shape[:ax]) + list(it.shape) + list(x.shape[ax + k:])
        y = vals[1].dev()
        if dev.TORCH_TO_NP[y.dtype] != self.dtype:
            from .nodes_cast import cast_to

            y = cast_to(y, self.dtype)
        yb = _broadcast_view(y, yshape)
        yc = dev.contiguous(yb) if not yb.is_contiguous() else yb
        n = 1
        for s in yshape:
            n *= s
        isz = x.element_size()
        if (n and inner == 1 and it.dim() == 1 and not self.set_instead_of_inc and self.dtype in ("float32", "float64")
                and outer >= 64 and n_dst + 1 <= 12000 and it.numel() * isz <= 48 * 1024):
            # many rows share one index vector: deterministic segmented reduction instead of atomics
            L = _lib.lib()
            wsb = int(L.ptk_put_rows_workspace_bytes(n_dst, it.numel()))
            ws = dev.empty_t((wsb,), torch.uint8)
            flag = _err_flag(f"{self.name}: index out of bounds")
            _lib.check(L.ptk_put_rows(dev.ptr(x), dev.ptr(yc), dev.ptr(it), outer, n_dst, it.numel(),
                                      _lib.DTYPE_CODE[self.dtype], dev.ptr(ws), wsb, flag, dev.stream_ptr()),
                       "ptk_put_rows")
            return [Val(d=x)]
        if n:
            flag = _err_flag(f"{self.name}: index out of bounds")
            _lib.check(_lib.lib().ptk_put(dev.ptr(x), dev.ptr(yc), dev.ptr(it), outer, n_dst, it.numel(), inner,
                                          _lib.DTYPE_CODE[self.dtype], 0 if self.set_instead_of_inc else 1,
                                          flag, dev.stream_ptr()), "ptk_put")
        return [Val(d=x)]


# ---- deferred device-side error flags ------------------------------------------------------------------------------------
class FlagSink:
    """Per-Executor error words (ADVICE r1): every gather/scatter launch of one compiled function reports out-of-bounds
    indices into its own slot of ONE persistent int32 array (kernels `atomicExch(slot, 1)`: sticky, never cleared on the
    device while a call is in flight).  The array is mirrored into page-locked host memory by an asynchronous copy that
    is queued behind the call's kernels (inside the captured CUDA graph when the call replays one), so
      * a call that returns host arrays reads the mirror right after its single synchronisation (no extra D2H sync),
      * a call that returns device tensors never synchronises: the mirror is inspected (non-blocking) at the start of the
        function's next call and by `check(sync=True)` (`CudaVM.check_errors()`), so an out-of-bounds index is never
        dropped and never attributed to a different compiled function."""

    SLOTS = 64

    def __init__(self):
        self.words = None     # device int32[SLOTS]
        self.mirror = None    # pinned host int32[SLOTS]
        self.msgs = [None] * self.SLOTS   # (message, exception class) of each slot
        self.cursor = 0
        self.used = False     # some launch of the current call took a slot
        self.in_flight = False

    def _ensure(self):
        if self.words is None:
            st = dev.alloc_state
            arena, st.arena = st.arena, None   # persistent: never inside a capture arena
            measuring, st.measuring = st.measuring, False
            try:
                self.words = dev.empty_t((self.SLOTS,), torch.int32)
            finally:
                st.arena, st.measuring = arena, measuring
            side = dev._side_stream() if dev.alloc_state.capturing else None
            sp = side.cuda_stream if side is not None else dev.stream_ptr()
            _lib.check(_lib.lib().ptk_memset_async(dev.ptr(self.words), 0, 4 * self.SLOTS, sp), "memset")
            _lib.check(_lib.lib().ptk_sync_stream(sp), "sync")
            self.mirror = dev.pinned_empty((self.SLOTS,), "int32") if not _lib.TRACE_ONLY else np.zeros(self.SLOTS, "int32")
            self.mirror[:] = 0

    def begin_call(self):
        self.cursor = 0
        self.used = False

    def slot(self, msg, exc=IndexError) -> int:
        """Device address of the next error word of this call (program order -> the same slot on every call); a flagged
        word raises `exc(msg)`."""
        self._ensure()
        k = min(self.cursor, self.SLOTS - 1)
        self.cursor += 1
        self.msgs[k] = (msg, exc) if self.cursor <= self.SLOTS or exc is not IndexError else ("index out of bounds", exc)
        self.used = True
        return dev.ptr(self.words) + 4 * k

    def queue_mirror(self):
        """Queue words -> pinned mirror behind the work of the current stream (capturable: becomes a memcpy node)."""
        if self.words is None or _lib.TRACE_ONLY:
            return
        _lib.check(_lib.lib().ptk_memcpy_d2h_async(self.mirror.ctypes.data, dev.ptr(self.words), 4 * self.SLOTS,
                                                   dev.stream_ptr()), "d2h flags")
        self.in_flight = True

    def check(self, sync=False):
        """Raise the exception of the first flagged slot (IndexError for an out-of-bounds index, like the reference's C
        code; ValueError for a parameter a random sampler rejects) if a completed call flagged one."""
        if self.words is None or not self.in_flight:
            return
        if sync:
            if dev.alloc_state.capturing:
                return
            dev.synchronize()
        bad = np.flatnonzero(self.mirror)
        if bad.size:
            msg, exc = self.msgs[int(bad[0])] or ("index out of bounds", IndexError)
            self.mirror[:] = 0
            _lib.check(_lib.lib().ptk_memset_async(dev.ptr(self.words), 0, 4 * self.SLOTS, dev.stream_ptr()), "memset")
            raise exc(msg)
        if sync:
            self.in_flight = False


_default_sink = FlagSink()   # nodes run outside an Executor (unit tests drive node.run directly)
_sink_stack: list = []


def current_sink() -> FlagSink:
    return _sink_stack[-1] if _sink_stack else _default_sink


def _err_flag(msg="index out of bounds", exc=IndexError) -> int:
    """Device ADDRESS (int) of an error word owned by the running Executor."""
    return current_sink().slot(msg, exc)


def check_pending_flags():
    """Synchronising check of the default sink (direct node use)."""
    _default_sink.queue_mirror()
    _default_sink.check(sync=True)


class AssertNode(Node):
    """Reference: Assert / CheckAndRaise, pytensor/raise_op.py:148 (view of input 0 when all conditions hold)."""

    def __init__(self, msg, exc_name="AssertionError", exc_module="builtins"):
        self.msg = msg
        self.exc_name = exc_name       # qualified name + module: resolved at raise time (keeps the node picklable)
        self.exc_module = exc_module
        self.name = "Assert"

    def _exc_class(self):
        import importlib

        try:
            obj = importlib.import_module(self.exc_module)
            for part in self.exc_name.split("."):
                obj = getattr(obj, part)
            if isinstance(obj, type) and issubclass(obj, BaseException):
                return obj
        except Exception:  # noqa: BLE001 - the class may live in a module this box does not have
            pass
        return AssertionError

    def run(self, vals):
        for c in vals[1:]:
            if not bool(np.all(np.asarray(c.host()))):
                raise self._exc_class()(self.msg)
        v = vals[0]
        return [Val(h=v.h, d=v.d)]


class JoinNode(Node):
    """Reference: Join, pytensor/tensor/basic.py:2405 (concatenate along the static `axis`)."""

    def __init__(self, dtype, axis, name="Join"):
        self.dtype = dtype
        self.axis = axis
        self.name = name

    def run(self, vals):
        axis = self.axis
        parts = [v.dev() for v in vals]
        nd = parts[0].dim()
        axis %= nd
        oshape = list(parts[0].shape)
        for p in parts[1:]:
            if p.dim() != nd or any(p.shape[d] != oshape[d] for d in range(nd) if d != axis):
                raise ValueError("all the input array dimensions except for the concatenation axis must match exactly, "
                                 f"but got shapes {[tuple(q.shape) for q in parts]} for axis {axis}")
        oshape[axis] = sum(p.shape[axis] for p in parts)
        out = dev.empty(oshape, self.dtype)
        pos = 0
        for p in parts:
            n = p.shape[axis]
            if p.numel():
                dev.copy_strided(out.narrow(axis, pos, n), p)
            pos += n
        return [Val(d=out)]
