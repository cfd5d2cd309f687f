"""`CUDALinker`: the H100 execution backend behind PyTensor's Linker plugin surface.

Boundary (reference file:line):
  * `Linker` / `LocalLinker` ABCs — pytensor/link/basic.py:138,228 (`make_thunk` :235-246 returns
    (fn, input Containers, output Containers)); `required_rewrites` / `incompatible_rewrites` :154-155.
  * `accept(fgraph, no_recycling, profile)` returning a NEW linker when already bound — pytensor/link/vm.py:849-913.
  * `accept_var_updates` — pytensor/link/vm.py:915-925 (called from compile/maker.py:611-620).
  * the VM object the `Function` drives — pytensor/compile/executor.py:651-760 reads `allow_gc`, `position_of_error`,
    `nodes`, `thunks`, `storage_map`, `time_thunks`/`call_times`/`call_counts`/`update_profile`
    (pytensor/link/vm.py:161-271), `need_update_inputs` (:186-193).
Per-node work is lowered ONCE at link time (lower.py) to executable CUDA nodes; unsupported ops raise
NotImplementedError at compile time.  There is no CPU fallback.
"""

from __future__ import annotations

from types import SimpleNamespace

import numpy as np

from pytensor.configdefaults import config
from pytensor.graph.basic import Constant
from pytensor.link.basic import Container, LocalLinker
from pytensor.link.utils import map_storage, raise_with_op

from pytensor_b200.link.cuda.lower import lower_node
from pytensor_b200.vm.vm import Executor, Program, Step, outputs_to_host


class CudaVM:
    """Callable handed to `Function` (role of pytensor.link.vm.VM)."""

    need_update_inputs = True

    def __init__(self, fgraph, nodes, executor, input_storage, output_storage, storage_map, allow_gc,
                 device_outputs, thunks):
        self.fgraph = fgraph
        self.nodes = nodes
        self.executor = executor
        self.input_storage = input_storage
        self.output_storage = output_storage
        self.storage_map = storage_map
        self.allow_gc = allow_gc
        self.device_outputs = device_outputs
        self.thunks = thunks
        self.position_of_error = -1
        self.time_thunks = False
        self.borrow_outputs = False
        # device-resident shared variables (pytensor_b200.shared): fgraph input positions whose cell may hold a torch
        # CUDA tensor, and update outputs (output index -> input index) that are written back on the device
        self.dev_shared = []
        self.dev_updates = {}
        self._shared_dev = {}
        self.call_times = executor.call_times
        self.call_counts = executor.call_counts

    def __call__(self, output_subset=None):
        ex = self.executor
        ex.time_nodes = self.time_thunks
        ex.host_outputs = not self.device_outputs
        if self.dev_shared:
            self._promote_shared()
        try:
            out_vals = ex.run([cell[0] for cell in self.input_storage])
        except Exception:
            self.position_of_error = ex.position_of_error
            raise
        if self.dev_updates:
            return self._finish_with_device_updates(out_vals, output_subset)
        if ex.last_from_graph and self.device_outputs and self.borrow_outputs and output_subset is None:
            # replayed graph, borrowed device outputs: hand out the arena views directly (no copies, no sync)
            outs = [v.d if v.d is not None else v.h for v in out_vals]
            for cell, o in zip(self.output_storage, outs):
                cell[0] = o
            return outs
        outs = outputs_to_host(out_vals, self.device_outputs, copy_device=ex.last_from_graph and not self.borrow_outputs,
                               sink=ex.sink)
        for cell, o in zip(self.output_storage, outs):
            cell[0] = o
        if output_subset is not None:
            return [o if i in output_subset else None for i, o in enumerate(outs)]
        return outs

    # ---- device-resident shared variables (SURVEY.md §8(f).1) -------------------------------------------------------
    def _promote_shared(self):
        """A CudaSharedVariable whose cell still holds a NumPy array (fresh, or after set_value(ndarray)) is uploaded
        once and the device tensor is left in the cell.  The previous device buffer is reused when the layout allows, so
        captured CUDA graphs (keyed on input addresses) keep replaying after a `set_value`."""
        from pytensor_b200.runtime import device as dev

        for k in self.dev_shared:
            cell = self.input_storage[k]
            v = cell[0]
            if v is None or hasattr(v, "is_cuda"):
                continue
            a = np.asarray(v)
            last = self._shared_dev.get(k)
            if (last is not None and tuple(last.shape) == a.shape and dev.TORCH_TO_NP[last.dtype] == a.dtype.name
                    and last.is_contiguous()):
                dev.to_device_async(a, out=last)
                dev.synchronize()  # the host array is dropped from the cell below: the copy must have completed
                dev.bump_version(last)   # same object, new content: staged copies of the old value are stale
                t = last
            else:
                t = dev.to_device(a)
            cell[0] = t
            self._shared_dev[k] = t

    def _finish_with_device_updates(self, out_vals, output_subset):
        """Outputs that are `updates=` of device-resident shared variables stay in HBM: the new value is copied
        device-to-device INTO the variable's current buffer (stable address -> the CUDA graph keeps replaying) and that
        same tensor object is handed back, which `Function.__call__` stores into the container
        (pytensor/compile/executor.py:712-716).  Everything else takes the usual host/device output path."""
        from pytensor_b200.runtime import device as dev

        ex = self.executor
        res = [None] * len(out_vals)
        for j, k in self.dev_updates.items():
            v = out_vals[j]
            cur = self.input_storage[k][0]
            cur_ok = hasattr(cur, "is_cuda")
            if v.d is None:  # small value computed on the host (shape arithmetic, scalars)
                h = np.ascontiguousarray(np.asarray(v.h))
                if cur_ok and tuple(cur.shape) == h.shape and dev.TORCH_TO_NP[cur.dtype] == h.dtype.name \
                        and cur.is_contiguous():
                    dev.to_device_async(h, out=cur)
                    dev.synchronize()
                    dev.bump_version(cur)
                    res[j] = cur
                else:
                    res[j] = dev.to_device(h)
                continue
            src = v.d
            same_layout = cur_ok and tuple(cur.shape) == tuple(src.shape) and cur.dtype == src.dtype
            if same_layout and cur.data_ptr() == src.data_ptr() and cur.stride() == src.stride():
                res[j] = cur  # computed in place on the variable's buffer (destroy_map on a mutable input)
                dev.bump_version(cur)
            elif same_layout and cur.untyped_storage().data_ptr() != src.untyped_storage().data_ptr():
                dev.copy_strided(cur, src)
                dev.bump_version(cur)
                res[j] = cur
            else:  # new shape, or a view overlapping the old value: give the variable a new buffer
                res[j] = dev.clone(src)
            self._shared_dev[k] = res[j]
        rest = [j for j in range(len(out_vals)) if j not in self.dev_updates]
        if rest:
            outs = outputs_to_host([out_vals[j] for j in rest], self.device_outputs,
                                   copy_device=ex.last_from_graph and not self.borrow_outputs, sink=ex.sink)
            for j, o in zip(rest, outs):
                res[j] = o
        # (an updates-only call never synchronises: its error words are inspected when the function is called again)
        for cell, o in zip(self.output_storage, res):
            cell[0] = o
        if output_subset is not None:
            return [o if (i in output_subset or i in self.dev_updates) else None for i, o in enumerate(res)]
        return res

    def check_errors(self):
        """Synchronise and raise the error (IndexError, or ValueError for a rejected sampler parameter) that an earlier
        device-output / updates-only call may have flagged (those calls never synchronise themselves; the next call of
        this function would raise it too)."""
        self.executor.sink.check(sync=True)

    def clear_storage(self):
        for i in range(len(self.executor.vals)):
            if i not in self.executor.program.constants:
                self.executor.vals[i] = None

    def update_profile(self, profile):
        for node, t, c in zip(self.nodes, self.call_times, self.call_counts):
            profile.apply_time[(self.fgraph, node)] += t
            profile.apply_callcount[(self.fgraph, node)] += c
            profile.apply_cimpl[node] = True
        for i in range(len(self.call_times)):
            self.call_times[i] = 0.0
            self.call_counts[i] = 0


class CUDALinker(LocalLinker):
    """Linker whose VM keeps every intermediate in HBM and runs hand-written sm_90a kernels through libptk.

    Parameters
    ----------
    gemm_precision : "fp32" (native FMA, <=1e-5 vs the C linker) or "bf16" (wgmma tensor cores: operands rounded to
        bf16, fp32 accumulation; parity vs the C linker at the half-precision tolerance, see DESIGN.md).
    device_outputs : return torch.cuda tensors instead of NumPy arrays (no device->host copy, no sync).
    """

    required_rewrites: tuple[str, ...] = ("minimum_compile",)
    incompatible_rewrites: tuple[str, ...] = ("cxx_only",)

    def __init__(self, allow_gc=None, gemm_precision="fp32", device_outputs=False, schedule=None, fuse=True,
                 use_graph=True, borrow_outputs=False):
        if allow_gc is None:
            allow_gc = config.allow_gc
        self.fgraph = None
        self.gemm_precision = gemm_precision
        self.device_outputs = device_outputs
        self.fuse = fuse
        self.use_graph = use_graph
        self.borrow_outputs = borrow_outputs  # device outputs may alias VM-owned memory that the next call overwrites
        self.updated_vars = {}
        super().__init__(allow_gc=allow_gc, scheduler=schedule)

    def accept(self, fgraph, no_recycling=None, profile=None):
        if no_recycling is None:
            no_recycling = []
        if self.fgraph is not None and self.fgraph is not fgraph:
            return type(self)(
                allow_gc=self.allow_gc, gemm_precision=self.gemm_precision, device_outputs=self.device_outputs,
                schedule=self._scheduler, fuse=self.fuse, use_graph=self.use_graph,
                borrow_outputs=self.borrow_outputs,
            ).accept(fgraph, no_recycling, profile)
        self.fgraph = fgraph
        self.no_recycling = no_recycling
        self.profile = profile
        return self

    def accept_var_updates(self, updated_vars):
        self.updated_vars = updated_vars

    def lowering_options(self):
        return {"gemm_precision": 1 if self.gemm_precision == "bf16" else 0, "fuse": self.fuse, "linker": self}

    def make_all(self, input_storage=None, output_storage=None, storage_map=None):
        fgraph = self.fgraph
        order = self.schedule(fgraph)
        input_storage, output_storage, storage_map = map_storage(
            fgraph, order, input_storage, output_storage, storage_map
        )
        program, thunks = build_program(fgraph, order, self.lowering_options(), storage_map)
        executor = Executor(program, allow_gc=bool(self.allow_gc), use_graph=bool(self.use_graph))
        vm = CudaVM(fgraph, order, executor, input_storage, output_storage, storage_map, bool(self.allow_gc),
                    self.device_outputs, thunks)
        vm.borrow_outputs = self.borrow_outputs
        from pytensor_b200.sharedvar import CudaSharedVariable

        vm.dev_shared = [k for k, v in enumerate(fgraph.inputs) if isinstance(v, CudaSharedVariable)]
        mapping = getattr(fgraph, "update_mapping", None) or {}
        vm.dev_updates = {int(o): int(i) for o, i in mapping.items() if i in vm.dev_shared}
        return (
            vm,
            [Container(i, s) for i, s in zip(fgraph.inputs, input_storage, strict=True)],
            [Container(o, s, readonly=True) for o, s in zip(fgraph.outputs, output_storage, strict=True)],
            thunks,
            order,
        )


def build_program(fgraph, order, opts, storage_map=None):
    """FunctionGraph + schedule -> (Program, thunk-like records for error reporting)."""
    slots = {}

    def slot(v):
        if v not in slots:
            slots[v] = len(slots)
        return slots[v]

    for v in fgraph.inputs:
        slot(v)
    constants = {}
    steps = []
    thunks = []
    from pytensor_b200.link.cuda.fusion import fuse_steps

    for node in order:
        for v in node.inputs:
            if v not in slots:
                if isinstance(v, Constant):
                    constants[slot(v)] = np.asarray(v.data)
                elif v.owner is None:
                    # orphan non-constant (e.g. a shared variable's container): its cell is filled by the caller
                    if storage_map is not None and v in storage_map:
                        slot(v)
                    else:
                        raise ValueError(f"CUDALinker: variable {v} has no producer")
        try:
            impl = lower_node(node, opts)
        except Exception:
            raise_with_op(fgraph, node)
        st = Step(impl, [slot(v) for v in node.inputs], [slot(v) for v in node.outputs], origin=len(steps))
        steps.append(st)
        cells_in = [storage_map[v] for v in node.inputs] if storage_map is not None else []
        cells_out = [storage_map[v] for v in node.outputs] if storage_map is not None else []
        thunks.append(SimpleNamespace(inputs=cells_in, outputs=cells_out, lazy=False, impl=impl))
    for v in fgraph.outputs:
        if v not in slots:
            if isinstance(v, Constant):
                constants[slot(v)] = np.asarray(v.data)
            else:
                slot(v)
    if opts.get("fuse", True):
        # static types of every slot (dtype, ndim, broadcast pattern) + the constants: what the region finder needs
        fopts = dict(opts)
        fopts["slot_types"] = {k: (v.type.dtype, v.type.ndim, tuple(v.type.broadcastable))
                               for v, k in slots.items() if hasattr(v.type, "broadcastable")}
        fopts["constants"] = constants
        steps = fuse_steps(steps, [slots[v] for v in fgraph.outputs], fopts)
    program = Program(len(slots), [slots[v] for v in fgraph.inputs], [slots[v] for v in fgraph.outputs], constants,
                      steps)
    return program, thunks
