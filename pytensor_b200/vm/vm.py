"""The CUDA VM: executes a lowered program (a topologically ordered list of executable nodes) over device buffers.

Role of the reference's `Loop`/`Stack`/CVM (pytensor/link/vm.py:330,415; link/c/c_code/lazylinker_c.c:749-897):
run every thunk in order, drop intermediates after their last use, hand the outputs back, record the failing
position for `raise_with_op`.  Differences that matter on a GPU:
  * values are `Val`s (device buffers; host copies only for inputs/constants/shape integers);
  * input cells are read, never overwritten (so `SharedVariable.get_value` keeps seeing NumPy);
  * outputs are copied device->host once at the end (one synchronisation per call) unless `device_outputs`.
No pytensor import here: a program can be pickled and replayed on a box with only torch + libptk.
"""

from __future__ import annotations

import time
from ctypes import byref as ctypes_byref
from ctypes import c_void_p as ctypes_void_p

import numpy as np

from ..runtime import device as dev
from . import nodes_basic
from .values import Val, wrap


class Step:
    __slots__ = ("impl", "ins", "outs", "free", "origin")

    def __init__(self, impl, ins, outs, origin=-1):
        self.impl, self.ins, self.outs, self.free, self.origin = impl, list(ins), list(outs), [], origin

    def __getstate__(self):
        return (self.impl, self.ins, self.outs, self.free, self.origin)

    def __setstate__(self, st):
        self.impl, self.ins, self.outs, self.free, self.origin = st


class Program:
    """Flat, pytensor-free description of a compiled graph.

    n_slots value slots; `inputs` / `outputs` are slot ids; `constants` maps slot -> numpy array."""

    def __init__(self, n_slots, inputs, outputs, constants, steps):
        self.n_slots = n_slots
        self.inputs = list(inputs)
        self.outputs = list(outputs)
        self.constants = dict(constants)
        self.steps = list(steps)
        self._plan_gc()

    # ---- dependency structure for multi-stream execution ------------------------------------------------------------
    def plan_streams(self, max_streams=4):
        """Static stream assignment for the captured (graph) execution: `self.stream_of[i]` and `self.deps[i]`.

        Hazards honoured (the role `fgraph.orderings()` / `get_destroy_dependencies` play for the reference's VMs,
        pytensor/link/utils.py:831-847): true dependencies through slots, and — conservatively — any pair of steps where
        one WRITES into an alias group (views + in-place outputs share a group) that the other touches."""
        n = len(self.steps)
        parent = {}

        def find(x):
            while parent.setdefault(x, x) != x:
                parent[x] = parent[parent[x]]
                x = parent[x]
            return x

        def union(a, b):
            ra, rb = find(a), find(b)
            if ra != rb:
                parent[ra] = rb

        VIEW = ("DimShuffleNode", "ViewNode", "SubtensorNode", "ReshapeNode", "AssertNode")
        writers = [False] * n
        for i, st in enumerate(self.steps):
            name = type(st.impl).__name__
            if name in VIEW and st.ins and st.outs:
                union(st.ins[0], st.outs[0])
            if getattr(st.impl, "views_input0", False) and st.ins:  # every output is a view of input 0 (Split, ...)
                for o in st.outs:
                    union(st.ins[0], o)
            destroy = getattr(st.impl, "destroy", None) or {}
            for o, k in destroy.items():
                if o < len(st.outs) and k < len(st.ins):
                    union(st.outs[o], st.ins[k])
                    writers[i] = True
            if name in ("ScanNode", "ScanFusedElemwiseNode"):
                writers[i] = writers[i] or bool(destroy)
        producer = {}
        for i, st in enumerate(self.steps):
            for o in st.outs:
                producer[o] = i
        group_touch = {}   # group -> list of (step, is_write)
        deps = [set() for _ in range(n)]
        last_serial = {}
        for i, st in enumerate(self.steps):
            sg = getattr(st.impl, "serial_group", None)
            if sg is not None:
                if sg in last_serial:
                    deps[i].add(last_serial[sg])
                last_serial[sg] = i
            for sl in st.ins:
                if sl in producer and producer[sl] < i:
                    deps[i].add(producer[sl])
            groups_r = {find(sl) for sl in st.ins}
            groups_w = {find(st.ins[k]) for k in (getattr(st.impl, "destroy", None) or {}).values() if k < len(st.ins)}
            for g in groups_r | groups_w:
                for j, was_write in group_touch.get(g, []):
                    if was_write or g in groups_w:
                        deps[i].add(j)
            for g in groups_r | groups_w:
                group_touch.setdefault(g, []).append((i, g in groups_w))
        # greedy assignment: continue on the stream of a dependency whose last op is that dependency; else a free stream
        stream_of = [0] * n
        last_on = {}   # stream -> last step index
        for i in range(n):
            cand = None
            for d in sorted(deps[i], reverse=True):
                sd = stream_of[d]
                if last_on.get(sd) == d:
                    cand = sd
                    break
            if cand is None:
                used = set(last_on)
                free = [k for k in range(max_streams) if k not in used]
                if not deps[i] and free:
                    cand = free[0]
                elif free and deps[i]:
                    cand = free[0]
                else:
                    # reuse the stream whose last op is oldest
                    cand = min(range(max_streams), key=lambda k: last_on.get(k, -1))
            stream_of[i] = cand
            last_on[cand] = i
        self.deps = [sorted(d) for d in deps]
        self.stream_of = stream_of
        self.n_streams = max(stream_of) + 1 if stream_of else 1

    def weight_inputs(self):
        """{position in `inputs`: slot} of the program inputs (and the set of constant slots) that some GEMM node reads
        directly as its B operand — the candidates for the staged-operand cache (nodes_blas.staged_weight)."""
        if not hasattr(self, "_weight_inputs"):
            b_pos = {"Dot22Node": 1, "GemmBiasActNode": 1, "GemmNode": 3}
            slots = {st.ins[b_pos[type(st.impl).__name__]] for st in self.steps
                     if type(st.impl).__name__ in b_pos and len(st.ins) > b_pos[type(st.impl).__name__]}
            for st in self.steps:   # fused nodes that still read weight matrices directly (MlpChainNode)
                slots.update(st.ins[p] for p in getattr(st.impl, "weight_in_positions", ()) if p < len(st.ins))
            self._weight_inputs = ({k: s for k, s in enumerate(self.inputs) if s in slots},
                                   {s for s in self.constants if s in slots})
        return self._weight_inputs

    def streamable(self):
        """True when every step is row-independent along axis 0: fused Elemwise over non-broadcast operands, and
        reductions that keep axis 0.  Such a program can be run chunk by chunk along axis 0, which lets the executor
        overlap the host->device copy of chunk c+1 and the device->host copy of chunk c-1 with the kernels of chunk c
        (PCIe is full duplex; see Executor._run_chunked)."""
        ok = getattr(self, "_streamable", None)
        if ok is None:
            from .nodes_elemwise import CAReduceNode, ElemwiseNode, ElemwiseReduceNode

            def ew_ok(n):
                return n.ndim >= 1 and not any(any(b) for b in n.in_bcast)

            def red_ok(n):
                return n.ndim >= 2 and 0 not in n.axes

            ok = bool(self.steps) and bool(self.inputs)
            produced = set()
            for st in self.steps:
                t = type(st.impl)
                if t is ElemwiseNode:
                    good = ew_ok(st.impl)
                elif t is CAReduceNode:
                    good = red_ok(st.impl)
                elif t is ElemwiseReduceNode:
                    good = ew_ok(st.impl.ew) and red_ok(st.impl.red)
                else:
                    good = False
                if not good or any(j in self.constants for j in st.ins):
                    ok = False
                    break
                produced.update(st.outs)
            if ok:
                ok = all(s in produced for s in self.outputs) and len(set(self.outputs)) == len(self.outputs)
            self._streamable = ok
        return ok

    def _plan_gc(self):
        last = {}
        for i, st in enumerate(self.steps):
            for s in st.ins:
                last[s] = i
        keep = set(self.inputs) | set(self.outputs) | set(self.constants)
        for st in self.steps:
            st.free = []
        produced = set()
        for st in self.steps:
            produced.update(st.outs)
        for s, i in last.items():
            if s not in keep and s in produced:
                self.steps[i].free.append(s)
        # values never read and not outputs die right after they are produced
        for i, st in enumerate(self.steps):
            for s in st.outs:
                if s not in last and s not in keep:
                    st.free.append(s)


class _GraphEntry:
    __slots__ = ("stage", "nbytes", "arena", "gexec", "static_in", "out_vals", "flags", "keep")

    def __init__(self, nbytes):
        self.stage, self.nbytes = 1, nbytes
        self.arena = self.gexec = self.out_vals = None
        self.static_in, self.flags, self.keep = [], None, []   # flags: the sink's slot messages of this signature

    def __del__(self):
        g, self.gexec = self.gexec, None
        if g:
            try:
                from ..runtime import lib as _lib

                _lib.lib().ptk_graph_destroy(g)
            except Exception:
                pass


import itertools as _itertools

_executor_uid = _itertools.count(1)


class Executor:
    """Runs a Program.  `run(input_values) -> list of output Vals` (no host conversion).

    With `use_graph`, the launch list of a call signature (input shapes/dtypes, device-input addresses, values of tiny
    host inputs) is captured once into a CUDA graph over an arena of stable addresses and replayed with one
    cudaGraphLaunch per call afterwards — the device-side analogue of the CVM's precomputed instruction arrays
    (pytensor/link/vm.py:1057-1168).  First call of a signature: eager run that also measures the arena; second call:
    capture + launch; later calls: replay.  Anything that cannot live in a graph (a device->host read inside a node)
    abandons the capture and pins that signature to eager execution.
    """

    MAX_GRAPHS = 8
    STREAM_MIN_BYTES = 24 << 20   # host inputs smaller than this are not worth pipelining over PCIe
    STREAM_CHUNKS = 8              # at most this many chunks ... (measured: 4-8 best; every extra chunk costs ~30 us
    STREAM_CHUNK_BYTES = 16 << 20  # ... of about this many input bytes each     of copy-engine turnaround)

    def __getstate__(self):
        return {"program": self.program, "allow_gc": self.allow_gc, "use_graph": self.use_graph}

    def __setstate__(self, d):
        self.__init__(d["program"], d["allow_gc"], d["use_graph"])

    def __init__(self, program: Program, allow_gc=True, use_graph=False):
        self.use_graph = use_graph
        self.multi_stream = True   # independent branches on side streams inside captured graphs
        self.host_outputs = False  # set by the caller when results go back to NumPy (enables the chunked PCIe pipeline)
        self._d2h_stream = self._h2d_stream = None
        self.chunked_calls = 0
        self._chunk_plan = None
        self._side_streams = []
        self.last_from_graph = False
        self._graphs = {}
        self._id_cache = {}
        self._graph_misses = 0
        self.program = program
        self.allow_gc = allow_gc
        self.vals = [None] * program.n_slots
        for s, arr in program.constants.items():
            self.vals[s] = Val(h=np.asarray(arr))
        self._uid = next(_executor_uid)
        w_in, w_const = program.weight_inputs()
        for s in w_const:
            # a graph constant never changes: its staged copy stays resident (a process-unique number, not id(): ids recycle)
            self.vals[s].key = ("const", self._uid, s)
        self._w_in = w_in
        self._w_track = {}    # input position -> [tensor object (strong ref), torch version, identical calls in a row, volatile]
        self._w_keys = {}     # input position -> content key of THIS call (stable inputs only)
        self.position_of_error = -1
        self.time_nodes = False
        n = max([len(program.steps)] + [st.origin + 1 for st in program.steps])
        self.call_times = [0.0] * n
        self.call_counts = [0] * n
        self.event_log = None  # when a list: (step index, start event, stop event) per executed step (no syncs)
        self.sink = nodes_basic.FlagSink()  # this function's device-side error words (out-of-bounds indices)
        self.epilogue = None  # callable(out_vals) run on the VM stream right after the last node (e.g. the in-graph
        #                       all-reduce of a batch-sharded evaluation, pytensor_b200/sharded.py); captured with the graph

    # ---- CUDA-graph path ------------------------------------------------------------------------------------------
    @staticmethod
    def _signature(inputs):
        import torch

        sig = []
        for x in inputs:
            if isinstance(x, Val):
                return None
            if isinstance(x, torch.Tensor):
                if not x.is_cuda:
                    return None
                sig.append(("d", x.data_ptr(), tuple(x.shape), tuple(x.stride()), x.dtype))
            elif isinstance(x, np.random.Generator):
                return None   # random draws are keyed per call: never a CUDA graph
            else:
                a = np.asarray(x)
                small = tuple(a.reshape(-1).tolist()) if a.size <= 8 else None
                sig.append(("h", a.shape, a.dtype.str, small))
        return tuple(sig)

    def _track_weights(self, inputs):
        """Which B operands of this call are KNOWN to hold what they held on the previous calls: the same caller-owned
        torch tensor object (kept alive here, so its address cannot be recycled) at the same `Tensor._version` for the
        third call in a row.  A tensor whose version ever moves between calls is treated as volatile from then on
        (training-style in-place updates: staging it inside the graph is the right thing).  Returns the keys as a
        hashable tuple — part of the graph signature, because a graph captured over a resident staged copy must only be
        replayed for exactly that content."""
        keys = self._w_keys
        keys.clear()
        for k in self._w_in:
            x = inputs[k]
            tr = self._w_track.get(k)
            if not hasattr(x, "is_cuda") or not x.is_cuda:
                if tr is not None:
                    self._forget(self._w_track.pop(k)[4])
                continue
            v = x._version
            if tr is None or tr[0] is not x:
                # another object: a new process-unique serial (an id() could be the recycled id of a dead tensor, and the
                # key is part of the graph signature), and everything staged for the previous object is dropped
                if tr is not None:
                    self._forget(tr[4])
                self._w_track[k] = [x, v, 0, False, next(_executor_uid)]
                continue
            if tr[1] != v:
                tr[1], tr[2], tr[3] = v, 0, True
                self._forget(tr[4])
                continue
            tr[2] += 1
            if tr[2] >= 2 and not tr[3]:
                keys[k] = ("in", tr[4], v)
        return tuple(sorted(keys.items())) if keys else ()

    @staticmethod
    def _forget(serial, kind="in"):
        from . import nodes_blas

        nodes_blas.forget_weights(kind, serial)

    def __del__(self):
        try:   # staged copies only this executor's keys (and captured graphs) can reach
            for tr in self._w_track.values():
                self._forget(tr[4])
            self._forget(self._uid, "const")
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass

    def _wrap_inputs(self, inputs):
        vals = self.vals
        keys = self._w_keys
        for k, (s, x) in enumerate(zip(self.program.inputs, inputs)):
            v = wrap(x)
            if keys and k in keys and v.key is None:
                v.key = keys[k]
            vals[s] = v

    def run(self, inputs):
        """Outermost executors own the error-word sink of the call; nested ones (OpFromGraph, Scan bodies, pipeline
        chunks) report into their caller's."""
        stack = nodes_basic._sink_stack
        if stack:
            return self._run(inputs)
        sink = self.sink
        sink.check()          # non-blocking: an out-of-bounds index flagged by an earlier device-output call
        sink.begin_call()
        stack.append(sink)
        try:
            outs = self._run(inputs)
            if sink.used and not self.last_from_graph:
                sink.queue_mirror()   # (a replayed graph carries the mirror copy as its last node)
            return outs
        finally:
            stack.pop()

    def _run(self, inputs):
        from ..runtime import lib as _lib

        self.last_from_graph = False
        wkeys = self._track_weights(inputs) if self._w_in else ()
        if (not self.use_graph or _lib.TRACE_ONLY or self.time_nodes or self.event_log is not None
                or dev.alloc_state.capturing or dev.alloc_state.measuring):
            return self._run_eager(inputs)
        if self.host_outputs and self._chunkable(inputs):
            outs = self._run_chunked(inputs)
            if outs is not None:
                return outs
        # hot path: the very same input OBJECTS as an earlier replayed call (device tensors / large host arrays whose
        # metadata cannot change under us) -> skip building the signature
        ids = tuple(map(id, inputs))
        hit = self._id_cache.get(ids)
        if hit is not None and hit[1].stage == 2 and hit[2] == wkeys:
            e = hit[1]
            sig = None
        else:
            sig = self._signature(inputs)
            if sig is None:
                return self._run_eager(inputs)
            if wkeys:
                sig = sig + (("resident", wkeys),)   # graphs over resident staged weights are content-specific
            e = self._graphs.get(sig)
            if e is not None and e.stage == 2 and all(
                    (hasattr(x, "is_cuda") or np.asarray(x).size > 8) for x in inputs):
                if len(self._id_cache) > 16:
                    self._id_cache.clear()
                self._id_cache[ids] = (list(inputs), e, wkeys)  # strong refs keep the ids from being recycled
        if e is None:
            if len(self._graphs) >= self.MAX_GRAPHS:
                self._graph_misses += 1
                return self._run_eager(inputs)
            st = dev.alloc_state
            st.measuring, st.measured = True, 0
            try:
                outs = self._run_eager(inputs)
            finally:
                st.measuring = False
            extra = sum(int(np.asarray(x).nbytes) + 512 for x in inputs if not hasattr(x, "is_cuda"))
            self._graphs[sig] = _GraphEntry(st.measured + extra + 4096)
            return outs
        if e.stage == 1:
            return self._capture(e, inputs)
        if e.stage == 2:
            L = _lib.lib()
            sp = dev.stream_ptr()
            for k, t in e.static_in:
                a = np.asarray(inputs[k])
                if not a.flags.c_contiguous:
                    a = np.ascontiguousarray(a)
                    e.keep.append(a)
                if a.size:
                    _lib.check(L.ptk_memcpy_h2d_async(dev.ptr(t), a.ctypes.data, a.nbytes, sp), "h2d")
            _lib.check(L.ptk_graph_launch(e.gexec, sp), "graph launch")
            if e.flags is not None:
                sink = nodes_basic.current_sink()
                sink.msgs, sink.used, sink.in_flight = e.flags, True, True
            e.keep.clear() if len(e.keep) > 64 else None
            self.last_from_graph = True
            return e.out_vals
        return self._run_eager(inputs)

    # ---- chunked host pipeline --------------------------------------------------------------------------------------
    def _chunkable(self, inputs):
        if not inputs:
            return False
        a0 = inputs[0]
        if type(a0) is not np.ndarray or a0.ndim < 1 or a0.shape[0] < 2 or not self.program.streamable():
            return False
        rows = a0.shape[0]
        nbytes = 0
        for a in inputs:
            if type(a) is not np.ndarray or a.ndim < 1 or a.shape[0] != rows or not a.flags.c_contiguous:
                return False
            nbytes += a.nbytes
        return nbytes >= self.STREAM_MIN_BYTES

    def _run_chunked(self, inputs):
        """Host arrays in, host arrays out, row-independent program: split axis 0 into chunks and pipeline
        H2D(c+1) | kernels(c) | D2H(c-1).  Uploads run back to back on their own stream (the static input buffers are
        full size, so they never wait for a kernel), the kernels of chunk c wait on the VM stream for upload c, and
        downloads run on a third stream behind the kernels: both PCIe directions stay busy and a call costs about
        max(upload, download) plus one chunk of latency instead of their sum.

        The per-chunk device work runs through a private Executor over STATIC device input buffers: with `use_graph` its
        kernels are captured once per chunk and replayed with a single cudaGraphLaunch, which keeps the host cost per
        chunk (2 copies + 1 launch + 1 event) far below the chunk's DMA time.  Returns host Vals (pinned-pool arrays),
        or None if the first chunk shows the program does not keep axis 0 (the caller then takes the normal path)."""
        import torch

        from ..runtime import lib as _lib

        L = _lib.lib()
        main = torch.cuda.current_stream()
        if self._d2h_stream is None:
            self._d2h_stream = torch.cuda.Stream()
            self._h2d_stream = torch.cuda.Stream()
        side, up = self._d2h_stream, self._h2d_stream
        sp_up, sp2 = up.cuda_stream, side.cuda_stream
        key = tuple((a.shape, a.dtype.str) for a in inputs)
        plan = self._chunk_plan
        if plan is None or plan["key"] != key:
            rows = inputs[0].shape[0]
            in_bytes = sum(a.nbytes for a in inputs)
            nch = max(2, min(self.STREAM_CHUNKS, rows, in_bytes // self.STREAM_CHUNK_BYTES))
            bounds = [(rows * c // nch, rows * (c + 1) // nch) for c in range(nch)]
            static = [dev.empty(a.shape, a.dtype.name) for a in inputs]
            ev0 = torch.cuda.Event()  # the allocator may hand out blocks with work still queued on the VM stream
            ev0.record(main)
            up.wait_event(ev0)
            sub = Executor(self.program, self.allow_gc, self.use_graph)
            sub.MAX_GRAPHS = nch + 1
            sub.multi_stream = False
            plan = self._chunk_plan = {
                "key": key, "rows": rows, "bounds": bounds, "static": static, "sub": sub,
                "views": [[t[r0:r1] for t in static] for r0, r1 in bounds],
                "rowbytes": [a.nbytes // rows for a in inputs],
                "events": [torch.cuda.Event() for _ in bounds],
                "up_events": [torch.cuda.Event() for _ in bounds],
                "out_meta": None,
            }
        rows, sub = plan["rows"], plan["sub"]
        hbase = [a.ctypes.data for a in inputs]
        rowbytes = plan["rowbytes"]
        host_out = obase = None
        for c, (r0, r1) in enumerate(plan["bounds"]):
            views = plan["views"][c]
            for k, t in enumerate(views):
                nb = (r1 - r0) * rowbytes[k]
                if nb:
                    _lib.check(L.ptk_memcpy_h2d_async(t.data_ptr(), hbase[k] + r0 * rowbytes[k], nb, sp_up), "h2d")
            uev = plan["up_events"][c]
            uev.record(up)
            main.wait_event(uev)
            outs = sub.run(views)
            if host_out is None:
                meta = plan["out_meta"]
                if meta is None:
                    if any(v is None or v.d is None or v.d.dim() < 1 or v.d.shape[0] != r1 - r0
                           or not v.d.is_contiguous() for v in outs):
                        self.program._streamable = False
                        self._chunk_plan = None
                        return None
                    meta = plan["out_meta"] = [(tuple(v.d.shape[1:]), dev.TORCH_TO_NP[v.d.dtype]) for v in outs]
                host_out = [dev.host_empty((rows,) + tail, dt, always_pinned=True) for tail, dt in meta]
                obase = [(h.ctypes.data, h.nbytes // rows) for h in host_out]
            ev = plan["events"][c]
            ev.record(main)
            side.wait_event(ev)
            for v, (base, rb) in zip(outs, obase):
                nb = (r1 - r0) * rb
                if nb:
                    _lib.check(L.ptk_memcpy_d2h_async(base + r0 * rb, v.d.data_ptr(), nb, sp2), "d2h")
            if not sub.last_from_graph:
                # eagerly allocated results: keep them until the download stream is done with them
                plan.setdefault("keep", []).append(outs)
        _lib.check(L.ptk_sync_stream(sp2), "sync")
        plan.pop("keep", None)
        self.chunked_calls += 1
        return [Val(h=h, fresh=True) for h in host_out]

    def _capture(self, e, inputs):
        import torch

        from ..runtime import lib as _lib

        L = _lib.lib()
        st = dev.alloc_state
        sp = dev.stream_ptr()
        e.arena = dev.Arena(e.nbytes)
        st.arena = e.arena
        vals_in = []
        try:
            for k, x in enumerate(inputs):
                if isinstance(x, torch.Tensor):
                    vals_in.append(Val(d=x))
                else:
                    a = np.asarray(x)
                    if not a.flags.c_contiguous:  # (np.ascontiguousarray would also turn a 0-d array into 1-d)
                        a = np.ascontiguousarray(a)
                    t = dev.empty(a.shape, a.dtype.name)
                    if a.size:
                        _lib.check(L.ptk_memcpy_h2d_async(dev.ptr(t), a.ctypes.data, a.nbytes, sp), "h2d")
                    e.static_in.append((k, t))
                    vals_in.append(Val(h=a if a.size <= 8 else None, d=t))
            _lib.check(L.ptk_sync_stream(sp), "sync")
            sink = nodes_basic.current_sink()
            sink._ensure()
            sink.begin_call()
            _lib.check(L.ptk_graph_begin_capture(sp), "begin capture")
            st.capturing = True
            ok = True
            try:
                outs = self._run_streams(vals_in) if self.multi_stream else self._run_eager(vals_in)
                if sink.used:
                    sink.queue_mirror()   # memcpy node at the end of the graph: every replay refreshes the mirror
            except dev.GraphUnsupported:
                ok = False
            finally:
                st.capturing = False
                g = ctypes_void_p()
                rc = L.ptk_graph_end_capture(sp, ctypes_byref(g))
            if not ok or rc != 0:
                sink.begin_call()
                if rc == 0 and g.value:
                    L.ptk_graph_destroy(g)
                e.stage, e.arena, e.static_in = -1, None, []
                st.arena = None
                return self._run_eager(inputs)
            e.gexec = g.value
            e.flags = list(sink.msgs) if sink.used else None
            e.out_vals = outs
            e.stage = 2
        finally:
            st.arena = None
            st.capturing = False
        _lib.check(L.ptk_graph_launch(e.gexec, sp), "graph launch")
        if e.flags is not None:
            sink.in_flight = True
        self.last_from_graph = True
        return e.out_vals

    def _run_streams(self, inputs):
        """Capture-time execution with independent branches on side streams: the cross-stream event waits recorded here
        become the dependency edges of the CUDA graph, so replays run independent nodes concurrently."""
        import torch

        p = self.program
        if not hasattr(p, "stream_of"):
            p.plan_streams()
        if p.n_streams <= 1:
            return self._run_eager(inputs)
        main = torch.cuda.current_stream()
        while len(self._side_streams) < p.n_streams - 1:
            self._side_streams.append(torch.cuda.Stream())
        streams = [main] + self._side_streams[: p.n_streams - 1]
        vals = self.vals
        self._wrap_inputs(inputs)
        fork = torch.cuda.Event()
        fork.record(main)
        for sd in streams[1:]:
            sd.wait_event(fork)
        done = [None] * len(p.steps)
        try:
            for i, st in enumerate(p.steps):
                S = streams[p.stream_of[i]]
                for d in p.deps[i]:
                    if p.stream_of[d] != p.stream_of[i]:
                        S.wait_event(done[d])
                torch.cuda.set_stream(S)
                try:
                    res = st.impl.run([vals[j] for j in st.ins])
                except Exception:
                    self.position_of_error = st.origin if st.origin >= 0 else i
                    raise
                ev = torch.cuda.Event()
                ev.record(S)
                done[i] = ev
                for j, r in zip(st.outs, res):
                    vals[j] = r
        finally:
            torch.cuda.set_stream(main)
            for sd in streams[1:]:
                ev = torch.cuda.Event()
                ev.record(sd)
                main.wait_event(ev)
        outs = [vals[s] for s in p.outputs]
        if self.epilogue is not None:
            self.epilogue(outs)
        for s in range(len(vals)):
            if s not in p.constants:
                vals[s] = None
        return outs

    def _run_eager(self, inputs):
        p = self.program
        vals = self.vals
        self._wrap_inputs(inputs)
        timing = self.time_nodes
        for i, st in enumerate(p.steps):
            try:
                if timing:
                    dev.synchronize()
                    t0 = time.perf_counter()
                if self.event_log is not None:
                    import torch

                    e0 = torch.cuda.Event(enable_timing=True)
                    e1 = torch.cuda.Event(enable_timing=True)
                    e0.record()
                    res = st.impl.run([vals[j] for j in st.ins])
                    e1.record()
                    self.event_log.append((i, e0, e1))
                else:
                    res = st.impl.run([vals[j] for j in st.ins])
                if timing:
                    dev.synchronize()
                    k = st.origin if st.origin >= 0 else i
                    self.call_times[k] += time.perf_counter() - t0
                    self.call_counts[k] += 1
            except Exception:
                self.position_of_error = st.origin if st.origin >= 0 else i
                raise
            for j, r in zip(st.outs, res):
                vals[j] = r  # a fused node may return None for a value that is never materialised (and never read)
            if self.allow_gc:
                for j in st.free:
                    vals[j] = None
        outs = [vals[s] for s in p.outputs]
        if self.epilogue is not None:
            self.epilogue(outs)
        if self.allow_gc:
            for s in p.inputs:
                vals[s] = None
            for s in p.outputs:
                if s not in p.constants:
                    vals[s] = None
        return outs


def outputs_to_host(out_vals, device_outputs=False, copy_device=False, sink=None):
    """Val -> what Function.__call__ hands to the user: NumPy arrays (one sync) or device tensors.
    `copy_device`: device outputs may live in a graph arena that the next call overwrites -> hand out copies.
    `sink`: the executor's error words; their mirror copy was queued behind the call's kernels, so after the one
    synchronisation of a host-output call it is inspected for free.  Device outputs never synchronise: their flags are
    looked at when the function is called again (or by `CudaVM.check_errors()`)."""
    res = []
    pending = []
    for v in out_vals:
        if isinstance(v.h, np.random.Generator):
            res.append(v.h)   # the advanced generator of a RandomVariable node goes back as the object it is
        elif v.h is not None and v.d is None:
            # host-only values (shape vectors ...) are cached inside the VM: hand out a fresh object per call.  The
            # chunked host pipeline's results (Val.fresh: page-locked arrays it filled for THIS call) already are.
            res.append(np.asarray(v.h) if v.fresh else np.array(v.h, copy=True))
        elif device_outputs:
            res.append(dev.clone(v.d) if copy_device else v.d)
        else:
            res.append(None)
            pending.append((len(res) - 1, v))
    for k, v in pending:
        res[k] = dev.to_host(v.d, sync=False)
    if pending:
        dev.synchronize()
        if sink is not None:
            sink.check()
    elif sink is not None and sink.used and not device_outputs:
        sink.check(sync=True)
    return res
