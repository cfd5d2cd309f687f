"""`pytensor.link.cuda` — the H100 CUDA backend package (aliased into the `pytensor.link` namespace on registration).

Registration uses the reference's own hooks: `register_linker` / `register_mode` (pytensor/compile/mode.py:59,624)
and the inner-graph `singledispatch`es every linker must register with (`rewrite_scan_inner_graph`,
pytensor/scan/rewriting/inner_graph.py:28-33; `rewrite_ofg_inner_graph`, pytensor/compile/rewriting.py:128-134).
"""

from __future__ import annotations

import sys

from pytensor_b200.link.cuda.linker import CUDALinker, CudaVM  # noqa: F401

_registered = False


def register():
    """Make `pytensor.function(..., mode="CUDA")` (and "CUDA_BF16") resolve to the CUDALinker. Idempotent."""
    global _registered
    if _registered:
        return
    import pytensor.link
    from pytensor.compile import mode as pmode
    from pytensor.compile.rewriting import rewrite_ofg_inner_graph
    from pytensor.graph.rewriting.db import RewriteDatabaseQuery
    from pytensor.scan.rewriting.inner_graph import rewrite_scan_inner_graph, scan_inner_optimizer

    this = sys.modules[__name__]
    sys.modules.setdefault("pytensor.link.cuda", this)
    if not hasattr(pytensor.link, "cuda"):
        pytensor.link.cuda = this

    @rewrite_scan_inner_graph.register(CUDALinker)
    def _cuda_rewrite_scan_inner_graph(linker, op, node, inner, *, mode):
        # The device loop / persistent kernel manages the tap buffers itself, so no in-place taps are baked into the
        # inner graph (functional variant, inner_graph.py:85-90) — and every inner input is protected from destruction
        # (they are views into the circular buffers); in-place between inner intermediates is still allowed.
        from pytensor.compile.aliasing import add_supervisor_to_fgraph
        from pytensor.compile.io import In

        specs = [In(x, borrow=True, mutable=False) for x in inner.inputs]
        add_supervisor_to_fgraph(fgraph=inner, input_specs=specs, accept_inplace=True)
        scan_inner_optimizer(op, mode).rewrite(inner)

    @rewrite_ofg_inner_graph.register(CUDALinker)
    def _cuda_rewrite_ofg_inner_graph(linker, op, node, inner, *, mode):
        # Same contract as the reference's destructive variant (compile/rewriting.py:141-152): an OpFromGraph declares
        # no destroy_map / view_map, so its inner graph must neither write into its inputs (the outer VM hands the
        # caller's device buffers straight to the inner Executor) nor return views of them; in-place between purely
        # internal buffers stays allowed.
        from pytensor.compile.aliasing import add_supervisor_to_fgraph, insert_deepcopy
        from pytensor.compile.io import In, Out
        from pytensor.compile.rewriting import _ofg_inner_optimizer

        specs = [In(x, borrow=True, mutable=False) for x in inner.inputs]
        add_supervisor_to_fgraph(fgraph=inner, input_specs=specs, accept_inplace=True)
        _ofg_inner_optimizer(mode, op).rewrite(inner)
        insert_deepcopy(inner, wrapped_inputs=specs, wrapped_outputs=[Out(o, borrow=False) for o in inner.outputs])

    query = RewriteDatabaseQuery(include=["fast_run"], exclude=["cxx_only"])
    if "cuda" not in pmode.predefined_linkers:
        pmode.register_linker("cuda", CUDALinker())
        pmode.register_linker("cuda_bf16", CUDALinker(gemm_precision="bf16"))
    if "CUDA" not in pmode.predefined_modes:
        pmode.register_mode("CUDA", pmode.Mode(CUDALinker(), query))
        pmode.register_mode("CUDA_BF16", pmode.Mode(CUDALinker(gemm_precision="bf16"), query))
    _registered = True


def cuda_mode(**linker_kwargs):
    """A `Mode` with a customised CUDALinker, e.g. cuda_mode(device_outputs=True, gemm_precision="bf16")."""
    from pytensor.compile.mode import Mode
    from pytensor.graph.rewriting.db import RewriteDatabaseQuery

    register()
    return Mode(CUDALinker(**linker_kwargs), RewriteDatabaseQuery(include=["fast_run"], exclude=["cxx_only"]))
