"""CPU suite: every BASELINE.json config lowers under mode="CUDA" and its launch logic runs in trace-only mode
(NVRTC compiles each generated kernel for sm_90a; no device, no results)."""

import numpy as np
import pytest

from helpers import pytensor

import pytensor.tensor as pt
from pytensor_b200 import workloads as W
from pytensor_b200.precompile import trace_function


def pytensor_b200_mode(**kw):
    from pytensor_b200.link.cuda import cuda_mode

    return cuda_mode(**kw)


def _steps(f):
    return [type(st.impl).__name__ for st in f.vm.executor.program.steps]


def test_cfg2_is_one_fused_kernel():
    pytensor.config.floatX = "float32"
    ins, outs, mk, meta = W.cfg2_fused_elemwise(4096)
    f = pytensor.function(ins, outs, mode="CUDA")
    assert _steps(f) == ["ElemwiseReduceNode"]
    prog = f.vm.executor.program.steps[0].impl.ew.prog
    assert len(prog.insts) == 32 and prog.n_transcendental() == 2  # the "32-op" graph, HBM-bound by construction
    assert trace_function(f, mk()) == 1
    assert meta["bytes"] == 201342976  # SURVEY.md §8d


def test_cfg1_readme_has_gemv():
    ins, outs, mk, _ = W.cfg1_readme(128)
    f = pytensor.function(ins, outs, mode="CUDA")
    assert "GemvNode" in _steps(f)
    assert trace_function(f, mk()) >= 2


def test_cfg3_keeps_blas_ops_and_uses_the_tensor_core_mode():
    pytensor.config.floatX = "float32"
    ins, outs, mk, _ = W.cfg3_mlp(512)
    f = pytensor.function(ins, outs, mode="CUDA_BF16")
    names = _steps(f)
    # BlasOpt kept (3 x Dot22), each fused with its bias+tanh Elemwise into one tensor-core launch (K5)
    assert names.count("GemmBiasActNode") == 3 and "ElemwiseNode" not in names
    assert all(st.impl.precision == 1 and st.impl.act == 1 for st in f.vm.executor.program.steps
               if type(st.impl).__name__ == "GemmBiasActNode")
    trace_function(f, mk())
    f2 = pytensor.function(ins, outs, mode=__import__("pytensor_b200").link.cuda.cuda_mode(fuse=False))
    assert _steps(f2).count("Dot22Node") == 3


def test_cfg4_scan_lowers_to_the_persistent_kernel():
    pytensor.config.floatX = "float32"
    ins, outs, mk, _ = W.cfg4_scan(256, 64, 100)
    f = pytensor.function(ins, outs, mode="CUDA")
    assert "ScanFusedElemwiseNode" in _steps(f)
    assert trace_function(f, mk()) == 1  # ONE launch for all 100 steps
    # h <- tanh(h @ W + b): a chain of GEMM launches, one per step, each writing into the tap buffer (FMA kernel at this size)
    ins, outs, mk, _ = W.cfg4_scan(64, 64, 10, matmul=True)
    f = pytensor.function(ins, outs, mode="CUDA")
    assert "ScanMatmulRecurrenceNode" in _steps(f)
    assert trace_function(f, mk()) <= 10 + 6
    # tensor-core sizes: W and the initial state staged once (2 launches), then ONE launch per step
    ins, outs, mk, _ = W.cfg4_scan(512, 256, 12, matmul=True)
    f = pytensor.function(ins, outs, mode="CUDA")
    assert "ScanMatmulRecurrenceNode" in _steps(f)
    n_tc = trace_function(f, mk())
    f_loop = pytensor.function(ins, outs, mode=pytensor_b200_mode(fuse=False))
    assert "ScanNode" in _steps(f_loop)  # the general device loop stays available
    assert n_tc <= 12 + 2 + 6
    # anything else in the loop keeps the general node
    import pytensor.tensor as pt2

    h0, Wm = pt2.fmatrix("h0"), pt2.fmatrix("W")
    hs = pytensor.scan(lambda h, W: pt2.tanh(pt2.dot(h, W)) * 0.5 + h, outputs_info=[h0], non_sequences=[Wm], n_steps=3,
                       return_updates=False)
    assert "ScanNode" in _steps(pytensor.function([h0, Wm], hs[-1], mode="CUDA"))


def test_cfg5_and_metric_graph_lower():
    pytensor.config.floatX = "float32"
    ins, outs, mk, _ = W.cfg5_logp_grad(B=256, n=64, J=8, K=4)
    f = pytensor.function(ins, outs, mode="CUDA")
    names = _steps(f)
    # gather, both skinny Gemms, the Composites, the scatter-add and every Sum run as ONE row-fused region kernel ...
    assert names.count("RowRegionNode") == 1 and "TakeNode" not in names and "GemmNode" not in names
    region = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "RowRegionNode"][0]
    inner = [type(st.impl).__name__ for st in region.sub_steps]   # ... which keeps its constituent steps as the fallback
    assert "TakeNode" in inner and "PutNode" in inner and "GemmNode" in inner
    assert trace_function(f, mk()) <= 8   # region kernel + finishing kernel + the five tiny Join copies
    assert region.fused_calls == 1 and region.unfused_calls == 0
    ins, outs, mk, _ = W.metric_graph(n=16, layers=84, scan_steps=16)
    f = pytensor.function(ins, outs, mode="CUDA")
    assert len(f.maker.fgraph.toposort()) >= 256
    trace_function(f, mk())


def test_unsupported_ops_fail_at_compile_time_not_at_run_time():
    x = pt.dmatrix("x")
    with pytest.raises(NotImplementedError, match="no sm_90a implementation"):
        pytensor.function([x], pt.linalg.inv(x), mode="CUDA")
    c = pt.zmatrix("c")
    with pytest.raises(NotImplementedError):
        pytensor.function([c], c * 2, mode="CUDA")


def test_running_without_a_gpu_raises():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from pytensor_b200.runtime.lib import PtkError

    x = pt.dvector("x")
    f = pytensor.function([x], x * 2, mode="CUDA")
    with pytest.raises(PtkError, match="no CPU fallback"):
        f(np.ones(3))


def test_scalar_table_matches_reference_through_host_emulation(tmp_path):
    """The generated scalar body is plain C++: compile it for the host with a shim for the few device intrinsics and
    compare against the reference C linker on the same inputs (validates the codegen table without a GPU)."""
    import ctypes
    import subprocess

    from pytensor_b200.codegen.scalar import CTYPE, emit_body

    pytensor.config.floatX = "float32"
    a, b = pt.fvector("a"), pt.fvector("b")
    i = pt.lvector("i")
    out = [pt.tanh(a * b) + pt.exp(-pt.abs(b)) * pt.maximum(a, b) - pt.switch(a > b, pt.sqr(a), pt.log1p(pt.abs(b))),
           pt.sigmoid(a) + pt.softplus(b) + pt.erf(a) + pt.cast(i // 3 + i % 5, "float32") + pt.sign(a) * pt.floor(b)]
    f = pytensor.function([a, b, i], out, mode="CUDA")
    f_ref = pytensor.function([a, b, i], out, mode="CVM")
    steps = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "ElemwiseNode"]
    assert len(steps) == 1
    prog = steps[0].prog
    shim = r"""
#include <cmath>
#include <cstring>
#include <cstdint>
#define __device__
#define __forceinline__ inline
static inline float __int_as_float(int v) { float f; std::memcpy(&f, &v, 4); return f; }
static inline double __longlong_as_double(long long v) { double f; std::memcpy(&f, &v, 8); return f; }
static inline float ptk_max_nan_f32(float a, float b) { return (b > a) ? b : ((a >= b) ? a : NAN); }
static inline float ptk_min_nan_f32(float a, float b) { return (b < a) ? b : ((a <= b) ? a : NAN); }
using std::isnan; using std::isinf;
template <typename T> static inline T ptk_floordiv(T x, T y) { if (y == 0) return 0; T q = x / y; if ((x % y != 0) && ((x < 0) != (y < 0))) --q; return q; }
template <typename T> static inline T ptk_imod_py(T x, T y) { if (y == 0) return 0; T r = x % y; if (r != 0 && ((r < 0) != (y < 0))) r += y; return r; }
template <typename T> static inline T ptk_fmod_py(T x, T y) { T r = std::fmod(x, y); if (r != 0 && ((r < 0) != (y < 0))) r += y; return r; }
"""
    ins_decl = ", ".join(f"const {CTYPE[d]}* i{k}" for k, d in enumerate(prog.in_dtypes))
    outs_decl = ", ".join(f"{CTYPE[d]}* o{k}" for k, d in enumerate(prog.out_dtypes))
    call = ", ".join([f"i{k}[n]" for k in range(len(prog.in_dtypes))] + [f"o{k}[n]" for k in range(len(prog.out_dtypes))])
    src = shim + emit_body(prog) + f'\nextern "C" void run(long long N, {ins_decl}, {outs_decl}) {{ for (long long n = 0; n < N; ++n) ptk_body({call}); }}\n'
    cpp = tmp_path / "body.cpp"
    cpp.write_text(src)
    so = tmp_path / "body.so"
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", str(cpp), "-o", str(so)], check=True)
    L = ctypes.CDLL(str(so))
    rng = np.random.default_rng(91)
    N = 4000
    av, bv = rng.standard_normal(N).astype("float32") * 3, rng.standard_normal(N).astype("float32") * 3
    iv = rng.integers(-40, 40, size=N)
    order = [x.name for x in f.maker.fgraph.inputs]
    vals = {"a": av, "b": bv, "i": iv}
    node_inputs = [v for v in f.maker.fgraph.toposort() if type(v.op).__name__ == "Elemwise"][0].inputs
    arrays = []
    for v in node_inputs:
        src_name = v.name if v.name in vals else None
        assert src_name is not None, f"unexpected Elemwise input {v} (graph inputs {order})"
        arrays.append(np.ascontiguousarray(vals[src_name]))
    outs_np = [np.empty(N, dtype=d) for d in prog.out_dtypes]
    L.run(ctypes.c_longlong(N), *[x.ctypes.data_as(ctypes.c_void_p) for x in arrays],
          *[x.ctypes.data_as(ctypes.c_void_p) for x in outs_np])
    ref = f_ref(av, bv, iv)
    node_outs = [v for v in f.maker.fgraph.toposort() if type(v.op).__name__ == "Elemwise"][0].outputs
    for k, o in enumerate(node_outs):
        j = f.maker.fgraph.outputs.index(o)
        np.testing.assert_allclose(outs_np[k], ref[j], rtol=2e-6, atol=2e-6)


def test_device_resident_shared_variables_are_recognised_by_the_linker():
    # pytensor_b200.shared: the VM must find the shared input and its update output (trace-only: no device needed)
    import pytensor_b200
    from pytensor_b200.sharedvar import CudaSharedVariable

    pytensor.config.floatX = "float32"
    Wd = pytensor_b200.shared(np.ones((8, 4), "float32"), name="W")
    b = pytensor.shared(np.zeros(4, "float32"), name="b")
    x = pt.fmatrix("x")
    loss = (pt.tanh(pt.dot(x, Wd) + b) ** 2).sum()
    f = pytensor.function([x], loss, updates={Wd: Wd - np.float32(0.1) * pytensor.grad(loss, Wd)}, mode="CUDA")
    k = [i for i, v in enumerate(f.maker.fgraph.inputs) if isinstance(v, CudaSharedVariable)]
    assert f.vm.dev_shared == k and len(k) == 1
    assert f.vm.dev_updates == {1: k[0]}
    assert isinstance(Wd.type, pt.TensorType) and type(Wd.type) is pt.TensorType  # rewrites see a dense tensor
    assert "GemmNode" in _steps(f)  # ... so the BLAS rewrites still fire on it
    assert not Wd.on_device
    assert trace_function(f, [np.ones((5, 8), "float32")]) >= 2


def test_glue_ops_lower_and_trace():
    # §8(f).3 ops lower to their own nodes (no CPU fallback) and their launch logic runs in trace-only mode
    x = pt.dmatrix("x")
    i, j = pt.lvector("i"), pt.lvector("j")
    a, b = pt.split(x, [2, 3], n_splits=2, axis=1)
    outs = [pt.argmax(x, axis=0), pt.cumsum(x, axis=1), pt.eye(x.shape[0], x.shape[1], 1), pt.arange(x.shape[0] * 5000),
            a.sum() + b.sum(), pt.diagonal(x, offset=1), x[i, j], pt.inc_subtensor(x[i, j], 1.0)]
    f = pytensor.function([x, i, j], outs, mode="CUDA")
    names = _steps(f)
    for want in ("ArgmaxNode", "CumOpNode", "EyeNode", "ARangeNode", "SplitNode", "ExtractDiagNode", "TakeNode", "PutNode"):
        assert want in names, (want, names)
    take = next(st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "TakeNode")
    assert take.naxes == 2 and take.axis == 0
    assert trace_function(f, [np.ones((5, 5)), np.array([0, 1]), np.array([1, -1])]) >= 1  # (counts JIT kernels only)


def test_streamable_programs_are_row_independent_only():
    # the chunked host pipeline (Executor._run_chunked) may only split programs whose steps keep axis 0
    pytensor.config.floatX = "float32"
    ins, outs, _, _ = W.cfg2_fused_elemwise(64)
    assert pytensor.function(ins, outs, mode="CUDA").vm.executor.program.streamable()
    x, y = pt.fmatrix("x"), pt.fvector("y")
    assert pytensor.function([x], [pt.exp(x) + 1, x.sum(axis=1)], mode="CUDA").vm.executor.program.streamable()
    assert not pytensor.function([x], x.sum(axis=0), mode="CUDA").vm.executor.program.streamable()   # reduces axis 0
    assert not pytensor.function([x, y], x * y, mode="CUDA").vm.executor.program.streamable()       # broadcast operand
    assert not pytensor.function([x], pt.dot(x, x.T), mode="CUDA").vm.executor.program.streamable()  # not elementwise


def test_shape_errors_raise_the_reference_exception_types():
    # the boundary mirrors the reference's error behaviour: shape problems found by the host-side launch logic raise the
    # same exception TYPE as the C linker (trace-only mode runs exactly that logic, no device needed)
    pytensor.config.floatX = "float64"
    x, y = pt.dmatrix("x"), pt.dmatrix("y")
    v = pt.dvector("v")
    n = pt.lscalar("n")
    iv = pt.lvector("iv")
    cases = [
        ([x, y], x + y, [np.ones((3, 4)), np.ones((3, 5))]),                      # Elemwise dimension mismatch
        ([x, y], x * y, [np.ones((3, 4)), np.ones((1, 4))]),                      # runtime broadcasting is an error
        ([x, y], pt.dot(x, y), [np.ones((3, 4)), np.ones((5, 2))]),
        ([x, v], pt.dot(x, v), [np.ones((3, 4)), np.ones(5)]),
        ([x, n], x.reshape((n, 5)), [np.ones((3, 4)), np.asarray(2)]),
        ([x, y], pt.concatenate([x, y], axis=0), [np.ones((3, 4)), np.ones((2, 5))]),
        ([v, n], v[n], [np.ones(3), np.asarray(7)]),
        ([x, iv], pt.split(x, iv, n_splits=2, axis=1)[0], [np.ones((3, 4)), np.array([1, 1])]),
        ([x, v], pt.set_subtensor(x[0], v), [np.ones((3, 4)), np.ones(5)]),
        ([x], pt.linalg.cholesky(x), [np.ones((3, 4))]),
        ([x], pt.argmax(x, axis=1), [np.ones((3, 0))]),
    ]
    for ins, out, vals in cases:
        with pytest.raises(Exception) as ref:
            pytensor.function(ins, out, mode="CVM")(*vals)
        f = pytensor.function(ins, out, mode="CUDA")
        with pytest.raises(Exception) as got:
            trace_function(f, vals)
        assert got.type is ref.type, (str(out), got.type, ref.type, str(got.value).split("\\n")[0])


def test_opfromgraph_inner_graph_never_destroys_its_inputs():
    """ADVICE r1: the CUDA OpFromGraph rewrite must protect inner inputs and deep-copy aliased outputs like the
    reference's destructive variant (pytensor/compile/rewriting.py:141-152)."""
    from pytensor.compile.builders import OpFromGraph
    from pytensor.compile.ops import DeepCopyOp

    xi = pt.fmatrix("xi")
    x = pt.fmatrix("x")
    y = x * np.float32(2)
    f = pytensor.function([x], y + OpFromGraph([xi], [pt.exp(-xi)])(y), mode="CUDA")
    inner_nodes = [m for n in f.maker.fgraph.toposort() if isinstance(n.op, OpFromGraph) for m in n.op.fgraph.toposort()]
    assert inner_nodes and all(not getattr(m.op, "destroy_map", None) for m in inner_nodes)
    f2 = pytensor.function([x], OpFromGraph([xi], [xi.T])(y), mode="CUDA")
    inner2 = [m.op for n in f2.maker.fgraph.toposort() if isinstance(n.op, OpFromGraph) for m in n.op.fgraph.toposort()]
    assert any(isinstance(o, DeepCopyOp) for o in inner2)


def test_random_variables_lower_to_the_device_sampler_and_keep_the_generator_protocol():
    pytensor.config.floatX = "float32"
    rng = pytensor.shared(np.random.default_rng(3), name="rng")
    mu = pt.fvector("mu")
    nr, x = pt.random.normal(mu, 2.0, size=(4, 3), rng=rng).owner.outputs
    f = pytensor.function([mu], [x, pt.random.gamma(2.0, scale=1.0, size=(5,), rng=rng)], updates={rng: nr}, mode="CUDA")
    assert _steps(f).count("RandomVariableNode") == 2
    st0 = rng.get_value(borrow=True).bit_generator.state["state"]["state"]
    trace_function(f, [np.zeros(3, dtype="float32")])
    # multivariate / unsupported samplers are compile-time errors, like every other unsupported op
    with pytest.raises(NotImplementedError, match="no device sampler"):
        pytensor.function([], pt.random.multivariate_normal(np.zeros(2), np.eye(2), rng=rng), mode="CUDA")
    del st0


def test_runs_of_dense_layers_become_one_chain_node_only_when_nothing_else_reads_them():
    pytensor.config.floatX = "float32"
    # the metric graph: 84 layers -> ONE MlpChainNode reading x, 84 weights and 84 bias rows
    ins, outs, mk, _ = W.metric_graph(n=16, layers=84, scan_steps=4)
    f = pytensor.function(ins, outs, mode="CUDA")
    chain = [st for st in f.vm.executor.program.steps if type(st.impl).__name__ == "MlpChainNode"]
    assert len(chain) == 1 and len(chain[0].impl.layers) == 84
    assert len(chain[0].ins) == 1 + sum(2 if has_bias else 1 for _, has_bias in chain[0].impl.layers)
    assert "GemmBiasActNode" not in _steps(f) and "Dot22Node" not in _steps(f)
    # its weight inputs stay visible to the resident-weights bookkeeping
    w_in, _ = f.vm.executor.program.weight_inputs()
    assert len(w_in) == 84
    # three layers (cfg3) are left alone; so is a run whose intermediate is also an output
    ins, outs, mk, _ = W.cfg3_mlp(64)
    assert "MlpChainNode" not in _steps(pytensor.function(ins, outs, mode="CUDA"))
    x = pt.fmatrix("x")
    Ws = [pt.fmatrix(f"W{i}") for i in range(6)]
    hs = [x]
    for Wi in Ws:
        hs.append(pt.tanh(pt.dot(hs[-1], Wi)))
    f = pytensor.function([x, *Ws], [hs[-1], hs[3]], mode="CUDA")       # layer 3's result escapes: no run of >= 4 remains
    assert "MlpChainNode" not in _steps(f)
    f = pytensor.function([x, *Ws], [hs[-1], hs[1]], mode="CUDA")       # layers 2..6 still form a run of five
    chain = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == "MlpChainNode"]
    assert len(chain) == 1 and len(chain[0].layers) == 5
    trace_function(f, [np.zeros((8, 16), dtype="float32")] + [np.zeros((16, 16), dtype="float32")] * 6)


def test_advanced_indexing_dispatch_between_the_fast_and_the_general_nodes():
    """Integer index arrays on consecutive axes with everything else taken in full -> TakeNode / PutNode (one gather /
    scatter kernel); boolean masks, index arrays separated by a slice, partial slices next to an index array and
    `ignore_duplicates` increments -> the general AdvIndexNode / AdvIndexPutNode with the template NumPy's rules need
    (pytensor/tensor/subtensor.py:1932-2236)."""
    pytensor.config.floatX = "float32"
    x = pt.ftensor3("x")
    i, j = pt.lvector("i"), pt.lvector("j")
    mb = pt.tensor("mb", dtype="bool", shape=(None, None))
    y = pt.fmatrix("y")

    def only(f, name):
        nodes = [st.impl for st in f.vm.executor.program.steps if type(st.impl).__name__ == name]
        assert len(nodes) == 1, _steps(f)
        return nodes[0]

    assert "TakeNode" in _steps(pytensor.function([x, i], x[:, i], mode="CUDA"))
    assert "TakeNode" in _steps(pytensor.function([x, i, j], x[i, j], mode="CUDA"))
    n = only(pytensor.function([x, i, j], x[i, :, j], mode="CUDA"), "AdvIndexNode")           # separated by a slice
    assert [e[0] for e in n.template] == ["a", "s", "a"] and set(n.kinds.values()) == {("int", 1)}
    n = only(pytensor.function([x, mb], x[mb], mode="CUDA"), "AdvIndexNode")                   # 2-d mask over axes 0, 1
    assert n.template == [("a", 0)] and n.kinds == {0: ("bool", 2)}
    n = only(pytensor.function([x, i], x[1:, i], mode="CUDA"), "AdvIndexNode")                 # partial slice + index array
    assert n.template[0][0] == "s" and n.template[1] == ("a", n.template[1][1])
    assert _steps(pytensor.function([x, i, y], pt.inc_subtensor(x[:, i, 0], y), mode="CUDA")) == ["PutNode"]
    n = only(pytensor.function([x, mb, pt.fscalar("s")], pt.set_subtensor(x[mb], 0.5), mode="CUDA", on_unused_input="ignore"),
             "AdvIndexPutNode")
    assert n.set_instead_of_inc and n.kinds == {0: ("bool", 2)}
    n = only(pytensor.function([x, i, y], pt.inc_subtensor(x[i, :, 0], y, ignore_duplicates=True), mode="CUDA"), "AdvIndexPutNode")
    assert n.ignore_duplicates and not n.set_instead_of_inc


def test_scalar_ops_applied_to_scalar_typed_values_lower_as_zero_d_elemwise():
    """The reference's shape arithmetic sometimes survives as a ScalarOp applied to SCALAR-typed values between
    ScalarFromTensor and TensorFromScalar (here `maximum(shape_i, shape_j)` sizing the Gemv output of a broadcast sum; found
    by tests/lowering_fuzz.py): lowered as the same scalar program over 0-d values, evaluated on the host."""
    import pytensor.scalar.basic as ps
    from oracle import numpy_port

    pytensor.config.floatX = "float64"
    a, b, w, v = pt.dmatrix("a"), pt.dmatrix("b"), pt.dmatrix("w"), pt.dvector("v")
    k = a * 0.5 + b
    out = pt.dot(0.6 * k - 1.5 * pt.dot(pt.dot(k, w), w.T), v)
    f_ref = pytensor.function([a, b, w, v], out, mode="CVM")
    assert any(isinstance(n.op, ps.ScalarOp) for n in f_ref.maker.fgraph.toposort())   # the situation exists in this graph
    f = pytensor.function([a, b, w, v], out, mode="CUDA")
    rng = np.random.default_rng(5)
    vals = [rng.standard_normal((6, 4)), rng.standard_normal((6, 4)), rng.standard_normal((4, 3)), rng.standard_normal(4)]
    got = numpy_port.evaluate_program(f.vm.executor.program, vals)
    np.testing.assert_allclose(got[0], f_ref(*vals), rtol=1e-12, atol=1e-12)
    assert trace_function(f, vals) >= 1      # the host shape arithmetic really runs in trace-only mode


def test_host_integer_evaluator_leaves_c_conversion_corner_cases_to_the_device():
    """Small integer programs over host values are evaluated with NumPy (shape arithmetic).  Where C's usual arithmetic
    conversions — which the reference's generated code and the device kernels follow — differ from NumPy's promotion (a
    signed operand meeting an unsigned one of at least its width: int8(-3) * uint32(2) is 4294967290 in C, -6 in NumPy) the
    evaluator declines and the node takes the device path.  (Found with the port-oracle fuzzer over mixed integer dtypes.)"""
    from pytensor_b200.codegen.scalar import ScalarInst, ScalarProgram
    from pytensor_b200.vm.nodes_elemwise import host_eval_program

    def prog(op, in_dt, out_dt):
        return ScalarProgram(list(in_dt), [out_dt], [], [ScalarInst(op, [("i", k) for k in range(len(in_dt))], list(in_dt), out_dt)],
                             [("t", 0)])

    a8, u32 = np.array([-3, 2], dtype="int8"), np.array([2, 5], dtype="uint32")
    assert host_eval_program(prog("Mul", ["int8", "uint32"], "int64"), [a8, u32]) is None
    assert host_eval_program(prog("LT", ["int32", "uint64"], "bool"), [a8.astype("int32"), u32.astype("uint64")]) is None
    assert host_eval_program(prog("Switch", ["bool", "int32", "uint32"], "int64"), [a8 > 0, a8.astype("int32"), u32]) is None
    # no corner case: signed with a NARROWER unsigned (C promotes both to the signed type), and all-int64 shape arithmetic
    r = host_eval_program(prog("Mul", ["int64", "uint32"], "int64"), [a8.astype("int64"), u32])
    np.testing.assert_array_equal(r[0], np.array([-6, 10], dtype="int64"))
    r = host_eval_program(prog("Maximum", ["int64", "int64"], "int64"), [np.int64(7), np.int64(9)])
    assert int(r[0]) == 9


def test_floor_division_of_two_integers_with_a_float_result_compiles_for_the_device():
    """uint64 // int32 has the common type float64: the generated `floor(x / y)` got an INTEGER argument, which the device
    compiler rejects as ambiguous (the host compiler does not) — found by tracing random mixed-dtype graphs; the quotient
    is now converted explicitly."""
    p, q = pt.tensor("p", dtype="uint64", shape=(None,)), pt.tensor("q", dtype="int32", shape=(None,))
    f = pytensor.function([p, q], p // pt.switch(pt.eq(q, 0), 1, q), mode="CUDA")
    assert trace_function(f, [np.arange(1, 70, dtype="uint64"), np.arange(-34, 35, dtype="int32")]) >= 1   # NVRTC compiles it


def test_broadcast_shape_checks_stay_on_the_host():
    """With statically unknown shapes the reference guards a broadcast by Assert(All(MakeVector(eq(shape_i, shape_j), ...))).
    The tiny bool reduction used to be uploaded and reduced on the device, so the Assert needed a device round trip (and such
    a program could not be captured into a CUDA graph); integer / bool reductions of small host values now run on the host.
    In trace-only mode (no device values) the whole check therefore works — found by tracing random graphs."""
    from pytensor_b200.vm.nodes_elemwise import CAReduceNode

    pytensor.config.floatX = "float64"
    x, y, z = pt.dmatrix("x"), pt.lmatrix("y"), pt.lmatrix("z")
    from pytensor.raise_op import Assert

    same = pt.all(pt.stack([pt.eq(y.shape[0], z.shape[0]), pt.eq(y.shape[1], z.shape[1])]))   # the reference's own idiom
    out = Assert("shapes differ")(x.max(axis=1, keepdims=True), same) * pt.ones_like(y + z)
    f = pytensor.function([x, y, z], out, mode="CUDA")
    steps = f.vm.executor.program.steps
    assert any(type(s.impl).__name__ == "AssertNode" for s in steps) and any(
        type(s.impl) is CAReduceNode and s.impl.red_op == "and" for s in steps), [type(s.impl).__name__ for s in steps]
    assert trace_function(f, [np.zeros((70, 33)), np.ones((70, 33), dtype="int64"), np.ones((70, 33), dtype="int64")]) >= 1
    # the host reduction follows the declared accumulator / output types
    n = CAReduceNode("add", (0,), 2, "int8", "int64", "int64", 0)
    v = np.array([[100, -3], [100, 7], [100, 1]], dtype="int8")
    np.testing.assert_array_equal(n._run_host(v), np.array([300, 5], dtype="int64"))
    n = CAReduceNode("and", None, 1, "bool", "bool", "bool", 1)
    assert n._run_host(np.array([True, True])) == np.bool_(True) and n._run_host(np.array([True, False])) == np.bool_(False)
    assert n._run_host(np.zeros((0,), dtype=bool)) == np.bool_(True)      # empty: the identity
