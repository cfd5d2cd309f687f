"""The row-fused region kernel (codegen/rowfuse.py `gen_region_kernel`, found by link/cuda/fusion_rows.py, run by
vm/nodes_rowfuse.py `RowRegionNode`) in every code form its generator emits, at its size and layout edges.

a. Integer grid: operands are small integers (|n| <= 7) or powers of two, the maps use only + - *, maximum, abs, switch
   and comparisons, alpha / beta are powers of two, and every partial sum is checked up front to fit in 24 bits.  Each
   output must then equal a NumPy fp64 restatement of the graph exactly (up to the sign of a zero), in fp32 and fp64,
   whatever order the kernel's shared-memory atomics and warp shuffles add in.  `pt.prod(w[:, idx], axis=1)` reaches the
   `mul` row reduction directly (with `no_zeros_in_input=True` its lowering adds ShapeI / MakeVector and no region forms).
b. Size regimes: the batch around MIN_ROWS and past one row per resident warp, domains of 1 / 31 / 32 / 33, the staging
   boundary (4096 bytes), the per-CTA index table boundary (8192 entries), the skinny-product form boundaries
   (reduce: q <= 16 and p > q; pointwise: p <= 32) and the fallbacks (domain > 65536, shared memory > 160 KB).
c. fp64 scatter-add adds the lanes of an iteration in lane order: the result equals x + s bit for bit, s being the
   sequential scatter-add of y into zeros in j order, with heavy duplicates and partial last iterations.
d. Layouts: strided and column-major operands, (B, 1) column slices, strided index vectors, X and X.T in one group,
   matrix operands that force the scalar loads, negative indices.
e. NaN / ±inf in gathered sources and scattered values; out-of-bounds indices through both index paths.
f. Replay: device inputs and outputs, six calls on two alternating input sets (eager, capture, replay).

Every fused case asserts one RowRegionNode with the intended op kinds that ran fused; every fallback case asserts the
unfused path and its reason.  In the dry run (PTK_DRY=1) the graphs are traced (lowering, finder, code generation and
NVRTC, fused / unfused decision) and the device results are not read; the tests that need the device skip."""

import os
import re

import numpy as np
import pytest

from helpers import pytensor

import pytensor.tensor as pt
from pytensor_b200.codegen import rowfuse as cg
from pytensor_b200.vm.nodes_rowfuse import RowRegionNode

pytestmark = pytest.mark.gpu

DRY = os.environ.get("PTK_DRY") == "1"
B0 = 203                    # default batch: more than MIN_ROWS, not a multiple of 8 warps


# ---- harness ------------------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _device(gpu, monkeypatch):
    for v in ("PTK_ROWFUSE", "PTK_ROWFUSE_CTA_INDEX"):
        monkeypatch.delenv(v, raising=False)
    yield


def _needs_device():
    if DRY:
        pytest.skip("reads device results")


def T(name, dtype="float32", nd=2):
    return pt.tensor(name, dtype=dtype, shape=(None,) * nd)


def _region(f):
    nodes = [st.impl for st in f.vm.executor.program.steps if isinstance(st.impl, RowRegionNode)]
    assert len(nodes) == 1, [type(st.impl).__name__ for st in f.vm.executor.program.steps]
    return nodes[0]


def _sources(node):
    return [hit[0].source for hit in node._kernels.values()]


def _has(node, pattern):
    """Every fused specialisation of the node contains `pattern` (a regex)."""
    srcs = _sources(node)
    assert srcs, "no fused kernel was generated"
    return all(re.search(pattern, s) for s in srcs)


def _same(got, exp, what=""):
    """Equal values (a zero of either sign equals a zero), NaN where NaN, same dtype and shape."""
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.dtype == exp.dtype and got.shape == exp.shape, (what, got.dtype, exp.dtype, got.shape, exp.shape)
    bad = ~((got == exp) | (np.isnan(got) & np.isnan(exp)))
    if bad.any():
        idx = np.argwhere(bad)[:5]
        raise AssertionError(f"{what}: {int(bad.sum())} of {exp.size} differ; first {idx.tolist()}: "
                             f"got {[got[tuple(i)] for i in idx]} expected {[exp[tuple(i)] for i in idx]}")


def _fits(bound, unit=1.0):
    """Exactness precondition: every partial sum (bounded by `bound`) is an integer multiple of `unit` below 2^24 units."""
    assert np.all(np.asarray(bound) < 2.0 ** 24 * unit), "test operands break the exactness precondition"


def _run(ins, outs, args, refs, kinds, fused=True, reason=None, device=False):
    """Compile, check the region's op kinds, call once and compare every output with `refs` exactly; `fused=False`:
    the node must have run its constituent steps for `reason`.  `device`: inputs and outputs stay on the device, so
    that views of the inputs reach the kernel with their own strides (host inputs are uploaded contiguous)."""
    if device:
        _needs_device()
        from pytensor_b200.link.cuda import cuda_mode

        f = pytensor.function(ins, outs, mode=cuda_mode(device_outputs=True), trust_input=True)
    else:
        f = pytensor.function(ins, outs, mode="CUDA")
    node = _region(f)
    assert [o.kind for o in node.plan.ops] == kinds, [o.kind for o in node.plan.ops]
    args = [np.array(a, copy=True) for a in args]
    if DRY:
        from pytensor_b200.precompile import trace_function

        trace_function(f, args)
        got = None
    elif device:
        import torch

        got = [o.cpu().numpy() for o in f(*[torch.from_numpy(a).cuda() for a in args])]
    else:
        got = f(*args)
    if fused:
        assert node.fused_calls >= 1 and node.unfused_calls == 0, node.last_reason
    else:
        assert node.fused_calls == 0 and node.unfused_calls >= 1
        assert reason in (node.last_reason or ""), node.last_reason
    if got is not None:
        assert len(got) == len(refs)
        for k, (g, e) in enumerate(zip(got, refs)):
            _same(g, e, f"output {k}")
    return f, node


def _ints(rng, shape, lo=-7, hi=7):
    return rng.integers(lo, hi + 1, shape).astype(np.float64)


def _idx(rng, n, m, dtype="int64", neg=False):
    """`n` indices into an axis of `m` (repeats, both ends of the axis present); `neg`: some written as i - m."""
    i = rng.integers(0, m, n)
    i[: min(n, 2)] = [m - 1, 0][: min(n, 2)]
    if neg:
        i = np.where(rng.random(n) < 0.4, i - m, i)
    return i.astype(dtype)


# ---- a. integer grid ------------------------------------------------------------------------------------------------------
DT = ["float32", "float64"]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("red", ["max", "min_map", "prod", "sum"])
def test_gather_row_reductions(dtype, red):
    rng = np.random.default_rng(1)
    m, n = 37, 45
    w, idx = T("w", dtype), T("idx", "int64", 1)
    g = w[:, idx]
    W, I = _ints(rng, (B0, m)), _idx(rng, n, m)
    G = W[:, I]
    if red == "max":
        out, ref, kinds, op = g.max(axis=1), G.max(axis=1), ["take", "rsum"], "maximum"
    elif red == "min_map":
        out = pt.min(pt.switch(g > 1, g * 2 - 3, pt.abs(g) - g), axis=1)
        ref, kinds, op = np.where(G > 1, G * 2 - 3, np.abs(G) - G).min(axis=1), ["take", "ew", "rsum"], "minimum"
    elif red == "prod":       # powers of two, mostly ±1: every product exact, far inside the fp32 range
        W = rng.choice([1.0, -1.0, 2.0, -2.0, 0.5, -0.5], (B0, m), p=[0.4, 0.4, 0.05, 0.05, 0.05, 0.05])
        G = W[:, I]
        out, ref, kinds, op = pt.prod(g, axis=1), G.prod(axis=1), ["take", "rsum"], "mul"
        assert np.all(np.abs(np.log2(np.abs(G)).sum(axis=1)) < 100)
    else:
        out, ref, kinds, op = g.sum(axis=1), G.sum(axis=1), ["take", "rsum"], "add"
        _fits(np.abs(G).sum(axis=1))
    f, node = _run([w, idx], [out], [W.astype(dtype), I], [ref.astype(dtype)], kinds)
    assert node.plan.ops[-1].red == op


def _product_case(case, dtype, rng, p=None, q=None):
    """(inputs, outputs, arrays, refs, kinds, form) of one skinny-product graph on the integer grid."""
    w, idx, X = T("w", dtype), T("idx", "int64", 1), T("X", dtype)
    m = 23
    if case == "reduce":                      # dot(map(w[:, idx]), X): n = p > q
        p, q = p or 45, q or 5
        g = w[:, idx]
        W, I, Xv = _ints(rng, (B0, m)), _idx(rng, p, m), _ints(rng, (p, q))
        Gm = np.maximum(W[:, I], 0) * 2 - W[:, I]
        _fits(np.abs(Gm) @ np.abs(Xv))
        return ([w, idx, X], [pt.dot(pt.maximum(g, 0) * 2 - g, X)], [W, I, Xv], [Gm @ Xv], ["take", "ew", "gemm"],
                "reduce")
    if case == "plain":                       # dot(w[:, idx], X) at given p, q
        g = w[:, idx]
        W, I, Xv = _ints(rng, (B0, m)), _idx(rng, p, m), _ints(rng, (p, q))
        _fits(np.abs(W[:, I]) @ np.abs(Xv))
        return [w, idx, X], [pt.dot(g, X)], [W, I, Xv], [W[:, I] @ Xv], ["take", "gemm"], None
    if case == "pointwise":                   # w[:, idx] + dot(bt, X.T): p = 7 operand values per row
        p, n = 7, 41
        bt = T("bt", dtype)
        W, I, Bt, Xv = _ints(rng, (B0, m)), _idx(rng, n, m), _ints(rng, (B0, p)), _ints(rng, (n, p))
        _fits(np.abs(W[:, I]) + np.abs(Bt) @ np.abs(Xv).T)
        return ([w, idx, bt, X], [w[:, idx] + pt.dot(bt, X.T)], [W, I, Bt, Xv], [W[:, I] + Bt @ Xv.T],
                ["take", "gemm"], "pointwise")
    # Gemm with z: 0.5 * z + 2 * dot(w[:, idx], X)
    n, q = 30, 6
    z = T("z", dtype)
    W, I, Xv, Z = _ints(rng, (B0, m)), _idx(rng, n, m), _ints(rng, (n, q)), _ints(rng, (B0, q))
    _fits(2 * (0.5 * np.abs(Z) + 2 * np.abs(W[:, I]) @ np.abs(Xv)))        # unit 0.5
    return ([w, idx, z, X], [0.5 * z + 2 * pt.dot(w[:, idx], X)], [W, I, Z, Xv], [0.5 * Z + 2 * (W[:, I] @ Xv)],
            ["take", "gemm"], "reduce")


def _form(node):
    red, pw = _has(node, r"\bgr\d+_0\b"), _has(node, r"\bga\d+_0\b")
    assert not (red and pw)
    return "reduce" if red else "pointwise" if pw else None


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("case", ["reduce", "pointwise", "gemm_z"])
def test_skinny_products(dtype, case):
    ins, outs, arrs, refs, kinds, form = _product_case(case, dtype, np.random.default_rng(2))
    arrs = [a.astype(dtype) if a.dtype == np.float64 else a for a in arrs]
    f, node = _run(ins, outs, arrs, [r.astype(dtype) for r in refs], kinds)
    assert _form(node) == form


def _np_put(x, y, idx):
    """x + sequential scatter-add of y's columns into zeros (j order), per row."""
    s = np.zeros_like(x)
    for j, k in enumerate(idx):
        s[:, k] += y[:, j]
    return x + s


@pytest.mark.parametrize("dtype", DT)
def test_scatter_add(dtype):
    rng = np.random.default_rng(3)
    m, n = 29, 70
    z, w, idx = T("z", dtype), T("w", dtype), T("idx", "int64", 1)
    Z, Wv, I = _ints(rng, (B0, m)), _ints(rng, (B0, n)), _idx(rng, n, m)
    ref = _np_put(Z, 2 * Wv, I)
    _fits(np.abs(Z) + _np_put(np.zeros_like(Z), 2 * np.abs(Wv), I))
    _run([z, w, idx], [pt.inc_subtensor(z[:, idx], 2 * w)], [Z.astype(dtype), Wv.astype(dtype), I], [ref.astype(dtype)],
         ["ew", "put"])


@pytest.mark.parametrize("dtype", DT)
def test_sums_over_the_batch(dtype):
    rng = np.random.default_rng(4)
    m, n = 31, 50
    w, idx = T("w", dtype), T("idx", "int64", 1)
    g = w[:, idx]
    W, I = _ints(rng, (B0, m)), _idx(rng, n, m)
    G = W[:, I]
    _fits(np.abs(G * 3).sum(axis=0))
    _fits(np.abs(G - 1).sum())
    _run([w, idx], [(g * 3).sum(axis=0), (g - 1).sum()], [W.astype(dtype), I],
         [(G * 3).sum(axis=0).astype(dtype), np.asarray((G - 1).sum()).astype(dtype)],
         ["take", "csum", "ew", "rsum", "csum"])


@pytest.mark.parametrize("dtype", DT)
def test_per_row_scalar_outputs(dtype):
    """A row sum as a (B,) output through a map and as a (B, 1) output (keepdims) through another."""
    rng = np.random.default_rng(5)
    m, n = 19, 40
    w, idx = T("w", dtype), T("idx", "int64", 1)
    g = w[:, idx]
    W, I = _ints(rng, (B0, m)), _idx(rng, n, m)
    S = W[:, I].sum(axis=1)
    f, node = _run([w, idx], [g.sum(axis=1) * 2 + 1, pt.sum(g, axis=1, keepdims=True) * 4], [W.astype(dtype), I],
                   [(S * 2 + 1).astype(dtype), (S[:, None] * 4).astype(dtype)], ["take", "rsum", "ew", "ew"])
    assert sorted(v.nd for v in node.plan.vals if v.out >= 0) == [1, 2]


@pytest.mark.parametrize("idt", ["int32", "int8"])
def test_narrow_index_dtypes(idt):
    rng = np.random.default_rng(6)
    m, n = 100, 77
    w, idx = T("w"), T("idx", idt, 1)
    W, I = _ints(rng, (B0, m)), _idx(rng, n, m, idt, neg=True)
    G = W[:, I]
    _run([w, idx], [(pt.abs(w[:, idx]) - 1).sum(axis=1)], [W.astype("float32"), I],
         [(np.abs(G) - 1).sum(axis=1).astype("float32")], ["take", "ew", "rsum"])


def _chain(dtype, rng, B=B0):
    """The shape of cfg5's backward pass: gather -> reduce-form product -> its finish -> map with a row sum ->
    scatter-add."""
    w, idx, X, z, jdx = T("w", dtype), T("idx", "int64", 1), T("X", dtype), T("z", dtype), T("jdx", "int64", 1)
    m, n, q, mz = 21, 40, 6, 11
    h = pt.dot(w[:, idx], X)
    out = pt.inc_subtensor(z[:, jdx], h - pt.abs(h).sum(axis=1, keepdims=True))
    W, I, Xv, Z, Jv = _ints(rng, (B, m)), _idx(rng, n, m), _ints(rng, (n, q), -3, 3), _ints(rng, (B, mz)), _idx(rng, q, mz)
    H = W[:, I] @ Xv
    Y = H - np.abs(H).sum(axis=1, keepdims=True)
    _fits(np.abs(W[:, I]) @ np.abs(Xv))
    _fits(2 * np.abs(H).sum(axis=1))
    _fits(np.abs(Z) + _np_put(np.zeros_like(Z), np.abs(Y), Jv))
    arrs = [W.astype(dtype), I, Xv.astype(dtype), Z.astype(dtype), Jv]
    return [w, idx, X, z, jdx], [out], arrs, [_np_put(Z, Y, Jv).astype(dtype)]


CHAIN_KINDS = ["take", "gemm", "ew", "rsum", "ew", "put"]


@pytest.mark.parametrize("dtype", DT)
def test_multi_level_chain(dtype):
    ins, outs, arrs, refs = _chain(dtype, np.random.default_rng(7))
    f, node = _run(ins, outs, arrs, refs, CHAIN_KINDS)
    assert _form(node) == "reduce"
    assert max(hit[0].n_loops for hit in node._kernels.values()) >= 3


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("stored", [False, True])
def test_gather_from_a_value_made_in_the_region(dtype, stored):
    """u = 2 w - 3 is gathered from: kept in the warp's shared-memory slab, or (when it is also an output) written to
    global memory and read back from there by the gather's loop."""
    rng = np.random.default_rng(8)
    m, n = 45, 60
    w, idx = T("w", dtype), T("idx", "int64", 1)
    u = w * 2 - 3
    W, I = _ints(rng, (B0, m)), _idx(rng, n, m, neg=True)
    U = W * 2 - 3
    outs, refs = [u[:, idx].sum(axis=1)], [U[:, I].sum(axis=1).astype(dtype)]
    if stored:
        outs, refs = [u] + outs, [U.astype(dtype)] + refs
    f, node = _run([w, idx], outs, [W.astype(dtype), I], refs, ["ew", "take", "rsum"])
    slab_gather = _has(node, r"= \(\w+\)\(sm\d+\[ix\d+\]\)")
    global_gather = _has(node, r"= \(\w+\)\(q\d+\[b \* \d+LL \+ \(ix\d+\)\]\)")
    assert (slab_gather, global_gather) == (not stored, stored)


# ---- b. sizes ----------------------------------------------------------------------------------------------------------
def _sms():
    if DRY:
        return 132
    from pytensor_b200.runtime import lib as _lib

    return _lib.sm_count()


def _map_graph(B, m, n, rng, dtype="float32"):
    w, idx = T("w", dtype), T("idx", "int64", 1)
    e = pt.abs(w[:, idx]) - 2
    W, I = _ints(rng, (B, m)), _idx(rng, n, m)
    E = np.abs(W[:, I]) - 2
    return [w, idx], [e, e.sum(axis=1)], [W.astype(dtype), I], [E.astype(dtype), E.sum(axis=1).astype(dtype)]


@pytest.mark.parametrize("B", [63, 64, 65, 203, "persistent"])
def test_batch_sizes(B):
    S = _sms()
    if B == "persistent":      # more rows than resident warps (8 CTAs of 8 warps per SM at most): warps take several rows
        B = S * 8 * 8 + 37
    ins, outs, arrs, refs = _map_graph(B, 33, 70, np.random.default_rng(9))
    f, node = _run(ins, outs, arrs, refs, ["take", "ew", "rsum"], fused=B >= 64, reason="batch of 63 rows")
    if B > 64 and not DRY:
        blocks = max(hit[3] for hit in node._kernels.values())
        assert blocks <= 8
        if B > S * 64:
            assert B > S * blocks * cg.WARPS


@pytest.mark.parametrize("d", [1, 31, 32, 33])
def test_domain_sizes(d):
    """Gather, map, scatter-add and row sum with every domain of size d (one partial iteration, one exact, one plus one)."""
    rng = np.random.default_rng(10)
    w, z, idx = T("w"), T("z"), T("idx", "int64", 1)
    y = w[:, idx] * 2 - 1
    W, Z, I = _ints(rng, (B0, d)), _ints(rng, (B0, d)), _idx(rng, d, d, neg=True)
    Y = W[:, I] * 2 - 1
    _run([w, idx, z], [pt.inc_subtensor(z[:, idx], y), y.sum(axis=1)], [W.astype("float32"), I, Z.astype("float32")],
         [_np_put(Z, Y, I).astype("float32"), Y.sum(axis=1).astype("float32")], ["take", "ew", "rsum", "put"])


@pytest.mark.parametrize("dtype,m", [("float32", 1024), ("float32", 1025), ("float64", 512), ("float64", 513)])
def test_staging_boundary(dtype, m):
    """A gathered source of at most STAGE_MAX_BYTES per row is copied to shared memory once per row."""
    rng = np.random.default_rng(11)
    w, idx = T("w", dtype), T("idx", "int64", 1)
    W, I = _ints(rng, (B0, m)), _idx(rng, 150, m)
    I[2:6] = [m - 2, 1, m - 1, m // 2]
    _fits(np.abs(W[:, I]).sum(axis=1))
    f, node = _run([w, idx], [w[:, idx].sum(axis=1), w[:, idx].max(axis=1)], [W.astype(dtype), I],
                   [W[:, I].sum(axis=1).astype(dtype), W[:, I].max(axis=1).astype(dtype)], ["take", "rsum", "rsum"])
    staged = m * np.dtype(dtype).itemsize <= cg.STAGE_MAX_BYTES
    assert _has(node, r"st\d+\[j\] = __ldg") == staged
    assert _has(node, r"\(st\d+\[ix\d+\]\)") == staged


@pytest.mark.parametrize("n", [8192, 8193])
def test_index_table_boundary(n):
    rng = np.random.default_rng(12)
    m = 50
    w, idx = T("w"), T("idx", "int64", 1)
    W, I = _ints(rng, (64, m)), _idx(rng, n, m, neg=True)
    G = W[:, I]
    _fits(np.abs(G).sum(axis=1))
    f, node = _run([w, idx], [w[:, idx].sum(axis=1)], [W.astype("float32"), I], [G.sum(axis=1).astype("float32")],
                   ["take", "rsum"])
    assert _has(node, r"\bcix0\[j\]") == (n * 4 <= cg.CTA_INDEX_MAX_BYTES)


@pytest.mark.parametrize("p,q,form", [(33, 16, "reduce"), (17, 16, "reduce"), (16, 16, "pointwise"),
                                      (32, 17, "pointwise"), (33, 17, None)])
def test_product_form_boundaries(p, q, form):
    rng = np.random.default_rng(13)
    ins, outs, arrs, refs, kinds, _ = _product_case("plain", "float32", rng, p, q)
    arrs = [a.astype("float32") if a.dtype == np.float64 else a for a in arrs]
    f, node = _run(ins, outs, arrs, [r.astype("float32") for r in refs], kinds, fused=form is not None,
                   reason="has no skinny side")
    if form:
        assert _form(node) == form


def test_fallback_domain_too_large():
    rng = np.random.default_rng(14)
    w, idx = T("w"), T("idx", "int64", 1)
    W, I = _ints(rng, (64, 40)), _idx(rng, 65537, 40)
    _run([w, idx], [w[:, idx].max(axis=1)], [W.astype("float32"), I], [W[:, I].max(axis=1).astype("float32")],
         ["take", "rsum"], fused=False, reason="domain size")


@pytest.mark.parametrize("m", [5120, 5124])
def test_shared_memory_budget(m):
    """A gathered in-region value of m fp32 per row takes 8 m * 4 bytes of slab: 160 KB exactly fits, 16 more bytes
    per warp send the node to its steps."""
    rng = np.random.default_rng(15)
    w, idx = T("w"), T("idx", "int64", 1)
    u = w * 2 - 3
    W, I = _ints(rng, (64, m)), _idx(rng, 300, m)
    U = W * 2 - 3
    fits = cg.WARPS * m * 4 <= cg.MAX_SMEM
    f, node = _run([w, idx], [u[:, idx].max(axis=1)], [W.astype("float32"), I], [U[:, I].max(axis=1).astype("float32")],
                   ["ew", "take", "rsum"], fused=fits, reason="bytes of shared memory")
    if fits:
        assert max(hit[0].smem_bytes for hit in node._kernels.values()) == cg.MAX_SMEM


# ---- c. fp64 scatter-add order -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dup", ["all_equal", "one_bin", "random"])
@pytest.mark.parametrize("n", [20, 64, 65, 95])
def test_fp64_scatter_add_is_sequential(dup, n):
    """y spans 12 decades, so the order of the adds shows in the low bits: the region output must equal x + s with s the
    scatter-add of y into zeros in j order (the C linker adds into x directly: equal within rounding)."""
    rng = np.random.default_rng(16 + n)
    m = {"all_equal": 9, "one_bin": 1, "random": 6}[dup]
    if dup == "all_equal":
        I = np.full(n, -4 if n % 2 else 5, dtype=np.int64)
    elif dup == "one_bin":
        I = np.zeros(n, dtype=np.int64)
    else:
        I = rng.integers(-m, m, n)
    x, y, idx = T("x", "float64"), T("y", "float64"), T("idx", "int64", 1)
    X = rng.standard_normal((B0, m))
    Y = rng.standard_normal((B0, n)) * 10.0 ** rng.uniform(-6, 6, (B0, n))
    ref = _np_put(X, Y, I % m)
    rev = _np_put(X, Y[:, ::-1], (I % m)[::-1])
    assert not np.array_equal(ref, rev), "the order of the adds does not show in these operands"
    out = pt.inc_subtensor(x[:, idx], y)
    f, node = _run([x, y, idx], [out], [X, Y, I], [ref], ["put"])
    if not DRY:
        exp = pytensor.function([x, y, idx], [out], mode="CVM")(X, Y, I)[0]
        scale = np.abs(X) + _np_put(np.zeros_like(X), np.abs(Y), I % m)
        assert np.all(np.abs(exp - ref) <= 1e-12 * scale)


def test_fp32_scatter_add_with_duplicates_on_the_grid():
    rng = np.random.default_rng(17)
    for n in (20, 65, 95):
        x, y, idx = T("x"), T("y"), T("idx", "int64", 1)
        X, Y, I = _ints(rng, (B0, 3)), _ints(rng, (B0, n)), rng.integers(-3, 3, n)
        _run([x, y, idx], [pt.inc_subtensor(x[:, idx], y)], [X.astype("float32"), Y.astype("float32"), I],
             [_np_put(X, Y, I % 3).astype("float32")], ["put"])


# ---- d. layouts ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["strided", "column_major", "column_slice_r0", "strided_index"])
def test_operand_layouts(layout):
    rng = np.random.default_rng(18)
    m, n = 26, 55
    idx = T("idx", "int64", 1)
    I = _idx(rng, n, m, neg=True)
    if layout == "strided":
        w2 = T("w2")
        W2 = _ints(rng, (2 * B0, 3 * m))
        W = W2[::2, ::3]
        ins, arrs, w = [w2, idx], [W2, I], w2[::2, ::3]
    elif layout == "column_major":
        wt = T("wt")
        W = _ints(rng, (B0, m))
        ins, arrs, w = [wt, idx], [np.ascontiguousarray(W.T), I], wt.T
    elif layout == "strided_index":
        w, i2 = T("w"), T("i2", "int64", 1)
        W = _ints(rng, (B0, m))
        I2 = np.stack([I, rng.integers(-1000, 1000, n)], axis=1).reshape(-1)    # every other entry is out of bounds
        ins, arrs, idx = [w, i2], [W, I2], i2[::2]
    else:
        w, s2 = T("w"), T("s2")
        W, S2 = _ints(rng, (B0, m)), _ints(rng, (B0, 3))
        ins, arrs = [w, s2, idx], [W, S2, I]
    g = w[:, idx]
    G = W[:, I]
    if layout == "column_slice_r0":
        s = pt.specify_broadcastable(s2[:, 1:2], 1)          # the rewrites take the (B, 1) factor out of the sum
        outs, refs, kinds = [(g * s).sum(axis=1)], [(G * S2[:, 1:2]).sum(axis=1)], ["take", "rsum", "ew"]
    else:
        outs, refs, kinds = [(g * 2).max(axis=1)], [(G * 2).max(axis=1)], ["take", "ew", "rsum"]
    arrs = [a.astype("float32") if a.dtype == np.float64 else a for a in arrs]
    f, node = _run(ins, outs, arrs, [r.astype("float32") for r in refs], kinds, device=True)
    strides = [e[1] for _, lay in node._kernels for e in lay]      # kernel key: (dims, ((grp, strides, ...), ...))
    want = {"strided": (2 * 3 * m, 3), "column_major": (1, B0), "strided_index": (2,), "column_slice_r0": (3,)}[layout]
    assert want in strides, strides


@pytest.mark.parametrize("dtype", DT)
def test_x_and_its_transpose_share_one_pointer_group(dtype):
    """h = dot(w[:, idx], X) (reduce form), then dot(h, X.T) (pointwise form): X and X.T are one kernel parameter."""
    rng = np.random.default_rng(19)
    m, n, q = 30, 40, 5
    w, idx, X = T("w", dtype), T("idx", "int64", 1), T("X", dtype)
    W, I, Xv = _ints(rng, (B0, m)), _idx(rng, n, m), _ints(rng, (n, q), -3, 3)
    H = W[:, I] @ Xv
    _fits(np.abs(np.abs(W[:, I]) @ np.abs(Xv)) @ np.abs(Xv).T)
    f, node = _run([w, idx, X], [pt.dot(pt.dot(w[:, idx], X), X.T)], [W.astype(dtype), I, Xv.astype(dtype)],
                   [(H @ Xv.T).astype(dtype)], ["take", "gemm", "gemm"], device=True)
    (dims, lay), = node._kernels                          # kernel key: (dims, ((grp, strides, offset, aligned), ...))
    mats = [e for e in lay if len(e[1]) == 2 and sorted(e[1]) == [1, q]]
    assert len(mats) == 2 and mats[0][0] == mats[1][0] and mats[0][1] != mats[1][1], lay
    assert _has(node, r"\bgr\d+_0\b") and _has(node, r"\bga\d+_0\b")


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("layout,vec", [("dense_q8", True), ("odd_pitch", False), ("misaligned_base", False),
                                        ("q_not_multiple_of_4", False)])
def test_matrix_loads(dtype, layout, vec):
    """float4 / double2 loads only for an aligned contiguous run of whole vectors; otherwise one load per element."""
    rng = np.random.default_rng(20)
    m, n = 25, 39
    w, idx, xb = T("w", dtype), T("idx", "int64", 1), T("xb", dtype)
    q, width, sl = {"dense_q8": (8, 8, None), "odd_pitch": (8, 9, (slice(None), slice(None, 8))),
                    "misaligned_base": (8, 9, (slice(None), slice(1, None))), "q_not_multiple_of_4": (5, 5, None)}[layout]
    Xb = _ints(rng, (n, width))
    Xv = Xb[sl] if sl else Xb
    X = xb[sl] if sl else xb
    W, I = _ints(rng, (B0, m)), _idx(rng, n, m)
    _fits(np.abs(W[:, I]) @ np.abs(Xv))
    f, node = _run([w, idx, xb], [pt.dot(w[:, idx], X)], [W.astype(dtype), I, Xb.astype(dtype)],
                   [(W[:, I] @ Xv).astype(dtype)], ["take", "gemm"], device=True)
    assert _form(node) == "reduce"
    assert _has(node, r"float4|double2") == vec
    assert _has(node, r"\bms\d+_0\b") == (not vec)


# ---- e. special values and errors ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT)
def test_nonfinite_values(dtype):
    """NaN / ±inf planted in a gathered source (row add / max / min) and in scattered values: NumPy's pattern exactly."""
    rng = np.random.default_rng(21)
    m, n = 35, 70
    w, z, y, idx = T("w", dtype), T("z", dtype), T("y", dtype), T("idx", "int64", 1)
    W, Z, Y, I = _ints(rng, (B0, m)), _ints(rng, (B0, m)), _ints(rng, (B0, n)), _idx(rng, n, m)
    specials = np.array([np.nan, np.inf, -np.inf])
    rows = np.arange(B0)
    live = rows % 7 != 6                                     # some rows keep only finite values
    W[rows[live], rng.integers(0, m, live.sum())] = specials[rows[live] % 3]
    two = rows % 5 == 0                                      # a second plant: +inf with -inf, NaN with ±inf
    W[rows[two], rng.integers(0, m, two.sum())] = specials[(rows[two] + 1) % 3]
    Y[rows[live], rng.integers(0, n, live.sum())] = specials[(rows[live] + 2) % 3]
    g = w[:, idx]
    G = W[:, I]
    with np.errstate(invalid="ignore"):
        refs = [G.sum(axis=1), G.max(axis=1), G.min(axis=1), _np_put(Z, Y, I)]
    for r in (refs[0], refs[3]):
        assert np.isnan(r).any() and np.isposinf(r).any() and np.isneginf(r).any()
    assert np.isnan(refs[1]).any() and np.isposinf(refs[1]).any() and np.isnan(refs[2]).any() and np.isneginf(refs[2]).any()
    _run([w, idx], [g.sum(axis=1), g.max(axis=1), g.min(axis=1)], [W.astype(dtype), I],
         [r.astype(dtype) for r in refs[:3]], ["take", "rsum", "rsum", "rsum"])
    _run([z, y, idx], [pt.inc_subtensor(z[:, idx], y)], [Z.astype(dtype), Y.astype(dtype), I], [refs[3].astype(dtype)],
         ["put"])


@pytest.mark.parametrize("path,idt", [("table", "int64"), ("table", "int32"), ("per_use", "int64"), ("per_use", "int32")])
@pytest.mark.parametrize("bad", ["too_large", "too_negative"])
def test_out_of_bounds_index_raises(monkeypatch, path, idt, bad):
    _needs_device()
    if path == "per_use":   # read when the source is generated: a new function builds a new kernel
        monkeypatch.setenv("PTK_ROWFUSE_CTA_INDEX", "0")
    rng = np.random.default_rng(22)
    m, n = 40, 90
    w, z, idx = T("w"), T("z"), T("idx", idt, 1)
    g = w[:, idx]
    f = pytensor.function([w, z, idx], [g.sum(axis=1), pt.inc_subtensor(z[:, idx], g)], mode="CUDA")
    node = _region(f)
    W, Z, I = _ints(rng, (B0, m)).astype("float32"), _ints(rng, (B0, m)).astype("float32"), _idx(rng, n, m, idt, neg=True)
    f(W, Z, I)                                              # in bounds, negative indices wrap
    assert node.fused_calls == 1 and node.unfused_calls == 0, node.last_reason
    assert _has(node, r"\bcix0\[j\]") == (path == "table")
    I_bad = I.copy()
    I_bad[n // 2] = m if bad == "too_large" else -m - 1
    with pytest.raises(IndexError):
        f(W, Z, I_bad)
    assert node.fused_calls == 2 and node.unfused_calls == 0


# ---- f. replay ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DT)
def test_replay_with_device_inputs_and_outputs(dtype):
    _needs_device()
    import torch

    from pytensor_b200.link.cuda import cuda_mode

    cases = [_chain(dtype, np.random.default_rng(23 + k)) for k in range(2)]
    ins, outs = cases[0][0], cases[0][1]
    f = pytensor.function(ins, outs, mode=cuda_mode(device_outputs=True), trust_input=True)
    node = _region(f)
    assert [o.kind for o in node.plan.ops] == CHAIN_KINDS
    dev_sets = [[torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in c[2]] for c in cases]
    for call in range(6):
        k = call % 2
        got = f(*dev_sets[k])
        for j, (g, e) in enumerate(zip(got, cases[k][3])):
            _same(g.cpu().numpy(), e, f"call {call} on set {k}, output {j}")
    assert f.vm.executor.last_from_graph, "the last call did not replay a captured graph"
    assert node.fused_calls >= 2 and node.unfused_calls == 0, node.last_reason
