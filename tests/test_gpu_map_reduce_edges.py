"""The fused map + row-reduce kernel (K3: codegen/careduce.py `gen_row_kernel` / `gen_row_kernel_tma`, launched by
vm/nodes_elemwise.py `ElemwiseReduceNode`) and the split paths of the CAReduce kernels, at their edges.

a. Integer grid: integer-valued inputs from small ranges and a map built from operations that are exact on them
   (+ - *, maximum, abs, sqr, switch, comparisons, casts), so every map value is exact and the fp64 accumulator sums
   them exactly: a stored map output must equal NumPy bit for bit and the reduction must equal the exact row sum
   rounded once.  Every row carries an adjacent +G pair and an adjacent -G pair (G = 3 * 2^22; G + G exceeds 2^24):
   the exact sum does not see them, an fp32 running sum or an fp32 pre-sum of a vector's lanes does.
b. Launch regimes derived from the SM count S: 32 threads per row (TPR) for cols < 1024, 128 for 1 K <= cols < 16 K
   with at least 8 S rows, 256 otherwise; fewer row blocks than SMs falls back to the two-kernel path; more rows than
   the resident CTAs hold makes every CTA stride over several row blocks.
c. NaN / ±inf / the row extreme planted at every position where a vector, a thread's stride or the tail starts or
   ends: max, min, sum and prod match the C linker exactly, NaN pattern included.
d. The transcendental cfg2 map: e against the C linker at 1e-5 on a row slice, r against an exact sum of the kernel's
   own stored e (|r - fsum(e)| <= 1 ulp32(r) + n 2^-52 sum|e|, independent of libm).
e. Every load scheme (PTK_K3_PIPE none / l2 / regs / tma, PTK_K3_ADDR=idx, PTK_K3_MINB 4 / 6) accumulates in the same
   order with the same combine tree: for each forced TPR their results must be bit-identical.
f. Every K3 function is called six times on two alternating input sets (eager, capture, replay of each) in the mode
   the benchmark uses (device inputs and outputs), and every call must return its own input's result.
g. CAReduce row kernel split over blocks (nsplit up to 4 S, finished by the warp-per-output kernel's lane loop), the
   split column kernel, and the scalar-load (vw = 1) row kernel of a misaligned slice, on the integer grid.

Every K3 test asserts that the graph ran the fused kernel with the intended (in_modes, vw, tpr, store, tma) key and
never fell back; the fallback cases assert the opposite."""

import math

import numpy as np
import pytest

from helpers import pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu

G = 3 << 22
SCHEMES = [("none", {}), ("l2", {"PTK_K3_PIPE": "l2"}), ("regs", {"PTK_K3_PIPE": "regs"}), ("tma", {"PTK_K3_PIPE": "tma"}),
           ("idx", {"PTK_K3_ADDR": "idx"}), ("minb4", {"PTK_K3_MINB": "4"}), ("minb6", {"PTK_K3_MINB": "6"})]
K3_ENV = ("PTK_K3_PIPE", "PTK_K3_ADDR", "PTK_K3_MINB", "PTK_K3_TPR")


# ---- fixtures and harness ----------------------------------------------------------------------------------------------
@pytest.fixture
def fallbacks(gpu, monkeypatch):
    """Records every ElemwiseReduceNode that ran its two constituent kernels instead of the fused one; K3 switches are
    cleared so that each test starts from the default scheme."""
    if not gpu:
        pytest.skip("runs the fused kernel on the device")
    from pytensor_b200.vm.nodes_elemwise import ElemwiseReduceNode

    for v in K3_ENV:
        monkeypatch.delenv(v, raising=False)
    calls = []
    given, unfused = ElemwiseReduceNode._unfused_given, ElemwiseReduceNode._unfused

    def rec_given(self, vals, ins, outs):
        calls.append(self)
        return given(self, vals, ins, outs)

    def rec_unfused(self, vals):
        calls.append(self)
        return unfused(self, vals)

    monkeypatch.setattr(ElemwiseReduceNode, "_unfused_given", rec_given)
    monkeypatch.setattr(ElemwiseReduceNode, "_unfused", rec_unfused)
    return calls


def _sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _compile(ins, outs):
    from pytensor_b200.link.cuda import cuda_mode

    return pytensor.function(ins, outs, mode=cuda_mode(device_outputs=True), trust_input=True)


def _alternate(f, sets, calls=6):
    """Host copies of f's results over `calls` calls alternating between the input sets: [(set index, outputs)]."""
    import torch

    dev_sets = [[torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in s] for s in sets]
    res = []
    for i in range(calls):
        k = i % len(sets)
        outs = f(*dev_sets[k])
        res.append((k, [o.cpu().numpy() for o in outs]))
    if calls >= 2 * len(sets) + 1:
        assert f.vm.executor.last_from_graph, "the last call did not replay a captured graph"
    return res


def _k3_node(f):
    from pytensor_b200.vm.nodes_elemwise import ElemwiseReduceNode

    steps = f.vm.executor.program.steps
    nodes = [st.impl for st in steps if isinstance(st.impl, ElemwiseReduceNode)]
    assert len(nodes) == 1, [type(st.impl).__name__ for st in steps]
    return nodes[0]


def _assert_fused(f, fallbacks, **want):
    """The fused kernel ran, only with keys matching `want` (in_modes / vw / tpr / store / tma), and nothing fell back."""
    node = _k3_node(f)
    assert not fallbacks, "the graph fell back to the unfused two-kernel path"
    assert node._kernels, "no fused kernel was launched"
    for in_modes, vw, tpr, store, tma in node._kernels:
        got = dict(in_modes=in_modes, vw=vw, tpr=tpr, store=store, tma=tma)
        assert all(got[k] == v for k, v in want.items()), (got, want)
    return node


def _same(got, exp, what=""):
    """Bit-exact up to the NaN payload: equal values, equal signs of zero, NaN where NaN."""
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.dtype == exp.dtype and got.shape == exp.shape, (what, got.dtype, exp.dtype, got.shape, exp.shape)
    if exp.dtype.kind == "f":
        bad = ~((got == exp) & (np.signbit(got) == np.signbit(exp)) | (np.isnan(got) & np.isnan(exp)))
    else:
        bad = got != exp
    if bad.any():
        idx = np.argwhere(bad)[:5]
        raise AssertionError(f"{what}: {int(bad.sum())} of {exp.size} differ; first {idx.tolist()}: "
                             f"got {[got[tuple(i)] for i in idx]} expected {[exp[tuple(i)] for i in idx]}")


def _check(res, refs):
    for k, got in res:
        assert len(got) == len(refs[k])
        for j, (g, e) in enumerate(zip(got, refs[k])):
            _same(g, e, f"call on set {k}, output {j}")


# ---- integer grid ------------------------------------------------------------------------------------------------------
def _plant_cancelling(rng, c):
    """An adjacent +G pair and an adjacent -G pair, each starting at an even column, in every row of the last axis (rows of
    at least 8)."""
    c2 = c.reshape(-1, c.shape[-1])
    n = c2.shape[1]
    if n < 8:
        return
    m = n // 2 - 1                                   # pair starts 0, 2, ..., 2 (m - 1)
    s1 = rng.integers(0, m, c2.shape[0])
    s2 = (s1 + rng.integers(1, m, c2.shape[0])) % m
    i = np.arange(c2.shape[0])
    for s, v in ((s1, G), (s2, -G)):
        c2[i, 2 * s] = v
        c2[i, 2 * s + 1] = v


def _grid_sets(shape, dtype="float32", seed=0, n=2):
    """`n` input sets (a, b, c) on the integer grid, as the given float dtype and as int32."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        a = rng.integers(-8, 9, shape, dtype=np.int32)
        b = rng.integers(-4, 5, shape, dtype=np.int32)
        c = rng.integers(-8, 9, shape, dtype=np.int32)
        _plant_cancelling(rng, c)
        out.append(([x.astype(dtype) for x in (a, b, c)], (a, b, c)))
    return out


def _grid_map_pt(a, b, c):
    return pt.switch(a > b, a * b, pt.maximum(pt.sqr(b) - a, pt.abs(a) - b)) + c


def _grid_map_np(a, b, c):
    return np.where(a > b, a * b, np.maximum(b * b - a, np.abs(a) - b)) + c


def _grid_graph(ndim, dtype, sl, store):
    a, b, c = (pt.tensor(n, dtype=dtype, shape=(None,) * ndim) for n in "abc")
    e = _grid_map_pt(*((x[sl] if sl is not None else x) for x in (a, b, c)))
    r = e.sum(axis=tuple(range(1, ndim)))
    return [a, b, c], ([e, r] if store else [r])


def _grid_refs(sets, dtype, sl, store):
    refs = []
    for _, ints in sets:
        e = _grid_map_np(*((x[sl] if sl is not None else x) for x in ints))
        r = e.reshape(e.shape[0], -1).sum(axis=1, dtype=np.int64)   # exact
        assert np.all(np.abs(e) < 2 ** 24)
        refs.append(([e.astype(dtype)] if store else []) + [r.astype(np.float64).astype(dtype)])
    return refs


def _run_grid(fallbacks, shape, dtype="float32", sl=None, stored=True, calls=6, **want):
    """The integer-grid graph on two input sets of `shape`; `want`: the expected kernel key, or tpr=None for a graph
    that must take the two-kernel fallback."""
    ins, outs = _grid_graph(len(shape), dtype, sl, stored)
    sets = _grid_sets(shape, dtype)
    f = _compile(ins, outs)
    res = _alternate(f, [s for s, _ in sets], calls)
    if want.get("tpr", 0) is None:
        node = _k3_node(f)
        assert fallbacks, "expected the two-kernel fallback"
    else:
        node = _assert_fused(f, fallbacks, **want)
    _check(res, _grid_refs(sets, dtype, sl, stored))
    return f, node


def _regime(cols, S):
    """(rows, expected TPR) that put `cols` into its natural regime."""
    if cols < 1024:
        return 8 * S + 3, 32
    if cols < 16384:
        return 8 * S + 1, 128
    return S + 1, 256


@pytest.mark.parametrize("cols", [1, 3, 4, 5, 31, 33, 127, 1000, 1023, 1024, 1028, 4096, 16383, 16384, 70001])
def test_integer_grid_in_its_regime(fallbacks, cols):
    rows, tpr = _regime(cols, _sms())
    if cols == 1:
        tpr = None      # one column collapses to a broadcast-like stride 0 for every operand: the two-kernel path
    _run_grid(fallbacks, (rows, cols), tpr=tpr, vw=4 if cols % 4 == 0 else 1, store=(True,), in_modes=(1, 1, 1),
              tma=False)


# rows = m * S + d
@pytest.mark.parametrize("cols,m,d,tpr", [
    (1028, 1, 0, 256), (4096, 8, -1, 256),        # 1 K <= cols < 16 K with S <= rows < 8 S
    (16384, 8, 1, 256),                           # long rows of tall matrices stay at 256
    (1028, 1, -1, None), (100, 8, -8, None),      # fewer row blocks than SMs: two kernels
])
def test_integer_grid_tpr256_and_fallback(fallbacks, cols, m, d, tpr):
    _run_grid(fallbacks, (m * _sms() + d, cols), calls=2, tpr=tpr, vw=4, store=(True,))


@pytest.mark.parametrize("cols,tpr", [(100, 32), (1028, 128), (16384, 256)])
def test_integer_grid_persistent_striding(fallbacks, cols, tpr):
    """More row blocks than resident CTAs (rows > S * occupancy * rows per block, not a multiple of rows per block):
    every CTA strides over several row blocks and the last block is partial."""
    S, rpb = _sms(), 256 // tpr
    rows = 9 * S * rpb + 1                   # resident CTAs per SM are at most 2048 / 256 = 8
    _, node = _run_grid(fallbacks, (rows, cols), calls=3, tpr=tpr, vw=4, store=(True,))
    occ = max(node._occupancy.values())
    assert rows > S * occ * rpb, (rows, S, occ, rpb)


@pytest.mark.parametrize("name,width,sl,vw,stored", [
    ("misaligned_base", 1001, (slice(None), slice(1, None)), 1, False),   # 4-byte offset: scalar loads
    ("misaligned_base_stored", 1001, (slice(None), slice(1, None)), 1, True),
    ("odd_pitch", 1001, (slice(None), slice(None, 1000)), 1, False),       # aligned base, row pitch 1001
    ("vector_tail", 1024, (slice(None), slice(None, 1001)), 4, False),     # 250 vectors + 1 tail element per row
    ("no_full_vector", 8, (slice(None), slice(None, 3)), 4, False),        # cols < vw: the tail loop alone
])
def test_integer_grid_layouts(fallbacks, name, width, sl, vw, stored):
    _run_grid(fallbacks, (8 * _sms() + 3, width), sl=sl, stored=stored, tpr=32, vw=vw, in_modes=(1, 1, 1),
              store=(stored,))


def test_integer_grid_3d_collapses_to_columns(fallbacks):
    # (rows, 7, 152): the reduced axes (1, 2) collapse to 1064 contiguous columns
    _run_grid(fallbacks, (8 * _sms() + 1, 7, 152), tpr=128, vw=4, store=(True,), in_modes=(1, 1, 1))


def test_integer_grid_non_collapsible_slice_falls_back(fallbacks):
    # (rows, 7, 152)[:, :, :150]: the reduced axes have strides 152 and 1 over 7 x 150 -- not one run of columns
    _run_grid(fallbacks, (8 * _sms() + 1, 7, 152), sl=(slice(None), slice(None), slice(None, 150)), tpr=None)


def test_operand_modes_column_row_and_constant(fallbacks):
    """A (rows, 1) operand (one value per row), a (1, cols) operand (row stride 0) and constants."""
    S = _sms()
    rows, cols = 8 * S + 3, 1028
    a = pt.fmatrix("a")
    x = pt.tensor("x", dtype="float32", shape=(None, 1))
    y = pt.tensor("y", dtype="float32", shape=(1, None))
    kc = (np.arange(cols) % 7 - 3).astype("float32")[None, :]
    e = pt.switch(a > x, a + y, a - pt.abs(x)) + pt.constant(kc) + np.float32(3)
    f = _compile([a, x, y], [e, e.sum(axis=1)])
    rng = np.random.default_rng(3)
    sets, refs = [], []
    for _ in range(2):
        ai = rng.integers(-8, 9, (rows, cols))
        _plant_cancelling(rng, ai)
        xi, yi = rng.integers(-8, 9, (rows, 1)), rng.integers(-4, 5, (1, cols))
        ei = np.where(ai > xi, ai + yi, ai - np.abs(xi)) + kc.astype(np.int64) + 3
        sets.append([v.astype("float32") for v in (ai, xi, yi)])
        refs.append([ei.astype("float32"), ei.sum(axis=1).astype("float32")])
    _check(_alternate(f, sets), refs)
    node = _assert_fused(f, fallbacks, tpr=128, vw=4, store=(True,))
    (in_modes, *_), = node._kernels
    assert 0 in in_modes and in_modes.count(1) >= 2, in_modes


def _multi_graph(kind):
    """A two- or three-output Elemwise, one of whose outputs is reduced."""
    a, b, c = (pt.fmatrix(n) for n in "abc")
    e0 = a * b + c
    e1 = pt.maximum(e0, pt.abs(c)) - b
    e2 = pt.sqr(b) - e0
    r = e1.sum(axis=1)
    outs = {"reduced_not_stored": [e0, r], "reduced_stored": [e0, e1, r], "several_stored": [e2, e0, r],
            "not_first_and_stored": [e2, e0, e1, r]}[kind]
    return [a, b, c], outs


def _multi_ref(kind, a, b, c):
    e0 = a * b + c
    e1 = np.maximum(e0, np.abs(c)) - b
    e2 = b * b - e0
    r = e1.sum(axis=1).astype(np.float64).astype("float32")
    f32 = np.float32
    return {"reduced_not_stored": [e0.astype(f32), r], "reduced_stored": [e0.astype(f32), e1.astype(f32), r],
            "several_stored": [e2.astype(f32), e0.astype(f32), r],
            "not_first_and_stored": [e2.astype(f32), e0.astype(f32), e1.astype(f32), r]}[kind]


@pytest.mark.parametrize("kind", ["reduced_not_stored", "reduced_stored", "several_stored", "not_first_and_stored"])
def test_multi_output_elemwise(fallbacks, kind):
    rows = 8 * _sms() + 1
    ins, outs = _multi_graph(kind)
    f = _compile(ins, outs)
    sets = _grid_sets((rows, 1028))
    _check(_alternate(f, [s for s, _ in sets]), [_multi_ref(kind, *ints) for _, ints in sets])
    node = _assert_fused(f, fallbacks, tpr=128, vw=4)
    assert node.ew.n_out >= 2
    assert node.store_reduced_input == (kind in ("reduced_stored", "not_first_and_stored"))
    if kind in ("several_stored", "not_first_and_stored"):
        assert node.which != 0, "the reduced map output is output 0 of the Elemwise"



def test_inplace_elemwise_on_an_intermediate(fallbacks):
    """The map overwrites its input, a Join result nothing else reads (a destroyed intermediate)."""
    rows = 8 * _sms() + 3
    a, b = pt.fmatrix("a"), pt.fmatrix("b")
    j = pt.concatenate([a, b], axis=1)
    e = pt.sqr(j) - j * np.float32(3)
    f = _compile([a, b], [e, e.sum(axis=1)])
    sets, refs = [], []
    rng = np.random.default_rng(5)
    for _ in range(2):
        ai, bi = rng.integers(-50, 51, (rows, 500)), rng.integers(-50, 51, (rows, 500))
        ji = np.concatenate([ai, bi], axis=1)
        ei = ji * ji - 3 * ji
        sets.append([ai.astype("float32"), bi.astype("float32")])
        refs.append([ei.astype("float32"), ei.sum(axis=1).astype("float32")])
    _check(_alternate(f, sets), refs)
    node = _assert_fused(f, fallbacks, tpr=32, vw=4)
    assert node.ew.inplace, "the Elemwise is not in place"


# ---- dtypes ------------------------------------------------------------------------------------------------------------
def test_float64_grid_with_32_byte_vectors_never_takes_tma(fallbacks, monkeypatch):
    monkeypatch.setenv("PTK_K3_PIPE", "tma")
    _run_grid(fallbacks, (8 * _sms() + 1, 1028), dtype="float64", tpr=128, vw=4, tma=False, store=(True,))


def test_tma_staging_of_three_inputs_takes_the_plain_kernel(fallbacks, monkeypatch):
    # three streamed inputs would need 3 x 4 stages x 256 x 16 B = 48 KiB of staging plus the mbarriers: more static
    # shared memory than a kernel may declare
    monkeypatch.setenv("PTK_K3_PIPE", "tma")
    _run_grid(fallbacks, (8 * _sms() + 1, 1028), tpr=128, vw=4, tma=False, store=(True,), in_modes=(1, 1, 1))


def _cvm(ins, outs, arrays):
    return pytensor.function(ins, outs, mode="CVM")(*[np.array(x, copy=True) for x in arrays])


def test_int8_map_sums_into_int64_with_wraparound(fallbacks):
    rows = 8 * _sms() + 3
    a, b = pt.bmatrix("a"), pt.bmatrix("b")
    e = a * b + np.int8(7)                      # wraps in int8, like the C linker's expression
    r = e.sum(axis=1)                           # int64 accumulator and result
    assert r.dtype == "int64"
    f = _compile([a, b], [e, r])
    rng = np.random.default_rng(7)
    sets = [[rng.integers(-128, 128, (rows, 1008)).astype("int8") for _ in range(2)] for _ in range(2)]
    refs = [_cvm([a, b], [e, r], s) for s in sets]
    for s, ref in zip(sets, refs):
        wrapped = (s[0].astype(np.int64) * s[1] + 7).astype(np.int8)
        _same(ref[0], wrapped, "C linker vs NumPy int8")
    _check(_alternate(f, sets), refs)
    _assert_fused(f, fallbacks, tpr=32, vw=16, store=(True,))


@pytest.mark.parametrize("op", ["all", "any"])
def test_bool_all_any_of_a_comparison(fallbacks, op):
    S = _sms()
    rows, cols = 8 * S + 1, 1028
    a, b = pt.fmatrix("a"), pt.fmatrix("b")
    r = getattr(pt, op)(a > b, axis=1)
    f = _compile([a, b], [r])
    rng = np.random.default_rng(8)
    sets = []
    for _ in range(2):
        bv = rng.integers(-8, 9, (rows, cols)).astype("float32")
        av = bv + (1 if op == "all" else 0)                      # all rows true (all) / all rows false (any) ...
        flip = np.arange(rows) % 3 != 0                          # ... except one element in two rows of three
        pos = np.array([0, 3, 4, 511, 512, 1023, 1024, 1027])[np.arange(rows) % 8]
        av[flip, pos[flip]] += -1 if op == "all" else 1
        sets.append([av, bv])
    refs = [[getattr(np, op)(s[0] > s[1], axis=1)] for s in sets]
    for s, ref in zip(sets, refs):
        _same(_cvm([a, b], [r], s)[0], ref[0], "C linker vs NumPy")
    _check(_alternate(f, sets), refs)
    _assert_fused(f, fallbacks, tpr=128, store=(False,))


def test_int32_input_with_a_float32_map(fallbacks):
    rows = 8 * _sms() + 3
    i, x = pt.imatrix("i"), pt.fmatrix("x")
    e = pt.cast(i, "float32") * x - pt.cast(i > 0, "float32")
    r = e.sum(axis=1)
    assert e.dtype == "float32"
    f = _compile([i, x], [e, r])
    rng = np.random.default_rng(9)
    sets, refs = [], []
    for _ in range(2):
        iv = rng.integers(-1000, 1001, (rows, 1000))
        xv = rng.integers(-8, 9, (rows, 1000))
        _plant_cancelling(rng, iv)                               # (G * x stays below 2^24 only for |x| = 1)
        xv[np.abs(iv) == G] = 1
        ev = iv.astype("float32") * xv.astype("float32") - (iv > 0).astype("float32")   # exact; 0 * -3 is -0
        sets.append([iv.astype("int32"), xv.astype("float32")])
        refs.append([ev, ev.astype(np.float64).sum(axis=1).astype("float32")])
    _check(_alternate(f, sets), refs)
    _assert_fused(f, fallbacks, tpr=32, vw=4, store=(True,))


# ---- non-finite values, max / min / sum / prod -------------------------------------------------------------------------
def _planted_positions(cols, vw, tpr):
    ncv = cols // vw
    pos = [0, vw - 1, vw, tpr * vw - 1, tpr * vw, 2 * tpr * vw, ncv * vw - vw, ncv * vw - 1]
    pos += list(range(ncv * vw, cols)) + [cols - 1]
    return sorted({p for p in pos if 0 <= p < cols})


@pytest.mark.parametrize("red", ["max", "min", "sum", "prod"])
@pytest.mark.parametrize("tpr,width,cols", [(32, 1004, 1001), (128, 4100, 4099), (256, 16388, 16387)])
def test_nonfinite_and_extremes_match_the_c_linker(fallbacks, red, tpr, width, cols):
    """Factors ±0.5 / ±1 / ±2 keep every sum and product exact; NaN, ±inf or the row extreme planted where vectors,
    thread strides and the tail begin and end (one or two plants per row)."""
    S = _sms()
    rows = S + 1 if tpr == 256 else 8 * S + 3
    a, b = pt.fmatrix("a"), pt.fmatrix("b")
    r = getattr(pt, red)(a[:, :cols] * b[:, :cols], axis=1)
    f = _compile([a, b], [r])
    pos = _planted_positions(cols, 4, tpr)
    extreme = {"max": 100.0, "min": -100.0, "sum": 2.0 ** 20, "prod": 0.0}[red]
    kinds = [np.nan, np.inf, -np.inf, extreme]
    rng = np.random.default_rng(10)
    sets = []
    for _ in range(2):
        # mostly ±1: a row's product stays far inside the float32 range in every order
        av = rng.choice(np.float32([0.5, 1, 2, -0.5, -1, -2]), (rows, width), p=[0.01, 0.48, 0.01, 0.01, 0.48, 0.01])
        bv = rng.choice(np.float32([1, -1]), (rows, width))
        i = np.arange(rows)
        p, k = i % len(pos), (i // len(pos)) % len(kinds)
        live = i % 11 != 10                                      # some rows keep no plant
        av[i[live], np.take(pos, p[live])] = np.take(kinds, k[live])
        two = i % 5 == 0                                         # a second plant: +inf with -inf, NaN with an extreme
        av[i[two], np.take(pos, (p[two] + len(pos) // 2) % len(pos))] = np.take(kinds, (k[two] + 1) % len(kinds))
        sets.append([av, bv])
    refs = [_cvm([a, b], [r], s) for s in sets]
    _check(_alternate(f, sets), refs)
    _assert_fused(f, fallbacks, tpr=tpr, vw=4, store=(False,))


# ---- transcendental map: cfg2 ------------------------------------------------------------------------------------------
def _cfg2():
    a, b = pt.fmatrix("a"), pt.fmatrix("b")
    e = a
    for c in [0.5, -0.25, 0.125, 0.75]:
        e = (e * b + np.float32(c)) * np.float32(0.9)
        e = pt.maximum(e, -e) + pt.sqr(a) * np.float32(0.1)
    e = pt.tanh(e * np.float32(0.01)) + pt.exp(-pt.abs(b))
    return [a, b], [e, e.sum(axis=1)]


def _cfg2_sets(rows, cols, n=2, seed=1):
    rng = np.random.default_rng(seed)
    return [[rng.standard_normal((rows, cols)).astype("float32") for _ in range(2)] for _ in range(n)]


def _assert_sum_bound(e, r):
    """|r - fsum(e_row)| <= 1 ulp32(r) + n 2^-52 sum|e_row| for every row."""
    e64 = e.astype(np.float64)
    exact = np.array([math.fsum(row.tolist()) for row in e64])
    n = e.shape[1]
    bound = np.spacing(np.abs(r)).astype(np.float64) + n * 2.0 ** -52 * np.abs(e64).sum(axis=1)
    err = np.abs(r.astype(np.float64) - exact)
    assert np.all(err <= bound), (float(np.max(err / bound)), int(np.argmax(err / bound)))


def _run_cfg2(fallbacks, rows, cols, calls=6, slice_rows=64, **want):
    ins, outs = _cfg2()
    f = _compile(ins, outs)
    sets = _cfg2_sets(rows, cols)
    res = _alternate(f, sets, calls)
    node = _assert_fused(f, fallbacks, **want)
    f_ref = pytensor.function(ins, outs, mode="CVM")
    ref_e = [f_ref(*[x[:slice_rows] for x in s])[0] for s in sets]    # rows are independent: the C linker on a slice
    for k, (e, r) in res:
        assert e.dtype == np.float32 and r.dtype == np.float32
        np.testing.assert_allclose(e[:slice_rows], ref_e[k], rtol=1e-5, atol=1e-5)
    for k in range(len(sets)):                                          # one bound check per input set
        e, r = next(got for kk, got in res if kk == k)
        _assert_sum_bound(e, r)
        for kk, (e2, r2) in res:
            if kk == k:
                _same(e2, e, "e across calls")
                _same(r2, r, "r across calls")
    return f, node, res


@pytest.mark.parametrize("m,d,cols,tpr", [(8, 3, 1000, 32), (8, 1, 1028, 128), (1, 1, 16384, 256),
                                         (0, 4096, 4096, 128)])         # rows = m * S + d; the last is cfg2 itself
def test_cfg2_map_in_each_regime(fallbacks, m, d, cols, tpr):
    _run_cfg2(fallbacks, m * _sms() + d, cols, calls=6 if cols < 4096 else 3, tpr=tpr, vw=4, store=(True,))


# ---- every load scheme computes the same bits --------------------------------------------------------------------------
def _schemes_for(tpr):
    return [(name, env) for name, env in SCHEMES if not (name == "tma" and tpr < 64)]


@pytest.mark.parametrize("tpr", [32, 64, 128, 256])
def test_load_schemes_are_bit_identical(fallbacks, monkeypatch, tpr):
    """Forced TPR, persistent striding (more row blocks than resident CTAs), odd trip counts: the integer grid with a
    vector tail (exact) and cfg2 with a stored e (bounded), both bit-identical across every load scheme."""
    S, rpb = _sms(), 256 // tpr
    rows = 8 * S * rpb + 3
    ncv = 5 * tpr // 2 + 3                     # two double trips, then part of the lanes take one more vector
    cols = 4 * ncv
    monkeypatch.setenv("PTK_K3_TPR", str(tpr))
    sl = (slice(None), slice(None, cols + 3))  # + 3 tail elements, row pitch cols + 4
    grid_sets, grid_refs = [], []
    for (_, (ai, bi, ci)) in _grid_sets((rows, cols + 4)):
        ai = np.where(np.abs(ci) == G, ci, ai)                    # the cancelling pairs, carried by a
        ei = np.where(np.abs(ai) > 64, ai, ai * bi + bi * bi)[sl]
        grid_sets.append([ai.astype("float32"), bi.astype("float32")])
        grid_refs.append([ei.sum(axis=1, dtype=np.int64).astype(np.float64).astype("float32")])
    cfg_sets = _cfg2_sets(rows, cols)
    first = None
    for name, env in _schemes_for(tpr):
        for v in K3_ENV[:3]:
            monkeypatch.delenv(v, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        tma = name == "tma"
        a, b = pt.fmatrix("a"), pt.fmatrix("b")
        a_, b_ = a[sl], b[sl]
        f = _compile([a, b], [pt.switch(pt.abs(a_) > 64, a_, a_ * b_ + pt.sqr(b_)).sum(axis=1)])
        _check(_alternate(f, grid_sets, 3), grid_refs)
        _assert_fused(f, fallbacks, tpr=tpr, vw=4, tma=tma, store=(False,))
        ins, outs = _cfg2()
        f = _compile(ins, outs)
        res = _alternate(f, cfg_sets, 3)
        _assert_fused(f, fallbacks, tpr=tpr, vw=4, tma=tma, store=(True,))
        if first is None:
            first = res
            for k in range(2):
                _assert_sum_bound(*res[k][1])
        for (k, got), (k0, ref) in zip(res, first):
            for g, e in zip(got, ref):
                _same(g, e, f"scheme {name} vs {SCHEMES[0][0]}, TPR {tpr}")
    assert rows > S * max(_k3_node(f)._occupancy.values()) * rpb


def test_load_schemes_at_the_benchmark_shape(fallbacks, monkeypatch):
    """cfg2 at 4096 x 4096 (128 threads per row, persistent CTAs) under every load scheme: the same bits."""
    sets = _cfg2_sets(4096, 4096)
    first = None
    for name, env in _schemes_for(128):
        for v in K3_ENV:
            monkeypatch.delenv(v, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        ins, outs = _cfg2()
        f = _compile(ins, outs)
        res = _alternate(f, sets, 3)
        _assert_fused(f, fallbacks, tpr=128, vw=4, tma=name == "tma", store=(True,))
        if first is None:
            first = res
            _assert_sum_bound(*res[0][1])
        for (k, got), (k0, ref) in zip(res, first):
            for g, e in zip(got, ref):
                _same(g, e, f"scheme {name} vs {SCHEMES[0][0]}")


def test_host_inputs_replay(fallbacks):
    """mode="CUDA" with NumPy inputs (below the size that is pipelined in row chunks): eager, capture, replay."""
    rows = 8 * _sms() + 1
    ins, outs = _grid_graph(2, "float32", None, True)
    f = pytensor.function(ins, outs, mode="CUDA")
    sets = _grid_sets((rows, 1028))
    refs = _grid_refs(sets, "float32", None, True)
    for i in range(6):
        k = i % 2
        _check([(k, f(*sets[k][0]))], refs)
    assert f.vm.executor.last_from_graph and not f.vm.executor.chunked_calls
    _assert_fused(f, fallbacks, tpr=128, vw=4, store=(True,))


# ---- CAReduce split paths ----------------------------------------------------------------------------------------------
@pytest.fixture
def splits(gpu, monkeypatch):
    """Records the nsplit of every finishing pass of a CAReduceNode."""
    if not gpu:
        pytest.skip("runs the reduction kernels on the device")
    from pytensor_b200.vm.nodes_elemwise import CAReduceNode

    seen = []
    finish = CAReduceNode._finish

    def rec(self, part, out, n_out, nsplit, stride_o, stride_s):
        seen.append(nsplit)
        return finish(self, part, out, n_out, nsplit, stride_o, stride_s)

    monkeypatch.setattr(CAReduceNode, "_finish", rec)
    return seen


def _red_node(f):
    from pytensor_b200.vm.nodes_elemwise import CAReduceNode

    nodes = [st.impl for st in f.vm.executor.program.steps if isinstance(st.impl, CAReduceNode)]
    assert len(nodes) == 1, [type(st.impl).__name__ for st in f.vm.executor.program.steps]
    return nodes[0]


@pytest.mark.parametrize("case", ["row_split_4", "row_split_full_sum", "row_vw1_misaligned_full_sum", "col_split",
                                  "col_split_outer"])
def test_careduce_split_paths_on_the_integer_grid(splits, case):
    S = _sms()
    rng = np.random.default_rng(12)
    if case == "row_split_4":        # 64 rows < 2 S row blocks, 8192 vectors: nsplit = min(ceil(4 S / 64), 4) = 4
        x = pt.fmatrix("x")
        out, shape, axis, want = x.sum(axis=1), (64, 32768), 1, (4, ("row", 4, 256))
    elif case == "row_split_full_sum":   # 2^22 values: nsplit = min(4 S, 2^20 / 2048) > 32, the finish lane loop
        x = pt.fvector("x")
        out, shape, axis, want = x.sum(), (1 << 22,), None, (min(4 * S, 512), ("row", 4, 256))
    elif case == "row_vw1_misaligned_full_sum":
        x = pt.fvector("x")
        out, shape, axis, want = x[1:].sum(), ((1 << 22) + 1,), None, (min(4 * S, 1024), ("row", 1, 256))
    elif case == "col_split":        # (70000, 3) over axis 0: one CTA column, nsplit = min(4 S, 70000 / 16)
        x = pt.fmatrix("x")
        out, shape, axis, want = x.sum(axis=0), (70000, 3), 0, (min(4 * S, 4375), ("col",))
    else:                            # (2, 50000, 5) over axis 1
        x = pt.ftensor3("x")
        out, shape, axis, want = x.sum(axis=1), (2, 50000, 5), 1, (min(2 * S, 3125), ("col",))
    f = _compile([x], [out])
    sets, refs = [], []
    for _ in range(2):
        xi = rng.integers(-8, 9, shape)
        flat = xi.reshape(-1)
        m = flat.size // 4 - 1                                   # cancelling ±G pairs across the whole input
        s = rng.choice(m, 64, replace=False)
        flat[4 * s[:32]] = flat[4 * s[:32] + 1] = G
        flat[4 * s[32:]] = flat[4 * s[32:] + 1] = -G
        src = xi[1:] if case == "row_vw1_misaligned_full_sum" else xi
        sets.append([xi.astype("float32")])
        refs.append([np.asarray(src.sum(axis=axis)).astype(np.float64).astype("float32")])
    _check(_alternate(f, sets), refs)
    nsplit, key = want
    assert splits and set(splits) == {nsplit}, (splits, nsplit)
    assert nsplit > 1 and (case != "row_split_full_sum" or nsplit > 32)
    assert key in _red_node(f)._kernels, list(_red_node(f)._kernels)
