"""CPU suite: the generated sync-free CUDA kernels (fused Elemwise vec / flat / generic, fused Scan) executed thread by
thread on the host (tests/kernel_emulator.py) against NumPy — index arithmetic, vector tails, broadcasting strides and the
circular trace-buffer protocol, without a GPU."""

import ctypes
from ctypes import c_int, c_longlong, c_uint, c_void_p

import numpy as np
import pytest

from kernel_emulator import EmulatedKernel
from pytensor_b200.codegen import elemwise as cg_ew
from pytensor_b200.codegen import scan as cg_scan
from pytensor_b200.codegen.scalar import ScalarInst, ScalarProgram


def _prog_fma_tanh(dtype="float32"):
    # o0 = tanh(i0 * i1 + i2), o1 = i0 - i2
    p = ScalarProgram(in_dtypes=[dtype] * 3, out_dtypes=[dtype, dtype])
    p.insts = [ScalarInst("Mul", [("i", 0), ("i", 1)], [dtype, dtype], dtype),
               ScalarInst("Add", [("t", 0), ("i", 2)], [dtype, dtype], dtype),
               ScalarInst("Tanh", [("t", 1)], [dtype], dtype),
               ScalarInst("Sub", [("i", 0), ("i", 2)], [dtype, dtype], dtype)]
    p.outputs = [("t", 2), ("t", 3)]
    return p


def _ptr(a):
    return c_void_p(a.ctypes.data)


def _aligned(shape, dtype, rng=None, align=64):
    n = int(np.prod(shape))
    raw = np.empty(n * np.dtype(dtype).itemsize + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    a = raw[off:off + n * np.dtype(dtype).itemsize].view(dtype).reshape(shape)
    a[...] = rng.standard_normal(shape).astype(dtype) if rng is not None else 0
    return a


@pytest.mark.parametrize("n,grid", [(1003, 3), (7, 1), (4096, 2), (3, 1), (260 * 4 * 4 + 5, 1)])
def test_flat_vector_kernel_with_scalar_broadcast_and_tail(tmp_path, n, grid):
    rng = np.random.default_rng(1)
    prog = _prog_fma_tanh()
    src = cg_ew.gen_vec_kernel(prog, "k_flat", (1, 0, 1, 1, 1), {}, 4, flat=True)   # input 1 is a broadcast scalar
    k = EmulatedKernel(src, "k_flat", tmp_path)
    a, c = _aligned((n,), "float32", rng), _aligned((n,), "float32", rng)
    b = np.array([0.7], dtype="float32")
    o0, o1 = _aligned((n,), "float32"), _aligned((n,), "float32")
    nchunks = n // 4
    args = [_ptr(a), _ptr(b), _ptr(c), _ptr(o0), _ptr(o1)] + [c_longlong(0)] * 5 + \
           [c_longlong(nchunks), c_uint(0), c_longlong(nchunks * 4), c_longlong(n)]
    k.launch(grid, 256, args)
    np.testing.assert_allclose(o0, np.tanh(a * b + c), rtol=2e-6, atol=1e-7)
    np.testing.assert_array_equal(o1, a - c)


@pytest.mark.parametrize("rows,cols,grid", [(5, 16, 1), (37, 64, 2), (1000, 8, 3)])
def test_row_vector_kernel_with_row_broadcast_operand_and_pitched_rows(tmp_path, rows, cols, grid):
    rng = np.random.default_rng(2)
    prog = _prog_fma_tanh()
    src = cg_ew.gen_vec_kernel(prog, "k_rows", (1, 0, 1, 1, 1), {}, 4, flat=False)  # input 1: one value per row
    k = EmulatedKernel(src, "k_rows", tmp_path)
    pitch = cols + 8                                                                   # input 0 lives in a wider buffer
    abuf = _aligned((rows, pitch), "float32", rng)
    a = abuf[:, :cols]
    b = _aligned((rows,), "float32", rng)
    c = _aligned((rows, cols), "float32", rng)
    o0, o1 = _aligned((rows, cols), "float32"), _aligned((rows, cols), "float32")
    cpr = cols // 4
    args = [_ptr(abuf), _ptr(b), _ptr(c), _ptr(o0), _ptr(o1),
            c_longlong(pitch), c_longlong(1), c_longlong(cols), c_longlong(cols), c_longlong(cols),
            c_longlong(rows * cpr), c_uint(cpr), c_longlong(cols), c_longlong(cols)]
    k.launch(grid, 256, args)
    np.testing.assert_allclose(o0, np.tanh(a * b[:, None] + c), rtol=2e-6, atol=1e-7)
    np.testing.assert_array_equal(o1, a - c)


def test_generic_kernel_with_transposed_broadcast_and_negative_strides(tmp_path):
    rng = np.random.default_rng(3)
    prog = _prog_fma_tanh("float64")
    src = cg_ew.gen_generic_kernel(prog, "k_gen", {})
    k = EmulatedKernel(src, "k_gen", tmp_path)
    shape = (4, 5, 6)
    a = rng.standard_normal((6, 5, 4)).transpose(2, 1, 0)             # transposed view
    b = rng.standard_normal((1, 5, 1))                                 # broadcast along dims 0 and 2
    cfull = rng.standard_normal(shape)
    c = cfull[:, ::-1, :]                                              # negative stride along dim 1
    o0, o1 = np.empty(shape), np.empty(shape[::-1]).transpose(2, 1, 0)  # second output written through a transposed view
    ops = [a, b, c, o0, o1]

    class EwDims(ctypes.Structure):
        _fields_ = [("ndim", c_int), ("shape", c_longlong * cg_ew.MAX_DIMS), ("st", (c_longlong * cg_ew.MAX_DIMS) * len(ops))]

    d = EwDims()
    d.ndim = 3
    for i, s in enumerate(shape):
        d.shape[i] = s
    for j, t in enumerate(ops):
        for i in range(3):
            d.st[j][i] = 0 if t.shape[i] == 1 else t.strides[i] // t.itemsize
    total = int(np.prod(shape))
    k.launch(2, 256, [_ptr(t) for t in ops] + [d, c_longlong(total)])
    np.testing.assert_allclose(o0, np.tanh(a * b + c), rtol=1e-14)
    np.testing.assert_array_equal(o1, a - c)


def _scan_reference(T, store, taps, h_init, seq, a, b):
    """NumPy statement of the buffer protocol (codegen/scan.py docstring): `store` slots, the first L hold the initial
    taps, step i writes slot (L + i) % store, a value survives iff i >= T - store."""
    L = -min(taps)
    buf = np.zeros((store,) + h_init.shape[1:], dtype=h_init.dtype)
    buf[:L] = h_init
    window = [h_init[j].copy() for j in range(L)]
    for i in range(T):
        args = [window[L + t] for t in taps]
        new = np.tanh(args[-1] * a + b) + (0.5 * args[0] if len(taps) > 1 else 0) + (seq[i] if seq is not None else 0)
        window = window[1:] + [new.astype(h_init.dtype)]
        if i >= T - store:
            buf[(L + i) % store] = window[-1]
    return buf


@pytest.mark.parametrize("T,store,taps,with_seq", [(10, 11, (-1,), False), (10, 2, (-1,), False), (7, 3, (-1,), True),
                                                    (1, 2, (-1,), False), (0, 2, (-1,), False), (9, 4, (-2, -1), True),
                                                    (6, 8, (-2, -1), False), (25, 5, (-1,), True)])
def test_fused_scan_kernel_trace_buffers_taps_and_sequences(tmp_path, T, store, taps, with_seq):
    rng = np.random.default_rng(4)
    dt = "float32"
    L = -min(taps)
    S = (3, 5)
    # scalar program: inputs [seq?] + taps (in tap order) + nonseq a, b ; output: new state
    n_seq = 1 if with_seq else 0
    n_in = n_seq + len(taps) + 2
    p = ScalarProgram(in_dtypes=[dt] * n_in, out_dtypes=[dt])
    last_tap = n_seq + len(taps) - 1
    a_i, b_i = n_seq + len(taps), n_seq + len(taps) + 1
    insts = [ScalarInst("Mul", [("i", last_tap), ("i", a_i)], [dt, dt], dt), ScalarInst("Add", [("t", 0), ("i", b_i)], [dt, dt], dt),
             ScalarInst("Tanh", [("t", 1)], [dt], dt)]
    cur = 2
    if len(taps) > 1:
        insts += [ScalarInst("Mul", [("i", n_seq), ("c", 0)], [dt, dt], dt), ScalarInst("Add", [("t", cur), ("t", cur + 1)], [dt, dt], dt)]
        p.consts = [(dt, 0.5)]
        cur += 2
    if with_seq:
        insts += [ScalarInst("Add", [("t", cur), ("i", 0)], [dt, dt], dt)]
        cur += 1
    p.insts, p.outputs = insts, [("t", cur)]
    src = cg_scan.gen_fused_scan_kernel(p, "k_scan", n_seq, [taps], 0, 2)
    k = EmulatedKernel(src, "k_scan", tmp_path)

    h_init = rng.standard_normal((L,) + S).astype(dt)
    seq = rng.standard_normal((max(T, 1),) + S).astype(dt) * 0.1 if with_seq else None
    a = rng.uniform(0.5, 1.0, S[1]).astype(dt)          # broadcast over rows
    b = (rng.standard_normal(S) * 0.1).astype(dt)
    buf = np.zeros((store,) + S, dtype=dt)
    buf[:L] = h_init
    ops = ([seq] if with_seq else []) + [buf, a, b]
    nops = len(ops)

    class ScDims(ctypes.Structure):
        _fields_ = [("ndim", c_int), ("shape", c_longlong * cg_scan.MAX_DIMS), ("st", (c_longlong * cg_scan.MAX_DIMS) * nops),
                    ("tstride", c_longlong * nops), ("store", c_longlong * 1)]

    d = ScDims()
    d.ndim = 2
    d.shape[0], d.shape[1] = S
    for j, t in enumerate(ops):
        per_elem = j >= n_seq + 1
        if per_elem:
            full = np.broadcast_to(t, S)
            for kk in range(2):
                d.st[j][kk] = full.strides[kk] // t.itemsize
            d.tstride[j] = 0
        else:
            for kk in range(2):
                d.st[j][kk] = t.strides[kk + 1] // t.itemsize
            d.tstride[j] = t.strides[0] // t.itemsize
    d.store[0] = store
    total = int(np.prod(S))
    k.launch(2, 256, [_ptr(t) for t in ops] + [d, c_longlong(total), c_longlong(T)])
    expect = _scan_reference(T, store, taps, h_init, seq, a[None, :], b)
    np.testing.assert_allclose(buf, expect, rtol=3e-6, atol=1e-6)


# ---- kernels with warp shuffles / __syncthreads / __shared__ (threaded emulator: one OS thread per simulated thread) ------
from pytensor_b200.codegen import careduce as cg_red  # noqa: E402


@pytest.mark.parametrize("rows,cols,tpr,vw,store", [(9, 64, 32, 4, True), (3, 1024, 256, 4, True), (10, 70, 32, 1, True),
                                                     (5, 260, 32, 4, False), (2, 2052, 256, 4, True), (5, 2060, 128, 4, True),
                                                     (7, 1024, 64, 4, False)])
@pytest.mark.parametrize("tma", [False, True])
def test_fused_map_row_reduce_kernel_k3(tmp_path, rows, cols, tpr, vw, store, tma):
    """The bench's dominant kernel shape (gen_row_kernel): map over (rows, cols), store the map result (or not), reduce each
    row with fp64 accumulation — warp-shuffle tree, cross-warp combine through shared memory for TPR = 256, scalar tail for
    cols % VW, rows that do not fill the last block."""
    if tma and vw != 4:
        pytest.skip("the TMA-staged variant moves 16-byte vectors")
    rng = np.random.default_rng(6)
    dt = "float32"
    prog = ScalarProgram(in_dtypes=[dt, dt, dt], out_dtypes=[dt])
    prog.insts = [ScalarInst("Mul", [("i", 0), ("i", 1)], [dt, dt], dt), ScalarInst("Add", [("t", 0), ("i", 2)], [dt, dt], dt),
                  ScalarInst("Tanh", [("t", 1)], [dt], dt)]
    prog.outputs = [("t", 2)]
    in_modes = (1, 0, 1)                                      # input 1: one value per row
    gen = cg_red.gen_row_kernel_tma if tma else cg_red.gen_row_kernel
    src = gen(prog, "k_row", in_modes, (store,), "add", "float64", "float32", 0, vw, tpr)
    k = EmulatedKernel(src, "k_row", tmp_path, threaded=True, warp_shim=tma)   # (a real __syncwarp before the slot release)
    a, c = _aligned((rows, cols), dt, rng), _aligned((rows, cols), dt, rng)
    b = _aligned((rows,), dt, rng)
    e = _aligned((rows, cols), dt)
    r = _aligned((rows,), dt)
    args = [_ptr(a), _ptr(b), _ptr(c)] + ([_ptr(e)] if store else []) + [_ptr(r), c_longlong(cols), c_longlong(1), c_longlong(cols)] \
        + ([c_longlong(cols)] if store else []) + [c_longlong(rows), c_longlong(cols), c_int(1)]
    rows_per_block = 256 // tpr
    # fewer CTAs than row blocks: the persistent launch (CTAs stride over the row blocks) is what the VM uses
    k.launch((min(2, (rows + rows_per_block - 1) // rows_per_block), 1), 256, args)
    expect = np.tanh(a * b[:, None] + c)
    if store:
        np.testing.assert_allclose(e, expect, rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(r, expect.astype(np.float64).sum(axis=1).astype(np.float32), rtol=3e-6, atol=1e-6)


K3_SCHEMES = {"none": {}, "l2": {"PTK_K3_PIPE": "l2"}, "regs": {"PTK_K3_PIPE": "regs"}, "tma": {"PTK_K3_PIPE": "tma"},
              "idx": {"PTK_K3_ADDR": "idx"}}
_k3_scheme_kernels = {}


@pytest.mark.parametrize("layout", ["no_full_vector", "one_leftover_vector", "tail"])
@pytest.mark.parametrize("scheme,tpr", [(s, t) for s in K3_SCHEMES for t in (32, 64, 128, 256)
                                        if not (s == "tma" and t < 64)])   # (the launcher stages from 64 threads per row)
def test_fused_map_row_reduce_load_schemes_on_the_integer_grid(tmp_path_factory, monkeypatch, scheme, tpr, layout):
    """Every load scheme of the row kernel (PTK_K3_PIPE / PTK_K3_ADDR) at every TPR, bit for bit: integer-valued inputs
    make the map a * s + c exact and its fp64 row sum exact, and an adjacent +G pair and -G pair per row (G + G > 2^24)
    breaks any fp32 step in the accumulation.  Two CTAs stride over four row blocks (the register pipeline pre-loads the
    first trip of a thread's next row), the last block is partial; cols give no full vector, one vector left over after
    the two-vector trips, or a scalar tail behind an uneven share of vectors."""
    G = 3 << 22
    for v in ("PTK_K3_PIPE", "PTK_K3_ADDR", "PTK_K3_MINB"):
        monkeypatch.delenv(v, raising=False)
    for k, v in K3_SCHEMES[scheme].items():
        monkeypatch.setenv(k, v)
    dt, vw, rpb = "float32", 4, 256 // tpr
    key = (scheme, tpr)
    if key not in _k3_scheme_kernels:
        prog = ScalarProgram(in_dtypes=[dt, dt, dt], out_dtypes=[dt])
        prog.insts = [ScalarInst("Mul", [("i", 0), ("i", 1)], [dt, dt], dt), ScalarInst("Add", [("t", 0), ("i", 2)], [dt, dt], dt)]
        prog.outputs = [("t", 1)]
        gen = cg_red.gen_row_kernel_tma if scheme == "tma" else cg_red.gen_row_kernel
        src = gen(prog, "k_row_s", (1, 0, 1), (True,), "add", "float64", "float32", 0, vw, tpr)
        _k3_scheme_kernels[key] = EmulatedKernel(src, "k_row_s", tmp_path_factory.mktemp(f"k3_{scheme}_{tpr}"), threaded=True,
                                                 warp_shim=scheme == "tma")
    k = _k3_scheme_kernels[key]
    ncv, tail = {"no_full_vector": (0, 3), "one_leftover_vector": (2 * tpr + 1, 0), "tail": (3 * tpr + 5, 2)}[layout]
    cols = ncv * vw + tail
    pitch = cols + (-cols) % vw + vw          # aligned row pitch with padding that must stay untouched
    rows = 3 * rpb + 1
    rng = np.random.default_rng(tpr + ncv)
    a, c, e = _aligned((rows, pitch), dt), _aligned((rows, pitch), dt), _aligned((rows, pitch), dt)
    s = _aligned((rows,), dt)
    ai, ci = rng.integers(-8, 9, (rows, cols)), rng.integers(-8, 9, (rows, cols))
    si = rng.integers(-4, 5, rows)
    if cols >= 8:
        m = cols // 2 - 1
        p1 = rng.integers(0, m, rows)
        p2 = (p1 + rng.integers(1, m, rows)) % m
        for p, v in ((p1, G), (p2, -G)):
            ci[np.arange(rows), 2 * p] = ci[np.arange(rows), 2 * p + 1] = v
    a[:, :cols], c[:, :cols], s[:] = ai, ci, si
    e[...] = 12345.0
    r = _aligned((rows,), dt)
    args = [_ptr(a), _ptr(s), _ptr(c), _ptr(e), _ptr(r), c_longlong(pitch), c_longlong(1), c_longlong(pitch), c_longlong(pitch),
            c_longlong(rows), c_longlong(cols), c_int(1)]
    k.launch((2, 1), 256, args)
    exact = ai * si[:, None] + ci
    np.testing.assert_array_equal(e[:, :cols], exact.astype(dt))
    assert np.all(e[:, cols:] == 12345.0)
    np.testing.assert_array_equal(r, exact.sum(axis=1).astype(np.float64).astype(dt))


@pytest.mark.parametrize("red_op,np_fn,identity", [("add", np.sum, 0), ("maximum", np.max, float("-inf")), ("mul", np.prod, 1)])
def test_column_and_generic_reduce_kernels(tmp_path, red_op, np_fn, identity):
    rng = np.random.default_rng(7)
    x = rng.uniform(0.5, 1.5, size=(3, 37, 70))            # (outer, red, inner)
    # column kernel: reduce the middle axis, threads along the contiguous inner axis, optional split of the reduced axis
    src = cg_red.gen_col_kernel("k_col", "float64", red_op, "float64", "float64", identity)
    k = EmulatedKernel(src, "k_col", tmp_path, threaded=True)
    out = np.empty((3, 70))
    k.launch((1, 3, 1), 256, [_ptr(x), _ptr(out), c_longlong(3), c_longlong(37), c_longlong(70), c_int(1)])
    np.testing.assert_allclose(out, np_fn(x, axis=1), rtol=1e-13)
    if red_op == "add":  # split into 4 partial sums [split][outer][inner], finished by the warp-per-output kernel
        part = np.empty((4, 3, 70))
        k.launch((1, 2, 4), 256, [_ptr(x), _ptr(part), c_longlong(3), c_longlong(37), c_longlong(70), c_int(4)])
        np.testing.assert_allclose(part.sum(axis=0), x.sum(axis=1), rtol=1e-13)
        fsrc = cg_red.gen_finish_kernel("k_fin", "add", "float64", "float64", 0)
        fk = EmulatedKernel(fsrc, "k_fin", tmp_path, threaded=True)
        out2 = np.empty(3 * 70)
        fk.launch(2, 256, [_ptr(part), _ptr(out2), c_longlong(210), c_int(4), c_longlong(1), c_longlong(210)])
        np.testing.assert_allclose(out2.reshape(3, 70), x.sum(axis=1), rtol=1e-13)
    # generic kernel: keep dims (0, 2) of a TRANSPOSED view, reduce dim 1 and a broadcast-free extra dim
    xt = x.transpose(2, 1, 0)                                # shape (70, 37, 3), non-contiguous
    src = cg_red.gen_generic_kernel("k_rgen", "float64", red_op, "float64", "float64", identity)
    gk = EmulatedKernel(src, "k_rgen", tmp_path, threaded=True)

    class RdDims(ctypes.Structure):
        _fields_ = [("nk", c_int), ("nr", c_int), ("kshape", c_longlong * cg_red.MAX_DIMS), ("kst", c_longlong * cg_red.MAX_DIMS),
                    ("rshape", c_longlong * cg_red.MAX_DIMS), ("rst", c_longlong * cg_red.MAX_DIMS)]

    d = RdDims()
    d.nk, d.nr = 2, 1
    es = [s // 8 for s in xt.strides]
    d.kshape[0], d.kshape[1], d.kst[0], d.kst[1] = 70, 3, es[0], es[2]
    d.rshape[0], d.rst[0] = 37, es[1]
    outg = np.empty((70, 3))
    base = x  # the kernel indexes from the base pointer of the view (offset 0 here)
    gk.launch(1, 256, [_ptr(base), _ptr(outg), d, c_longlong(210), c_longlong(37)])
    np.testing.assert_allclose(outg, np_fn(xt, axis=1), rtol=1e-13)


@pytest.mark.parametrize("in_dt,red_op,acc_dt,out_dt,identity,np_fn", [
    ("int8", "add", "int64", "int64", 0, lambda a: a.astype(np.int64).sum(axis=1)),
    ("uint8", "maximum", "uint8", "uint8", 0, lambda a: a.max(axis=1)),
    ("int16", "minimum", "int16", "int16", 32767, lambda a: a.min(axis=1)),
    ("bool", "and", "bool", "bool", 1, lambda a: a.all(axis=1)),
    ("bool", "or", "bool", "bool", 0, lambda a: a.any(axis=1)),
    ("int32", "xor", "int32", "int32", 0, lambda a: np.bitwise_xor.reduce(a, axis=1)),
    ("int64", "mul", "int64", "int64", 1, lambda a: a.prod(axis=1)),
    ("float32", "maximum", "float32", "float32", float("-inf"), lambda a: a.max(axis=1)),
    ("float64", "add", "float64", "float64", 0, lambda a: a.sum(axis=1)),
])
@pytest.mark.parametrize("cols,tpr,nsplit", [(100, 32, 1), (4100, 256, 1), (4096, 32, 4)])
def test_careduce_row_kernel_dtypes_accumulators_and_splits(tmp_path, in_dt, red_op, acc_dt, out_dt, identity, np_fn, cols, tpr, nsplit):
    """Pure CAReduce row kernel (identity map): the reference's accumulator / output dtypes (`_acc_dtype`,
    pytensor/tensor/elemwise.py:1383-1417: small ints accumulate in int64), the shuffle specialisations for 1- and 2-byte
    accumulators, NaN-free max/min, and the split-row variant finished by the warp-per-output kernel."""
    rng = np.random.default_rng(8)
    rows = 5
    if in_dt == "bool":
        a = _aligned((rows, cols), "uint8")
        a[...] = rng.integers(0, 2, size=(rows, cols)) if red_op == "or" else 1
        a[1, cols // 2] = 0 if red_op == "and" else a[1, cols // 2]
        a[2] = 0 if red_op == "or" else a[2]
    elif in_dt.startswith("float"):
        a = _aligned((rows, cols), in_dt, rng)
    else:
        a = _aligned((rows, cols), in_dt)
        lo, hi = (-3, 4) if red_op != "mul" else (1, 2)
        a[...] = rng.integers(max(lo, np.iinfo(in_dt).min), hi, size=(rows, cols)).astype(in_dt)
        if red_op == "mul":
            a[:, ::97] = -1
    isz = a.itemsize
    vw = 4 if isz >= 4 else (8 if isz == 2 else 16)
    if cols % vw:
        vw = 1
    prog = cg_red.identity_program(in_dt)
    src = cg_red.gen_row_kernel(prog, "k_red", (1,), (False,), red_op, acc_dt, out_dt, identity, vw, tpr)
    k = EmulatedKernel(src, "k_red", tmp_path, threaded=True)
    np_out = np.dtype("uint8" if out_dt == "bool" else out_dt)
    np_acc = np.dtype("uint8" if acc_dt == "bool" else acc_dt)
    rows_per_block = 256 // tpr
    gx = (rows + rows_per_block - 1) // rows_per_block
    if nsplit == 1:
        out = np.zeros(rows, dtype=np_out)
        k.launch((gx, 1), 256, [_ptr(a), _ptr(out), c_longlong(cols), c_longlong(rows), c_longlong(cols), c_int(1)])
    else:
        part = np.zeros((rows, nsplit), dtype=np_acc)
        k.launch((gx, nsplit), 256, [_ptr(a), _ptr(part), c_longlong(cols), c_longlong(rows), c_longlong(cols), c_int(nsplit)])
        fk = EmulatedKernel(cg_red.gen_finish_kernel("k_fin2", red_op, acc_dt, out_dt, identity), "k_fin2", tmp_path, threaded=True)
        out = np.zeros(rows, dtype=np_out)
        fk.launch(1, 256, [_ptr(part), _ptr(out), c_longlong(rows), c_int(nsplit), c_longlong(nsplit), c_longlong(1)])
    ref = np_fn(a.view(np.bool_) if in_dt == "bool" else a)
    if np_out.kind == "f":
        np.testing.assert_allclose(out, ref, rtol=1e-5 if in_dt == "float32" else 1e-12)
    else:
        np.testing.assert_array_equal(out.astype(ref.dtype) if in_dt != "bool" else out.astype(bool), ref)


# ---- hand-written libptk kernels, extracted from the .cu source and instantiated for the host ----------------------------
import os  # noqa: E402

from kernel_emulator import extract_static_kernel  # noqa: E402
from ctypes import c_double, c_float  # noqa: E402

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytensor_b200", "csrc")


def _smallk_case(tmp_path, kernel, M, N, K, KM, beta, dtype="float32"):
    rng = np.random.default_rng(9)
    cT, ct = ("float", c_float) if dtype == "float32" else ("double", c_double)
    src = extract_static_kernel(os.path.join(CSRC, "ptk_blas.cu"), kernel)
    k = EmulatedKernel(src, kernel, tmp_path, threaded=True, template_args=f"{cT}, {KM}", type_subst={"T": cT})
    A = _aligned((M, K), dtype, rng)
    B = _aligned((K, N), dtype, rng)
    C = _aligned((M, N), dtype, rng)
    expect = 1.5 * (A.astype(np.float64) @ B.astype(np.float64)) + beta * C.astype(np.float64)
    args = [c_longlong(M), c_longlong(N), c_int(K), ct(1.5), _ptr(A), c_longlong(K), c_longlong(1), _ptr(B), c_longlong(N),
            c_longlong(1), ct(beta), _ptr(C), c_longlong(N)]
    k.launch(((N + 255) // 256, 2), 256, args)
    np.testing.assert_allclose(C, expect, rtol=1e-5 if dtype == "float32" else 1e-12, atol=1e-5 if dtype == "float32" else 1e-12)


@pytest.mark.parametrize("M,N,K,KM,beta", [(130, 256, 8, 8, 0.0), (300, 70, 8, 8, 0.75), (65, 1024, 3, 4, 1.0), (200, 260, 13, 16, 0.5)])
def test_skinny_gemm_small_k_kernel(tmp_path, M, N, K, KM, beta):
    """gemm_smallk_kernel (csrc/ptk_blas.cu): C = alpha*A[M,K<=16] @ B[K,N] + beta*C with A tiles staged in shared memory,
    ragged last row tile, columns that do not fill the last block, vector and scalar epilogues."""
    _smallk_case(tmp_path, "gemm_smallk_kernel", M, N, K, KM, beta)


def _smalln_case(tmp_path, kernel, M, N_act, NT, K, beta, grid=3, R=None):
    rng = np.random.default_rng(10)
    src = extract_static_kernel(os.path.join(CSRC, "ptk_blas.cu"), kernel)
    targs = f"float, {NT}" + (f", {R}" if R else "")
    k = EmulatedKernel(src, kernel, tmp_path, threaded=True, template_args=targs, type_subst={"T": "float"},
                       dynamic_smem="sn_smem")
    A = _aligned((M, K), "float32", rng)
    B = _aligned((K, N_act), "float32", rng)
    C = _aligned((M, N_act), "float32", rng)
    expect = 0.5 * (A.astype(np.float64) @ B.astype(np.float64)) + beta * C.astype(np.float64)
    unit = 32 * 4 * 4   # launch_smalln's sweep unit (a multiple of the v2 kernel's 32 * V * U as well)
    kchunk = (K + unit - 1) // unit * unit
    args = [c_longlong(M), c_int(N_act), c_longlong(K), c_int(kchunk), c_float(0.5), _ptr(A), c_longlong(K), _ptr(B),
            c_longlong(N_act), c_longlong(1), c_float(beta), _ptr(C), c_longlong(N_act), c_longlong(1)]
    k.launch(grid, 256, args)
    np.testing.assert_allclose(C, expect, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("M,N_act,NT,K,beta", [(50, 8, 8, 1024, 0.0), (27, 5, 8, 700, 1.0), (64, 1, 1, 512, 0.5), (40, 16, 16, 96, 0.0)])
def test_skinny_gemm_small_n_kernel(tmp_path, M, N_act, NT, K, beta):
    """gemm_smalln_kernel: C[M, N<=16] = alpha*A[M,K] @ B[K,N] + beta*C, one warp per row, B transposed in shared memory,
    vector path with a K that is not a multiple of the sweep, padded template width (n_act < N)."""
    _smalln_case(tmp_path, "gemm_smalln_kernel", M, N_act, NT, K, beta)


@pytest.mark.parametrize("M,N,K,KM,beta", [(130, 256, 8, 8, 0.0), (300, 70, 8, 8, 0.75), (65, 1024, 3, 4, 1.0), (200, 260, 13, 16, 0.5),
                                           (61, 64, 8, 8, 1.0), (259, 513, 8, 8, 0.25)])
def test_skinny_gemm_small_k_kernel_v2(tmp_path, M, N, K, KM, beta):
    """The software-pipelined variant (PTK_BLAS_V2=1): the group's reads of C are issued before its stores — same results,
    incl. ragged row groups (M not a multiple of 16 / 64), misaligned rows (N = 513: only every 4th row is 16-byte aligned)
    and the scalar edge columns."""
    _smallk_case(tmp_path, "gemm_smallk_v2_kernel", M, N, K, KM, beta)


@pytest.mark.parametrize("M,N_act,NT,K,beta,R", [(50, 8, 8, 1024, 0.0, 4), (27, 5, 8, 700, 1.0, 4), (64, 1, 1, 512, 0.5, 4), (41, 16, 16, 96, 0.0, 2),
                                                 (3, 8, 8, 1024, 1.0, 4), (130, 4, 4, 2100, 0.5, 4)])
def test_skinny_gemm_small_n_kernel_v2(tmp_path, M, N_act, NT, K, beta, R):
    """The R-rows-per-warp variant: row groups that run past M, fewer rows than one group, K spanning several sweeps."""
    _smalln_case(tmp_path, "gemm_smalln_v2_kernel", M, N_act, NT, K, beta, R=R)


# ---- boolean-mask compaction (ptk_nonzero_count / ptk_nonzero_fill, csrc/ptk_misc.cu) -----------------------------------
def _nonzero_sources():
    import re

    text = open(os.path.join(CSRC, "ptk_misc.cu")).read()
    consts = "\n".join(re.findall(r"^constexpr int NZ_[A-Z]+ = [^;]+;", text, re.M))
    i = text.index("__device__ __forceinline__ int nz_count16")
    helper = text[i:text.index("\n}\n", i) + 3]
    shim = "struct alignas(16) uint4 { unsigned x, y, z, w; };\n"
    return shim + consts + "\n" + helper


@pytest.mark.parametrize("n,density,misalign", [(0, 0.5, 0), (1, 1.0, 0), (37, 0.5, 0), (4096, 0.3, 0), (4097, 0.9, 0),
                                                (3 * 4096 + 123, 0.05, 3), (9000, 0.0, 0), (70001, 0.6, 1)])
def test_nonzero_count_scan_fill_kernels(tmp_path, n, density, misalign):
    """np.flatnonzero of a byte mask through the three device passes (tile counts with 16-byte loads and the byte-fold
    popcount, single-CTA exclusive scan with carried totals, ordered per-tile compaction), tails and unaligned bases."""
    rng = np.random.default_rng(n + 1)
    raw = np.zeros(n + 64, dtype=np.uint8)
    mask = raw[misalign:misalign + n]
    mask[:] = (rng.random(n) < density) * rng.integers(1, 256, size=n)  # "true" is any non-zero byte
    pre = _nonzero_sources()
    TILE = 4096
    tiles = (n + TILE - 1) // TILE
    ws = np.full(tiles + 1, -7, dtype=np.int64)
    if tiles:
        k = EmulatedKernel(pre + extract_static_kernel(os.path.join(CSRC, "ptk_misc.cu"), "nonzero_count_kernel"),
                           "nonzero_count_kernel", tmp_path, threaded=True)
        k.launch(min(tiles, 3), 256, [_ptr(mask), ctypes.c_longlong(n), _ptr(ws), ctypes.c_longlong(tiles)])
        per_tile = [int(np.count_nonzero(mask[t * TILE:(t + 1) * TILE])) for t in range(tiles)]
        assert ws[:tiles].tolist() == per_tile
    k = EmulatedKernel(extract_static_kernel(os.path.join(CSRC, "ptk_misc.cu"), "nonzero_scan_kernel"), "nonzero_scan_kernel",
                       tmp_path, threaded=True)
    k.launch(1, 1024, [_ptr(ws), ctypes.c_longlong(tiles)])
    expect = np.flatnonzero(mask)
    assert ws[tiles] == expect.size
    if tiles:
        assert ws[:tiles].tolist() == np.concatenate([[0], np.cumsum(per_tile)[:-1]]).tolist()
        out = np.full(max(expect.size, 1), -1, dtype=np.int64)
        k = EmulatedKernel(pre + extract_static_kernel(os.path.join(CSRC, "ptk_misc.cu"), "nonzero_fill_kernel"),
                           "nonzero_fill_kernel", tmp_path, threaded=True)
        k.launch(min(tiles, 2), 256, [_ptr(mask), ctypes.c_longlong(n), _ptr(ws), ctypes.c_longlong(tiles), _ptr(out)])
        np.testing.assert_array_equal(out[:expect.size], expect)


# ---- error-free leading pieces of the fp32-accurate GEMM (row_absmax_kernel / split_aligned_kernel, ptk_gemm_tc.cu) ------
BF16_SHIM = r"""
#include <cmath>
struct __nv_bfloat16 { unsigned short u; };
struct __nv_bfloat162 { __nv_bfloat16 x, y; };
static inline __nv_bfloat16 __float2bfloat16_rn(float f) {
  unsigned int b; std::memcpy(&b, &f, 4);
  if ((b & 0x7fffffffu) > 0x7f800000u) { __nv_bfloat16 n; n.u = (unsigned short)((b >> 16) | 0x40); return n; }
  b += 0x7fffu + ((b >> 16) & 1u);   // round to nearest even on the dropped 16 bits
  __nv_bfloat16 r; r.u = (unsigned short)(b >> 16); return r;
}
static inline float __bfloat162float(__nv_bfloat16 h) { unsigned int b = (unsigned int)h.u << 16; float f; std::memcpy(&f, &b, 4); return f; }
"""


ATOMIC_SHIM = r"""
static inline unsigned int atomicMax(unsigned int* p, unsigned int v) {
  unsigned int old = __atomic_load_n(p, __ATOMIC_RELAXED);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}
static inline unsigned int __float_as_uint(float f) { unsigned int u; std::memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(unsigned int u) { float f; std::memcpy(&f, &u, 4); return f; }
"""


@pytest.mark.parametrize("lead_bits", [7, 5])
@pytest.mark.parametrize("R,Cc,row_major", [(70, 130, True), (130, 70, False), (64, 64, True), (5, 9, False)])
def test_aligned_three_piece_split_is_exact_and_on_the_row_grid(tmp_path, R, Cc, row_major, lead_bits):
    """x = x1 + x2 + x3 to 2^-(b+16) of the row's largest magnitude; x1 * 2^s is an integer of magnitude <= 2^b with
    s = b - 1 - ilogb(row max), so that the A1 x B1 products of a dot product are integers on one common unit (b = 7 for
    K <= 1024 ... 4 for K > 16384: 2^2b * K <= 2^24 keeps the whole accumulation exact)."""
    rng = np.random.default_rng(R * 1000 + Cc)
    x = (rng.standard_normal((R, Cc)) * np.exp(rng.uniform(-6, 6, (R, 1)))).astype(np.float32)
    x[1 % R, :] = 0.0                       # an all-zero row
    x[2 % R, 3 % Cc] = 1e-30                # tiny next to the row maximum
    src = np.ascontiguousarray(x if row_major else x.T)   # the kernel reads src[r * sr + c * sc]
    sr, sc = (Cc, 1) if row_major else (1, R)
    text = open(os.path.join(CSRC, "ptk_gemm_tc.cu")).read()
    i0 = text.index("__device__ __forceinline__ int scale_exp_of")
    helper = text[i0:text.index("\n}\n", i0) + 3]
    maxbits = np.zeros(R, dtype=np.uint32)
    k1 = EmulatedKernel(BF16_SHIM + ATOMIC_SHIM + extract_static_kernel(os.path.join(CSRC, "ptk_gemm_tc.cu"), "row_absmax_kernel"),
                        "row_absmax_kernel", tmp_path, threaded=True)
    k1.launch(((Cc + 63) // 64, (R + 63) // 64), 256, [_ptr(src), c_longlong(sr), c_longlong(sc), c_longlong(R), c_longlong(Cc),
                                                     _ptr(maxbits)])
    rowmax = np.abs(x).max(axis=1)
    np.testing.assert_array_equal(maxbits.view(np.float32), rowmax)
    sexp = np.where(rowmax > 0, lead_bits - 1 - np.floor(np.log2(np.where(rowmax > 0, rowmax, 1.0))).astype(np.int64),
                    0).astype(np.int32)
    ld, pr = (Cc + 7) // 8 * 8, (R + 255) // 256 * 256
    dst = np.zeros((3 * pr, ld), dtype=np.uint16)
    k2 = EmulatedKernel(BF16_SHIM + ATOMIC_SHIM + helper + extract_static_kernel(os.path.join(CSRC, "ptk_gemm_tc.cu"), "split_aligned_kernel"),
                        "split_aligned_kernel", tmp_path, threaded=True)
    k2.launch(((Cc + 63) // 64, (R + 63) // 64), 256, [_ptr(src), c_longlong(sr), c_longlong(sc), _ptr(dst), c_longlong(ld),
                                                     c_longlong(R), c_longlong(Cc), c_longlong(pr), _ptr(maxbits), c_int(lead_bits)])
    pieces = [(dst[k * pr:k * pr + R, :Cc].astype(np.uint32) << 16).view(np.float32).astype(np.float64) for k in range(3)]
    lead_units = pieces[0] * np.exp2(sexp.astype(np.float64))[:, None]
    assert np.all(lead_units == np.rint(lead_units)) and np.abs(lead_units).max() <= 2 ** lead_bits
    err = np.abs(pieces[0] + pieces[1] + pieces[2] - x.astype(np.float64))
    assert np.all(err <= np.maximum(rowmax[:, None].astype(np.float64) * 2.0 ** -(lead_bits + 16), 1e-45))
    # every product of two leading pieces is an integer (<= 2^14 for the shipped width 7) on the unit 2^-(s_i + s_j)
    from pytensor_b200.runtime import lib as L

    assert L.load_library().ptk_gemm_lead_bits(4096) == 7 and L._TraceLib().ptk_gemm_lead_bits(4096) == 7
    assert (2 ** 7) ** 2 * 1024 <= 2 ** 24


# ---- a chain of small dense layers in one launch (mlp_chain_kernel, csrc/ptk_blas.cu) -----------------------------------------
@pytest.mark.parametrize("M,widths,acts,with_bias", [
    (37, [64, 64, 64, 64, 64], [1, 1, 1, 1], True),          # the metric graph's layer shape, rows not a multiple of 16
    (16, [20, 128, 4, 68, 128], [1, 0, 1, 0], True),         # ragged widths, both column groups, no activation on some layers
    (5, [128, 128], [1], False),                             # a single widest layer without bias
    (50, [8, 12, 8, 12, 8, 12, 8], [0, 0, 1, 1, 0, 1], True),
])
def test_small_mlp_chain_kernel(tmp_path, M, widths, acts, with_bias):
    """h <- act(h @ W_l + b_l) for all layers inside one CTA per 16 rows: activations ping-pong between two shared-memory
    buffers, the next layer's weights stream in while the current layer is computed; fp32 FMA, k ascending."""
    rng = np.random.default_rng(len(widths) * 100 + M)
    text = open(os.path.join(CSRC, "ptk_blas.cu")).read()
    i0 = text.index("constexpr int MC_MAXW")
    i1 = text.index("__device__ __forceinline__ void mc_cp_async16")
    defs = text[i0:i1]
    shim = ("#define __grid_constant__\nstruct alignas(16) float4 { float x, y, z, w; };\n" + defs +
            "static inline void mc_cp_async16(float* d, const float* s) { std::memcpy(d, s, 16); }\n"
            "static inline void mc_cp_async_wait_all() {}\nusing std::fmaf;\n"
            "template <typename T> static inline T __ldg(const T* p) { return *p; }\n")
    src = shim + extract_static_kernel(os.path.join(CSRC, "ptk_blas.cu"), "mlp_chain_kernel").replace(
        "extern __shared__ float mc_smem[];", "alignas(16) static float mc_smem[2 * 16 * 128 + 2 * 128 * 128];")
    k = EmulatedKernel(src, "mlp_chain_kernel", tmp_path, threaded=True)

    class MlpLayer(ctypes.Structure):
        _fields_ = [("W", c_void_p), ("bias", c_void_p), ("K", c_int), ("N", c_int), ("act", c_int), ("pad_", c_int)]

    class MlpChain(ctypes.Structure):
        _fields_ = [("L", c_int), ("pad_", c_int), ("layer", MlpLayer * 96)]

    L = len(widths) - 1
    x = _aligned((M, widths[0]), "float32", rng)
    Ws = [_aligned((widths[l], widths[l + 1]), "float32") for l in range(L)]
    bs = [_aligned((widths[l + 1],), "float32", rng) for l in range(L)]
    ch = MlpChain()
    ch.L = L
    ref = x.astype(np.float64)
    for l in range(L):
        Ws[l][...] = (rng.standard_normal(Ws[l].shape) / np.sqrt(widths[l])).astype("float32")
        ch.layer[l].W = Ws[l].ctypes.data
        ch.layer[l].bias = bs[l].ctypes.data if with_bias else None
        ch.layer[l].K, ch.layer[l].N, ch.layer[l].act = widths[l], widths[l + 1], acts[l]
        ref = ref @ Ws[l].astype(np.float64) + (bs[l].astype(np.float64) if with_bias else 0.0)
        if acts[l]:
            ref = np.tanh(ref)
    y = _aligned((M, widths[-1]), "float32")
    y[...] = -7.0
    k.launch((M + 15) // 16, 256, [_ptr(x), c_longlong(widths[0]), _ptr(y), c_longlong(widths[-1]), c_longlong(M), ch])
    np.testing.assert_allclose(y, ref, rtol=2e-5, atol=2e-6)


# ---- counter-based random draws (random_kernel, ptk_random.cu) -------------------------------------------------------------
RNG_SHIM = r"""
static inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
static inline double sinpi(double x) { return std::sin(M_PI * x); }
static inline double cospi(double x) { return std::cos(M_PI * x); }
using std::sqrt; using std::log; using std::exp; using std::pow; using std::fabs; using std::floor; using std::copysign;
"""

RNG_KAT = r"""
extern "C" void emu_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  Philox p; p.k0 = key[0]; p.k1 = key[1];
  uint32_t c[4] = {ctr[0], ctr[1], ctr[2], ctr[3]};
  p.block(c);
  for (int i = 0; i < 4; ++i) out[i] = c[i];
}
"""


def _random_kernel(tmp_path, out_type="double"):
    text = open(os.path.join(CSRC, "ptk_random.cu")).read()
    body = text[text.index("struct Philox"):text.index("}  // namespace")]
    return EmulatedKernel(RNG_SHIM + body + RNG_KAT, "random_kernel", tmp_path, template_args=out_type, type_subst={"OUT": out_type})


def _draw(k, dist, n, key, seed, params=(), dtype=np.float64, grid=3):
    out = np.full(n, -12345, dtype=dtype)
    ps, keep = [], []   # `keep`: the parameter arrays must outlive the launch
    for p in list(params) + [None] * (3 - len(params)):
        if p is None:
            ps += [c_void_p(None), c_longlong(0)]
        else:
            p = np.ascontiguousarray(p, dtype=np.float64)
            ps += [_ptr(p), c_longlong(0 if p.size == 1 else 1)]
            keep.append(p)
    k.launch(grid, 256, [c_int(dist), _ptr(out), c_longlong(n), ctypes.c_uint64(key), ctypes.c_uint64(seed), *ps])
    return out


def test_philox_block_matches_the_published_known_answers(tmp_path):
    """Philox4x32-10 (Salmon et al., SC'11) known-answer vectors of the Random123 distribution: zero, all-ones and the
    digits-of-pi counter/key."""
    k = _random_kernel(tmp_path)
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        c, kk, out = np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32), np.zeros(4, dtype=np.uint32)
        k.lib.emu_philox(_ptr(c), _ptr(kk), _ptr(out))
        assert tuple(int(v) for v in out) == want


def test_random_kernel_streams_are_per_element_and_keyed(tmp_path):
    """An element's draw depends on (key, seed, element index) only — not on the launch geometry — and changes with either
    key word; uniforms lie strictly inside (0, 1)."""
    k = _random_kernel(tmp_path)
    a = _draw(k, 0, 5000, 0x1234567890abcdef, 42, grid=1)
    b = _draw(k, 0, 5000, 0x1234567890abcdef, 42, grid=7)
    np.testing.assert_array_equal(a, b)
    assert np.all((a > 0) & (a < 1)) and len(np.unique(a)) == a.size
    assert not np.array_equal(a, _draw(k, 0, 5000, 0x1234567890abcdee, 42))
    assert not np.array_equal(a, _draw(k, 0, 5000, 0x1234567890abcdef, 43))
    # a prefix of a longer fill is the shorter fill (streams are indexed, not consumed)
    np.testing.assert_array_equal(_draw(k, 1, 100, 7, 9), _draw(k, 1, 5000, 7, 9)[:100])


@pytest.mark.parametrize("dist,params,ref", [
    (0, (-2.0, 3.0), ("uniform", dict(loc=-2.0, scale=5.0))),
    (1, (1.5, 0.5), ("norm", dict(loc=1.5, scale=0.5))),
    (2, (0.0, 2.0), ("halfnorm", dict(loc=0.0, scale=2.0))),
    (3, (0.2, 0.4), ("lognorm", dict(s=0.4, scale=float(np.exp(0.2))))),
    (4, (2.5,), ("expon", dict(scale=2.5))),
    (5, (1.0, 0.7), ("laplace", dict(loc=1.0, scale=0.7))),
    (6, (-1.0, 0.6), ("logistic", dict(loc=-1.0, scale=0.6))),
    (7, (0.5, 1.5), ("gumbel_r", dict(loc=0.5, scale=1.5))),
    (8, (0.3, 2.0), ("cauchy", dict(loc=0.3, scale=2.0))),
    (15, (0.0, 1.5), ("halfcauchy", dict(loc=0.0, scale=1.5))),
    (10, (0.4, 2.0), ("gamma", dict(a=0.4, scale=2.0))),
    (10, (7.5, 0.5), ("gamma", dict(a=7.5, scale=0.5))),
    (16, (3.0, 2.0), ("invgamma", dict(a=3.0, scale=2.0))),
    (11, (0.7, 2.2), ("beta", dict(a=0.7, b=2.2))),
    (13, (1.7,), ("weibull_min", dict(c=1.7))),
    (14, (2.5, 1.5), ("pareto", dict(b=2.5, scale=1.5))),
    (17, (4.0, 0.5, 2.0), ("t", dict(df=4.0, loc=0.5, scale=2.0))),
])
def test_random_kernel_distributions(tmp_path, dist, params, ref):
    """Kolmogorov-Smirnov of 20000 emulated draws against scipy's CDF of the distribution the reference's RandomVariable
    of that name samples (pytensor/tensor/random/basic.py)."""
    import scipy.stats as st

    k = _random_kernel(tmp_path)
    x = _draw(k, dist, 20000, 0xfeedfacecafebeef, 1234 + dist, [np.array([p]) for p in params])
    name, kw = ref
    stat, p = st.kstest(x, getattr(st, name)(**kw).cdf)
    assert p > 1e-3, (name, stat, p)


def test_random_kernel_discrete_and_broadcast_parameters(tmp_path):
    k = _random_kernel(tmp_path)
    n = 20000
    # Bernoulli with a per-element probability vector; integers in [low, high)
    pvec = np.linspace(0.05, 0.95, n)
    b = _draw(k, 9, n, 11, 22, [pvec])
    assert set(np.unique(b)) <= {0.0, 1.0}
    halves = b[: n // 2].mean(), b[n // 2:].mean()
    assert abs(halves[0] - pvec[: n // 2].mean()) < 0.02 and abs(halves[1] - pvec[n // 2:].mean()) < 0.02
    (tmp_path / "i64").mkdir()
    ki = _random_kernel(tmp_path / "i64", "int64_t")
    r = _draw(ki, 12, n, 5, 6, [np.array([-3.0]), np.array([4.0])], dtype=np.int64)
    vals, counts = np.unique(r, return_counts=True)
    assert vals.tolist() == list(range(-3, 4))
    assert np.all(np.abs(counts / n - 1 / 7) < 0.015)
    # per-element location vector with a scalar scale: the stride-0 / stride-1 parameter walk
    loc = np.arange(n, dtype=np.float64)
    x = _draw(k, 1, n, 3, 4, [loc, np.array([0.01])])
    assert np.max(np.abs(x - loc)) < 0.1 and np.std(x - loc) == pytest.approx(0.01, rel=0.05)


# ---- native-precision BLAS family: gemm_simt_kernel / gemv_row|col_kernel / ger_kernel (ptk_blas.cu) ---------------------
def _blas_text():
    return open(os.path.join(CSRC, "ptk_blas.cu")).read()


@pytest.mark.parametrize("dtype,a_kfast,b_nfast,M,N,K,beta,with_bias,act", [
    ("float32", True, True, 70, 130, 37, 0.0, True, 1),       # row-major A and B, ragged tiles in all three dims, bias + tanh
    ("float32", False, True, 64, 64, 16, 0.6, False, 0),      # A transposed view (M fast), exact tiles, beta * C
    ("float64", True, False, 33, 47, 29, -1.0, False, 0),     # B transposed view (K fast)
    ("float64", False, False, 5, 200, 3, 1.0, True, 0),       # both transposed, K smaller than one k-tile
    ("float32", True, False, 300, 70, 20, -0.5, True, 0),     # 5 m-tiles on 2 y-blocks: the grid-stride m-tile loop turns
])
def test_fma_gemm_kernel_strides_edges_and_epilogue(tmp_path, dtype, a_kfast, b_nfast, M, N, K, beta, with_bias, act):
    """C = act(alpha*A@B + beta*C + bias) over arbitrary element strides; beta == 0 never reads C (NaN-poisoned here, the
    AllocEmpty contract of pytensor/tensor/blas/gemm.py:194-198)."""
    rng = np.random.default_rng(31)
    cT, ct = ("float", c_float) if dtype == "float32" else ("double", c_double)
    text = _blas_text()
    src = text[text.index("constexpr int BM = 64"):text.index("// ---- skinny shapes")]
    k = EmulatedKernel(src, "gemm_simt_kernel", tmp_path, threaded=True,
                       template_args=f"{cT}, {str(a_kfast).lower()}, {str(b_nfast).lower()}", type_subst={"T": cT})
    A = rng.standard_normal((M, K)).astype(dtype) if a_kfast else rng.standard_normal((K, M)).astype(dtype).T
    B = rng.standard_normal((K, N)).astype(dtype) if b_nfast else rng.standard_normal((N, K)).astype(dtype).T
    # C: every second column of a wider buffer (a non-unit column stride)
    Cbuf = rng.standard_normal((M, 2 * N)).astype(dtype)
    if beta == 0.0:
        Cbuf[:] = np.nan
    C = Cbuf[:, ::2]
    bias = rng.standard_normal(N).astype(dtype)
    expect = 0.7 * (A.astype(np.float64) @ B.astype(np.float64))
    if beta != 0.0:
        expect = expect + beta * C.astype(np.float64)
    if with_bias:
        expect = expect + bias
    if act:
        expect = np.tanh(expect)
    isz = A.itemsize
    args = [c_longlong(M), c_longlong(N), c_longlong(K), ct(0.7), c_void_p(A.ctypes.data), c_longlong(A.strides[0] // isz),
            c_longlong(A.strides[1] // isz), c_void_p(B.ctypes.data), c_longlong(B.strides[0] // isz),
            c_longlong(B.strides[1] // isz), ct(beta), c_void_p(C.ctypes.data), c_longlong(C.strides[0] // isz),
            c_longlong(C.strides[1] // isz), _ptr(bias) if with_bias else c_void_p(None), c_int(act)]
    untouched = Cbuf[:, 1::2].copy()
    k.launch(((N + 63) // 64, min((M + 63) // 64, 2)), 256, args)   # (fewer y-blocks than m-tiles where M > 128)
    tol = 2e-5 if dtype == "float32" else 1e-12
    np.testing.assert_allclose(C, expect, rtol=tol, atol=tol)
    np.testing.assert_array_equal(Cbuf[:, 1::2], untouched)   # the columns between the strided ones are not written


@pytest.mark.parametrize("dtype,M,N,nchunks,beta", [("float32", 70, 1300, 1, 0.5), ("float64", 9, 5000, 3, 1.0), ("float32", 33, 17, 1, 0.0)])
def test_gemv_row_kernel(tmp_path, dtype, M, N, nchunks, beta):
    """y = alpha*A@x + beta*y, one warp per (row, column chunk): strided x and y, split rows accumulate atomically into the
    pre-scaled y, beta == 0 never reads y (pytensor/tensor/blas/gemv.py:79-86)."""
    rng = np.random.default_rng(32)
    cT, ct = ("float", c_float) if dtype == "float32" else ("double", c_double)
    src = extract_static_kernel(os.path.join(CSRC, "ptk_blas.cu"), "gemv_row_kernel")
    k = EmulatedKernel(src, "gemv_row_kernel", tmp_path, threaded=True, template_args=cT, type_subst={"T": cT}, warp_shim=True)
    A = rng.standard_normal((M, N)).astype(dtype)
    xb = rng.standard_normal(3 * N).astype(dtype)
    yb = rng.standard_normal(2 * M).astype(dtype)
    x, y = xb[::3], yb[::2]
    y0 = y.astype(np.float64).copy()
    if beta == 0.0:
        y[:] = np.nan
    if nchunks > 1:
        y *= np.asarray(beta, dtype=dtype)   # what scale_vec_kernel does before a split launch
    expect = 1.25 * (A.astype(np.float64) @ x.astype(np.float64)) + (beta * y0 if beta != 0.0 else 0.0)
    chunk = (N + nchunks - 1) // nchunks
    args = [c_longlong(M), c_longlong(N), ct(1.25), _ptr(A), c_longlong(N), c_longlong(1), c_void_p(x.ctypes.data), c_longlong(3),
            ct(beta), c_void_p(y.ctypes.data), c_longlong(2), c_longlong(chunk), c_longlong(nchunks)]
    k.launch(2, 256, args)
    tol = 3e-5 if dtype == "float32" else 1e-11
    np.testing.assert_allclose(y, expect, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype,M,N,nchunks", [("float64", 70, 1300, 4), ("float32", 31, 9, 1), ("float32", 100, 300, 2)])
def test_gemv_col_kernel(tmp_path, dtype, M, N, nchunks):
    """The column-fast variant (A.T views: sa0 == 1): lanes own consecutive rows, 8 column groups reduced through shared memory,
    column chunks accumulate atomically into the pre-scaled y."""
    rng = np.random.default_rng(33)
    cT, ct = ("float", c_float) if dtype == "float32" else ("double", c_double)
    src = extract_static_kernel(os.path.join(CSRC, "ptk_blas.cu"), "gemv_col_kernel")
    k = EmulatedKernel(src, "gemv_col_kernel", tmp_path, threaded=True, template_args=cT, type_subst={"T": cT}, warp_shim=True)
    At = rng.standard_normal((N, M)).astype(dtype)   # A = At.T: element (m, n) at m*1 + n*M
    x = rng.standard_normal(N).astype(dtype)
    y = rng.standard_normal(M).astype(dtype)
    expect = 0.5 * (At.T.astype(np.float64) @ x.astype(np.float64)) + y.astype(np.float64)
    chunk = (N + nchunks - 1) // nchunks
    args = [c_longlong(M), c_longlong(N), ct(0.5), _ptr(At), c_longlong(1), c_longlong(M), _ptr(x), c_longlong(1), _ptr(y),
            c_longlong(1), c_longlong(chunk)]
    k.launch(((M + 31) // 32, nchunks), 256, args)
    tol = 3e-5 if dtype == "float32" else 1e-11
    np.testing.assert_allclose(y, expect, rtol=tol, atol=tol)


def test_ger_kernel_strided_update(tmp_path):
    """A += alpha * outer(x, y) in place over a column-strided A and strided vectors (pytensor/tensor/blas/ger.py:8)."""
    rng = np.random.default_rng(34)
    src = extract_static_kernel(os.path.join(CSRC, "ptk_blas.cu"), "ger_kernel")
    k = EmulatedKernel(src, "ger_kernel", tmp_path, template_args="double", type_subst={"T": "double"})
    M, N = 40, 50
    Abuf = rng.standard_normal((M, 2 * N))
    A = Abuf[:, ::2]
    xb, yb = rng.standard_normal(2 * M), rng.standard_normal(3 * N)
    expect = A + 0.3 * np.outer(xb[::2], yb[::3])
    other = Abuf[:, 1::2].copy()
    args = [c_longlong(M), c_longlong(N), c_double(0.3), c_void_p(xb.ctypes.data), c_longlong(2), c_void_p(yb.ctypes.data),
            c_longlong(3), c_void_p(A.ctypes.data), c_longlong(2 * N), c_longlong(2)]
    k.launch(3, 256, args)
    np.testing.assert_allclose(A, expect, rtol=1e-14, atol=1e-14)
    np.testing.assert_array_equal(Abuf[:, 1::2], other)


# ---- gather / scatter kernels (ptk_index.cu) ---------------------------------------------------------------------------------
INDEX_SHIM = r"""
struct alignas(16) uint4 { unsigned x, y, z, w; };
static inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline void emu_atomic_add(int* p, int v) { __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline void emu_atomic_add(long* p, long v) { __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
static inline void emu_atomic_add(float* p, float v) { atomicAdd(p, v); }    // (the float / double atomicAdd of the warp shim)
static inline void emu_atomic_add(double* p, double v) { atomicAdd(p, v); }
"""


def _index_kernel(tmp_path, name, targs, subst, smem=None, fix=None):
    src = extract_static_kernel(os.path.join(CSRC, "ptk_index.cu"), name)
    for a, b in (fix or {}).items():
        assert a in src
        src = src.replace(a, b)
    return EmulatedKernel(INDEX_SHIM + src, name, tmp_path, threaded=True, template_args=targs, type_subst=subst,
                          dynamic_smem=smem, warp_shim=True)


@pytest.mark.parametrize("outer,n_src,n_idx,inner", [(3, 11, 7, 5), (1, 40, 300, 1), (4, 6, 9, 2)])
def test_take_kernel_negative_and_out_of_range_indices(tmp_path, outer, n_src, n_idx, inner):
    """out[o, j, i] = src[o, idx[j], i] with NumPy's negative-index wrap; an index outside [-n, n) raises the error word and
    leaves that output element alone (the host turns the word into IndexError, like tensor/subtensor.py:2164)."""
    rng = np.random.default_rng(41)
    k = _index_kernel(tmp_path, "take_kernel", "uint32_t", {"T": "uint32_t"})
    src = rng.integers(0, 1 << 31, size=(outer, n_src, inner), dtype=np.uint32)
    idx = rng.integers(-n_src, n_src, size=n_idx).astype(np.int64)
    out = np.full((outer, n_idx, inner), 77, dtype=np.uint32)
    err = np.zeros(1, dtype=np.int32)
    args = [_ptr(out), _ptr(src), _ptr(idx), c_longlong(outer), c_longlong(n_src), c_longlong(n_idx), c_longlong(inner), _ptr(err)]
    k.launch(2, 256, args)
    np.testing.assert_array_equal(out, src[:, idx, :])
    assert err[0] == 0
    idx[n_idx // 2] = n_src          # one past the end
    out[:] = 77
    k.launch(2, 256, args)
    assert err[0] == 1
    good = np.ones(n_idx, dtype=bool)
    good[n_idx // 2] = False
    np.testing.assert_array_equal(out[:, good, :], src[:, idx[good], :])
    assert np.all(out[:, n_idx // 2, :] == 77)


@pytest.mark.parametrize("kernel,outer,n_src,n_idx,misalign", [
    ("take_lastaxis_kernel", 37, 500, 256, 0),      # vector path: 4 rows in flight + the row remainder
    ("take_lastaxis_kernel", 9, 64, 70, 0),         # n_idx not a multiple of 4: scalar stores, ragged last thread
    ("take_lastaxis_kernel", 20, 100, 128, 1),      # output base not 16-byte aligned
    ("take_lastaxis_smem_kernel", 70, 50, 256, 0),  # staged source rows, last row block short (70 = 4*16 + 6)
    ("take_lastaxis_smem_kernel", 64, 33, 130, 0),  # scalar tail
])
def test_take_along_the_last_axis_kernels(tmp_path, kernel, outer, n_src, n_idx, misalign):
    rng = np.random.default_rng(42)
    smem = kernel.endswith("smem_kernel")
    k = _index_kernel(tmp_path, kernel, "uint32_t, 16" if smem else "uint32_t", {"T": "uint32_t"}, smem="take_smem" if smem else None)
    src = rng.integers(0, 1 << 31, size=(outer, n_src), dtype=np.uint32)
    idx = rng.integers(-n_src, n_src, size=n_idx).astype(np.int64)
    buf = _aligned((outer * n_idx + 8,), "uint32")
    out = buf[misalign:misalign + outer * n_idx].reshape(outer, n_idx)
    out[:] = 5
    err = np.zeros(1, dtype=np.int32)
    args = [c_void_p(out.ctypes.data), _ptr(src), _ptr(idx), c_longlong(outer), c_longlong(n_src), c_longlong(n_idx), _ptr(err)]
    grid = (1, (outer + 15) // 16) if smem else ((n_idx + 1023) // 1024, 3)
    k.launch(grid, 256, args)
    np.testing.assert_array_equal(out, src[:, idx])
    assert err[0] == 0
    idx[3] = -n_src - 1
    out[:] = 5
    k.launch(grid, 256, args)
    assert err[0] == 1
    keep = np.arange(n_idx) != 3
    np.testing.assert_array_equal(out[:, keep], src[:, idx[keep]])
    assert np.all(out[:, 3] == 5)


@pytest.mark.parametrize("ctype,dtype,op", [("float", np.float32, 1), ("double", np.float64, 1), ("int64_t", np.int64, 1),
                                            ("int32_t", np.int32, 0)])
def test_put_kernel_set_and_accumulate(tmp_path, ctype, dtype, op):
    """x[:, idx, :] = y (unique indices) / np.add.at(x, (:, idx, :), y) with repeated and negative indices — the atomics
    path of AdvancedIncSubtensor (tensor/subtensor.py:2275)."""
    rng = np.random.default_rng(43)
    k = _index_kernel(tmp_path, "put_kernel", f"{ctype}, {op}", {"T": ctype},
                      fix={"atomic_add_t<T>(p, y[t])": "emu_atomic_add(p, y[t])"})
    outer, n_dst, n_idx, inner = 3, 13, 40 if op else 9, 4
    x = (rng.standard_normal((outer, n_dst, inner)) * 8).astype(dtype)
    y = (rng.standard_normal((outer, n_idx, inner)) * 8).astype(dtype)
    idx = (rng.integers(-n_dst, n_dst, size=n_idx) if op else rng.permutation(n_dst)[:n_idx] - n_dst * (np.arange(n_idx) % 2)).astype(np.int64)
    want = x.copy()
    if op:
        np.add.at(want, (slice(None), idx, slice(None)), y)
    else:
        want[:, idx, :] = y
    err = np.zeros(1, dtype=np.int32)
    k.launch(2, 256, [_ptr(x), _ptr(y), _ptr(idx), c_longlong(outer), c_longlong(n_dst), c_longlong(n_idx), c_longlong(inner), _ptr(err)])
    if np.issubdtype(dtype, np.floating):
        np.testing.assert_allclose(x, want, rtol=1e-5 if dtype == np.float32 else 1e-13, atol=1e-4 if dtype == np.float32 else 1e-12)
    else:
        np.testing.assert_array_equal(x, want)
    assert err[0] == 0


@pytest.mark.parametrize("dtype,ctype,outer,n_dst,n_idx", [(np.float32, "float", 21, 64, 1024), (np.float64, "double", 5, 7, 300),
                                                          (np.float32, "float", 3, 130, 33)])
def test_put_rows_segmented_scatter_add(tmp_path, dtype, ctype, outer, n_dst, n_idx):
    """x[:, idx] += y with ONE index vector shared by all rows (the group index of a hierarchical model): histogram + exclusive
    scan, stable permutation, one warp per row adding each bin's contributions in ascending source order — the order of
    np.add.at, so the result is deterministic and, in fp64, bit-identical to NumPy's."""
    rng = np.random.default_rng(44)
    idx = rng.integers(-n_dst, n_dst, size=n_idx).astype(np.int64)
    idx[rng.integers(0, n_idx, size=3)] = n_dst - 1
    offsets = np.full(n_dst + 1, -1, dtype=np.int32)
    perm = np.full(n_idx, -1, dtype=np.int32)
    err = np.zeros(1, dtype=np.int32)
    (tmp_path / "a").mkdir(), (tmp_path / "b").mkdir(), (tmp_path / "c").mkdir()
    k1 = _index_kernel(tmp_path / "a", "put_rows_offsets_kernel", "", None, fix={"extern __shared__ int cnt[];": "static int cnt[16384];"})
    k1.launch(1, 1024, [_ptr(idx), c_longlong(n_idx), c_longlong(n_dst), _ptr(offsets), _ptr(err)])
    norm = np.where(idx < 0, idx + n_dst, idx)
    counts = np.bincount(norm, minlength=n_dst)
    assert offsets.tolist() == np.concatenate([[0], np.cumsum(counts)]).tolist() and err[0] == 0
    k2 = _index_kernel(tmp_path / "b", "put_rows_perm_kernel", "", None, fix={"extern __shared__ int sidx[];": "static int sidx[16384];"})
    k2.launch((n_dst + 255) // 256, 256, [_ptr(idx), c_longlong(n_idx), c_longlong(n_dst), _ptr(offsets), _ptr(perm)])
    assert perm.tolist() == np.argsort(norm, kind="stable").tolist()
    k3 = _index_kernel(tmp_path / "c", "put_rows_kernel", ctype, {"T": ctype}, smem="put_smem")
    x = rng.standard_normal((outer, n_dst)).astype(dtype)
    y = rng.standard_normal((outer, n_idx)).astype(dtype)
    want = x.copy()
    np.add.at(want, (slice(None), idx), y)
    wpb = 4
    k3.launch(2, 256, [_ptr(x), _ptr(y), _ptr(offsets), _ptr(perm), c_longlong(outer), c_longlong(n_dst), c_longlong(n_idx), c_int(wpb)])
    if dtype == np.float64:
        np.testing.assert_array_equal(x, want)
    else:
        np.testing.assert_allclose(x, want, rtol=1e-5, atol=1e-5)


class _Dims(ctypes.Structure):
    _fields_ = [("ndim", c_int), ("shape", c_longlong * 8), ("a", c_longlong * 8), ("b", c_longlong * 8)]


COLLAPSE_EXPORT = r"""
extern "C" long long emu_collapse(Dims* d, const int64_t* shape, const int64_t* sa, const int64_t* sb, int ndim) {
  return collapse(*d, shape, sa, sb, ndim);
}
"""


@pytest.mark.parametrize("kernel,ctype,dtype", [("copy_strided_kernel", "uint32_t", np.float32), ("copy_strided_kernel", "uint64_t", np.float64),
                                                ("inc_strided_kernel", "float", np.float32), ("inc_strided_kernel", "int16_t", np.int16)])
def test_strided_copy_and_increment_with_collapsed_dims(tmp_path, kernel, ctype, dtype):
    """dst[...] = src[...] / dst[...] += src[...] over up-to-8-d element strides: the host-side dimension collapse (size-1 dims
    dropped, neighbours contiguous in BOTH operands merged) and the kernel's mixed-radix walk, on a transposed + reversed +
    broadcast source and a sliced destination (DeepCopyOp / Alloc / IncSubtensor: compile/ops.py:121, tensor/basic.py:1545,
    tensor/subtensor.py:1441)."""
    rng = np.random.default_rng(45)
    text = open(os.path.join(CSRC, "ptk_index.cu")).read()
    src_txt = text[text.index("constexpr int kMaxDims"):text.index("// Contiguous destination and source both 16-byte aligned")]
    if kernel == "inc_strided_kernel":
        src_txt += extract_static_kernel(os.path.join(CSRC, "ptk_index.cu"), kernel)
    k = EmulatedKernel(src_txt + COLLAPSE_EXPORT, kernel, tmp_path, template_args=ctype, type_subst={"T": ctype})
    mk = (lambda shape: (rng.standard_normal(shape) * 50).astype(dtype))
    dbuf = mk((6, 5, 4, 10))
    sbuf = mk((7, 1, 4, 6))
    dst = dbuf[1:6, :, :, 2:9:2]                       # (5, 5, 4, 4): sliced rows, strided last axis
    src = np.broadcast_to(sbuf.transpose(3, 1, 2, 0)[::-1][:5, :, :, 1:5], (5, 5, 4, 4))   # reversed, broadcast, transposed
    want = src.copy() if kernel == "copy_strided_kernel" else (dst + src).astype(dtype)
    isz = dbuf.itemsize
    shape = (c_longlong * 4)(*dst.shape)
    sa = (c_longlong * 4)(*[s // isz for s in dst.strides])
    sb = (c_longlong * 4)(*[s // isz for s in src.strides])
    d = _Dims()
    k.lib.emu_collapse.restype = c_longlong
    total = k.lib.emu_collapse(ctypes.byref(d), shape, sa, sb, 4)
    assert total == dst.size and 1 <= d.ndim <= 4
    before = dbuf.copy()
    k.launch(3, 256, [c_void_p(dst.ctypes.data), c_void_p(src.ctypes.data), d, c_longlong(total)])
    np.testing.assert_array_equal(dst, want)
    mask = np.ones(dbuf.shape, dtype=bool)
    mask[1:6, :, :, 2:9:2] = False
    np.testing.assert_array_equal(dbuf[mask], before[mask])      # nothing outside the destination window is touched
    # fully contiguous operands collapse to ONE dimension (the 128-bit streaming copy's precondition)
    c_shape = (c_longlong * 3)(4, 1, 6)
    c_st = (c_longlong * 3)(6, 6, 1)
    assert k.lib.emu_collapse(ctypes.byref(d), c_shape, c_st, c_st, 3) == 24 and d.ndim == 1 and d.shape[0] == 24 and d.a[0] == 1


# ---- Cholesky / triangular solve kernels (ptk_linalg.cu) -------------------------------------------------------------------
LINALG_SHIM = r"""
#define CUDART_NAN_F NAN
#define CUDART_NAN ((double)NAN)
using std::sqrt;
template <typename T> static inline T __shfl_sync(unsigned, T v, int src) { return emu_exchange(v, (int)((threadIdx.x & ~31u) + src)); }
"""


def _linalg_kernel(tmp_path, name, ctype, smem=None):
    text = open(os.path.join(CSRC, "ptk_linalg.cu")).read()
    head = text[text.index("constexpr int NB = 64;"):text.index("// ---- small path")]
    src = LINALG_SHIM + head + extract_static_kernel(os.path.join(CSRC, "ptk_linalg.cu"), name)
    return EmulatedKernel(src, name, tmp_path, threaded=True, template_args=ctype, type_subst={"T": ctype}, dynamic_smem=smem)


def _spd(rng, n, dtype):
    a = rng.standard_normal((n, n))
    return (a @ a.T + n * np.eye(n)).astype(dtype)


@pytest.mark.parametrize("dtype,ctype,n,lower,threads", [("float64", "double", 37, True, 64), ("float32", "float", 96, True, 256),
                                                        ("float64", "double", 20, False, 64), ("float64", "double", 1, True, 64)])
def test_small_cholesky_kernel(tmp_path, dtype, ctype, n, lower, threads):
    """One CTA per matrix of a batch, left-looking, lanes along the dot-product index; upper = the lower algorithm on the
    transposed view; the other triangle is zeroed; a matrix that is not positive definite comes back all-NaN while its batch
    neighbours are factored (pytensor/tensor/linalg/decomposition/cholesky.py:52-83)."""
    rng = np.random.default_rng(51)
    k = _linalg_kernel(tmp_path, "potrf_small_kernel", ctype, smem="smem_raw")
    batch = 3
    A = np.stack([_spd(rng, n, dtype) for _ in range(batch)])
    A0 = A.copy()
    if n > 1:
        A[1, n // 2, n // 2] = -1.0     # breaks positive definiteness of the middle matrix only
    rs, cs = (n, 1) if lower else (1, n)
    k.launch(batch, threads, [_ptr(A), c_longlong(n), c_longlong(rs), c_longlong(cs), c_longlong(n * n)])
    tol = 2e-4 if dtype == "float32" else 1e-11
    for b in range(batch):
        if b == 1 and n > 1:
            assert np.all(np.isnan(A[b]))
            continue
        L = np.linalg.cholesky(A0[b].astype(np.float64))
        np.testing.assert_allclose(A[b], L if lower else L.T, rtol=tol, atol=tol * np.abs(L).max())


@pytest.mark.parametrize("dtype,ctype,n", [("float64", "double", 150), ("float32", "float", 130)])
def test_blocked_cholesky_kernels_compose(tmp_path, dtype, ctype, n):
    """The right-looking blocked algorithm of ptk_potrf (n > 128) step by step: diagonal-block kernel, warp-per-row panel solve,
    trailing update (NumPy stands in for ptk_gemm here), final clean-up; 64-wide panels with a short last one."""
    rng = np.random.default_rng(52)
    (tmp_path / "d").mkdir(), (tmp_path / "p").mkdir(), (tmp_path / "c").mkdir()
    kd = _linalg_kernel(tmp_path / "d", "potrf_diag_kernel", ctype)
    kp = _linalg_kernel(tmp_path / "p", "potrf_panel_kernel", ctype)
    kc = _linalg_kernel(tmp_path / "c", "potrf_clean_kernel", ctype)
    A = _spd(rng, n, dtype)
    want = np.linalg.cholesky(A.astype(np.float64))
    flag = np.zeros(1, dtype=np.int32)
    isz = A.itemsize
    at = lambda r, c: c_void_p(A.ctypes.data + (r * n + c) * isz)  # noqa: E731
    for k0 in range(0, n, 64):
        kb = min(64, n - k0)
        kd.launch(1, 64, [at(k0, k0), c_longlong(n), c_longlong(1), c_int(kb), _ptr(flag)])
        m = n - k0 - kb
        if m > 0:
            kp.launch(2, 256, [at(k0, k0), at(k0 + kb, k0), c_longlong(n), c_longlong(1), c_int(kb), c_longlong(m)])
            A21 = A[k0 + kb:, k0:k0 + kb]
            A[k0 + kb:, k0 + kb:] -= A21 @ A21.T
    kc.launch(3, 256, [_ptr(A), c_longlong(n), c_longlong(n), c_longlong(1), _ptr(flag)])
    assert flag[0] == 0
    tol = 3e-4 if dtype == "float32" else 1e-10
    np.testing.assert_allclose(A, want, rtol=tol, atol=tol * np.abs(want).max())
    # a non-positive pivot inside a diagonal block raises the flag; the clean-up kernel then NaN-fills the whole matrix
    B = _spd(rng, 40, dtype)
    B[17, 17] = -5.0
    kd.launch(1, 64, [_ptr(B), c_longlong(40), c_longlong(1), c_int(40), _ptr(flag)])
    assert flag[0] == 1
    kc.launch(1, 256, [_ptr(B), c_longlong(40), c_longlong(40), c_longlong(1), _ptr(flag)])
    assert np.all(np.isnan(B))


@pytest.mark.parametrize("dtype,ctype,n,nrhs,lower,trans,unit", [("float64", "double", 45, 70, 1, 0, 0), ("float32", "float", 33, 5, 0, 0, 0),
                                                                 ("float64", "double", 20, 33, 1, 1, 0), ("float64", "double", 16, 8, 0, 1, 1)])
def test_small_triangular_solve_kernel(tmp_path, dtype, ctype, n, nrhs, lower, trans, unit):
    """op(A) X = B by substitution, one CTA per 32 right-hand sides, `trans` folded into the strides; unit_diag never reads the
    diagonal; an exactly-zero diagonal element NaN-fills the solution (pytensor/tensor/linalg/solvers/triangular.py:41-71)."""
    import scipy.linalg as sl

    rng = np.random.default_rng(53)
    k = _linalg_kernel(tmp_path, "trsm_small_kernel", ctype)
    batch = 2
    tri = np.tril if lower else np.triu
    A = np.stack([tri(rng.standard_normal((n, n))) + 4 * np.eye(n) for _ in range(batch)]).astype(dtype)
    if unit:
        for b in range(batch):
            A[b][np.diag_indices(n)] = np.nan    # must not be read
    B = rng.standard_normal((batch, n, nrhs)).astype(dtype)
    B0 = B.copy()
    ars, acs = (1, n) if trans else (n, 1)
    fwd = 1 if (bool(lower) != bool(trans)) else 0
    args = [_ptr(A), _ptr(B), c_longlong(n), c_longlong(nrhs), c_longlong(ars), c_longlong(acs), c_int(fwd), c_int(unit)]
    k.launch(((nrhs + 31) // 32, batch), 256, args)
    tol = 2e-4 if dtype == "float32" else 1e-10
    for b in range(batch):
        Ab = A[b].astype(np.float64)
        if unit:
            Ab[np.diag_indices(n)] = 1.0
        want = sl.solve_triangular(Ab, B0[b].astype(np.float64), lower=bool(lower), trans=trans, unit_diagonal=bool(unit))
        np.testing.assert_allclose(B[b], want, rtol=tol, atol=tol * np.abs(want).max())
    if not unit:
        A[0, n // 3, n // 3] = 0.0
        B[:] = B0
        k.launch(((nrhs + 31) // 32, batch), 256, args)
        assert np.all(np.isnan(B[0])) and np.all(np.isfinite(B[1]))


@pytest.mark.parametrize("fwd,unit", [(1, 0), (0, 0), (1, 1)])
def test_blocked_triangular_solve_diagonal_block_kernel(tmp_path, fwd, unit):
    rng = np.random.default_rng(54)
    import scipy.linalg as sl

    k = _linalg_kernel(tmp_path, "trsm_diag_kernel", "double")
    kb, nrhs, n = 50, 200, 70      # a kb x kb diagonal block inside an n x n matrix (row stride n)
    A = (np.tril(rng.standard_normal((n, n))) if fwd else np.triu(rng.standard_normal((n, n)))) + 5 * np.eye(n)
    B = rng.standard_normal((kb, nrhs))
    B0 = B.copy()
    off = 10
    A11 = A[off:off + kb, off:off + kb]
    k.launch((nrhs + 127) // 128, 128, [c_void_p(A.ctypes.data + (off * n + off) * 8), c_longlong(n), c_longlong(1), _ptr(B),
                                         c_longlong(nrhs), c_int(kb), c_int(fwd), c_int(unit)])
    want = sl.solve_triangular(A11, B0, lower=bool(fwd), unit_diagonal=bool(unit))
    np.testing.assert_allclose(B, want, rtol=1e-10, atol=1e-10 * np.abs(want).max())


# ---- ARange / Argmax / CumOp / index linearisation (ptk_misc.cu) --------------------------------------------------------------
MISC_SHIM = r"""
#include <type_traits>
static inline float __fmul_rn(float a, float b) { volatile float p = a * b; return p; }     // volatile: no FMA contraction
static inline float __fadd_rn(float a, float b) { volatile float s = a + b; return s; }
static inline double __dmul_rn(double a, double b) { volatile double p = a * b; return p; }
static inline double __dadd_rn(double a, double b) { volatile double s = a + b; return s; }
template <typename T> static inline T __shfl_sync(unsigned, T v, int src) { return emu_exchange(v, (int)((threadIdx.x & ~31u) + src)); }
"""


def _misc_kernel(tmp_path, name, targs, subst, head=""):
    src = MISC_SHIM + head + extract_static_kernel(os.path.join(CSRC, "ptk_misc.cu"), name)
    return EmulatedKernel(src, name, tmp_path, threaded=True, template_args=targs, type_subst=subst)


def test_arange_kernels_round_like_numpy(tmp_path):
    """out[i] = first + i*delta in the OUTPUT type with two roundings (no FMA), like NumPy's <type>_fill; integers wrap."""
    (tmp_path / "f").mkdir(), (tmp_path / "d").mkdir(), (tmp_path / "i").mkdir()
    n = 3000
    kf = _misc_kernel(tmp_path / "f", "arange_float_kernel", "float", {"T": "float"})
    out = np.zeros(n, dtype=np.float32)
    kf.launch(3, 256, [_ptr(out), c_longlong(n), c_float(0.1), c_float(0.3)])
    i = np.arange(n, dtype=np.float32)
    np.testing.assert_array_equal(out, np.float32(0.1) + i * np.float32(0.3))
    kd = _misc_kernel(tmp_path / "d", "arange_float_kernel", "double", {"T": "double"})
    outd = np.zeros(n, dtype=np.float64)
    kd.launch(3, 256, [_ptr(outd), c_longlong(n), c_double(-7.7), c_double(1e-3)])
    np.testing.assert_array_equal(outd, -7.7 + np.arange(n, dtype=np.float64) * 1e-3)
    ki = _misc_kernel(tmp_path / "i", "arange_int_kernel", "int8_t", {"T": "int8_t"})
    outi = np.zeros(n, dtype=np.int8)
    ki.launch(2, 256, [_ptr(outi), c_longlong(n), c_longlong(-5), c_longlong(3)])
    np.testing.assert_array_equal(outi, (-5 + 3 * np.arange(n, dtype=np.int64)).astype(np.int8))


def _argmax_head():
    text = open(os.path.join(CSRC, "ptk_misc.cu")).read()
    return text[text.index("template <typename T>\n__device__ __forceinline__ bool is_nan_v"):text.index("// inner == 1: one warp (small rows)")]


@pytest.mark.parametrize("threads,rows,n", [(32, 70, 100), (256, 5, 3000), (256, 3, 7), (32, 4, 1)])
def test_argmax_rows_kernel_first_maximum_and_nan(tmp_path, threads, rows, n):
    """np.argmax along the last axis: the FIRST maximal element wins across lanes, warps and strides; the first NaN wins
    over everything (pytensor/tensor/math.py Argmax.perform = np.argmax)."""
    rng = np.random.default_rng(61)
    k = _misc_kernel(tmp_path, "argmax_rows_kernel", f"float, {threads}", {"T": "float"}, head=_argmax_head())
    x = rng.integers(0, 6, size=(rows, n)).astype(np.float32)     # few distinct values: many ties
    if n > 5:
        x[1, n // 2] = np.nan
        x[1, n - 1] = np.nan
        x[2, :] = 3.0
    out = np.full(rows, -1, dtype=np.int64)
    k.launch(2, threads, [_ptr(x), _ptr(out), c_longlong(rows), c_longlong(n)])
    np.testing.assert_array_equal(out, np.argmax(x, axis=1))


def test_argmax_cols_kernel(tmp_path):
    rng = np.random.default_rng(62)
    k = _misc_kernel(tmp_path, "argmax_cols_kernel", "int32_t", {"T": "int32_t"}, head=_argmax_head())
    x = rng.integers(-4, 4, size=(3, 17, 40)).astype(np.int32)
    out = np.full((3, 40), -1, dtype=np.int64)
    k.launch(2, 256, [_ptr(x), _ptr(out), c_longlong(3), c_longlong(17), c_longlong(40)])
    np.testing.assert_array_equal(out, np.argmax(x, axis=1))


@pytest.mark.parametrize("ctype,dtype,op", [("int64_t", np.int64, 0), ("double", np.float64, 0), ("int32_t", np.int32, 1), ("float", np.float32, 1)])
def test_cumulative_kernels(tmp_path, ctype, dtype, op):
    """CumOp (pytensor/tensor/extra_ops.py: np.cumsum / np.cumprod): warp scan with a carried total along the last axis,
    one sequential thread per line otherwise — integers bit-exact (wrapping products included), floats within rounding
    (rows kernel) or bit-exact (columns kernel, same order as NumPy)."""
    rng = np.random.default_rng(63)
    (tmp_path / "r").mkdir(), (tmp_path / "c").mkdir()
    head = ("template <typename T, int OP>\n__device__ __forceinline__ T cum_combine(T a, T b) {\n"
            "  return OP == 0 ? (T)(a + b) : (T)(a * b);\n}\n")
    assert head in open(os.path.join(CSRC, "ptk_misc.cu")).read()
    kr = _misc_kernel(tmp_path / "r", "cum_rows_kernel", f"{ctype}, {op}", {"T": ctype}, head=head)
    kc = _misc_kernel(tmp_path / "c", "cum_cols_kernel", f"{ctype}, {op}", {"T": ctype}, head=head)
    f = np.cumsum if op == 0 else np.cumprod
    if np.issubdtype(dtype, np.integer):
        x = rng.integers(-3, 4, size=(9, 77)).astype(dtype)
    else:
        x = (1.0 + 0.1 * rng.standard_normal((9, 77))).astype(dtype)
    out = np.zeros_like(x)
    kr.launch(1, 256, [_ptr(x), _ptr(out), c_longlong(9), c_longlong(77)])
    want = f(x, axis=1, dtype=dtype)
    if np.issubdtype(dtype, np.integer):
        np.testing.assert_array_equal(out, want)
    else:
        np.testing.assert_allclose(out, want, rtol=2e-5 if dtype == np.float32 else 1e-13)
    x3 = x.reshape(3, 3, 77).transpose(0, 2, 1).copy()       # (outer 3, n 77, inner 3)
    out3 = np.zeros_like(x3)
    kc.launch(1, 256, [_ptr(x3), _ptr(out3), c_longlong(3), c_longlong(77), c_longlong(3)])
    np.testing.assert_array_equal(out3, f(x3, axis=1, dtype=dtype))


class _LinIdxArgs(ctypes.Structure):
    _fields_ = [("idx", c_void_p * 8), ("dim", c_longlong * 8), ("stride", c_longlong * 8), ("k", c_int)]


def test_linearize_index_kernel(tmp_path):
    """Several integer index arrays on consecutive axes -> one linear index (np.ravel_multi_index with NumPy's per-axis
    negative wrap); any out-of-range component raises the error word."""
    rng = np.random.default_rng(64)
    text = open(os.path.join(CSRC, "ptk_misc.cu")).read()
    head = text[text.index("struct LinIdxArgs {"):text.index("__global__ void linearize_index_kernel")]
    k = _misc_kernel(tmp_path, "linearize_index_kernel", "", None, head=head)
    dims, n = (5, 7, 3), 500
    idx = [rng.integers(-d, d, size=n).astype(np.int64) for d in dims]
    a = _LinIdxArgs()
    a.k = 3
    for j, d in enumerate(dims):
        a.idx[j] = idx[j].ctypes.data
        a.dim[j] = d
        a.stride[j] = int(np.prod(dims[j + 1:]))
    out = np.zeros(n, dtype=np.int64)
    err = np.zeros(1, dtype=np.int32)
    k.launch(2, 256, [a, c_longlong(n), _ptr(out), _ptr(err)])
    np.testing.assert_array_equal(out, np.ravel_multi_index([np.where(i < 0, i + d, i) for i, d in zip(idx, dims)], dims))
    assert err[0] == 0
    idx[1][123] = 7
    k.launch(2, 256, [a, c_longlong(n), _ptr(out), _ptr(err)])
    assert err[0] == 1


BF16_PAIR_SHIM = r"""
static inline __nv_bfloat162 __floats2bfloat162_rn(float a, float b) { __nv_bfloat162 r; r.x = __float2bfloat16_rn(a); r.y = __float2bfloat16_rn(b); return r; }
"""


def _bf16_round(x):
    """float32 -> bf16 (round to nearest even) -> float64, NumPy restatement."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    return (b.astype(np.uint32) << 16).view(np.float32).astype(np.float64)


@pytest.mark.parametrize("R,Cc,row_major", [(70, 130, True), (130, 70, False), (64, 63, True), (3, 9, False)])
def test_plain_bf16_staging_kernels(tmp_path, R, Cc, row_major):
    """ptk_stage_operand's plain variants: one bf16 matrix (bf16 mode), or the three-piece split x1 = bf16(x), x2 = bf16(x - x1),
    x3 = bf16(x - x1 - x2) stacked with a pitch of piece_rows rows; either source stride may be the unit one (the B operand
    is staged transposed); odd column counts end in a zero / untouched pad inside the 8-element row pitch."""
    rng = np.random.default_rng(R + 7 * Cc)
    x = (rng.standard_normal((R, Cc)) * np.exp(rng.uniform(-8, 8, (R, Cc)))).astype(np.float32)
    src = np.ascontiguousarray(x if row_major else x.T)
    sr, sc = (Cc, 1) if row_major else (1, R)
    ld, pr = (Cc + 7) // 8 * 8, (R + 255) // 256 * 256
    grid = ((Cc + 63) // 64, (R + 63) // 64)
    (tmp_path / "c").mkdir(), (tmp_path / "s").mkdir()
    shim = BF16_SHIM + BF16_PAIR_SHIM
    kc = EmulatedKernel(shim + extract_static_kernel(os.path.join(CSRC, "ptk_gemm_tc.cu"), "convert_bf16_kernel"),
                        "convert_bf16_kernel", tmp_path / "c", threaded=True)
    one = np.full((R, ld), 0xABCD, dtype=np.uint16)
    kc.launch(grid, 256, [_ptr(src), c_longlong(sr), c_longlong(sc), _ptr(one), c_longlong(ld), c_longlong(R), c_longlong(Cc)])
    got = (one[:, :Cc].astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    np.testing.assert_array_equal(got, _bf16_round(x))
    ks = EmulatedKernel(shim + extract_static_kernel(os.path.join(CSRC, "ptk_gemm_tc.cu"), "split_bf16x3_kernel"),
                        "split_bf16x3_kernel", tmp_path / "s", threaded=True)
    dst = np.zeros((3 * pr, ld), dtype=np.uint16)
    ks.launch(grid, 256, [_ptr(src), c_longlong(sr), c_longlong(sc), _ptr(dst), c_longlong(ld), c_longlong(R), c_longlong(Cc),
                          c_longlong(pr)])
    p = [(dst[k * pr:k * pr + R, :Cc].astype(np.uint32) << 16).view(np.float32).astype(np.float64) for k in range(3)]
    x64 = x.astype(np.float64)
    np.testing.assert_array_equal(p[0], _bf16_round(x))
    r1 = (x64 - p[0]).astype(np.float32)          # exact in fp32
    np.testing.assert_array_equal(p[1], _bf16_round(r1))
    np.testing.assert_array_equal(p[2], _bf16_round((r1.astype(np.float64) - p[1]).astype(np.float32)))
    assert np.all(np.abs(p[0] + p[1] + p[2] - x64) <= np.abs(x64) * 2.0 ** -22)
    assert not dst[R:pr].any() and not dst[pr + R:2 * pr].any()     # rows between the pieces stay untouched


def _special_rows(R, Cc, rng):
    """Finite normal values except: ±inf next to zeros, tiny and normal values (row 0), NaN (row 1), a row whose largest
    magnitude lies in the top binade above 127.5 * 2^121 (row 2), fp32 denormals (row 3), -inf alone (row 4)."""
    x = rng.standard_normal((R, Cc)).astype(np.float32)
    x[0, :6] = [np.inf, 0.0, 1e-3, -1e-3, -np.inf, 2.0]
    x[1, 3] = np.nan
    x[2, :] = (rng.uniform(-1, 1, Cc) * 3.0e38).astype(np.float32)
    x[2, 1] = np.float32(3.40e38)          # (rounds to inf in bf16)
    x[3, :] = (rng.standard_normal(Cc) * 1e-40).astype(np.float32)
    x[4, :] = 0.0
    x[4, Cc - 1] = -np.inf
    return x


@pytest.mark.parametrize("aligned", [False, True])
@pytest.mark.parametrize("R,Cc,row_major", [(70, 130, True), (9, 67, False)])
def test_three_piece_splits_of_non_finite_and_extreme_values(tmp_path, R, Cc, row_major, aligned):
    """Both three-piece splits (split_bf16x3_kernel, split_aligned_kernel): a non-finite x is staged as (x, 0, 0) — a NaN
    remainder would turn every piece product into NaN — and every finite x, the top binade and denormals included, as
    finite pieces summing to x.  The row maxima row_absmax_kernel leaves (ptk_stage_operand runs it for either split) are
    +inf exactly for the rows holding ±inf: the flags that make the GEMM recompute those rows' outputs."""
    rng = np.random.default_rng(R + Cc)
    x = _special_rows(R, Cc, rng)
    src = np.ascontiguousarray(x if row_major else x.T)
    sr, sc = (Cc, 1) if row_major else (1, R)
    ld, pr = (Cc + 7) // 8 * 8, (R + 255) // 256 * 256
    grid = ((Cc + 63) // 64, (R + 63) // 64)
    cu = os.path.join(CSRC, "ptk_gemm_tc.cu")
    text = open(cu).read()
    dst = np.zeros((3 * pr, ld), dtype=np.uint16)
    flags = np.zeros(R, dtype=np.uint32)
    (tmp_path / "m").mkdir(), (tmp_path / "s").mkdir()
    k1 = EmulatedKernel(BF16_SHIM + ATOMIC_SHIM + extract_static_kernel(cu, "row_absmax_kernel"), "row_absmax_kernel",
                        tmp_path / "m", threaded=True)
    k1.launch(grid, 256, [_ptr(src), c_longlong(sr), c_longlong(sc), c_longlong(R), c_longlong(Cc), _ptr(flags)])
    if aligned:
        i0 = text.index("__device__ __forceinline__ int scale_exp_of")
        helper = text[i0:text.index("\n}\n", i0) + 3]
        k2 = EmulatedKernel(BF16_SHIM + ATOMIC_SHIM + helper + extract_static_kernel(cu, "split_aligned_kernel"),
                            "split_aligned_kernel", tmp_path / "s", threaded=True)
        k2.launch(grid, 256, [_ptr(src), c_longlong(sr), c_longlong(sc), _ptr(dst), c_longlong(ld), c_longlong(R),
                              c_longlong(Cc), c_longlong(pr), _ptr(flags), c_int(7)])
    else:
        ks = EmulatedKernel(BF16_SHIM + BF16_PAIR_SHIM + extract_static_kernel(cu, "split_bf16x3_kernel"),
                            "split_bf16x3_kernel", tmp_path / "s", threaded=True)
        ks.launch(grid, 256, [_ptr(src), c_longlong(sr), c_longlong(sc), _ptr(dst), c_longlong(ld), c_longlong(R),
                              c_longlong(Cc), c_longlong(pr)])
    has_inf = np.isinf(x).any(axis=1)
    np.testing.assert_array_equal(flags == 0x7F800000, has_inf)
    p = [(dst[k * pr:k * pr + R, :Cc].astype(np.uint32) << 16).view(np.float32).astype(np.float64) for k in range(3)]
    x64 = x.astype(np.float64)
    fin = np.isfinite(x)
    np.testing.assert_array_equal(p[0][~fin], x64[~fin])               # inf keeps its sign, NaN stays NaN
    assert not p[1][~fin].any() and not p[2][~fin].any()
    assert all(np.isfinite(q[fin]).all() for q in p)
    err = np.abs((p[0] + p[1] + p[2])[fin] - x64[fin])
    if aligned:
        # finite rows: 2^-23 of the row maximum; a row holding ±inf has no scale (unit 1): the remainder |x - rint(x)| <= 1/2
        # carries 16 bits through the two correction pieces
        rowmax = np.abs(np.where(fin, x64, 0.0)).max(axis=1)
        bound = np.where(has_inf, 2.0 ** -17, rowmax * 2.0 ** -23)[:, None] * np.ones_like(x64)
        bound = np.maximum(bound, 2.0 ** -134)[fin]
    else:
        bound = np.maximum(np.abs(x64) * 2.0 ** -22, 2.0 ** -134)[fin]   # (bf16 denormals end at 2^-133)
    assert np.all(err <= bound), (err - bound).max()
