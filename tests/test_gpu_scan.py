"""Scan on the device (K7): general loop and the persistent fused kernel, against the reference (Cython loop + CVM).
Known-answer cases follow tests/scan/test_basic.py (ScanCompatibilityTests :4060-4173, [44, 38] :3984-4057)."""

import numpy as np
import pytest

from helpers import compare_cuda_and_cvm, pytensor

import pytensor.tensor as pt
from pytensor.scan.basic import scan

pytestmark = pytest.mark.gpu


def _is_fused(f):
    return any("ScanFused" in type(st.impl).__name__ for st in f.vm.executor.program.steps)


@pytest.mark.parametrize("last_only", [True, False])
def test_cfg4_elementwise_recurrence(gpu, last_only):
    pytensor.config.floatX = "float32"
    from pytensor_b200 import workloads as W

    ins, outs, make_args, _ = W.cfg4_scan(96, 40, 57, full_trace=not last_only)
    args = make_args()
    # contractive gain (|a| < 1): libm-vs-CUDA tanhf ulp differences must not be amplified step after step, otherwise the
    # comparison measures the recurrence's Lyapunov growth instead of the kernel
    args[1] = np.random.default_rng(5).uniform(0.3, 0.9, args[1].shape).astype("float32")
    f, _ = compare_cuda_and_cvm(ins, outs, args, rtol=2e-5, atol=2e-5)
    assert _is_fused(f)


def test_cfg4_matmul_recurrence_general_loop(gpu):
    pytensor.config.floatX = "float32"
    from pytensor_b200 import workloads as W

    ins, outs, make_args, _ = W.cfg4_scan(64, 32, 20, matmul=True)
    f, _ = compare_cuda_and_cvm(ins, outs, make_args(), rtol=1e-4, atol=1e-5)
    assert not _is_fused(f)
    # h <- tanh(h @ W + b) alone in the loop: a chain of GEMM launches writing straight into the tap buffer
    assert any(type(st.impl).__name__ == "ScanMatmulRecurrenceNode" for st in f.vm.executor.program.steps)


def _contractive(args, gain=0.6):
    # |W| scaled below the edge of chaos: rounding differences between two sgemm implementations must decay, not grow
    args = list(args)
    args[1] = (args[1] * gain).astype("float32")
    return args


@pytest.mark.parametrize("full_trace", [False, True])
@pytest.mark.parametrize("rows,cols,steps", [(300, 256, 9), (512, 384, 25)])
def test_matmul_recurrence_on_tensor_cores_chained_operands(gpu, rows, cols, steps, full_trace):
    """dims >= 256: the fp32-accurate tensor-core path — W staged once, every step's epilogue writes the three-piece staged
    operand of the next step (nodes_scan_matmul.py); final state (2-slot circular buffer) and full trace, vs the C linker."""
    pytensor.config.floatX = "float32"
    from pytensor_b200 import workloads as W

    ins, outs, make_args, _ = W.cfg4_scan(rows, cols, steps, matmul=True, full_trace=full_trace)
    f, _ = compare_cuda_and_cvm(ins, outs, _contractive(make_args()), rtol=1e-5, atol=1e-5)
    assert any(type(st.impl).__name__ == "ScanMatmulRecurrenceNode" for st in f.vm.executor.program.steps)


def test_matmul_recurrence_variants(gpu):
    pytensor.config.floatX = "float32"
    rng = np.random.default_rng(61)
    h0, Wm = pt.fmatrix("h0"), pt.fmatrix("W")
    n = pt.lscalar("n")
    h0v = rng.standard_normal((260, 256)).astype("float32")
    Wv = (rng.standard_normal((256, 256)) * 0.03).astype("float32")
    # no bias, no activation, symbolic n_steps (0, 1 and many), last three states only (truncated buffer)
    hs = scan(lambda h, W: pt.dot(h, W), outputs_info=[h0], non_sequences=[Wm], n_steps=n, return_updates=False)
    for steps in (0, 1, 7):
        outs = [hs] if steps == 0 else [hs, hs[-1]]
        compare_cuda_and_cvm([h0, Wm, n], outs, [h0v, Wv, steps], rtol=1e-5, atol=1e-5)
    hs = scan(lambda h, W: pt.tanh(pt.dot(h, W)), outputs_info=[h0], non_sequences=[Wm], n_steps=12, return_updates=False)
    f, _ = compare_cuda_and_cvm([h0, Wm], [hs[-3:]], [h0v, Wv], rtol=1e-5, atol=1e-5)
    assert any(type(st.impl).__name__ == "ScanMatmulRecurrenceNode" for st in f.vm.executor.program.steps)
    # bf16 tensor-core mode: the chained operand is the bf16 copy; compared at bf16 accuracy
    f16 = pytensor.function([h0, Wm], hs[-1], mode="CUDA_BF16")
    ref = pytensor.function([h0, Wm], hs[-1], mode="CVM")(h0v, Wv)
    assert np.abs(f16(h0v, Wv) - ref).max() < 2e-2
    # fp64 state: FMA kernel per step, still in place
    pytensor.config.floatX = "float64"
    g0, Wd = pt.dmatrix("g0"), pt.dmatrix("Wd")
    gs = scan(lambda h, W: pt.tanh(pt.dot(h, W)), outputs_info=[g0], non_sequences=[Wd], n_steps=5, return_updates=False)
    compare_cuda_and_cvm([g0, Wd], [gs, gs[-1]], [h0v[:, :64].astype("float64"), Wv[:64, :64].astype("float64")])


def test_sequences_mit_sot_nit_sot(gpu):
    rng = np.random.default_rng(51)
    u = pt.dmatrix("u")          # sequence (T, n)
    x0 = pt.dmatrix("x0")        # two initial taps (2, n)
    w = pt.dvector("w")

    def step(u_t, x_tm2, x_tm1, w):
        x_t = 0.5 * x_tm1 - 0.25 * x_tm2 + pt.tanh(u_t * w)
        return x_t, pt.exp(-x_t * x_t)

    (xs, ys) = scan(step, sequences=[u], outputs_info=[dict(initial=x0, taps=[-2, -1]), None], non_sequences=[w],
                    return_updates=False)
    uv = rng.standard_normal((23, 17))
    x0v = rng.standard_normal((2, 17))
    wv = rng.standard_normal(17)
    f, _ = compare_cuda_and_cvm([u, x0, w], [xs, ys, xs[-1], ys[-3:].sum(axis=0)], [uv, x0v, wv], rtol=1e-9, atol=1e-9)
    assert _is_fused(f)


def test_scalar_power_recurrence_and_grad(gpu):
    # x ** 16 via repeated multiplication and its gradient (ScanCompatibilityTests, tests/scan/test_basic.py:4060-4110)
    x = pt.dscalar("x")
    ys = scan(lambda acc, x: acc * x, outputs_info=[pt.ones((), dtype="float64")], non_sequences=[x], n_steps=16,
              return_updates=False)
    y = ys[-1]
    g = pytensor.grad(y, x)
    compare_cuda_and_cvm([x], [y, g], [np.float64(1.1)], rtol=1e-9)


def test_until_and_n_steps_zero(gpu):
    n = pt.lscalar("n")
    from pytensor.scan.utils import until

    zs = scan(lambda z: (z + 1.0, until(z > 2)), outputs_info=[pt.zeros((), dtype="float64")], n_steps=n,
              return_updates=False)
    compare_cuda_and_cvm([n], [zs, zs.sum()], [np.int64(10)])
    compare_cuda_and_cvm([n], [zs.sum()], [np.int64(2)])
    compare_cuda_and_cvm([n], [zs.sum()], [np.int64(0)])


def test_grad_through_scan_mit_mot(gpu):
    rng = np.random.default_rng(52)
    h0 = pt.dvector("h0")
    W = pt.dmatrix("W")
    hs = scan(lambda h, W: pt.tanh(pt.dot(h, W)), outputs_info=[h0], non_sequences=[W], n_steps=6,
              return_updates=False)
    cost = (hs ** 2).sum()
    gW, gh = pytensor.grad(cost, [W, h0])
    compare_cuda_and_cvm([h0, W], [cost, gW, gh], [rng.standard_normal(7), rng.standard_normal((7, 7)) * 0.5],
                         rtol=1e-8, atol=1e-9)


def test_known_answer_two_mit_mots(gpu):
    # hand-built Scan with two MIT-MOTs: expected [44, 38] (tests/scan/test_basic.py:3984-4057)
    from pytensor.scan.op import Scan, ScanInfo
    from pytensor.tensor import as_tensor

    info = ScanInfo(n_seqs=1, mit_mot_in_slices=((0, 1), (0, 1)), mit_mot_out_slices=((1,), (1,)),
                    mit_sot_in_slices=(), sit_sot_in_slices=(), n_nit_sot=0, n_untraced_sit_sot=0, n_non_seqs=0,
                    as_while=False)
    bool_seq = pt.scalar(dtype="bool")
    A0, A1, B0, B1 = (pt.matrix(shape=(2, 2), dtype="float64") for _ in range(4))
    outputs = [pt.add(bool_seq + A0, A1), pt.add(bool_seq * B0, B1)]
    op = Scan([bool_seq, A0, A1, B0, B1], outputs, info=info)
    n_steps = 5
    vals = [np.array(n_steps, dtype="int64"), np.array([1, 1, 0, 1, 0], dtype="bool"),
            np.zeros(n_steps + 1)[:, None, None] * np.eye(2), np.arange(n_steps + 1)[:, None, None] * np.eye(2)]
    tins = [as_tensor(v, dtype=v.dtype).type() for v in vals]
    touts = [o.sum() for o in op(*tins)]
    f = pytensor.function(tins, touts, mode="CUDA")
    np.testing.assert_allclose(f(*vals), [44, 38])


def test_nested_scan_with_until_known_answer(gpu):
    # nested Scan whose inner Scan stops early (tests/scan/test_basic.py:3852-3898 expects [3, 1, 0])
    from pytensor.scan.utils import until

    def fn(n):
        s_in_y = scan(fn=lambda z: (z + 1, until(z > 2)),
                      outputs_info=[{"taps": [-1], "initial": pt.as_tensor(0.0, dtype=np.float64)}],
                      n_steps=n - 1, return_updates=False)
        return s_in_y.sum()

    s_y = scan(fn=fn, outputs_info=[None], sequences=[pt.as_tensor([3, 2, 1], dtype=np.int64)], return_updates=False)
    f = pytensor.function([], s_y, mode="CUDA")
    np.testing.assert_array_equal(f(), np.array([3, 1, 0]))


def test_truncated_trace_buffers_and_taps(gpu):
    # save-mem rewrites shrink trace buffers to the taps actually used (circular buffers + final rotation)
    rng = np.random.default_rng(53)
    x0 = pt.dmatrix("x0")  # (3, n) initial taps
    u = pt.dmatrix("u")

    def step(u_t, x3, x1):
        return 0.3 * x1 + 0.2 * x3 + pt.sin(u_t)

    xs = scan(step, sequences=[u], outputs_info=[dict(initial=x0, taps=[-3, -1])], return_updates=False)
    uv = rng.standard_normal((40, 9))
    x0v = rng.standard_normal((3, 9))
    compare_cuda_and_cvm([u, x0], [xs[-1], xs[-2] + xs[-4], xs[::7]], [uv, x0v], rtol=1e-10, atol=1e-12)


def test_scan_with_shared_non_sequence_and_sum_of_nit_sot(gpu):
    rng = np.random.default_rng(54)
    W = pytensor.shared(rng.standard_normal((6, 6)) * 0.3, name="W")
    v = pt.dvector("v")
    seq = pt.dmatrix("seq")
    hs, ys = scan(lambda s_t, h: (pt.tanh(pt.dot(h, W) + s_t), (h ** 2).sum()), sequences=[seq],
                  outputs_info=[v, None], return_updates=False)
    compare_cuda_and_cvm([v, seq], [hs[-1], ys, ys.sum()], [rng.standard_normal(6), rng.standard_normal((11, 6))],
                         rtol=1e-9, atol=1e-10)
