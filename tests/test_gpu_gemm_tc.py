"""The bf16 tensor-core (wgmma) GEMM path (K4/K5) against the reference C linker's fp32 sgemm.

Tolerance: operands are rounded to bf16 (8-bit mantissa, rel 2^-9 per operand), products accumulate in fp32, so a
K-term dot product of O(1) values carries an absolute error ~ sqrt(K) * 2^-9 * |a||b|.  This is the reference's own
half-precision notion of "close" (float16: atol=rtol=1e-3 relative to the output scale, pytensor/tensor/math.py:92-139)
scaled by the output magnitude; the 1e-5 bar applies to the native fp32 path (test_gpu_blas.py)."""

import numpy as np
import pytest

from helpers import pytensor

import pytensor.tensor as pt

pytestmark = pytest.mark.gpu


def _check(got, ref, K):
    scale = np.abs(ref).max() + 1e-30
    err = np.abs(got - ref).max() / scale
    assert err < 4e-3, f"bf16 tensor-core GEMM deviates {err:.2e} of the output scale (K={K})"


# the last shapes have more 128x128 output tiles than the H100 has SMs (132), ragged M / N / K edges included, and the
# last two have >= 8 k-blocks
@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (512, 768, 320), (1000, 520, 264), (384, 256, 1024),
                                   (2560, 2048, 256), (2500, 2000, 264), (3072, 3328, 320),
                                   (2500, 2000, 520), (2560, 2048, 1032)])
def test_dot22_bf16(gpu, M, N, K):
    rng = np.random.default_rng(41)
    x, y = pt.fmatrix("x"), pt.fmatrix("y")
    f = pytensor.function([x, y], pt.dot(x, y), mode="CUDA_BF16")
    xv = rng.standard_normal((M, K)).astype("float32")
    yv = rng.standard_normal((K, N)).astype("float32")
    got = f(xv, yv)
    ref = xv.astype(np.float64) @ yv.astype(np.float64)
    _check(got, ref, K)
    # bit-level structure: the result must equal an fp32-accumulated product of the bf16-rounded operands closely
    import torch

    xb = torch.from_numpy(xv).bfloat16().double().numpy()
    yb = torch.from_numpy(yv).bfloat16().double().numpy()
    np.testing.assert_allclose(got, xb @ yb, rtol=2e-5, atol=2e-4 * np.sqrt(K))


def test_gemm_bf16_alpha_beta_and_transposes(gpu):
    rng = np.random.default_rng(42)
    z, x, y = pt.fmatrix("z"), pt.fmatrix("x"), pt.fmatrix("y")
    f = pytensor.function([z, x, y], 0.5 * z + 2.0 * pt.dot(x.T, y), mode="CUDA_BF16")
    xv = rng.standard_normal((512, 300)).astype("float32")
    yv = rng.standard_normal((512, 260)).astype("float32")
    zv = rng.standard_normal((300, 260)).astype("float32")
    got = f(zv, xv, yv)
    ref = 0.5 * zv + 2.0 * (xv.T.astype(np.float64) @ yv.astype(np.float64))
    _check(got, ref, 512)


def test_mlp_chain_bf16_vs_cvm(gpu):
    # BASELINE.json configs[2] at reduced size: 3 x tanh(h @ W + b); CUDA_BF16 vs the C linker's fp32 result
    from pytensor_b200 import workloads as W

    pytensor.config.floatX = "float32"
    ins, outs, make_args, _ = W.cfg3_mlp(512)
    f = pytensor.function(ins, outs, mode="CUDA_BF16")
    f_ref = pytensor.function(ins, outs, mode="CVM")
    a = make_args()
    got, ref = f(*a)[0], f_ref(*a)[0]
    assert np.abs(got - ref).max() < 2e-3 * max(1.0, np.abs(ref).max())
    # and the native-precision linker meets the 1e-5 class bar on the same graph
    f32 = pytensor.function(ins, outs, mode="CUDA")
    np.testing.assert_allclose(f32(*a)[0], ref, rtol=1e-5, atol=1e-5)   # outputs of tanh: scale 1


# ---- fp32-accurate tensor-core GEMM (bf16x3 operand split, ptk_gemm_tc_split): the DEFAULT mode="CUDA" path for large fp32 ----
def _scale_err(got, ref):
    return float(np.abs(np.asarray(got, dtype=np.float64) - ref).max() / (np.abs(ref).max() + 1e-30))


@pytest.mark.parametrize("M,N,K", [(256, 256, 256), (512, 768, 320), (1000, 520, 264), (2500, 2000, 520), (300, 4096, 4096)])
def test_dot22_fp32_on_tensor_cores_is_more_accurate_than_1e5(gpu, M, N, K):
    """6 piece products per k-block: the only dropped products are O(2^-24).  What remains is the tensor core's own fp32
    accumulation (it truncates: ~3x the rounding noise of an FMA sgemm over a short chain, and a bias growing with the
    chain length — hence the accumulation chunks of EpiParams::kchunk, without which K = 4096 sits at 2.4e-5): the result
    must stay within 5e-6 of the output scale of an fp64 product (cuBLAS sgemm: 1-3e-6) and within 1e-5 of the C linker."""
    rng = np.random.default_rng(43)
    x, y = pt.fmatrix("x"), pt.fmatrix("y")
    f = pytensor.function([x, y], pt.dot(x, y), mode="CUDA")
    xv = rng.standard_normal((M, K)).astype("float32")
    yv = rng.standard_normal((K, N)).astype("float32")
    got = f(xv, yv)
    ref = xv.astype(np.float64) @ yv.astype(np.float64)
    assert _scale_err(got, ref) < 5e-6, _scale_err(got, ref)
    f_ref = pytensor.function([x, y], pt.dot(x, y), mode="CVM")
    exp = f_ref(xv, yv)
    np.testing.assert_allclose(got, exp, rtol=1e-5, atol=1e-5 * np.abs(exp).max())


def test_gemm_fp32_split_alpha_beta_strides_bias_tanh(gpu):
    rng = np.random.default_rng(44)
    z, x, y, b = pt.fmatrix("z"), pt.fmatrix("x"), pt.fmatrix("y"), pt.fvector("b")
    outs = [0.5 * z + 2.0 * pt.dot(x.T, y), pt.tanh(pt.dot(x.T, y) + b), pt.dot(x.T[:, ::2], y[::2])]
    f = pytensor.function([z, x, y, b], outs, mode="CUDA")
    f_ref = pytensor.function([z, x, y, b], outs, mode="CVM")
    xv = (rng.standard_normal((640, 300)) / 16).astype("float32")
    yv = (rng.standard_normal((640, 260)) / 16).astype("float32")
    zv = rng.standard_normal((300, 260)).astype("float32")
    bv = rng.standard_normal(260).astype("float32")
    for g, e in zip(f(zv, xv, yv, bv), f_ref(zv, xv, yv, bv)):
        np.testing.assert_allclose(g, e, rtol=1e-5, atol=1e-5 * max(1.0, float(np.abs(e).max())))


def test_three_term_split_meets_the_1e5_bar(gpu, monkeypatch):
    from pytensor_b200.vm import nodes_blas

    monkeypatch.setattr(nodes_blas, "FP32_MODE", "tc3")
    rng = np.random.default_rng(45)
    x, y = pt.fmatrix("x"), pt.fmatrix("y")
    f = pytensor.function([x, y], pt.dot(x, y), mode="CUDA")
    xv = rng.standard_normal((512, 4096)).astype("float32")
    yv = rng.standard_normal((4096, 512)).astype("float32")
    ref = xv.astype(np.float64) @ yv.astype(np.float64)
    err = _scale_err(f(xv, yv), ref)
    assert 1e-8 < err < 1e-5, err
    monkeypatch.setattr(nodes_blas, "FP32_MODE", "simt")
    f2 = pytensor.function([x, y], pt.dot(x, y), mode="CUDA")
    assert _scale_err(f2(xv, yv), ref) < 1e-5


# ---- resident staged weights (nodes_blas.staged_weight, Executor._track_weights) ------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_resident_weights_follow_the_tensor_version(gpu, precision):
    """A weight matrix handed over as the same device tensor object at the same torch version is staged once and the staged
    copy stays resident (also inside the captured graph); an in-place change through torch, or another tensor object, must be
    seen by the very next call.  Constants are resident from the first call."""
    import torch

    from pytensor_b200.link.cuda import cuda_mode
    from pytensor_b200.runtime import device as dev
    from pytensor_b200.vm import nodes_blas

    pytensor.config.floatX = "float32"
    rng = np.random.default_rng(46)
    x, W1, W2, b = pt.fmatrix("x"), pt.fmatrix("W1"), pt.fmatrix("W2"), pt.fvector("b")
    Wc = (rng.standard_normal((384, 256)) / 20).astype("float32")
    out = pt.dot(pt.tanh(pt.dot(pt.tanh(pt.dot(x, W1) + b), W2)), pt.constant(Wc))
    f = pytensor.function([x, W1, W2, b], out, mode=cuda_mode(device_outputs=True, gemm_precision=precision), trust_input=True)
    f_ref = pytensor.function([x, W1, W2, b], out, mode="CVM")
    xv = rng.standard_normal((300, 320)).astype("float32")
    W1v = (rng.standard_normal((320, 512)) / 18).astype("float32")
    W2v = (rng.standard_normal((512, 384)) / 22).astype("float32")
    bv = (rng.standard_normal(512) * 0.1).astype("float32")
    tol = dict(rtol=1e-5, atol=1e-5) if precision == "fp32" else dict(rtol=0, atol=2e-2)
    d = [dev.to_device(v) for v in (xv, W1v, W2v, bv)]
    h0 = nodes_blas._stage_cache_stats["hits"]
    for call in range(7):   # eager+measure, capture, (keys appear) measure, capture, replays
        np.testing.assert_allclose(dev.to_host(f(*d)), f_ref(xv, W1v, W2v, bv), **tol)
    assert nodes_blas._stage_cache_stats["hits"] > h0, "weights were never served from the resident cache"
    assert f.vm.executor.last_from_graph
    # in-place change through torch: version moves, the next call must see the new values
    d[1].mul_(0.5)
    torch.cuda.synchronize()
    for call in range(4):
        np.testing.assert_allclose(dev.to_host(f(*d)), f_ref(xv, W1v * np.float32(0.5), W2v, bv), **tol)
    # another tensor object of the same shape
    W2b = (W2v * np.float32(-1.0)).astype("float32")
    d[2] = dev.to_device(W2b)
    for call in range(4):
        np.testing.assert_allclose(dev.to_host(f(*d)), f_ref(xv, W1v * np.float32(0.5), W2b, bv), **tol)
