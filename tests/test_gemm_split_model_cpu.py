"""NumPy model of the fp32-accurate tensor-core GEMM (DESIGN.md §4 K4x), kept beside the kernel as the statement of WHY it
works.  The tensor core accumulates bf16 x bf16 products into an fp32 accumulator that may TRUNCATE (a systematic shrink
of about 1e-7 per accumulation step).  The model reproduces such an accumulator and shows, on the same operands:

  * the plain three-piece split (x1 = bf16(x), ...) inherits the shrink: the result is biased towards zero by ~K * 2^-24;
  * with error-free leading pieces (x1 = rint(x * 2^s) * 2^-s, |rint| <= 2^7, s per row of A / column of B) every A1*B1
    product is an integer on one common unit, their running sum is exact in fp32, and the truncation only touches the five
    correction products, which carry 2^-7 of the total: the bias disappears.

Only the accumulation order inside one MMA (16 products at a time) is a guess; the conclusions do not depend on it."""

import numpy as np
import pytest


def _bf16(x):
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    return (b.astype(np.uint32) << 16).view(np.float32)


def _trunc_add(acc, inc):
    """fp32 accumulator += exact increment, rounded TOWARDS ZERO (acc, inc: float64 arrays holding fp32-representable acc)."""
    s = acc + inc                                     # exact enough in float64 for 24-bit operands of similar scale
    f = s.astype(np.float32)                          # round to nearest ...
    over = np.abs(f.astype(np.float64)) > np.abs(s)   # ... then step back where that rounded away from zero
    f = np.where(over, np.nextafter(f, np.float32(0)), f)
    return f.astype(np.float64)


def _accumulate(terms, K, mma_k=16):
    """terms: list of (A_piece [M,K], B_piece [K,N]) float32; one truncating accumulator; per k-slab of 16 the products of a
    term are summed exactly (the tensor core's internal adder tree is wider than fp32) and then added with truncation."""
    M, N = terms[0][0].shape[0], terms[0][1].shape[1]
    acc = np.zeros((M, N))
    for k0 in range(0, K, mma_k):
        for A, B in terms:
            acc = _trunc_add(acc, A[:, k0:k0 + mma_k].astype(np.float64) @ B[k0:k0 + mma_k].astype(np.float64))
    return acc


def _plain_split(x):
    x1 = _bf16(x)
    x2 = _bf16(x - x1)
    x3 = _bf16(x - x1 - x2)
    return x1, x2, x3


def _aligned_split(x, axis, lead_bits=7):
    """Leading piece on a power-of-two grid chosen per row (axis=1: rows of A) or per column (axis=0: columns of B)."""
    m = np.abs(x).max(axis=axis, keepdims=True)
    e = np.floor(np.log2(np.where(m > 0, m, 1.0)))
    s = lead_bits - 1 - e
    x1 = (np.rint(x.astype(np.float64) * np.exp2(s)) * np.exp2(-s)).astype(np.float32)
    r = (x.astype(np.float64) - x1).astype(np.float32)
    x2 = _bf16(r)
    x3 = _bf16(r - x2)
    assert np.all(_bf16(x1) == x1)          # <= 8 significant bits: representable in bf16
    return x1, x2, x3


@pytest.mark.parametrize("K", [512, 2048])
def test_error_free_leading_pieces_remove_the_truncation_bias(K):
    rng = np.random.default_rng(K)
    M, N = 24, 24
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = (rng.standard_normal((K, N)) / np.sqrt(K)).astype(np.float32)
    B += np.float32(0.5 / np.sqrt(K))       # a non-zero mean makes a shrink visible as a signed bias
    A = np.abs(A)
    exact = A.astype(np.float64) @ B.astype(np.float64)
    scale = np.abs(exact).max()

    a, b = _plain_split(A), _plain_split(B)
    six = [(a[2], b[0]), (a[1], b[1]), (a[0], b[2]), (a[1], b[0]), (a[0], b[1]), (a[0], b[0])]
    plain = _accumulate(six, K)
    shrink_plain = float(np.sum(plain * exact) / np.sum(exact * exact) - 1.0)

    a, b = _aligned_split(A, 1), _aligned_split(B, 0)
    main = _accumulate([(a[0], b[0])], K)
    corr = _accumulate([(a[2], b[0]), (a[1], b[1]), (a[0], b[2]), (a[1], b[0]), (a[0], b[1])], K)
    ours = (main + corr).astype(np.float32).astype(np.float64)          # the epilogue adds the two accumulators with RN
    shrink_ours = float(np.sum(ours * exact) / np.sum(exact * exact) - 1.0)

    # 1. the main term is EXACT: integer products on one unit, partial sums below 2^24 units
    np.testing.assert_array_equal(main, a[0].astype(np.float64) @ b[0].astype(np.float64))
    # 2. plain split: biased towards zero, growing with the length of the accumulation chain
    assert shrink_plain < -0.3e-7 * K / 16      # (K=2048: -1.7e-5 in this model; measured on the device at K=4096: -2.5e-5)
    # 3. exact main term: bias two orders of magnitude smaller, max error at the fp32 rounding level
    assert abs(shrink_ours) < abs(shrink_plain) / 30
    assert np.abs(ours - exact).max() / scale < 1e-6
    assert np.abs(plain - exact).max() / scale > np.abs(ours - exact).max() / scale
