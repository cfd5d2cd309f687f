"""CPU suite: how nodes_blas.gemm routes a product, seen from the C-ABI calls it makes (trace-only mode, a recording
library).  Every tensor-core product is staging (ptk_stage_operand, zero to two calls) followed by exactly one
ptk_gemm_tc_staged; the table below is what decides the staging, the kernel's arguments and the operand a product hands
to the next one:

  product                        A                                         B                   result operand
  fp64 / a dim < 256 / simt      FMA kernels                                                   none
  bf16 mode                      chained one-piece copy, else staged       resident or staged  one piece when asked
  fp32-accurate (tc6 / tc3)      chained pieces only with a resident B     resident or staged  three pieces only with a
                                 whose `aligned` matches, else staged                          resident B and a tanh
                                                                                               (or an unaligned split)
"""

import itertools

import pytest
import torch

from pytensor_b200.runtime import device as dev
from pytensor_b200.runtime import lib as _lib
from pytensor_b200.vm import nodes_blas as nb

M, N, K = 512, 384, 256

STAGED_ARGS = ("M", "N", "K", "alpha", "A", "lda", "a_rows", "B", "ldb", "b_rows", "terms", "beta", "C", "sc0", "sc1", "bias",
               "act", "C_stage", "ldc_stage", "c_rows", "out_pieces", "exact_main", "out_exp", "a_flags", "b_flags", "c_flags",
               "stream")
STAGE_ARGS = ("src", "sr", "sc", "rows", "cols", "pieces", "aligned", "dst", "ld", "piece_rows", "stream")
RECORDED = ("ptk_stage_operand", "ptk_gemm_tc_staged", "ptk_gemm_tc_ex", "ptk_gemm_tc_split", "ptk_gemm", "ptk_gemm_bias_act")


class Recorder:
    """The trace-only library, recording the GEMM-family calls in order."""

    def __init__(self, exact_default=1):
        self.calls, self.exact_default, self._trace = [], exact_default, _lib._TraceLib()

    def __getattr__(self, name):
        if name == "ptk_gemm_exact_main_default":
            return lambda: self.exact_default
        if name in RECORDED:
            return lambda *a: self.calls.append((name, a)) or 0
        return getattr(self._trace, name)

    def names(self):
        return [n for n, _ in self.calls]


@pytest.fixture
def rec(monkeypatch):
    monkeypatch.setattr(_lib, "TRACE_ONLY", True)
    r = Recorder()
    monkeypatch.setattr(_lib, "lib", lambda: r)
    # meta tensors have no addresses: hand out a distinct fake one per buffer so that the calls say which buffer they read
    addr, keep = {}, []

    def fake_ptr(t):
        if id(t) not in addr:
            keep.append(t)
            addr[id(t)] = (len(addr) + 1) << 32
        return addr[id(t)]

    monkeypatch.setattr(dev, "ptr", fake_ptr)
    return r


def _t(*shape, dtype=torch.float32):
    return torch.empty(shape, dtype=dtype, device="meta")


def _run(rec, monkeypatch, mode, precision, resident, chained=None, want=False, act=0, dtype="float32", dims=(M, N, K),
         exact_default=1):
    """One gemm() call; returns (result, [stage_operand calls as dicts], tc_staged call as a dict or None)."""
    monkeypatch.setattr(nb, "FP32_MODE", mode)
    rec.exact_default = exact_default
    m, n, k = dims
    tdt = torch.float64 if dtype == "float64" else torch.float32
    A, B, C = _t(m, k, dtype=tdt), _t(k, n, dtype=tdt), _t(m, n, dtype=tdt)
    plan = nb.tc_plan(dtype, precision, m, n, k)
    Bres = nb.stage_operand(B, plan[0], transposed=True) if resident and plan else None
    monkeypatch.setattr(nb, "staged_weight", lambda key, t, pieces: Bres if key is not None else None)
    a_staged = chained(plan) if chained is not None and plan else None
    rec.calls.clear()
    ret = nb.gemm(dtype, 1.0, A, B, 0.0, C, precision, act=act, a_staged=a_staged, want_staged=want,
                  b_key=("const", 1, 0) if resident else None)
    assert not any(name in ("ptk_gemm_tc_ex", "ptk_gemm_tc_split") for name in rec.names())
    stages = [dict(zip(STAGE_ARGS, a)) for nm, a in rec.calls if nm == "ptk_stage_operand"]
    staged = [dict(zip(STAGED_ARGS, a)) for nm, a in rec.calls if nm == "ptk_gemm_tc_staged"]
    if staged:
        assert len(staged) == 1 and rec.names()[-1] == "ptk_gemm_tc_staged"   # staging first, then one product
    ctx = {"A": A, "B": B, "C": C, "Bres": Bres, "a_staged": a_staged}
    return ret, stages, (staged[0] if staged else None), ctx


@pytest.mark.parametrize("case", ["float64", "small", "simt"])
def test_fma_products_never_touch_the_tensor_cores(rec, monkeypatch, case):
    kw = {"float64": dict(dtype="float64"), "small": dict(dims=(M, N, 255)), "simt": dict()}[case]
    mode = "simt" if case == "simt" else "tc6"
    for act in (0, 1):
        ret, stages, staged, _ = _run(rec, monkeypatch, mode, 0, resident=True, want=True, act=act, **kw)
        assert ret is None and not stages and staged is None
        assert rec.names() == ["ptk_gemm_bias_act" if act else "ptk_gemm"]


def _one_piece(plan):
    return nb.Staged(M, K, 1)


def _three_piece(aligned):
    def make(plan):
        st = nb.Staged(M, K, 3, aligned=aligned)
        st.flagged = not aligned   # as an epilogue leaves it (gemm_staged): a tanh output needs no ±inf flags
        return st
    return make


@pytest.mark.parametrize("resident,chain,want", list(itertools.product([False, True], [False, True], [False, True])))
def test_bf16_mode(rec, monkeypatch, resident, chain, want):
    ret, stages, p, ctx = _run(rec, monkeypatch, "tc6", 1, resident, chained=_one_piece if chain else None, want=want, act=1)
    # staging: B^T unless resident, then A unless the previous product's one-piece copy is chained
    expect = ([] if resident else [("B", N, K)]) + ([] if chain else [("A", M, K)])
    assert [("B" if s["src"] == dev.ptr(ctx["B"]) else "A", s["rows"], s["cols"]) for s in stages] == expect
    assert all(s["pieces"] == 1 and s["aligned"] == 0 for s in stages)
    if not resident:
        assert (stages[0]["sr"], stages[0]["sc"]) == (ctx["B"].stride(1), ctx["B"].stride(0))
    assert (p["M"], p["N"], p["K"], p["terms"], p["exact_main"], p["out_exp"]) == (M, N, K, 1, 0, nb.NO_EXP)
    assert p["a_flags"] is None and p["b_flags"] is None and p["c_flags"] is None
    assert p["C"] == dev.ptr(ctx["C"])
    assert p["A"] == (ctx["a_staged"].ptr if chain else stages[-1]["dst"])
    assert p["B"] == (ctx["Bres"].ptr if resident else stages[0]["dst"])
    if want:
        assert isinstance(ret, nb.Staged) and (ret.pieces, ret.rows, ret.cols, ret.aligned) == (1, M, N, False)
        assert (p["C_stage"], p["ldc_stage"], p["out_pieces"]) == (ret.ptr, ret.ld, 1)
    else:
        assert ret is None and p["C_stage"] is None and p["out_pieces"] == 1


@pytest.mark.parametrize("mode,exact_default", [("tc6", 1), ("tc3", 1), ("tc6", 0)])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("chain_aligned", [None, False, True])
@pytest.mark.parametrize("resident", [False, True])
def test_fp32_accurate_mode(rec, monkeypatch, mode, exact_default, act, chain_aligned, resident):
    terms = 6 if mode == "tc6" else 3
    aligned = mode == "tc6" and exact_default == 1
    chained = None if chain_aligned is None else _three_piece(chain_aligned)
    ret, stages, p, ctx = _run(rec, monkeypatch, mode, 0, resident, chained=chained, want=True, act=act,
                               exact_default=exact_default)
    # chained pieces only together with a resident B whose alignment they share
    use_chain = resident and chain_aligned is not None and chain_aligned == aligned
    expect = ([] if resident else [("B", N, K)]) + ([] if use_chain else [("A", M, K)])
    assert [("B" if s["src"] == dev.ptr(ctx["B"]) else "A", s["rows"], s["cols"]) for s in stages] == expect
    assert all(s["pieces"] == 3 and s["aligned"] == int(aligned) for s in stages)
    assert (p["terms"], p["exact_main"]) == (terms, int(aligned))
    assert p["A"] == (ctx["a_staged"].ptr if use_chain else stages[-1]["dst"])
    assert p["B"] == (ctx["Bres"].ptr if resident else stages[0]["dst"])
    # ±inf flags: those of every staged operand, those of a chained one when its epilogue raised them
    if use_chain:
        assert p["a_flags"] == (ctx["a_staged"].flags_ptr if ctx["a_staged"].flagged else None)
    else:
        assert p["a_flags"] is not None
    if resident:
        assert p["b_flags"] == ctx["Bres"].flags_ptr
    else:
        assert p["b_flags"] is not None
    # the three-piece result only for a resident B, and with error-free leading pieces only after a tanh
    emits = resident and (act == 1 or not aligned)
    if emits:
        assert isinstance(ret, nb.Staged) and (ret.pieces, ret.rows, ret.cols, ret.aligned) == (3, M, N, aligned)
        assert (p["C_stage"], p["out_pieces"], p["c_rows"]) == (ret.ptr, 3, ret.piece_rows)
        assert p["out_exp"] == (6 if aligned else nb.NO_EXP)
        assert (p["c_flags"] is None) == aligned
    else:
        assert ret is None
        assert (p["C_stage"], p["out_pieces"], p["out_exp"], p["c_flags"]) == (None, 1, nb.NO_EXP, None)
