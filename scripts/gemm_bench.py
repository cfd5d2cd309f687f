"""Micro-benchmark of the bf16 tensor-core (wgmma) GEMM through the C-ABI (ptk_gemm_tc_ex) with A already in bf16 (the chained-layer
case): the conversion of B and the GEMM kernel are timed together.
usage: python scripts/gemm_bench.py [M N K]..."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pytensor_b200.runtime import lib as _lib

L = _lib.init(0)
shapes = [(4096, 4096, 4096), (8192, 8192, 4096), (2560, 2048, 4096), (3072, 3328, 2048)]
for M, N, K in shapes:
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(K, N, device="cuda")
    C = torch.empty(M, N, device="cuda")
    Abf = A.bfloat16().contiguous()
    ws_bytes = L.ptk_gemm_workspace_bytes(M, N, K, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def run():
        _lib.check(L.ptk_gemm_tc_ex(M, N, K, 1.0, A.data_ptr(), A.stride(0), A.stride(1), Abf.data_ptr(), Abf.stride(0),
                                    B.data_ptr(), B.stride(0), B.stride(1), 0.0, C.data_ptr(), C.stride(0), C.stride(1),
                                    None, 0, None, 0, ws.data_ptr(), ws_bytes, s), "gemm")

    for _ in range(5):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 30
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    ref = Abf.float() @ B.bfloat16().float()
    err = ((C - ref).abs().max() / ref.abs().max()).item()
    print(f"M={M} N={N} K={K} {ms*1e3:.1f} us (incl. B convert) "
          f"{2*M*N*K/ms/1e9:.0f} TF/s  rel.err {err:.2e}", flush=True)
