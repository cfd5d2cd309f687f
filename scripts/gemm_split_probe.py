"""fp32-accurate tensor-core GEMM (ptk_gemm_tc_split) through the C-ABI: error against an fp64 product and time per call.
The accumulation chunk (EpiParams::kchunk) is read once per process from PTK_GEMM_KCHUNK: run once per setting.
usage: PTK_GEMM_KCHUNK=8 python scripts/gemm_split_probe.py [terms]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pytensor_b200.runtime import lib as _lib

L = _lib.init(0)
terms = int(sys.argv[1]) if len(sys.argv) > 1 else 6
torch.manual_seed(0)
for M, N, K in [(4096, 4096, 4096), (2048, 2048, 8192), (512, 768, 320), (2500, 2000, 520), (300, 4096, 4096), (1024, 1024, 1024)]:
    A = torch.randn(M, K, device="cuda")
    B = torch.randn(K, N, device="cuda")
    C = torch.empty(M, N, device="cuda")
    wsb = L.ptk_gemm_split_workspace_bytes(M, N, K)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def run():
        _lib.check(L.ptk_gemm_tc_split(M, N, K, 1.0, A.data_ptr(), A.stride(0), A.stride(1), B.data_ptr(), B.stride(0),
                                       B.stride(1), 0.0, C.data_ptr(), C.stride(0), C.stride(1), None, 0, terms, ws.data_ptr(),
                                       wsb, s), "split")

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 10
    e0.record()
    for _ in range(n):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    ref = A.double() @ B.double()
    d = (C.double() - ref)
    err = (d.abs().max() / ref.abs().max()).item()
    bias = (d.mean() / ref.abs().mean()).item()
    shrink = ((d * ref).sum() / (ref * ref).sum()).item()   # least-squares slope of the error against the exact result
    sg = torch.matmul(A, B)  # cuBLAS sgemm for scale: what a RN fp32 GEMM gets
    torch.backends.cuda.matmul.allow_tf32 = False
    err_sg = ((sg.double() - ref).abs().max() / ref.abs().max()).item()
    print(f"kchunk={os.environ.get('PTK_GEMM_KCHUNK', 'default')} terms={terms} M={M} N={N} K={K}: {ms*1e3:8.1f} us "
          f"{2*M*N*K/ms/1e9:6.0f} TF/s(fp32-equiv)  max err/scale {err:.2e} (cuBLAS fp32: {err_sg:.2e})  mean signed err {bias:+.1e}  shrink {shrink:+.2e}  exact={os.environ.get('PTK_GEMM_EXACT', '1')}",
          flush=True)
