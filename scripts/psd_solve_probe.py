"""Device time of ptk_potrs (the Cholesky solve behind CholeskySolve and positive-definite Solve), timed with CUDA events
after warm-up, and of a Gaussian-process marginal log-likelihood plus its gradient through pytensor.function(mode="CUDA")
beside the C linker.  Records the card name and power limit, which are part of every number.

  batched small systems (potrs_small_kernel, one warp per (system, column)): achieved bytes/s against 3.35 TB/s, counting
  the least traffic the solve needs — each factor once (n*n elements, the whole stored matrix), b read and x written;
  large systems (the blocked triangular solves, diagonal-block kernel + ptk_gemm updates): time and GFLOP/s at
  2 n^2 nrhs flop.

`--registers` needs no GPU: it compiles csrc/ptk_linalg.cu for sm_90a with ptxas -v and prints potrs_small_kernel's
registers and spill bytes.
usage: python scripts/psd_solve_probe.py [--reps 20] [--registers]"""
import argparse
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def registers():
    src = os.path.join(REPO, "pytensor_b200", "csrc", "ptk_linalg.cu")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run(["/usr/local/cuda/bin/nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                            "-I" + os.path.join(REPO, "include"), "-I" + os.path.dirname(src), "-Xptxas", "-v", "-c", src,
                            "-o", os.path.join(d, "x.o")], capture_output=True, text=True, check=True)
    lines = r.stderr.splitlines()
    for i, ln in enumerate(lines):
        m = re.search(r"Compiling entry function '(\S*potrs_small_kernelI([fd])\S*)'", ln)
        if m:
            spill = next(x for x in lines[i + 1:i + 4] if "spill" in x).strip()
            regs = next(x for x in lines[i + 1:i + 4] if "registers" in x).strip()
            print(f"potrs_small_kernel<{'float' if m.group(2) == 'f' else 'double'}>: {regs} | {spill}")


def power_limit():
    try:   # a read-only query
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def time_potrs(systems, n, nrhs, dtype, reps):
    import torch

    from pytensor_b200.runtime import device as dev
    from pytensor_b200.runtime import lib as _lib

    dev.device()
    g = torch.Generator(device="cuda").manual_seed(n + nrhs)
    tdt = getattr(torch, dtype)
    M = torch.randn((systems, n, n), generator=g, device="cuda", dtype=torch.float64)
    C = torch.linalg.cholesky(M @ M.transpose(1, 2) / n + torch.eye(n, device="cuda", dtype=torch.float64)).to(tdt).contiguous()
    del M
    B0 = torch.randn((systems, n, nrhs), generator=g, device="cuda", dtype=tdt)
    B = B0.clone()
    L = _lib.lib()
    shape, strides = dev.i64_array([systems]), dev.i64_array([n * n])

    def run():
        _lib.check(L.ptk_potrs(_lib.DTYPE_CODE[dtype], C.data_ptr(), B.data_ptr(), n, nrhs, 1, 1, shape, strides,
                               dev.stream_ptr()), "ptk_potrs")

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    # correctness of the timed kernel: one solve from b against A x
    B.copy_(B0)
    run()
    torch.cuda.synchronize()
    A = C.double() @ C.double().transpose(1, 2)
    res = (A @ B.double() - B0.double()).abs().max().item() / max(B0.abs().max().item(), 1e-300)
    return ms, res


def gp(n, reps):
    from oracle import cvm

    pytensor = cvm.configure()
    import pytensor_b200  # noqa: F401

    sys.path.insert(0, os.path.join(REPO, "tests"))
    import psd_cases

    ins, outs = psd_cases.gp_graph()
    outs = outs[:4]   # logp and its gradient
    vals = psd_cases.gp_inputs(n, 4, 0)
    f = pytensor.function(ins, outs, mode="CUDA", on_unused_input="ignore")
    f_ref = pytensor.function(ins, outs, mode="CVM", on_unused_input="ignore")
    got = f(*vals)
    for _ in range(2):
        f(*vals)
    t0 = time.perf_counter()
    for _ in range(reps):
        f(*vals)      # host outputs: every call ends in a device synchronise
    t_dev = (time.perf_counter() - t0) / reps
    exp = f_ref(*vals)
    nref = 2 if n <= 1000 else 1
    t0 = time.perf_counter()
    for _ in range(nref):
        f_ref(*vals)
    t_ref = (time.perf_counter() - t0) / nref
    err = max(abs(float(g) - float(e)) / max(abs(float(e)), 1e-300) for g, e in zip(got, exp))
    return t_dev, t_ref, err


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--registers", action="store_true")
    a = ap.parse_args()
    if a.registers:
        registers()
        return
    import torch

    print(f"card: {torch.cuda.get_device_name(0)} | name, power limit: {power_limit()}")
    print("batched small systems (potrs_small_kernel)")
    for systems, n, nrhs in ((1 << 16, 16, 1), (1 << 12, 128, 1), (1 << 12, 128, 32)):
        for dtype in ("float32", "float64"):
            ms, res = time_potrs(systems, n, nrhs, dtype, a.reps)
            isz = 4 if dtype == "float32" else 8
            nbytes = systems * (n * n + 2 * n * nrhs) * isz
            bw = nbytes / (ms * 1e-3)
            print(f"  {systems:6d} x n={n:4d} nrhs={nrhs:3d} {dtype}: {ms * 1e3:9.1f} us  {bw / 1e9:7.1f} GB/s "
                  f"({100 * bw / HBM_BYTES_PER_S:5.1f}% of 3.35 TB/s)  rel. residual {res:.1e}")
    print("large systems (blocked triangular solves)")
    for n in (4096, 8192):
        for nrhs in (1, 64):
            for dtype in ("float32", "float64"):
                ms, res = time_potrs(1, n, nrhs, dtype, max(3, a.reps // 4))
                print(f"  n={n:5d} nrhs={nrhs:3d} {dtype}: {ms:8.3f} ms  {2.0 * n * n * nrhs / (ms * 1e-3) / 1e9:7.1f} GFLOP/s  "
                      f"rel. residual {res:.1e}")
    print("GP marginal logp + gradient w.r.t. (ell, eta, sigma), float64, host inputs and outputs")
    for n in (1000, 4000):
        t_dev, t_ref, err = gp(n, 5)
        print(f"  n={n:5d}: CUDA {t_dev * 1e3:8.2f} ms/call   C linker {t_ref * 1e3:9.1f} ms/call   max rel. diff {err:.1e}")


if __name__ == "__main__":
    main()
