"""Device throughput of polygamma, gammaincinv, gammainccinv and betaincinv through pytensor.function(mode="CUDA") with
inputs and outputs on the device, timed with CUDA events after warm-up, beside the C linker's host rate for the same
graph; plus gammaincinv fused into a row sum (the map+row-reduce kernel).  Records the card name and power limit, which
are part of every number.  `--registers` needs no GPU: it prints ptxas's registers, spill-store / spill-load bytes
and stack frame for every kernel these graphs generate (each NVRTC program compiled again with `--ptxas-options=-v`).
usage: python scripts/special_probe.py [--n 16777216] [--reps 5] [--registers]"""
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


def graphs(pt, dtype):
    a, b, p, x = (pt.vector(nm, dtype=dtype) for nm in "abpx")
    k = pt.vector("k", dtype="int64")
    m, u = pt.vector("m", dtype=dtype), pt.matrix("u", dtype=dtype)
    return {
        "polygamma": ([k, x], pt.polygamma(k, x)),
        "gammaincinv": ([a, p], pt.gammaincinv(a, p)),
        "gammainccinv": ([a, p], pt.gammainccinv(a, p)),
        "betaincinv": ([a, b, p], pt.betaincinv(a, b, p)),
        "gammaincinv_rowsum": ([m, u], pt.gammaincinv(m[None, :], u).sum(axis=1)),
    }


def inputs(name, n, dtype, rng):
    a = np.exp(rng.uniform(np.log(0.05), np.log(50), n)).astype(dtype)
    p = rng.uniform(1e-6, 1 - 1e-6, n).astype(dtype)
    if name == "polygamma":
        return [rng.integers(0, 13, n).astype("int64"), rng.uniform(0.1, 40, n).astype(dtype)]
    if name == "betaincinv":
        return [a, a[::-1].copy(), p]
    if name == "gammaincinv_rowsum":
        cols = 4096
        return [a[:cols], p.reshape(-1, cols)]
    return [a, p]


def power_limit():
    try:   # a read-only query
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _ptxas_report(src, opts):
    """NVRTC log of `src` compiled again with the same options plus ptxas -v: registers and spill bytes per kernel."""
    import ctypes

    from pytensor_b200.runtime import lib as _lib

    L = _lib.load_library()
    opts = tuple(opts) + ("--ptxas-options=-v",)
    cubin, size, log = ctypes.c_void_p(), ctypes.c_size_t(), ctypes.c_void_p()
    c_opts = (ctypes.c_char_p * len(opts))(*[o.encode() for o in opts])
    st = L.ptk_jit_compile(src.encode(), c_opts, len(opts), ctypes.byref(cubin), ctypes.byref(size), ctypes.byref(log))
    txt = ctypes.string_at(log.value).decode("utf-8", "replace") if log.value else ""
    for ptr in (log, cubin):
        if ptr.value:
            L.ptk_free(ptr)
    if st != 0:
        raise RuntimeError(txt)
    return txt


def registers():
    """Compile every graph as mode="CUDA" would, without a device, and print ptxas's report for each new kernel."""
    os.environ["PTK_KCACHE"] = tempfile.mkdtemp(prefix="ptk_special_probe_")   # (a cold cache: every kernel compiles)
    from oracle import cvm

    pytensor = cvm.configure()
    import pytensor.tensor as pt

    import pytensor_b200  # noqa: F401
    from pytensor_b200.precompile import trace_function
    from pytensor_b200.runtime import jit

    compiled = []
    original = jit.compile_cubin

    def recording(src, opts=()):
        compiled.append((src, tuple(opts)))
        return original(src, opts)

    jit.compile_cubin = recording
    rng = np.random.default_rng(0)
    for dtype in ("float32", "float64"):
        for name, (ins, out) in graphs(pt, dtype).items():
            del compiled[:]
            f = pytensor.function(ins, out, mode="CUDA")
            trace_function(f, inputs(name, 1 << 16, dtype, rng))
            for src, opts in compiled:
                txt = _ptxas_report(src, opts)
                for fn, body in re.findall(r"Compiling entry function '(\S+)'.*?\n(.*?)(?=Compiling entry|\Z)", txt, re.S):
                    regs = re.search(r"Used (\d+) registers", body)
                    spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", body)
                    stack = re.search(r"(\d+) bytes stack frame", body)
                    print(f"{dtype:8s} {name:20s} {fn[:40]:40s} regs {regs.group(1) if regs else '?':>3s}  "
                          f"spill stores {spill.group(1) if spill else '?':>4s} B  loads {spill.group(2) if spill else '?':>4s} B  "
                          f"stack {stack.group(1) if stack else '?'} B")


def throughput(n, reps):
    import torch

    from oracle import cvm

    pytensor = cvm.configure()
    import pytensor.tensor as pt

    import pytensor_b200  # noqa: F401
    from pytensor_b200.link.cuda import cuda_mode

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: throughput is measured on the GPU only")
    print("card:", power_limit())
    rng = np.random.default_rng(0)
    for dtype in ("float32", "float64"):
        for name, (ins, out) in graphs(pt, dtype).items():
            vals = inputs(name, n, dtype, rng)
            f = pytensor.function(ins, out, mode=cuda_mode(device_outputs=True), trust_input=True)
            dv = [torch.as_tensor(v, device="cuda") for v in vals]
            for _ in range(2):
                f(*dv)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                f(*dv)
            e1.record()
            torch.cuda.synchronize()
            dev_ms = e0.elapsed_time(e1) / reps
            nh = min(n, 1 << 18)     # host rate on a slice: the C linker evaluates these ops through SciPy
            hv = [v[:nh] if v.ndim == 1 or name != "gammaincinv_rowsum" else v[: nh // v.shape[1]] for v in vals]
            if name == "gammaincinv_rowsum":
                hv[0] = vals[0]
            fh = pytensor.function(ins, out, mode="CVM")
            fh(*hv)
            t0 = time.perf_counter()
            fh(*hv)
            host_s = time.perf_counter() - t0
            nel = int(np.prod(vals[-1].shape))
            nhel = int(np.prod(hv[-1].shape))
            print(f"{dtype:8s} {name:20s} n={nel:>9d}  device {dev_ms:8.3f} ms  {nel / dev_ms / 1e6:8.2f} Gelem/s   "
                  f"C linker {nhel / host_s / 1e6:8.3f} Melem/s")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 24)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--registers", action="store_true")
    args = ap.parse_args()
    if args.registers:
        registers()
    else:
        throughput(args.n, args.reps)
