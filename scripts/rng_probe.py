"""Throughput of the discrete-count and row samplers (ptk_random_count / ptk_random_rows) through the C-ABI, timed with CUDA
events after warm-up, beside the reference's host sampler (NumPy's Generator / SciPy) for the same draws.
Prints one line per case and records the card name and its power limit, which are part of every number.
usage: python scripts/rng_probe.py [--reps R]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pytensor_b200.runtime import lib as _lib

L = _lib.init(0)
I64, F64 = _lib.DTYPE_CODE["int64"], _lib.DTYPE_CODE["float64"]


def power_limit():
    try:   # a read-only query
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device="cuda")


def time_ms(run, reps):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def host_ms(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    print(f"# {torch.cuda.get_device_name(0)}, power limit {power_limit()}", flush=True)
    s = torch.cuda.current_stream().cuda_stream
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    g = np.random.default_rng(0)
    n = 1 << 24
    out = torch.empty(n, dtype=torch.int64, device="cuda")
    count_cases = [("poisson lam=3", 0, [3.0], lambda: g.poisson(3.0, n)),
                   ("poisson lam=1e4", 0, [1e4], lambda: g.poisson(1e4, n)),
                   ("binomial n=1000 p=0.5", 1, [1000.0, 0.5], lambda: g.binomial(1000, 0.5, n)),
                   ("geometric p=0.01", 3, [0.01], lambda: g.geometric(0.01, n))]
    for name, code, params, ref in count_cases:
        ps = [dev([p]) for p in params] + [None] * (3 - len(params))
        ptr = [p.data_ptr() if p is not None else None for p in ps]

        def run():
            _lib.check(L.ptk_random_count(code, I64, out.data_ptr(), n, 1234, 5678, ptr[0], 0, ptr[1], 0, ptr[2], 0,
                                          err.data_ptr(), s), "count")

        ms = time_ms(run, args.reps)
        print(f"{name:<34} {n:>9} draws  device {ms:9.3f} ms {n / ms / 1e3:10.1f} M draws/s   host reference "
              f"{n / host_ms(ref) / 1e3:8.1f} M draws/s", flush=True)
    row_cases = [("categorical 2^20 rows x k=3", 0, 1 << 20, 3, None),
                 ("categorical 64 rows x k=100000", 0, 64, 100_000, None),
                 ("multinomial 2^18 rows n=100 k=10", 1, 1 << 18, 10, 100.0),
                 ("dirichlet 2^18 rows x k=10", 2, 1 << 18, 10, None)]
    for name, kind, rows, k, nval in row_cases:
        P = g.dirichlet(np.ones(k), size=rows) if kind != 2 else np.full((rows, k), 1.5)
        Pd = dev(P)
        nv = dev(np.full(rows, nval if nval is not None else 0.0))
        o = torch.empty((rows,) if kind == 0 else (rows, k), dtype=torch.float64 if kind == 2 else torch.int64, device="cuda")
        dt = F64 if kind == 2 else I64

        def run():
            _lib.check(L.ptk_random_rows(kind, dt, o.data_ptr(), rows, k, 1234, 5678, Pd.data_ptr(), k, nv.data_ptr(), 1,
                                         err.data_ptr(), s), "rows")

        ms = time_ms(run, args.reps)
        if kind == 0:
            def ref():
                u = g.random(rows)
                cs = np.cumsum(P, axis=1)
                return [np.searchsorted(cs[i], u[i]) for i in range(rows)]
        elif kind == 1:
            def ref():
                return g.multinomial(int(nval), P)
        else:
            def ref():
                return g.dirichlet(np.full(k, 1.5), size=rows)
        print(f"{name:<34} {rows:>9} rows   device {ms:9.3f} ms {rows / ms / 1e3:10.3f} M rows/s   host reference "
              f"{rows / host_ms(ref) / 1e3:8.3f} M rows/s", flush=True)
    assert int(err.item()) == 0


if __name__ == "__main__":
    main()
