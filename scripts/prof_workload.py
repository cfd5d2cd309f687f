#!/usr/bin/env python
"""Run a BASELINE workload a few times eagerly (a target for a profiler).  usage: prof_workload.py cfg3|cfg4|cfg5|metric [steps]"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import cvm  # noqa: E402

pytensor = cvm.configure("float32")
import torch  # noqa: E402

import pytensor_b200  # noqa: E402,F401
from pytensor_b200 import workloads as W  # noqa: E402
from pytensor_b200.link.cuda import cuda_mode  # noqa: E402
from pytensor_b200.runtime import device as dev  # noqa: E402

which = sys.argv[1]
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 2
kw = {}
if which == "cfg3":
    ins, outs, mk, meta = W.cfg3_mlp(4096)
    kw = dict(gemm_precision="bf16")
elif which == "cfg4":
    ins, outs, mk, meta = W.cfg4_scan(8192, 512, 1000)
elif which == "cfg4full":
    ins, outs, mk, meta = W.cfg4_scan(8192, 512, 1000, full_trace=True)
elif which == "cfg4mm":
    ins, outs, mk, meta = W.cfg4_scan(8192, 512, int(os.environ.get("T", "40")), matmul=True)
    kw = dict(gemm_precision=os.environ.get("PREC", "bf16"))
elif which == "cfg5":
    ins, outs, mk, meta = W.cfg5_logp_grad(B=1 << 17, n=1024, J=64, K=8)
elif which == "metric":
    ins, outs, mk, meta = W.metric_graph(n=int(os.environ.get("N", "64")))
else:
    raise SystemExit("unknown workload")
f = pytensor.function(ins, outs, mode=cuda_mode(device_outputs=True, use_graph=False, **kw), trust_input=True)
a = [dev.to_device(x) for x in mk()]
for _ in range(steps):
    f(*a)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(steps):
    f(*a)
e1.record()
torch.cuda.synchronize()
print(which, "eager ms/eval", e0.elapsed_time(e1) / steps)
