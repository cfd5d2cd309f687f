"""Static instruction count of the cfg2 map+row-reduce kernel (K3): generates the kernel exactly as `mode="CUDA"` would
(trace-only mode + NVRTC, no GPU needed), disassembles the cubin and reports the SASS size of its loops — the main loop
processes 8 elements per thread and trip.  Where the kernel is instruction-issue bound, instructions per element are the
quantity that matters.

    python scripts/k3_sass_count.py                      # shipped configuration
    PTK_K3_ADDR=idx PTK_SCALAR_SIMPLIFY=0 python scripts/k3_sass_count.py   # index addressing, no scalar simplification
"""
import collections
import os
import re
import subprocess
import sys
import tempfile

cache = tempfile.mkdtemp(prefix="ptk_k3_sass_")
os.environ["PTK_KCACHE"] = cache
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

from pytensor_b200._host import ensure_pytensor  # noqa: E402

ensure_pytensor()
import pytensor  # noqa: E402

import pytensor_b200  # noqa: E402,F401
from pytensor_b200 import precompile  # noqa: E402
from pytensor_b200 import workloads as W  # noqa: E402

pytensor.config.floatX = "float32"
ins, outs, mk, _ = W.cfg2_fused_elemwise(4096)
f = pytensor.function(ins, outs, mode="CUDA")
precompile.trace_function(f, [np.empty_like(a) for a in mk()])
prog = f.vm.executor.program.steps[0].impl.prog
print("scalar program:", collections.Counter(i.op for i in prog.insts).most_common())
cub = [os.path.join(cache, n) for n in os.listdir(cache) if n.endswith(".cubin")]
assert len(cub) == 1, cub
sass = subprocess.run(["cuobjdump", "-sass", cub[0]], capture_output=True, text=True, check=True).stdout
res = subprocess.run(["cuobjdump", "-res-usage", cub[0]], capture_output=True, text=True, check=True).stdout
print(res.strip().splitlines()[-1].strip())
ins_ = [(int(m.group(1), 16), m.group(2).strip()) for m in re.finditer(r"/\*([0-9a-f]{4})\*/\s+(.*?);", sass)]
print("kernel:", len(ins_), "SASS instructions")
for addr, txt in ins_:
    m = re.search(r"BRA\S*\s+(?:!?U?P\d,\s*)?0x([0-9a-f]+)", txt)
    if m and int(m.group(1), 16) < addr:
        body = [t for a, t in ins_ if int(m.group(1), 16) <= a <= addr]
        nld = sum("LDG.E.128" in t for t in body)
        print(f"  loop 0x{int(m.group(1), 16):04x}..0x{addr:04x}: {len(body)} instructions, {nld} LDG.E.128")
        if nld == 4:
            hist = collections.Counter(re.sub(r"^@!?U?P\w+\s+", "", t).split()[0] for t in body)
            print(f"    main loop = {len(body) / 8:.2f} instructions per element:", dict(hist.most_common()))
