"""CUDA source generation for ROW-FUSED regions: one persistent kernel for a whole sub-graph whose tensors all carry an
independent leading batch axis (PyMC-style logp+grad over chains, SURVEY.md §8(f).4 / BASELINE.json configs[4]).

The reference executes such a sub-graph node by node and materialises every (B, n) intermediate
(`AdvancedSubtensor` -> `Gemm` -> `Composite` -> `Sum` / `Gemm` / `AdvancedIncSubtensor`, one C loop or BLAS call each;
its newest rewriter only starts to fuse indexing into Elemwise: pytensor/tensor/rewriting/fused_elemwise.py:107,278).
Here one WARP owns one batch row at a time and walks the region's ops as a short sequence of fused loops over the row's
own index spaces ("domains": n data rows, J groups, K covariates ...): gathers, skinny matrix products, elementwise
programs, row reductions, scatter-adds and the final sums over the batch all happen on values that live in registers or
in a few hundred bytes of the warp's shared memory.  Nothing of shape (B, n) is ever written to HBM.

Value kinds (B = batch rows):   R1 (B, m) per-row vector  |  R0 (B,) / (B, 1) per-row scalar
                                S1 (m,) / (1, m) shared vector  |  S0 shared scalar  |  S2 (p, q) shared matrix
Region ops (`ROp.kind`):
    ew    Elemwise ScalarProgram over R1 / R0 / S1 / S0 operands           (pytensor/tensor/elemwise.py:375)
    take  out[b, j] = x[b, idx[j]]                                        (AdvancedSubtensor, subtensor.py:1932)
    put   out[b, :] = x[b, :];  out[b, idx[j]] += y[b, j]                 (AdvancedIncSubtensor, subtensor.py:2275)
    gemm  out[b, :] = beta * z[b, :] + alpha * a[b, :] @ M                (Gemm / Dot22 with one skinny side, gemm.py:76,248)
    rsum  R1 -> R0 reduction over the row (CAReduce axis=1)               (elemwise.py:1233)
    csum  R1 -> S1 / R0 -> S0 sum over the batch axis (terminal: the region's cross-row outputs)
Every size except B is baked into the kernel (one NVRTC specialisation per set of domain sizes).

Schedule: each op runs in the loop of one domain (or in the per-row scalar phase); ops of the same (level, domain) share
ONE loop and hand values over in registers.  A value that a later loop needs (a different domain, or random access by a
gather / the skinny product) is materialised in the warp's shared memory; the level of an op is the number of such
hand-overs on its longest dependency chain.
"""

from __future__ import annotations

from dataclasses import dataclass, field

from .scalar import CTYPE, ITEMSIZE, PRELUDE, ScalarProgram, emit_body, literal

WARPS = 8            # warps per CTA (one batch row per warp at a time)
MAX_SMEM = 160 * 1024
GEMM_R_MAX_Q = 16    # "reduce" form: q accumulators in registers
GEMM_P_MAX_P = 32    # "pointwise" form: p operand values in registers
STAGE_MAX_BYTES = 4096
CTA_INDEX_MAX_BYTES = 32 * 1024   # shared index vectors up to 8192 entries get a per-CTA int32 table


def _cta_index_enabled() -> bool:
    import os

    return os.environ.get("PTK_ROWFUSE_CTA_INDEX", "1") != "0"


class NotFusable(Exception):
    """These sizes / layouts do not fit the row-fused kernel; the node then runs its constituent steps one by one."""


@dataclass
class RV:
    kind: str               # R1 | R0 | S1 | S0 | S2
    dtype: str
    dom: int = -1           # R1 / S1: length symbol;  S2: rows symbol
    dom2: int = -1          # S2: columns symbol
    ext: int = -1           # >= 0: index into the node's inputs
    out: int = -1           # >= 0: index into the node's outputs
    const: object = None    # S0 only: value baked into the source
    nd: int = 1             # ndim of the original tensor (outputs: (B,) vs (B, 1))


@dataclass
class ROp:
    kind: str
    ins: list
    outs: list
    prog: ScalarProgram | None = None   # ew
    red: str = "add"                    # rsum
    acc_dtype: str = "float64"          # rsum / csum
    alpha: int = -1                     # gemm: value ids of the S0 scalars (const or external)
    beta: int = -1
    name: str = ""


@dataclass
class RegionPlan:
    vals: list = field(default_factory=list)   # RV
    ops: list = field(default_factory=list)    # ROp, topological
    n_ext: int = 0
    n_out: int = 0

    def signature(self):
        return repr(([(v.kind, v.dtype, v.dom, v.dom2, v.ext, v.out, repr(v.const), v.nd) for v in self.vals],
                     [(o.kind, o.ins, o.outs, o.prog.signature() if o.prog else None, o.red, o.acc_dtype, o.alpha, o.beta)
                      for o in self.ops]))


@dataclass
class ExtLayout:
    """Runtime layout of one external input (element strides; `grp` = pointer-parameter index: inputs that are views of
    the same memory share one parameter so that the compiler sees identical loads)."""
    grp: int
    strides: tuple
    offset: int = 0          # element offset from the group's base pointer
    aligned16: bool = True


@dataclass
class KernelSpec:
    source: str
    name: str
    finish_name: str
    smem_bytes: int
    acc_len: int
    n_groups: int
    out_order: list          # node-output indices of the R-kind outputs, in parameter order
    csum_out: list           # (node-output index, offset into the accumulator vector, length, out dtype)
    params: list             # human-readable parameter list (tests)
    n_loops: int = 0


_HELPERS = r"""
template <typename T> __device__ __forceinline__ T ptk_shx(T v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
template <typename T> __device__ __forceinline__ T ptk_nanmax(T a, T b) { return (b > a) ? b : ((a >= b) ? a : (a + b)); }
template <typename T> __device__ __forceinline__ T ptk_nanmin(T a, T b) { return (b < a) ? b : ((a <= b) ? a : (a + b)); }
"""

_RED = {
    "add": lambda a, b: f"(({a}) + ({b}))", "mul": lambda a, b: f"(({a}) * ({b}))",
    "maximum": lambda a, b: f"ptk_nanmax(({a}), ({b}))", "minimum": lambda a, b: f"ptk_nanmin(({a}), ({b}))",
}
_RED_ID = {"add": 0, "mul": 1, "maximum": float("-inf"), "minimum": float("inf")}


@dataclass
class _Micro:
    kind: str
    op: ROp
    loop_dom: int | None
    reads: list              # (value id, "pt" | "full")
    writes: list             # (value id, "pt" | "red" | "scalar")
    extra: dict = field(default_factory=dict)
    level: int = 0


def _expand(plan: RegionPlan, dims: dict):
    """Region ops -> micro-ops with their loop domain; picks the form of each skinny product from the concrete sizes.
    Returns (micro list, extended value list)."""
    vals = list(plan.vals)
    micro = []

    def new_val(kind, dtype, dom):
        vals.append(RV(kind, dtype, dom=dom))
        return len(vals) - 1

    for op in plan.ops:
        if op.kind == "ew":
            outk = vals[op.outs[0]].kind
            dom = vals[op.outs[0]].dom if outk == "R1" else None
            reads = []
            for i in op.ins:
                k = vals[i].kind
                reads.append((i, "pt" if k in ("R1", "S1") else "full"))
            micro.append(_Micro("ew", op, dom, reads, [(o, "pt" if outk == "R1" else "scalar") for o in op.outs]))
        elif op.kind == "take":
            x, idx = op.ins
            micro.append(_Micro("take", op, vals[op.outs[0]].dom, [(x, "full"), (idx, "pt")], [(op.outs[0], "pt")]))
        elif op.kind == "put":
            x, y, idx = op.ins
            buf = new_val("R1", vals[y].dtype, vals[x].dom)
            micro.append(_Micro("put_acc", op, vals[y].dom, [(y, "pt"), (idx, "pt")], [(buf, "red")], {"buf": buf}))
            micro.append(_Micro("put_fin", op, vals[x].dom, [(x, "pt"), (buf, "pt")], [(op.outs[0], "pt")], {"buf": buf}))
        elif op.kind == "gemm":
            z, a, m = op.ins
            out = op.outs[0]
            p, q = dims[vals[a].dom], dims[vals[out].dom]
            if q <= GEMM_R_MAX_Q and p > q:
                acc = new_val("R1", vals[out].dtype, vals[out].dom)
                micro.append(_Micro("gemm_acc", op, vals[a].dom, [(a, "pt"), (m, "full")], [(acc, "red")], {"acc": acc, "q": q}))
                reads = [(acc, "pt")] + ([(z, "pt")] if z >= 0 else [])
                micro.append(_Micro("gemm_fin", op, vals[out].dom, reads, [(out, "pt")], {"acc": acc}))
            elif p <= GEMM_P_MAX_P:
                reads = [(a, "full"), (m, "full")] + ([(z, "pt")] if z >= 0 else [])
                micro.append(_Micro("gemm_pt", op, vals[out].dom, reads, [(out, "pt")], {"p": p}))
            else:
                raise NotFusable(f"matrix product {p} x {q} has no skinny side")
        elif op.kind == "rsum":
            micro.append(_Micro("rsum", op, vals[op.ins[0]].dom, [(op.ins[0], "pt")], [(op.outs[0], "red")]))
        elif op.kind == "csum":
            k = vals[op.ins[0]].kind
            if k == "R1":
                micro.append(_Micro("csum_v", op, vals[op.ins[0]].dom, [(op.ins[0], "pt")], []))
            else:
                micro.append(_Micro("csum_s", op, None, [(op.ins[0], "full")], []))
        else:
            raise NotFusable(f"unknown region op {op.kind}")
    return micro, vals


def _schedule(micro, vals):
    producer = {}
    for m in micro:
        for v, mode in m.writes:
            producer[v] = (m, mode)
    for m in micro:
        lvl = 0
        for v, need in m.reads:
            if v not in producer:
                continue
            pm, mode = producer[v]
            if mode == "scalar":
                lvl = max(lvl, pm.level)
            elif need == "pt" and mode == "pt" and pm.loop_dom is not None and pm.loop_dom == m.loop_dom:
                lvl = max(lvl, pm.level)
            else:
                lvl = max(lvl, pm.level + 1)
        m.level = lvl
    return producer


def gen_region_kernel(plan: RegionPlan, dims: dict, ext: list, name: str, idx_check: bool = True) -> KernelSpec:
    """`dims`: domain symbol -> size; `ext[k]`: ExtLayout of node input k."""
    micro, vals = _expand(plan, dims)
    producer = _schedule(micro, vals)
    for v in vals:
        if v.kind in ("R1", "R0") and v.dtype not in ("float32", "float64"):
            raise NotFusable(f"per-row values of dtype {v.dtype}")

    def is_ext(i):
        return vals[i].ext >= 0

    # ---- which values need memory between loops ------------------------------------------------------------------------
    consumers = {}
    for m in micro:
        for v, need in m.reads:
            consumers.setdefault(v, []).append((m, need))
    in_smem = {}        # value id -> byte offset in the warp's slab
    staged = {}         # external R1 value id -> byte offset (copied to smem once per row)
    off = 0

    def slab(nbytes):
        nonlocal off
        o = off
        off = (off + nbytes + 15) // 16 * 16
        return o

    for i, v in enumerate(vals):
        if v.kind != "R1":
            continue
        if is_ext(i):
            full = any(need == "full" for _, need in consumers.get(i, []))
            nb = dims[v.dom] * ITEMSIZE[v.dtype]
            if full and nb <= STAGE_MAX_BYTES:
                staged[i] = slab(nb)
            continue
        if i not in producer:
            continue
        pm, mode = producer[i]
        need_mem = mode == "red"
        for cm, need in consumers.get(i, []):
            if need == "full" or cm.loop_dom != pm.loop_dom or cm.level != pm.level:
                need_mem = True
        if need_mem and v.out < 0:
            in_smem[i] = slab(dims[v.dom] * ITEMSIZE[v.dtype])
        elif need_mem and mode == "red":
            in_smem[i] = slab(dims[v.dom] * ITEMSIZE[v.dtype])
    warp_bytes = off

    # ---- cross-row accumulators ------------------------------------------------------------------------------------------
    acc_len = 0
    csum_out = []
    acc_off = {}
    for m in micro:
        if m.kind in ("csum_v", "csum_s"):
            o = m.op.outs[0]
            n = dims[vals[m.op.ins[0]].dom] if m.kind == "csum_v" else 1
            acc_off[id(m)] = acc_len
            csum_out.append((vals[o].out, acc_len, n, vals[o].dtype))
            acc_len += n
    acc_bytes = (acc_len * 8 + 15) // 16 * 16
    smem_bytes = acc_bytes + WARPS * warp_bytes
    if smem_bytes > MAX_SMEM:
        raise NotFusable(f"{smem_bytes} bytes of shared memory per CTA")

    # ---- parameters -------------------------------------------------------------------------------------------------------
    n_groups = max([e.grp for e in ext], default=-1) + 1
    grp_dtype = {}
    for i, v in enumerate(vals):
        if v.ext >= 0 and v.const is None:
            grp_dtype.setdefault(ext[v.ext].grp, v.dtype)
    params, pdesc = [], []
    for g in range(n_groups):
        T = CTYPE[grp_dtype.get(g, "float32")]
        params.append(f"const {T}* __restrict__ p{g}")
        pdesc.append(("ext", g))
    out_order = []
    for i, v in enumerate(vals):
        if v.out >= 0 and v.kind in ("R1", "R0"):
            params.append(f"{CTYPE[v.dtype]}* __restrict__ q{v.out}")
            pdesc.append(("out", v.out))
            out_order.append(v.out)
    params += ["double* __restrict__ partials", "int* err", "long long B"]
    pdesc += [("partials",), ("err",), ("B",)]

    def gptr(i):
        """Typed base pointer expression of external value i (its group's pointer may have another element type)."""
        v = vals[i]
        e = ext[v.ext]
        T = CTYPE[v.dtype]
        base = f"p{e.grp}" if grp_dtype.get(e.grp) == v.dtype else f"reinterpret_cast<const {T}*>(p{e.grp})"
        return f"({base} + {e.offset}LL)" if e.offset else base

    # ---- expression helpers ------------------------------------------------------------------------------------------------
    lines = []
    bodies = []

    def scalar_expr(i):
        v = vals[i]
        if v.const is not None:
            return literal(v.dtype, v.const)
        if v.kind == "S0":
            return f"s{i}"
        return f"v{i}"

    def full_access(i, ix):
        """Element `ix` of the row vector i (complete before the current loop)."""
        if i in staged:
            return f"st{i}[{ix}]"
        if i in in_smem:
            return f"sm{i}[{ix}]"
        v = vals[i]
        if is_ext(i):
            e = ext[v.ext]
            return f"__ldg({gptr(i)} + b * {e.strides[0]}LL + (long long)({ix}) * {e.strides[-1] if v.kind == 'R1' else 0}LL)"
        if v.out >= 0:
            return f"q{v.out}[b * {dims[v.dom]}LL + ({ix})]"
        raise NotFusable("internal: value has no storage")

    class Loop:
        def __init__(self, dom, level):
            self.dom, self.level = dom, level
            self.pre, self.body, self.post = [], [], []
            self.loaded = {}
            self.local = set()
            self.writes_smem = False

        def pt(self, i):
            """Value i at the loop index j."""
            v = vals[i]
            if v.kind in ("R0", "S0"):
                return scalar_expr(i)
            if i in self.local:
                return f"v{i}"
            if i in self.loaded:
                return self.loaded[i]
            T = CTYPE[v.dtype]
            if is_ext(i):
                e = ext[v.ext]
                if v.kind == "R1":
                    src = f"__ldg({gptr(i)} + b * {e.strides[0]}LL + (long long)j * {e.strides[1]}LL)"
                else:
                    src = f"__ldg({gptr(i)} + (long long)j * {e.strides[-1]}LL)"
            elif i in in_smem:
                src = f"sm{i}[j]"
            elif v.out >= 0:
                src = f"q{v.out}[b * {dims[v.dom]}LL + j]"
            else:
                raise NotFusable("internal: pointwise read of a value that was never materialised")
            nm = f"l{i}"
            self.body.append(f"const {T} {nm} = {src};")
            self.loaded[i] = nm
            return nm

        def define(self, i, expr):
            v = vals[i]
            T = CTYPE[v.dtype]
            self.body.append(f"const {T} v{i} = ({T})({expr});")
            self.local.add(i)
            self.finish_value(i)

        def finish_value(self, i):
            v = vals[i]
            if i in in_smem:
                self.body.append(f"sm{i}[j] = v{i};")
                self.writes_smem = True
            if v.out >= 0:
                self.body.append(f"q{v.out}[b * {dims[v.dom]}LL + j] = v{i};")

    cta_idx = {}        # (index value, axis length) -> (name, byte offset inside the CTA index region, entries)
    cta_idx_bytes = 0
    cta_idx_code = []

    def index_expr(L, idx, n_src):
        """Bounds-checked (negative wrap like NumPy) index expression; flags `err` and clamps on out-of-bounds.

        An index vector SHARED by all batch rows (the group index of a hierarchical model) is wrapped and checked ONCE per
        CTA into an int32 table in shared memory; the per-row loops then read one LDS instead of re-validating a 64-bit
        global load for every (row, element) — in the cfg5 kernel that check was ~20 of 70 instructions per element, twice
        (gather and scatter) inside divergence-guarded regions.  PTK_ROWFUSE_CTA_INDEX=0 keeps the per-use form."""
        nonlocal cta_idx_bytes
        v = vals[idx]
        n_ent = dims[v.dom]
        if (v.kind == "S1" and is_ext(idx) and v.const is None and L.dom == v.dom and _cta_index_enabled()
                and n_src < 2 ** 31 and n_ent * 4 <= CTA_INDEX_MAX_BYTES):
            key = (idx, n_src)
            if key not in cta_idx and smem_bytes + cta_idx_bytes + n_ent * 4 + 16 <= MAX_SMEM:
                nm = f"cix{len(cta_idx)}"
                e = ext[v.ext]
                cta_idx[key] = (nm, cta_idx_bytes, n_ent)
                chk = f" if ((unsigned long long)t >= {n_src}ULL) {{ atomicExch(err, 1); t = 0; }}" if idx_check else ""
                cta_idx_code.append(
                    f"int* const {nm} = reinterpret_cast<int*>(ptk_smem + {smem_bytes + cta_idx_bytes});\n"
                    f"  for (int jj = threadIdx.x; jj < {n_ent}; jj += {WARPS * 32}) {{\n"
                    f"    long long t = (long long)__ldg({gptr(idx)} + (long long)jj * {e.strides[-1]}LL);\n"
                    f"    if (t < 0) t += {n_src};{chk}\n"
                    f"    {nm}[jj] = (int)t;\n  }}")
                cta_idx_bytes += (n_ent * 4 + 15) // 16 * 16
            if key in cta_idx:
                nm = f"ix{len(L.body)}"
                L.body.append(f"const int {nm} = {cta_idx[key][0]}[j];")
                return nm
        raw = L.pt(idx)
        nm = f"ix{len(L.body)}"
        L.body.append(f"long long {nm} = (long long)({raw});")
        L.body.append(f"if ({nm} < 0) {nm} += {n_src};")
        if idx_check:
            L.body.append(f"if ((unsigned long long){nm} >= {n_src}ULL) {{ atomicExch(err, 1); {nm} = 0; }}")
        return nm

    def vec_matrix_row(L, m, fixed_dom_is_rows, fixed_ix, count, tag):
        """`count` consecutive logical elements of the shared matrix m along its OTHER axis at position `fixed_ix` of the
        fixed axis; 128-bit loads when that run is contiguous and aligned.  Returns the list of element expressions."""
        v = vals[m]
        e = ext[v.ext]
        T = CTYPE[v.dtype]
        s_fixed, s_run = (e.strides[0], e.strides[1]) if fixed_dom_is_rows else (e.strides[1], e.strides[0])
        vw = 16 // ITEMSIZE[v.dtype]
        base = f"({gptr(m)} + (long long)({fixed_ix}) * {s_fixed}LL)"
        if s_run == 1 and count % vw == 0 and s_fixed % vw == 0 and e.aligned16 and e.offset % vw == 0:
            VT = "float4" if v.dtype == "float32" else "double2"
            comps = ["x", "y", "z", "w"][:vw]
            out = []
            for c in range(count // vw):
                nm = f"mv{tag}_{c}"
                L.body.append(f"const {VT} {nm} = __ldg(reinterpret_cast<const {VT}*>({base}) + {c});")
                out += [f"{nm}.{x}" for x in comps]
            return out
        out = []
        for c in range(count):
            nm = f"ms{tag}_{c}"
            L.body.append(f"const {T} {nm} = __ldg({base} + {c * s_run}LL);")
            out.append(nm)
        return out

    # ---- emit -----------------------------------------------------------------------------------------------------------------
    max_level = max([m.level for m in micro], default=0)
    row = []            # statements of one batch row
    decl_row = []
    n_loops = 0

    # staging of small externals that are gathered from / multiplied as a whole
    for i, o in staged.items():
        v = vals[i]
        e = ext[v.ext]
        n = dims[v.dom]
        row.append(f"for (int j = lane; j < {n}; j += 32) st{i}[j] = __ldg({gptr(i)} + b * {e.strides[0]}LL + (long long)j * {e.strides[1]}LL);")
    if staged:
        row.append("__syncwarp();")
    for i, v in enumerate(vals):  # per-row scalars handed in from outside: one load per row
        if v.kind == "R0" and is_ext(i):
            row.append(f"const {CTYPE[v.dtype]} v{i} = __ldg({gptr(i)} + b * {ext[v.ext].strides[0]}LL);")

    body_id = 0
    for lvl in range(max_level + 1):
        # scalar phase
        for m in micro:
            if m.level != lvl or m.loop_dom is not None:
                continue
            if m.kind == "ew":
                fn = f"ptk_body_{body_id}"
                body_id += 1
                bodies.append(emit_body(m.op.prog, fn))
                for o in m.op.outs:
                    row.append(f"{CTYPE[vals[o].dtype]} v{o};")
                row.append(f"{fn}({', '.join([scalar_expr(i) for i in m.op.ins] + [f'v{o}' for o in m.op.outs])});")
                for o in m.op.outs:
                    if vals[o].out >= 0:
                        row.append(f"if (lane == 0) q{vals[o].out}[b] = v{o};")
            elif m.kind == "csum_s":
                row.append(f"if (lane == 0) atomicAdd(&cta_acc[{acc_off[id(m)]}], (double)({scalar_expr(m.op.ins[0])}));")
        # loops
        doms = []
        for m in micro:
            if m.level == lvl and m.loop_dom is not None and m.loop_dom not in doms:
                doms.append(m.loop_dom)
        for d in doms:
            L = Loop(d, lvl)
            n = dims[d]
            for m in micro:
                if m.level != lvl or m.loop_dom != d:
                    continue
                op = m.op
                if m.kind == "ew":
                    fn = f"ptk_body_{body_id}"
                    body_id += 1
                    bodies.append(emit_body(op.prog, fn))
                    args = [L.pt(i) for i in op.ins]
                    for o in op.outs:
                        L.body.append(f"{CTYPE[vals[o].dtype]} v{o};")
                        L.local.add(o)
                    L.body.append(f"{fn}({', '.join(args + [f'v{o}' for o in op.outs])});")
                    for o in op.outs:
                        L.finish_value(o)
                elif m.kind == "take":
                    x, idx = op.ins
                    ix = index_expr(L, idx, dims[vals[x].dom])
                    L.define(op.outs[0], full_access(x, ix))
                elif m.kind == "put_acc":
                    x, y, idx = op.ins
                    buf = m.extra["buf"]
                    nb = dims[vals[buf].dom]
                    L.pre.append(f"for (int jj = lane; jj < {nb}; jj += 32) sm{buf}[jj] = 0;")
                    L.pre.append("__syncwarp();")
                    ix = index_expr(L, idx, nb)
                    if vals[buf].dtype == "float64":
                        # fp64 shared-memory atomicAdd is a compare-and-swap loop on sm_90, so lanes that hit the same
                        # bin would add in an arbitrary order; adding in lane order (the lanes of one iteration are
                        # consecutive positions j) keeps the sum bit-equal to a sequential scatter-add
                        L.body.append("#ifdef __CUDA_ARCH__")
                        L.body.append(f"{{ const int pix = {ix}; const double pv = {L.pt(y)};"
                                      f" const unsigned pm = ({n} - (j - lane) >= 32) ? 0xffffffffu"
                                      f" : ((1u << ({n} - (j - lane))) - 1u);"
                                      f" for (int q = 0; q < 32; ++q) {{ if (lane == q) sm{buf}[pix] += pv; __syncwarp(pm); }} }}")
                        L.body.append("#else")
                        L.body.append(f"atomicAdd(&sm{buf}[{ix}], {L.pt(y)});")
                        L.body.append("#endif")
                    else:
                        L.body.append(f"atomicAdd(&sm{buf}[{ix}], {L.pt(y)});")
                    L.writes_smem = True
                elif m.kind == "put_fin":
                    x = op.ins[0]
                    L.define(op.outs[0], f"{L.pt(x)} + {L.pt(m.extra['buf'])}")
                elif m.kind in ("gemm_pt", "gemm_acc", "gemm_fin"):
                    z, a, mm = op.ins
                    out = op.outs[0]
                    T = CTYPE[vals[out].dtype]
                    al, be = scalar_expr(op.alpha), scalar_expr(op.beta)
                    beta_zero = vals[op.beta].const is not None and float(vals[op.beta].const) == 0.0
                    if m.kind == "gemm_pt":
                        p = m.extra["p"]
                        for k in range(p):  # the row's p operand values: registers, loaded once per row
                            L.pre.append(f"const {T} ga{out}_{k} = {full_access(a, k)};")
                        elems = vec_matrix_row(L, mm, False, "j", p, f"{out}")
                        acc = f"gs{out}"
                        L.body.append(f"{T} {acc} = ({T})0;")
                        for k in range(p):
                            L.body.append(f"{acc} = fma(ga{out}_{k}, {elems[k]}, {acc});")
                        expr = f"{al} * {acc}" if (z < 0 or beta_zero) else f"{be} * {L.pt(z)} + {al} * {acc}"
                        L.define(out, expr)
                    elif m.kind == "gemm_acc":
                        q = m.extra["q"]
                        acc = m.extra["acc"]
                        for k in range(q):
                            L.pre.append(f"{T} gr{acc}_{k} = ({T})0;")
                        elems = vec_matrix_row(L, mm, True, "j", q, f"{acc}")
                        av = L.pt(a)
                        for k in range(q):
                            L.body.append(f"gr{acc}_{k} = fma({av}, {elems[k]}, gr{acc}_{k});")
                        for k in range(q):
                            L.post.append(f"#pragma unroll\n      for (int s = 16; s > 0; s >>= 1) gr{acc}_{k} += ptk_shx(gr{acc}_{k}, s);")
                        L.post.append("if (lane == 0) { " + " ".join(f"sm{acc}[{k}] = gr{acc}_{k};" for k in range(q)) + " }")
                        L.writes_smem = True
                    else:
                        acc = m.extra["acc"]
                        expr = (f"{al} * {L.pt(acc)}" if (z < 0 or beta_zero) else f"{be} * {L.pt(z)} + {al} * {L.pt(acc)}")
                        L.define(out, expr)
                elif m.kind == "rsum":
                    o = op.outs[0]
                    A = CTYPE[op.acc_dtype]
                    L.pre.append(f"{A} ra{o} = ({A}){literal(op.acc_dtype, _RED_ID[op.red])};")
                    L.body.append(f"ra{o} = {_RED[op.red](f'ra{o}', f'({A})(' + L.pt(op.ins[0]) + ')')};")
                    L.post.append(f"#pragma unroll\n      for (int s = 16; s > 0; s >>= 1) ra{o} = {_RED[op.red](f'ra{o}', f'ptk_shx(ra{o}, s)')};")
                    L.post.append(f"const {CTYPE[vals[o].dtype]} v{o} = ({CTYPE[vals[o].dtype]})ra{o};")
                    if vals[o].out >= 0:
                        L.post.append(f"if (lane == 0) q{vals[o].out}[b] = v{o};")
                elif m.kind == "csum_v":
                    L.body.append(f"atomicAdd(&cta_acc[{acc_off[id(m)]} + j], (double)({L.pt(op.ins[0])}));")
            n_loops += 1
            row += L.pre
            row.append(f"#pragma unroll 4\n    for (int j = lane; j < {n}; j += 32) {{")
            row += ["  " + s for s in L.body]
            row.append("}")
            row += L.post
            row.append("__syncwarp();")
    row.append("__syncwarp();")

    sm_decl = []
    for i, o in list(staged.items()):
        sm_decl.append(f"{CTYPE[vals[i].dtype]}* const st{i} = reinterpret_cast<{CTYPE[vals[i].dtype]}*>(wsm + {o});")
    for i, o in in_smem.items():
        sm_decl.append(f"{CTYPE[vals[i].dtype]}* const sm{i} = reinterpret_cast<{CTYPE[vals[i].dtype]}*>(wsm + {o});")
    s0_decl = []
    for i, v in enumerate(vals):
        if v.kind == "S0" and v.const is None and v.ext >= 0:
            s0_decl.append(f"const {CTYPE[v.dtype]} s{i} = __ldg({gptr(i)});")

    finish_name = name + "_fin"
    fin_params = ["const double* __restrict__ partials", "int nblocks"]
    fin_body = []
    for (oi, o, n, dt) in csum_out:
        fin_params.append(f"{CTYPE[dt]}* __restrict__ o{oi}")
        fin_body.append(f"    if (e >= {o} && e < {o + n}) o{oi}[e - {o}] = ({CTYPE[dt]})acc;")
    nl = "\n"
    src = f"""{PRELUDE}
{_HELPERS}
{nl.join(bodies)}

#define ACC_LEN {acc_len}
extern "C" __global__ void __launch_bounds__({WARPS * 32}) {name}({', '.join(params)}) {{
  extern __shared__ __align__(16) unsigned char ptk_smem[];
  double* const cta_acc = reinterpret_cast<double*>(ptk_smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char* const wsm = ptk_smem + {acc_bytes} + warp * {warp_bytes};
  {(nl + '  ').join(sm_decl)}
  for (int i = threadIdx.x; i < ACC_LEN; i += {WARPS * 32}) cta_acc[i] = 0.0;
  {(nl + '  ').join(cta_idx_code)}
  __syncthreads();
  {(nl + '  ').join(s0_decl)}
  const long long nwarps = (long long)gridDim.x * {WARPS};
  for (long long b = (long long)blockIdx.x * {WARPS} + warp; b < B; b += nwarps) {{
    {(nl + '    ').join(row)}
  }}
  __syncthreads();
  for (int i = threadIdx.x; i < ACC_LEN; i += {WARPS * 32}) partials[(long long)blockIdx.x * ACC_LEN + i] = cta_acc[i];
}}

// sums the per-CTA partial accumulators (fp64) and casts to the outputs' dtypes: one warp per accumulator element
extern "C" __global__ void __launch_bounds__(256) {finish_name}({', '.join(fin_params)}) {{
  const int lane = threadIdx.x & 31;
  const int e = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (e >= ACC_LEN) return;
  double acc = 0.0;
  for (int k = lane; k < nblocks; k += 32) acc += partials[(long long)k * ACC_LEN + e];
  #pragma unroll
  for (int s = 16; s > 0; s >>= 1) acc += ptk_shx(acc, s);
  if (lane == 0) {{
{nl.join(fin_body)}
  }}
}}
"""
    return KernelSpec(src, name, finish_name, smem_bytes + cta_idx_bytes, acc_len, n_groups, out_order, csum_out, pdesc, n_loops)
