"""CUDA source generation for CAReduce kernels (K2) and the fused map+reduce kernel (K3).

Replaces `CAReduce._c_all` (pytensor/tensor/elemwise.py:1520-1678; loop generators elemwise_cgen.py:467,578).
Accumulator dtype follows the reference (`_acc_dtype` elemwise.py:1383-1417: fp32 sums accumulate in fp64, small
ints in int64); the combine order is a tree instead of the C loop's sequential order, which is why the parity bar
for floating-point reductions is a tolerance and not bit-exactness.

Kernel shapes (the host normalises every reduction to one of them):
* `row`     — input(s) viewed as (rows, cols), reduce over the contiguous `cols`; TPR threads per row, 128-bit loads.
              Optional fused map stage: a ScalarProgram applied to n_in operands (each contiguous or constant along
              cols) whose outputs may also be stored — this is the Elemwise->Sum fusion the reference cannot do for
              multi-input Elemwise (rewriting/elemwise.py:1119-1121).
* `col`     — input viewed as (outer, red, inner) contiguous, reduce over the strided middle axis; threads along
              `inner` (coalesced), optional split of `red` across blockIdx.z with a finishing pass.
* `generic` — any strides: one thread per output element walks the reduced index space.
* `finish`  — reduces `nsplit` partial accumulators per output (second pass of split reductions).
"""

from __future__ import annotations

from .scalar import CTYPE, PRELUDE, ScalarProgram, emit_body, is_float, literal, single_op_program
from .elemwise import _VEC_HELPERS, MAX_DIMS

REDUCE_OPS = {
    "add": lambda a, b, dt: f"(({a}) + ({b}))",
    "mul": lambda a, b, dt: f"(({a}) * ({b}))",
    "maximum": lambda a, b, dt: (f"ptk_nanmax(({a}), ({b}))" if is_float(dt) else f"((({b}) > ({a})) ? ({b}) : ({a}))"),
    "minimum": lambda a, b, dt: (f"ptk_nanmin(({a}), ({b}))" if is_float(dt) else f"((({b}) < ({a})) ? ({b}) : ({a}))"),
    "and": lambda a, b, dt: f"(({a}) & ({b}))",
    "or": lambda a, b, dt: f"(({a}) | ({b}))",
    "xor": lambda a, b, dt: f"(({a}) ^ ({b}))",
}

_RED_HELPERS = r"""
template <typename T> __device__ __forceinline__ T ptk_nanmax(T a, T b) { return (b > a) ? b : ((a >= b) ? a : (a + b)); }
template <typename T> __device__ __forceinline__ T ptk_nanmin(T a, T b) { return (b < a) ? b : ((a <= b) ? a : (a + b)); }
template <typename T> __device__ __forceinline__ T ptk_shfl_xor(T v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
template <> __device__ __forceinline__ unsigned char ptk_shfl_xor<unsigned char>(unsigned char v, int m) { return (unsigned char)__shfl_xor_sync(0xffffffffu, (int)v, m); }
template <> __device__ __forceinline__ signed char ptk_shfl_xor<signed char>(signed char v, int m) { return (signed char)__shfl_xor_sync(0xffffffffu, (int)v, m); }
template <> __device__ __forceinline__ short ptk_shfl_xor<short>(short v, int m) { return (short)__shfl_xor_sync(0xffffffffu, (int)v, m); }
template <> __device__ __forceinline__ unsigned short ptk_shfl_xor<unsigned short>(unsigned short v, int m) { return (unsigned short)__shfl_xor_sync(0xffffffffu, (int)v, m); }
"""


def _combine(op, acc_dtype):
    fn = REDUCE_OPS[op]
    return f"__device__ __forceinline__ ACC ptk_red(ACC a, ACC b) {{ return (ACC){fn('a', 'b', acc_dtype)}; }}"


def _block_reduce_code(tpr: int) -> str:
    """Reduce `acc` across the TPR threads that share a row; result valid in the first of them."""
    if tpr == 32:
        return """
    #pragma unroll
    for (int m = 16; m > 0; m >>= 1) acc = ptk_red(acc, ptk_shfl_xor<ACC>(acc, m));
"""
    return f"""
    #pragma unroll
    for (int m = 16; m > 0; m >>= 1) acc = ptk_red(acc, ptk_shfl_xor<ACC>(acc, m));
    __shared__ ACC s_part[8];                 // one partial per warp of the CTA; a row owns {tpr // 32} consecutive warps
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if ((threadIdx.x & (TPR - 1)) == 0) {{
      #pragma unroll
      for (int w = 1; w < {tpr // 32}; ++w) acc = ptk_red(acc, s_part[(threadIdx.x >> 5) + w]);
    }}
    __syncthreads();
"""


def _k3_pipeline() -> str:
    """How the row kernel keeps memory busy while the scalar bodies run: "none" (occupancy only: 40 registers, 6 CTAs per SM),
    "l2" (same, plus an L2 prefetch of the next trip), "regs" (register software pipeline with pinned loads: 64-68
    registers, 3-4 CTAs per SM — measured SLOWER on cfg2, 43.5-44.7 us vs 39.1 us: the long dependent scalar chains need the
    warps more than the loads need the head start).  PTK_K3_PIPE overrides."""
    import os

    return os.environ.get("PTK_K3_PIPE", "none")   # also: "tma" = gen_row_kernel_tma (bulk-copy staging through shared memory)


def _k3_running_pointers() -> bool:
    """Column walk of the default row kernel: running pointers (one 64-bit add per operand and trip; a trip's second vector
    is addressed at a compile-time distance from the first) instead of re-deriving every address from the 32-bit column
    index — 425 -> 408 SASS instructions per 8-element trip of the cfg2 kernel at the same 40 registers.  PTK_K3_ADDR=idx
    restores the index form."""
    import os

    return os.environ.get("PTK_K3_ADDR", "ptr") != "idx"


def _k3_min_blocks() -> int:
    """CTAs per SM the row kernel is compiled for (register cap 65536 / (256 * n)): 4 leaves 64 registers — enough for
    the two-trip software pipeline of a 2-input Composite with a couple of spilled words; PTK_K3_MINB overrides (A/B)."""
    import os

    # "none": capped at 42 registers like the L2 variant — left alone the compiler hoists the trip's four loads and takes
    # 64 registers (4 CTAs/SM): 40.1 us vs 39.1 us on cfg2
    return int(os.environ.get("PTK_K3_MINB", {"regs": "4"}.get(_k3_pipeline(), "6")))


def gen_row_kernel(prog: ScalarProgram, name: str, col_modes: tuple, store_map: tuple, red_op: str, acc_dtype: str,
                   out_dtype: str, identity, vw: int, tpr: int, inplace: dict | None = None) -> str:
    """Fused map + row reduction.

    prog: n_in inputs -> n_map outputs; output 0 of `prog` feeds the reduction.  store_map[k] tells whether map
    output k is also written to memory (po{k}); col_modes as in the vec elemwise kernel (inputs then stored outputs).
    Params: pi*, po* (stored map outputs only), pred (reduction result or partials), row strides (inputs, stored
    outputs), rows, cols, nsplit.  grid = (row_blocks, nsplit); a block owns 256/TPR rows.
    When nsplit > 1 `pred` holds ACC partials laid out [row][split], finished by the `finish` kernel.
    """
    n_in, n_map = len(prog.in_dtypes), len(prog.out_dtypes)
    ACC, OUT = CTYPE[acc_dtype], CTYPE[out_dtype]
    restrict = "" if inplace else " __restrict__"
    params = [f"const {CTYPE[d]}*{restrict} pi{k}" for k, d in enumerate(prog.in_dtypes)]
    stored = [k for k in range(n_map) if store_map[k]]
    params += [f"{CTYPE[prog.out_dtypes[k]]}*{restrict} po{k}" for k in stored]
    params += ["void* __restrict__ pred"]
    params += [f"long long rsi{k}" for k in range(n_in)]
    params += [f"long long rso{k}" for k in stored]
    params += ["long long rows", "long long cols", "int nsplit"]
    rows_per_block = 256 // tpr

    # Row base pointers are formed once per row (64-bit); the column walk uses 32-bit vector indices (the launcher keeps
    # cols < 2^31) and no integer division: VW and TPR are powers of two, the split bounds only exist when nsplit > 1.
    base_in = "\n".join(f"      const {CTYPE[d]}* q{k} = pi{k} + r * rsi{k};" for k, d in enumerate(prog.in_dtypes))
    base_out = "\n".join(f"      {CTYPE[prog.out_dtypes[k]]}* w{k} = po{k} + r * rso{k};" for k in stored)

    def loads(tag, cexpr):
        out = []
        for k, d in enumerate(prog.in_dtypes):
            T = CTYPE[d]
            if col_modes[k] == 1:
                out.append(f"          const PVec<{T}, VW> v{tag}{k} = ptk_ldv<{T}, VW>(q{k} + {cexpr});")
        return "\n".join(out)

    row_scalars = "\n".join(f"      const {CTYPE[d]} s{k} = q{k}[0];" for k, d in enumerate(prog.in_dtypes) if col_modes[k] != 1)
    # (A float32 map output is promoted to the accumulator type element by element: adding the VW lanes of a vector in fp32
    # first would save conversions but breaks the reference's "fp32 sums accumulate in float64" contract on cancelling sums —
    # measured 2e-6 on a 200000-term row, tests/test_gpu_careduce.py::test_fp32_sum_accumulates_in_fp64.)

    def compute(tag, cexpr):
        call_in = [f"v{tag}{k}.v[e]" if col_modes[k] == 1 else f"s{k}" for k in range(n_in)]
        decl = "\n".join(f"          PVec<{CTYPE[d]}, VW> o{tag}{k};" for k, d in enumerate(prog.out_dtypes))
        call_out = [f"o{tag}{k}.v[e]" for k in range(n_map)]
        st_ = "\n".join(f"          ptk_stv<{CTYPE[prog.out_dtypes[k]]}, VW>(w{k} + {cexpr}, o{tag}{k});" for k in stored)
        body = f"""          #pragma unroll
          for (int e = 0; e < VW; ++e) {{
            ptk_body({', '.join(call_in + call_out)});
            acc = ptk_red(acc, (ACC)o{tag}0.v[e]);
          }}"""
        return f"{decl}\n{body}\n{st_}"

    vec_in = [k for k in range(n_in) if col_modes[k] == 1]

    def pin_loads(tag, base, ea, eb):
        out = []
        for k in vec_in:
            T = CTYPE[prog.in_dtypes[k]]
            out.append(f"            v{tag}a{k} = ptk_ldv_pin<{T}, VW>({base}{k} + {ea});")
            out.append(f"            v{tag}b{k} = ptk_ldv_pin<{T}, VW>({base}{k} + {eb});")
        return "\n".join(out)

    pipe_decl = "\n".join(f"  PVec<{CTYPE[prog.in_dtypes[k]]}, VW> vpa{k}, vpb{k}, vna{k}, vnb{k};" for k in vec_in)
    next_row_ptrs = "\n".join(f"            const {CTYPE[prog.in_dtypes[k]]}* z{k} = pi{k} + r2 * rsi{k};" for k in vec_in)
    advance = "\n".join(f"          vpa{k} = vna{k}; vpb{k} = vnb{k};" for k in vec_in)

    pipe = _k3_pipeline()
    if pipe == "regs":
        main_loop = f"""      int cv = cv_lo + lane_in_row;
      // Software pipeline over trips of two vectors: the (pinned) loads of trip t+1 are issued before trip t is computed,
      // and the last trip of a row issues the first trip of this thread's NEXT row, so the memory system always has a
      // trip in flight per thread while the scalar bodies run.
      if (cv + TPR < cv_hi) {{
        if (!primed) {{
{pin_loads('p', 'q', 'cv * VW', '(cv + TPR) * VW')}
        }}
        primed = false;
        for (;;) {{
          const int nx = cv + 2 * TPR;
          const bool more = nx + TPR < cv_hi;
          const long long r2 = r + (long long)gridDim.x * {rows_per_block};
          if (more) {{
{pin_loads('n', 'q', 'nx * VW', '(nx + TPR) * VW')}
          }} else if (r2 < rows) {{
{next_row_ptrs}
            const int c2 = cv_lo + lane_in_row;
{pin_loads('n', 'z', 'c2 * VW', '(c2 + TPR) * VW')}
            primed = true;
          }}
          const int ca = cv * VW, cb = (cv + TPR) * VW;
          {{
{compute('pa', 'ca')}
{compute('pb', 'cb')}
          }}
          cv = nx;
{advance}
          if (!more) break;
        }}
      }}
"""
    else:
        if pipe == "l2":
            # ask L2 for the trip after this one (and, on a row's last trip, for the first trip of the thread's next row):
            # no registers, one instruction per 128-byte line (lanes 0, 8, 16, 24 of a warp cover its 512 contiguous bytes)
            pf_lines = []
            for k in vec_in:
                pf_lines.append(f"          ptk_prefetch_l2(pfq{k} + pfa); ptk_prefetch_l2(pfq{k} + pfb);")
            pf_ptr = "\n".join(f"          const {CTYPE[prog.in_dtypes[k]]}* pfq{k} = more ? q{k} : pi{k} + r2 * rsi{k};" for k in vec_in)
            prefetch = f"""        if ((threadIdx.x & 7) == 0) {{{{
          const int nx = cv + 2 * TPR;
          const bool more = nx + TPR < cv_hi;
          const long long r2 = r + (long long)gridDim.x * {rows_per_block};
          if (more || r2 < rows) {{{{
            const int pfa = (more ? nx : cv_lo + lane_in_row) * VW, pfb = pfa + TPR * VW;
{pf_ptr}
{chr(10).join(pf_lines)}
          }}}}
        }}}}"""
            pf_note = "; the NEXT trip's lines are requested from L2 first (prefetch.global.L2)"
        else:
            prefetch, pf_note = "", ""
    use_ptr = pipe not in ("regs", "l2") and _k3_running_pointers()
    if use_ptr:
        def loads_p(tag, off):
            return "\n".join(f"          const PVec<{CTYPE[prog.in_dtypes[k]]}, VW> v{tag}{k} = ptk_ldv<{CTYPE[prog.in_dtypes[k]]}, VW>(a{k}{off});"
                             for k in vec_in)

        def compute_p(tag, off):
            return "\n".join(_compute_ptr(tag, off))

        def _compute_ptr(tag, off):
            call_in = [f"v{tag}{k}.v[e]" if col_modes[k] == 1 else f"s{k}" for k in range(n_in)]
            call_out = [f"o{tag}{k}.v[e]" for k in range(n_map)]
            for k, d in enumerate(prog.out_dtypes):
                yield f"          PVec<{CTYPE[d]}, VW> o{tag}{k};"
            yield "          #pragma unroll"
            yield "          for (int e = 0; e < VW; ++e) {"
            yield f"            ptk_body({', '.join(call_in + call_out)});"
            yield f"            acc = ptk_red(acc, (ACC)o{tag}0.v[e]);"
            yield "          }"
            for k in stored:
                yield f"          ptk_stv<{CTYPE[prog.out_dtypes[k]]}, VW>(u{k}{off}, o{tag}{k});"

        ptr_decl = "\n".join([f"      const {CTYPE[prog.in_dtypes[k]]}* a{k} = q{k} + cv * VW;" for k in vec_in]
                             + [f"      {CTYPE[prog.out_dtypes[k]]}* u{k} = w{k} + cv * VW;" for k in stored])

        def advance_p(n):
            return " ".join([f"a{k} += {n} * TPR * VW;" for k in vec_in] + [f"u{k} += {n} * TPR * VW;" for k in stored])

        main_loop = f"""      int cv = cv_lo + lane_in_row;
{ptr_decl}
      // two vectors per trip, running pointers: the second vector sits at a compile-time distance from the first
      for (; cv + TPR < cv_hi; cv += 2 * TPR) {{
        {{
{loads_p('a', '')}
{loads_p('b', ' + TPR * VW')}
{compute_p('a', '')}
{compute_p('b', ' + TPR * VW')}
        }}
        {advance_p(2)}
      }}
      for (; cv < cv_hi; cv += TPR) {{
        {{
{loads_p('a', '')}
{compute_p('a', '')}
        }}
        {advance_p(1)}
      }}
"""
    elif pipe != "regs":
        main_loop = f"""      int cv = cv_lo + lane_in_row;
      // two vectors per trip{pf_note}
      for (; cv + TPR < cv_hi; cv += 2 * TPR) {{
        const int ca = cv * VW, cb = (cv + TPR) * VW;
{prefetch}
        {{
{loads('a', 'ca')}
{loads('b', 'cb')}
{compute('a', 'ca')}
{compute('b', 'cb')}
        }}
      }}
"""

    tail_in = [f"q{k}[c]" if col_modes[k] == 1 else f"s{k}" for k in range(n_in)]
    tail_tmp = "\n".join(f"          {CTYPE[d]} to{k};" for k, d in enumerate(prog.out_dtypes))
    tail_st = "\n".join(f"          w{k}[c] = to{k};" for k in stored)
    single_loop = "" if use_ptr else f"""
      for (; cv < cv_hi; cv += TPR) {{
        const int ca = cv * VW;
        {{
{loads('a', 'ca')}
{compute('a', 'ca')}
        }}
      }}"""

    return f"""{PRELUDE}
{_VEC_HELPERS}
{_RED_HELPERS}
{emit_body(prog)}
typedef {ACC} ACC;
typedef {OUT} OUT;
{_combine(red_op, acc_dtype)}
#define VW {vw}
#define TPR {tpr}

extern "C" __global__ void __launch_bounds__(256, {_k3_min_blocks()}) {name}({', '.join(params)}) {{
  const int lane_in_row = threadIdx.x & (TPR - 1);
  const int row_in_block = threadIdx.x / TPR;
  const int ncv = (int)(cols / VW);                      // vector chunks per row (VW is a power of two: a shift)
  int cv_lo = 0, cv_hi = ncv;
  if (nsplit > 1) {{
    const int per_split = (ncv + nsplit - 1) / nsplit;
    cv_lo = (int)blockIdx.y * per_split;
    cv_hi = (cv_lo + per_split < ncv) ? (cv_lo + per_split) : ncv;
  }}
  const bool last_split = (int)blockIdx.y == nsplit - 1;
{pipe_decl}
  bool primed = false;   // vpa* / vpb* already hold the first trip of the row this thread starts next
  for (long long rb = (long long)blockIdx.x * {rows_per_block}; rb < rows; rb += (long long)gridDim.x * {rows_per_block}) {{
    const long long r = rb + row_in_block;
    ACC acc = (ACC){literal(acc_dtype, identity)};
    if (r < rows) {{
{base_in}
{base_out}
{row_scalars}
{main_loop}{single_loop}
      if (last_split) {{
        for (int c = ncv * VW + lane_in_row; c < (int)cols; c += TPR) {{
{tail_tmp}
          ptk_body({', '.join(tail_in + [f'to{k}' for k in range(n_map)])});
          acc = ptk_red(acc, (ACC)to0);
{tail_st}
        }}
      }}
    }}
{_block_reduce_code(tpr)}
    if (lane_in_row == 0 && r < rows) {{
      if (nsplit == 1) reinterpret_cast<OUT*>(pred)[r] = (OUT)acc;
      else reinterpret_cast<ACC*>(pred)[r * nsplit + split_of_block()] = acc;
    }}
  }}
}}
""".replace("split_of_block()", "(int)blockIdx.y")


# ---- K3 with TMA staging: a producer thread streams the rows through shared memory with bulk async copies ------------------
_TMA_HELPERS = r"""
// mbarrier + bulk-copy (TMA 1-D) wrappers used by the staged row kernel
__device__ __forceinline__ unsigned ptk_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ptk_mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ptk_smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void ptk_mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void ptk_mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ptk_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ptk_mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(ptk_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void ptk_mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(ptk_smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
// global -> shared bulk copy (bytes and both addresses multiples of 16) completing on `bar`
__device__ __forceinline__ void ptk_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(ptk_smem_u32(dst)), "l"(src), "r"(bytes), "r"(ptk_smem_u32(bar)) : "memory");
}
"""

TMA_STAGES = 4
STATIC_SMEM_LIMIT = 48 * 1024   # statically declared __shared__ bytes a kernel may use


def tma_smem_bytes(n_vec: int) -> int:
    """Shared memory of gen_row_kernel_tma with `n_vec` streamed inputs: a ring of TMA_STAGES trips of 256 16-byte vectors
    per input, plus the full / empty mbarriers."""
    return n_vec * TMA_STAGES * 256 * 16 + 2 * TMA_STAGES * 8


def _k3_tma_min_blocks() -> int:
    import os

    return int(os.environ.get("PTK_K3_MINB", "6"))   # 6 CTAs/SM: 42 registers, 6 x 34 KB of staging buffers


def gen_row_kernel_tma(prog: ScalarProgram, name: str, col_modes: tuple, store_map: tuple, red_op: str, acc_dtype: str,
                       out_dtype: str, identity, vw: int, tpr: int, inplace: dict | None = None) -> str:
    """gen_row_kernel with the north star's "TMA staging into shared memory": thread 0 of the CTA issues one bulk
    asynchronous copy (cp.async.bulk, completion counted on an mbarrier) per input row chunk, TMA_STAGES trips ahead of the
    consumers; all 256 threads then read their 16-byte vector of every input from shared memory, release the stage
    (one mbarrier arrival per warp) and run the scalar bodies.  No load instruction, no address arithmetic and no register
    is spent on the prefetch, so occupancy stays that of the plain kernel while the memory system always has
    TMA_STAGES - 1 trips in flight per CTA.  Same parameters / launch geometry as gen_row_kernel; requires every
    vector-mode input to have 16-byte vectors (vw * itemsize == 16) and the ring to fit the static shared memory
    (tma_smem_bytes: at most two such inputs) — the launcher uses gen_row_kernel otherwise."""
    from .scalar import ITEMSIZE

    n_in, n_map = len(prog.in_dtypes), len(prog.out_dtypes)
    ACC, OUT = CTYPE[acc_dtype], CTYPE[out_dtype]
    restrict = "" if inplace else " __restrict__"
    params = [f"const {CTYPE[d]}*{restrict} pi{k}" for k, d in enumerate(prog.in_dtypes)]
    stored = [k for k in range(n_map) if store_map[k]]
    params += [f"{CTYPE[prog.out_dtypes[k]]}*{restrict} po{k}" for k in stored]
    params += ["void* __restrict__ pred"]
    params += [f"long long rsi{k}" for k in range(n_in)]
    params += [f"long long rso{k}" for k in stored]
    params += ["long long rows", "long long cols", "int nsplit"]
    rpb = 256 // tpr
    vec_in = [k for k in range(n_in) if col_modes[k] == 1]
    for k in vec_in:
        assert vw * ITEMSIZE[prog.in_dtypes[k]] == 16, "TMA staging moves 16-byte vectors"
    smem_decl = "\n".join(f"  __shared__ __align__(128) {CTYPE[prog.in_dtypes[k]]} s_in{k}[STG][{rpb}][TPR * VW];" for k in vec_in)
    issue_rows = "\n".join(
        f"          ptk_bulk_g2s(&s_in{k}[p_stage][rr][0], pi{k} + rp * rsi{k} + (long long)cvb * VW, nbytes, &s_full[p_stage]);"
        for k in vec_in)
    base_in = "\n".join(f"      const {CTYPE[d]}* q{k} = pi{k} + r * rsi{k};" for k, d in enumerate(prog.in_dtypes))
    base_out = "\n".join(f"      {CTYPE[prog.out_dtypes[k]]}* w{k} = po{k} + r * rso{k};" for k in stored)
    row_scalars = "\n".join(f"      const {CTYPE[d]} s{k} = q{k}[0];" for k, d in enumerate(prog.in_dtypes) if col_modes[k] != 1)
    ld_smem = "\n".join(f"        if (mine) va{k} = *reinterpret_cast<const PVec<{CTYPE[prog.in_dtypes[k]]}, VW>*>(&s_in{k}[c_stage][row_in_block][lane_in_row * VW]);"
                        for k in vec_in)
    vdecl = "\n".join(f"        PVec<{CTYPE[prog.in_dtypes[k]]}, VW> va{k};" for k in vec_in)
    call_in = [f"va{k}.v[e]" if col_modes[k] == 1 else f"s{k}" for k in range(n_in)]
    odecl = "\n".join(f"          PVec<{CTYPE[d]}, VW> oa{k};" for k, d in enumerate(prog.out_dtypes))
    call_out = [f"oa{k}.v[e]" for k in range(n_map)]
    st_ = "\n".join(f"          ptk_stv<{CTYPE[prog.out_dtypes[k]]}, VW>(w{k} + ca, oa{k});" for k in stored)
    tail_in = [f"q{k}[c]" if col_modes[k] == 1 else f"s{k}" for k in range(n_in)]
    tail_tmp = "\n".join(f"          {CTYPE[d]} to{k};" for k, d in enumerate(prog.out_dtypes))
    tail_st = "\n".join(f"          w{k}[c] = to{k};" for k in stored)
    n_vec = len(vec_in)
    return f"""{PRELUDE}
{_VEC_HELPERS}
{_RED_HELPERS}
{_TMA_HELPERS}
{emit_body(prog)}
typedef {ACC} ACC;
typedef {OUT} OUT;
{_combine(red_op, acc_dtype)}
#define VW {vw}
#define TPR {tpr}
#define STG {TMA_STAGES}

extern "C" __global__ void __launch_bounds__(256, {_k3_tma_min_blocks()}) {name}({', '.join(params)}) {{
{smem_decl}
  __shared__ unsigned long long s_full[STG], s_empty[STG];
  const int lane_in_row = threadIdx.x & (TPR - 1);
  const int row_in_block = threadIdx.x / TPR;
  const int ncv = (int)(cols / VW);
  int cv_lo = 0, cv_hi = ncv;
  if (nsplit > 1) {{
    const int per_split = (ncv + nsplit - 1) / nsplit;
    cv_lo = (int)blockIdx.y * per_split;
    cv_hi = (cv_lo + per_split < ncv) ? (cv_lo + per_split) : ncv;
  }}
  const bool last_split = (int)blockIdx.y == nsplit - 1;
  const int trips = (cv_hi > cv_lo) ? (cv_hi - cv_lo + TPR - 1) / TPR : 0;   // per row block (one division per CTA)
  if (threadIdx.x == 0) {{
    for (int s = 0; s < STG; ++s) {{ ptk_mbar_init(&s_full[s], 1); ptk_mbar_init(&s_empty[s], 8); }}
    ptk_mbar_fence_init();
  }}
  __syncthreads();
  // producer cursor (thread 0 only): next (row block, trip) to request and the ring slot it goes to
  long long p_rb = (long long)blockIdx.x * {rpb};
  int p_t = 0, p_stage = 0;
  unsigned p_par = 1;          // parity to wait for on s_empty: a fresh barrier's previous phase counts as complete
  auto issue = [&]() {{
    if (trips == 0 || p_rb >= rows) return;
    ptk_mbar_wait(&s_empty[p_stage], p_par);
    const int cvb = cv_lo + p_t * TPR;
    const int nvec = (cv_hi - cvb < TPR) ? (cv_hi - cvb) : TPR;
    const unsigned nbytes = (unsigned)nvec * 16u;
    int nrows = 0;
    for (int rr = 0; rr < {rpb}; ++rr) nrows += (p_rb + rr < rows) ? 1 : 0;
    ptk_mbar_expect_tx(&s_full[p_stage], nbytes * (unsigned)nrows * {n_vec}u);
    for (int rr = 0; rr < {rpb}; ++rr) {{
      const long long rp = p_rb + rr;
      if (rp < rows) {{
{issue_rows}
      }}
    }}
    if (++p_stage == STG) {{ p_stage = 0; p_par ^= 1u; }}
    if (++p_t == trips) {{ p_t = 0; p_rb += (long long)gridDim.x * {rpb}; }}
  }};
  if (threadIdx.x == 0) {{
    for (int s = 0; s < STG - 1; ++s) issue();
  }}
  int c_stage = 0;
  unsigned c_par = 0;
  for (long long rb = (long long)blockIdx.x * {rpb}; rb < rows; rb += (long long)gridDim.x * {rpb}) {{
    const long long r = rb + row_in_block;
    const bool row_ok = r < rows;
    ACC acc = (ACC){literal(acc_dtype, identity)};
    {{
      const long long rc = row_ok ? r : rb;     // (threads of a missing row idle through the trips: they still hit the barriers)
{base_in.replace(" r * ", " rc * ")}
{base_out.replace(" r * ", " rc * ")}
{row_scalars}
      for (int t = 0; t < trips; ++t) {{
        if (threadIdx.x == 0) issue();           // keeps STG - 1 trips in flight
        const int cv = cv_lo + t * TPR + lane_in_row;
        const bool mine = row_ok && cv < cv_hi;
        ptk_mbar_wait(&s_full[c_stage], c_par);
{vdecl}
{ld_smem}
        __syncwarp();
        if ((threadIdx.x & 31) == 0) ptk_mbar_arrive(&s_empty[c_stage]);   // this warp is done with the slot
        if (++c_stage == STG) {{ c_stage = 0; c_par ^= 1u; }}
        if (mine) {{
          const int ca = cv * VW;
{odecl}
          #pragma unroll
          for (int e = 0; e < VW; ++e) {{
            ptk_body({', '.join(call_in + call_out)});
            acc = ptk_red(acc, (ACC)oa0.v[e]);
          }}
{st_}
        }}
      }}
      if (row_ok && last_split) {{
        for (int c = ncv * VW + lane_in_row; c < (int)cols; c += TPR) {{
{tail_tmp}
          ptk_body({', '.join(tail_in + [f'to{k}' for k in range(n_map)])});
          acc = ptk_red(acc, (ACC)to0);
{tail_st}
        }}
      }}
    }}
{_block_reduce_code(tpr)}
    if (lane_in_row == 0 && row_ok) {{
      if (nsplit == 1) reinterpret_cast<OUT*>(pred)[r] = (OUT)acc;
      else reinterpret_cast<ACC*>(pred)[r * nsplit + (int)blockIdx.y] = acc;
    }}
  }}
}}
"""


def gen_finish_kernel(name: str, red_op: str, acc_dtype: str, out_dtype: str, identity) -> str:
    """out[o] = (OUT) reduce_s partial[o*nsplit + s]; one warp per output."""
    ACC, OUT = CTYPE[acc_dtype], CTYPE[out_dtype]
    return f"""{PRELUDE}
{_RED_HELPERS}
typedef {ACC} ACC;
typedef {OUT} OUT;
{_combine(red_op, acc_dtype)}
extern "C" __global__ void __launch_bounds__(256) {name}(const ACC* __restrict__ part, OUT* __restrict__ out,
                                                         long long n_out, int nsplit, long long part_stride_o,
                                                         long long part_stride_s) {{
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long o = warp; o < n_out; o += nwarps) {{
    ACC acc = (ACC){literal(acc_dtype, identity)};
    for (int s = lane; s < nsplit; s += 32) acc = ptk_red(acc, part[o * part_stride_o + s * part_stride_s]);
    #pragma unroll
    for (int m = 16; m > 0; m >>= 1) acc = ptk_red(acc, ptk_shfl_xor<ACC>(acc, m));
    if (lane == 0) out[o] = (OUT)acc;
  }}
}}
"""


def gen_col_kernel(name: str, in_dtype: str, red_op: str, acc_dtype: str, out_dtype: str, identity) -> str:
    """Input (outer, red, inner) contiguous; out (outer, inner) [nsplit == 1] or ACC partials laid out
    [split][outer][inner]. grid = (ceil(inner/256), outer, nsplit)."""
    ACC, OUT, T = CTYPE[acc_dtype], CTYPE[out_dtype], CTYPE[in_dtype]
    return f"""{PRELUDE}
{_RED_HELPERS}
typedef {ACC} ACC;
typedef {OUT} OUT;
{_combine(red_op, acc_dtype)}
extern "C" __global__ void __launch_bounds__(256) {name}(const {T}* __restrict__ in, void* __restrict__ outp,
                                                         long long outer, long long red, long long inner, int nsplit) {{
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= inner) return;
  const long long per = (red + nsplit - 1) / nsplit;
  const long long r_lo = (long long)blockIdx.z * per;
  const long long r_hi = (r_lo + per < red) ? (r_lo + per) : red;
  for (long long o = blockIdx.y; o < outer; o += gridDim.y) {{
    const {T}* p = in + o * red * inner + i;
    ACC a0 = (ACC){literal(acc_dtype, identity)}, a1 = a0, a2 = a0, a3 = a0;
    long long r = r_lo;
    for (; r + 3 < r_hi; r += 4) {{
      const {T} x0 = p[r * inner], x1 = p[(r + 1) * inner], x2 = p[(r + 2) * inner], x3 = p[(r + 3) * inner];
      a0 = ptk_red(a0, (ACC)x0); a1 = ptk_red(a1, (ACC)x1); a2 = ptk_red(a2, (ACC)x2); a3 = ptk_red(a3, (ACC)x3);
    }}
    for (; r < r_hi; ++r) a0 = ptk_red(a0, (ACC)p[r * inner]);
    const ACC acc = ptk_red(ptk_red(a0, a1), ptk_red(a2, a3));
    if (nsplit == 1) reinterpret_cast<OUT*>(outp)[o * inner + i] = (OUT)acc;
    else reinterpret_cast<ACC*>(outp)[((long long)blockIdx.z * outer + o) * inner + i] = acc;
  }}
}}
"""


def gen_generic_kernel(name: str, in_dtype: str, red_op: str, acc_dtype: str, out_dtype: str, identity) -> str:
    """One thread per output element. dims: kept dims (shape, input strides) then reduced dims (shape, strides)."""
    ACC, OUT, T = CTYPE[acc_dtype], CTYPE[out_dtype], CTYPE[in_dtype]
    return f"""{PRELUDE}
{_RED_HELPERS}
typedef {ACC} ACC;
typedef {OUT} OUT;
{_combine(red_op, acc_dtype)}
struct RdDims {{ int nk; int nr; long long kshape[{MAX_DIMS}]; long long kst[{MAX_DIMS}]; long long rshape[{MAX_DIMS}]; long long rst[{MAX_DIMS}]; }};
extern "C" __global__ void __launch_bounds__(256) {name}(const {T}* __restrict__ in, OUT* __restrict__ out,
                                                         const RdDims d, long long n_out, long long n_red) {{
  const long long gstride = (long long)gridDim.x * blockDim.x;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < n_out; o += gstride) {{
    long long rem = o, base = 0;
    for (int k = d.nk - 1; k >= 0; --k) {{ const long long q = rem / d.kshape[k]; base += (rem - q * d.kshape[k]) * d.kst[k]; rem = q; }}
    ACC acc = (ACC){literal(acc_dtype, identity)};
    for (long long j = 0; j < n_red; ++j) {{
      long long rj = j, off = base;
      for (int k = d.nr - 1; k >= 0; --k) {{ const long long q = rj / d.rshape[k]; off += (rj - q * d.rshape[k]) * d.rst[k]; rj = q; }}
      acc = ptk_red(acc, (ACC)in[off]);
    }}
    out[o] = (OUT)acc;
  }}
}}
"""


def identity_program(dtype: str) -> ScalarProgram:
    return single_op_program("Identity", [dtype], dtype)
