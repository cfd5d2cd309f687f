// bf16 tensor-core GEMM for fp32 graphs on sm_90a (H100): warpgroup MMA (wgmma.mma_async m64n128k16, bf16 x bf16 ->
// fp32 accumulators in registers), operands staged by TMA (cp.async.bulk.tensor, SWIZZLE_128B) through a 6-stage
// mbarrier ring.  One CTA per 128 x 128 output tile, three warpgroups: warpgroup 0 = TMA producer (one thread),
// warpgroups 1 and 2 = consumers, each owning 64 rows of the tile: they issue the wgmmas and run the epilogue
// (alpha/beta/bias/tanh -> global) straight from their accumulator registers.
//
// Replaces the sgemm_ call the C linker emits for Dot22 / Gemm (pytensor/tensor/blas/c_code/codegen.py:463-540) on the
// "bf16 tensor core" configuration of BASELINE.json: the graph dtype stays float32 (the reference has no bfloat16 dtype,
// pytensor/tensor/type.py:40-55), operands are rounded to bf16 by a conversion pass into a caller-owned workspace
// (A as [M,K] K-major, B transposed to [N,K] K-major), products accumulate in fp32.
#include <cuda_bf16.h>
#include <stdlib.h>
#include <algorithm>
#include "ptk_common.h"

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_N = 128;
constexpr int BLOCK_K = 64;   // 64 bf16 = 128 bytes = one SWIZZLE_128B row
constexpr int WG_K = 16;      // K of one wgmma
constexpr int STAGES = 6;
constexpr int NUM_THREADS = 384;
constexpr uint32_t A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;  // 16 KiB
constexpr uint32_t B_STAGE_BYTES = BLOCK_N * BLOCK_K * 2;  // 16 KiB
constexpr uint32_t STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(SMEM_BYTES <= 227 * 1024, "H100 allows at most 227 KiB of shared memory per block");

// ---- PTX wrappers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem_dst, int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Ties the accumulator registers to the surrounding asm statements: the compiler may neither read them before the
// wgmma.wait_group that completes them nor move an epilogue write past the wgmma.fence that precedes the next MMA.
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int j = 0; j < N; ++j) asm volatile("" : "+f"(r[j])::"memory");
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}

// D (+)= A[smem desc] * B[smem desc]^T for a 64 x 128 x 16 slice, bf16 x bf16 -> fp32, both operands K-major.
// Accumulator fragment: thread t of the warpgroup holds rows 16 * (t / 32) + (t % 32) / 4 (+ 8) and columns
// 8 * j + 2 * (t % 4) (+ 1): d[4j + 2h + e] = D[row + 8h][8j + 2(t % 4) + e].
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// K-major SWIZZLE_128B shared-memory matrix descriptor (sm_90 wgmma layout):
//  [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (unused for swizzled K-major) |
//  [32,46) stride byte offset >> 4 (8 rows x 128 B = 1024 B between row groups) | [62,64) layout type = 1 (SWIZZLE_128B)
// Stepping K by 16 inside the 128-byte swizzle row advances the start address by 32 bytes (the tile is 1024-aligned).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

struct EpiParams {
  float alpha, beta;
  float* C;
  long long sc0, sc1;
  const float* bias;
  int act;
  int M, N, K;
  __nv_bfloat16* Cbf;  // optional bf16 copy of the result, row-major [M, ldcbf] (the next layer's K-major A operand)
  long long ldcbf;
  int out_pieces;      // 1 = Cbf is a plain bf16 copy; 3 = the three-piece split of the result (piece i at rows
  long long cbf_rows;  // [i * cbf_rows, ...) of Cbf) — the staged A operand of a following fp32-accurate product
  // fp32-accurate mode: every fp32 operand is staged as THREE bf16 pieces x = x1 + x2 + x3 (8 mantissa bits each) stacked
  // along the rows of the staging matrix (piece i of A at rows [i * a_rows, ...)); per k-block the kernel accumulates
  // `terms` piece products into the same fp32 accumulator, smallest first:
  //   terms = 6: A3B1 + A2B2 + A1B3 + A2B1 + A1B2 + A1B1   (drops only O(2^-24) terms: below sgemm's own rounding noise)
  //   terms = 3:                      A2B1 + A1B2 + A1B1   (~4e-6 of the output scale at K = 4096)
  //   terms = 1: plain bf16 operands (the CUDA_BF16 mode)
  int terms;
  int a_rows, b_rows;  // row pitch between the stacked pieces
  // k-blocks per ACCUMULATION CHUNK (0 = the whole K in one chunk).  The tensor core adds into its fp32 accumulator with
  // truncation, a bias that grows linearly with the length of the accumulation chain.  With chunks the register
  // accumulator only ever holds the sum over `kchunk` k-blocks; the epilogue adds every chunk into C in global memory with
  // round-to-nearest fp32 adds (the same thread owns the same elements for all chunks of a tile, so the read-modify-write
  // needs no synchronisation) and applies bias / activation / the bf16 copy after the last chunk.
  int kchunk;
  // fp32-accurate mode with an error-free leading piece (see row_absmax_kernel): the A1 x B1 products go to the main
  // accumulator, the correction products to a second one; the epilogue adds the two (round to nearest).
  int exact_main;
  // staged output pieces (Cbf, out_pieces == 3): leading piece aligned to the fixed exponent out_exp (operands known to lie
  // in [-1, 1]) so that it can feed an exact-main product; PTK_NO_EXP: ordinary bf16 split
  int out_exp;
  float out_scale, out_inv;   // 2^out_exp and 2^-out_exp (exact powers of two: the alignment is two multiplies and a rint)
  // ±inf operands (fp32-accurate modes).  An infinite x is staged as (x, 0, 0), so the piece products that pair it with a
  // zero piece of the other operand are inf * 0 = NaN where sgemm has ±inf.  fa / fb flag the rows of A / columns of B
  // that hold ±inf (kInfBits, the row maximum row_absmax_kernel leaves; null = no flags): a consumer thread owning such an
  // output skips its epilogue, and nonfinite_fixup_kernel recomputes that thread's outputs from the staged pieces As / Bs
  // (pitch lda / ldb, piece pitch a_rows / b_rows).  fc (nullable, zeroed by the caller) receives the same flags for the
  // rows of a three-piece Cbf.
  const unsigned int* fa;
  const unsigned int* fb;
  unsigned int* fc;
  const __nv_bfloat16* As;
  const __nv_bfloat16* Bs;
  long long lda, ldb;
};
#define PTK_NO_EXP (-100000)
constexpr unsigned int kInfBits = 0x7f800000u;
// piece indices of the term sequence; a run of `terms` entries ending at index 5 is used
__device__ __constant__ int kPieceA[6] = {2, 1, 0, 1, 0, 0};
__device__ __constant__ int kPieceB[6] = {0, 1, 2, 0, 1, 0};

// sum over k of A[row, k] * B[k, col], each operand rebuilt exactly from its three staged pieces (p0 + p1 + p2), products
// summed in fp64 and rounded once: the outputs nonfinite_fixup_kernel recomputes.  ±inf / NaN come out as sgemm has them.
__device__ float nonfinite_dot(const __nv_bfloat16* As, long long lda, long long a_rows, const __nv_bfloat16* Bs, long long ldb,
                               long long b_rows, int K, long long row, long long col) {
  const __nv_bfloat16* a = As + row * lda;
  const __nv_bfloat16* b = Bs + col * ldb;
  double s = 0.0;
  for (int k = 0; k < K; ++k) {
    const double x = (double)__bfloat162float(a[k]) + (double)__bfloat162float(a[a_rows * lda + k]) +
                     (double)__bfloat162float(a[2 * a_rows * lda + k]);
    const double y = (double)__bfloat162float(b[k]) + (double)__bfloat162float(b[b_rows * ldb + k]) +
                     (double)__bfloat162float(b[2 * b_rows * ldb + k]);
    s = fma(x, y, s);
  }
  return (float)s;
}

__device__ __forceinline__ bool inf_flagged(const unsigned int* f, long long i) { return f != nullptr && f[i] == kInfBits; }

// One output element pair (row, col), (row, col + 1) of a finished chunk: alpha * acc (+ beta * C) (+ bias) (tanh), the
// bf16 / three-piece copy.  The vector and the scalar branch compute the same values.
__device__ __forceinline__ void epi_pair(const EpiParams& p, long long row, long long col, float v0, float v1, float beta,
                                         const float* bias, int act, __nv_bfloat16* cbf) {
  if (row >= p.M || col >= p.N) return;
  const bool two = col + 1 < p.N;
  float* dst = p.C + row * p.sc0 + col * p.sc1;
  const bool vec = two && p.sc1 == 1 && ((((uintptr_t)dst) & 7) == 0);
  float x[2] = {p.alpha * v0, p.alpha * v1};
  if (beta != 0.0f) {
    if (vec) {
      const float2 o = __ldcg(reinterpret_cast<const float2*>(dst));
      x[0] += beta * o.x;
      x[1] += beta * o.y;
    } else {
      x[0] += beta * dst[0];
      if (two) x[1] += beta * dst[p.sc1];
    }
  }
  if (bias) {
    x[0] += bias[col];
    if (two) x[1] += bias[col + 1];
  }
  if (act == 1) {
    x[0] = tanhf(x[0]);
    x[1] = tanhf(x[1]);
  }
  if (vec) {
    *reinterpret_cast<float2*>(dst) = make_float2(x[0], x[1]);
  } else {
    dst[0] = x[0];
    if (two) dst[p.sc1] = x[1];
  }
  if (cbf) {
    const float inf = __int_as_float(kInfBits), bfmax = __int_as_float(0x7f7f0000);   // (bfmax: the largest bf16)
    if (p.fc != nullptr && (fabsf(x[0]) == inf || (two && fabsf(x[1]) == inf))) p.fc[row] = kInfBits;
    for (int pc = 0; pc < p.out_pieces; ++pc) {   // piece pc = bf16 of what the earlier pieces left over
      __nv_bfloat16 b[2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        b[e] = (pc == 0 && p.out_exp != PTK_NO_EXP) ? __float2bfloat16_rn(rintf(x[e] * p.out_scale) * p.out_inv)
                                                    : __float2bfloat16_rn(fabsf(x[e]) < inf ? fminf(fmaxf(x[e], -bfmax), bfmax) : x[e]);
        x[e] = fabsf(x[e]) < inf ? x[e] - __bfloat162float(b[e]) : 0.0f;   // ±inf / NaN ride in the leading piece alone
      }
      __nv_bfloat16* d = cbf + ((long long)pc * p.cbf_rows + row) * p.ldcbf + col;
      if (two && ((((uintptr_t)d) & 3) == 0)) {
        __nv_bfloat162 pk;
        pk.x = b[0];
        pk.y = b[1];
        *reinterpret_cast<__nv_bfloat162*>(d) = pk;
      } else {
        d[0] = b[0];
        if (two) d[1] = b[1];
      }
    }
  }
}

// Does this consumer thread own an output whose row of A or column of B holds ±inf?  (two rows, 32 columns)
__device__ __forceinline__ bool thread_flagged(const unsigned int* fa, const unsigned int* fb, int M, int N, long long row0,
                                            long long col0) {
  bool any = false;
  for (int h = 0; h < 2; ++h) any |= row0 + 8 * h < M && inf_flagged(fa, row0 + 8 * h);
  for (int j = 0; j < 32; ++j) {
    const long long col = col0 + 8 * (j >> 1) + (j & 1);
    any |= col < N && inf_flagged(fb, col);
  }
  return any;
}

// kExact: compile-time copy of EpiParams::exact_main — the plain instantiation carries no second accumulator.
template <bool kExact>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b, EpiParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smem_a = smem;                              // STAGES x 16 KiB
  uint8_t* smem_b = smem + STAGES * A_STAGE_BYTES;     // STAGES x 16 KiB
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;                    // [STAGES]  TMA bytes landed
  uint64_t* empty_bar = bars + STAGES;          // [STAGES]  8 arrivals: every consumer warp is done reading

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int tm = (int)(blockIdx.x % (unsigned)m_tiles), tn = (int)(blockIdx.x / (unsigned)m_tiles);
  const int k_blocks = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int kchunk = (p.kchunk > 0 && p.kchunk < k_blocks) ? p.kchunk : max(k_blocks, 1);
  const int n_chunks = max(1, (k_blocks + kchunk - 1) / kchunk);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===== TMA producer: one thread streams k-block x piece-product stages in the consumers' order =====
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < k_blocks; ++kb) {
        for (int t = 6 - p.terms; t < 6; ++t) {   // one ring stage per piece product (a single pass when terms == 1)
          const int arow = kPieceA[t] * p.a_rows, brow = kPieceB[t] * p.b_rows;
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          tma_load_2d(&tmap_a, &full_bar[stage], smem_a + stage * A_STAGE_BYTES, kb * BLOCK_K, arow + tm * BLOCK_M);
          tma_load_2d(&tmap_b, &full_bar[stage], smem_b + stage * B_STAGE_BYTES, kb * BLOCK_K, brow + tn * BLOCK_N);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup 1 -> rows [0, 64) of the tile, warpgroup 2 -> rows [64, 128) =====
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  float acc[64];
  float cor[kExact ? 64 : 1];
  int stage = 0;
  uint32_t phase = 0;
  const int terms_m1 = p.terms - 1;
  const long long row0 = (long long)tm * BLOCK_M + cw * 64 + (warp & 3) * 16 + (lane >> 2);
  const long long col0 = (long long)tn * BLOCK_N + (lane & 3) * 2;
  // a thread owning an output whose row of A / column of B holds ±inf leaves all its outputs to nonfinite_fixup_kernel
  const bool flagged = (p.fa != nullptr || p.fb != nullptr) && thread_flagged(p.fa, p.fb, p.M, p.N, row0, col0);
#pragma unroll 1
  for (int ch = 0; ch < n_chunks; ++ch) {
    const int kb_n = min(kchunk, k_blocks - ch * kchunk);
    const int n_stages = kb_n * p.terms;   // piece products of one k-block accumulate into the same tile
    if (n_stages == 0) {                   // K == 0: the product is zero
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.0f;
    }
    int term = 0;                          // position inside the k-block's term sequence
    int prev = -1;                         // stage whose wgmmas may still be reading shared memory
#pragma unroll 1
    for (int it = 0; it < n_stages; ++it) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem_a + stage * A_STAGE_BYTES + cw * (64 * BLOCK_K * 2));
      const uint32_t b_addr = smem_u32(smem_b + stage * B_STAGE_BYTES);
      // term order within a k-block: the correction products first, A1 x B1 last (kPieceA / kPieceB)
      const bool to_corr = kExact && term != terms_m1;
      const bool first = kExact ? (to_corr ? it == 0 : it == terms_m1) : it == 0;
      term = (term == terms_m1) ? 0 : term + 1;
      wg_fence();
      fence_regs(acc);
      if constexpr (kExact) fence_regs(cor);
      if constexpr (kExact) {
        if (to_corr) {
#pragma unroll
          for (int k = 0; k < BLOCK_K / WG_K; ++k)
            wgmma_m64n128k16(cor, make_smem_desc(a_addr + k * WG_K * 2), make_smem_desc(b_addr + k * WG_K * 2),
                             (!first || k > 0) ? 1u : 0u);
        } else {
#pragma unroll
          for (int k = 0; k < BLOCK_K / WG_K; ++k)
            wgmma_m64n128k16(acc, make_smem_desc(a_addr + k * WG_K * 2), make_smem_desc(b_addr + k * WG_K * 2),
                             (!first || k > 0) ? 1u : 0u);
        }
      } else {
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k)
          wgmma_m64n128k16(acc, make_smem_desc(a_addr + k * WG_K * 2), make_smem_desc(b_addr + k * WG_K * 2),
                           (!first || k > 0) ? 1u : 0u);
      }
      wg_commit();
      wg_wait<1>();   // the previous stage's wgmmas are complete: its shared memory may be refilled
      if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wg_wait<0>();
    fence_regs(acc);
    if constexpr (kExact) fence_regs(cor);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    if constexpr (kExact) {
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] += cor[j];
    }
    // chunk 0 combines with the caller's C (beta), later chunks add onto the partial sum this thread stored before;
    // bias / activation / the bf16 copy belong to the completed sum
    const float beta = ch == 0 ? p.beta : 1.0f;
    const bool last = ch == n_chunks - 1;
    const float* bias = last ? p.bias : nullptr;
    const int act = last ? p.act : 0;
    __nv_bfloat16* cbf = last ? p.Cbf : nullptr;
    if (flagged) continue;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        epi_pair(p, row0 + 8 * h, col0 + 8 * j, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], beta, bias, act, cbf);
    }
  }
}

// The outputs the GEMM kernel left alone (thread_flagged): one block per output tile, thread t standing for consumer thread
// t of the GEMM (same fragment mapping), the GEMM's own epilogue over dot products from nonfinite_dot.  C still holds the
// caller's values there, so beta, bias, tanh and the staged output pieces come out as for any other output.  A tile without
// a flagged row or column costs one flag load per thread.
__global__ void __launch_bounds__(256) nonfinite_fixup_kernel(const EpiParams p) {
  const int m_tiles = (p.M + BLOCK_M - 1) / BLOCK_M;
  const int tm = (int)(blockIdx.x % (unsigned)m_tiles), tn = (int)(blockIdx.x / (unsigned)m_tiles);
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const long long r = (long long)tm * BLOCK_M + (t & 127), c = (long long)tn * BLOCK_N + (t & 127);
  const bool mine = t < 128 ? (r < p.M && inf_flagged(p.fa, r)) : (c < p.N && inf_flagged(p.fb, c));
  if (!__syncthreads_or(mine)) return;
  const long long row0 = (long long)tm * BLOCK_M + (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
  const long long col0 = (long long)tn * BLOCK_N + (lane & 3) * 2;
  if (!thread_flagged(p.fa, p.fb, p.M, p.N, row0, col0)) return;
  for (int j = 0; j < 16; ++j) {
    for (int h = 0; h < 2; ++h) {
      const long long row = row0 + 8 * h, col = col0 + 8 * j;
      if (row >= p.M || col >= p.N) continue;
      const float v0 = nonfinite_dot(p.As, p.lda, p.a_rows, p.Bs, p.ldb, p.b_rows, p.K, row, col);
      const float v1 = col + 1 < p.N ? nonfinite_dot(p.As, p.lda, p.a_rows, p.Bs, p.ldb, p.b_rows, p.K, row, col + 1) : 0.0f;
      epi_pair(p, row, col, v0, v1, p.beta, p.bias, p.act, p.Cbf);
    }
  }
}

// ---- fp32 -> bf16 operand staging: dst[r][c] (row-major, pitch ld) = bf16(src[r*sr + c*sc]) ----------------------------
// Tiled through shared memory so that both the read (along whichever source stride is 1) and the write (along c) coalesce.
__global__ void __launch_bounds__(256) convert_bf16_kernel(const float* __restrict__ src, long long sr, long long sc,
                                                           __nv_bfloat16* __restrict__ dst, long long ld, long long R,
                                                           long long Cc) {
  // 64 x 64 tile: reads walk the source's unit-stride direction (128 B per warp), writes are packed bf16x2 along c
  // (128 B per warp-row).  ld is even and dst 4-byte aligned (workspace rows are padded to 8 elements).
  __shared__ float tile[64][65];
  const long long r0 = (long long)blockIdx.y * 64, c0 = (long long)blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const bool col_fast = (sc == 1) || (sr != 1);
  if (col_fast) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + ty + 8 * i, c = c0 + tx + 32 * h;
        tile[ty + 8 * i][tx + 32 * h] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  } else {  // source is row-fast (sr == 1): read with threads along r, transpose through shared memory
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + tx + 32 * h, c = c0 + ty + 8 * i;
        tile[tx + 32 * h][ty + 8 * i] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long r = r0 + ty + 8 * i, c = c0 + 2 * tx;
    if (r < R && c < Cc) {
      const float lo = tile[ty + 8 * i][2 * tx], hi = tile[ty + 8 * i][2 * tx + 1];
      if (c + 1 < Cc || c + 1 < ld) {
        *reinterpret_cast<__nv_bfloat162*>(dst + r * ld + c) = __floats2bfloat162_rn(lo, (c + 1 < Cc) ? hi : 0.0f);
      } else {
        dst[r * ld + c] = __float2bfloat16_rn(lo);
      }
    }
  }
}

// ---- fp32 -> 3 x bf16 operand split: piece i of src[r*sr + c*sc] goes to dst[(i * piece_rows + r) * ld + c] ----------------
// x1 = bf16(x), x2 = bf16(x - x1), x3 = bf16(x - x1 - x2): the residuals are exact in fp32, so x1 + x2 + x3 carries 24
// mantissa bits of x.  Same 64 x 64 shared-memory tile as convert_bf16_kernel (coalesced reads along either source stride).
// A non-finite x is staged as (x, 0, 0); a finite x beyond the largest bf16 (3.3895e38) gets that largest value as its
// leading piece instead of inf, so that its remainder stays finite.
__global__ void __launch_bounds__(256) split_bf16x3_kernel(const float* __restrict__ src, long long sr, long long sc,
                                                           __nv_bfloat16* __restrict__ dst, long long ld, long long R,
                                                           long long Cc, long long piece_rows) {
  __shared__ float tile[64][65];
  const long long r0 = (long long)blockIdx.y * 64, c0 = (long long)blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const bool col_fast = (sc == 1) || (sr != 1);
  if (col_fast) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + ty + 8 * i, c = c0 + tx + 32 * h;
        tile[ty + 8 * i][tx + 32 * h] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + tx + 32 * h, c = c0 + ty + 8 * i;
        tile[tx + 32 * h][ty + 8 * i] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long r = r0 + ty + 8 * i, c = c0 + 2 * tx;
    if (r < R && c < Cc) {
      float lo = tile[ty + 8 * i][2 * tx], hi = (c + 1 < Cc) ? tile[ty + 8 * i][2 * tx + 1] : 0.0f;
      const float inf = __int_as_float(0x7f800000), bfmax = __int_as_float(0x7f7f0000);
#pragma unroll
      for (int pc = 0; pc < 3; ++pc) {
        const __nv_bfloat16 bl = __float2bfloat16_rn(fabsf(lo) < inf ? fminf(fmaxf(lo, -bfmax), bfmax) : lo);
        const __nv_bfloat16 bh = __float2bfloat16_rn(fabsf(hi) < inf ? fminf(fmaxf(hi, -bfmax), bfmax) : hi);
        __nv_bfloat16* d = dst + (pc * piece_rows + r) * ld + c;
        if (c + 1 < ld) {
          __nv_bfloat162 pk;
          pk.x = bl;
          pk.y = bh;
          *reinterpret_cast<__nv_bfloat162*>(d) = pk;
        } else {
          *d = bl;
        }
        lo = fabsf(lo) < inf ? lo - __bfloat162float(bl) : 0.0f;   // ±inf / NaN ride in the leading piece alone
        hi = fabsf(hi) < inf ? hi - __bfloat162float(bh) : 0.0f;
      }
    }
  }
}

// ---- error-free leading piece (fp32-accurate mode, "exact main term") ---------------------------------------------------
// The tensor core truncates when it adds into its fp32 accumulator; over a chain of MMAs that is a systematic shrink of the
// result (~1e-7 per MMA of the chain, measured) which, unlike rounding noise, adds up coherently through chained layers.
// Truncation cannot bite when every partial sum is exactly representable: the LEADING piece of each operand is therefore
// taken as an integer multiple of a per-row power of two, x1 = rint(x * 2^s) * 2^-s with |rint| <= 2^b (s = b - 1 - ilogb of
// the row's largest magnitude; a row of A, a column of B).  All products A1[i,k] * B1[k,j] of one output element are then
// integers (<= 2^2b, b = 7: lead_bits_for) on the common unit 2^-(s_i + s_j), and they sum exactly in fp32 as long as the
// partial sums stay below 2^24 units; the operand carries b + 16 = 23 bits plus sign through its three pieces.  The remainder x - x1 is
// exact in fp32 and is split into two ordinary bf16 pieces; the five correction products go to a second accumulator, whose
// own truncation shrink is 2^-7 of the total.
// Pass 1: largest magnitude of every row, as the bit pattern of a non-negative float (ordered like an unsigned integer):
// 64 x 64 tiles through shared memory exactly like the split kernels (coalesced whichever source stride is 1), four
// threads per tile row, one atomicMax per tile row.  `maxbits` must be zeroed beforehand.  NaN / inf count as "no scale".
__global__ void __launch_bounds__(256) row_absmax_kernel(const float* __restrict__ src, long long sr, long long sc,
                                                         long long R, long long Cc, unsigned int* __restrict__ maxbits) {
  __shared__ float tile[64][65];
  const long long r0 = (long long)blockIdx.y * 64, c0 = (long long)blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const bool col_fast = (sc == 1) || (sr != 1);
  if (col_fast) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + ty + 8 * i, c = c0 + tx + 32 * h;
        tile[ty + 8 * i][tx + 32 * h] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + tx + 32 * h, c = c0 + ty + 8 * i;
        tile[tx + 32 * h][ty + 8 * i] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  }
  __syncthreads();
  const int row = threadIdx.x >> 2, part = threadIdx.x & 3;
  float m = 0.0f;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const float v = fabsf(tile[row][part * 16 + j]);
    m = (v > m) ? v : m;   // NaN never wins; +inf does (and then disables the scale below)
  }
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
  if (part == 0 && r0 + row < R && m > 0.0f) atomicMax(maxbits + r0 + row, __float_as_uint(m));
}

// per-row scale exponent from the row maximum: (lead_bits - 1) - ilogb(max), so that |x| * 2^s < 2^lead_bits; 0 for empty /
// non-finite rows
__device__ __forceinline__ int scale_exp_of(unsigned int bits, int lead_bits) {
  const float m = __uint_as_float(bits);
  return (m > 0.0f && m < __int_as_float(0x7f800000)) ? (lead_bits - 1) - ilogbf(m) : 0;
}

// piece 0 = rint(x * 2^s[r]) * 2^-s[r] (exact in bf16), pieces 1, 2 = bf16 split of the exact remainder; same tiling and
// output layout as split_bf16x3_kernel.  fixed_exp != INT_MIN: use that exponent for every row (operands known to lie in
// [-1, 1], e.g. tanh outputs written by a previous product's epilogue) instead of sexp.
__global__ void __launch_bounds__(256) split_aligned_kernel(const float* __restrict__ src, long long sr, long long sc,
                                                            __nv_bfloat16* __restrict__ dst, long long ld, long long R,
                                                            long long Cc, long long piece_rows,
                                                            const unsigned int* __restrict__ maxbits, int lead_bits) {
  __shared__ float tile[64][65];
  const long long r0 = (long long)blockIdx.y * 64, c0 = (long long)blockIdx.x * 64;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  const bool col_fast = (sc == 1) || (sr != 1);
  if (col_fast) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + ty + 8 * i, c = c0 + tx + 32 * h;
        tile[ty + 8 * i][tx + 32 * h] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long r = r0 + tx + 32 * h, c = c0 + ty + 8 * i;
        tile[tx + 32 * h][ty + 8 * i] = (r < R && c < Cc) ? src[r * sr + c * sc] : 0.0f;
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const long long r = r0 + ty + 8 * i, c = c0 + 2 * tx;
    if (r < R && c < Cc) {
      int sx = scale_exp_of(maxbits[r], lead_bits);
      sx = sx > 126 ? 126 : (sx < -126 ? -126 : sx);   // 2^sx and 2^-sx must be normal floats (rows of denormal size lose bits)
      const float up = __int_as_float((127 + sx) << 23), dn = __int_as_float((127 - sx) << 23);
      float v[2] = {tile[ty + 8 * i][2 * tx], (c + 1 < Cc) ? tile[ty + 8 * i][2 * tx + 1] : 0.0f};
      __nv_bfloat16 pc[3][2];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float q = rintf(v[e] * up);   // |q| <= 2^lead_bits: exact in bf16; x - lead exact in fp32
        float lead = q * dn;
        if (fabsf(lead) == __int_as_float(0x7f800000) && fabsf(v[e]) < __int_as_float(0x7f800000))
          lead = (q - copysignf(1.0f, q)) * dn;   // the top binade: 2^lead_bits * 2^-sx = 2^128 overflows
        pc[0][e] = __float2bfloat16_rn(lead);
        float rem = v[e] - lead;
        if (!(fabsf(v[e]) < __int_as_float(0x7f800000))) rem = 0.0f;  // inf / NaN ride in the leading piece only
        pc[1][e] = __float2bfloat16_rn(rem);
        rem -= __bfloat162float(pc[1][e]);
        pc[2][e] = __float2bfloat16_rn(rem);
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        __nv_bfloat16* d = dst + (k * piece_rows + r) * ld + c;
        if (c + 1 < ld) {
          __nv_bfloat162 pk;
          pk.x = pc[k][0];
          pk.y = pc[k][1];
          *reinterpret_cast<__nv_bfloat162*>(d) = pk;
        } else {
          *d = pc[k][0];
        }
      }
    }
  }
}

ptk_status make_tmap(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems, uint32_t box_rows) {
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = ptk::drv().TensorMapEncodeTiled(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr,
                                               box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return ptk::check_cu(r, "cuTensorMapEncodeTiled");
}

inline long long round_up(long long x, long long m) { return (x + m - 1) / m * m; }

// One CTA per 128 x 128 tile of C; A and B^T are bf16 K-major matrices behind the two tensor maps.
ptk_status launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const EpiParams& p, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    PTK_CUDA(cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    PTK_CUDA(cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    attr_set = true;
  }
  const long long tiles = (long long)((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + BLOCK_N - 1) / BLOCK_N);
  if (tiles > 2147483647LL) return ptk::fail(PTK_ERR_ARG, "gemm_tc: too many output tiles");
  if (p.exact_main) gemm_bf16_wgmma_kernel<true><<<(unsigned)tiles, NUM_THREADS, SMEM_BYTES, st>>>(ta, tb, p);
  else gemm_bf16_wgmma_kernel<false><<<(unsigned)tiles, NUM_THREADS, SMEM_BYTES, st>>>(ta, tb, p);
  PTK_LAUNCH_CHECK("gemm_bf16_wgmma");
  if (p.fa != nullptr || p.fb != nullptr) {
    nonfinite_fixup_kernel<<<(unsigned)tiles, 256, 0, st>>>(p);
    PTK_LAUNCH_CHECK("nonfinite_fixup");
  }
  return PTK_OK;
}

}  // namespace

namespace ptk {

size_t gemm_tc_workspace(int64_t M, int64_t N, int64_t K) {
  long long Kp = round_up(K, 8);
  return (size_t)(round_up(M * Kp * 2, 256) + round_up(N * Kp * 2, 256) + 256);
}

size_t gemm_tc_split_workspace(int64_t M, int64_t N, int64_t K) {
  long long Kp = round_up(K, 8), Mp = round_up(M, 256), Np = round_up(N, 256);
  return (size_t)(round_up(3 * Mp * Kp * 2, 256) + round_up(3 * Np * Kp * 2, 256) + round_up(4 * (M + N), 256) + 256);
}

// error-free leading pieces on/off for the fp32-accurate mode (PTK_GEMM_EXACT=0: plain bf16x3 split, one accumulator)
// Leading-piece width: |rint(x * 2^s)| <= 2^7.  Products are then integers <= 2^14 and every partial sum below 2^24 units is
// exact: always for K <= 1024, and for longer contractions unless more than a thousand near-maximal products line up in
// sign — past 2^24 the accumulator merely drops its lowest one or two unit bits (a 2^-24-level effect, no worse than the
// plain split, and only on such data).  Measured alternative (width shrinking with K so that exactness is unconditional:
// 6 bits at K = 4096, 5 at 8192): max error 2.5e-6 / 9.3e-6 of the output scale instead of 6e-7 — the operand then only
// carries b + 16 bits — so the width stays 7 and the accumulation is cut into chunks only beyond K = 16384.
static int lead_bits_for(int64_t K) {
  (void)K;
  return 7;
}

static int exact_main_default() {
  static int g = -1;
  if (g < 0) {
    const char* e = getenv("PTK_GEMM_EXACT");
    g = (e && e[0] == '0') ? 0 : 1;
  }
  return g;
}

// accumulation chunk of the fp32-accurate modes: 8 k-blocks (K = 512) keeps the tensor core's truncation bias near 1e-6 of
// the output scale; PTK_GEMM_KCHUNK=<k-blocks> overrides (0 = one chunk)
static int split_kchunk(int64_t K, int exact) {
  static int g_kchunk = -1;
  if (g_kchunk < 0) {
    const char* e = getenv("PTK_GEMM_KCHUNK");
    g_kchunk = e ? atoi(e) : -1;
  }
  const long long kb = (K + BLOCK_K - 1) / BLOCK_K;
  if (exact) {
    const long long cap = 256;   // k-blocks (K = 16384) per accumulation, see lead_bits_for
    const long long c = g_kchunk > 0 ? std::min<long long>(g_kchunk, cap) : cap;
    return kb > c ? (int)c : 0;
  }
  const int c = g_kchunk >= 0 ? g_kchunk : 8;
  return (c > 0 && kb > c + c / 4) ? c : 0;
}

// Operand staging on its own (so that an operand that does not change between calls is staged ONCE): dst = `pieces` (1 | 3)
// bf16 matrices [R, Cc] stacked with a pitch of piece_rows rows, row pitch ld elements, from fp32 src[r*sr + c*sc].
// sexp (R words, required when aligned): the row maxima (row_absmax_kernel), which are +inf for a row holding ±inf — the
// flags of EpiParams::fa / fb, kept for the plain split too.
ptk_status stage_operand(const float* src, int64_t sr, int64_t sc, int64_t R, int64_t Cc, int pieces, void* dst, int64_t ld,
                         int64_t piece_rows, int aligned, int* sexp, cudaStream_t st) {
  if (pieces != 1 && pieces != 3) return fail(PTK_ERR_ARG, "stage_operand: pieces must be 1 or 3");
  if (aligned && (pieces != 3 || sexp == nullptr)) return fail(PTK_ERR_ARG, "stage_operand: aligned staging needs 3 pieces and the exponent scratch");
  if (ld % 8 != 0 || ld < Cc || ((uintptr_t)dst & 15) != 0) return fail(PTK_ERR_ARG, "stage_operand: pitch must be a multiple of 8 >= cols, base 16-byte aligned");
  if (R == 0 || Cc == 0) return PTK_OK;
  dim3 g((unsigned)((Cc + 63) / 64), (unsigned)((R + 63) / 64));
  unsigned int* flags = reinterpret_cast<unsigned int*>(sexp);
  if (pieces == 3 && flags != nullptr) {
    PTK_CUDA(cudaMemsetAsync(flags, 0, (size_t)R * 4, st));
    row_absmax_kernel<<<g, 256, 0, st>>>(src, sr, sc, R, Cc, flags);
  }
  if (pieces == 1) {
    convert_bf16_kernel<<<g, 256, 0, st>>>(src, sr, sc, (__nv_bfloat16*)dst, ld, R, Cc);
  } else if (aligned) {
    split_aligned_kernel<<<g, 256, 0, st>>>(src, sr, sc, (__nv_bfloat16*)dst, ld, R, Cc, piece_rows, flags, lead_bits_for(Cc));
  } else {
    split_bf16x3_kernel<<<g, 256, 0, st>>>(src, sr, sc, (__nv_bfloat16*)dst, ld, R, Cc, piece_rows);
  }
  PTK_LAUNCH_CHECK("stage_operand");
  return PTK_OK;
}

// The tensor-core kernel over operands that are ALREADY staged (see stage_operand): A_stage = pieces of A [M,K] (K-major,
// pitch lda, piece pitch a_rows rows), B_stage = pieces of B^T [N,K]; terms 1 (plain bf16) | 3 | 6.  C_stage (optional)
// receives `out_pieces` (1 | 3) staged pieces of the RESULT [M,N] (pitch ldc_stage, piece pitch c_rows) — the A operand
// of the next product of a chain / recurrence, so that only the very first operand is ever staged by a separate pass.
// The only code that builds the kernel's tensor maps and EpiParams: gemm_tc_ex / gemm_tc_split stage and come here.
ptk_status gemm_tc_staged(int64_t M, int64_t N, int64_t K, float alpha, const void* A_stage, int64_t lda, int64_t a_rows,
                          const void* B_stage, int64_t ldb, int64_t b_rows, int terms, float beta, float* C, int64_t sc0,
                          int64_t sc1, const float* bias, int act, void* C_stage, int64_t ldc_stage, int64_t c_rows,
                          int out_pieces, int exact_main, int out_exp, const unsigned int* a_flags,
                          const unsigned int* b_flags, unsigned int* c_flags, cudaStream_t st) {
  if (M == 0 || N == 0) return PTK_OK;
  if (terms != 1 && terms != 3 && terms != 6) return fail(PTK_ERR_ARG, "gemm_tc_staged: terms must be 1, 3 or 6");
  // Three stacked pieces put row coordinates up to 2 * a_rows + M into the tensor map: M, N <= 5e8 keep them in int32.
  // The one-piece product accepts what ptk_gemm_tc_ex always has: M, N up to int32 and a C_stage at any pitch (the
  // epilogue checks the alignment of every store).
  const bool one = terms == 1;
  const long long max_mn = one ? 2147483647LL : 500000000LL;
  if (M > max_mn || N > max_mn || K > 2147483647LL || K <= 0) return fail(PTK_ERR_ARG, "gemm_tc_staged: bad dims");
  if (lda % 8 || ldb % 8 || ((uintptr_t)A_stage & 15) || ((uintptr_t)B_stage & 15))
    return fail(PTK_ERR_ARG, "gemm_tc_staged: operand pitch must be a multiple of 8 elements, base 16-byte aligned");
  if (C_stage != nullptr && (out_pieces != 1 && out_pieces != 3)) return fail(PTK_ERR_ARG, "gemm_tc_staged: out_pieces must be 1 or 3");
  if (C_stage != nullptr && !one && (ldc_stage % 8 || ((uintptr_t)C_stage & 15)))
    return fail(PTK_ERR_ARG, "gemm_tc_staged: misaligned C_stage");
  const int pa = one ? 1 : 3;
  CUtensorMap ta, tb;
  ptk_status s;
  // rows past M (N) inside a piece hold whatever the staging buffer held: they only reach output rows (columns) the
  // epilogue masks, never a stored element; columns past K and rows past the last piece are zero-filled by TMA
  const uint64_t a_total = (uint64_t)((pa - 1) * a_rows + M), b_total = (uint64_t)((pa - 1) * b_rows + N);
  if ((s = make_tmap(&ta, A_stage, a_total, (uint64_t)K, (uint64_t)lda, BLOCK_M)) != PTK_OK) return s;
  if ((s = make_tmap(&tb, B_stage, b_total, (uint64_t)K, (uint64_t)ldb, BLOCK_N)) != PTK_OK) return s;
  EpiParams p;
  p.alpha = alpha; p.beta = beta; p.C = C; p.sc0 = sc0; p.sc1 = sc1; p.bias = bias; p.act = act;
  p.M = (int)M; p.N = (int)N; p.K = (int)K;
  p.Cbf = reinterpret_cast<__nv_bfloat16*>(C_stage);
  p.ldcbf = ldc_stage;
  p.out_pieces = C_stage ? out_pieces : 1;
  p.cbf_rows = c_rows;
  p.terms = terms; p.a_rows = one ? 0 : (int)a_rows; p.b_rows = one ? 0 : (int)b_rows;
  p.exact_main = (!one && exact_main) ? 1 : 0;
  p.out_exp = (C_stage && out_pieces == 3) ? out_exp : PTK_NO_EXP;
  p.out_scale = 1.0f; p.out_inv = 1.0f;
  if (p.out_exp != PTK_NO_EXP) {
    if (p.out_exp < -100 || p.out_exp > 100) return fail(PTK_ERR_ARG, "gemm_tc_staged: out_exp out of range");
    p.out_scale = ldexpf(1.0f, p.out_exp);
    p.out_inv = ldexpf(1.0f, -p.out_exp);
  }
  p.kchunk = one ? 0 : split_kchunk(K, p.exact_main);
  p.fa = one ? nullptr : a_flags; p.fb = one ? nullptr : b_flags;   // (flags only mean something for three-piece operands)
  p.fc = (C_stage && out_pieces == 3) ? c_flags : nullptr;
  p.As = reinterpret_cast<const __nv_bfloat16*>(A_stage); p.Bs = reinterpret_cast<const __nv_bfloat16*>(B_stage);
  p.lda = lda; p.ldb = ldb;
  return launch_gemm(ta, tb, p, st);
}

// bf16 product with fp32 operands: A (unless given as A_bf16: row-major, pitch lda_bf16 elements, multiple of 8, 16-byte
// aligned base) and B^T are staged as one bf16 piece each in the workspace, then multiplied by gemm_tc_staged.
ptk_status gemm_tc_ex(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t sa0, int64_t sa1,
                      const void* A_bf16, int64_t lda_bf16, const float* B, int64_t sb0, int64_t sb1, float beta, float* C,
                      int64_t sc0, int64_t sc1, const float* bias, int act, void* C_bf16, int64_t ldc_bf16, void* workspace,
                      size_t workspace_bytes, cudaStream_t st) {
  if (M == 0 || N == 0) return PTK_OK;
  if (M > 2147483647LL || N > 2147483647LL || K > 2147483647LL) return fail(PTK_ERR_ARG, "gemm_tc: dims exceed int32");
  if (workspace == nullptr || workspace_bytes < gemm_tc_workspace(M, N, K))
    return fail(PTK_ERR_ARG, "gemm_tc: workspace too small (see ptk_gemm_workspace_bytes)");
  const long long Kp = round_up(K, 8);
  uintptr_t w = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
  void* Bbf = reinterpret_cast<void*>(w + round_up(M * Kp * 2, 256));
  ptk_status s;
  if (A_bf16 == nullptr) {
    void* Abf = reinterpret_cast<void*>(w);
    if ((s = stage_operand(A, sa0, sa1, M, K, 1, Abf, Kp, 0, 0, nullptr, st)) != PTK_OK) return s;
    A_bf16 = Abf;
    lda_bf16 = Kp;
  }
  if ((s = stage_operand(B, sb1, sb0, N, K, 1, Bbf, Kp, 0, 0, nullptr, st)) != PTK_OK) return s;   // B[K,N] -> Bt[N,K]
  return gemm_tc_staged(M, N, K, alpha, A_bf16, lda_bf16, 0, Bbf, Kp, 0, 1, beta, C, sc0, sc1, bias, act, C_bf16, ldc_bf16, 0,
                        1, 0, PTK_NO_EXP, nullptr, nullptr, nullptr, st);
}

// fp32-accurate product on the tensor cores: both operands split into three bf16 pieces in the workspace (the per-row
// words behind them: sexp for A, sexp + M for B^T), then `terms` (3 or 6) piece products per k-block by gemm_tc_staged
// (see EpiParams::terms).
ptk_status gemm_tc_split(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t sa0, int64_t sa1, const float* B,
                         int64_t sb0, int64_t sb1, float beta, float* C, int64_t sc0, int64_t sc1, const float* bias, int act,
                         int terms, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (M == 0 || N == 0) return PTK_OK;
  if (terms != 3 && terms != 6) return fail(PTK_ERR_ARG, "gemm_tc_split: terms must be 3 or 6");
  if (M > 500000000LL || N > 500000000LL || K > 2147483647LL) return fail(PTK_ERR_ARG, "gemm_tc_split: dims exceed int32");
  if (workspace == nullptr || workspace_bytes < gemm_tc_split_workspace(M, N, K))
    return fail(PTK_ERR_ARG, "gemm_tc_split: workspace too small (see ptk_gemm_split_workspace_bytes)");
  const long long Kp = round_up(K, 8), Mp = round_up(M, 256), Np = round_up(N, 256);
  uintptr_t w = ((uintptr_t)workspace + 255) & ~(uintptr_t)255;
  void* Abf = reinterpret_cast<void*>(w);
  void* Bbf = reinterpret_cast<void*>(w + round_up(3 * Mp * Kp * 2, 256));
  int* sexp = reinterpret_cast<int*>(w + round_up(3 * Mp * Kp * 2, 256) + round_up(3 * Np * Kp * 2, 256));
  const int exact = terms == 6 ? exact_main_default() : 0;   // (3 terms need the 8-bit leading pieces of the plain split)
  ptk_status s;
  if ((s = stage_operand(A, sa0, sa1, M, K, 3, Abf, Kp, Mp, exact, sexp, st)) != PTK_OK) return s;
  if ((s = stage_operand(B, sb1, sb0, N, K, 3, Bbf, Kp, Np, exact, sexp + M, st)) != PTK_OK) return s;   // B[K,N] -> Bt[N,K]
  const unsigned int* flags = reinterpret_cast<const unsigned int*>(sexp);
  return gemm_tc_staged(M, N, K, alpha, Abf, Kp, Mp, Bbf, Kp, Np, terms, beta, C, sc0, sc1, bias, act, nullptr, 0, 0, 1, exact,
                        PTK_NO_EXP, flags, flags + M, nullptr, st);
}

}  // namespace ptk

extern "C" ptk_status ptk_gemm_tc_ex(int64_t M, int64_t N, int64_t K, double alpha, const void* A_f32, int64_t sa0,
                                     int64_t sa1, const void* A_bf16, int64_t lda_bf16, const void* B_f32, int64_t sb0,
                                     int64_t sb1, double beta, void* C, int64_t sc0, int64_t sc1, const void* bias, int act,
                                     void* C_bf16, int64_t ldc_bf16, void* workspace, size_t workspace_bytes, void* stream) {
  PTK_REQUIRE_INIT();
  if (A_f32 == nullptr && A_bf16 == nullptr) return ptk::fail(PTK_ERR_ARG, "ptk_gemm_tc_ex: no A operand");
  return ptk::gemm_tc_ex(M, N, K, (float)alpha, (const float*)A_f32, sa0, sa1, A_bf16, lda_bf16, (const float*)B_f32, sb0, sb1,
                         (float)beta, (float*)C, sc0, sc1, (const float*)bias, act, C_bf16, ldc_bf16, workspace,
                         workspace_bytes, (cudaStream_t)stream);
}

extern "C" size_t ptk_gemm_split_workspace_bytes(int64_t M, int64_t N, int64_t K) { return ptk::gemm_tc_split_workspace(M, N, K); }

extern "C" ptk_status ptk_gemm_tc_split(int64_t M, int64_t N, int64_t K, double alpha, const void* A_f32, int64_t sa0,
                                        int64_t sa1, const void* B_f32, int64_t sb0, int64_t sb1, double beta, void* C,
                                        int64_t sc0, int64_t sc1, const void* bias, int act, int terms, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  PTK_REQUIRE_INIT();
  if (A_f32 == nullptr || B_f32 == nullptr) return ptk::fail(PTK_ERR_ARG, "ptk_gemm_tc_split: null operand");
  return ptk::gemm_tc_split(M, N, K, (float)alpha, (const float*)A_f32, sa0, sa1, (const float*)B_f32, sb0, sb1, (float)beta,
                            (float*)C, sc0, sc1, (const float*)bias, act, terms, workspace, workspace_bytes,
                            (cudaStream_t)stream);
}

extern "C" size_t ptk_stage_bytes(int64_t rows, int64_t cols, int pieces) {
  const long long ld = (cols + 7) / 8 * 8, pr = (rows + 255) / 256 * 256;
  const size_t mats = (size_t)(pieces <= 1 ? rows : 3 * pr) * (size_t)ld * 2;
  return (mats + 255) / 256 * 256 + (pieces <= 1 ? 0 : (size_t)rows * 4) + 256;   // + the per-row exponents of an aligned split
}

extern "C" ptk_status ptk_stage_operand(const void* src_f32, int64_t sr, int64_t sc, int64_t rows, int64_t cols, int pieces,
                                        int aligned, void* dst, int64_t ld, int64_t piece_rows, void* stream) {
  PTK_REQUIRE_INIT();
  if (src_f32 == nullptr || dst == nullptr) return ptk::fail(PTK_ERR_ARG, "ptk_stage_operand: null pointer");
  int* sexp = nullptr;
  const bool default_pitch = ld == (cols + 7) / 8 * 8 && piece_rows == (rows + 255) / 256 * 256;
  if (aligned && (pieces != 3 || !default_pitch))
    return ptk::fail(PTK_ERR_ARG, "ptk_stage_operand: aligned staging uses the default pitch / piece pitch of ptk_stage_bytes");
  if (pieces == 3 && default_pitch) {   // the row words behind the pieces: row maxima / ±inf row flags
    const size_t mats = (size_t)(3 * piece_rows) * (size_t)ld * 2;
    sexp = reinterpret_cast<int*>((char*)dst + (mats + 255) / 256 * 256);
  }
  return ptk::stage_operand((const float*)src_f32, sr, sc, rows, cols, pieces, dst, ld, piece_rows, aligned, sexp,
                            (cudaStream_t)stream);
}

extern "C" ptk_status ptk_gemm_tc_staged(int64_t M, int64_t N, int64_t K, double alpha, const void* A_stage, int64_t lda,
                                         int64_t a_rows, const void* B_stage, int64_t ldb, int64_t b_rows, int terms,
                                         double beta, void* C, int64_t sc0, int64_t sc1, const void* bias, int act,
                                         void* C_stage, int64_t ldc_stage, int64_t c_rows, int out_pieces, int exact_main,
                                         int out_exp, const void* a_flags, const void* b_flags, void* c_flags,
                                         void* stream) {
  PTK_REQUIRE_INIT();
  if (A_stage == nullptr || B_stage == nullptr || C == nullptr) return ptk::fail(PTK_ERR_ARG, "ptk_gemm_tc_staged: null operand");
  return ptk::gemm_tc_staged(M, N, K, (float)alpha, A_stage, lda, a_rows, B_stage, ldb, b_rows, terms, (float)beta, (float*)C,
                             sc0, sc1, (const float*)bias, act, C_stage, ldc_stage, c_rows, out_pieces, exact_main,
                             out_exp == PTK_STAGE_NO_EXP ? PTK_NO_EXP : out_exp, (const unsigned int*)a_flags,
                             (const unsigned int*)b_flags, (unsigned int*)c_flags, (cudaStream_t)stream);
}

extern "C" int ptk_gemm_exact_main_default(void) { return ptk::exact_main_default(); }

extern "C" int ptk_gemm_lead_bits(int64_t K) { return ptk::lead_bits_for(K); }
