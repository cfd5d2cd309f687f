// Native-precision BLAS family (fp32 / fp64 FMA pipes): GEMM with arbitrary element strides, GEMV, GER.
// These are the "<= 1e-5 vs the C linker" paths behind Gemm / Dot22 / Dot22Scalar / Gemv / Ger
// (pytensor/tensor/blas/gemm.py:76,248,298, gemv.py:16, ger.py:8); the bf16 tensor-core path is ptk_gemm_tc.cu.
#include <algorithm>
#include <cstdlib>
#include "ptk_common.h"

namespace ptk {
ptk_status gemm_tc_ex(int64_t M, int64_t N, int64_t K, float alpha, const float* A, int64_t sa0, int64_t sa1,
                      const void* A_bf16, int64_t lda_bf16, const float* B, int64_t sb0, int64_t sb1, float beta, float* C,
                      int64_t sc0, int64_t sc1, const float* bias, int act, void* C_bf16, int64_t ldc_bf16, void* workspace,
                      size_t workspace_bytes, cudaStream_t st);
size_t gemm_tc_workspace(int64_t M, int64_t N, int64_t K);
}  // namespace ptk

namespace {

constexpr int BM = 64, BN = 64, BK = 16, TM = 4, TN = 4;

template <typename T>
__device__ __forceinline__ T act_apply(T v, int act) {
  if (act == 1) return tanh(v);
  return v;
}
template <>
__device__ __forceinline__ float act_apply<float>(float v, int act) {
  if (act == 1) return tanhf(v);
  return v;
}

// C = alpha * A @ B + beta * C (+ bias[n], act). A_KFAST: A's K stride is 1; B_NFAST: B's N stride is 1 — only the
// thread->element mapping of the global loads changes so that a warp always walks the unit-stride direction.  The m-tiles
// are walked grid-stride along y (gridDim.y is capped at 65535, so products with more than 65535 * 64 rows loop).
template <typename T, bool A_KFAST, bool B_NFAST>
__global__ void __launch_bounds__(256) gemm_simt_kernel(int64_t M, int64_t N, int64_t K, T alpha,
                                                        const T* __restrict__ A, int64_t sa0, int64_t sa1,
                                                        const T* __restrict__ B, int64_t sb0, int64_t sb1, T beta,
                                                        T* __restrict__ C, int64_t sc0, int64_t sc1,
                                                        const T* __restrict__ bias, int act) {
  __shared__ T As[BK][BM + 4];
  __shared__ T Bs[BK][BN + 4];
  const int t = threadIdx.x;
  const int tx = t % 16, ty = t / 16;
  const int64_t n0 = (int64_t)blockIdx.x * BN;
  for (int64_t m0 = (int64_t)blockIdx.y * BM; m0 < M; m0 += (int64_t)gridDim.y * BM) {  // uniform per block
    T acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = T(0);

    for (int64_t k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int m, k;
        if (A_KFAST) { k = t % BK; m = t / BK + 16 * i; }
        else         { m = t % BM; k = t / BM + 4 * i; }
        int64_t gm = m0 + m, gk = k0 + k;
        As[k][m] = (gm < M && gk < K) ? A[gm * sa0 + gk * sa1] : T(0);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        int n, k;
        if (B_NFAST) { n = t % BN; k = t / BN + 4 * i; }
        else         { k = t % BK; n = t / BK + 16 * i; }
        int64_t gn = n0 + n, gk = k0 + k;
        Bs[k][n] = (gn < N && gk < K) ? B[gk * sb0 + gn * sb1] : T(0);
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < BK; ++k) {
        T a[TM], b[TN];
#pragma unroll
        for (int i = 0; i < TM; ++i) a[i] = As[k][ty * TM + i];
#pragma unroll
        for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
        for (int i = 0; i < TM; ++i)
#pragma unroll
          for (int j = 0; j < TN; ++j) acc[i][j] += a[i] * b[j];
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      int64_t gm = m0 + ty * TM + i;
      if (gm >= M) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        int64_t gn = n0 + tx * TN + j;
        if (gn >= N) continue;
        T* p = C + gm * sc0 + gn * sc1;
        T v = alpha * acc[i][j];
        if (beta != T(0)) v += beta * (*p);  // beta == 0 must not read C (it may hold NaNs from AllocEmpty)
        if (bias) v += bias[gn];
        *p = act_apply<T>(v, act);
      }
    }
  }
}

// ---- skinny shapes (PyMC-style regressions: (B x K)(K x n) with K ~ 8 and (B x n)(n x K)): HBM-bound on the big operand --------
constexpr int SK_MAXK = 16;
// K <= KMAX (4 / 8 / 16), C unit-stride along N.  A CTA owns 256 output columns; every thread keeps its K x 4 slab of B in
// registers.  Rows are processed in tiles of 64: the tile's 64 x K block of A is staged in shared memory with ONE coalesced
// global load per thread (latency paid once per 64 rows, hidden by the other resident CTAs), then each thread produces
// 16 rows x 4 columns from broadcast LDS + FMAs and writes them with 128-bit stores.  Bound by the write of C.
template <typename T, int KMAX>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 ? 3 : 2)) gemm_smallk_kernel(
    int64_t M, int64_t N, int K, T alpha, const T* __restrict__ A, int64_t sa0, int64_t sa1, const T* __restrict__ B,
    int64_t sb0, int64_t sb1, T beta, T* __restrict__ C, int64_t sc0) {
  constexpr int TR = 64;
  __shared__ T As[TR][KMAX + 1];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;  // 64 column-threads x 4 row-threads
  const int64_t n0 = ((int64_t)blockIdx.x * 64 + tx) * 4;
  T b[KMAX][4];
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) b[k][j] = (k < K && n0 + j < N) ? B[k * sb0 + (n0 + j) * sb1] : T(0);
  const bool col_ok = n0 < N;
  for (int64_t m0 = (int64_t)blockIdx.y * TR; m0 < M; m0 += (int64_t)gridDim.y * TR) {
    __syncthreads();
    for (int e = threadIdx.x; e < TR * KMAX; e += blockDim.x) {
      const int r = e / KMAX, k = e - r * KMAX;
      As[r][k] = (m0 + r < M && k < K) ? A[(m0 + r) * sa0 + k * sa1] : T(0);
    }
    __syncthreads();
    if (!col_ok) continue;
#pragma unroll 4
    for (int rr = 0; rr < TR / 4; ++rr) {
      const int r = rr * 4 + ty;
      const int64_t m = m0 + r;
      if (m >= M) break;
      T acc[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll
      for (int k = 0; k < KMAX; ++k) {
        const T a = As[r][k];
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] += a * b[k][j];
      }
      T* c = C + m * sc0 + n0;
      if (n0 + 3 < N && ((((uintptr_t)c) & (4 * sizeof(T) - 1)) == 0)) {
        struct __align__(4 * sizeof(T)) V4 { T v[4]; } out;
        if (beta != T(0)) {  // Gemm accumulating into Z: vector read-modify-write, never touched when beta == 0
          const V4 old = *reinterpret_cast<const V4*>(c);
#pragma unroll
          for (int j = 0; j < 4; ++j) out.v[j] = alpha * acc[j] + beta * old.v[j];
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) out.v[j] = alpha * acc[j];
        }
        *reinterpret_cast<V4*>(c) = out;  // one 128-bit (fp32) / 256-bit (fp64) access: full 32-byte sectors
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (n0 + j < N) {
            T v = alpha * acc[j];
            if (beta != T(0)) v += beta * c[j];
            c[j] = v;
          }
        }
      }
    }
  }
}

// v2 of the small-K kernel (selected with PTK_BLAS_V2=1 until measured on the device): identical arithmetic, but the
// read-modify-write of C is software-pipelined.  In v1 every row's `old = C[m, n0..n0+3]` load sits behind the previous row's
// store to the same array, which the compiler must keep in order, so each thread has ONE 16-byte load in flight and the
// kernel is latency-bound (ncu: 31 % of DRAM peak at 36 % warps active).  Here the loads of G = 4 rows are issued together,
// before any of the group's stores.
template <typename T, int KMAX>
__global__ void __launch_bounds__(256, (sizeof(T) == 4 ? 2 : 1)) gemm_smallk_v2_kernel(
    int64_t M, int64_t N, int K, T alpha, const T* __restrict__ A, int64_t sa0, int64_t sa1, const T* __restrict__ B,
    int64_t sb0, int64_t sb1, T beta, T* __restrict__ C, int64_t sc0) {
  constexpr int TR = 64, G = 4;
  struct __align__(4 * sizeof(T)) V4 { T v[4]; };
  __shared__ T As[TR][KMAX + 1];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;  // 64 column-threads x 4 row-threads
  const int64_t n0 = ((int64_t)blockIdx.x * 64 + tx) * 4;
  T b[KMAX][4];
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) b[k][j] = (k < K && n0 + j < N) ? B[k * sb0 + (n0 + j) * sb1] : T(0);
  const bool col_ok = n0 < N;
  const bool full4 = n0 + 3 < N;
  for (int64_t m0 = (int64_t)blockIdx.y * TR; m0 < M; m0 += (int64_t)gridDim.y * TR) {
    __syncthreads();
    for (int e = threadIdx.x; e < TR * KMAX; e += blockDim.x) {
      const int r = e / KMAX, k = e - r * KMAX;
      As[r][k] = (m0 + r < M && k < K) ? A[(m0 + r) * sa0 + k * sa1] : T(0);
    }
    __syncthreads();
    if (!col_ok) continue;
    for (int rr0 = 0; rr0 < TR / 4; rr0 += G) {
      V4 old[G];
      bool vec[G];
      // phase 1: all of the group's reads of C (independent loads, nothing of this group has been stored yet)
#pragma unroll
      for (int u = 0; u < G; ++u) {
        const int64_t m = m0 + (rr0 + u) * 4 + ty;
        T* c = C + m * sc0 + n0;
        vec[u] = m < M && full4 && ((((uintptr_t)c) & (4 * sizeof(T) - 1)) == 0);
        if (vec[u] && beta != T(0)) old[u] = *reinterpret_cast<const V4*>(c);
      }
      // phase 2: products, epilogue, stores
#pragma unroll
      for (int u = 0; u < G; ++u) {
        const int r = (rr0 + u) * 4 + ty;
        const int64_t m = m0 + r;
        if (m >= M) continue;
        T acc[4] = {T(0), T(0), T(0), T(0)};
#pragma unroll
        for (int k = 0; k < KMAX; ++k) {
          const T a = As[r][k];
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[j] += a * b[k][j];
        }
        T* c = C + m * sc0 + n0;
        if (vec[u]) {
          V4 out;
          if (beta != T(0)) {
#pragma unroll
            for (int j = 0; j < 4; ++j) out.v[j] = alpha * acc[j] + beta * old[u].v[j];
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) out.v[j] = alpha * acc[j];
          }
          *reinterpret_cast<V4*>(c) = out;
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (n0 + j < N) {
              T v = alpha * acc[j];
              if (beta != T(0)) v += beta * c[j];
              c[j] = v;
            }
          }
        }
      }
    }
  }
}

constexpr int SN_MAXN = 16;
// N <= 16, A unit-stride along K: one warp per row of A; each lane streams 16-byte vectors of the row (4 in flight) and
// multiplies them with B, which is staged TRANSPOSED in shared memory ONCE per CTA and K-chunk (Bs[n][k], k contiguous ->
// conflict-free LDS.128).  The CTA's warps then walk all their rows without further synchronisation.
template <typename T, int N>
__global__ void __launch_bounds__(256) gemm_smalln_kernel(int64_t M, int n_act, int64_t K, int kchunk, T alpha,
                                                          const T* __restrict__ A, int64_t sa0, const T* __restrict__ B,
                                                          int64_t sb0, int64_t sb1, T beta, T* __restrict__ C, int64_t sc0,
                                                          int64_t sc1) {
  constexpr int V = 16 / sizeof(T);  // elements per 16-byte vector
  extern __shared__ __align__(16) unsigned char sn_smem[];
  T* Bs = reinterpret_cast<T*>(sn_smem);  // [N][kchunk + V]
  const int ldb = kchunk + V;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t warps_total = (int64_t)gridDim.x * 8;
  const int64_t gw = (int64_t)blockIdx.x * 8 + warp;
  const bool vec_ok = (sa0 % V == 0) && ((((uintptr_t)A) & 15) == 0) && (kchunk % (32 * V) == 0);
  for (int64_t k0 = 0; k0 < K; k0 += kchunk) {
    const int kc = (int)min((int64_t)kchunk, K - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < N * kchunk; e += blockDim.x) {
      const int n = e / kchunk, k = e - n * kchunk;
      Bs[n * ldb + k] = (k < kc && n < n_act) ? B[(k0 + k) * sb0 + n * sb1] : T(0);
    }
    __syncthreads();
    const bool first = k0 == 0;
    for (int64_t m = gw; m < M; m += warps_total) {
      T acc[N];
#pragma unroll
      for (int n = 0; n < N; ++n) acc[n] = T(0);
      const T* arow = A + m * sa0 + k0;
      if (vec_ok && ((k0 % V) == 0)) {
        // kc is padded with zeros in Bs up to kchunk, but A must not be read past K: guard the vector index
        for (int kb = 0; kb < kchunk; kb += 32 * V * 4) {
          T a[4][V];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int kk = kb + (u * 32 + lane) * V;
            if (kk + V <= kc) *reinterpret_cast<uint4*>(a[u]) = *reinterpret_cast<const uint4*>(arow + kk);
            else {
#pragma unroll
              for (int e = 0; e < V; ++e) a[u][e] = (kk + e < kc) ? arow[kk + e] : T(0);
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int kk = kb + (u * 32 + lane) * V;
            if (kk < kchunk) {
#pragma unroll
              for (int n = 0; n < N; ++n) {
                T bv[V];
                *reinterpret_cast<uint4*>(bv) = *reinterpret_cast<const uint4*>(&Bs[n * ldb + kk]);
#pragma unroll
                for (int e = 0; e < V; ++e) acc[n] += a[u][e] * bv[e];
              }
            }
          }
        }
      } else {
        for (int k = lane; k < kc; k += 32) {
          const T av = arow[k];
#pragma unroll
          for (int n = 0; n < N; ++n) acc[n] += av * Bs[n * ldb + k];
        }
      }
#pragma unroll
      for (int n = 0; n < N; ++n) {
        T v = acc[n];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == 0 && n < n_act) {
          T* c = C + m * sc0 + n * sc1;
          T out = alpha * v;
          if (first) { if (beta != T(0)) out += beta * (*c); }
          else out += *c;
          *c = out;
        }
      }
    }
  }
}

// PTK_BLAS_V2=1 selects the restructured skinny-GEMM kernels below (validated on the host emulator, tests/; to be timed on
// the device before they become the default).
static bool blas_v2() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("PTK_BLAS_V2");
    v = (e && e[0] == '1') ? 1 : 0;
  }
  return v == 1;
}

// v2 of the small-N kernel (PTK_BLAS_V2=1): one warp owns R rows at a time.  v1 re-reads the N vectors of B from shared
// memory for every row (8 x 16 B of LDS per 16 B of A: ~16 TB/s of shared-memory traffic at 2 TB/s of HBM — the
// shared-memory pipe, not DRAM, is what saturates); with R rows per warp each LDS.128 of B feeds R rows' FMAs, and the
// R x U row vectors are independent global loads in flight.
template <typename T, int N, int R>
__global__ void __launch_bounds__(256) gemm_smalln_v2_kernel(int64_t M, int n_act, int64_t K, int kchunk, T alpha,
                                                             const T* __restrict__ A, int64_t sa0, const T* __restrict__ B,
                                                             int64_t sb0, int64_t sb1, T beta, T* __restrict__ C,
                                                             int64_t sc0, int64_t sc1) {
  constexpr int V = 16 / sizeof(T);  // elements per 16-byte vector
  constexpr int U = 2;               // vectors per lane and row in flight
  extern __shared__ __align__(16) unsigned char sn_smem[];
  T* Bs = reinterpret_cast<T*>(sn_smem);  // [N][kchunk + V]
  const int ldb = kchunk + V;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t warps_total = (int64_t)gridDim.x * 8;
  const int64_t gw = (int64_t)blockIdx.x * 8 + warp;
  const bool vec_ok = (sa0 % V == 0) && ((((uintptr_t)A) & 15) == 0) && (kchunk % (32 * V * U) == 0);
  for (int64_t k0 = 0; k0 < K; k0 += kchunk) {
    const int kc = (int)min((int64_t)kchunk, K - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < N * kchunk; e += blockDim.x) {
      const int n = e / kchunk, k = e - n * kchunk;
      Bs[n * ldb + k] = (k < kc && n < n_act) ? B[(k0 + k) * sb0 + n * sb1] : T(0);
    }
    __syncthreads();
    const bool first = k0 == 0;
    for (int64_t mb = gw * R; mb < M; mb += warps_total * R) {
      T acc[R][N];
#pragma unroll
      for (int r = 0; r < R; ++r)
#pragma unroll
        for (int n = 0; n < N; ++n) acc[r][n] = T(0);
      const T* arow[R];
#pragma unroll
      for (int r = 0; r < R; ++r) arow[r] = A + min(mb + r, M - 1) * sa0 + k0;  // rows past M alias the last row (not stored)
      if (vec_ok && ((k0 % V) == 0)) {
        for (int kb = 0; kb < kchunk; kb += 32 * V * U) {
          T a[R][U][V];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int kk = kb + (u * 32 + lane) * V;
#pragma unroll
            for (int r = 0; r < R; ++r) {
              if (kk + V <= kc) *reinterpret_cast<uint4*>(a[r][u]) = *reinterpret_cast<const uint4*>(arow[r] + kk);
              else {
#pragma unroll
                for (int e = 0; e < V; ++e) a[r][u][e] = (kk + e < kc) ? arow[r][kk + e] : T(0);
              }
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int kk = kb + (u * 32 + lane) * V;
#pragma unroll
            for (int n = 0; n < N; ++n) {
              T bv[V];
              *reinterpret_cast<uint4*>(bv) = *reinterpret_cast<const uint4*>(&Bs[n * ldb + kk]);
#pragma unroll
              for (int r = 0; r < R; ++r)
#pragma unroll
                for (int e = 0; e < V; ++e) acc[r][n] += a[r][u][e] * bv[e];
            }
          }
        }
      } else {
        for (int k = lane; k < kc; k += 32) {
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const T av = arow[r][k];
#pragma unroll
            for (int n = 0; n < N; ++n) acc[r][n] += av * Bs[n * ldb + k];
          }
        }
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
#pragma unroll
        for (int n = 0; n < N; ++n) {
          T v = acc[r][n];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0 && n < n_act && mb + r < M) {
            T* c = C + (mb + r) * sc0 + n * sc1;
            T out = alpha * v;
            if (first) { if (beta != T(0)) out += beta * (*c); }
            else out += *c;
            *c = out;
          }
        }
      }
    }
  }
}

template <typename T, int N>
ptk_status launch_smalln(int64_t M, int n_act, int64_t K, T alpha, const T* A, int64_t sa0, const T* B, int64_t sb0,
                         int64_t sb1, T beta, T* C, int64_t sc0, int64_t sc1, unsigned grid, cudaStream_t st) {
  constexpr int V = 16 / sizeof(T);
  const int unit = 32 * V * 4;  // one unrolled sweep of a warp
  int64_t kchunk = (K + unit - 1) / unit * unit;
  const int64_t max_elems = (96 * 1024) / ((int64_t)sizeof(T) * N) - V;
  if (kchunk > max_elems) kchunk = std::max<int64_t>(unit, max_elems / unit * unit);
  const size_t smem = (size_t)N * (kchunk + V) * sizeof(T);
  static bool attr_done = false;
  (void)attr_done;
  cudaError_t e = cudaFuncSetAttribute(gemm_smalln_kernel<T, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
  if (e != cudaSuccess) return ptk::check_cuda(e, "cudaFuncSetAttribute(gemm_smalln)");
  if (blas_v2()) {
    constexpr int R = (N <= 8) ? 4 : 2;  // R x N accumulators per lane
    e = cudaFuncSetAttribute(gemm_smalln_v2_kernel<T, N, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024);
    if (e != cudaSuccess) return ptk::check_cuda(e, "cudaFuncSetAttribute(gemm_smalln_v2)");
    const unsigned g2 = (unsigned)std::max<int64_t>(1, std::min<int64_t>((M + 8 * R - 1) / (8 * R), grid));
    gemm_smalln_v2_kernel<T, N, R><<<g2, 256, smem, st>>>(M, n_act, K, (int)kchunk, alpha, A, sa0, B, sb0, sb1, beta, C, sc0, sc1);
    return PTK_OK;
  }
  gemm_smalln_kernel<T, N><<<grid, 256, smem, st>>>(M, n_act, K, (int)kchunk, alpha, A, sa0, B, sb0, sb1, beta, C, sc0, sc1);
  return PTK_OK;
}

template <typename T>
ptk_status launch_gemm(int64_t M, int64_t N, int64_t K, double alpha, const void* A, int64_t sa0, int64_t sa1,
                       const void* B, int64_t sb0, int64_t sb1, double beta, void* C, int64_t sc0, int64_t sc1,
                       const void* bias, int act, cudaStream_t st) {
  if (M == 0 || N == 0) return PTK_OK;
  const int sms = std::max(1, ptk::sm_count());
  if (bias == nullptr && act == 0 && K >= 1 && K <= SK_MAXK && sc1 == 1 && M >= 256 && N >= 64) {
    unsigned gx = (unsigned)((N + 255) / 256);
    unsigned gy = (unsigned)std::min<int64_t>((M + 63) / 64, std::max<int64_t>(1, (int64_t)sms * 12 / gx));
#define PTK_SK(KM) gemm_smallk_kernel<T, KM><<<dim3(gx, gy), 256, 0, st>>>(M, N, (int)K, (T)alpha, (const T*)A, sa0, sa1, \
                                                                      (const T*)B, sb0, sb1, (T)beta, (T*)C, sc0)
#define PTK_SK2(KM) gemm_smallk_v2_kernel<T, KM><<<dim3(gx, gy), 256, 0, st>>>(M, N, (int)K, (T)alpha, (const T*)A, sa0, sa1, \
                                                                          (const T*)B, sb0, sb1, (T)beta, (T*)C, sc0)
    if (blas_v2()) {
      if (K <= 4) PTK_SK2(4);
      else if (K <= 8) PTK_SK2(8);
      else PTK_SK2(16);
    } else if (K <= 4) PTK_SK(4);
    else if (K <= 8) PTK_SK(8);
    else PTK_SK(16);
#undef PTK_SK2
#undef PTK_SK
    PTK_LAUNCH_CHECK("gemm_smallk");
    return PTK_OK;
  }
  if (bias == nullptr && act == 0 && N <= SN_MAXN && sa1 == 1 && M >= 256 && K >= 64) {
    unsigned gx = (unsigned)std::min<int64_t>((M + 7) / 8, (int64_t)sms * 4);
#define PTK_SN(NN) launch_smalln<T, NN>(M, (int)N, K, (T)alpha, (const T*)A, sa0, (const T*)B, sb0, sb1, (T)beta, (T*)C, sc0, sc1, gx, st)
    ptk_status sn;
    if (N <= 1) sn = PTK_SN(1);
    else if (N <= 2) sn = PTK_SN(2);
    else if (N <= 4) sn = PTK_SN(4);
    else if (N <= 8) sn = PTK_SN(8);
    else sn = PTK_SN(16);
#undef PTK_SN
    if (sn != PTK_OK) return sn;
    PTK_LAUNCH_CHECK("gemm_smalln");
    return PTK_OK;
  }
  dim3 grid((unsigned)((N + BN - 1) / BN), (unsigned)std::min<int64_t>((M + BM - 1) / BM, 65535));
  bool akf = (sa1 == 1) || K == 1, bnf = (sb1 == 1) || N == 1;
  if (sa0 == 1 && sa1 != 1) akf = false;
  if (sb0 == 1 && sb1 != 1) bnf = false;
#define PTK_G(AK, BNF)                                                                                       \
  gemm_simt_kernel<T, AK, BNF><<<grid, 256, 0, st>>>(M, N, K, (T)alpha, (const T*)A, sa0, sa1, (const T*)B, \
                                                      sb0, sb1, (T)beta, (T*)C, sc0, sc1, (const T*)bias, act)
  if (akf && bnf) PTK_G(true, true);
  else if (akf && !bnf) PTK_G(true, false);
  else if (!akf && bnf) PTK_G(false, true);
  else PTK_G(false, false);
#undef PTK_G
  PTK_LAUNCH_CHECK("gemm_simt");
  return PTK_OK;
}

// ---- GEMV ----------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) scale_vec_kernel(T* y, int64_t sy, int64_t M, T beta) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < M) y[i * sy] = (beta == T(0)) ? T(0) : beta * y[i * sy];
}

// One warp per (row, column-chunk); lanes walk the unit-stride (or sa1-strided) direction of the row.
template <typename T>
__global__ void __launch_bounds__(256) gemv_row_kernel(int64_t M, int64_t N, T alpha, const T* __restrict__ A,
                                                       int64_t sa0, int64_t sa1, const T* __restrict__ x, int64_t sx,
                                                       T beta, T* __restrict__ y, int64_t sy, int64_t chunk,
                                                       int64_t nchunks) {
  const int lane = threadIdx.x & 31;
  int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w = warp; w < M * nchunks; w += nwarps) {
    int64_t m = w / nchunks, c = w - m * nchunks;
    int64_t n_lo = c * chunk, n_hi = min(N, n_lo + chunk);
    const T* row = A + m * sa0;
    T s = T(0);
    for (int64_t n = n_lo + lane; n < n_hi; n += 32) s += row[n * sa1] * x[n * sx];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) {
      if (nchunks == 1) {
        T v = alpha * s;
        if (beta != T(0)) v += beta * y[m * sy];
        y[m * sy] = v;
      } else {
        atomicAdd(&y[m * sy], alpha * s);  // y was pre-scaled by beta
      }
    }
  }
}

// A is "column fast" (sa0 == 1): lanes own consecutive rows m, each block walks one chunk of columns.
template <typename T>
__global__ void __launch_bounds__(256) gemv_col_kernel(int64_t M, int64_t N, T alpha, const T* __restrict__ A,
                                                       int64_t sa0, int64_t sa1, const T* __restrict__ x, int64_t sx,
                                                       T* __restrict__ y, int64_t sy, int64_t chunk) {
  __shared__ T red[8][33];
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;  // 32 rows x 8 column groups
  int64_t m = (int64_t)blockIdx.x * 32 + lane;
  int64_t n_lo = (int64_t)blockIdx.y * chunk, n_hi = min(N, n_lo + chunk);
  T s = T(0);
  if (m < M)
    for (int64_t n = n_lo + grp; n < n_hi; n += 8) s += A[m * sa0 + n * sa1] * x[n * sx];
  red[grp][lane] = s;
  __syncthreads();
  if (grp == 0 && m < M) {
    T tot = T(0);
#pragma unroll
    for (int g = 0; g < 8; ++g) tot += red[g][lane];
    atomicAdd(&y[m * sy], alpha * tot);  // y was pre-scaled by beta
  }
}

template <typename T>
ptk_status launch_gemv(int64_t M, int64_t N, double alpha, const void* A, int64_t sa0, int64_t sa1, const void* x,
                       int64_t sx, double beta, void* y, int64_t sy, cudaStream_t st) {
  if (M == 0) return PTK_OK;
  const int sms = std::max(1, ptk::sm_count());
  if (sa0 == 1 && sa1 != 1 && N > 1) {
    scale_vec_kernel<T><<<(unsigned)((M + 255) / 256), 256, 0, st>>>((T*)y, sy, M, (T)beta);
    int64_t mblocks = (M + 31) / 32;
    int64_t want = std::max<int64_t>(1, (int64_t)sms * 4 / mblocks);
    int64_t nchunks = std::min<int64_t>(want, (N + 63) / 64);
    nchunks = std::max<int64_t>(1, std::min<int64_t>(nchunks, 65535));
    int64_t chunk = (N + nchunks - 1) / nchunks;
    dim3 grid((unsigned)mblocks, (unsigned)nchunks);
    gemv_col_kernel<T><<<grid, 256, 0, st>>>(M, N, (T)alpha, (const T*)A, sa0, sa1, (const T*)x, sx, (T*)y, sy, chunk);
    PTK_LAUNCH_CHECK("gemv_col");
    return PTK_OK;
  }
  // row kernel: split long rows so that at least ~4 warps per SM exist
  int64_t nchunks = 1;
  int64_t target = (int64_t)sms * 32;
  if (M < target && N > 4096) nchunks = std::min<int64_t>((target + M - 1) / M, (N + 1023) / 1024);
  int64_t chunk = (N + nchunks - 1) / nchunks;
  if (nchunks > 1) scale_vec_kernel<T><<<(unsigned)((M + 255) / 256), 256, 0, st>>>((T*)y, sy, M, (T)beta);
  int64_t warps = M * nchunks;
  unsigned blocks = (unsigned)std::min<int64_t>((warps + 7) / 8, (int64_t)sms * 16);
  gemv_row_kernel<T><<<blocks, 256, 0, st>>>(M, N, (T)alpha, (const T*)A, sa0, sa1, (const T*)x, sx, (T)beta, (T*)y,
                                             sy, chunk, nchunks);
  PTK_LAUNCH_CHECK("gemv_row");
  return PTK_OK;
}

// ---- a whole chain of small dense layers in ONE launch ----------------------------------------------------------------------
// h <- act_l(h @ W_l + b_l), l = 0..L-1, with every layer at most 128 wide (the "256-node Elemwise+Gemm+Scan" metric graph of
// BASELINE.json at n = 64: 84 such layers).  Node by node that is one launch per layer at ~3 us of launch + drain each, for
// ~0.5 MFLOP of work; here a CTA owns 16 rows for ALL layers: the activations live in shared memory (two buffers), the weights
// of layer l+1 stream into shared memory with cp.async while layer l is computed, and nothing but the final activations
// goes back to HBM.  Thread (r, c) = (tid / 16, tid % 16) accumulates 4 consecutive columns [4c + 64j, +4) of row r:
// per k one broadcast LDS of h and one LDS.128 of W per 4 FMAs.  fp32 FMA, k ascending (the SIMT GEMM's arithmetic).
constexpr int MC_MAXW = 128;   // widest layer
constexpr int MC_ROWS = 16;    // rows of the batch per CTA
constexpr int MC_MAXL = 96;    // layers per launch
struct MlpLayer {
  const float* W;      // [K, N] row-major, contiguous, 16-byte aligned, N % 4 == 0
  const float* bias;   // [N] or null
  int K, N, act, pad_;
};
struct MlpChain {
  int L, pad_;
  MlpLayer layer[MC_MAXL];
};

__device__ __forceinline__ void mc_cp_async16(float* dst_smem, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void mc_cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

__global__ void __launch_bounds__(256) mlp_chain_kernel(const float* __restrict__ x, long long sx0, float* __restrict__ y,
                                                        long long sy0, long long M, const __grid_constant__ MlpChain c) {
  extern __shared__ float mc_smem[];
  // Buffer l & 1 of the activations / weights, as ARITHMETIC on the shared array: an indexed array of pointers would live in
  // local memory and turn every access of the k-loop into a generic load behind 64-bit address arithmetic.
  auto hbuf = [&](int i) -> float* { return mc_smem + i * (MC_ROWS * MC_MAXW); };
  auto wbuf = [&](int i) -> float* { return mc_smem + 2 * MC_ROWS * MC_MAXW + i * (MC_MAXW * MC_MAXW); };
  const int tid = threadIdx.x, r = tid >> 4, c0 = tid & 15;
  const long long row0 = (long long)blockIdx.x * MC_ROWS;
  // layer 0's weights start streaming; meanwhile the input rows are copied in (zeros for rows past M)
  {
    const MlpLayer& l0 = c.layer[0];
    const int n4 = (l0.K * l0.N) >> 2;
    for (int i = tid; i < n4; i += 256) mc_cp_async16(wbuf(0) + 4 * i, l0.W + 4 * i);
    for (int i = tid; i < MC_ROWS * l0.K; i += 256) {
      const int rr = i / l0.K, kk = i - rr * l0.K;
      hbuf(0)[rr * MC_MAXW + kk] = (row0 + rr < M) ? x[(row0 + rr) * sx0 + kk] : 0.0f;
    }
  }
  for (int l = 0; l < c.L; ++l) {
    const MlpLayer& ly = c.layer[l];
    mc_cp_async_wait_all();          // this thread's part of W_l has landed ...
    __syncthreads();                 // ... and everybody's, together with the activations the previous layer wrote
    if (l + 1 < c.L) {               // W_{l+1} goes into the buffer layer l-1 used (all its readers passed the barrier above)
      const MlpLayer& nx = c.layer[l + 1];
      const int n4 = (nx.K * nx.N) >> 2;
      float* dst = wbuf((l + 1) & 1);
      for (int i = tid; i < n4; i += 256) mc_cp_async16(dst + 4 * i, nx.W + 4 * i);
    }
    const float* h = hbuf(l & 1) + r * MC_MAXW;
    const float* W = wbuf(l & 1);
    const int K = ly.K, N = ly.N;
    float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    const int ca = 4 * c0, cb = 64 + 4 * c0;
    const bool use_a = ca < N, use_b = cb < N;
    // the bias values are requested BEFORE the product loop (their L2 latency hides behind it); read after it
    float bv[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
    if (ly.bias != nullptr) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (use_a) bv[0][e] = __ldg(ly.bias + ca + e);
        if (use_b) bv[1][e] = __ldg(ly.bias + cb + e);
      }
    }
    for (int k = 0; k < K; ++k) {
      const float hv = h[k];
      if (use_a) {
        const float4 w = *reinterpret_cast<const float4*>(W + k * N + ca);
        acc[0][0] = fmaf(hv, w.x, acc[0][0]); acc[0][1] = fmaf(hv, w.y, acc[0][1]);
        acc[0][2] = fmaf(hv, w.z, acc[0][2]); acc[0][3] = fmaf(hv, w.w, acc[0][3]);
      }
      if (use_b) {
        const float4 w = *reinterpret_cast<const float4*>(W + k * N + cb);
        acc[1][0] = fmaf(hv, w.x, acc[1][0]); acc[1][1] = fmaf(hv, w.y, acc[1][1]);
        acc[1][2] = fmaf(hv, w.z, acc[1][2]); acc[1][3] = fmaf(hv, w.w, acc[1][3]);
      }
    }
    const bool last = l + 1 == c.L;
    float* hn = hbuf((l + 1) & 1) + r * MC_MAXW;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int cc = j ? cb : ca;
      if (cc < N) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = acc[j][e] + bv[j][e];
          if (ly.act == 1) v = tanhf(v);
          if (last) {
            if (row0 + r < M) y[(row0 + r) * sy0 + cc + e] = v;
          } else {
            hn[cc + e] = v;
          }
        }
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) ger_kernel(int64_t M, int64_t N, T alpha, const T* __restrict__ x, int64_t sx,
                                                  const T* __restrict__ y, int64_t sy, T* __restrict__ A, int64_t sa0,
                                                  int64_t sa1) {
  int64_t total = M * N, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int64_t m = i / N, n = i - m * N;
    A[m * sa0 + n * sa1] += alpha * x[m * sx] * y[n * sy];
  }
}

}  // namespace

using namespace ptk;

extern "C" {

size_t ptk_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K, int precision) {
  if (precision == 1) return ptk::gemm_tc_workspace(M, N, K);
  return 0;
}

ptk_status ptk_gemm_bias_act(int dtype, int64_t M, int64_t N, int64_t K, const void* A, int64_t sa0, int64_t sa1,
                             const void* B, int64_t sb0, int64_t sb1, const void* bias, int act, void* C, int64_t sc0,
                             int64_t sc1, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  PTK_REQUIRE_INIT();
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == 1) {
    if (dtype != PTK_F32) return fail(PTK_ERR_UNSUPPORTED, "ptk_gemm: the bf16 tensor-core path takes fp32 graphs only");
    return ptk::gemm_tc_ex(M, N, K, 1.0f, (const float*)A, sa0, sa1, nullptr, 0, (const float*)B, sb0, sb1, 0.0f, (float*)C,
                           sc0, sc1, (const float*)bias, act, nullptr, 0, workspace, workspace_bytes, st);
  }
  if (dtype == PTK_F32) return launch_gemm<float>(M, N, K, 1.0, A, sa0, sa1, B, sb0, sb1, 0.0, C, sc0, sc1, bias, act, st);
  if (dtype == PTK_F64) return launch_gemm<double>(M, N, K, 1.0, A, sa0, sa1, B, sb0, sb1, 0.0, C, sc0, sc1, bias, act, st);
  return fail(PTK_ERR_UNSUPPORTED, "ptk_gemm: dtype must be float32 or float64");
}

ptk_status ptk_mlp_chain(const void* x, int64_t sx0, void* y, int64_t sy0, int64_t M, int L, const void* const* W,
                         const void* const* bias, const int* K, const int* N, const int* act, void* stream) {
  PTK_REQUIRE_INIT();
  if (L < 1 || L > MC_MAXL) return fail(PTK_ERR_ARG, "ptk_mlp_chain: 1..96 layers");
  if (M <= 0) return PTK_OK;
  MlpChain c;
  c.L = L;
  c.pad_ = 0;
  for (int l = 0; l < L; ++l) {
    if (K[l] < 1 || N[l] < 4 || K[l] > MC_MAXW || N[l] > MC_MAXW || (N[l] & 3) || (l > 0 && K[l] != N[l - 1]))
      return fail(PTK_ERR_ARG, "ptk_mlp_chain: layer widths must be <= 128, N a multiple of 4, K_l == N_(l-1)");
    if (((uintptr_t)W[l] & 15) != 0) return fail(PTK_ERR_ARG, "ptk_mlp_chain: weights must be 16-byte aligned");
    c.layer[l].W = (const float*)W[l];
    c.layer[l].bias = bias ? (const float*)bias[l] : nullptr;
    c.layer[l].K = K[l];
    c.layer[l].N = N[l];
    c.layer[l].act = act ? act[l] : 0;
    c.layer[l].pad_ = 0;
  }
  const int smem = (2 * MC_ROWS * MC_MAXW + 2 * MC_MAXW * MC_MAXW) * (int)sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    PTK_CUDA(cudaFuncSetAttribute(mlp_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  const unsigned grid = (unsigned)((M + MC_ROWS - 1) / MC_ROWS);
  mlp_chain_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>((const float*)x, sx0, (float*)y, sy0, M, c);
  PTK_LAUNCH_CHECK("mlp_chain");
  return PTK_OK;
}

ptk_status ptk_gemm(int dtype, int64_t M, int64_t N, int64_t K, double alpha, const void* A, int64_t sa0,
                    int64_t sa1, const void* B, int64_t sb0, int64_t sb1, double beta, void* C, int64_t sc0,
                    int64_t sc1, int precision, void* workspace, size_t workspace_bytes, void* stream) {
  PTK_REQUIRE_INIT();
  cudaStream_t st = (cudaStream_t)stream;
  if (precision == 1) {
    if (dtype != PTK_F32) return fail(PTK_ERR_UNSUPPORTED, "ptk_gemm: the bf16 tensor-core path takes fp32 graphs only");
    return ptk::gemm_tc_ex(M, N, K, (float)alpha, (const float*)A, sa0, sa1, nullptr, 0, (const float*)B, sb0, sb1,
                           (float)beta, (float*)C, sc0, sc1, nullptr, 0, nullptr, 0, workspace, workspace_bytes, st);
  }
  if (dtype == PTK_F32) return launch_gemm<float>(M, N, K, alpha, A, sa0, sa1, B, sb0, sb1, beta, C, sc0, sc1, nullptr, 0, st);
  if (dtype == PTK_F64) return launch_gemm<double>(M, N, K, alpha, A, sa0, sa1, B, sb0, sb1, beta, C, sc0, sc1, nullptr, 0, st);
  return fail(PTK_ERR_UNSUPPORTED, "ptk_gemm: dtype must be float32 or float64");
}

ptk_status ptk_gemv(int dtype, int64_t M, int64_t N, double alpha, const void* A, int64_t sa0, int64_t sa1,
                    const void* x, int64_t sx, double beta, void* y, int64_t sy, void* stream) {
  PTK_REQUIRE_INIT();
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == PTK_F32) return launch_gemv<float>(M, N, alpha, A, sa0, sa1, x, sx, beta, y, sy, st);
  if (dtype == PTK_F64) return launch_gemv<double>(M, N, alpha, A, sa0, sa1, x, sx, beta, y, sy, st);
  return fail(PTK_ERR_UNSUPPORTED, "ptk_gemv: dtype must be float32 or float64");
}

ptk_status ptk_ger(int dtype, int64_t M, int64_t N, double alpha, const void* x, int64_t sx, const void* y,
                   int64_t sy, void* A, int64_t sa0, int64_t sa1, void* stream) {
  PTK_REQUIRE_INIT();
  cudaStream_t st = (cudaStream_t)stream;
  int64_t total = M * N;
  if (total == 0) return PTK_OK;
  unsigned g = (unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)std::max(1, ptk::sm_count()) * 16);
  if (dtype == PTK_F32)
    ger_kernel<float><<<g, 256, 0, st>>>(M, N, (float)alpha, (const float*)x, sx, (const float*)y, sy, (float*)A, sa0, sa1);
  else if (dtype == PTK_F64)
    ger_kernel<double><<<g, 256, 0, st>>>(M, N, alpha, (const double*)x, sx, (const double*)y, sy, (double*)A, sa0, sa1);
  else return fail(PTK_ERR_UNSUPPORTED, "ptk_ger: dtype must be float32 or float64");
  PTK_LAUNCH_CHECK("ger");
  return PTK_OK;
}

}  // extern "C"
