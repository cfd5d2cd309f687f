// Dense factor / triangular-solve kernels for Cholesky, SolveTriangular and CholeskySolve
// (pytensor/tensor/linalg/decomposition/cholesky.py:18 potrf :52-83; solvers/triangular.py:13 trtrs :41-71;
// solvers/psd.py:14 potrs :35-54).
//
// Small matrices (n <= 128, typically batched through Blockwise): one CTA per matrix / per 32-RHS panel, warp-cooperative
// (lanes along the dot-product index).  Large matrices: right-looking BLOCKED algorithms with 64-wide panels — a
// shared-memory diagonal-block kernel, a row-parallel panel solve, and the trailing update on the GEMM kernel
// (ptk_gemm, native precision) — so that O(n^3) work runs on all SMs.
// Failure is signalled the reference's way: NaN-fill, never an exception (cholesky.py:78-80, triangular.py:68-69).
// All matrices are addressed through element strides (rs, cs): "upper" is the lower algorithm on the transposed view.
#include <math_constants.h>
#include <algorithm>
#include <atomic>
#include <mutex>
#include "ptk_common.h"

namespace {

constexpr int NB = 64;  // panel width of the blocked algorithms

template <typename T> __device__ __forceinline__ T nan_of();
template <> __device__ __forceinline__ float nan_of<float>() { return CUDART_NAN_F; }
template <> __device__ __forceinline__ double nan_of<double>() { return CUDART_NAN; }

// ---- small path: left-looking Cholesky, one CTA per matrix ------------------------------------------------------------
// Element (i,j) of the lower factor lives at A[i*rs + j*cs]. Column j: every warp owns rows i>j and forms
// dot(L[i,:j], L[j,:j]) with lanes along k.
template <typename T>
__global__ void __launch_bounds__(512) potrf_small_kernel(T* __restrict__ Aall, int64_t n, int64_t rs, int64_t cs,
                                                          int64_t batch_stride) {
  T* A = Aall + (int64_t)blockIdx.x * batch_stride;
  extern __shared__ unsigned char smem_raw[];
  T* rowj = reinterpret_cast<T*>(smem_raw);  // L[j, 0..j)
  __shared__ T s_d;
  __shared__ int s_bad;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  auto at = [&](int64_t i, int64_t j) -> T& { return A[i * rs + j * cs]; };
  if (tid == 0) s_bad = 0;
  __syncthreads();
  for (int64_t j = 0; j < n; ++j) {
    for (int64_t k = tid; k < j; k += blockDim.x) rowj[k] = at(j, k);
    __syncthreads();
    if (warp == 0) {
      T s = T(0);
      for (int64_t k = lane; k < j; k += 32) s += rowj[k] * rowj[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        T d = at(j, j) - s;
        if (!(d > T(0))) s_bad = 1;
        d = sqrt(d);
        at(j, j) = d;
        s_d = d;
      }
    }
    __syncthreads();
    if (s_bad) break;
    const T inv = T(1) / s_d;
    for (int64_t i = j + 1 + warp; i < n; i += nwarps) {
      T s = T(0);
      for (int64_t k = lane; k < j; k += 32) s += at(i, k) * rowj[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) at(i, j) = (at(i, j) - s) * inv;
    }
    __syncthreads();
  }
  const bool bad = s_bad != 0;
  const T nanv = nan_of<T>();
  for (int64_t e = tid; e < n * n; e += blockDim.x) {
    int64_t r = e / n, c = e - r * n;
    if (bad) at(r, c) = nanv;
    else if (c > r) at(r, c) = T(0);  // clean=True: zero the other triangle
  }
}

// ---- blocked path ----------------------------------------------------------------------------------------------------
// (1) factor the kb x kb diagonal block in shared memory: left-looking, ONE thread per row, ONE barrier per column.  Every
// thread recomputes the pivot column's dot product (row j . row j) itself, so no thread waits for another one's sqrt.
template <typename T>
__global__ void __launch_bounds__(64) potrf_diag_kernel(T* __restrict__ A, int64_t rs, int64_t cs, int kb, int* flag) {
  __shared__ T s[NB][NB + 1];
  const int i = threadIdx.x;
  for (int e = i; e < kb * kb; e += blockDim.x) {
    int r = e / kb, c = e - r * kb;
    s[r][c] = (c <= r) ? A[r * rs + c * cs] : T(0);
  }
  __syncthreads();
  bool bad = false;
  for (int j = 0; j < kb; ++j) {
    T sj0 = T(0), sj1 = T(0), si0 = T(0), si1 = T(0);  // two partial sums each: break the serial FMA dependency
    const bool below = i > j && i < kb;
    int k = 0;
    for (; k + 1 < j; k += 2) {
      const T l0 = s[j][k], l1 = s[j][k + 1];
      sj0 += l0 * l0;
      sj1 += l1 * l1;
      if (below) {
        si0 += s[i][k] * l0;
        si1 += s[i][k + 1] * l1;
      }
    }
    if (k < j) {
      const T l0 = s[j][k];
      sj0 += l0 * l0;
      if (below) si0 += s[i][k] * l0;
    }
    const T sj = sj0 + sj1, si = si0 + si1;
    const T d = s[j][j] - sj;
    if (!(d > T(0))) bad = true;
    const T ljj = sqrt(d);
    T mine = T(0);
    if (i > j && i < kb) mine = (s[i][j] - si) / ljj;
    __syncthreads();  // everyone has read column j / row j before it is overwritten
    if (i == j) s[j][j] = ljj;
    else if (i > j && i < kb) s[i][j] = mine;
    __syncthreads();
  }
  if (bad && i == 0) *flag = 1;
  for (int e = i; e < kb * kb; e += blockDim.x) {
    int r = e / kb, c = e - r * kb;
    if (c <= r) A[r * rs + c * cs] = s[r][c];
  }
}

// (2) panel: rows below the diagonal block solve X * L11^T = A21.  One WARP per row: lane l owns columns l and l+32; the
// forward substitution broadcasts each finished x_j with a shuffle and every lane updates its two pending columns.
template <typename T>
__global__ void __launch_bounds__(256) potrf_panel_kernel(const T* __restrict__ L11, T* __restrict__ A21, int64_t rs,
                                                          int64_t cs, int kb, int64_t m) {
  __shared__ T s[NB][NB + 1];
  for (int e = threadIdx.x; e < kb * kb; e += blockDim.x) {
    int r = e / kb, c = e - r * kb;
    s[r][c] = (c <= r) ? L11[r * rs + c * cs] : T(0);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = warp; i < m; i += nwarps) {
    T* row = A21 + i * rs;
    T a0 = (lane < kb) ? row[lane * cs] : T(0);
    T a1 = (lane + 32 < kb) ? row[(lane + 32) * cs] : T(0);
    for (int j = 0; j < kb; ++j) {
      const int owner = j & 31;
      T x = (j < 32) ? a0 : a1;
      x = x / s[j][j];                       // only the owner lane's value is used
      const T xj = __shfl_sync(0xffffffffu, x, owner);
      if (lane == owner) { if (j < 32) a0 = xj; else a1 = xj; }
      if (lane > j && lane < kb) a0 -= xj * s[lane][j];
      if (lane + 32 > j && lane + 32 < kb) a1 -= xj * s[lane + 32][j];
    }
    if (lane < kb) row[lane * cs] = a0;
    if (lane + 32 < kb) row[(lane + 32) * cs] = a1;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) potrf_clean_kernel(T* __restrict__ A, int64_t n, int64_t rs, int64_t cs,
                                                          const int* flag) {
  const bool bad = *flag != 0;
  const T nanv = nan_of<T>();
  int64_t total = n * n, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    int64_t r = e / n, c = e - r * n;
    if (bad) A[r * rs + c * cs] = nanv;
    else if (c > r) A[r * rs + c * cs] = T(0);
  }
}

// ---- triangular solve --------------------------------------------------------------------------------------------------
// small path: substitution for op(A) X = B, one CTA per (matrix, panel of 32 RHS columns); 32 columns x 8 k-groups.
// opA(i,k) = A[i*ars + k*acs] (the caller folds `trans` into the strides).
template <typename T>
__global__ void __launch_bounds__(256) trsm_small_kernel(const T* __restrict__ Aall, T* __restrict__ Ball, int64_t n,
                                                         int64_t nrhs, int64_t ars, int64_t acs, int fwd, int unit_diag) {
  const T* A = Aall + (int64_t)blockIdx.y * n * n;
  T* B = Ball + (int64_t)blockIdx.y * n * nrhs;
  __shared__ T red[8][33];
  __shared__ int s_sing;
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 5;
  const int64_t col = (int64_t)blockIdx.x * 32 + lane;
  const bool active = col < nrhs;
  if (threadIdx.x == 0) s_sing = 0;
  __syncthreads();
  if (!unit_diag) {
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x)
      if (A[i * (ars + acs)] == T(0)) s_sing = 1;
  }
  __syncthreads();
  if (s_sing) {
    const T nanv = nan_of<T>();
    for (int64_t i = grp; i < n; i += 8)
      if (active) B[i * nrhs + col] = nanv;
    return;
  }
  for (int64_t step = 0; step < n; ++step) {
    const int64_t i = fwd ? step : (n - 1 - step);
    T s = T(0);
    if (active) {
      if (fwd) for (int64_t k = grp; k < i; k += 8) s += A[i * ars + k * acs] * B[k * nrhs + col];
      else     for (int64_t k = i + 1 + grp; k < n; k += 8) s += A[i * ars + k * acs] * B[k * nrhs + col];
    }
    red[grp][lane] = s;
    __syncthreads();
    if (grp == 0 && active) {
      T tot = T(0);
#pragma unroll
      for (int g = 0; g < 8; ++g) tot += red[g][lane];
      T v = B[i * nrhs + col] - tot;
      if (!unit_diag) v = v / A[i * (ars + acs)];
      B[i * nrhs + col] = v;
    }
    __syncthreads();
  }
}

// blocked path, diagonal block: solve the kb x kb triangular system for all RHS columns (threads along columns)
template <typename T>
__global__ void __launch_bounds__(128) trsm_diag_kernel(const T* __restrict__ A11, int64_t ars, int64_t acs,
                                                        T* __restrict__ B1, int64_t nrhs, int kb, int fwd, int unit_diag) {
  __shared__ T s[NB][NB + 1];
  for (int e = threadIdx.x; e < kb * kb; e += blockDim.x) {
    int r = e / kb, c = e - r * kb;
    s[r][c] = A11[r * ars + c * acs];
  }
  __syncthreads();
  const int64_t col = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= nrhs) return;
  T x[NB];
  if (fwd) {
#pragma unroll 1
    for (int i = 0; i < kb; ++i) {
      T v = B1[i * nrhs + col];
      for (int k = 0; k < i; ++k) v -= s[i][k] * x[k];
      x[i] = unit_diag ? v : v / s[i][i];
    }
  } else {
#pragma unroll 1
    for (int i = kb - 1; i >= 0; --i) {
      T v = B1[i * nrhs + col];
      for (int k = i + 1; k < kb; ++k) v -= s[i][k] * x[k];
      x[i] = unit_diag ? v : v / s[i][i];
    }
  }
  for (int i = 0; i < kb; ++i) B1[i * nrhs + col] = x[i];
}

template <typename T>
__global__ void __launch_bounds__(256) diag_zero_check_kernel(const T* __restrict__ A, int64_t n, int64_t step, int* flag) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    if (A[i * step] == T(0)) *flag = 1;
}
template <typename T>
__global__ void __launch_bounds__(256) nan_fill_if_kernel(T* __restrict__ B, int64_t total, const int* flag) {
  if (*flag == 0) return;
  const T nanv = nan_of<T>();
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    B[i] = nanv;
}

template <typename T>
ptk_status potrf_blocked(int dtype, T* A, int64_t n, int64_t rs, int64_t cs, int* flag, cudaStream_t st) {
  PTK_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
  for (int64_t k0 = 0; k0 < n; k0 += NB) {
    const int kb = (int)std::min<int64_t>(NB, n - k0);
    T* A11 = A + k0 * rs + k0 * cs;
    potrf_diag_kernel<T><<<1, 64, 0, st>>>(A11, rs, cs, kb, flag);
    const int64_t m = n - k0 - kb;
    if (m > 0) {
      T* A21 = A + (k0 + kb) * rs + k0 * cs;
      potrf_panel_kernel<T><<<(unsigned)std::min<int64_t>((m + 7) / 8, (int64_t)std::max(1, ptk::sm_count()) * 4), 256, 0, st>>>(A11, A21, rs, cs, kb, m);
      T* A22 = A + (k0 + kb) * rs + (k0 + kb) * cs;
      // A22 -= A21 * A21^T on the GEMM kernel (full square; only the lower triangle is read afterwards)
      ptk_status s = ptk_gemm(dtype, m, m, kb, -1.0, A21, rs, cs, A21, cs, rs, 1.0, A22, rs, cs, 0, nullptr, 0, (void*)st);
      if (s != PTK_OK) return s;
    }
  }
  unsigned g = (unsigned)std::min<int64_t>((n * n + 255) / 256, (int64_t)std::max(1, ptk::sm_count()) * 8);
  potrf_clean_kernel<T><<<g, 256, 0, st>>>(A, n, rs, cs, flag);
  PTK_LAUNCH_CHECK("potrf_blocked");
  return PTK_OK;
}

// ---- Cholesky solve (potrs) --------------------------------------------------------------------------------------------
// Batch layout of ptk_potrs: system i of the output is decomposed over `shape` (row-major); its factor lies at
// sum_d idx_d * stride[d] elements from the base (stride 0 = broadcast).  Passed by value, so nothing is uploaded.
constexpr int POTRS_MAX_DIMS = 8;
struct PotrsBatch {
  int nd;
  int64_t shape[POTRS_MAX_DIMS];
  int64_t stride[POTRS_MAX_DIMS];
};

constexpr int POTRS_WARPS = 8;      // warps per CTA of potrs_small_kernel
constexpr int POTRS_SMALL_N = 128;  // largest n of the one-launch path

// small path: A = C C^T (lower) or U^T U (upper), both triangular sweeps in one launch.  One warp per (system, RHS column);
// the column lives in the warp's shared-memory row `x`.  Warps are independent (no block barrier) and take consecutive
// pairs with the column index fastest, so the columns of one system read its factor through L1.  The stored triangle is
// read by rows in every sweep: where row i holds the coefficients of unknowns already solved, lanes run along k and a
// shuffle reduction forms the dot product; where it holds those of pending unknowns, x_i is finished first and the lanes
// update the pending entries.  Division by the diagonal, no zero check: a zero pivot gives IEEE inf / NaN like ?potrs.
template <typename T>
__global__ void __launch_bounds__(POTRS_WARPS * 32) potrs_small_kernel(const T* __restrict__ C, T* __restrict__ B, int64_t n,
                                                                       int64_t nrhs, int lower, PotrsBatch bat, int64_t npairs) {
  __shared__ T xs[POTRS_WARPS][POTRS_SMALL_N];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T* x = xs[warp];
  const int64_t nwarps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t p = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; p < npairs; p += nwarps) {
    const int64_t sys = p / nrhs, col = p - sys * nrhs;
    int64_t off = 0, rem = sys;
    for (int d = bat.nd - 1; d >= 0; --d) {
      const int64_t q = rem / bat.shape[d];
      off += (rem - q * bat.shape[d]) * bat.stride[d];
      rem = q;
    }
    const T* A = C + off;
    T* b = B + sys * n * nrhs + col;
    for (int64_t i = lane; i < n; i += 32) x[i] = b[i * nrhs];
    __syncwarp();
    // sweep 1 runs forward, sweep 2 backward.  lower: C y = b (dot form), C^T x = y (axpy form);
    // upper: U^T y = b (axpy form), U x = y (dot form).
    for (int sweep = 0; sweep < 2; ++sweep) {
      const bool fwd = sweep == 0, dot = (sweep == 0) == (lower != 0);
      for (int64_t step = 0; step < n; ++step) {
        const int64_t i = fwd ? step : n - 1 - step;
        const T* row = A + i * n;
        if (dot) {
          T s = T(0);
          if (fwd) for (int64_t k = lane; k < i; k += 32) s += row[k] * x[k];
          else     for (int64_t k = i + 1 + lane; k < n; k += 32) s += row[k] * x[k];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (lane == 0) x[i] = (x[i] - s) / row[i];
        } else {
          T xi = T(0);
          if (lane == 0) xi = x[i] / row[i];
          xi = __shfl_sync(0xffffffffu, xi, 0);  // (only lane 0 reads x[i], so its store below races with no read)
          if (fwd) for (int64_t j = i + 1 + lane; j < n; j += 32) x[j] -= row[j] * xi;
          else     for (int64_t j = lane; j < i; j += 32) x[j] -= row[j] * xi;
          if (lane == 0) x[i] = xi;
        }
        __syncwarp();
      }
    }
    for (int64_t i = lane; i < n; i += 32) b[i * nrhs] = x[i];
    __syncwarp();  // the next pair's loads must not overtake this pair's stores of x
  }
}

// `check` != 0 gives trtrs semantics (an exactly-zero diagonal NaN-fills B); 0 gives potrs semantics (IEEE inf / NaN
// from the division, nothing checked) and leaves `flag` unused.
template <typename T>
ptk_status trsm_blocked(int dtype, const T* A, T* B, int64_t n, int64_t nrhs, int64_t ars, int64_t acs, int fwd,
                        int unit_diag, int check, int* flag, cudaStream_t st) {
  if (check) PTK_CUDA(cudaMemsetAsync(flag, 0, sizeof(int), st));
  if (check && !unit_diag) diag_zero_check_kernel<T><<<(unsigned)std::min<int64_t>((n + 255) / 256, 1024), 256, 0, st>>>(A, n, ars + acs, flag);
  const int64_t nblk = (n + NB - 1) / NB;
  for (int64_t b = 0; b < nblk; ++b) {
    const int64_t blk = fwd ? b : (nblk - 1 - b);
    const int64_t k0 = blk * NB;
    const int kb = (int)std::min<int64_t>(NB, n - k0);
    const T* A11 = A + k0 * ars + k0 * acs;
    T* B1 = B + k0 * nrhs;
    trsm_diag_kernel<T><<<(unsigned)((nrhs + 127) / 128), 128, 0, st>>>(A11, ars, acs, B1, nrhs, kb, fwd, unit_diag);
    if (fwd) {
      const int64_t m = n - k0 - kb;
      if (m > 0) {  // B2 -= A21 * X1
        ptk_status s = ptk_gemm(dtype, m, nrhs, kb, -1.0, A + (k0 + kb) * ars + k0 * acs, ars, acs, B1, nrhs, 1, 1.0,
                                B + (k0 + kb) * nrhs, nrhs, 1, 0, nullptr, 0, (void*)st);
        if (s != PTK_OK) return s;
      }
    } else if (k0 > 0) {  // B0 -= A01 * X1
      ptk_status s = ptk_gemm(dtype, k0, nrhs, kb, -1.0, A + k0 * acs, ars, acs, B1, nrhs, 1, 1.0, B, nrhs, 1, 0, nullptr, 0,
                              (void*)st);
      if (s != PTK_OK) return s;
    }
  }
  if (check) nan_fill_if_kernel<T><<<(unsigned)std::min<int64_t>((n * nrhs + 255) / 256, 2048), 256, 0, st>>>(B, n * nrhs, flag);
  PTK_LAUNCH_CHECK("trsm_blocked");
  return PTK_OK;
}

// Status word of one blocked factorisation / solve.  Calls on different streams (parallel branches of a captured graph) must
// not share a word, so every call takes the next one of a small ring; a captured node keeps the word it was captured with.
int* scratch_flag() {
  constexpr unsigned kWords = 1024;
  static int* p = nullptr;
  static std::atomic<unsigned> next{0};
  static std::once_flag once;
  std::call_once(once, [] { if (cudaMalloc(&p, kWords * sizeof(int)) != cudaSuccess) p = nullptr; });
  return p ? p + (next.fetch_add(1) % kWords) : nullptr;
}

}  // namespace

using namespace ptk;

extern "C" {

ptk_status ptk_potrf(int dtype, void* A, int64_t n, int64_t batch, int lower, void* stream) {
  PTK_REQUIRE_INIT();
  if (n == 0 || batch == 0) return PTK_OK;
  if (batch > 2147483647LL) return fail(PTK_ERR_ARG, "ptk_potrf: batch too large");
  if (dtype != PTK_F32 && dtype != PTK_F64) return fail(PTK_ERR_UNSUPPORTED, "ptk_potrf: dtype must be float32 or float64");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t rs = lower ? n : 1, cs = lower ? 1 : n;  // upper = the lower algorithm on the transposed view
  if (n <= 128) {
    size_t smem = (size_t)n * dtype_size(dtype);
    int threads = n >= 64 ? 256 : 64;
    if (dtype == PTK_F32) potrf_small_kernel<float><<<(unsigned)batch, threads, smem, st>>>((float*)A, n, rs, cs, n * n);
    else potrf_small_kernel<double><<<(unsigned)batch, threads, smem, st>>>((double*)A, n, rs, cs, n * n);
    PTK_LAUNCH_CHECK("potrf_small");
    return PTK_OK;
  }
  int* flag = scratch_flag();
  if (!flag) return fail(PTK_ERR_CUDA, "ptk_potrf: cannot allocate the status word");
  for (int64_t b = 0; b < batch; ++b) {
    ptk_status s = dtype == PTK_F32 ? potrf_blocked<float>(dtype, (float*)A + b * n * n, n, rs, cs, flag, st)
                                    : potrf_blocked<double>(dtype, (double*)A + b * n * n, n, rs, cs, flag, st);
    if (s != PTK_OK) return s;
  }
  return PTK_OK;
}

ptk_status ptk_trsm(int dtype, const void* A, void* B, int64_t n, int64_t nrhs, int64_t batch, int lower, int trans,
                    int unit_diag, void* stream) {
  PTK_REQUIRE_INIT();
  if (n == 0 || nrhs == 0 || batch == 0) return PTK_OK;
  if (batch > 65535) return fail(PTK_ERR_ARG, "ptk_trsm: batch > 65535");
  if (dtype != PTK_F32 && dtype != PTK_F64) return fail(PTK_ERR_UNSUPPORTED, "ptk_trsm: dtype must be float32 or float64");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t ars = trans ? 1 : n, acs = trans ? n : 1;  // op(A)(i,k) = A[i*ars + k*acs]
  const int fwd = ((lower != 0) != (trans != 0)) ? 1 : 0;
  if (n <= 128) {
    dim3 grid((unsigned)((nrhs + 31) / 32), (unsigned)batch);
    if (dtype == PTK_F32)
      trsm_small_kernel<float><<<grid, 256, 0, st>>>((const float*)A, (float*)B, n, nrhs, ars, acs, fwd, unit_diag);
    else
      trsm_small_kernel<double><<<grid, 256, 0, st>>>((const double*)A, (double*)B, n, nrhs, ars, acs, fwd, unit_diag);
    PTK_LAUNCH_CHECK("trsm_small");
    return PTK_OK;
  }
  int* flag = scratch_flag();
  if (!flag) return fail(PTK_ERR_CUDA, "ptk_trsm: cannot allocate the status word");
  for (int64_t b = 0; b < batch; ++b) {
    ptk_status s = dtype == PTK_F32
                       ? trsm_blocked<float>(dtype, (const float*)A + b * n * n, (float*)B + b * n * nrhs, n, nrhs, ars, acs,
                                             fwd, unit_diag, 1, flag, st)
                       : trsm_blocked<double>(dtype, (const double*)A + b * n * n, (double*)B + b * n * nrhs, n, nrhs, ars,
                                              acs, fwd, unit_diag, 1, flag, st);
    if (s != PTK_OK) return s;
  }
  return PTK_OK;
}

ptk_status ptk_potrs(int dtype, const void* C, void* B, int64_t n, int64_t nrhs, int lower, int nbatch_dims,
                     const int64_t* batch_shape, const int64_t* factor_batch_strides, void* stream) {
  PTK_REQUIRE_INIT();
  if (dtype != PTK_F32 && dtype != PTK_F64) return fail(PTK_ERR_UNSUPPORTED, "ptk_potrs: dtype must be float32 or float64");
  if (nbatch_dims < 0 || nbatch_dims > POTRS_MAX_DIMS) return fail(PTK_ERR_ARG, "ptk_potrs: at most 8 batch dimensions");
  if (n < 0 || nrhs < 0) return fail(PTK_ERR_ARG, "ptk_potrs: negative size");
  PotrsBatch bat{};
  bat.nd = nbatch_dims;
  int64_t systems = 1;
  for (int d = 0; d < nbatch_dims; ++d) {
    if (batch_shape[d] < 0) return fail(PTK_ERR_ARG, "ptk_potrs: negative batch dimension");
    bat.shape[d] = batch_shape[d];
    bat.stride[d] = factor_batch_strides[d];
    systems *= batch_shape[d];
  }
  if (n == 0 || nrhs == 0 || systems == 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (n <= POTRS_SMALL_N) {
    const int64_t pairs = systems * nrhs;
    const unsigned grid = (unsigned)std::min<int64_t>((pairs + POTRS_WARPS - 1) / POTRS_WARPS,
                                                      (int64_t)std::max(1, ptk::sm_count()) * 16);
    if (dtype == PTK_F32)
      potrs_small_kernel<float><<<grid, POTRS_WARPS * 32, 0, st>>>((const float*)C, (float*)B, n, nrhs, lower, bat, pairs);
    else
      potrs_small_kernel<double><<<grid, POTRS_WARPS * 32, 0, st>>>((const double*)C, (double*)B, n, nrhs, lower, bat, pairs);
    PTK_LAUNCH_CHECK("potrs_small");
    return PTK_OK;
  }
  // blocked path: two triangular solves per system.  lower: C y = b, then C^T x = y; upper: U^T y = b, then U x = y.
  // op(A)(i,k) = A[i*ars + k*acs]: (n, 1) reads the stored triangle as is, (1, n) its transpose.
  for (int64_t s = 0; s < systems; ++s) {
    int64_t off = 0, rem = s;
    for (int d = nbatch_dims - 1; d >= 0; --d) {
      const int64_t q = rem / bat.shape[d];
      off += (rem - q * bat.shape[d]) * bat.stride[d];
      rem = q;
    }
    for (int sweep = 0; sweep < 2; ++sweep) {
      const int fwd = sweep == 0 ? 1 : 0;
      const bool plain = (sweep == 0) == (lower != 0);
      const int64_t ars = plain ? n : 1, acs = plain ? 1 : n;
      ptk_status r = dtype == PTK_F32
                         ? trsm_blocked<float>(dtype, (const float*)C + off, (float*)B + s * n * nrhs, n, nrhs, ars, acs, fwd,
                                               0, 0, nullptr, st)
                         : trsm_blocked<double>(dtype, (const double*)C + off, (double*)B + s * n * nrhs, n, nrhs, ars, acs,
                                                fwd, 0, 0, nullptr, st);
      if (r != PTK_OK) return r;
    }
  }
  return PTK_OK;
}

}  // extern "C"
