// Data-movement glue kernels (HBM-bound byte work): strided copy / set / inc, take (gather) and put (scatter).
// Replaces the C loops the reference emits for DeepCopyOp, Alloc, IncSubtensor, AdvancedSubtensor and
// AdvancedIncSubtensor (pytensor/compile/ops.py:121, tensor/basic.py:1545, tensor/subtensor.py:1441,1932,2275).
#include <algorithm>
#include "ptk_common.h"

namespace {

constexpr int kMaxDims = 8;

struct Dims {
  int ndim;
  int64_t shape[kMaxDims];
  int64_t a[kMaxDims];  // dst strides (elements)
  int64_t b[kMaxDims];  // src strides (elements)
};

// Drop size-1 dims and merge neighbours that are contiguous in BOTH operands; returns total element count.
int64_t collapse(Dims& d, const int64_t* shape, const int64_t* sa, const int64_t* sb, int ndim) {
  int64_t total = 1;
  int n = 0;
  for (int i = 0; i < ndim; ++i) {
    total *= shape[i];
    if (shape[i] == 1) continue;
    if (n > 0 && d.a[n - 1] == sa[i] * shape[i] && d.b[n - 1] == sb[i] * shape[i]) {
      d.shape[n - 1] *= shape[i];
      d.a[n - 1] = sa[i];
      d.b[n - 1] = sb[i];
    } else {
      d.shape[n] = shape[i];
      d.a[n] = sa[i];
      d.b[n] = sb[i];
      ++n;
    }
  }
  if (n == 0) {
    d.shape[0] = 1;
    d.a[0] = 0;
    d.b[0] = 0;
    n = 1;
  }
  d.ndim = n;
  return total;
}

template <typename T>
__global__ void __launch_bounds__(256) copy_strided_kernel(T* __restrict__ dst, const T* __restrict__ src, Dims d,
                                                           int64_t total) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int64_t r = i, oa = 0, ob = 0;
#pragma unroll
    for (int k = kMaxDims - 1; k >= 0; --k) {
      if (k < d.ndim) {
        int64_t c = r;                        // the outermost axis (k == 0) keeps what is left: no division
        if (k > 0) {
          const int64_t q = r / d.shape[k];
          c = r - q * d.shape[k];
          r = q;
        }
        oa += c * d.a[k];
        ob += c * d.b[k];
      }
    }
    dst[oa] = src[ob];
  }
}

// Contiguous destination and source both 16-byte aligned: plain 128-bit streaming copy.
__global__ void __launch_bounds__(256) copy_vec16_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src,
                                                         int64_t n16) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += stride) dst[i] = src[i];
}

template <typename T>
__device__ __forceinline__ void atomic_add_t(T* p, T v) { atomicAdd(p, v); }
template <>
__device__ __forceinline__ void atomic_add_t<int64_t>(int64_t* p, int64_t v) {
  atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}
template <>
__device__ __forceinline__ void atomic_add_t<uint64_t>(uint64_t* p, uint64_t v) {
  atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
}

template <typename T>
__global__ void __launch_bounds__(256) inc_strided_kernel(T* __restrict__ dst, const T* __restrict__ src, Dims d,
                                                          int64_t total) {
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int64_t r = i, oa = 0, ob = 0;
#pragma unroll
    for (int k = kMaxDims - 1; k >= 0; --k) {
      if (k < d.ndim) {
        int64_t c = r;                        // the outermost axis (k == 0) keeps what is left: no division
        if (k > 0) {
          const int64_t q = r / d.shape[k];
          c = r - q * d.shape[k];
          r = q;
        }
        oa += c * d.a[k];
        ob += c * d.b[k];
      }
    }
    dst[oa] = dst[oa] + src[ob];
  }
}

template <typename T>
__global__ void __launch_bounds__(256) take_kernel(T* __restrict__ out, const T* __restrict__ src,
                                                   const int64_t* __restrict__ idx, int64_t outer, int64_t n_src,
                                                   int64_t n_idx, int64_t inner, int* err) {
  int64_t total = outer * n_idx * inner;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    int64_t i = t % inner;
    int64_t r = t / inner;
    int64_t j = r % n_idx;
    int64_t o = r / n_idx;
    int64_t k = idx[j];
    if (k < 0) k += n_src;
    if (k < 0 || k >= n_src) {
      if (err) atomicExch(err, 1);
      continue;
    }
    out[t] = src[(o * n_src + k) * inner + i];
  }
}

template <typename T, int OP>
__global__ void __launch_bounds__(256) put_kernel(T* __restrict__ dst, const T* __restrict__ y,
                                                  const int64_t* __restrict__ idx, int64_t outer, int64_t n_dst,
                                                  int64_t n_idx, int64_t inner, int* err) {
  int64_t total = outer * n_idx * inner;
  int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {
    int64_t i = t % inner;
    int64_t r = t / inner;
    int64_t j = r % n_idx;
    int64_t o = r / n_idx;
    int64_t k = idx[j];
    if (k < 0) k += n_dst;
    if (k < 0 || k >= n_dst) {
      if (err) atomicExch(err, 1);
      continue;
    }
    T* p = dst + (o * n_dst + k) * inner + i;
    if (OP == 0) *p = y[t];
    else atomic_add_t<T>(p, y[t]);
  }
}

// take along the LAST axis (inner == 1): out[o, j] = src[o, idx[j]].  A thread owns 4 consecutive j (one 128-bit store per
// row for 4-byte types) and reuses its 4 indices over ROWS rows; no integer division in the hot loop.
template <typename T>
__global__ void __launch_bounds__(256) take_lastaxis_kernel(T* __restrict__ out, const T* __restrict__ src,
                                                            const int64_t* __restrict__ idx, int64_t outer, int64_t n_src,
                                                            int64_t n_idx, int* err) {
  const int64_t j0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (j0 >= n_idx) return;
  int64_t k[4];
  bool ok[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    ok[e] = j0 + e < n_idx;
    int64_t v = ok[e] ? idx[j0 + e] : 0;
    if (v < 0) v += n_src;
    if (v < 0 || v >= n_src) {
      if (ok[e] && err) atomicExch(err, 1);
      ok[e] = false;
      v = 0;
    }
    k[e] = v;
  }
  const bool vec = ok[0] && ok[1] && ok[2] && ok[3] && (n_idx % 4 == 0) && sizeof(T) == 4 && (((uintptr_t)out & 15) == 0);
  int64_t o = blockIdx.y;
  if (vec) {
    for (; o + 3 * (int64_t)gridDim.y < outer; o += 4 * (int64_t)gridDim.y) {  // 4 rows = 16 independent gathers in flight
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const T* s = src + (o + u * (int64_t)gridDim.y) * n_src;
        v[u].x = (uint32_t)s[k[0]]; v[u].y = (uint32_t)s[k[1]]; v[u].z = (uint32_t)s[k[2]]; v[u].w = (uint32_t)s[k[3]];
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        *reinterpret_cast<uint4*>(out + (o + u * (int64_t)gridDim.y) * n_idx + j0) = v[u];
    }
  }
  for (; o < outer; o += gridDim.y) {
    const T* s = src + o * n_src;
    T* d = out + o * n_idx + j0;
    if (vec) {
      uint4 v;
      v.x = (uint32_t)s[k[0]]; v.y = (uint32_t)s[k[1]]; v.z = (uint32_t)s[k[2]]; v.w = (uint32_t)s[k[3]];
      *reinterpret_cast<uint4*>(d) = v;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (ok[e]) d[e] = s[k[e]];
    }
  }
}

// take along the last axis when the source rows are small: a CTA stages ROWS source rows in shared memory (coalesced), then
// every thread gathers 4 consecutive j for each staged row from shared memory and stores 128-bit — no global-memory
// latency inside the gather, fully coalesced writes (the kernel is bound by the output write).
template <typename T, int ROWS>
__global__ void __launch_bounds__(256) take_lastaxis_smem_kernel(T* __restrict__ out, const T* __restrict__ src,
                                                                 const int64_t* __restrict__ idx, int64_t outer, int64_t n_src,
                                                                 int64_t n_idx, int* err) {
  extern __shared__ unsigned char take_smem[];
  T* rows = reinterpret_cast<T*>(take_smem);  // [ROWS][n_src]
  const int64_t o0 = (int64_t)blockIdx.y * ROWS;
  const int nrows = (int)min((int64_t)ROWS, outer - o0);
  const T* s0 = src + o0 * n_src;
  for (int64_t e = threadIdx.x; e < (int64_t)nrows * n_src; e += blockDim.x) rows[e] = s0[e];
  __syncthreads();
  for (int64_t j0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; j0 < n_idx; j0 += (int64_t)gridDim.x * blockDim.x * 4) {
    int k[4];
    bool ok[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      ok[e] = j0 + e < n_idx;
      int64_t v = ok[e] ? idx[j0 + e] : 0;
      if (v < 0) v += n_src;
      if (v < 0 || v >= n_src) {
        if (ok[e] && err) atomicExch(err, 1);
        ok[e] = false;
        v = 0;
      }
      k[e] = (int)v;
    }
    const bool vec = ok[0] && ok[1] && ok[2] && ok[3] && (n_idx % 4 == 0) && sizeof(T) == 4 && (((uintptr_t)out & 15) == 0);
    for (int r = 0; r < nrows; ++r) {
      const T* sr = rows + (int64_t)r * n_src;
      T* d = out + (o0 + r) * n_idx + j0;
      if (vec) {
        uint4 v;
        v.x = (uint32_t)sr[k[0]]; v.y = (uint32_t)sr[k[1]]; v.z = (uint32_t)sr[k[2]]; v.w = (uint32_t)sr[k[3]];
        *reinterpret_cast<uint4*>(d) = v;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (ok[e]) d[e] = sr[k[e]];
      }
    }
  }
}

// ---- scatter-add along the last axis with an index vector shared by all rows: a deterministic segmented reduction ----------
// (1) histogram + exclusive scan of the destination bins; (2) stable fill of the permutation; (3) one warp per row.
__global__ void __launch_bounds__(1024) put_rows_offsets_kernel(const int64_t* __restrict__ idx, int64_t n_idx, int64_t n_dst,
                                                                int* __restrict__ offsets, int* err) {
  extern __shared__ int cnt[];
  for (int64_t j = threadIdx.x; j <= n_dst; j += blockDim.x) cnt[j] = 0;
  __syncthreads();
  for (int64_t i = threadIdx.x; i < n_idx; i += blockDim.x) {
    int64_t k = idx[i];
    if (k < 0) k += n_dst;
    if (k < 0 || k >= n_dst) {
      if (err) atomicExch(err, 1);
      continue;
    }
    atomicAdd(&cnt[k], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int64_t j = 0; j < n_dst; ++j) {
      int c = cnt[j];
      offsets[j] = run;
      run += c;
    }
    offsets[n_dst] = run;
  }
}
__global__ void __launch_bounds__(256) put_rows_perm_kernel(const int64_t* __restrict__ idx, int64_t n_idx, int64_t n_dst,
                                                            const int* __restrict__ offsets, int* __restrict__ perm) {
  extern __shared__ int sidx[];  // normalised indices, shared by the block
  for (int64_t i = threadIdx.x; i < n_idx; i += blockDim.x) {
    int64_t k = idx[i];
    if (k < 0) k += n_dst;
    sidx[i] = (k >= 0 && k < n_dst) ? (int)k : -1;
  }
  __syncthreads();
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;  // one destination bin per thread
  if (j >= n_dst) return;
  int p = offsets[j];
  for (int i = 0; i < (int)n_idx; ++i)
    if (sidx[i] == (int)j) perm[p++] = i;  // ascending i: the same accumulation order as np.add.at
}
template <typename T>
__global__ void __launch_bounds__(256) put_rows_kernel(T* __restrict__ dst, const T* __restrict__ y,
                                                       const int* __restrict__ offsets, const int* __restrict__ perm,
                                                       int64_t outer, int64_t n_dst, int64_t n_idx, int warps_per_block) {
  extern __shared__ unsigned char put_smem[];
  int* s_off = reinterpret_cast<int*>(put_smem);            // [n_dst + 1]
  int* s_perm = s_off + (n_dst + 1);                        // [n_idx]
  T* ys = reinterpret_cast<T*>(s_perm + n_idx + ((n_dst + 1 + n_idx) & 1));  // 8-byte aligned rows
  for (int64_t i = threadIdx.x; i <= n_dst; i += blockDim.x) s_off[i] = offsets[i];
  for (int64_t i = threadIdx.x; i < n_idx; i += blockDim.x) s_perm[i] = perm[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp >= warps_per_block) return;
  T* mine = ys + (int64_t)warp * n_idx;
  for (int64_t o = (int64_t)blockIdx.x * warps_per_block + warp; o < outer; o += (int64_t)gridDim.x * warps_per_block) {
    const T* yrow = y + o * n_idx;
    int64_t i = lane;
    for (; i + 7 * 32 < n_idx; i += 8 * 32) {  // 8 independent 128-byte warp loads in flight before the first smem store
      T t[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) t[u] = yrow[i + u * 32];
#pragma unroll
      for (int u = 0; u < 8; ++u) mine[i + u * 32] = t[u];
    }
    for (; i < n_idx; i += 32) mine[i] = yrow[i];
    __syncwarp();
    T* drow = dst + o * n_dst;
    for (int64_t j = lane; j < n_dst; j += 64) {   // two destination bins per lane, their chains interleaved
      const int64_t j2 = j + 32;
      const bool has2 = j2 < n_dst;
      T acc0 = drow[j], acc1 = has2 ? drow[j2] : T(0);
      int p0 = s_off[j], e0 = s_off[j + 1];
      int p1 = has2 ? s_off[j2] : 0, e1 = has2 ? s_off[j2 + 1] : 0;
      while (p0 < e0 || p1 < e1) {
        if (p0 < e0) acc0 += mine[s_perm[p0++]];
        if (p1 < e1) acc1 += mine[s_perm[p1++]];
      }
      drow[j] = acc0;
      if (has2) drow[j2] = acc1;
    }
    __syncwarp();
  }
}

inline unsigned grid_for(int64_t total, int threads = 256) {
  int64_t blocks = (total + threads - 1) / threads;
  int64_t cap = (int64_t)ptk::sm_count() * 16;
  if (cap <= 0) cap = 132 * 16;  // H100 SXM
  return (unsigned)std::max<int64_t>(1, std::min(blocks, cap));
}

}  // namespace

using namespace ptk;

extern "C" {

ptk_status ptk_copy_strided(void* dst, const int64_t* dst_strides, const void* src, const int64_t* src_strides,
                            const int64_t* shape, int ndim, int itemsize, void* stream) {
  PTK_REQUIRE_INIT();
  if (ndim < 0 || ndim > kMaxDims) return fail(PTK_ERR_ARG, "ptk_copy_strided: ndim > 8");
  Dims d;
  int64_t total = collapse(d, shape, dst_strides, src_strides, ndim);
  if (total == 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (d.ndim == 1 && d.a[0] == 1 && d.b[0] == 1) {
    size_t bytes = (size_t)total * itemsize;
    if (bytes % 16 == 0 && ((uintptr_t)dst % 16 == 0) && ((uintptr_t)src % 16 == 0)) {
      copy_vec16_kernel<<<grid_for(bytes / 16), 256, 0, st>>>((uint4*)dst, (const uint4*)src, bytes / 16);
      PTK_LAUNCH_CHECK("copy_vec16");
      return PTK_OK;
    }
  }
  unsigned g = grid_for(total);
  switch (itemsize) {
    case 1: copy_strided_kernel<uint8_t><<<g, 256, 0, st>>>((uint8_t*)dst, (const uint8_t*)src, d, total); break;
    case 2: copy_strided_kernel<uint16_t><<<g, 256, 0, st>>>((uint16_t*)dst, (const uint16_t*)src, d, total); break;
    case 4: copy_strided_kernel<uint32_t><<<g, 256, 0, st>>>((uint32_t*)dst, (const uint32_t*)src, d, total); break;
    case 8: copy_strided_kernel<uint64_t><<<g, 256, 0, st>>>((uint64_t*)dst, (const uint64_t*)src, d, total); break;
    default: return fail(PTK_ERR_ARG, "ptk_copy_strided: itemsize must be 1, 2, 4 or 8");
  }
  PTK_LAUNCH_CHECK("copy_strided");
  return PTK_OK;
}

ptk_status ptk_inc_strided(void* dst, const int64_t* dst_strides, const void* src, const int64_t* src_strides,
                           const int64_t* shape, int ndim, int dtype, int op, void* stream) {
  PTK_REQUIRE_INIT();
  if (op == 0) return ptk_copy_strided(dst, dst_strides, src, src_strides, shape, ndim, dtype_size(dtype), stream);
  if (ndim < 0 || ndim > kMaxDims) return fail(PTK_ERR_ARG, "ptk_inc_strided: ndim > 8");
  Dims d;
  int64_t total = collapse(d, shape, dst_strides, src_strides, ndim);
  if (total == 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned g = grid_for(total);
#define PTK_INC(T) inc_strided_kernel<T><<<g, 256, 0, st>>>((T*)dst, (const T*)src, d, total); break;
  switch (dtype) {
    case PTK_F32: PTK_INC(float)
    case PTK_F64: PTK_INC(double)
    case PTK_I8: PTK_INC(int8_t)
    case PTK_I16: PTK_INC(int16_t)
    case PTK_I32: PTK_INC(int32_t)
    case PTK_I64: PTK_INC(int64_t)
    case PTK_U8: PTK_INC(uint8_t)
    case PTK_U16: PTK_INC(uint16_t)
    case PTK_U32: PTK_INC(uint32_t)
    case PTK_U64: PTK_INC(uint64_t)
    default: return fail(PTK_ERR_UNSUPPORTED, "ptk_inc_strided: dtype");
  }
#undef PTK_INC
  PTK_LAUNCH_CHECK("inc_strided");
  return PTK_OK;
}

ptk_status ptk_take(void* out, const void* src, const int64_t* idx, int64_t outer, int64_t n_src, int64_t n_idx,
                    int64_t inner, int itemsize, int* err_flag, void* stream) {
  PTK_REQUIRE_INIT();
  int64_t total = outer * n_idx * inner;
  if (total == 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (inner == 1 && outer >= 64 && n_idx >= 64 && n_src * 16 * itemsize <= 40 * 1024 && outer / 16 <= 65535 * 16LL) {
    constexpr int ROWS = 16;
    unsigned gx = (unsigned)std::min<int64_t>((n_idx + 1023) / 1024, 8);
    dim3 grid(gx, (unsigned)((outer + ROWS - 1) / ROWS));
    if (grid.y <= 65535u * 16u && grid.y <= 2147483647u) {
      size_t smem = (size_t)ROWS * n_src * itemsize;
      if (grid.y > 65535) grid = dim3(gx, 65535);  // (guarded above; kept for clarity)
      switch (itemsize) {
        case 1: take_lastaxis_smem_kernel<uint8_t, ROWS><<<dim3(gx, (unsigned)((outer + ROWS - 1) / ROWS)), 256, smem, st>>>((uint8_t*)out, (const uint8_t*)src, idx, outer, n_src, n_idx, err_flag); break;
        case 2: take_lastaxis_smem_kernel<uint16_t, ROWS><<<dim3(gx, (unsigned)((outer + ROWS - 1) / ROWS)), 256, smem, st>>>((uint16_t*)out, (const uint16_t*)src, idx, outer, n_src, n_idx, err_flag); break;
        case 4: take_lastaxis_smem_kernel<uint32_t, ROWS><<<dim3(gx, (unsigned)((outer + ROWS - 1) / ROWS)), 256, smem, st>>>((uint32_t*)out, (const uint32_t*)src, idx, outer, n_src, n_idx, err_flag); break;
        case 8: take_lastaxis_smem_kernel<uint64_t, ROWS><<<dim3(gx, (unsigned)((outer + ROWS - 1) / ROWS)), 256, smem, st>>>((uint64_t*)out, (const uint64_t*)src, idx, outer, n_src, n_idx, err_flag); break;
        default: return fail(PTK_ERR_ARG, "ptk_take: itemsize must be 1, 2, 4 or 8");
      }
      PTK_LAUNCH_CHECK("take_lastaxis_smem");
      return PTK_OK;
    }
  }
  if (inner == 1 && outer >= 8 && n_idx >= 64) {
    unsigned gx = (unsigned)((n_idx + 1023) / 1024);
    unsigned gy = (unsigned)std::min<int64_t>(outer, std::max<int64_t>(1, (int64_t)std::max(1, ptk::sm_count()) * 16 / gx));
    dim3 grid(gx, gy);
    switch (itemsize) {
      case 1: take_lastaxis_kernel<uint8_t><<<grid, 256, 0, st>>>((uint8_t*)out, (const uint8_t*)src, idx, outer, n_src, n_idx, err_flag); break;
      case 2: take_lastaxis_kernel<uint16_t><<<grid, 256, 0, st>>>((uint16_t*)out, (const uint16_t*)src, idx, outer, n_src, n_idx, err_flag); break;
      case 4: take_lastaxis_kernel<uint32_t><<<grid, 256, 0, st>>>((uint32_t*)out, (const uint32_t*)src, idx, outer, n_src, n_idx, err_flag); break;
      case 8: take_lastaxis_kernel<uint64_t><<<grid, 256, 0, st>>>((uint64_t*)out, (const uint64_t*)src, idx, outer, n_src, n_idx, err_flag); break;
      default: return fail(PTK_ERR_ARG, "ptk_take: itemsize must be 1, 2, 4 or 8");
    }
    PTK_LAUNCH_CHECK("take_lastaxis");
    return PTK_OK;
  }
  unsigned g = grid_for(total);
#define PTK_TAKE(T) \
  take_kernel<T><<<g, 256, 0, st>>>((T*)out, (const T*)src, idx, outer, n_src, n_idx, inner, err_flag); break;
  switch (itemsize) {
    case 1: PTK_TAKE(uint8_t)
    case 2: PTK_TAKE(uint16_t)
    case 4: PTK_TAKE(uint32_t)
    case 8: PTK_TAKE(uint64_t)
    default: return fail(PTK_ERR_ARG, "ptk_take: itemsize must be 1, 2, 4 or 8");
  }
#undef PTK_TAKE
  PTK_LAUNCH_CHECK("take");
  return PTK_OK;
}

ptk_status ptk_put(void* dst, const void* y, const int64_t* idx, int64_t outer, int64_t n_dst, int64_t n_idx,
                   int64_t inner, int dtype, int op, int* err_flag, void* stream) {
  PTK_REQUIRE_INIT();
  int64_t total = outer * n_idx * inner;
  if (total == 0) return PTK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned g = grid_for(total);
#define PTK_PUT(T)                                                                                              \
  if (op == 0) put_kernel<T, 0><<<g, 256, 0, st>>>((T*)dst, (const T*)y, idx, outer, n_dst, n_idx, inner, err_flag); \
  else put_kernel<T, 1><<<g, 256, 0, st>>>((T*)dst, (const T*)y, idx, outer, n_dst, n_idx, inner, err_flag);   \
  break;
  switch (dtype) {
    case PTK_F32: PTK_PUT(float)
    case PTK_F64: PTK_PUT(double)
    case PTK_I32: PTK_PUT(int32_t)
    case PTK_I64: PTK_PUT(int64_t)
    case PTK_U32: PTK_PUT(uint32_t)
    case PTK_U64: PTK_PUT(uint64_t)
    default: return fail(PTK_ERR_UNSUPPORTED, "ptk_put: dtype (f32/f64/i32/i64/u32/u64 only)");
  }
#undef PTK_PUT
  PTK_LAUNCH_CHECK("put");
  return PTK_OK;
}

size_t ptk_put_rows_workspace_bytes(int64_t n_dst, int64_t n_idx) { return (size_t)(n_dst + 1 + n_idx) * sizeof(int) + 64; }

ptk_status ptk_put_rows(void* dst, const void* y, const int64_t* idx, int64_t outer, int64_t n_dst, int64_t n_idx, int dtype,
                        void* workspace, size_t workspace_bytes, int* err_flag, void* stream) {
  PTK_REQUIRE_INIT();
  if (outer == 0 || n_idx == 0) return PTK_OK;
  if (dtype != PTK_F32 && dtype != PTK_F64) return fail(PTK_ERR_UNSUPPORTED, "ptk_put_rows: dtype must be float32 or float64");
  const int isz = dtype_size(dtype);
  if (n_dst + 1 > 12000 || n_idx * isz > 48 * 1024 || n_dst < 1)
    return fail(PTK_ERR_UNSUPPORTED, "ptk_put_rows: n_dst <= 11999 and n_idx * itemsize <= 48 KiB required");
  if (workspace == nullptr || workspace_bytes < ptk_put_rows_workspace_bytes(n_dst, n_idx))
    return fail(PTK_ERR_ARG, "ptk_put_rows: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  int* offsets = reinterpret_cast<int*>(workspace);
  int* perm = offsets + (n_dst + 1);
  put_rows_offsets_kernel<<<1, 1024, (size_t)(n_dst + 1) * sizeof(int), st>>>(idx, n_idx, n_dst, offsets, err_flag);
  put_rows_perm_kernel<<<(unsigned)((n_dst + 255) / 256), 256, (size_t)n_idx * sizeof(int), st>>>(idx, n_idx, n_dst, offsets, perm);
  const size_t meta = (size_t)(n_dst + 1 + n_idx + 1) * sizeof(int);
  if (meta + (size_t)n_idx * isz > 96 * 1024) return fail(PTK_ERR_UNSUPPORTED, "ptk_put_rows: index set too large for shared memory");
  int wpb = (int)std::max<int64_t>(1, std::min<int64_t>(8, (int64_t)(96 * 1024 - meta) / (n_idx * isz)));
  size_t smem = meta + (size_t)wpb * n_idx * isz;
  PTK_CUDA(cudaFuncSetAttribute(put_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
  PTK_CUDA(cudaFuncSetAttribute(put_rows_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
  unsigned grid = (unsigned)std::min<int64_t>((outer + wpb - 1) / wpb, (int64_t)std::max(1, ptk::sm_count()) * 8);
  if (dtype == PTK_F32)
    put_rows_kernel<float><<<grid, 256, smem, st>>>((float*)dst, (const float*)y, offsets, perm, outer, n_dst, n_idx, wpb);
  else
    put_rows_kernel<double><<<grid, 256, smem, st>>>((double*)dst, (const double*)y, offsets, perm, outer, n_dst, n_idx, wpb);
  PTK_LAUNCH_CHECK("put_rows");
  return PTK_OK;
}

}  // extern "C"
