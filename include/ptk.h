/*
 * ptk.h — C-ABI of libptk.so, the H100 (sm_90a) kernel library behind pytensor.link.cuda.CUDALinker.
 *
 * Conventions (mirrors the reference's C-thunk ABI: `int (*fn)(void* data)` returning 0 on success and stashing
 * the error beside it — /root/reference/pytensor/link/c/c_code/lazylinker_c.c:498-534, link/c/basic.py:1690-1761):
 *   - every entry point returns `ptk_status` (0 = ok); the message is fetched with ptk_last_error() (thread local);
 *   - only plain pointers / integers / doubles cross the boundary — no torch, no numpy, no C++ types;
 *   - device pointers are raw `void*` (e.g. torch.Tensor.data_ptr()); the caller owns ALL memory incl. workspaces;
 *   - strides are in ELEMENTS, shapes int64; `stream` is a cudaStream_t passed as void* (0 = legacy default);
 *   - nothing here synchronises the device unless its name says so.
 *
 * Each group cites the reference interface it replaces (file:line under /root/reference/).
 */
#ifndef PTK_H
#define PTK_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int ptk_status;
#define PTK_OK 0
#define PTK_ERR_CUDA 1
#define PTK_ERR_NVRTC 2
#define PTK_ERR_ARG 3
#define PTK_ERR_UNSUPPORTED 4

/* dtype codes (numpy kinds the reference's TensorType supports, pytensor/tensor/type.py:40-55; no bf16 there) */
enum ptk_dtype {
  PTK_BOOL = 0, PTK_I8 = 1, PTK_I16 = 2, PTK_I32 = 3, PTK_I64 = 4,
  PTK_U8 = 5, PTK_U16 = 6, PTK_U32 = 7, PTK_U64 = 8,
  PTK_F16 = 9, PTK_F32 = 10, PTK_F64 = 11
};

/* ---- runtime ---------------------------------------------------------------------------------------------- */
int          ptk_version(void);
const char*  ptk_last_error(void);
/* Binds the driver API (libcuda.so.1 via cudaGetDriverEntryPoint) and queries the device. Must be called once per
 * process before any other call that touches the GPU. Fails (never falls back) when no CUDA device is present. */
ptk_status   ptk_init(int device);
int          ptk_sm_count(void);
int          ptk_device(void);
ptk_status   ptk_sync_stream(void* stream);
ptk_status   ptk_memcpy_h2d_async(void* dst_dev, const void* src_host, size_t bytes, void* stream);
ptk_status   ptk_memcpy_d2h_async(void* dst_host, const void* src_dev, size_t bytes, void* stream);
ptk_status   ptk_memcpy_d2d_async(void* dst_dev, const void* src_dev, size_t bytes, void* stream);
ptk_status   ptk_memset_async(void* dst_dev, int byte, size_t bytes, void* stream);
ptk_status   ptk_host_alloc_pinned(void** out, size_t bytes);
ptk_status   ptk_host_free_pinned(void* p);

/* ---- JIT: the per-Composite kernels (replaces the per-node g++ compile of the C linker:
 *      pytensor/link/c/cmodule.py:2454-2643 GCC_compiler.compile_str, link/c/basic.py:1585 cthunk_factory) -------- */
/* Compile CUDA C++ `src` for sm_90a with NVRTC. On success *cubin / *cubin_size receive a malloc'd image the caller
 * releases with ptk_free(). `log` (may be NULL) receives a malloc'd compile log (also on failure). */
ptk_status   ptk_jit_compile(const char* src, const char* const* opts, int n_opts,
                             void** cubin, size_t* cubin_size, char** log);
void         ptk_free(void* p);
ptk_status   ptk_module_load(const void* image, size_t size, void** module);
ptk_status   ptk_module_unload(void* module);
ptk_status   ptk_module_get_function(void* module, const char* name, void** func);
ptk_status   ptk_func_set_max_dynamic_smem(void* func, int bytes);
ptk_status   ptk_func_max_active_blocks(void* func, int block_threads, int dyn_smem, int* out);
/* flags: bit0 = cooperative launch (grid-wide barrier allowed); cluster_x > 1 launches thread-block clusters. */
ptk_status   ptk_launch(void* func, unsigned gx, unsigned gy, unsigned gz, unsigned bx, unsigned by, unsigned bz,
                        unsigned dyn_smem, void* stream, void** args, int flags, int cluster_x);

/* ---- CUDA graphs: the replayable launch list of the VM (replaces the CVM per-call interpreter loop,
 *      lazylinker_c.c:749-897 CLazyLinker_call) --------------------------------------------------------------- */
ptk_status   ptk_graph_begin_capture(void* stream);
ptk_status   ptk_graph_end_capture(void* stream, void** graph_exec);
ptk_status   ptk_graph_launch(void* graph_exec, void* stream);
ptk_status   ptk_graph_destroy(void* graph_exec);

/* ---- events (profiling: VM.call_times, pytensor/link/vm.py:243-271) ------------------------------------------- */
ptk_status   ptk_event_create(void** ev);
ptk_status   ptk_event_record(void* ev, void* stream);
ptk_status   ptk_event_elapsed_ms(void* start, void* stop, float* ms);   /* synchronises on `stop` */
ptk_status   ptk_event_destroy(void* ev);
ptk_status   ptk_stream_wait_event(void* stream, void* ev);

/* ---- data movement glue (G3/G4: DeepCopyOp compile/ops.py:121, Alloc tensor/basic.py:1545,
 *      IncSubtensor tensor/subtensor.py:1441, AdvancedSubtensor :1932, AdvancedIncSubtensor :2275) ------------ */
/* dst[idx] = src[idx] for an ndim<=8 strided pair of equal shape; itemsize in {1,2,4,8}; a 0 src stride broadcasts. */
ptk_status   ptk_copy_strided(void* dst, const int64_t* dst_strides, const void* src, const int64_t* src_strides,
                              const int64_t* shape, int ndim, int itemsize, void* stream);
/* dst[idx] (op)= src[idx]; op 0 = set (same as copy), 1 = add. dtype gives the arithmetic for add. */
ptk_status   ptk_inc_strided(void* dst, const int64_t* dst_strides, const void* src, const int64_t* src_strides,
                             const int64_t* shape, int ndim, int dtype, int op, void* stream);
/* out[o, j, i] = src[o, idx[j], i]  (take along one axis; src viewed as (outer, n_src, inner), contiguous). Bit-exact. */
ptk_status   ptk_take(void* out, const void* src, const int64_t* idx, int64_t outer, int64_t n_src, int64_t n_idx,
                      int64_t inner, int itemsize, int* err_flag, void* stream);
/* dst[o, idx[j], i] (op)= y[o, j, i]; op 0 = set, 1 = add (atomic; duplicates accumulate, order not defined —
 * np.add.at semantics up to fp reassociation, tensor/subtensor.py:2513-2531). */
ptk_status   ptk_put(void* dst, const void* y, const int64_t* idx, int64_t outer, int64_t n_dst, int64_t n_idx,
                     int64_t inner, int dtype, int op, int* err_flag, void* stream);

/* Row-batched scatter-ADD along the last axis with ONE index vector shared by all rows: dst[o, idx[j]] += y[o, j]
 * (dst (outer, n_dst) and y (outer, n_idx) contiguous; float32/float64).  A deterministic segmented reduction — sources are
 * accumulated in ascending j per destination, the same order as np.add.at (tensor/subtensor.py:2513-2531) — instead of
 * atomics.  `workspace` (ptk_put_rows_workspace_bytes) holds the CSR of `idx` built on the device each call. */
size_t       ptk_put_rows_workspace_bytes(int64_t n_dst, int64_t n_idx);
ptk_status   ptk_put_rows(void* dst, const void* y, const int64_t* idx, int64_t outer, int64_t n_dst, int64_t n_idx,
                          int dtype, void* workspace, size_t workspace_bytes, int* err_flag, void* stream);

/* Advanced indexing with k integer index arrays on k CONSECUTIVE axes (AdvancedSubtensor / AdvancedIncSubtensor,
 * tensor/subtensor.py:1932,2275; NumPy semantics :2164): out[t] = sum_j wrap(idx[j][t], dims[j]) * prod(dims[j+1:]) — the
 * row-major position inside the indexed block, which ptk_take / ptk_put then use as a single axis.  All k arrays are int64,
 * contiguous and already broadcast to n elements; an out-of-range entry sets *err_flag (checked at the call's sync). */
ptk_status   ptk_linearize_index(int k, const void* const* idx, const int64_t* dims, int64_t n, int64_t* out,
                                 int* err_flag, void* stream);

/* Boolean-mask indexing (AdvancedSubtensor / AdvancedIncSubtensor with a bool index, tensor/subtensor.py:2026-2051: the
 * reference turns the mask into `mask.nonzero()` and lets NumPy index): ascending flat positions of the non-zero bytes
 * of a contiguous mask of n bytes.  ptk_nonzero_count leaves the per-tile exclusive offsets in `workspace`
 * (ptk_nonzero_workspace_bytes(n) bytes, int64) with the TOTAL in its last int64 — the caller reads that one number back
 * (the output shape is data dependent), allocates `out[total]` and calls ptk_nonzero_fill with the same workspace. */
size_t       ptk_nonzero_workspace_bytes(int64_t n);
ptk_status   ptk_nonzero_count(const void* mask, int64_t n, void* workspace, size_t workspace_bytes, void* stream);
ptk_status   ptk_nonzero_fill(const void* mask, int64_t n, const void* workspace, int64_t* out, void* stream);

/* ---- more glue of the Op library (SURVEY.md §8(f).3) ------------------------------------------------------------
 * ARange (tensor/basic.py:3139; perform = np.arange): out[i] = first + i*delta evaluated in the output type like NumPy's
 * <type>_fill loops (first/delta = the first element and the difference of the first two, computed by the caller);
 * the float variants take first_f/delta_f, the integer variants first_i/delta_i. */
ptk_status   ptk_arange(int dtype, void* out, int64_t n, double first_f, double delta_f, int64_t first_i, int64_t delta_i,
                        void* stream);
/* Argmax (tensor/math.py:188-206): x viewed as contiguous (outer, n, inner) -> out (outer, inner) int64 = index of the
 * FIRST maximal element along the middle axis; NaN counts as maximal (np.argmax). Bit-exact. */
ptk_status   ptk_argmax(int dtype, const void* x, int64_t* out, int64_t outer, int64_t n, int64_t inner, void* stream);
/* CumOp (tensor/extra_ops.py:295-321; np.cumsum / np.cumprod along one axis): x, out contiguous (outer, n, inner);
 * op 0 = add, 1 = mul; float32/float64/int64/uint64 (the dtypes np.cumsum does not widen).  inner > 1: sequential per
 * line (bit-exact); inner == 1: warp scan (integers exact, floats within rounding). */
ptk_status   ptk_cumop(int dtype, int op, const void* x, void* out, int64_t outer, int64_t n, int64_t inner, void* stream);

/* ---- random draws (SURVEY.md §8(f).3: RandomVariable, tensor/random/op.py:49; perform :457-468 draws from a host
 *      numpy Generator) ---------------------------------------------------------------------------------------------------
 * out[i] (i < n, contiguous) = one draw of distribution `dist` with parameters p0[i*s0], p1[i*s1], p2[i*s2] (float64 device
 * arrays; stride 0 = one value for all, 1 = one per output element; NULL = the distribution's default).  Counter-based
 * Philox4x32-10 stream per element, keyed by (key, seed): same key/seed => same draws.  dist: 0 uniform(low, high),
 * 1 normal(loc, scale), 2 halfnormal(loc, scale), 3 lognormal(mean, sigma), 4 exponential(scale), 5 laplace(loc, scale),
 * 6 logistic(loc, scale), 7 gumbel(loc, scale), 8 cauchy(loc, scale), 9 bernoulli(p), 10 gamma(shape, scale),
 * 11 beta(a, b), 12 integers[low, high), 13 weibull(shape), 14 pareto(shape, scale), 15 halfcauchy(loc, scale),
 * 16 invgamma(shape, scale), 17 studentt(df, loc, scale).  The values are NOT numpy's (its PCG64 rejection samplers are
 * sequential): parity with the reference is distributional. */
ptk_status   ptk_random_fill(int dist, int dtype, void* out, int64_t n, uint64_t key, uint64_t seed, const void* p0, int64_t s0,
                             const void* p1, int64_t s1, const void* p2, int64_t s2, void* stream);

/* ---- BLAS family (A5/A6: Gemm tensor/blas/gemm.py:76, Dot22 :248, Dot22Scalar :298, Gemv tensor/blas/gemv.py:16,
 *      Ger tensor/blas/ger.py:8; the C linker calls sgemm_/dgemm_/sgemv_/dgemv_ at blas/c_code/codegen.py:463-805) */
/* C[M,N] = alpha * A[M,K] @ B[K,N] + beta * C, arbitrary element strides, dtype PTK_F32 | PTK_F64.
 * beta == 0 never reads C (so an AllocEmpty C holding NaNs is fine — gemv.py:79-86 contract).
 * precision: 0 = native (fp32/fp64 FMA, <=1e-5 rel vs BLAS), 1 = bf16 operands on wgmma tensor cores with fp32
 * accumulation (fp32 graphs only; needs `workspace` of ptk_gemm_workspace_bytes()). */
size_t       ptk_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K, int precision);
ptk_status   ptk_gemm(int dtype, int64_t M, int64_t N, int64_t K, double alpha,
                      const void* A, int64_t sa0, int64_t sa1, const void* B, int64_t sb0, int64_t sb1,
                      double beta, void* C, int64_t sc0, int64_t sc1,
                      int precision, void* workspace, size_t workspace_bytes, void* stream);
/* Fused epilogue variant used by the linker peephole K5: C = act(alpha*A@B + bias[N]) with act 0=none, 1=tanh. */
ptk_status   ptk_gemm_bias_act(int dtype, int64_t M, int64_t N, int64_t K,
                      const void* A, int64_t sa0, int64_t sa1, const void* B, int64_t sb0, int64_t sb1,
                      const void* bias, int act, void* C, int64_t sc0, int64_t sc1,
                      int precision, void* workspace, size_t workspace_bytes, void* stream);
/* Extended tensor-core entry point (fp32 graphs, bf16 operands, fp32 accumulation):
 *   C = act(alpha * A @ B + beta * C + bias[N]);
 * A comes either as fp32 (A_f32, element strides sa0/sa1; staged to bf16 in the workspace) or ALREADY staged as bf16
 * (A_bf16: row-major [M,K], pitch lda_bf16 elements (multiple of 8), 16-byte aligned) — e.g. the C_bf16 copy a previous
 * call emitted, so that a chain of layers re-stages only the weights.  C_bf16 (optional, row-major pitch ldc_bf16) receives
 * a bf16 copy of the result. */
ptk_status   ptk_gemm_tc_ex(int64_t M, int64_t N, int64_t K, double alpha, const void* A_f32, int64_t sa0, int64_t sa1,
                      const void* A_bf16, int64_t lda_bf16, const void* B_f32, int64_t sb0, int64_t sb1, double beta,
                      void* C, int64_t sc0, int64_t sc1, const void* bias, int act, void* C_bf16, int64_t ldc_bf16,
                      void* workspace, size_t workspace_bytes, void* stream);
/* fp32-ACCURATE product on the tensor cores — what mode="CUDA" runs for large fp32 Dot22 / Gemm (the reference calls sgemm_
 * here: pytensor/tensor/blas/c_code/codegen.py:463-540; parity bar <= 1e-5 vs that result):
 *   C = act(alpha * A @ B + beta * C + bias[N]),  A, B, C fp32 with arbitrary element strides.
 * Each operand is staged as THREE bf16 pieces x = x1 + x2 + x3 (24 mantissa bits in total); per 64-wide k-block the
 * wgmma kernel accumulates `terms` piece products in its fp32 register accumulator, smallest first:
 *   terms = 6: A3B1+A2B2+A1B3+A2B1+A1B2+A1B1 (only O(2^-24) products dropped: below sgemm's own rounding noise),
 *   terms = 3: A2B1+A1B2+A1B1 (about 4e-6 of the output scale at K = 4096; twice as fast).
 * workspace >= ptk_gemm_split_workspace_bytes(M, N, K), caller-owned. */
size_t       ptk_gemm_split_workspace_bytes(int64_t M, int64_t N, int64_t K);
ptk_status   ptk_gemm_tc_split(int64_t M, int64_t N, int64_t K, double alpha, const void* A_f32, int64_t sa0, int64_t sa1,
                      const void* B_f32, int64_t sb0, int64_t sb1, double beta, void* C, int64_t sc0, int64_t sc1,
                      const void* bias, int act, int terms, void* workspace, size_t workspace_bytes, void* stream);
/* Operands staged ONCE, products chained: the two halves of ptk_gemm_tc_ex / ptk_gemm_tc_split as separate entry points,
 * for operands that do not change between calls (graph constants, shared weights, the non-sequences of a Scan — the C
 * linker's sgemm_ has no such state: every call of pytensor/tensor/blas/c_code/codegen.py:463-540 reads fp32 operands) and for
 * recurrences h <- act(h @ W + b) (Scan inner graphs, scan/scan_perform.pyx:311-541) where the epilogue of step t writes
 * the staged A operand of step t+1.
 *   ptk_stage_operand: dst = `pieces` (1 = bf16 | 3 = x1+x2+x3 split) matrices [rows, cols] from fp32 src[r*sr + c*sc],
 *     row pitch ld (multiple of 8, >= cols), piece i at rows [i*piece_rows, ...); dst >= ptk_stage_bytes(rows, cols, pieces)
 *     with ld = round_up(cols, 8), piece_rows = round_up(rows, 256).  For the B operand of C = A @ B stage B^T:
 *     rows = N, cols = K, sr = B's column stride, sc = B's row stride.
 *     aligned != 0 (3 pieces, default pitches): the LEADING piece of every row is an integer multiple (|.| <= 2^b, b from `cols`) of a
 *     per-row power of two, so that the A1 x B1 products of a dot product accumulate EXACTLY in the tensor core's fp32
 *     accumulator (which truncates otherwise: a systematic shrink of ~1e-7 per MMA of the accumulation chain) — the
 *     operand layout ptk_gemm_tc_staged's exact_main mode expects for both A and B.
 *   ptk_gemm_tc_staged: C = act(alpha * A @ B + beta * C + bias[N]) from staged A [M,K] / B^T [N,K]; terms 1 (bf16
 *     operands) | 3 | 6 (fp32-accurate, see ptk_gemm_tc_split; 3 and 6 need 3-piece operands).  exact_main != 0 (both
 *     operands staged `aligned`): A1 x B1 accumulates in its own accumulator — exactly while its partial sums stay below
 *     2^24 units (always for K <= 1024; see ptk_gemm_tc.cu lead_bits_for), in chunks only beyond K = 16384; the
 *     correction products in a second one; the epilogue adds them with round-to-nearest.  C_stage (optional) receives
 *     out_pieces (1 | 3) staged pieces of the result [M,N] (pitch ldc_stage, piece pitch c_rows); out_exp != PTK_STAGE_NO_EXP
 *     aligns the leading output piece to that fixed exponent (results known to lie in [-1, 1], e.g. tanh),
 *     which makes the pieces a valid `aligned` A operand of a following exact_main product.
 *   ptk_gemm_exact_main_default: 1 unless PTK_GEMM_EXACT=0 — what ptk_gemm_tc_split uses. */
#define PTK_STAGE_NO_EXP (-100000)
size_t       ptk_stage_bytes(int64_t rows, int64_t cols, int pieces);
ptk_status   ptk_stage_operand(const void* src_f32, int64_t sr, int64_t sc, int64_t rows, int64_t cols, int pieces, int aligned,
                      void* dst, int64_t ld, int64_t piece_rows, void* stream);
ptk_status   ptk_gemm_tc_staged(int64_t M, int64_t N, int64_t K, double alpha, const void* A_stage, int64_t lda, int64_t a_rows,
                      const void* B_stage, int64_t ldb, int64_t b_rows, int terms, double beta, void* C, int64_t sc0,
                      int64_t sc1, const void* bias, int act, void* C_stage, int64_t ldc_stage, int64_t c_rows,
                      int out_pieces, int exact_main, int out_exp, void* stream);
int          ptk_gemm_exact_main_default(void);
/* Width b of the aligned leading piece for a contraction of length K (|leading integer| <= 2^b; 7 today for every K);
 * out_exp of a chained tanh epilogue feeding a product of contraction length K' is ptk_gemm_lead_bits(K') - 1. */
int          ptk_gemm_lead_bits(int64_t K);
/* A chain of L <= 96 small dense layers in one launch: h <- act_l(h @ W_l + bias_l), every K_l, N_l <= 128, N_l % 4 == 0,
 * K_l == N_(l-1), W_l contiguous row-major fp32 [K_l, N_l] (16-byte aligned), bias_l [N_l] or NULL, act_l 0 | 1 (tanh).
 * x [M, K_0] (row stride sx0, unit column stride) -> y [M, N_(L-1)] (row stride sy0).  Replaces L sgemm_ calls plus L
 * Composite{tanh(x + b)} loops of the C linker (tensor/blas/c_code/codegen.py:463-540) when the matrices are so small that
 * a launch per layer costs more than the layer: the BASELINE metric graph at n = 64. */
ptk_status   ptk_mlp_chain(const void* x, int64_t sx0, void* y, int64_t sy0, int64_t M, int L, const void* const* W,
                           const void* const* bias, const int* K, const int* N, const int* act, void* stream);
/* y[M] = alpha * A[M,N] @ x[N] + beta * y   (beta == 0 never reads y). */
ptk_status   ptk_gemv(int dtype, int64_t M, int64_t N, double alpha, const void* A, int64_t sa0, int64_t sa1,
                      const void* x, int64_t sx, double beta, void* y, int64_t sy, void* stream);
/* A[M,N] += alpha * x[M] y[N]^T */
ptk_status   ptk_ger(int dtype, int64_t M, int64_t N, double alpha, const void* x, int64_t sx,
                     const void* y, int64_t sy, void* A, int64_t sa0, int64_t sa1, void* stream);

/* ---- dense linear algebra (A8/A9: Cholesky tensor/linalg/decomposition/cholesky.py:18 (potrf :52-83),
 *      SolveTriangular tensor/linalg/solvers/triangular.py:13 (trtrs :41-71)) ------------------------------------ */
/* In-place factorisation of `batch` column-or-row-major (n,n) matrices (row-major, ld = n). lower != 0 -> L with
 * A = L L^T, the other triangle zeroed; non positive definite -> the whole matrix is NaN-filled (cholesky.py:78-80).*/
ptk_status   ptk_potrf(int dtype, void* A, int64_t n, int64_t batch, int lower, void* stream);
/* Solve op(A) X = B in place in B (n, nrhs) row-major, A (n,n) row-major; trans: 0 = A, 1 = A^T; unit_diag;
 * singular (zero diagonal) -> B NaN-filled (triangular.py:68-69). */
ptk_status   ptk_trsm(int dtype, const void* A, void* B, int64_t n, int64_t nrhs, int64_t batch,
                      int lower, int trans, int unit_diag, void* stream);

/* ---- multi-GPU exchange (SURVEY.md §8e C1; no counterpart in the reference, which has no collectives) ----------------------
 * One-shot all-reduce (sum) of a small vector (n <= nmax) over NVLink peer memory.  `peer_ptrs[world]` (host array) are the
 * addresses of every rank's symmetric buffer of ptk_allreduce_oneshot_buffer_bytes() bytes, zero-initialised once;
 * `epoch_ctr` is a zero-initialised device uint32 owned by this rank.  Collective: every rank must call it the same number of
 * times.  The result (sum in rank order, identical on all ranks) lands in `out`; no host synchronisation. */
size_t       ptk_allreduce_oneshot_buffer_bytes(int world, int64_t nmax, int itemsize);
ptk_status   ptk_allreduce_oneshot(int dtype, const void* in, void* out, int64_t n, const uint64_t* peer_ptrs, int rank,
                                   int world, int64_t nmax, void* epoch_ctr, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PTK_H */
