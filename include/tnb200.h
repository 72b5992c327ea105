/* tnb200.h — C ABI of libtnb200.so, the H100-native (sm_90a) dense contraction + split
 * engine that sits beneath the `cuda_b200` TensorNetwork backend.
 *
 * This is the drop-in boundary of SURVEY.md section 8(b): the reference's plug-in surface is
 * the Python class `AbstractBackend` (tensornetwork/backends/abstract_backend.py:22); the
 * adapter class `tensornetwork_b200.backend.CudaB200Backend` implements that class and
 * forwards every compute method to one of the entry points below through ctypes.
 * No torch / Python types appear here: plain device pointers, sizes, a cudaStream_t passed
 * as void*.  All calls are stream-ordered and asynchronous unless stated; all return 0 on
 * success or a negative tnb200_status_t, with a message available from tnb200_last_error().
 *
 * Each entry point cites the reference method it replaces (file:line relative to the
 * reference repo root).
 */
#ifndef TNB200_H_
#define TNB200_H_

#include <stdint.h>

#if defined(TNB200_BUILD)
#define TNB200_API __attribute__((visibility("default")))
#else
#define TNB200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

#define TNB200_MAX_NDIM 16
#define TNB200_ABI_VERSION 1

typedef enum {
  TNB200_OK = 0,
  TNB200_ERR_INVALID = -1,   /* bad argument / shape mismatch  -> Python ValueError   */
  TNB200_ERR_DTYPE = -2,     /* unsupported dtype combination  -> Python TypeError    */
  TNB200_ERR_CUDA = -3,      /* CUDA runtime / driver failure  -> Python RuntimeError */
  TNB200_ERR_UNSUPPORTED = -4,/* valid request this build cannot serve -> NotImplementedError */
  TNB200_ERR_NOCONV = -5     /* iterative kernel did not converge -> RuntimeError */
} tnb200_status_t;

typedef enum {
  TNB200_F64 = 0,
  TNB200_F32 = 1,
  TNB200_F16 = 2,
  TNB200_BF16 = 3,
  TNB200_C64 = 4,   /* interleaved (re, im) float  */
  TNB200_C128 = 5,  /* interleaved (re, im) double */
  TNB200_I32 = 6,
  TNB200_I64 = 7,
  TNB200_BOOL = 8   /* one byte, 0 or 1: a mask.  Only tnb200_compare (output) and tnb200_index_update (mask)
                       accept it; every other entry point refuses a bool descriptor. */
} tnb200_dtype_t;

/* A strided view of device memory.  Strides are in ELEMENTS (like torch), may be 0
 * (broadcast) and need not describe a contiguous block. */
typedef struct tnb200_tensor {
  void* data;
  int32_t dtype;
  int32_t ndim;
  int64_t shape[TNB200_MAX_NDIM];
  int64_t stride[TNB200_MAX_NDIM];
} tnb200_tensor_t;

/* flags for tnb200_tensordot */
#define TNB200_CONJ_A 0x1
#define TNB200_CONJ_B 0x2
/* math mode, bits [4,8): how fp32 / fp64 inputs use the tensor cores */
#define TNB200_MATH_DEFAULT (0 << 4) /* f64: DMMA fp64; f32: TF32 wgmma when large; 16-bit: wgmma */
#define TNB200_MATH_STRICT (1 << 4)  /* never lower the input precision (f32 -> fp32 FMA path)      */
#define TNB200_MATH_SIMT (2 << 4)    /* force the generic strided CUDA-core kernel (any dtype)     */

TNB200_API const char* tnb200_last_error(void);
TNB200_API int32_t tnb200_abi_version(void);
/* sm count, compute capability and HBM bytes of the current device */
TNB200_API int32_t tnb200_device_info(int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor,
                           int64_t* total_mem);
/* name of the kernel family the last tnb200_tensordot call on this thread dispatched to
 * ("simt", "dmma_f64", "wgmma_bf16", ...): used by tests to prove which path ran. */
TNB200_API const char* tnb200_last_kernel(void);
/* number of kernel launches issued by this library since process start (all threads) */
TNB200_API int64_t tnb200_launch_count(void);

/* ---- a1: NumPyBackend.tensordot  (backends/numpy/numpy_backend.py:35-54,
 *          AbstractBackend.tensordot abstract_backend.py:27-38), and the batched form used by
 *          NumPyBackend.matmul (:609-612) / ncon's _batch_cont (ncon_interface.py:280-354).
 * c[batch..., free_a..., free_b...] = sum over contracted axes of a * b.
 * `c` must be a preallocated tensor of that shape (any strides); transposes of a/b are fused:
 * a and b are arbitrary strided views and are never materialised unless the planner has to
 * repack an operand the TMA engine cannot address (see DESIGN.md).
 * batch_a/batch_b list `nbatch` axes of a/b that are carried, not summed (nbatch may be 0). */
TNB200_API int32_t tnb200_tensordot(const tnb200_tensor_t* a, const tnb200_tensor_t* b,
                         const tnb200_tensor_t* c, int32_t naxes, const int32_t* axes_a,
                         const int32_t* axes_b, int32_t nbatch, const int32_t* batch_a,
                         const int32_t* batch_b, int32_t flags, void* stream);

/* ---- a2 helpers: NumPyBackend.transpose/reshape materialisation (numpy_backend.py:56-62).
 * dst[i...] = (conj?) src[i...] with dtype conversion; shapes must match; any strides. */
TNB200_API int32_t tnb200_copy(const tnb200_tensor_t* src, const tnb200_tensor_t* dst, int32_t conj,
                    void* stream);

/* ---- a6: elementwise helpers (numpy_backend.py:536-575 add/sub/mul/div + broadcast_*,
 *          :89-90 sqrt, :162-163 conj, :709-730 abs/sign, :577-589 sin/cos/exp/log, :763-782 power).
 * c = a (op) b with numpy broadcasting expressed by 0-strides; all three same ndim/shape. */
typedef enum { TNB200_ADD = 0, TNB200_SUB = 1, TNB200_MUL = 2, TNB200_DIV = 3,
               TNB200_POW = 4 } tnb200_binop_t;
TNB200_API int32_t tnb200_binary(int32_t op, const tnb200_tensor_t* a, const tnb200_tensor_t* b,
                      const tnb200_tensor_t* c, void* stream);
typedef enum { TNB200_CONJ = 0, TNB200_SQRT = 1, TNB200_ABS = 2, TNB200_NEG = 3,
               TNB200_EXP = 4, TNB200_LOG = 5, TNB200_SIN = 6, TNB200_COS = 7,
               TNB200_SIGN = 8, TNB200_REAL = 9, TNB200_IMAG = 10 } tnb200_unop_t;
TNB200_API int32_t tnb200_unary(int32_t op, const tnb200_tensor_t* a, const tnb200_tensor_t* c,
                     void* stream);
/* x = alpha * x + beta  (in place; `x /= norm` of dmrg.py:225,298 and base_mps.py:172) */
TNB200_API int32_t tnb200_affine_inplace(const tnb200_tensor_t* x, double alpha_re, double alpha_im,
                              double beta_re, double beta_im, void* stream);
/* x = x * (*alpha_dev)^power, alpha read on the device (no host sync): power = -1 divides */
TNB200_API int32_t tnb200_scale_by_device_scalar(const tnb200_tensor_t* x, const void* alpha_dev,
                                      int32_t alpha_dtype, int32_t power, void* stream);
/* y += alpha * x, alpha given on host or (alpha_dev != NULL) as sign * (*alpha_dev) on device */
TNB200_API int32_t tnb200_axpy(const tnb200_tensor_t* x, const tnb200_tensor_t* y, double alpha_re,
                    double alpha_im, const void* alpha_dev, double sign, void* stream);
TNB200_API int32_t tnb200_fill(const tnb200_tensor_t* c, double re, double im, void* stream);
/* ---- elementwise comparison masks (numpy's `a <= b` etc., used by InfiniteMPS.canonicalize,
 *      matrixproductstates/infinite_mps.py:237,263).  c (TNB200_BOOL) = a (op) b with the operand conventions of
 *      tnb200_binary: same ndim and shape, broadcasting by 0-strides, a and b of one dtype.  IEEE semantics: any
 *      comparison with NaN is false.  f64 / f32 / f16 / bf16 / i32 / i64; complex: TNB200_ERR_DTYPE. */
typedef enum { TNB200_LT = 0, TNB200_LE = 1, TNB200_GT = 2, TNB200_GE = 3 } tnb200_cmpop_t;
TNB200_API int32_t tnb200_compare(int32_t op, const tnb200_tensor_t* a, const tnb200_tensor_t* b, const tnb200_tensor_t* c,
                                  void* stream);
/* ---- NumPyBackend.index_update (numpy_backend.py:548-552: t = copy(a); t[mask] = value):
 *      out = where(mask, value, a) in one strided launch.  mask (TNB200_BOOL) has a's shape (0-strides broadcast it) or
 *      is NULL, which selects every element.  The value is (re, im) from the host, or, when value_dev is not NULL, the
 *      scalar of dtype value_dtype read on the device (no host sync; an i64 scalar stored into an i64 tensor is copied
 *      exactly, so integers beyond 2^53, which a double rounds, go that way).  It is cast to a's dtype as numpy casts: a float
 *      stored into an integer tensor is truncated toward zero; a complex value into a real tensor is TNB200_ERR_DTYPE
 *      (host values: im != 0).  out has a's shape and dtype, any strides. */
TNB200_API int32_t tnb200_index_update(const tnb200_tensor_t* a, const tnb200_tensor_t* mask, double re, double im,
                                       const void* value_dev, int32_t value_dtype, const tnb200_tensor_t* out,
                                       void* stream);
/* c[i, j] = (j - i == k) — NumPyBackend.eye :110-116 */
TNB200_API int32_t tnb200_eye(const tnb200_tensor_t* c, int64_t k, void* stream);
/* standard normal fill (Philox4x32-10 + Box-Muller), NumPyBackend.randn :132-144; complex
 * dtypes get independent re/im parts.  uniform: random_uniform :146-160. */
TNB200_API int32_t tnb200_randn(const tnb200_tensor_t* c, uint64_t seed, void* stream);
TNB200_API int32_t tnb200_uniform(const tnb200_tensor_t* c, double lo, double hi, uint64_t seed,
                       void* stream);

/* ---- a6: reductions.  out is a device scalar/tensor; nothing syncs.
 * norm: Frobenius norm (numpy_backend.py:108-109) -> *out (real dtype of a: f64 for f64/c128,
 *       f32 otherwise).  dot: sum(conj?(x) * y) -> *out in a's dtype (Lanczos :503-504). */
TNB200_API int32_t tnb200_norm(const tnb200_tensor_t* a, void* out, void* stream);
TNB200_API int32_t tnb200_dot(const tnb200_tensor_t* x, const tnb200_tensor_t* y, int32_t conj_x, void* out,
                   void* stream);
/* sum over `naxes` axes (numpy_backend.py:603-607); c has the reduced axes removed */
TNB200_API int32_t tnb200_sum(const tnb200_tensor_t* a, const tnb200_tensor_t* c, int32_t naxes,
                   const int32_t* axes, void* stream);
/* trace over (axis1, axis2) with offset (numpy_backend.py:684-707); c = remaining axes */
TNB200_API int32_t tnb200_trace(const tnb200_tensor_t* a, const tnb200_tensor_t* c, int64_t offset,
                     int32_t axis1, int32_t axis2, void* stream);
/* c (n+|k|, n+|k|) = 0 except the k-th diagonal = ravel(a) (numpy_backend.py:673-682) */
TNB200_API int32_t tnb200_diagflat(const tnb200_tensor_t* a, const tnb200_tensor_t* c, int64_t k,
                        void* stream);

/* ---- a4: decompositions.svd (backends/numpy/decompositions.py:21-74).
 * Thin SVD of the m x n matrix view `a` (any strides) by one-sided Jacobi:
 *   u (m x r), s (r, real dtype, DESCENDING), vh (r x n), r = min(m, n); all preallocated and
 *   contiguous.  `info` (device int32[4], may be NULL): [0] sweeps used, [1] converged flag.
 * Truncation is a second call so the data-dependent `keep` needs exactly one D2H of an int. */
TNB200_API int32_t tnb200_svd(const tnb200_tensor_t* a, const tnb200_tensor_t* u, const tnb200_tensor_t* s,
                   const tnb200_tensor_t* vh, int32_t* info_dev, void* stream);
/* decompositions.py:38-57: keep = min(max_singular_values, #{ sqrt(cumsum(s[::-1]^2)) > eps })
 * with eps = max_truncation_error * (relative ? s[0] : 1); max_singular_values < 0 means None,
 * use_error = 0 means max_truncation_error is None.  Writes one int64 to *keep_dev. */
TNB200_API int32_t tnb200_svd_truncation_count(const tnb200_tensor_t* s, int64_t max_singular_values,
                                    int32_t use_error, double max_truncation_error,
                                    int32_t relative, int64_t* keep_dev, void* stream);

/* ---- NumPyBackend.eigh (backends/numpy/numpy_backend.py:165-166, AbstractBackend.eigh
 *      abstract_backend.py:320-330): np.linalg.eigh of the n x n view `a` (any strides) by parallel two-sided
 *      block Jacobi.  Only the lower triangle is read (LAPACK's UPLO='L'): the upper triangle is taken as its
 *      conjugate and the imaginary part of the diagonal is ignored.  w (n, real dtype, ASCENDING) and v (n x n, the
 *      input dtype, eigenvectors as columns) are preallocated, any strides.  f32 / c64 iterate in double.
 *      `info` (device int32[4], may be NULL): [0] sweeps used, [1] converged flag.  Synchronises with the host once
 *      per sweep.  Non-square: TNB200_ERR_INVALID; other dtypes: TNB200_ERR_DTYPE; no convergence: TNB200_ERR_NOCONV. */
TNB200_API int32_t tnb200_eigh(const tnb200_tensor_t* a, const tnb200_tensor_t* w, const tnb200_tensor_t* v,
                               int32_t* info_dev, void* stream);

/* ---- NumPyBackend.eigs (backends/numpy/numpy_backend.py:216-298, which hands off to scipy's ARPACK): one Arnoldi
 *      step's orthogonalisation, two passes of classical Gram-Schmidt (CGS2) of w against rows 0..j of the Krylov
 *      basis v, a row-major matrix view (rows >= j + 2, contiguous rows, any row stride; row i = Krylov vector i).
 *      Writes the normalised result into row j+1 of v, h_dev[0..j] = V[0..j]^H w (the sum of both passes) and
 *      h_dev[j+1] = beta, the norm before normalising.  h_dev holds j + 2 values of the double-precision form of the
 *      basis dtype (f64 for f64 / f32, c128 for c128 / c64).  w (contiguous, n elements, the basis dtype) is only
 *      read.  If beta <= 16 sqrt(j + 2) eps(dtype) ||w||, w lies in span(V) to rounding: row j+1 is written as zeros
 *      and beta as 0.  f64 / c128 / f32 / c64, accumulation in double, j + 1 <= 1024 (TNB200_ERR_UNSUPPORTED above).
 *      Four launches per call for any j and n, three reads of rows 0..j; no host synchronisation. */
TNB200_API int32_t tnb200_arnoldi_orth(const tnb200_tensor_t* v, int32_t j, const tnb200_tensor_t* w, void* h_dev,
                                       void* stream);

/* ---- a5: decompositions.qr / rq (decompositions.py:77-124).  Reduced QR of the m x n view
 * `a`: q (m x r), r (r x n), r = min(m, n), Householder (LAPACK geqrf sign convention) with the
 * optional non_negative_diagonal phase fix (:91-94).  rq is qr of the conjugate transpose and is
 * composed by the adapter. */
TNB200_API int32_t tnb200_qr(const tnb200_tensor_t* a, const tnb200_tensor_t* q, const tnb200_tensor_t* r,
                  int32_t non_negative_diagonal, void* stream);

/* ---- LU with partial pivoting: LAPACK getrf, as scipy.linalg.lu_factor computes it; the factorisation behind
 *      NumPyBackend.inv (numpy_backend.py:554-558).  lu_factor factors the n x n view `a` (any strides) and writes the
 *      packed factors into `lu` (n x n, any strides): unit L strictly below the diagonal, U on and above it.
 *      piv_dev[n] (device int32) receives the 0-based row interchanges in LAPACK's order (row i was swapped with row
 *      piv[i], i <= piv[i] < n); the pivot of column j is the FIRST row of largest |x| (real) or |re| + |im| (complex),
 *      with NaN treated as reference BLAS idamax / izamax treat it: a NaN on the diagonal stays the pivot, a NaN below
 *      it is never chosen, and the NaNs propagate through the factors.  Complex pivots are divided by without forming
 *      |x|^2 (Smith's algorithm), so the whole double range is safe.
 *      info_dev[0] (device int32) is set to 0, or to 1 + the index of the first pivot that is exactly zero (LAPACK's
 *      info); the factorisation still completes, as in LAPACK.
 *      Right-looking and blocked, panels of 32 columns, four launches per panel and none per column:
 *        - the panel: ONE cluster of 8 CTAs; its rows are dealt to the CTAs and held in shared memory while they fit
 *          (n - j0 <= ~6900 rows for f64, ~3400 for c128; above that the same kernel works on the panel in global
 *          memory, where it stays L2-resident).  Per column one cluster-wide exchange through distributed shared
 *          memory carries each CTA's pivot candidate (|x|, index, row) and the diagonal row; the swap, the scale and
 *          the rank-1 update of the panel are then local;
 *        - the row interchanges left and right of the panel (laswp), the U12 triangular solve, and the trailing update
 *          A22 -= L21 U12.
 *      f64 runs the trailing update on the FP64 tensor pipe (DMMA m8n8k4); c128 runs it with CUDA-core FMA.
 *      f32 / c64 are widened to f64 / c128, factored, and rounded back.  Other dtypes: TNB200_ERR_DTYPE; not square:
 *      TNB200_ERR_INVALID; n = 0: no-op.  Does not synchronise with the host. */
TNB200_API int32_t tnb200_lu_factor(const tnb200_tensor_t* a, const tnb200_tensor_t* lu, int32_t* piv_dev,
                                    int32_t* info_dev, void* stream);
/* ---- NumPyBackend.inv (numpy_backend.py:554-558, np.linalg.inv): x = a^-1, x preallocated (n x n, any strides).
 *      The factorisation above, then tnb200_lu_solve's blocked solve against the identity (the row interchanges, then
 *      forward with unit L and backward with U, 32 rows per step: a triangular solve and one update launch each, the
 *      update on DMMA for f64).  Launches:
 *      at most 8 ceil(n / 32) + 8.  info_dev[0] as for tnb200_lu_factor: nonzero means the matrix is singular and x
 *      holds no inverse.  Same dtypes and errors as tnb200_lu_factor.  Does not synchronise with the host. */
TNB200_API int32_t tnb200_inv(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int32_t* info_dev, void* stream);
/* ---- LAPACK getrs / scipy.linalg.lu_solve on tnb200_lu_factor's output: x = a^-1 b with lu (n x n) and piv_dev[n] as
 *      lu_factor wrote them; b and x are n x k, any strides (x may not overlap b).  The row interchanges on b, then the
 *      blocked forward (unit L) and backward (U) substitution of tnb200_inv, 32 rows per step.  Same dtypes, widening
 *      and errors as tnb200_lu_factor; all three of one dtype.  n = 0 or k = 0: no-op.  Does not synchronise with the
 *      host. */
TNB200_API int32_t tnb200_lu_solve(const tnb200_tensor_t* lu, const int32_t* piv_dev, const tnb200_tensor_t* b,
                                   const tnb200_tensor_t* x, void* stream);

/* ---- NumPyBackend.expm (numpy_backend.py:589-598, scipy.linalg.expm): x = exp(a) for the n x n view `a`, x
 *      preallocated n x n, any strides.  Scaling and squaring with Pade degrees 3, 5, 7, 9, 13 (Al-Mohy & Higham 2009,
 *      Algorithm 5.1) and the degree / squaring choice of scipy.sparse.linalg._matfuncs._expm with exact 1-norms.  f32 /
 *      c64 are widened to f64 / c128 and rounded back.  Any NaN or Inf in `a` gives an all-NaN x, as scipy returns.
 *      info_dev (device int32[4], may be NULL) receives {m, s, path, lu_info}: the Pade degree, the number of squarings,
 *      0 for the fused path or 1 for the blocked one, and the getrf info of the Q factorisation.
 *        - n <= TNB200_EXPM_FUSED_MAX_N: ONE launch, one CTA, no host synchronisation (capturable);
 *        - larger n: GEMMs through tnb200_tensordot's dispatch in strict mode (DMMA for f64), Q factored and solved as
 *          in tnb200_inv; the host reads the selection at most three times (once per stage that decides which power
 *          of a to form next).
 *      Other dtypes: TNB200_ERR_DTYPE; not square: TNB200_ERR_INVALID; n = 0: no-op. */
#define TNB200_EXPM_FUSED_MAX_N 48
TNB200_API int32_t tnb200_expm(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int32_t* info_dev, void* stream);

/* ---- a11: block_sparse.tensordot per-sector loop (block_sparse/blocksparsetensor.py:1094-1101).
 * For each sector q: C.data[c_map[q]] = A.data[a_map[q]].reshape(m_q,k_q) @ B.data[b_map[q]]
 * .reshape(k_q,n_q), all sectors in ONE launch.  maps are int64 element indices into the flat
 * data vectors; *_off[q] is where sector q's maps start, and they run for m_q k_q (a), k_q n_q (b)
 * and m_q n_q (c) entries, with dims holding the (m_q, k_q, n_q) triples.  Offsets need not
 * increase, and only the first nsect entries are read.  All arrays are device pointers. */
TNB200_API int32_t tnb200_blocksparse_tensordot(const void* a_data, const void* b_data, void* c_data,
                                     int32_t dtype, int32_t nsect, const int64_t* dims_dev,
                                     const int64_t* a_map_dev, const int64_t* a_off_dev,
                                     const int64_t* b_map_dev, const int64_t* b_off_dev,
                                     const int64_t* c_map_dev, const int64_t* c_off_dev,
                                     int64_t max_m, int64_t max_n, int32_t conj_b, void* stream);

/* ---- a12: the per-sector SVDs of backends/symmetric/decompositions.py:54-61 (a Python loop of
 * np.linalg.svd there): `nprob` independent small SVDs in ONE launch, one CTA per matrix, warp-shuffle
 * Jacobi in shared memory.  Problem q: A_q is m_q x n_q, row-major contiguous at a_data + a_off[q]
 * (element offsets); outputs U_q (m x r), S_q (r, real dtype, descending), Vh_q (r x n), r = min(m, n),
 * row-major at the given offsets.  dims holds (m_q, n_q) pairs.  All arrays are device pointers.
 * *status_dev (may be NULL) is set to 1 if any problem failed to converge. */
TNB200_API int32_t tnb200_svd_batched(const void* a_data, int32_t dtype, int32_t nprob, const int64_t* dims_dev,
                                      const int64_t* a_off_dev, void* u_data, const int64_t* u_off_dev, void* s_data,
                                      const int64_t* s_off_dev, void* vh_data, const int64_t* vh_off_dev,
                                      int64_t max_m, int64_t max_n, int32_t* status_dev, void* stream);

/* ---- the per-sector QRs of block_sparse/linalg.py:300-393 (a Python loop of np.linalg.qr there): `nprob` independent
 * reduced Householder QRs in ONE launch, one CTA per matrix, staged column-major in shared memory (f32 / c64 widened
 * to f64 / c128).  Problem q: A_q is m_q x n_q, row-major contiguous at a_data + a_off[q] (element offsets); dims holds
 * (m_q, n_q) pairs; r = min(m, n).  The reflectors are tnb200_qr's (LAPACK geqrf + orgqr: beta = -sign(Re alpha) |x|),
 * so each Q_q, R_q is np.linalg.qr(A_q) to rounding.  Outputs are row-major at the given offsets:
 *   adjoint = 0:  Q_q (m x r) and R_q (r x n, upper trapezoidal with explicit zeros): A_q = Q_q R_q;
 *   adjoint = 1:  the factors of A_q^H = Q' R', written as R_q = R'^H (m x r) and Q_q = Q'^H (r x n): A_q = R_q Q_q,
 *                 the block-sparse RQ of backends/symmetric/decompositions.py:234-248.
 * max_elems bounds m_q n_q over all problems and sizes the shared memory: sizeof(f64 or c128) * max_elems must not
 * exceed TNB200_QR_BATCHED_MAX_BYTES (TNB200_ERR_UNSUPPORTED; use tnb200_qr for such a problem).  A problem with
 * m_q n_q > max_elems is skipped.  All arrays are device pointers; nprob = 0 and empty problems are no-ops; no host
 * synchronisation.  Bad sizes or null pointers: TNB200_ERR_INVALID; dtypes other than f64 / f32 / c128 / c64:
 * TNB200_ERR_DTYPE.  The limit is what fits in shared memory, not a measured crossover (README: one problem alone beats
 * tnb200_qr up to n = 64 in f64 and n = 112 in c128 on an H100 80GB HBM3 at 700 W; a batch runs its problems at once). */
#define TNB200_QR_BATCHED_MAX_BYTES (200 * 1024)
TNB200_API int32_t tnb200_qr_batched(const void* a_data, int32_t dtype, int32_t nprob, const int64_t* dims_dev,
                                     const int64_t* a_off_dev, void* q_data, const int64_t* q_off_dev, void* r_data,
                                     const int64_t* r_off_dev, int64_t max_elems, int32_t adjoint, void* stream);

/* ---- f3: the int64 element maps of a block-sparse matrix view, built on the device (the reference builds them on the host
 * with numpy unique / intersect: block_sparse/blocksparse_utils.py:330-634, cached only on request, caching.py:22-88).
 * The tensor has `nlegs` stored legs; leg t has dims[t] states with SIGNED charges (flow applied, int64) at
 * charges_dev[leg_off[t] ...].  Matrix view: rows = legs order[0..partition), columns = order[partition..nlegs).
 * Output map_dev[nnz]: sector-major (ascending row charge), inside a sector row-major (rows x columns, both ascending):
 * the position in the data vector of every element — bit-identical to the reference's maps.  `split` cuts the stored legs
 * into the two groups whose states are enumerated; shift = sum of max|charge| over the legs (U(1)), modulus = N for Z_N
 * (0: U(1)); nbins = 2*shift+1 or N; tables_dev = int64 [start_right(nbins) | sect_off(nbins) | ncols(nbins)], the
 * per-charge tables the caller derives from the legs' charge histograms (charge-degeneracy arithmetic).
 * dims / leg_off / order are HOST arrays.  This is tnb200_blocksparse_maps_nsym (include/tnb200_symmetry.h) with
 * nsym = 1. */
TNB200_API int32_t tnb200_blocksparse_maps(int32_t nlegs, const int64_t* dims, const int64_t* charges_dev, const int64_t* leg_off,
                                           const int32_t* order, int32_t partition, int32_t split, int64_t modulus, int64_t shift,
                                           int32_t nbins, const int64_t* tables_dev, int64_t nnz, int64_t* map_dev, void* stream);

/* dst[i] = src[idx[i]] (gather) or dst[idx[i]] = src[i] (scatter = 1), i < n; idx is a device int64 array.
 * The fancy-index gathers of block_sparse (blocksparsetensor.py:1094-1101, symmetric decompositions.py:55). */
TNB200_API int32_t tnb200_gather(const void* src, const int64_t* idx_dev, void* dst, int64_t n, int32_t dtype,
                                 int32_t scatter, void* stream);

/* ---- a8/a9: a RUN of dependent pairwise contractions of one path (the sequential `contract_between` loop of
 * contractors/opt_einsum_paths/path_contractors.py:87-90, e.g. the MPS zipper) as ONE persistent launch.
 * Step i is the contraction tnb200_tensordot(a, b, c, ...) would perform; dep_a / dep_b name the earlier step
 * of the chain whose output `c` is this step's operand (or -1 when the operand exists before the launch).
 * Every step must be a tensor-core GEMM addressable in place (M >= 128, N >= 128, 16/32-bit float, one batch
 * mode shared by all steps, C row-major with 16-byte aligned rows); otherwise create() returns
 * TNB200_ERR_UNSUPPORTED with *first_unsupported = the first offending step, and the caller can split the run
 * around it.  When the chain as a whole is declined (too few tiles per step to fill the GPU,
 * not enough shared memory) create() returns TNB200_ERR_UNSUPPORTED with *first_unsupported = -1 and the caller
 * launches the steps one by one.  create() allocates device tables (not capturable); launch() is stream-ordered
 * and capturable; operand addresses are frozen at create(). */
typedef struct {
  tnb200_tensor_t a, b, c;
  int32_t naxes, nbatch;
  int32_t axes_a[TNB200_MAX_NDIM], axes_b[TNB200_MAX_NDIM];
  int32_t batch_a[TNB200_MAX_NDIM], batch_b[TNB200_MAX_NDIM];
  int32_t dep_a, dep_b;
} tnb200_chain_step_t;
TNB200_API int32_t tnb200_chain_create(int32_t nsteps, const tnb200_chain_step_t* steps, int32_t* first_unsupported,
                                       void** handle);
TNB200_API int32_t tnb200_chain_launch(void* handle, void* stream);
TNB200_API int32_t tnb200_chain_destroy(void* handle);

/* ---- a RUN of 2..8 thin contractions (the ramp of an MPS contraction: a small matrix, K <= 64, applied to a long
 * operand) in which step i streams step i - 1's result: ONE persistent launch that reads the first long operand once,
 * keeps every intermediate on chip and writes only the last step's result, bit-identical to launching the steps one by
 * one.  Steps are described as for tnb200_chain_create; dep_a / dep_b of step i > 0 name step i - 1 for the long
 * operand and -1 for the small one, and the `data` of an intermediate result is not used (it may be NULL).  Each
 * step must take the 16-bit thin layout tnb200_tensordot would launch for it, all in one mode, with the previous
 * result's long axis innermost (columns) or outermost (rows) in the next long axis; otherwise create() returns
 * TNB200_ERR_UNSUPPORTED with *first_unsupported = the offending step (-1 when the run is declined as a whole).
 * create() allocates a device table (not capturable); launch() is stream-ordered and capturable. */
TNB200_API int32_t tnb200_thin_run_create(int32_t nsteps, const tnb200_chain_step_t* steps, int32_t* first_unsupported,
                                          void** handle);
TNB200_API int32_t tnb200_thin_run_launch(void* handle, void* stream);
TNB200_API int32_t tnb200_thin_run_destroy(void* handle);

#ifdef __cplusplus
}
#endif
#endif /* TNB200_H_ */
