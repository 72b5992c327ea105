// qr_small.cu — tnb200_qr_batched: many small independent Householder QRs in ONE launch, one CTA per matrix
// (the per-charge-sector QRs of block_sparse/linalg.py:300-393, which the reference runs as a Python loop of
// np.linalg.qr calls).
//
// The factored matrix F (M x N) is A_q, or A_q^H when `adjoint` is set (the block-sparse RQ of
// backends/symmetric/decompositions.py:234-248 is the QR of A^H).  F is staged column-major in shared memory, so a
// warp walking a column reads consecutive words.  The column loop is LAPACK geqr2: xLARFG on column j by one warp
// (beta = -sign(Re alpha) ||x||, tau as qr.cu's qr_larfg_kernel), then H_j^H applied to the trailing columns, one warp
// per column (a dot product by lane-strided partial sums and a shuffle reduction, then the axpy).  R is copied out, and
// Q is formed in place over the reflectors by backward accumulation (LAPACK org2r / ung2r).  These are the reflectors
// and the order of operations of geqrf + orgqr at these sizes, so each problem's Q and R are np.linalg.qr's to rounding.
#include "common.cuh"
#include "wide.cuh"
#include <math.h>

namespace tnb {

// tau of at most sqrt(TNB200_QR_BATCHED_MAX_BYTES / 8) = 160 reflectors: K^2 <= m n
constexpr int QR_SMALL_KMAX = 256;

// H x for the column x (rows j..M-1) of W, H = I - t v v^H, v = [1; W[j+1:, j]]; one warp
template <typename T>
__device__ __forceinline__ void qr_small_reflect(const T* __restrict__ v, T* __restrict__ x, int M, int j, T t, int lane) {
  T acc = lane == 0 ? x[j] : zero_<T>();
  for (int i = j + 1 + lane; i < M; i += 32) fmacc(acc, cj(v[i]), x[i]);
  const T w = mul(warp_sum(acc), t);
  if (lane == 0) x[j] = sub(x[j], w);
  for (int i = j + 1 + lane; i < M; i += 32) x[i] = sub(x[i], mul(w, v[i]));
}

// Shared memory: W[N][M], column c of F at W + c M.  Outputs, row-major at the caller's offsets:
//   adjoint = 0:  Q = Q_F (m x r),  R = R_F (r x n)
//   adjoint = 1:  R = R_F^H (m x r), Q = Q_F^H (r x n)      (F = A^H = Q_F R_F, so A = R_F^H Q_F^H)
template <typename Tin>
__global__ void __launch_bounds__(256) qr_small_kernel(const Tin* __restrict__ a_data, const long long* __restrict__ dims,
                                                       const long long* __restrict__ a_off, Tin* __restrict__ q_data,
                                                       const long long* __restrict__ q_off, Tin* __restrict__ r_data,
                                                       const long long* __restrict__ r_off, long long max_elems, int adjoint) {
  using T = typename Wide<Tin>::T;
  extern __shared__ __align__(16) unsigned char sm_raw[];
  __shared__ T tau[QR_SMALL_KMAX];
  const int p = blockIdx.x;
  const long long m = dims[2 * p], n = dims[2 * p + 1];
  if (m == 0 || n == 0 || m * n > max_elems) return;     // the shared memory was sized from max_elems
  const int M = (int)(adjoint ? n : m), N = (int)(adjoint ? m : n), K = M < N ? M : N;
  T* W = (T*)sm_raw;
  const Tin* A = a_data + a_off[p];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;

  // stage F, reading A in its row-major order: F[i][c] = A[i][c] (W[c M + i]), or F[b][a] = conj(A[a][b]) (W[a M + b])
  for (int idx = tid; idx < M * N; idx += blockDim.x) {
    const T a = widen(A[idx]);
    if (adjoint) W[idx] = cj(a);
    else W[(size_t)(idx % N) * M + idx / N] = a;
  }
  __syncthreads();

  // geqr2
  for (int j = 0; j < K; ++j) {
    T* col = W + (size_t)j * M;
    if (warp == 0) {
      double s2 = 0.0;
      for (int i = j + 1 + lane; i < M; i += 32) s2 += ab2(col[i]);
      s2 = warp_sum(s2);
      const T alpha = col[j];
      T t = zero_<T>();
      if (s2 != 0.0 || im_(alpha) != 0.0) {
        const double nrm = sqrt(ab2(alpha) + s2);
        const double beta = re_(alpha) >= 0.0 ? -nrm : nrm;
        const T scale = divz(one_<T>(), sub(alpha, mk(beta, 0.0, (T*)nullptr)));
        for (int i = j + 1 + lane; i < M; i += 32) col[i] = mul(col[i], scale);
        t = mk((beta - re_(alpha)) / beta, -im_(alpha) / beta, (T*)nullptr);
        if (lane == 0) col[j] = mk(beta, 0.0, (T*)nullptr);
      }
      if (lane == 0) tau[j] = t;
    }
    __syncthreads();
    const T tc = cj(tau[j]);
    if (re_(tc) != 0.0 || im_(tc) != 0.0)
      for (int c = j + 1 + warp; c < N; c += nwarps) qr_small_reflect(col, W + (size_t)c * M, M, j, tc, lane);
    __syncthreads();
  }

  // R_F = the upper trapezoid of rows 0..K-1
  if (!adjoint) {
    Tin* R = r_data + r_off[p];
    for (int idx = tid; idx < K * N; idx += blockDim.x) {
      const int i = idx / N, c = idx % N;
      narrow(R + idx, i <= c ? W[(size_t)c * M + i] : zero_<T>());
    }
  } else {
    Tin* R = r_data + r_off[p];                                     // R_F^H: N x K
    for (int idx = tid; idx < N * K; idx += blockDim.x) {
      const int c = idx / K, i = idx % K;
      narrow(R + idx, i <= c ? cj(W[(size_t)c * M + i]) : zero_<T>());
    }
  }
  __syncthreads();

  // org2r: Q_F = H_0 H_1 ... H_{K-1} [I_K; 0], accumulated backwards in columns 0..K-1 of W
  for (int j = K - 1; j >= 0; --j) {
    T* col = W + (size_t)j * M;
    const T t = tau[j];
    if (re_(t) != 0.0 || im_(t) != 0.0)
      for (int c = j + 1 + warp; c < K; c += nwarps) qr_small_reflect(col, W + (size_t)c * M, M, j, t, lane);
    __syncthreads();
    const T mt = mulr(t, -1.0);
    for (int i = tid; i < M; i += blockDim.x) col[i] = i < j ? zero_<T>() : (i == j ? sub(one_<T>(), t) : mul(mt, col[i]));
    __syncthreads();
  }

  Tin* Q = q_data + q_off[p];
  if (!adjoint) {
    for (int idx = tid; idx < M * K; idx += blockDim.x) narrow(Q + idx, W[(size_t)(idx % K) * M + idx / K]);
  } else {
    for (int idx = tid; idx < K * M; idx += blockDim.x) narrow(Q + idx, cj(W[idx]));     // Q_F^H: K x M
  }
}

template <typename Tin>
static int launch_qr_small(const void* a, int nprob, const int64_t* dims, const int64_t* a_off, void* q, const int64_t* q_off,
                           void* r, const int64_t* r_off, int64_t max_elems, int adjoint, cudaStream_t st) {
  using T = typename Wide<Tin>::T;
  const size_t smem = sizeof(T) * (size_t)max_elems;
  if (smem > TNB200_QR_BATCHED_MAX_BYTES) return TNB200_ERR_UNSUPPORTED;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(qr_small_kernel<Tin>, cudaFuncAttributeMaxDynamicSharedMemorySize, TNB200_QR_BATCHED_MAX_BYTES);
    if (e != cudaSuccess) { set_error("qr_batched: cannot raise dynamic smem: %s", cudaGetErrorString(e)); return TNB200_ERR_CUDA; }
    attr = true;
  }
  qr_small_kernel<Tin><<<nprob, 256, smem, st>>>((const Tin*)a, (const long long*)dims, (const long long*)a_off, (Tin*)q,
                                                 (const long long*)q_off, (Tin*)r, (const long long*)r_off, (long long)max_elems,
                                                 adjoint);
  TNB_LAUNCH_CHECK();
  count_launch();
  return 0;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_qr_batched(const void* a_data, int32_t dtype, int32_t nprob, const int64_t* dims_dev, const int64_t* a_off_dev,
                                     void* q_data, const int64_t* q_off_dev, void* r_data, const int64_t* r_off_dev, int64_t max_elems,
                                     int32_t adjoint, void* stream) {
  TNB_REQUIRE(nprob >= 0 && max_elems >= 0 && (adjoint == 0 || adjoint == 1), TNB200_ERR_INVALID, "qr_batched: bad sizes or flag");
  if (nprob == 0 || max_elems == 0) return 0;
  TNB_REQUIRE(a_data && dims_dev && a_off_dev && q_data && q_off_dev && r_data && r_off_dev, TNB200_ERR_INVALID,
              "qr_batched: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  set_kernel_name("qr_small_batched");
  int rc;
  switch (dtype) {
    case TNB200_F64: rc = launch_qr_small<double>(a_data, nprob, dims_dev, a_off_dev, q_data, q_off_dev, r_data, r_off_dev, max_elems, adjoint, st); break;
    case TNB200_F32: rc = launch_qr_small<float>(a_data, nprob, dims_dev, a_off_dev, q_data, q_off_dev, r_data, r_off_dev, max_elems, adjoint, st); break;
    case TNB200_C128: rc = launch_qr_small<cuDoubleComplex>(a_data, nprob, dims_dev, a_off_dev, q_data, q_off_dev, r_data, r_off_dev, max_elems, adjoint, st); break;
    case TNB200_C64: rc = launch_qr_small<cuFloatComplex>(a_data, nprob, dims_dev, a_off_dev, q_data, q_off_dev, r_data, r_off_dev, max_elems, adjoint, st); break;
    default: set_error("qr_batched: dtype %s is not supported", dtype_name(dtype)); return TNB200_ERR_DTYPE;
  }
  if (rc == TNB200_ERR_UNSUPPORTED)
    set_error("qr_batched: a problem of %lld elements is over TNB200_QR_BATCHED_MAX_BYTES; use tnb200_qr", (long long)max_elems);
  return rc;
}
