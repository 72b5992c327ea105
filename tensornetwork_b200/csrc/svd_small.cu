// svd_small.cu — tnb200_svd_batched: many small independent SVDs in ONE launch, one CTA per matrix
// (the per-charge-sector SVDs of backends/symmetric/decompositions.py:54-61, which the reference runs
// as a Python loop of np.linalg.svd calls).
//
// One-sided Jacobi with warp-shuffle Givens sweeps: the matrix is staged into shared memory as a set
// of `nv` vectors of length `len` (the rows of A when m <= n, its columns otherwise — whichever gives
// fewer, longer vectors), each vector contiguous so that every warp access is conflict-free.  A round
// of the round-robin tournament gives nv/2 disjoint vector pairs; each warp takes pairs, computes
// |x|^2, |y|^2 and <x, y> with lane-strided partial sums + __shfl_xor reductions, derives the plane
// rotation (complex-capable) and applies it to the two vectors and to the accumulated right factor.
// Converged when every pair is orthogonal to 4 sqrt(len) eps.  sigma = vector norms, sorted by rank
// counting; factors are written straight into the caller's packed U / S / Vh buffers.
#include "common.cuh"
#include "wide.cuh"
#include <math.h>

namespace tnb {

template <typename R> __device__ __forceinline__ void narrow_real(R* p, double v) { *p = (R)v; }

// Tin: storage type, R: its real type (for s).  Shared memory: X[nv][len] | V[nv][nv] | sig[nv] | rank[nv]
template <typename Tin, typename R>
__global__ void __launch_bounds__(256) svd_small_kernel(const Tin* __restrict__ a_data, const long long* __restrict__ dims,
                                                        const long long* __restrict__ a_off, Tin* __restrict__ u_data,
                                                        const long long* __restrict__ u_off, R* __restrict__ s_data,
                                                        const long long* __restrict__ s_off, Tin* __restrict__ vh_data,
                                                        const long long* __restrict__ vh_off, int* __restrict__ status) {
  using T = typename Wide<Tin>::T;
  extern __shared__ __align__(16) unsigned char sm_raw[];
  const int q = blockIdx.x;
  const int m = (int)dims[2 * q], n = (int)dims[2 * q + 1];
  if (m == 0 || n == 0) return;
  const bool rows_are_vectors = m <= n;         // orthogonalise the rows of A (vectors of length n)
  const int nv = rows_are_vectors ? m : n, len = rows_are_vectors ? n : m;
  const int nvp = (nv + 1) & ~1;                // tournament needs an even number of players
  T* X = (T*)sm_raw;                            // [nvp][len]
  T* V = X + (size_t)nvp * len;                 // [nvp][nvp], V[j][:] = coefficients of vector j
  double* sig = (double*)(V + (size_t)nvp * nvp);
  int* rank = (int*)(sig + nvp);
  __shared__ unsigned int offmax;
  const Tin* A = a_data + a_off[q];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nwarps = blockDim.x >> 5;

  // stage: X[v][i] = A[v][i] (rows) or conj-free transpose A[i][v] (columns); pad vector is zero
  for (int idx = tid; idx < nvp * len; idx += blockDim.x) {
    int v = idx / len, i = idx % len;
    T val = zero_<T>();
    if (v < nv) val = rows_are_vectors ? cj(widen(A[(size_t)v * n + i])) : widen(A[(size_t)i * n + v]);
    X[idx] = val;
  }
  for (int idx = tid; idx < nvp * nvp; idx += blockDim.x) V[idx] = (idx / nvp == idx % nvp) ? one_<T>() : zero_<T>();
  __syncthreads();
  // Work matrix M (len x nv) has the staged vectors as columns: M = A (columns) or A^H (rows).
  const double tol = 4.0 * sqrt((double)len) * 2.220446049250313e-16;
  int sweep = 0, converged = 0;
  for (; sweep < 60 && !converged; ++sweep) {
    if (tid == 0) offmax = 0u;
    __syncthreads();
    for (int round = 0; round < nvp - 1; ++round) {
      for (int pr = warp; pr < nvp / 2; pr += nwarps) {
        const int mm = nvp - 1;
        int p, r2;
        if (pr == 0) { p = mm; r2 = round % mm; } else { p = (round + pr) % mm; r2 = (round - pr + mm) % mm; }
        if (p > r2) { int t = p; p = r2; r2 = t; }
        T* x = X + (size_t)p * len;
        T* y = X + (size_t)r2 * len;
        double a = 0.0, b = 0.0;
        T g = zero_<T>();
        for (int i = lane; i < len; i += 32) { T xi = x[i], yi = y[i]; a += ab2(xi); b += ab2(yi); fmacc(g, cj(xi), yi); }
        a = warp_sum(a); b = warp_sum(b); g = warp_sum(g);
        const double mag = sqrt(ab2(g));
        if (a > 0.0 && b > 0.0) {
          const float rel = (float)(mag / sqrt(a * b));
          if (lane == 0) atomicMax(&offmax, __float_as_uint(rel));
          if ((double)rel > tol) {
            const T e = unit_conj_phase(g);                 // e^{-i phi}
            const double tau = (b - a) / (2.0 * mag);
            const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
            const double c = 1.0 / sqrt(1.0 + t * t), s = t * c;
            for (int i = lane; i < len; i += 32) {
              T xi = x[i], yi = mul(e, y[i]);
              x[i] = sub(mulr(xi, c), mulr(yi, s)); y[i] = add(mulr(xi, s), mulr(yi, c));
            }
            T* vx = V + (size_t)p * nvp;
            T* vy = V + (size_t)r2 * nvp;
            for (int i = lane; i < nvp; i += 32) {
              T xi = vx[i], yi = mul(e, vy[i]);
              vx[i] = sub(mulr(xi, c), mulr(yi, s)); vy[i] = add(mulr(xi, s), mulr(yi, c));
            }
          }
        }
      }
      __syncthreads();
    }
    if (__uint_as_float(offmax) <= (float)tol) converged = 1;
    __syncthreads();
  }
  // singular values and their descending rank
  for (int v = warp; v < nvp; v += nwarps) {
    double a = 0.0;
    for (int i = lane; i < len; i += 32) a += ab2(X[(size_t)v * len + i]);
    a = warp_sum(a);
    if (lane == 0) sig[v] = v < nv ? sqrt(a) : -1.0;   // the pad vector sorts last
  }
  __syncthreads();
  for (int v = tid; v < nvp; v += blockDim.x) {
    int r = 0;
    const double sv = sig[v];
    for (int j = 0; j < nvp; ++j) r += (sig[j] > sv) || (sig[j] == sv && j < v);
    rank[v] = r;
  }
  __syncthreads();
  // M = Xn S V^H with Xn = normalised vectors (len x nv), V[j][:] the j-th column of the right factor.
  //   columns case (M = A):    U[i][k] = Xn_j[i],  Vh[k][c] = conj(V_j[c])
  //   rows case    (M = A^H):  A = V S Xn^H  ->  U[r][k] = V_j[r],  Vh[k][i] = conj(Xn_j[i])
  const int r_out = nv;
  Tin* U = u_data + u_off[q];
  R* S = s_data + s_off[q];
  Tin* Vh = vh_data + vh_off[q];
  for (int v = 0; v < nv; ++v) {
    const int k = rank[v];
    if (k >= r_out) continue;
    const double sg = sig[v], inv = sg > 0.0 ? 1.0 / sg : 0.0;
    if (tid == 0) narrow_real<R>(S + k, sg);
    for (int i = tid; i < len; i += blockDim.x) {
      T xn = mulr(X[(size_t)v * len + i], inv);
      if (rows_are_vectors) narrow(Vh + (size_t)k * n + i, cj(xn)); else narrow(U + (size_t)i * r_out + k, xn);
    }
    for (int c2 = tid; c2 < nv; c2 += blockDim.x) {
      T vv = V[(size_t)v * nvp + c2];
      if (rows_are_vectors) narrow(U + (size_t)c2 * r_out + k, vv); else narrow(Vh + (size_t)k * n + c2, cj(vv));
    }
  }
  if (tid == 0 && !converged && status) atomicExch(status, 1);
}

template <typename Tin, typename R>
static int launch_small(const void* a, int nprob, const int64_t* dims, const int64_t* a_off, void* u, const int64_t* u_off, void* s,
                        const int64_t* s_off, void* vh, const int64_t* vh_off, int64_t max_m, int64_t max_n, int* status, cudaStream_t st) {
  using T = typename Wide<Tin>::T;
  const int64_t nv = max_m < max_n ? max_m : max_n, len = max_m < max_n ? max_n : max_m;
  const int64_t nvp = (nv + 1) & ~1LL;
  const size_t smem = sizeof(T) * (size_t)(nvp * len + nvp * nvp) + sizeof(double) * nvp + sizeof(int) * nvp + 16;
  if (smem > 200 * 1024) return TNB200_ERR_UNSUPPORTED;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(svd_small_kernel<Tin, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) { set_error("svd_batched: cannot raise dynamic smem: %s", cudaGetErrorString(e)); return TNB200_ERR_CUDA; }
    attr = true;
  }
  svd_small_kernel<Tin, R><<<nprob, 256, smem, st>>>((const Tin*)a, (const long long*)dims, (const long long*)a_off, (Tin*)u,
                                                     (const long long*)u_off, (R*)s, (const long long*)s_off, (Tin*)vh,
                                                     (const long long*)vh_off, status);
  TNB_LAUNCH_CHECK();
  count_launch();
  return 0;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_svd_batched(const void* a_data, int32_t dtype, int32_t nprob, const int64_t* dims_dev, const int64_t* a_off_dev,
                                      void* u_data, const int64_t* u_off_dev, void* s_data, const int64_t* s_off_dev, void* vh_data,
                                      const int64_t* vh_off_dev, int64_t max_m, int64_t max_n, int32_t* status_dev, void* stream) {
  TNB_REQUIRE(nprob >= 0 && max_m >= 0 && max_n >= 0, TNB200_ERR_INVALID, "svd_batched: bad sizes");
  if (nprob == 0 || max_m == 0 || max_n == 0) return 0;
  TNB_REQUIRE(a_data && dims_dev && a_off_dev && u_data && u_off_dev && s_data && s_off_dev && vh_data && vh_off_dev,
              TNB200_ERR_INVALID, "svd_batched: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  set_kernel_name("svd_small_batched");
  int rc;
  switch (dtype) {
    case TNB200_F64: rc = launch_small<double, double>(a_data, nprob, dims_dev, a_off_dev, u_data, u_off_dev, s_data, s_off_dev, vh_data, vh_off_dev, max_m, max_n, status_dev, st); break;
    case TNB200_F32: rc = launch_small<float, float>(a_data, nprob, dims_dev, a_off_dev, u_data, u_off_dev, s_data, s_off_dev, vh_data, vh_off_dev, max_m, max_n, status_dev, st); break;
    case TNB200_C128: rc = launch_small<cuDoubleComplex, double>(a_data, nprob, dims_dev, a_off_dev, u_data, u_off_dev, s_data, s_off_dev, vh_data, vh_off_dev, max_m, max_n, status_dev, st); break;
    case TNB200_C64: rc = launch_small<cuFloatComplex, float>(a_data, nprob, dims_dev, a_off_dev, u_data, u_off_dev, s_data, s_off_dev, vh_data, vh_off_dev, max_m, max_n, status_dev, st); break;
    default: set_error("svd_batched: dtype %s is not supported", dtype_name(dtype)); return TNB200_ERR_DTYPE;
  }
  if (rc == TNB200_ERR_UNSUPPORTED) set_error("svd_batched: a %lld x %lld problem does not fit shared memory; use tnb200_svd", (long long)max_m, (long long)max_n);
  return rc;
}
