// eigh.cu — tnb200_eigh: Hermitian eigendecomposition by parallel two-sided block Jacobi (np.linalg.eigh in
// backends/numpy/numpy_backend.py:165-166; LAPACK syevd / heevd there, which read the lower triangle).
//
// The lower triangle of the input is expanded into a Hermitian, column-major working copy A padded to np = 32 k
// (pad rows and columns zero), V = I.  Indices are grouped in nb = np / SB blocks; a sweep is the round-robin
// tournament of svd.cu on those blocks (nb - 1 rounds of nb / 2 disjoint pairs of PB = 2 SB indices), and one
// round is three launches:
//   1. eig    : diagonalise the PB x PB principal block S_p of every pair p in shared memory (the rotation sweeps of
//               jacobi.cuh) -> Q_p; the rotated S_p is written back as the new diagonal tile
//   2. tile   : every off-diagonal tile (p, k), p < k:  T = Q_p^H A[p, k] Q_k  -> (p, k), T^H -> (k, p)
//   3. update : V[:, pair p] <- V[:, pair p] Q_p
// A pad index has exactly zero coupling to everything, so its rotation is the identity and it never mixes with the
// matrix.  Converged when no pair of a sweep had an off-diagonal above a few eps * ||A||_F before its rotation;
// then w = diag(A) and the columns of V are sorted in ascending order of w by a rank-counting kernel.
#include "common.cuh"
#include "cplx.cuh"
#include "jacobi.cuh"
#include <math.h>

namespace tnb {

int copy_strided(const tnb200_tensor_t* src, const tnb200_tensor_t* dst, int conj, cudaStream_t st);

// A (np x np, column-major) = the Hermitian matrix whose lower triangle is a's: A[i, j] = a[i, j] (i > j),
// conj(a[j, i]) (i < j), real(a[i, i]) on the diagonal; zero outside n x n.  V = I.
template <typename T>
__global__ void eigh_init_kernel(const T* __restrict__ a, int64_t s0, int64_t s1, int n, int np, T* __restrict__ A, T* __restrict__ V) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= (int64_t)np * np) return;
  const int i = (int)(idx % np), j = (int)(idx / np);
  T x = zero_<T>();
  if (i < n && j < n) {
    if (i > j) x = a[i * s0 + j * s1];
    else if (i < j) x = cj(a[j * s0 + i * s1]);
    else x = mk(re_(a[i * s0 + i * s1]), 0.0, (T*)nullptr);
  }
  A[idx] = x;
  V[idx] = i == j ? one_<T>() : zero_<T>();
}

// ||A||_F: squared column norms, then their sum in a fixed order (one CTA), so the convergence test is reproducible
template <typename T>
__global__ void eigh_colsq_kernel(const T* __restrict__ A, int np, double* __restrict__ colsq) {
  const int j = blockIdx.x;
  double acc = 0.0;
  for (int i = threadIdx.x; i < np; i += blockDim.x) acc += ab2(A[(int64_t)j * np + i]);
  __shared__ double red[8];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    colsq[j] = t;
  }
}
__global__ void eigh_fnorm_kernel(const double* __restrict__ colsq, int np, double* __restrict__ fnorm) {
  double acc = 0.0;
  for (int j = threadIdx.x; j < np; j += blockDim.x) acc += colsq[j];
  __shared__ double red[8];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    *fnorm = sqrt(t);
  }
}

// One CTA per pair: diagonalise S_p = A[pair p, pair p] -> Q_p (row-major PB x PB), write the rotated S_p back
// (Hermitian: lower triangle mirrored, real diagonal), record the largest |s_ij| / ||A||_F seen BEFORE rotating.
// The measure is absolute: a relative one, |s_ij|^2 / (s_ii s_jj) as in the SVD's Gram matrix, has no meaning for an
// indefinite matrix.  Dynamic shared memory: eig_smem_bytes<T>().
template <typename T>
__global__ void __launch_bounds__(256) eigh_eig_kernel(T* __restrict__ A, int np, int nb, int round, const double* __restrict__ fnorm,
                                                       T* __restrict__ Qout, unsigned int* conv, double tol, int max_inner) {
  constexpr int LD = PB + 1;
  extern __shared__ __align__(16) unsigned char eigh_smem[];
  T* g = reinterpret_cast<T*>(eigh_smem);
  T* rm = g + PB * LD;
  double* cs = reinterpret_cast<double*>(rm + PB * LD);
  double* sn = cs + SB;
  T* ph = reinterpret_cast<T*>(sn + SB);
  int* pp = reinterpret_cast<int*>(ph + SB);
  int* qq = pp + SB;
  __shared__ float red[8];
  __shared__ float offmax;
  const int pair = blockIdx.x, tid = threadIdx.x;
  int bi, bj;
  rr_pair(nb, round, pair, bi, bj);
  for (int idx = tid; idx < PB * PB; idx += 256) {
    const int i = idx % PB, j = idx / PB;       // consecutive threads -> consecutive rows of A
    g[i * LD + j] = A[(int64_t)pair_col(bi, bj, j) * np + pair_col(bi, bj, i)];
    rm[i * LD + j] = i == j ? one_<T>() : zero_<T>();
  }
  const double inv = *fnorm > 0.0 ? 1.0 / *fnorm : 0.0;
  __syncthreads();
  for (int sweep = 0; sweep < max_inner; ++sweep) {
    float loc = 0.f;
    for (int idx = tid; idx < PB * PB; idx += 256) {
      const int i = idx / PB, j = idx % PB;
      if (i < j) loc = fmaxf(loc, (float)(mag_(g[i * LD + j]) * inv));
    }
    for (int o = 16; o > 0; o >>= 1) loc = fmaxf(loc, __shfl_xor_sync(0xffffffffu, loc, o));
    if ((tid & 31) == 0) red[tid >> 5] = loc;
    __syncthreads();
    if (tid == 0) {
      float m = 0.f;
      for (int w = 0; w < 8; ++w) m = fmaxf(m, red[w]);
      offmax = m;
      if (sweep == 0) atomicMax(conv, __float_as_uint(m));
    }
    __syncthreads();
    if (offmax <= (float)tol) break;
    jacobi_sweep(g, rm, cs, sn, ph, pp, qq);
  }
  for (int idx = tid; idx < PB * PB; idx += 256) {
    const int i = idx % PB, j = idx / PB;
    const T x = i > j ? g[i * LD + j] : (i < j ? cj(g[j * LD + i]) : mk(re_(g[i * LD + i]), 0.0, (T*)nullptr));
    A[(int64_t)pair_col(bi, bj, j) * np + pair_col(bi, bj, i)] = x;
  }
  T* qo = Qout + (int64_t)pair * PB * PB;
  for (int idx = tid; idx < PB * PB; idx += 256) qo[idx] = rm[(idx / PB) * LD + idx % PB];
}

// One CTA per off-diagonal tile (p, k), p < k, of the round's pair partition (blockIdx.x enumerates them row by
// row of k): T = Q_p^H A[p, k] Q_k, written to (p, k) and T^H to (k, p), so A stays exactly Hermitian and only half
// of the tiles are computed.  Thread: row i = tid % 32 of the tile, columns j = tid / 32 + 8 c.
template <typename T>
__global__ void __launch_bounds__(256) eigh_tile_kernel(T* __restrict__ A, int np, int nb, int round, const T* __restrict__ Q) {
  constexpr int LD = PB + 1, CPT = PB * PB / 256;
  __shared__ T qs[PB][LD], xs[PB][LD];
  const int64_t t = blockIdx.x;
  int k = (int)((1.0 + sqrt(1.0 + 8.0 * (double)t)) * 0.5);
  while ((int64_t)k * (k - 1) / 2 > t) --k;
  while ((int64_t)(k + 1) * k / 2 <= t) ++k;
  const int p = (int)(t - (int64_t)k * (k - 1) / 2);
  int pi, pj, ki, kj;
  rr_pair(nb, round, p, pi, pj);
  rr_pair(nb, round, k, ki, kj);
  const int tid = threadIdx.x, i = tid & (PB - 1), j0 = tid / PB;
  const T* qp = Q + (int64_t)p * PB * PB;
  const T* qk = Q + (int64_t)k * PB * PB;
  for (int idx = tid; idx < PB * PB; idx += 256) {
    const int r = idx % PB, c = idx / PB;
    xs[r][c] = A[(int64_t)pair_col(ki, kj, c) * np + pair_col(pi, pj, r)];
    qs[idx / PB][idx % PB] = qk[idx];
  }
  __syncthreads();
  T acc[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) acc[c] = zero_<T>();
#pragma unroll 8
  for (int l = 0; l < PB; ++l) {
    const T x = xs[i][l];
#pragma unroll
    for (int c = 0; c < CPT; ++c) fmacc(acc[c], x, qs[l][j0 + 8 * c]);      // Y = X Q_k
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < CPT; ++c) xs[i][j0 + 8 * c] = acc[c];
  for (int idx = tid; idx < PB * PB; idx += 256) qs[idx / PB][idx % PB] = qp[idx];
  __syncthreads();
#pragma unroll
  for (int c = 0; c < CPT; ++c) acc[c] = zero_<T>();
#pragma unroll 8
  for (int l = 0; l < PB; ++l) {
    const T q = cj(qs[l][i]);
#pragma unroll
    for (int c = 0; c < CPT; ++c) fmacc(acc[c], q, xs[l][j0 + 8 * c]);      // T = Q_p^H Y
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    const int j = j0 + 8 * c;
    A[(int64_t)pair_col(ki, kj, j) * np + pair_col(pi, pj, i)] = acc[c];
    xs[i][j] = acc[c];
  }
  __syncthreads();
  // (k, p) = T^H, row i of it is column i of T: read transposed from shared memory so the stores stay coalesced
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    const int j = j0 + 8 * c;
    A[(int64_t)pair_col(pi, pj, j) * np + pair_col(ki, kj, i)] = cj(xs[j][i]);
  }
}

// w[j] = real(A[j, j]) for the n matrix indices (never the pads: a singular input has zero eigenvalues too)
template <typename T>
__global__ void eigh_diag_kernel(const T* __restrict__ A, int np, int n, double* __restrict__ w) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) w[j] = re_(A[(int64_t)j * np + j]);
}
// ascending rank by counting (stable: ties keep index order)
__global__ void eigh_rank_kernel(const double* __restrict__ w, int n, int* __restrict__ rank) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double wj = w[j];
  int r = 0;
  for (int i = 0; i < n; ++i) { const double wi = w[i]; r += (wi < wj) || (wi == wj && i < j); }
  rank[j] = r;
}
// one CTA per eigenpair j: w_out[rank j] = w[j], v[:, rank j] = V[:n, j]
template <typename T>
__global__ void eigh_finalize_kernel(const T* __restrict__ V, const double* __restrict__ w, const int* __restrict__ rank, int n, int np,
                                     double* __restrict__ wo, int64_t w_s0, T* __restrict__ v, int64_t v_s0, int64_t v_s1) {
  const int j = blockIdx.x;
  const int k = rank[j];
  if (threadIdx.x == 0) wo[(int64_t)k * w_s0] = w[j];
  for (int i = threadIdx.x; i < n; i += blockDim.x) v[(int64_t)i * v_s0 + (int64_t)k * v_s1] = V[(int64_t)j * np + i];
}

template <typename T>
static int eigh_real(const tnb200_tensor_t* a, const tnb200_tensor_t* w, const tnb200_tensor_t* v, int32_t* info_dev, cudaStream_t st) {
  const int n = (int)a->shape[0];
  const int np = (n + PB - 1) / PB * PB;
  const int nb = np / SB, npairs = nb / 2, rounds = nb - 1;
  const int ntiles = npairs * (npairs - 1) / 2;
  T *A = nullptr, *V = nullptr, *Q = nullptr;
  double *colsq = nullptr, *fnorm = nullptr, *wd = nullptr;
  int* rank = nullptr;
  unsigned int* conv = nullptr;
  int rc;
  if ((rc = ws_alloc((void**)&A, sizeof(T) * (size_t)np * np, st))) return rc;
  if ((rc = ws_alloc((void**)&V, sizeof(T) * (size_t)np * np, st))) return rc;
  if ((rc = ws_alloc((void**)&Q, sizeof(T) * (size_t)npairs * PB * PB, st))) return rc;
  if ((rc = ws_alloc((void**)&colsq, sizeof(double) * (size_t)np, st))) return rc;
  if ((rc = ws_alloc((void**)&fnorm, sizeof(double), st))) return rc;
  if ((rc = ws_alloc((void**)&wd, sizeof(double) * (size_t)n, st))) return rc;
  if ((rc = ws_alloc((void**)&rank, sizeof(int) * (size_t)n, st))) return rc;
  if ((rc = ws_alloc((void**)&conv, sizeof(unsigned int), st))) return rc;
  eigh_init_kernel<T><<<(unsigned)(((int64_t)np * np + 255) / 256), 256, 0, st>>>((const T*)a->data, a->stride[0], a->stride[1], n, np, A, V);
  eigh_colsq_kernel<T><<<np, 256, 0, st>>>(A, np, colsq);
  eigh_fnorm_kernel<<<1, 256, 0, st>>>(colsq, np, fnorm);
  count_launch(3);

  // Rounding in the rotations of the last sweep that rotated leaves off-diagonals of a few eps * ||A||_F; below
  // 4 eps the off-diagonal part bounds every eigenvalue's error by about 4 n eps ||A||_F.  The same bound stops the
  // inner sweeps of a pair, so a converged block is left alone (Q_p = I).
  const double tol = 4.0 * 2.220446049250313e-16;
  const int max_inner = 10, max_sweeps = 40;
  const int usplit = (np + RT - 1) / RT;
  const size_t eig_bytes = eig_smem_bytes<T>();
  {
    static bool attr_done = false;      // per T instantiation
    if (!attr_done) {
      TNB_CHECK_CUDA(cudaFuncSetAttribute(eigh_eig_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)eig_bytes));
      attr_done = true;
    }
  }
  int sweeps = 0, converged = 0;
  unsigned int h_conv = 0;
  for (int sw = 0; sw < max_sweeps; ++sw) {
    TNB_CHECK_CUDA(cudaMemsetAsync(conv, 0, sizeof(unsigned int), st));
    for (int r = 0; r < rounds; ++r) {
      eigh_eig_kernel<T><<<npairs, 256, eig_bytes, st>>>(A, np, nb, r, fnorm, Q, conv, tol, max_inner);
      if (ntiles > 0) eigh_tile_kernel<T><<<ntiles, 256, 0, st>>>(A, np, nb, r, Q);
      svd_update_kernel<T><<<dim3(npairs, usplit), 256, 0, st>>>(V, np, nb, r, Q);
    }
    count_launch((ntiles > 0 ? 3 : 2) * rounds);
    TNB_LAUNCH_CHECK();
    TNB_CHECK_CUDA(cudaMemcpyAsync(&h_conv, conv, sizeof(unsigned int), cudaMemcpyDeviceToHost, st));
    TNB_CHECK_CUDA(cudaStreamSynchronize(st));
    ++sweeps;
    float off;
    memcpy(&off, &h_conv, 4);
    if (off <= (float)tol) { converged = 1; break; }     // the kernels' comparison, so a skipped pair is a converged one
  }
  eigh_diag_kernel<T><<<(n + 255) / 256, 256, 0, st>>>(A, np, n, wd);
  eigh_rank_kernel<<<(n + 255) / 256, 256, 0, st>>>(wd, n, rank);
  eigh_finalize_kernel<T><<<n, 256, 0, st>>>(V, wd, rank, n, np, (double*)w->data, w->stride[0], (T*)v->data, v->stride[0], v->stride[1]);
  count_launch(3);
  TNB_LAUNCH_CHECK();
  if (info_dev) {
    int32_t h[4] = {sweeps, converged, 0, 0};
    TNB_CHECK_CUDA(cudaMemcpyAsync(info_dev, h, sizeof(h), cudaMemcpyHostToDevice, st));
    TNB_CHECK_CUDA(cudaStreamSynchronize(st));
  }
  ws_free(A, st); ws_free(V, st); ws_free(Q, st); ws_free(colsq, st); ws_free(fnorm, st); ws_free(wd, st); ws_free(rank, st); ws_free(conv, st);
  if (!converged) { set_error("eigh: Jacobi did not converge in %d sweeps", max_sweeps); return TNB200_ERR_NOCONV; }
  return 0;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_eigh(const tnb200_tensor_t* a, const tnb200_tensor_t* w, const tnb200_tensor_t* v, int32_t* info_dev, void* stream) {
  TNB_REQUIRE(valid_tensor(a) && valid_tensor(w) && valid_tensor(v), TNB200_ERR_INVALID, "eigh: invalid tensor descriptor");
  TNB_REQUIRE(a->ndim == 2 && w->ndim == 1 && v->ndim == 2, TNB200_ERR_INVALID, "eigh: expects a matrix, a vector and a matrix");
  const int64_t n = a->shape[0];
  TNB_REQUIRE(a->shape[1] == n, TNB200_ERR_INVALID, "eigh: matrix must be square, got %lld x %lld", (long long)n, (long long)a->shape[1]);
  TNB_REQUIRE(w->shape[0] == n && v->shape[0] == n && v->shape[1] == n, TNB200_ERR_INVALID, "eigh: output shapes must be (n,) and (n, n)");
  const int dt = a->dtype;
  TNB_REQUIRE(dt == TNB200_F64 || dt == TNB200_C128 || dt == TNB200_F32 || dt == TNB200_C64, TNB200_ERR_DTYPE,
              "eigh: dtype %s is not supported (f32/f64/c64/c128)", dtype_name(dt));
  const bool single = dt == TNB200_F32 || dt == TNB200_C64, cplx = dt == TNB200_C64 || dt == TNB200_C128;
  TNB_REQUIRE(w->dtype == (single ? TNB200_F32 : TNB200_F64), TNB200_ERR_DTYPE, "eigh: w must have the real dtype of the input");
  TNB_REQUIRE(v->dtype == dt, TNB200_ERR_DTYPE, "eigh: v dtype must equal the input dtype");
  TNB_REQUIRE(n < (1LL << 16), TNB200_ERR_UNSUPPORTED, "eigh: matrix too large");
  cudaStream_t st = (cudaStream_t)stream;
  set_kernel_name("eigh_block_jacobi");
  if (n == 0) return 0;
  if (!single) return cplx ? eigh_real<zd>(a, w, v, info_dev, st) : eigh_real<double>(a, w, v, info_dev, st);
  // single precision input: iterate in double, then round the results back (as tnb200_svd does)
  const int wide_dt = cplx ? TNB200_C128 : TNB200_F64;
  const size_t esz = cplx ? 16 : 8;
  void *da = nullptr, *dv = nullptr;
  double* dw = nullptr;
  int rc;
  if ((rc = ws_alloc(&da, esz * (size_t)n * n, st))) return rc;
  if ((rc = ws_alloc((void**)&dw, sizeof(double) * (size_t)n, st))) return rc;
  if ((rc = ws_alloc(&dv, esz * (size_t)n * n, st))) return rc;
  auto mk = [](void* p, int dtype, int64_t d0, int64_t d1, int nd) {
    tnb200_tensor_t t; t.data = p; t.dtype = dtype; t.ndim = nd;
    t.shape[0] = d0; t.shape[1] = d1; t.stride[0] = nd == 2 ? d1 : 1; t.stride[1] = 1; return t;
  };
  tnb200_tensor_t ta = mk(da, wide_dt, n, n, 2), tw = mk(dw, TNB200_F64, n, 1, 1), tv = mk(dv, wide_dt, n, n, 2);
  if ((rc = copy_strided(a, &ta, 0, st))) return rc;
  rc = cplx ? eigh_real<zd>(&ta, &tw, &tv, info_dev, st) : eigh_real<double>(&ta, &tw, &tv, info_dev, st);
  if (rc == 0) rc = copy_strided(&tw, w, 0, st);
  if (rc == 0) rc = copy_strided(&tv, v, 0, st);
  ws_free(da, st); ws_free(dw, st); ws_free(dv, st);
  return rc;
}
