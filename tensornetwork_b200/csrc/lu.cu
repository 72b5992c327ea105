// lu.cu — tnb200_lu_factor / tnb200_lu_solve / tnb200_inv: LU with partial pivoting (LAPACK getrf, the pivots
// scipy.linalg.lu_factor returns), the solve on its factors (getrs, scipy.linalg.lu_solve) and the inverse built on both
// (np.linalg.inv, NumPyBackend.inv, backends/numpy/numpy_backend.py:554-558).
//
// Working storage is column-major (W[c * n + r]) in double or zd; f32 / c64 are widened by the strided copy in and
// rounded back by the copy out.  Right-looking blocked LU, panels of LB = 32 columns, four launches per panel:
//   lu_panel_kernel  : ONE cluster of 8 CTAs factors rows j0..n-1 of the panel.  Rows are dealt to the CTAs in
//                      contiguous ranges and kept in shared memory when they fit (in global memory, L2-resident, when
//                      they do not).  Per column ONE all-to-all exchange through distributed shared memory carries each
//                      CTA's pivot candidate (|x|, row index, the row) and the diagonal row; every CTA then picks the
//                      same winner (largest |x|, first index on ties: LAPACK's idamax / izamax), and the swap, the
//                      scale and the rank-1 update of the panel are local.
//   lu_laswp_kernel  : the panel's interchanges on the columns left and right of it (one thread per column).
//   lu_trsm_kernel   : U12 = L11^-1 A12 (unit lower, 32 x 32 in shared memory, one thread per column).
//   lu_update_*      : A22 -= L21 U12 — DMMA m8n8k4 for f64, CUDA-core FMA for c128.
// The solve (lu_solve_ws, shared with expm.cu) computes X = U^-1 (L^-1 (P B)): the row interchanges on B, then forward and
// backward block substitution, 32 rows per step, each step one triangular-solve launch and one update launch.  The
// inverse is the solve with B = I.
#include "common.cuh"
#include "cplx.cuh"
#include <float.h>
#include <math.h>

namespace tnb {

int copy_strided(const tnb200_tensor_t* src, const tnb200_tensor_t* dst, int conj, cudaStream_t st);

constexpr int LB = 32, LCL = 8, LTHR = 256;

__device__ __forceinline__ bool is_zero(double a) { return a == 0.0; }
__device__ __forceinline__ bool is_zero(zd a) { return a.x == 0.0 && a.y == 0.0; }

__device__ __forceinline__ uint32_t lu_cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void lu_cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void lu_st_remote(double* p, uint32_t rank, double v) {
  uint32_t a = (uint32_t)__cvta_generic_to_shared(p), r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(rank));
  asm volatile("st.shared::cluster.f64 [%0], %1;" ::"r"(r), "d"(v) : "memory");
}

// one CTA's message of a column step, in doubles: candidate row [LB T] | diagonal row [LB T] | |x| | row index
template <typename T> struct Msg {
  static constexpr int W = (int)(sizeof(T) / sizeof(double));
  static constexpr int CAND = 0, DIAG = LB * W, VAL = 2 * LB * W, IDX = 2 * LB * W + 1, SIZE = 2 * LB * W + 2;
};

template <typename T>
static size_t panel_smem(int rl, bool in_smem) {
  const int rlp = rl + (rl & 1);
  return sizeof(double) * ((size_t)(2 * LCL + 1) * Msg<T>::SIZE + 2 * 8 + 2) + (in_smem ? sizeof(T) * (size_t)LB * rlp : 0) + 16;
}

// Factor rows j0..n-1 of columns j0..j0+b-1 of W (column-major, leading dimension n).  CTA `rank` owns global rows
// [j0 + rank * rl, j0 + (rank + 1) * rl).  piv[j0 + j] = the global pivot row of column j0 + j; info[0] is set to
// 1 + the first exactly-zero pivot if it is still 0.
template <typename T>
__global__ void __cluster_dims__(LCL, 1, 1) __launch_bounds__(LTHR, 1)
lu_panel_kernel(T* __restrict__ W, int64_t n, int j0, int b, int rl, int in_smem, int* __restrict__ piv, int* __restrict__ info) {
  using M = Msg<T>;
  extern __shared__ __align__(16) double lsm[];
  double* part = lsm;                                   // [2][LCL][M::SIZE]: the messages of all CTAs, double-buffered
  double* mine = part + 2 * LCL * M::SIZE;              // [M::SIZE]
  double* rv = mine + M::SIZE;                          // [8] per-warp best |x|
  int* ri = (int*)(rv + 8);                             // [8] per-warp best local row  (+ 2 ints: the CTA's result)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = lu_cluster_rank();
  const int64_t row0 = (int64_t)j0 + (int64_t)rank * rl;
  int64_t nl64 = n - row0; if (nl64 > rl) nl64 = rl; if (nl64 < 0) nl64 = 0;
  const int nl = (int)nl64;
  T* P;
  int64_t ldp;
  if (in_smem) {
    const int rlp = rl + (rl & 1);
    P = reinterpret_cast<T*>(lsm + (2 * LCL + 1) * M::SIZE + 2 * 8 + 2 + ((2 * LCL + 1) * M::SIZE & 1));
    ldp = rlp;
    for (int idx = tid; idx < b * nl; idx += LTHR) {
      const int c = idx / nl, i = idx - c * nl;
      P[c * ldp + i] = W[(int64_t)(j0 + c) * n + row0 + i];
    }
  } else {
    P = W + (int64_t)j0 * n + row0;
    ldp = n;
  }
  int first_zero = -1;
  __syncthreads();
  lu_cluster_sync();                                    // every CTA of the cluster runs before any remote store
  for (int j = 0; j < b; ++j) {
    const int64_t gp = (int64_t)j0 + j;                 // global row of the diagonal
    int is = (int)(gp - row0); if (is < 0) is = 0;      // first local row at or below the diagonal
    // local candidate: the first row of largest |x| in column j (rows >= gp)
    double bv = -1.0;
    int bi = 0x7fffffff;
    for (int i = is + tid; i < nl; i += LTHR) {
      const double v = pivmag(P[j * ldp + i]);
      if (v > bv) { bv = v; bi = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_down_sync(0xffffffffu, bv, o);
      const int oi = __shfl_down_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { rv[warp] = bv; ri[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < LTHR / 32; ++w)
        if (rv[w] > bv || (rv[w] == bv && ri[w] < bi)) { bv = rv[w]; bi = ri[w]; }
      mine[M::VAL] = bv;
      mine[M::IDX] = bv >= 0.0 ? (double)(row0 + bi) : -1.0;
      ri[8] = bv >= 0.0 ? bi : -1;
    }
    __syncthreads();
    const int cand = ri[8];
    const bool own_diag = gp >= row0 && gp < row0 + nl;
    const int jl = (int)(gp - row0);
    T* mt = reinterpret_cast<T*>(mine);
    if (tid < b) {
      if (cand >= 0) mt[M::CAND / M::W + tid] = P[tid * ldp + cand];
      if (own_diag) mt[M::DIAG / M::W + tid] = P[tid * ldp + jl];
    }
    __syncthreads();
    const int buf = j & 1;
    for (int idx = tid; idx < LCL * M::SIZE; idx += LTHR) {
      const int q = idx / M::SIZE, w = idx - q * M::SIZE;
      lu_st_remote(part + ((size_t)buf * LCL + rank) * M::SIZE + w, (uint32_t)q, mine[w]);
    }
    lu_cluster_sync();
    // every CTA picks the same winner: largest |x|; CTAs hold ascending row ranges, so the first CTA wins a tie
    const double* pb = part + (size_t)buf * LCL * M::SIZE;
    int win = 0;
    double wv = pb[M::VAL];
    for (int q = 1; q < LCL; ++q)
      if (pb[q * M::SIZE + M::VAL] > wv) { wv = pb[q * M::SIZE + M::VAL]; win = q; }
    // NaN, as reference BLAS idamax treats it (dmax = |x(first)|, then only strictly greater |x| replace it): a NaN on
    // the diagonal stays the pivot, a NaN below it is never chosen.  No candidate at all (every |x| NaN) is covered
    // by the first rule, so the pivot row is always in range; the factorisation then carries the NaNs through.
    const T* drow = reinterpret_cast<const T*>(pb + (int)((gp - j0) / rl) * M::SIZE + M::DIAG);
    const bool keep_diag = pb[win * M::SIZE + M::IDX] < 0.0 || isnan(pivmag(drow[j]));
    const int64_t pr = keep_diag ? gp : (int64_t)pb[win * M::SIZE + M::IDX];        // global pivot row
    const T* prow = keep_diag ? drow : reinterpret_cast<const T*>(pb + win * M::SIZE + M::CAND);
    const T pivot = prow[j];
    if (rank == 0 && tid == 0) {
      piv[gp] = (int)pr;
      if (is_zero(pivot) && first_zero < 0) first_zero = (int)gp;
    }
    // the interchange inside the panel: row pr <- the diagonal row, the diagonal row <- row pr
    if (pr != gp && tid < b) {
      if (pr >= row0 && pr < row0 + nl) P[tid * ldp + (pr - row0)] = drow[tid];
      if (own_diag) P[tid * ldp + jl] = prow[tid];
    }
    __syncthreads();
    if (!is_zero(pivot)) {
      // as LAPACK's getrf2: multiply by the reciprocal unless |pivot| is below the smallest normal number
      const bool tiny = pivmag(pivot) < DBL_MIN;
      const T rp = divs(one_<T>(), pivot);
      int i0 = (int)(gp + 1 - row0); if (i0 < 0) i0 = 0;
      for (int i = i0 + tid; i < nl; i += LTHR) {
        const T l = tiny ? divs(P[j * ldp + i], pivot) : mul(P[j * ldp + i], rp);
        P[j * ldp + i] = l;
        for (int c = j + 1; c < b; ++c) P[c * ldp + i] = sub(P[c * ldp + i], mul(l, prow[c]));
      }
    }
    __syncthreads();
  }
  if (in_smem) {
    for (int idx = tid; idx < b * nl; idx += LTHR) {
      const int c = idx / nl, i = idx - c * nl;
      W[(int64_t)(j0 + c) * n + row0 + i] = P[c * ldp + i];
    }
  }
  if (rank == 0 && tid == 0 && first_zero >= 0 && info[0] == 0) info[0] = first_zero + 1;
}

// the interchanges of rows k0 .. k0+b-1 (piv) on the columns outside [k0, k0 + b)
template <typename T>
__global__ void lu_laswp_kernel(T* __restrict__ W, int64_t n, int k0, int b, const int* __restrict__ piv) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n - b) return;
  const int64_t col = t < k0 ? t : t + b;
  T* x = W + col * n;
  for (int k = k0; k < k0 + b; ++k) {
    const int r = piv[k];
    if (r != k) { const T v = x[k]; x[k] = x[r]; x[r] = v; }
  }
}

// X[r0 : r0+b, c0 + col] <- T^-1 X[...] for the b x b diagonal block T = A[r0 : r0+b, r0 : r0+b] (column-major, lda):
// unit lower (upper = 0) or upper (upper = 1) triangular.  One thread per column.
template <typename T>
__global__ void __launch_bounds__(128) lu_trsm_kernel(const T* __restrict__ A, int64_t lda, int r0, int b, int upper,
                                                      T* __restrict__ X, int64_t ldx, int64_t c0, int64_t ncols) {
  __shared__ T tri[LB][LB + 1];
  for (int idx = threadIdx.x; idx < LB * LB; idx += blockDim.x) {
    const int c = idx / LB, r = idx - c * LB;
    tri[r][c] = (r < b && c < b) ? A[(int64_t)(r0 + c) * lda + r0 + r] : zero_<T>();
  }
  __syncthreads();
  const int64_t col = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (col >= ncols) return;
  T* x = X + (c0 + col) * ldx + r0;
  T v[LB];
#pragma unroll
  for (int i = 0; i < LB; ++i) v[i] = i < b ? x[i] : zero_<T>();
  if (!upper) {
#pragma unroll
    for (int i = 0; i < LB; ++i)
#pragma unroll
      for (int r = i + 1; r < LB; ++r) v[r] = sub(v[r], mul(tri[r][i], v[i]));
  } else {
#pragma unroll
    for (int i = LB - 1; i >= 0; --i) {
      if (i < b) v[i] = divs(v[i], tri[i][i]);
#pragma unroll
      for (int r = 0; r < i; ++r) v[r] = sub(v[r], mul(tri[r][i], v[i]));
    }
  }
#pragma unroll
  for (int i = 0; i < LB; ++i) if (i < b) x[i] = v[i];
}

// C[M x N] -= A[M x K] B[K x N], all column-major, K <= 32, 64 x 64 tiles of C per CTA
template <typename T> struct LuUpd { const T* A; int64_t lda; const T* B; int64_t ldb; T* C; int64_t ldc; int64_t M, N; int K; };

constexpr int ULD = 36;
__device__ __forceinline__ void lu_dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(256) lu_update_dmma_kernel(const LuUpd<double> u) {
  __shared__ double As[64 * ULD], Bs[64 * ULD];           // As[row][k], Bs[col][k]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, fr = lane >> 2, fk = lane & 3;
  const int64_t rb = (int64_t)blockIdx.x * 64, cb = (int64_t)blockIdx.y * 64;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int idx = tid + 256 * i;
    const int r = idx & 63, k = idx >> 6;                 // A: 64 rows x 32 k, rows fastest (coalesced)
    As[r * ULD + k] = (rb + r < u.M && k < u.K) ? u.A[(int64_t)k * u.lda + rb + r] : 0.0;
    const int kb = idx & 31, c = idx >> 5;                // B: 32 k x 64 columns, k fastest
    Bs[c * ULD + kb] = (cb + c < u.N && kb < u.K) ? u.B[(cb + c) * u.ldb + kb] : 0.0;
  }
  __syncthreads();
  const int mrow = (warp & 3) * 16, ncol = (warp >> 2) * 32;
  double acc[2][4][2];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[a][j][0] = 0.0; acc[a][j][1] = 0.0; }
#pragma unroll
  for (int k4 = 0; k4 < LB; k4 += 4) {
    const double a0 = As[(mrow + fr) * ULD + k4 + fk], a1 = As[(mrow + 8 + fr) * ULD + k4 + fk];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double bb = Bs[(ncol + j * 8 + fr) * ULD + k4 + fk];
      lu_dmma(acc[0][j][0], acc[0][j][1], a0, bb);
      lu_dmma(acc[1][j][0], acc[1][j][1], a1, bb);
    }
  }
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int64_t r = rb + mrow + a * 8 + fr, c = cb + ncol + j * 8 + 2 * fk + e;
        if (r < u.M && c < u.N) u.C[c * u.ldc + r] -= acc[a][j][e];
      }
}

// the same product with CUDA-core FMA (c128); K in two halves of 16 so the tiles fit static shared memory
template <typename T>
__global__ void __launch_bounds__(256) lu_update_fma_kernel(const LuUpd<T> u) {
  __shared__ T As[16][64 + 1], Bs[16][64 + 1];            // As[k][row], Bs[k][col]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t rb = (int64_t)blockIdx.x * 64, cb = (int64_t)blockIdx.y * 64;
  T acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = zero_<T>();
  for (int k0 = 0; k0 < u.K; k0 += 16) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + 256 * i;
      const int r = idx & 63, k = idx >> 6;
      As[k][r] = (rb + r < u.M && k0 + k < u.K) ? u.A[(int64_t)(k0 + k) * u.lda + rb + r] : zero_<T>();
      const int kb = idx & 15, c = idx >> 4;
      Bs[kb][c] = (cb + c < u.N && k0 + kb < u.K) ? u.B[(cb + c) * u.ldb + k0 + kb] : zero_<T>();
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) fmacc(acc[i][j], As[k][tx + 16 * i], Bs[k][ty + 16 * j]);
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t r = rb + tx + 16 * i, c = cb + ty + 16 * j;
      if (r < u.M && c < u.N) u.C[c * u.ldc + r] = sub(u.C[c * u.ldc + r], acc[i][j]);
    }
}

static void lu_update(const LuUpd<double>& u, cudaStream_t st) {
  lu_update_dmma_kernel<<<dim3((unsigned)((u.M + 63) / 64), (unsigned)((u.N + 63) / 64)), 256, 0, st>>>(u);
}
static void lu_update(const LuUpd<zd>& u, cudaStream_t st) {
  lu_update_fma_kernel<zd><<<dim3((unsigned)((u.M + 63) / 64), (unsigned)((u.N + 63) / 64)), 256, 0, st>>>(u);
}

// B <- P B: the interchanges piv[0..n) of the factorisation applied in order to each of the nrhs columns of B (LAPACK's
// laswp on the right-hand side), one thread per column
template <typename T>
__global__ void lu_laswp_rhs_kernel(T* __restrict__ B, int64_t ldb, int64_t n, int64_t nrhs, const int* __restrict__ piv) {
  const int64_t col = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (col >= nrhs) return;
  T* x = B + col * ldb;
  for (int64_t k = 0; k < n; ++k) {
    const int r = piv[k];
    if (r != k) { const T v = x[k]; x[k] = x[r]; x[r] = v; }
  }
}

static unsigned lu_grid(int64_t work, int threads) {
  int64_t g = (work + threads - 1) / threads;
  if (g < 1) g = 1;
  return (unsigned)g;
}

// LU of W (n x n, column-major, in place); piv / info device arrays, info[0] must be 0 on entry
template <typename T>
int lu_factor_ws(T* W, int64_t n, int* piv, int* info, cudaStream_t st, int* launches) {
  static bool attr_done = false;
  if (!attr_done) {
    TNB_CHECK_CUDA(cudaFuncSetAttribute(lu_panel_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 1024));
    attr_done = true;
  }
  for (int64_t j0 = 0; j0 < n; j0 += LB) {
    const int b = (int)(n - j0 < LB ? n - j0 : LB);
    int rl = (int)((n - j0 + LCL - 1) / LCL);
    if (rl < 1) rl = 1;
    const bool in_smem = panel_smem<T>(rl, true) <= 226 * 1024;
    lu_panel_kernel<T><<<LCL, LTHR, panel_smem<T>(rl, in_smem), st>>>(W, n, (int)j0, b, rl, in_smem ? 1 : 0, piv, info);
    ++*launches;
    if (n - b > 0) {
      lu_laswp_kernel<T><<<lu_grid(n - b, 128), 128, 0, st>>>(W, n, (int)j0, b, piv);
      ++*launches;
    }
    const int64_t rest = n - j0 - b;
    if (rest > 0) {
      lu_trsm_kernel<T><<<lu_grid(rest, 128), 128, 0, st>>>(W, n, (int)j0, b, 0, W, n, j0 + b, rest);
      LuUpd<T> u{W + j0 * n + j0 + b, n, W + (j0 + b) * n + j0, n, W + (j0 + b) * n + j0 + b, n, rest, rest, b};
      lu_update(u, st);
      *launches += 2;
    }
  }
  TNB_LAUNCH_CHECK();
  return 0;
}

// B <- A^-1 B (LAPACK getrs) from the factors in W: the row interchanges, then forward (unit L) and backward (U) block
// substitution, 32 rows per step.  B is n x nrhs, column-major with leading dimension ldb.
template <typename T>
int lu_solve_ws(const T* W, int64_t n, const int* piv, T* B, int64_t ldb, int64_t nrhs, cudaStream_t st, int* launches) {
  lu_laswp_rhs_kernel<T><<<lu_grid(nrhs, 128), 128, 0, st>>>(B, ldb, n, nrhs, piv);
  ++*launches;
  for (int64_t r0 = 0; r0 < n; r0 += LB) {
    const int b = (int)(n - r0 < LB ? n - r0 : LB);
    lu_trsm_kernel<T><<<lu_grid(nrhs, 128), 128, 0, st>>>(W, n, (int)r0, b, 0, B, ldb, 0, nrhs);
    ++*launches;
    const int64_t below = n - r0 - b;
    if (below > 0) {
      LuUpd<T> u{W + r0 * n + r0 + b, n, B + r0, ldb, B + r0 + b, ldb, below, nrhs, b};
      lu_update(u, st);
      ++*launches;
    }
  }
  for (int64_t r0 = ((n - 1) / LB) * LB; r0 >= 0; r0 -= LB) {
    const int b = (int)(n - r0 < LB ? n - r0 : LB);
    lu_trsm_kernel<T><<<lu_grid(nrhs, 128), 128, 0, st>>>(W, n, (int)r0, b, 1, B, ldb, 0, nrhs);
    ++*launches;
    if (r0 > 0) {
      LuUpd<T> u{W + r0 * n, n, B + r0, ldb, B, ldb, r0, nrhs, b};
      lu_update(u, st);
      ++*launches;
    }
  }
  TNB_LAUNCH_CHECK();
  return 0;
}
template int lu_factor_ws<double>(double*, int64_t, int*, int*, cudaStream_t, int*);
template int lu_factor_ws<zd>(zd*, int64_t, int*, int*, cudaStream_t, int*);
template int lu_solve_ws<double>(const double*, int64_t, const int*, double*, int64_t, int64_t, cudaStream_t, int*);
template int lu_solve_ws<zd>(const zd*, int64_t, const int*, zd*, int64_t, int64_t, cudaStream_t, int*);

static tnb200_tensor_t colmajor(void* p, int dtype, int64_t n) {
  tnb200_tensor_t t;
  t.data = p; t.dtype = dtype; t.ndim = 2;
  t.shape[0] = n; t.shape[1] = n; t.stride[0] = 1; t.stride[1] = n;
  return t;
}

static int lu_check(const char* what, const tnb200_tensor_t* a, const tnb200_tensor_t* out) {
  TNB_REQUIRE(valid_tensor(a) && valid_tensor(out), TNB200_ERR_INVALID, "%s: invalid tensor descriptor", what);
  TNB_REQUIRE(a->ndim == 2 && out->ndim == 2, TNB200_ERR_INVALID, "%s: expects matrices", what);
  TNB_REQUIRE(a->shape[0] == a->shape[1], TNB200_ERR_INVALID, "%s: the matrix must be square, got %lld x %lld", what,
              (long long)a->shape[0], (long long)a->shape[1]);
  TNB_REQUIRE(out->shape[0] == a->shape[0] && out->shape[1] == a->shape[1], TNB200_ERR_INVALID, "%s: output shape mismatch", what);
  TNB_REQUIRE(out->dtype == a->dtype, TNB200_ERR_DTYPE, "%s: dtype mismatch", what);
  TNB_REQUIRE(a->dtype == TNB200_F64 || a->dtype == TNB200_F32 || a->dtype == TNB200_C128 || a->dtype == TNB200_C64,
              TNB200_ERR_DTYPE, "%s: dtype %s is not supported (f32/f64/c64/c128)", what, dtype_name(a->dtype));
  TNB_REQUIRE(a->shape[0] < (1LL << 31), TNB200_ERR_UNSUPPORTED, "%s: matrix too large", what);
  return 0;
}

// factor (and, when x != NULL, invert) in the wide type T; a / lu / x carry the caller's dtype, the copies convert
template <typename T>
static int lu_run(const tnb200_tensor_t* a, const tnb200_tensor_t* lu, const tnb200_tensor_t* x, int* piv, int* info,
                  cudaStream_t st) {
  const int64_t n = a->shape[0];
  const int wide = sizeof(T) == 16 ? TNB200_C128 : TNB200_F64;
  T* W = nullptr;
  int rc;
  if ((rc = ws_alloc((void**)&W, sizeof(T) * (size_t)n * n, st))) return rc;
  tnb200_tensor_t tw = colmajor(W, wide, n);
  int launches = 0;
  rc = copy_strided(a, &tw, 0, st);
  if (rc == 0) rc = lu_factor_ws<T>(W, n, piv, info, st, &launches);
  if (rc == 0 && lu) rc = copy_strided(&tw, lu, 0, st);
  if (rc == 0 && x) {                              // A X = I: the solve with B = I
    T* X = nullptr;
    rc = ws_alloc((void**)&X, sizeof(T) * (size_t)n * n, st);
    tnb200_tensor_t tx = colmajor(X, wide, n);
    if (rc == 0) rc = tnb200_eye(&tx, 0, st);
    if (rc == 0) rc = lu_solve_ws<T>(W, n, piv, X, n, n, st, &launches);
    if (rc == 0) rc = copy_strided(&tx, x, 0, st);
    ws_free(X, st);                                // (ws_free ignores NULL)
  }
  count_launch(launches);
  ws_free(W, st);
  return rc;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_lu_factor(const tnb200_tensor_t* a, const tnb200_tensor_t* lu, int32_t* piv_dev, int32_t* info_dev,
                                    void* stream) {
  int rc = lu_check("lu_factor", a, lu);
  if (rc) return rc;
  TNB_REQUIRE(info_dev && (piv_dev || a->shape[0] == 0), TNB200_ERR_INVALID, "lu_factor: piv and info must be device arrays");
  cudaStream_t st = (cudaStream_t)stream;
  TNB_CHECK_CUDA(cudaMemsetAsync(info_dev, 0, sizeof(int32_t), st));
  if (a->shape[0] == 0) return 0;
  set_kernel_name(a->dtype == TNB200_F64 || a->dtype == TNB200_F32 ? "lu_blocked_dmma" : "lu_blocked_fma");
  if (dtype_is_complex(a->dtype)) return lu_run<zd>(a, lu, nullptr, piv_dev, info_dev, st);
  return lu_run<double>(a, lu, nullptr, piv_dev, info_dev, st);
}

extern "C" int32_t tnb200_lu_solve(const tnb200_tensor_t* lu, const int32_t* piv_dev, const tnb200_tensor_t* b,
                                   const tnb200_tensor_t* x, void* stream) {
  TNB_REQUIRE(valid_tensor(lu) && valid_tensor(b) && valid_tensor(x), TNB200_ERR_INVALID, "lu_solve: invalid tensor descriptor");
  TNB_REQUIRE(lu->ndim == 2 && b->ndim == 2 && x->ndim == 2, TNB200_ERR_INVALID, "lu_solve: expects matrices");
  TNB_REQUIRE(lu->shape[0] == lu->shape[1], TNB200_ERR_INVALID, "lu_solve: the factors must be square, got %lld x %lld",
              (long long)lu->shape[0], (long long)lu->shape[1]);
  TNB_REQUIRE(b->shape[0] == lu->shape[0], TNB200_ERR_INVALID, "lu_solve: b has %lld rows, the factors %lld",
              (long long)b->shape[0], (long long)lu->shape[0]);
  TNB_REQUIRE(x->shape[0] == b->shape[0] && x->shape[1] == b->shape[1], TNB200_ERR_INVALID, "lu_solve: x must have b's shape");
  TNB_REQUIRE(b->dtype == lu->dtype && x->dtype == lu->dtype, TNB200_ERR_DTYPE, "lu_solve: dtype mismatch");
  TNB_REQUIRE(lu->dtype == TNB200_F64 || lu->dtype == TNB200_F32 || lu->dtype == TNB200_C128 || lu->dtype == TNB200_C64,
              TNB200_ERR_DTYPE, "lu_solve: dtype %s is not supported (f32/f64/c64/c128)", dtype_name(lu->dtype));
  TNB_REQUIRE(lu->shape[0] < (1LL << 31), TNB200_ERR_UNSUPPORTED, "lu_solve: matrix too large");
  const int64_t n = lu->shape[0], k = b->shape[1];
  if (n == 0 || k == 0) return 0;
  TNB_REQUIRE(piv_dev, TNB200_ERR_INVALID, "lu_solve: piv must be a device array");
  cudaStream_t st = (cudaStream_t)stream;
  const bool cplx = dtype_is_complex(lu->dtype);
  const int wide = cplx ? TNB200_C128 : TNB200_F64;
  const size_t es = cplx ? 16 : 8;
  set_kernel_name(cplx ? "lu_solve_fma" : "lu_solve_dmma");
  void *W = nullptr, *X = nullptr;
  int rc = ws_alloc(&W, es * (size_t)n * n, st);
  if (rc == 0) rc = ws_alloc(&X, es * (size_t)n * k, st);
  tnb200_tensor_t tw = colmajor(W, wide, n), tx = colmajor(X, wide, n);
  tx.shape[1] = k;
  int launches = 0;
  if (rc == 0) rc = copy_strided(lu, &tw, 0, st);
  if (rc == 0) rc = copy_strided(b, &tx, 0, st);
  if (rc == 0) rc = cplx ? lu_solve_ws<zd>((const zd*)W, n, piv_dev, (zd*)X, n, k, st, &launches)
                         : lu_solve_ws<double>((const double*)W, n, piv_dev, (double*)X, n, k, st, &launches);
  if (rc == 0) rc = copy_strided(&tx, x, 0, st);
  count_launch(launches);
  ws_free(W, st); ws_free(X, st);
  return rc;
}

extern "C" int32_t tnb200_inv(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int32_t* info_dev, void* stream) {
  int rc = lu_check("inv", a, x);
  if (rc) return rc;
  TNB_REQUIRE(info_dev, TNB200_ERR_INVALID, "inv: info must be a device array");
  cudaStream_t st = (cudaStream_t)stream;
  TNB_CHECK_CUDA(cudaMemsetAsync(info_dev, 0, sizeof(int32_t), st));
  const int64_t n = a->shape[0];
  if (n == 0) return 0;
  set_kernel_name(a->dtype == TNB200_F64 || a->dtype == TNB200_F32 ? "lu_blocked_dmma" : "lu_blocked_fma");
  int* piv = nullptr;
  if ((rc = ws_alloc((void**)&piv, sizeof(int) * (size_t)n, st))) return rc;
  rc = dtype_is_complex(a->dtype) ? lu_run<zd>(a, nullptr, x, piv, info_dev, st) : lu_run<double>(a, nullptr, x, piv, info_dev, st);
  ws_free(piv, st);
  return rc;
}
