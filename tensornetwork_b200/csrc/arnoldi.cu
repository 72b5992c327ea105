// arnoldi.cu — tnb200_arnoldi_orth: one Arnoldi step's orthogonalisation, classical Gram-Schmidt applied twice
// (CGS2), for the implicitly restarted Arnoldi driver behind CudaB200Backend.eigs (scipy's ARPACK in
// backends/numpy/numpy_backend.py:216-298; ARPACK's dnaitr does the same DGKS-style reorthogonalisation).
//
// With k = j + 1 basis rows V[0..j] (row-major, row stride ldv) and the vector w, one call is FOUR launches,
// whatever j and n are:
//   1. project : h1 = V^H w,                 ||w||                (reads V once)
//   2. update  : u = w - V h1 -> row j+1,    h2 = V^H u           (reads V once)
//   3. update  : r = u - V h2 -> row j+1,    beta = ||r||         (reads V once)
//   4. scale   : row j+1 *= 1 / beta (zeros when beta is below the breakdown threshold)
// Passes 1-3 share one kernel.  A CTA walks tiles of S elements (S a power of two, k * S elements staged in shared
// memory with 128-bit loads when the rows are 16-byte aligned), so the update of a tile and its projection read V
// from HBM once between them.  Each CTA writes its partial sums; the last CTA to arrive (an arrival counter, reset
// by that CTA) reduces them in CTA order, so results do not depend on scheduling.  Accumulation is in double.
#include "common.cuh"
#include "cplx.cuh"
#include <math.h>
#include <algorithm>
#include <type_traits>

namespace tnb {

namespace {

constexpr int OT = 256;                  // threads per CTA
constexpr int OR = 4;                    // basis rows per thread in the projection: k <= OT * OR
constexpr int kMaxRows = OT * OR;
constexpr int kTileBytes = 32 * 1024;    // staged basis tile

__device__ __forceinline__ double widen(float a) { return a; }
__device__ __forceinline__ double widen(double a) { return a; }
__device__ __forceinline__ zd widen(float2 a) { return zd{a.x, a.y}; }
__device__ __forceinline__ zd widen(double2 a) { return zd{a.x, a.y}; }
__device__ __forceinline__ void narrow(float& o, double a) { o = (float)a; }
__device__ __forceinline__ void narrow(double& o, double a) { o = a; }
__device__ __forceinline__ void narrow(float2& o, zd a) { o = make_float2((float)a.x, (float)a.y); }
__device__ __forceinline__ void narrow(double2& o, zd a) { o = make_double2(a.x, a.y); }

__device__ __forceinline__ double ldcg_acc(const double* p) { return __ldcg(p); }
__device__ __forceinline__ zd ldcg_acc(const zd* p) {
  const double* q = reinterpret_cast<const double*>(p);
  return zd{__ldcg(q), __ldcg(q + 1)};
}

// one 128-bit load of the basis into shared memory (the padded tile rows are not 16-byte aligned there)
__device__ __forceinline__ void stage16(float* t, const float* g) {
  const float4 q = __ldg(reinterpret_cast<const float4*>(g));
  t[0] = q.x; t[1] = q.y; t[2] = q.z; t[3] = q.w;
}
__device__ __forceinline__ void stage16(double* t, const double* g) {
  const double2 q = __ldg(reinterpret_cast<const double2*>(g));
  t[0] = q.x; t[1] = q.y;
}
__device__ __forceinline__ void stage16(float2* t, const float2* g) {
  const float4 q = __ldg(reinterpret_cast<const float4*>(g));
  t[0] = make_float2(q.x, q.y); t[1] = make_float2(q.z, q.w);
}
__device__ __forceinline__ void stage16(double2* t, const double2* g) { t[0] = __ldg(g); }

template <typename S> struct AccOf { using T = double; };
template <> struct AccOf<float2> { using T = zd; };
template <> struct AccOf<double2> { using T = zd; };

// block-wide sum in a fixed tree order (every thread gets the result)
template <typename A>
__device__ A block_sum(A v, A* red) {
  const int tid = threadIdx.x;
  __syncthreads();
  red[tid] = v;
  __syncthreads();
  for (int s = OT / 2; s > 0; s >>= 1) {
    if (tid < s) red[tid] = add(red[tid], red[tid + s]);
    __syncthreads();
  }
  const A r = red[0];
  __syncthreads();
  return r;
}

struct OrthArgs {
  const void* v;          // row 0 of the basis
  int64_t ldv;            // row stride (elements)
  int k;                  // rows 0..k-1 take part
  int64_t n;
  const void* x;          // source vector (w, or row k for pass 3)
  void* y;                // row k (written by passes 2 and 3)
  int S, lgS;             // tile width (a power of two, <= OT) and its log2
  int vec;                // 1: 128-bit tile loads
  void* part;             // [grid][k + 1] partial sums (accumulation type)
  unsigned* counter;
  void* h1;               // [k] accumulation type
  void* h2;               // [k]
  double* scal;           // [0] ||w||^2, [1] 1 / beta (0 on breakdown)
  void* h_out;            // caller's h (k + 1 values, accumulation type)
  double tau;             // breakdown threshold: beta <= tau * ||w||
};

// UPD: subtract V[0..k) c from x (c = h1 in pass 2, h2 in pass 3).  PROJ: partial V^H u.  NORM: partial ||u||^2.
// WRITE: store u into row k.  Dynamic shared memory: k * (S + 1) storage elements + OT accumulators + S accumulators
// + k accumulators of the coefficients.
template <typename ST, int PASS>
__global__ void __launch_bounds__(OT, 2) arnoldi_cgs_kernel(OrthArgs a) {
  using A = typename AccOf<ST>::T;
  constexpr bool UPD = PASS != 1, PROJ = PASS != 3, NORM = PASS != 2, WRITE = PASS != 1;
  extern __shared__ __align__(16) unsigned char orth_smem[];
  const int k = a.k, S = a.S, LD = S + 1, tid = threadIdx.x;
  A* red = reinterpret_cast<A*>(orth_smem);                 // [OT]
  A* us = red + OT;                                         // [S]
  A* cs = us + S;                                           // [k]
  ST* tile = reinterpret_cast<ST*>(cs + k);                 // [k][S + 1]
  __shared__ int is_last;
  const ST* __restrict__ V = reinterpret_cast<const ST*>(a.v);
  ST* Y = reinterpret_cast<ST*>(a.y);
  const ST* X = PASS == 3 ? Y : reinterpret_cast<const ST*>(a.x);      // pass 3 updates row k in place
  if (UPD)
    for (int i = tid; i < k; i += OT) cs[i] = reinterpret_cast<const A*>(PASS == 2 ? a.h1 : a.h2)[i];
  A acc[OR];
#pragma unroll
  for (int r = 0; r < OR; ++r) acc[r] = zero_<A>();
  double nacc = 0.0;
  const int lgS = a.lgS;                                    // S is a power of two: shifts, no 64-bit division
  const int64_t ntiles = (a.n + S - 1) >> lgS;
  const int G = OT >> lgS;                                  // row groups of the update
  const int e_t = tid & (S - 1), g_t = tid >> lgS;
  // projection: with k <= OT, RP threads share a row (rows tid / RP); otherwise thread tid owns rows tid + OT r
  int RP = 1;
  while (RP * 2 * k <= OT && RP * 2 <= S) RP *= 2;
  const int p_row = k <= OT ? tid / RP : tid, p_part = k <= OT ? tid % RP : 0;
  constexpr int VEC = 16 / sizeof(ST);
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int64_t e0 = t << lgS;
    const int w = (int)min((int64_t)S, a.n - e0);
    // ---- stage V[0..k, e0 .. e0 + S) (zeros past n)
    if (a.vec && w == S) {
      const int lg_row = lgS - (VEC == 4 ? 2 : VEC == 2 ? 1 : 0);     // log2(S / VEC)
      for (int idx = tid; idx < (k << lg_row); idx += OT) {
        const int i = idx >> lg_row, c = idx - (i << lg_row);
        stage16(tile + i * LD + c * VEC, V + i * a.ldv + e0 + c * VEC);
      }
    } else {
      for (int idx = tid; idx < (k << lgS); idx += OT) {
        const int i = idx >> lgS, c = idx - (i << lgS);
        tile[i * LD + c] = c < w ? V[i * a.ldv + e0 + c] : ST{};
      }
    }
    __syncthreads();
    // ---- u = x - V c on this tile (row groups, then a fixed-order sum over the groups)
    if (UPD) {
      A p = zero_<A>();
      for (int i = g_t; i < k; i += G) fmacc(p, widen(tile[i * LD + e_t]), cs[i]);
      red[tid] = p;
      __syncthreads();
    }
    if (tid < S) {
      A u = tid < w ? widen(X[e0 + tid]) : zero_<A>();
      if (UPD) {
        A s = zero_<A>();
        for (int g = 0; g < G; ++g) s = add(s, red[g * S + tid]);
        u = sub(u, s);
      }
      if (WRITE && tid < w) narrow(Y[e0 + tid], u);
      if (NORM) nacc += ab2(u);
      us[tid] = u;
    }
    __syncthreads();
    // ---- partial V^H u over the tile
    if (PROJ) {
#pragma unroll
      for (int r = 0; r < OR; ++r) {
        const int i = p_row + OT * r;
        if (i < k)
          for (int c = p_part; c < S; c += RP) fmacc(acc[r], cj(widen(tile[i * LD + c])), us[c]);
      }
    }
    __syncthreads();
  }
  // ---- partials, then the last CTA reduces them in CTA order
  A* part = reinterpret_cast<A*>(a.part) + (int64_t)blockIdx.x * (k + 1);
  if (PROJ) {
    if (k <= OT) {                                          // sum the RP shares of each row in order
      red[tid] = acc[0];
      __syncthreads();
      if (tid < k) {
        A s = zero_<A>();
        for (int q = 0; q < RP; ++q) s = add(s, red[tid * RP + q]);
        part[tid] = s;
      }
    } else {
#pragma unroll
      for (int r = 0; r < OR; ++r)
        if (tid + OT * r < k) part[tid + OT * r] = acc[r];
    }
  }
  if (NORM) {
    const double nb = block_sum(nacc, reinterpret_cast<double*>(red));
    if (tid == 0) reinterpret_cast<double*>(part + k)[0] = nb;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) is_last = atomicAdd(a.counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  const A* P = reinterpret_cast<const A*>(a.part);
  const int stride = k + 1;
  if (PROJ) {
    A* hout = reinterpret_cast<A*>(PASS == 1 ? a.h1 : a.h2);
    for (int i = tid; i < k; i += OT) {
      A s = zero_<A>();
      for (unsigned c = 0; c < gridDim.x; ++c) s = add(s, ldcg_acc(P + (int64_t)c * stride + i));
      hout[i] = s;
    }
  }
  if (NORM) {
    double s = 0.0;
    for (unsigned c = tid; c < gridDim.x; c += OT) s += __ldcg(reinterpret_cast<const double*>(P + (int64_t)c * stride + k));
    const double n2 = block_sum(s, reinterpret_cast<double*>(red));
    if (PASS == 1) {
      if (tid == 0) a.scal[0] = n2;
    } else {
      const double nrm = sqrt(n2);
      const bool brk = n2 <= a.tau * a.tau * a.scal[0];
      A* ho = reinterpret_cast<A*>(a.h_out);
      const A* g1 = reinterpret_cast<const A*>(a.h1);
      const A* g2 = reinterpret_cast<const A*>(a.h2);
      for (int i = tid; i < k; i += OT) ho[i] = add(g1[i], g2[i]);
      if (tid == 0) {
        ho[k] = mk(brk ? 0.0 : nrm, 0.0, (A*)nullptr);
        a.scal[1] = brk ? 0.0 : 1.0 / nrm;
      }
    }
  }
  if (tid == 0) *a.counter = 0u;                            // ready for the next pass
}

// row k *= scal[1]; an exact zero row on breakdown
template <typename ST>
__global__ void __launch_bounds__(OT) arnoldi_scale_kernel(ST* __restrict__ y, int64_t n, const double* __restrict__ scal) {
  using A = typename AccOf<ST>::T;
  const double s = scal[1];
  for (int64_t e = blockIdx.x * (int64_t)OT + threadIdx.x; e < n; e += (int64_t)gridDim.x * OT) {
    const A u = widen(y[e]);
    narrow(y[e], s == 0.0 ? zero_<A>() : mulr(u, s));
  }
}

template <typename ST>
int orth_run(const tnb200_tensor_t* v, int j, const tnb200_tensor_t* w, void* h_dev, cudaStream_t st) {
  using A = typename AccOf<ST>::T;
  const int k = j + 1;
  const int64_t n = v->shape[1], ldv = v->stride[0];
  constexpr int esz = sizeof(ST), VEC = 16 / sizeof(ST);
  int S = OT, lgS = 8;
  while (S > 1 && (int64_t)k * (S + 1) * esz > kTileBytes) { S >>= 1; --lgS; }
  const int64_t ntiles = (n + S - 1) / S;
  const int grid = (int)std::min<int64_t>((int64_t)2 * num_sms(), ntiles);      // two CTAs per SM are resident
  const uintptr_t base = (uintptr_t)v->data;
  const int vec = S % VEC == 0 && base % 16 == 0 && (ldv * esz) % 16 == 0;
  const size_t smem = sizeof(A) * (OT + S + k) + (size_t)esz * k * (S + 1);
  // workspace: partials, h1, h2, scal, counter
  const size_t part_b = sizeof(A) * (size_t)grid * (k + 1);
  const size_t bytes = part_b + 2 * sizeof(A) * k + 2 * sizeof(double) + 16;
  unsigned char* ws = nullptr;
  int rc;
  if ((rc = ws_alloc((void**)&ws, bytes, st))) return rc;
  OrthArgs a;
  a.v = v->data; a.ldv = ldv; a.k = k; a.n = n; a.x = w->data;
  a.y = (ST*)v->data + (int64_t)k * ldv;
  a.S = S; a.lgS = lgS; a.vec = vec;
  a.part = ws;
  a.h1 = ws + part_b;
  a.h2 = ws + part_b + sizeof(A) * k;
  a.scal = reinterpret_cast<double*>(ws + part_b + 2 * sizeof(A) * k);
  a.counter = reinterpret_cast<unsigned*>(a.scal + 2);
  a.h_out = h_dev;
  // CGS2 leaves a residual of a few eps (of the stored dtype) times ||w|| when w lies in span(V)
  constexpr bool single = std::is_same<ST, float>::value || std::is_same<ST, float2>::value;
  const double eps = single ? 1.1920928955078125e-07 : 2.220446049250313e-16;
  a.tau = 16.0 * sqrt((double)k + 1.0) * eps;
  {
    static bool attr_done = false;      // per ST instantiation
    if (!attr_done) {
      const int mx = (int)(sizeof(A) * (OT + OT + kMaxRows) + kTileBytes);
      TNB_CHECK_CUDA(cudaFuncSetAttribute(arnoldi_cgs_kernel<ST, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
      TNB_CHECK_CUDA(cudaFuncSetAttribute(arnoldi_cgs_kernel<ST, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
      TNB_CHECK_CUDA(cudaFuncSetAttribute(arnoldi_cgs_kernel<ST, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx));
      attr_done = true;
    }
  }
  TNB_CHECK_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned), st));
  arnoldi_cgs_kernel<ST, 1><<<grid, OT, smem, st>>>(a);
  arnoldi_cgs_kernel<ST, 2><<<grid, OT, smem, st>>>(a);
  arnoldi_cgs_kernel<ST, 3><<<grid, OT, smem, st>>>(a);
  arnoldi_scale_kernel<ST><<<(int)std::min<int64_t>((int64_t)4 * num_sms(), (n + OT - 1) / OT), OT, 0, st>>>((ST*)a.y, n, a.scal);
  count_launch(4);
  TNB_LAUNCH_CHECK();
  ws_free(ws, st);
  return 0;
}

}  // namespace

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_arnoldi_orth(const tnb200_tensor_t* v, int32_t j, const tnb200_tensor_t* w, void* h_dev, void* stream) {
  TNB_REQUIRE(valid_tensor(v) && valid_tensor(w), TNB200_ERR_INVALID, "arnoldi_orth: invalid tensor descriptor");
  TNB_REQUIRE(v->ndim == 2, TNB200_ERR_INVALID, "arnoldi_orth: the basis must be a matrix (rows = Krylov vectors)");
  const int64_t n = v->shape[1];
  TNB_REQUIRE(j >= 0 && (int64_t)j + 2 <= v->shape[0], TNB200_ERR_INVALID,
              "arnoldi_orth: j = %d needs rows 0..j+1 of a basis with %lld rows", (int)j, (long long)v->shape[0]);
  TNB_REQUIRE(j + 1 <= kMaxRows, TNB200_ERR_UNSUPPORTED, "arnoldi_orth: at most %d basis rows, got %d", kMaxRows, (int)j + 1);
  TNB_REQUIRE(n >= 1 && (n == 1 || v->stride[1] == 1) && v->stride[0] >= n, TNB200_ERR_INVALID,
              "arnoldi_orth: basis rows must be contiguous and must not overlap");
  TNB_REQUIRE(numel(w) == n, TNB200_ERR_INVALID, "arnoldi_orth: w has %lld elements, the basis rows %lld",
              (long long)numel(w), (long long)n);
  int64_t expect = 1;
  bool contiguous = true;
  for (int d = w->ndim - 1; d >= 0; --d) {
    if (w->shape[d] != 1 && w->stride[d] != expect) contiguous = false;
    expect *= w->shape[d];
  }
  TNB_REQUIRE(contiguous, TNB200_ERR_INVALID, "arnoldi_orth: w must be contiguous");
  const int dt = v->dtype;
  TNB_REQUIRE(w->dtype == dt, TNB200_ERR_DTYPE, "arnoldi_orth: w and the basis must share a dtype");
  TNB_REQUIRE(h_dev != nullptr, TNB200_ERR_INVALID, "arnoldi_orth: h_dev is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  set_kernel_name("arnoldi_cgs2");
  switch (dt) {
    case TNB200_F64: return orth_run<double>(v, j, w, h_dev, st);
    case TNB200_F32: return orth_run<float>(v, j, w, h_dev, st);
    case TNB200_C128: return orth_run<double2>(v, j, w, h_dev, st);
    case TNB200_C64: return orth_run<float2>(v, j, w, h_dev, st);
  }
  set_error("arnoldi_orth: dtype %s is not supported (f32/f64/c64/c128)", dtype_name(dt));
  return TNB200_ERR_DTYPE;
}
