// expm.cu — tnb200_expm: the matrix exponential by scaling and squaring with Padé approximants (Al-Mohy & Higham 2009,
// Algorithm 5.1), the algorithm and the degree / scaling choice of scipy.sparse.linalg._matfuncs._expm with exact
// 1-norms (scipy.linalg.expm, NumPyBackend.expm, backends/numpy/numpy_backend.py:589-598).
//
// Both paths work in double or zd (f32 / c64 are widened on the way in and rounded on the way out) on seven n x n
// column-major buffers: A, A2, A4, A6 and three more (R1, R2, R3) that hold A8, A10, the Padé terms, P, Q and the
// squarings in turn.  They share three pieces of device code:
//   expm_select  : the (m, s) rule, from the exact 1-norms of A, A4, A6 (A8, A10 once formed) and the vector sequence
//                  v_p = 1^T |A|^p, p = 1..27, whose maxima are the ||(|A|)^(2m+1)||_1 of every _ell term;
//   expm_plan    : the Padé assembly as a list of GEMMs and weighted sums (pade3 ... pade13_scaled, P = V + U and
//                  Q = V - U in one pass);
//   comb_at / ell_column : one element of a weighted sum, one column of the |A| product.
// Fused path (n <= TNB200_EXPM_FUSED_MAX_N): ONE CTA does everything in one launch — norms, the |A| sequence, the
// selection, the powers, U and V, Gaussian elimination with partial pivoting on [Q | P], and the s squarings — with
// the seven buffers in shared memory when they fit (a stream-ordered workspace otherwise).  No host synchronisation.
// Blocked path: the GEMMs go through tnb200_tensordot in strict mode (DMMA for f64), Q is factored by lu_factor_ws
// and solved by lu_solve_ws (lu.cu); the host reads the selection once per stage that decides which power to form next
// (at most three reads per call).
#include "common.cuh"
#include "cplx.cuh"
#include <float.h>
#include <math.h>

namespace tnb {

int copy_strided(const tnb200_tensor_t* src, const tnb200_tensor_t* dst, int conj, cudaStream_t st);
template <typename T> int lu_factor_ws(T* W, int64_t n, int* piv, int* info, cudaStream_t st, int* launches);
template <typename T>
int lu_solve_ws(const T* W, int64_t n, const int* piv, T* B, int64_t ldb, int64_t nrhs, cudaStream_t st, int* launches);

// ---------------------------------------------------------------------------------------------- the selection rule
// buffers
enum { XA = 0, XA2, XA4, XA6, XR1, XR2, XR3, XNBUF };
// the |A| sequence runs to p = 27 (= 2 * 13 + 1); _ell(A, m) reads p = 2m + 1
constexpr int ELL_P = 27;
enum { SEL_DONE = 0, SEL_NEED_A8 = 8, SEL_NEED_A10 = 10, SEL_NONFINITE = -1 };

// 1 / |c_{2m+1}| of _ell (Al-Mohy & Higham 2009, eq. (2.2) and (2.6) of the 2005 paper), m = 3, 5, 7, 9, 13
__host__ __device__ inline double ell_c(int m) {
  return m == 3 ? 100800. : m == 5 ? 10059033600. : m == 7 ? 4487938430976000. : m == 9 ? 5914384781877411840000.
                                                                                          : 113250775606021113483283660800000000.;
}

// the exponent that scales |A| in the sequence so that no column sum can overflow: ||2^-ea |A| ||_1 < 2
__host__ __device__ inline int ell_scale_exp(double a1) { return a1 > 0.0 ? ilogb(fmin(a1, DBL_MAX)) : 0; }
// the exponent that rescales v_p before the next product (v_0 = 1 carries none)
__host__ __device__ inline int ell_step_exp(double mx) { return mx > 0.0 && mx <= DBL_MAX ? ilogb(mx) : 0; }

// _ell(2^-s A, m): ||(|A|)^(2m+1)||_1 = mx[2m+1] * 2^E with E the exponents dropped along the sequence; the 2^-s scaling
// enters as 2^(-2ms) (numerator 2^(-(2m+1)s), denominator ||2^-s A||_1 = 2^-s ||A||_1)
__device__ inline int expm_ell(const double* nrm, const double* mx, int m, int s) {
  const int p = 2 * m + 1;
  if (!(mx[p] > 0.0)) return 0;
  const double a1 = fmin(nrm[0], DBL_MAX);
  double e = (double)p * ell_scale_exp(a1);
  for (int q = 1; q < p; ++q) e += ell_step_exp(mx[q]);
  const double l = log2(mx[p]) + e - 2.0 * m * (double)s - log2(a1) - log2(ell_c(m)) + 53.0;   // log2(alpha / u)
  const double v = ceil(l / (2 * m));
  return v > 0.0 ? (int)v : 0;
}

// The (m, s) choice of scipy's _expm(A, use_exact_onenorm=True).  nrm = {||A||_1, ||A^4||_1, ||A^6||_1, ||A^8||_1,
// ||A^10||_1}; `have` is the highest power formed (6, 8 or 10).  Returns SEL_DONE with *m, *s and *recompute set, or
// the power to form next.  A power norm that overflowed is replaced by ||A||_1, which bounds ||A^p||_1^(1/p); then the
// unscaled powers cannot be reused and *recompute asks for B = 2^-s A and its powers to be formed afresh.
__device__ inline int expm_select(const double* nrm, const double* mx, int have, int* m, int* s, int* recompute) {
  const double a1 = fmin(nrm[0], DBL_MAX);
  const double d4r = pow(nrm[1], 1 / 4.), d6r = pow(nrm[2], 1 / 6.);
  const double d4 = isfinite(d4r) ? d4r : a1, d6 = isfinite(d6r) ? d6r : a1;
  *s = 0;
  *recompute = 0;
  const double eta1 = fmax(d4, d6);
  if (eta1 < 1.495585217958292e-002 && expm_ell(nrm, mx, 3, 0) == 0) { *m = 3; return SEL_DONE; }
  if (eta1 < 2.539398330063230e-001 && expm_ell(nrm, mx, 5, 0) == 0) { *m = 5; return SEL_DONE; }
  if (have < 8) return SEL_NEED_A8;
  const double d8r = pow(nrm[3], 1 / 8.), d8 = isfinite(d8r) ? d8r : a1;
  const double eta3 = fmax(d6, d8);
  if (eta3 < 9.504178996162932e-001 && expm_ell(nrm, mx, 7, 0) == 0) { *m = 7; return SEL_DONE; }
  if (eta3 < 2.097847961257068e+000 && expm_ell(nrm, mx, 9, 0) == 0) { *m = 9; return SEL_DONE; }
  if (have < 10) return SEL_NEED_A10;
  const double d10r = pow(nrm[4], 1 / 10.), d10 = isfinite(d10r) ? d10r : a1;
  const double eta5 = fmin(eta3, fmax(d8, d10));
  int sc = 0;
  if (eta5 > 0.0) {
    const double c = ceil(log2(eta5 / 4.25));
    sc = c > 0.0 ? (int)c : 0;
  }
  sc += expm_ell(nrm, mx, 13, sc);
  *m = 13;
  *s = sc;
  *recompute = !(isfinite(d4r) && isfinite(d6r));
  return SEL_DONE;
}

// ---------------------------------------------------------------------------------------------- the Padé plan
// pade3 ... pade13 coefficients b_0 .. b_m (scipy's _ExpmPadeHelper)
#define TNB_EXPM_PADE_B                                                                                               \
  120., 60., 12., 1., 0., 0., 0., 0., 0., 0., 0., 0., 0., 0.,                                                         \
  30240., 15120., 3360., 420., 30., 1., 0., 0., 0., 0., 0., 0., 0., 0.,                                               \
  17297280., 8648640., 1995840., 277200., 25200., 1512., 56., 1., 0., 0., 0., 0., 0., 0.,                             \
  17643225600., 8821612800., 2075673600., 302702400., 30270240., 2162160., 110880., 3960., 90., 1., 0., 0., 0., 0.,   \
  64764752532480000., 32382376266240000., 7771770303897600., 1187353796428800., 129060195264000., 10559470521600.,    \
  670442572800., 33522128640., 1323241920., 40840800., 960960., 16380., 182., 1.
__constant__ double c_pade_b[5 * 14] = {TNB_EXPM_PADE_B};
[[maybe_unused]] static const double h_pade_b[5 * 14] = {TNB_EXPM_PADE_B};
__host__ __device__ inline double pade_b(int m, int i) {
  const int row = m == 13 ? 4 : (m - 3) / 2;
#ifdef __CUDA_ARCH__
  return c_pade_b[row * 14 + i];
#else
  return h_pade_b[row * 14 + i];
#endif
}

// one step: GEMM out = x y, or a weighted sum out = sum_i c_i 2^e_i in_i + c0 I; with q >= 0 the sum is V and the step
// writes P = U + V into out and Q = V - U into q, U being buffer u
struct ExpmOp {
  int gemm, out, k, u, q;
  int in[5], e[5];
  double c[5], c0;
};
constexpr int MAX_OPS = 12;

__host__ __device__ inline ExpmOp op_gemm(int out, int x, int y) {
  ExpmOp o{};
  o.gemm = 1; o.out = out; o.k = 2; o.in[0] = x; o.in[1] = y; o.u = o.q = -1;
  return o;
}
__host__ __device__ inline ExpmOp op_sum(int out, int k, const int* in, const double* c, double c0, int e0 = 0) {
  ExpmOp o{};
  o.out = out; o.k = k; o.c0 = c0; o.u = o.q = -1;
  for (int i = 0; i < k; ++i) { o.in[i] = in[i]; o.c[i] = c[i]; o.e[i] = e0; }
  return o;
}

// The Padé step of degree m (and, for m = 13, the scaling by 2^-s) as ops on the buffers; returns the count.  The
// result leaves P in R3 and Q in R2.  Sums run in scipy's order (highest power first, the identity last).
__host__ __device__ inline int expm_plan(int m, int s, int recompute, ExpmOp* ops) {
  int n = 0;
  if (m < 13) {
    const int pw[4] = {XA2, XA4, XA6, XR1};           // A2, A4, A6, A8
    const int k = (m - 1) / 2;                         // powers A2 .. A_{m-1}
    int in[4];
    double cu[4], cv[4];
    for (int i = 0; i < k; ++i) {
      in[i] = pw[k - 1 - i];
      cu[i] = pade_b(m, m - 2 * i);                    // b_m A_{m-1} + ... + b_3 A2
      cv[i] = pade_b(m, m - 1 - 2 * i);                // b_{m-1} A_{m-1} + ... + b_2 A2
    }
    ops[n++] = op_sum(XR2, k, in, cu, pade_b(m, 1));
    ops[n++] = op_gemm(XR3, XA, XR2);                  // U = A (...)
    ops[n] = op_sum(XR3, k, in, cv, pade_b(m, 0));
    ops[n].u = XR3; ops[n].q = XR2; ++n;
    return n;
  }
  const double one = 1.0;
  if (recompute) {                                     // B = 2^-s A and its powers afresh
    const int a[1] = {XA};
    ops[n++] = op_sum(XA, 1, a, &one, 0.0, -s);
    ops[n++] = op_gemm(XA2, XA, XA);
    ops[n++] = op_gemm(XA4, XA2, XA2);
    ops[n++] = op_gemm(XA6, XA4, XA2);
  } else {                                             // B_k = 2^(-ks) A_k in place
    const int pw[4] = {XA, XA2, XA4, XA6}, pk[4] = {1, 2, 4, 6};
    for (int i = 0; i < 4; ++i) ops[n++] = op_sum(pw[i], 1, &pw[i], &one, 0.0, -pk[i] * s);
  }
  const int b642[3] = {XA6, XA4, XA2};
  const double c1[3] = {pade_b(13, 13), pade_b(13, 11), pade_b(13, 9)};
  ops[n++] = op_sum(XR2, 3, b642, c1, 0.0);
  ops[n++] = op_gemm(XR3, XA6, XR2);                   // U2
  const int t[4] = {XR3, XA6, XA4, XA2};
  const double c2[4] = {1.0, pade_b(13, 7), pade_b(13, 5), pade_b(13, 3)};
  ops[n++] = op_sum(XR2, 4, t, c2, pade_b(13, 1));
  ops[n++] = op_gemm(XR3, XA, XR2);                    // U
  const double c3[3] = {pade_b(13, 12), pade_b(13, 10), pade_b(13, 8)};
  ops[n++] = op_sum(XR2, 3, b642, c3, 0.0);
  ops[n++] = op_gemm(XR1, XA6, XR2);                   // V2
  const int v[4] = {XR1, XA6, XA4, XA2};
  const double c4[4] = {1.0, pade_b(13, 6), pade_b(13, 4), pade_b(13, 2)};
  ops[n] = op_sum(XR3, 4, v, c4, pade_b(13, 0));
  ops[n].u = XR3; ops[n].q = XR2; ++n;
  return n;
}

// ---------------------------------------------------------------------------------------------- shared element code
__device__ __forceinline__ double sc2(double a, int e) { return ldexp(a, e); }
__device__ __forceinline__ zd sc2(zd a, int e) { return zd{ldexp(a.x, e), ldexp(a.y, e)}; }
__device__ __forceinline__ double sc(double a, double c) { return a * c; }
__device__ __forceinline__ zd sc(zd a, double c) { return zd{a.x * c, a.y * c}; }
__device__ __forceinline__ double absv(double a) { return fabs(a); }
__device__ __forceinline__ double absv(zd a) { return hypot(a.x, a.y); }     // numpy's complex abs
__device__ __forceinline__ bool finite_v(double a) { return isfinite(a); }
__device__ __forceinline__ bool finite_v(zd a) { return isfinite(a.x) && isfinite(a.y); }

// element (r, c) of a weighted-sum op; writes P / Q when the op carries them
template <typename T>
__device__ __forceinline__ void comb_at(const ExpmOp& o, T* base, int64_t n, int64_t r, int64_t c) {
  const int64_t idx = c * n + r, nn = n * n;
  T* const buf_ = base;
#define buf(i) (buf_ + (int64_t)(i) * nn)
  T acc = zero_<T>();
  for (int i = 0; i < o.k; ++i) {
    const T x = buf(o.in[i])[idx];
    acc = i == 0 ? sc(o.e[i] ? sc2(x, o.e[i]) : x, o.c[i]) : add(acc, sc(o.e[i] ? sc2(x, o.e[i]) : x, o.c[i]));
  }
  if (r == c) acc = add(acc, sc(one_<T>(), o.c0));
  if (o.q >= 0) {
    const T u = buf(o.u)[idx];
    buf(o.out)[idx] = add(u, acc);
    buf(o.q)[idx] = sub(acc, u);
  } else {
    buf(o.out)[idx] = acc;
  }
#undef buf
}

// v_p[c] = sum_r 2^-ea |A[r, c]| 2^-e v_{p-1}[r] for column c, summed by the 32 lanes of a warp (v_in == NULL: v_0 = 1)
template <typename T>
__device__ __forceinline__ double ell_column(const T* A, int64_t n, int64_t c, const double* v_in, int ea, int e, int lane) {
  double acc = 0.0;
  for (int64_t r = lane; r < n; r += 32)
    acc += ldexp(absv(A[c * n + r]), -ea) * (v_in ? ldexp(v_in[r], -e) : 1.0);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

template <typename T>
__device__ __forceinline__ double abs_column(const T* M, int64_t n, int64_t c, int lane) {
  double acc = 0.0;
  for (int64_t r = lane; r < n; r += 32) acc += absv(M[c * n + r]);
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// element (r, c) of a strided f64 / f32 (T = double) or c128 / c64 (T = zd) matrix, widened
template <typename T> __device__ __forceinline__ T ld_wide(const tnb200_tensor_t& t, int64_t r, int64_t c);
template <> __device__ __forceinline__ double ld_wide<double>(const tnb200_tensor_t& t, int64_t r, int64_t c) {
  const int64_t o = r * t.stride[0] + c * t.stride[1];
  return t.dtype == TNB200_F64 ? ((const double*)t.data)[o] : (double)((const float*)t.data)[o];
}
template <> __device__ __forceinline__ zd ld_wide<zd>(const tnb200_tensor_t& t, int64_t r, int64_t c) {
  const int64_t o = r * t.stride[0] + c * t.stride[1];
  if (t.dtype == TNB200_C128) return ((const zd*)t.data)[o];
  const float2 v = ((const float2*)t.data)[o];
  return zd{(double)v.x, (double)v.y};
}
__device__ __forceinline__ void st_narrow(const tnb200_tensor_t& t, int64_t r, int64_t c, double v) {
  const int64_t o = r * t.stride[0] + c * t.stride[1];
  if (t.dtype == TNB200_F64) ((double*)t.data)[o] = v; else ((float*)t.data)[o] = (float)v;
}
__device__ __forceinline__ void st_narrow(const tnb200_tensor_t& t, int64_t r, int64_t c, zd v) {
  const int64_t o = r * t.stride[0] + c * t.stride[1];
  if (t.dtype == TNB200_C128) ((zd*)t.data)[o] = v; else ((float2*)t.data)[o] = make_float2((float)v.x, (float)v.y);
}

// ---------------------------------------------------------------------------------------------- fused path
constexpr int XT = 512, XW = XT / 32;

struct FusedShared {
  double nrm[5];
  double mx[ELL_P + 1];
  double red[XW];
  int redi[XW];
  int sel, m, s, recompute, flag, piv, lu_info, nops;
  ExpmOp ops[MAX_OPS];
};

// max over the CTA of one value per warp (lane 0 holds it); the result is returned to every thread
__device__ __forceinline__ double cta_max(double v, FusedShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) sh.red[warp] = v;
  __syncthreads();
  double m = sh.red[0];
  for (int w = 1; w < XW; ++w) m = fmax(m, sh.red[w]);
  __syncthreads();
  return m;
}

template <typename T>
__device__ void cta_onenorm(const T* M, int n, double* out, FusedShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double best = 0.0;
  for (int c = warp; c < n; c += XW) best = fmax(best, abs_column(M, n, c, lane));
  const double m = cta_max(best, sh);
  if (threadIdx.x == 0) *out = m;
}

template <typename T>
__device__ void cta_gemm(T* C, const T* A, const T* B, int n) {
  for (int idx = threadIdx.x; idx < n * n; idx += XT) {
    const int c = idx / n, r = idx - c * n;
    T acc = zero_<T>();
    for (int k = 0; k < n; ++k) fmacc(acc, A[k * n + r], B[c * n + k]);
    C[idx] = acc;
  }
  __syncthreads();
}

// the selection at stage `have`, by thread 0, broadcast through shared memory
__device__ __forceinline__ int cta_select(int have, FusedShared& sh) {
  __syncthreads();
  if (threadIdx.x == 0) sh.sel = expm_select(sh.nrm, sh.mx, have, &sh.m, &sh.s, &sh.recompute);
  __syncthreads();
  return sh.sel;
}

// Q X = P by Gaussian elimination with partial pivoting (the pivot: first largest |x|, or |re| + |im|, as getrf
// picks it) and back substitution; X overwrites P.  sh.lu_info = 1 + the first exactly-zero pivot, as getrf's info.
template <typename T>
__device__ void cta_solve(T* Q, T* P, int n, FusedShared& sh) {
  const int tid = threadIdx.x, lane = tid & 31;
  for (int j = 0; j < n; ++j) {
    if (tid < 32) {
      double bv = -1.0;
      int bi = 0x7fffffff;
      for (int i = j + lane; i < n; i += 32) {
        const double v = pivmag(Q[j * n + i]);
        if (v > bv) { bv = v; bi = i; }
      }
      for (int o = 16; o > 0; o >>= 1) {
        const double ov = __shfl_down_sync(0xffffffffu, bv, o);
        const int oi = __shfl_down_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (lane == 0) sh.piv = bi < n ? bi : j;
    }
    __syncthreads();
    const int p = sh.piv;
    if (p != j) {                                      // swap rows j and p of [Q | P]
      for (int c = tid; c < 2 * n; c += XT) {
        T* M = c < n ? Q : P;
        const int cc = c < n ? c : c - n;
        const T t = M[cc * n + j]; M[cc * n + j] = M[cc * n + p]; M[cc * n + p] = t;
      }
      __syncthreads();
    }
    const T piv = Q[j * n + j];
    if (pivmag(piv) == 0.0) {                          // getrf goes on past a zero pivot, and so does this
      if (tid == 0 && sh.lu_info == 0) sh.lu_info = j + 1;
      __syncthreads();
      continue;
    }
    const T rp = divs(one_<T>(), piv);
    const bool tiny = pivmag(piv) < DBL_MIN;
    for (int i = j + 1 + tid; i < n; i += XT) Q[j * n + i] = tiny ? divs(Q[j * n + i], piv) : mul(Q[j * n + i], rp);
    __syncthreads();
    const int rows = n - j - 1;
    for (int idx = tid; idx < rows * (2 * n - j - 1); idx += XT) {   // trailing Q columns j+1.. and all of P
      const int cl = idx / rows, i = j + 1 + idx - cl * rows;
      const int c = j + 1 + cl;
      T* M = c < n ? Q : P;
      const int cc = c < n ? c : c - n;
      M[cc * n + i] = sub(M[cc * n + i], mul(Q[j * n + i], M[cc * n + j]));
    }
    __syncthreads();
  }
  for (int j = n - 1; j >= 0; --j) {                   // U X = P', one row at a time
    const T d = Q[j * n + j];
    for (int c = tid; c < n; c += XT) P[c * n + j] = divs(P[c * n + j], d);
    __syncthreads();
    for (int idx = tid; idx < j * n; idx += XT) {
      const int c = idx / j, i = idx - c * j;
      P[c * n + i] = sub(P[c * n + i], mul(Q[j * n + i], P[c * n + j]));
    }
    __syncthreads();
  }
}

template <typename T>
__global__ void __launch_bounds__(XT, 1) expm_fused_kernel(const tnb200_tensor_t a, const tnb200_tensor_t x, int n,
                                                          T* __restrict__ gws, int* __restrict__ info) {
  extern __shared__ __align__(16) double xsm[];
  FusedShared& sh = *reinterpret_cast<FusedShared*>(xsm);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t nn = (int64_t)n * n;
  T* base = gws ? gws : reinterpret_cast<T*>(xsm + (sizeof(FusedShared) + 15) / 16 * 2);
  auto buf = [&](int i) { return base + i * nn; };
  double* v0 = reinterpret_cast<double*>(buf(XR1));   // the |A| sequence runs before R1 / R2 are needed
  double* v1 = reinterpret_cast<double*>(buf(XR2));
  if (tid == 0) { sh.flag = 0; sh.lu_info = 0; }
  __syncthreads();
  T* A = buf(XA);
  for (int idx = tid; idx < nn; idx += XT) {
    const int c = idx / n, r = idx - c * n;
    const T v = ld_wide<T>(a, r, c);
    if (!finite_v(v)) sh.flag = 1;
    A[idx] = v;
  }
  __syncthreads();
  if (sh.flag) {                                       // any NaN / Inf: all NaN, as scipy.linalg.expm
    for (int idx = tid; idx < nn; idx += XT) {
      const int c = idx / n, r = idx - c * n;
      st_narrow(x, r, c, sc(one_<T>(), NAN));
    }
    if (info && tid == 0) { info[0] = 0; info[1] = 0; info[2] = 0; info[3] = 0; }
    return;
  }
  cta_onenorm(A, n, &sh.nrm[0], sh);
  __syncthreads();
  // the |A| sequence
  const int ea = ell_scale_exp(sh.nrm[0]);
  for (int p = 1; p <= ELL_P; ++p) {
    const double* vin = p == 1 ? nullptr : ((p & 1) ? v1 : v0);
    double* vout = (p & 1) ? v0 : v1;
    const int e = p == 1 ? 0 : ell_step_exp(sh.mx[p - 1]);
    double best = 0.0;
    for (int c = warp; c < n; c += XW) {
      const double v = ell_column(A, n, c, vin, ea, e, lane);
      if (lane == 0) vout[c] = v;
      best = fmax(best, v);
    }
    const double m = cta_max(best, sh);
    if (tid == 0) sh.mx[p] = m;
    __syncthreads();
  }
  cta_gemm(buf(XA2), A, A, n);
  cta_gemm(buf(XA4), buf(XA2), buf(XA2), n);
  cta_gemm(buf(XA6), buf(XA4), buf(XA2), n);
  cta_onenorm(buf(XA4), n, &sh.nrm[1], sh);
  cta_onenorm(buf(XA6), n, &sh.nrm[2], sh);
  if (cta_select(6, sh) == SEL_NEED_A8) {
    cta_gemm(buf(XR1), buf(XA6), buf(XA2), n);
    cta_onenorm(buf(XR1), n, &sh.nrm[3], sh);
    if (cta_select(8, sh) == SEL_NEED_A10) {
      cta_gemm(buf(XR2), buf(XA4), buf(XA6), n);
      cta_onenorm(buf(XR2), n, &sh.nrm[4], sh);
      cta_select(10, sh);
    }
  }
  if (tid == 0) sh.nops = expm_plan(sh.m, sh.s, sh.recompute, sh.ops);
  __syncthreads();
  for (int k = 0; k < sh.nops; ++k) {
    const ExpmOp& o = sh.ops[k];
    if (o.gemm) {
      cta_gemm(buf(o.out), buf(o.in[0]), buf(o.in[1]), n);
    } else {
      for (int idx = tid; idx < nn; idx += XT) {
        const int c = idx / n, r = idx - c * n;
        comb_at(o, base, n, r, c);
      }
      __syncthreads();
    }
  }
  cta_solve(buf(XR2), buf(XR3), n, sh);
  int cur = XR3, nxt = XR1;
  for (int i = 0; i < sh.s; ++i) {
    cta_gemm(buf(nxt), buf(cur), buf(cur), n);
    const int t = cur; cur = nxt; nxt = t;
  }
  for (int idx = tid; idx < nn; idx += XT) {
    const int c = idx / n, r = idx - c * n;
    st_narrow(x, r, c, buf(cur)[idx]);
  }
  if (info && tid == 0) { info[0] = sh.m; info[1] = sh.s; info[2] = 0; info[3] = sh.lu_info; }
}

template <typename T>
static int expm_fused(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int n, int* info, cudaStream_t st) {
  const size_t head = (sizeof(FusedShared) + 15) / 16 * 16;
  const size_t mats = sizeof(T) * (size_t)XNBUF * n * n;
  const bool in_smem = head + mats <= 200 * 1024;
  const size_t smem = head + (in_smem ? mats : 0);
  T* gws = nullptr;
  if (!in_smem) {
    int rc = ws_alloc((void**)&gws, mats, st);
    if (rc) return rc;
  }
  static bool attr_done = false;
  if (!attr_done) {
    TNB_CHECK_CUDA(cudaFuncSetAttribute(expm_fused_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024 + (int)head));
    attr_done = true;
  }
  expm_fused_kernel<T><<<1, XT, smem, st>>>(*a, *x, n, gws, info);
  count_launch();
  TNB_LAUNCH_CHECK();
  ws_free(gws, st);
  return 0;
}

// ---------------------------------------------------------------------------------------------- blocked path
// device state: the norms and sequence maxima as the bits of nonnegative doubles (ordered like the doubles, so
// atomicMax on the bits is a max), the non-finite flag and the selection
struct BlockedState {
  unsigned long long nrm[5], mx[ELL_P + 1];
  int nonfinite, sel, m, s, recompute, pad[3];
};

__device__ __forceinline__ void atomic_max_nonneg(unsigned long long* p, double v) {
  atomicMax(p, (unsigned long long)__double_as_longlong(v));
}

// ||M||_1 into *out (one warp per column); with flag != NULL, also flags any non-finite entry
template <typename T>
__global__ void __launch_bounds__(256) expm_onenorm_kernel(const T* __restrict__ M, int64_t n, unsigned long long* out,
                                                           int* flag) {
  const int lane = threadIdx.x & 31;
  const int64_t c = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (c >= n) return;
  if (flag) {
    bool bad = false;
    for (int64_t r = lane; r < n; r += 32) bad |= !finite_v(M[c * n + r]);
    if (__any_sync(0xffffffffu, bad) && lane == 0) *flag = 1;
  }
  const double v = abs_column(M, n, c, lane);
  if (lane == 0) atomic_max_nonneg(out, v);
}

// step p of the |A| sequence: v_out = (2^-e v_in)^T (2^-ea |A|), its max into mx[p]
template <typename T>
__global__ void __launch_bounds__(256) expm_ell_kernel(const T* __restrict__ A, int64_t n, const double* v_in, double* v_out,
                                                       BlockedState* stt, int p) {
  const int lane = threadIdx.x & 31;
  const int64_t c = blockIdx.x * 8LL + (threadIdx.x >> 5);
  if (c >= n) return;
  const double* mx = reinterpret_cast<const double*>(stt->mx);
  const int ea = ell_scale_exp(__longlong_as_double((long long)stt->nrm[0]));
  const int e = p == 1 ? 0 : ell_step_exp(mx[p - 1]);
  const double v = ell_column(A, n, c, p == 1 ? nullptr : v_in, ea, e, lane);
  if (lane == 0) { v_out[c] = v; atomic_max_nonneg(&stt->mx[p], v); }
}

__global__ void expm_select_kernel(BlockedState* stt, int have, int* info) {
  if (stt->nonfinite) { stt->sel = SEL_NONFINITE; stt->m = stt->s = 0; return; }
  int m = 0, s = 0, rec = 0;
  stt->sel = expm_select(reinterpret_cast<const double*>(stt->nrm), reinterpret_cast<const double*>(stt->mx), have, &m, &s,
                         &rec);
  stt->m = m; stt->s = s; stt->recompute = rec;
  if (info && stt->sel == SEL_DONE) { info[0] = m; info[1] = s; info[2] = 1; }
}

template <typename T>
__global__ void __launch_bounds__(256) expm_comb_kernel(const ExpmOp o, T* base, int64_t n) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < n * n; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = idx / n, r = idx - c * n;
    comb_at(o, base, n, r, c);
  }
}

static tnb200_tensor_t rowmajor(void* p, int dtype, int64_t n) {
  tnb200_tensor_t t;
  memset(&t, 0, sizeof(t));
  t.data = p; t.dtype = dtype; t.ndim = 2;
  t.shape[0] = n; t.shape[1] = n; t.stride[0] = n; t.stride[1] = 1;
  return t;
}

// C = A B for column-major n x n matrices through the library's GEMM dispatch, strict precision.  Column-major X is the
// row-major X^T, so the call is C^T = B^T A^T on row-major views.
template <typename T>
static int expm_gemm(const T* A, const T* B, T* C, int64_t n, cudaStream_t st) {
  const int dt = sizeof(T) == 16 ? TNB200_C128 : TNB200_F64;
  tnb200_tensor_t ta = rowmajor((void*)B, dt, n), tb = rowmajor((void*)A, dt, n), tc = rowmajor(C, dt, n);
  const int32_t ax_a[1] = {1}, ax_b[1] = {0}, none[1] = {0};
  return tnb200_tensordot(&ta, &tb, &tc, 1, ax_a, ax_b, 0, none, none, TNB200_MATH_STRICT, st);
}

static int read_state(const BlockedState* d, BlockedState* h, cudaStream_t st) {
  TNB_CHECK_CUDA(cudaMemcpyAsync(h, d, sizeof(BlockedState), cudaMemcpyDeviceToHost, st));
  TNB_CHECK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

template <typename T>
static int expm_blocked_run(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int64_t n, T* const* buf, BlockedState* dst,
                            double* v, int* piv, int* linfo, int* info, cudaStream_t st) {
  const int wide = sizeof(T) == 16 ? TNB200_C128 : TNB200_F64;
  const unsigned cgrid = (unsigned)((n + 7) / 8);
  const int64_t eg = (n * n + 255) / 256;
  const unsigned egrid = (unsigned)(eg < (int64_t)num_sms() * 16 ? eg : (int64_t)num_sms() * 16);
  int launches = 0, rc;
  tnb200_tensor_t ta = rowmajor(buf[XA], wide, n);
  ta.stride[0] = 1; ta.stride[1] = n;                 // column-major
  TNB_CHECK_CUDA(cudaMemsetAsync(dst, 0, sizeof(BlockedState), st));
  TNB_CHECK_CUDA(cudaMemsetAsync(linfo, 0, sizeof(int), st));
  if ((rc = copy_strided(a, &ta, 0, st))) return rc;
  expm_onenorm_kernel<T><<<cgrid, 256, 0, st>>>(buf[XA], n, &dst->nrm[0], &dst->nonfinite);
  for (int p = 1; p <= ELL_P; ++p)
    expm_ell_kernel<T><<<cgrid, 256, 0, st>>>(buf[XA], n, (p & 1) ? v + n : v, (p & 1) ? v : v + n, dst, p);
  launches += 1 + ELL_P;
  if ((rc = expm_gemm(buf[XA], buf[XA], buf[XA2], n, st))) return rc;
  if ((rc = expm_gemm(buf[XA2], buf[XA2], buf[XA4], n, st))) return rc;
  if ((rc = expm_gemm(buf[XA4], buf[XA2], buf[XA6], n, st))) return rc;
  expm_onenorm_kernel<T><<<cgrid, 256, 0, st>>>(buf[XA4], n, &dst->nrm[1], nullptr);
  expm_onenorm_kernel<T><<<cgrid, 256, 0, st>>>(buf[XA6], n, &dst->nrm[2], nullptr);
  expm_select_kernel<<<1, 1, 0, st>>>(dst, 6, info);
  launches += 3;
  BlockedState h;
  if ((rc = read_state(dst, &h, st))) return rc;
  if (h.sel == SEL_NONFINITE) {
    count_launch(launches);
    if (info) TNB_CHECK_CUDA(cudaMemsetAsync(info, 0, 4 * sizeof(int), st));
    return tnb200_fill(x, NAN, NAN, st);
  }
  if (h.sel == SEL_NEED_A8) {
    if ((rc = expm_gemm(buf[XA6], buf[XA2], buf[XR1], n, st))) return rc;
    expm_onenorm_kernel<T><<<cgrid, 256, 0, st>>>(buf[XR1], n, &dst->nrm[3], nullptr);
    expm_select_kernel<<<1, 1, 0, st>>>(dst, 8, info);
    launches += 2;
    if ((rc = read_state(dst, &h, st))) return rc;
    if (h.sel == SEL_NEED_A10) {
      if ((rc = expm_gemm(buf[XA4], buf[XA6], buf[XR2], n, st))) return rc;
      expm_onenorm_kernel<T><<<cgrid, 256, 0, st>>>(buf[XR2], n, &dst->nrm[4], nullptr);
      expm_select_kernel<<<1, 1, 0, st>>>(dst, 10, info);
      launches += 2;
      if ((rc = read_state(dst, &h, st))) return rc;
    }
  }
  ExpmOp ops[MAX_OPS];
  const int nops = expm_plan(h.m, h.s, h.recompute, ops);
  for (int k = 0; k < nops; ++k) {
    const ExpmOp& o = ops[k];
    if (o.gemm) {
      if ((rc = expm_gemm(buf[o.in[0]], buf[o.in[1]], buf[o.out], n, st))) return rc;
    } else {
      expm_comb_kernel<T><<<egrid, 256, 0, st>>>(o, buf[0], n);
      ++launches;
    }
  }
  if ((rc = lu_factor_ws<T>(buf[XR2], n, piv, linfo, st, &launches))) return rc;
  if ((rc = lu_solve_ws<T>(buf[XR2], n, piv, buf[XR3], n, n, st, &launches))) return rc;
  if (info) TNB_CHECK_CUDA(cudaMemcpyAsync(info + 3, linfo, sizeof(int), cudaMemcpyDeviceToDevice, st));
  int cur = XR3, nxt = XR1;
  for (int i = 0; i < h.s; ++i) {
    if ((rc = expm_gemm(buf[cur], buf[cur], buf[nxt], n, st))) return rc;
    const int t = cur; cur = nxt; nxt = t;
  }
  count_launch(launches);
  TNB_LAUNCH_CHECK();
  tnb200_tensor_t tx = ta;
  tx.data = buf[cur];
  return copy_strided(&tx, x, 0, st);
}

template <typename T>
static int expm_blocked(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int64_t n, int* info, cudaStream_t st) {
  const size_t mat = sizeof(T) * (size_t)n * n;
  T* base = nullptr;
  BlockedState* dst = nullptr;
  double* v = nullptr;
  int* piv = nullptr;
  int rc = ws_alloc((void**)&base, mat * XNBUF, st);
  if (rc == 0) rc = ws_alloc((void**)&dst, sizeof(BlockedState), st);
  if (rc == 0) rc = ws_alloc((void**)&v, sizeof(double) * 2 * (size_t)n, st);
  if (rc == 0) rc = ws_alloc((void**)&piv, sizeof(int) * ((size_t)n + 1), st);
  if (rc == 0) {
    T* buf[XNBUF];
    for (int i = 0; i < XNBUF; ++i) buf[i] = base + (size_t)i * n * n;
    rc = expm_blocked_run<T>(a, x, n, buf, dst, v, piv, piv + n, info, st);
  }
  ws_free(base, st); ws_free(dst, st); ws_free(v, st); ws_free(piv, st);
  return rc;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_expm(const tnb200_tensor_t* a, const tnb200_tensor_t* x, int32_t* info_dev, void* stream) {
  TNB_REQUIRE(valid_tensor(a) && valid_tensor(x), TNB200_ERR_INVALID, "expm: invalid tensor descriptor");
  TNB_REQUIRE(a->ndim == 2 && x->ndim == 2, TNB200_ERR_INVALID, "expm: expects matrices");
  TNB_REQUIRE(a->shape[0] == a->shape[1], TNB200_ERR_INVALID, "expm: the matrix must be square, got %lld x %lld",
              (long long)a->shape[0], (long long)a->shape[1]);
  TNB_REQUIRE(x->shape[0] == a->shape[0] && x->shape[1] == a->shape[1], TNB200_ERR_INVALID, "expm: output shape mismatch");
  TNB_REQUIRE(x->dtype == a->dtype, TNB200_ERR_DTYPE, "expm: dtype mismatch");
  TNB_REQUIRE(a->dtype == TNB200_F64 || a->dtype == TNB200_F32 || a->dtype == TNB200_C128 || a->dtype == TNB200_C64,
              TNB200_ERR_DTYPE, "expm: dtype %s is not supported (f32/f64/c64/c128)", dtype_name(a->dtype));
  TNB_REQUIRE(a->shape[0] < (1LL << 31), TNB200_ERR_UNSUPPORTED, "expm: matrix too large");
  const int64_t n = a->shape[0];
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const bool cplx = dtype_is_complex(a->dtype);
  if (n <= TNB200_EXPM_FUSED_MAX_N) {
    set_kernel_name("expm_fused");
    return cplx ? expm_fused<zd>(a, x, (int)n, info_dev, st) : expm_fused<double>(a, x, (int)n, info_dev, st);
  }
  const int rc = cplx ? expm_blocked<zd>(a, x, n, info_dev, st) : expm_blocked<double>(a, x, n, info_dev, st);
  set_kernel_name("expm_blocked");
  return rc;
}
