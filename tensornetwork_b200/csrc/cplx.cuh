// cplx.cuh — scalar abstraction shared by the split kernels (svd.cu, qr.cu): T is double (real) or
// zd (complex double, same layout as cuDoubleComplex); f32 / c64 inputs are widened by the callers.
#pragma once
#include <string.h>
namespace tnb {
// scalar abstraction: T is double (real) or zd (complex double); f32 / c64 inputs iterate in f64 / c128
struct zd { double x, y; };
__device__ __forceinline__ double cj(double a) { return a; }
__device__ __forceinline__ zd cj(zd a) { return zd{a.x, -a.y}; }
__device__ __forceinline__ double ab2(double a) { return a * a; }
__device__ __forceinline__ double ab2(zd a) { return a.x * a.x + a.y * a.y; }
__device__ __forceinline__ double mag_(double a) { return fabs(a); }          // |a| without the sqrt(a*a) round trip
__device__ __forceinline__ double mag_(zd a) { return sqrt(a.x * a.x + a.y * a.y); }
__device__ __forceinline__ double re_(double a) { return a; }
__device__ __forceinline__ double re_(zd a) { return a.x; }
__device__ __forceinline__ double mul(double a, double b) { return a * b; }
__device__ __forceinline__ zd mul(zd a, zd b) { return zd{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }
__device__ __forceinline__ double mulr(double a, double r) { return a * r; }
__device__ __forceinline__ zd mulr(zd a, double r) { return zd{a.x * r, a.y * r}; }
__device__ __forceinline__ double add(double a, double b) { return a + b; }
__device__ __forceinline__ zd add(zd a, zd b) { return zd{a.x + b.x, a.y + b.y}; }
__device__ __forceinline__ double sub(double a, double b) { return a - b; }
__device__ __forceinline__ zd sub(zd a, zd b) { return zd{a.x - b.x, a.y - b.y}; }
__device__ __forceinline__ void fmacc(double& c, double a, double b) { c = fma(a, b, c); }
__device__ __forceinline__ void fmacc(zd& c, zd a, zd b) {
  c.x = fma(a.x, b.x, c.x); c.x = fma(-a.y, b.y, c.x); c.y = fma(a.x, b.y, c.y); c.y = fma(a.y, b.x, c.y);
}
__device__ __forceinline__ void atomic_add(double* p, double v) { atomicAdd(p, v); }
__device__ __forceinline__ void atomic_add(zd* p, zd v) { atomicAdd(&p->x, v.x); atomicAdd(&p->y, v.y); }
template <typename T> __device__ __forceinline__ T zero_() { T z; memset(&z, 0, sizeof(T)); return z; }
template <typename T> __device__ __forceinline__ T one_();
template <> __device__ __forceinline__ double one_<double>() { return 1.0; }
template <> __device__ __forceinline__ zd one_<zd>() { return zd{1.0, 0.0}; }
// e^{-i phi} of g (1 for real / zero g)
__device__ __forceinline__ double unit_conj_phase(double g) { return g < 0 ? -1.0 : 1.0; }
__device__ __forceinline__ zd unit_conj_phase(zd g) {
  double a = sqrt(ab2(g));
  return a > 0 ? zd{g.x / a, -g.y / a} : zd{1.0, 0.0};
}

__device__ __forceinline__ zd divz(zd a, zd b) { double d = b.x * b.x + b.y * b.y; return zd{(a.x * b.x + a.y * b.y) / d, (a.y * b.x - a.x * b.y) / d}; }
__device__ __forceinline__ double divz(double a, double b) { return a / b; }
__device__ __forceinline__ double pivmag(double a) { return fabs(a); }
__device__ __forceinline__ double pivmag(zd a) { return fabs(a.x) + fabs(a.y); }   // dcabs1, as izamax ranks
// a / b without forming |b|^2 (Smith's algorithm): no overflow or underflow for |b| anywhere in the double range
__device__ __forceinline__ double divs(double a, double b) { return a / b; }
__device__ __forceinline__ zd divs(zd a, zd b) {
  if (fabs(b.x) >= fabs(b.y)) {
    const double r = b.y / b.x, d = b.x + b.y * r;
    return zd{(a.x + a.y * r) / d, (a.y - a.x * r) / d};
  }
  const double r = b.x / b.y, d = b.x * r + b.y;
  return zd{(a.x * r + a.y) / d, (a.y * r - a.x) / d};
}
__device__ __forceinline__ double im_(double) { return 0.0; }
__device__ __forceinline__ double im_(zd a) { return a.y; }
__device__ __forceinline__ double mk(double re, double, double*) { return re; }
__device__ __forceinline__ zd mk(double re, double im, zd*) { return zd{re, im}; }
}  // namespace tnb
