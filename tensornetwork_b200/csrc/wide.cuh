// wide.cuh — storage <-> compute types of the one-CTA-per-problem batched kernels (svd_small.cu, qr_small.cu):
// f64 / f32 iterate in double and c128 / c64 in zd; `widen` loads an element, `narrow` rounds it back on store.
#pragma once
#include "cplx.cuh"
#include <cuComplex.h>

namespace tnb {

template <typename Tin> struct Wide;
template <> struct Wide<double> { using T = double; };
template <> struct Wide<float> { using T = double; };
template <> struct Wide<cuDoubleComplex> { using T = zd; };
template <> struct Wide<cuFloatComplex> { using T = zd; };
__device__ __forceinline__ double widen(double x) { return x; }
__device__ __forceinline__ double widen(float x) { return (double)x; }
__device__ __forceinline__ zd widen(cuDoubleComplex x) { return zd{x.x, x.y}; }
__device__ __forceinline__ zd widen(cuFloatComplex x) { return zd{(double)x.x, (double)x.y}; }
__device__ __forceinline__ void narrow(double* p, double v) { *p = v; }
__device__ __forceinline__ void narrow(float* p, double v) { *p = (float)v; }
__device__ __forceinline__ void narrow(cuDoubleComplex* p, zd v) { *p = make_cuDoubleComplex(v.x, v.y); }
__device__ __forceinline__ void narrow(cuFloatComplex* p, zd v) { *p = make_cuFloatComplex((float)v.x, (float)v.y); }

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ zd warp_sum(zd v) { return zd{warp_sum(v.x), warp_sum(v.y)}; }

}  // namespace tnb
