// tensordot_thin.cu — HBM-streaming kernels for "thin" contractions: one operand is a small matrix S
// (<= 64 x 64, e.g. an MPS boundary site) and the other a long tensor X (10^5..10^6 elements per batch
// sample) that is read once and written once.  These are the ramp-up steps of a greedy MPS contraction
// path — (4 x 4).(4 x 131072) ... (64 x 64).(64 x 8192) — whose arithmetic intensity (<= 32 flop/B) puts
// them on the HBM roof: algorithmic bytes = (K + P) * L * sizeof(T) per sample, moved exactly once.
//
// Two layouts (after the planner's mode merging), L = long extent, K = contraction, P = short free extent:
//   mode A:  C[p][l] = sum_k S[p][k] * X[k][l]     X rows and C rows contiguous along l   (S is operand a)
//   mode D:  C[l][p] = sum_k X[l][k] * S[k][p]     X rows contiguous along k, C rows along p (S is operand b)
//
//  * thin_simt_{a,d}: K, P <= 8 — CUDA cores; every thread owns 16-byte vectors of X and of C.
//  * thin_mma_kernel : K in {16,32,64}, P <= 64, bf16/f16 — warp-level mma.sync.m16n8k16 with operands
//    loaded straight from global memory into fragments: no shared-memory staging of the stream, no block
//    barriers.  The mma column/k-slot <-> memory index maps are permuted (the contraction does not care
//    about the order of k, and a tile's columns can be any 8 columns) so that every thread's loads and
//    stores are 8/16-byte vectors and every warp instruction covers whole 32-byte sectors.
#include "common.cuh"
#include <algorithm>
#include <vector>

namespace tnb {

struct ThinParams {
  const void* X; const void* S; void* C;
  int64_t L;              // long extent (per batch sample)
  int K, P;
  int64_t sXl, sXk;       // X strides (elements) along l and k
  int64_t sCl;            // C stride along l (mode D); mode A: C rows are contiguous along l
  int64_t sSk;            // S stride along k
  int64_t bX, bS, bC;     // batch strides
  int64_t batch;
  DevModes mP;            // short free modes: s0 = offset in S, s1 = offset in C (mode A: row offsets)
};

enum ThinKind { THIN_SIMT = 0, THIN_MMA = 1, THIN_MMA_TF32 = 2 };   // kernel family of a thin step

template <typename T> struct Vec16 { static constexpr int N = 16 / (int)sizeof(T); };

__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }

// ------------------------------------------------------------------------------------------ SIMT, mode A
template <typename T> struct alignas(16) Pack16 { T v[Vec16<T>::N]; };

// One 16-byte unit of columns: C[i][cols] = sum_{k < K} w[k][i] * X[k][cols], fp32 fma in ascending k, rounded to T
// on the store.  cp points at the unit's first column of C row 0; row i lives at cp + co[i].  Shared by the per-step
// kernel and the fused run, so that both round the same values.
template <typename T, typename Acc, int KK, int PP>
__device__ __forceinline__ void simt_a_unit(const Acc (&w)[KK][PP], const Pack16<T> (&x)[KK], int K, int P, T* cp,
                                            const long long (&co)[PP]) {
  constexpr int VE = Vec16<T>::N;
  Acc acc[PP][VE];
#pragma unroll
  for (int i = 0; i < PP; ++i)
#pragma unroll
    for (int v = 0; v < VE; ++v) acc[i][v] = acc_zero((Acc*)nullptr);
#pragma unroll
  for (int k = 0; k < KK; ++k)
    if (k < K) {
#pragma unroll
      for (int v = 0; v < VE; ++v) {
        const Acc xv = to_acc(x[k].v[v]);
#pragma unroll
        for (int i = 0; i < PP; ++i) fma_acc(acc[i][v], w[k][i], xv);
      }
    }
#pragma unroll
  for (int i = 0; i < PP; ++i)
    if (i < P) {
      Pack16<T> o;
#pragma unroll
      for (int v = 0; v < VE; ++v) o.v[v] = FromAcc<T, Acc>::f(acc[i][v]);
      *reinterpret_cast<uint4*>(cp + co[i]) = *reinterpret_cast<uint4*>(&o);
    }
}

// KK / PP: compile-time upper bounds (2, 4, 8) of the runtime K and P, so that small problems keep few
// registers (high occupancy = more bytes in flight); U units of 16 bytes per thread are loaded before use.
template <typename T, typename Acc, int KK, int PP>
__global__ void __launch_bounds__(256) thin_simt_a_kernel(const __grid_constant__ ThinParams p) {
  constexpr int VE = Vec16<T>::N;
  constexpr int U = (KK * PP <= 16) ? 2 : 1;
  __shared__ __align__(16) Acc sS[KK][PP];    // [k][p], zero padded
  __shared__ long long cOff[PP];
  const int64_t bb = blockIdx.y;
  const T* Xb = (const T*)p.X + bb * p.bX;
  const T* Sb = (const T*)p.S + bb * p.bS;
  T* Cb = (T*)p.C + bb * p.bC;
  if (threadIdx.x < KK * PP) {
    const int k = threadIdx.x / PP, pp = threadIdx.x % PP;
    Acc v = acc_zero((Acc*)nullptr);
    if (pp < p.P) {
      int64_t os, oc;
      mode_offsets(p.mP, pp, os, oc);
      if (k < p.K) v = to_acc(Sb[os + k * p.sSk]);
      if (k == 0) cOff[pp] = oc;
    }
    sS[k][pp] = v;
  }
  __syncthreads();
  Acc w[KK][PP];
#pragma unroll
  for (int k = 0; k < KK; ++k)
#pragma unroll
    for (int i = 0; i < PP; ++i) w[k][i] = sS[k][i];
  long long co[PP];
#pragma unroll
  for (int i = 0; i < PP; ++i) co[i] = i < p.P ? cOff[i] : 0;
  const int64_t nunits = p.L / VE;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; u0 < nunits; u0 += stride * U) {
    Pack16<T> x[U][KK];
#pragma unroll
    for (int j = 0; j < U; ++j)
      if (u0 + j * stride < nunits) {
        const T* xp = Xb + (u0 + j * stride) * VE;
#pragma unroll
        for (int k = 0; k < KK; ++k)
          if (k < p.K) *reinterpret_cast<uint4*>(&x[j][k]) = ldg16(xp + k * p.sXk);
      }
#pragma unroll
    for (int j = 0; j < U; ++j)
      if (u0 + j * stride < nunits) simt_a_unit<T, Acc, KK, PP>(w, x[j], p.K, p.P, Cb + (u0 + j * stride) * VE, co);
  }
}

// ------------------------------------------------------------------------------------------ SIMT, mode D
// X rows (K contiguous elements) packed back to back, C rows (P contiguous elements) packed: thread owns
// a "unit" of UE = max(16B, one row) input elements = R whole rows and writes R*P contiguous outputs.
template <typename T, int KK, int PP> struct SimtD {
  static constexpr int VE = Vec16<T>::N;
  static constexpr int UE = VE > KK ? VE : KK;  // input elements per unit
  static constexpr int R = UE / KK;             // rows per unit
  static constexpr int NV = UE / VE;            // 16-byte vectors loaded per unit
  static constexpr int OE = R * PP;             // output elements per unit
  static constexpr int OB = OE * (int)sizeof(T);// output bytes per unit (power of two)
};

// One unit: C[r][j] = sum_k X[r][k] * w[k][j], fp32 fma in ascending k, rounded to T and stored at cp (R*P contiguous
// elements).  Shared by the per-step kernel and the fused run.
template <typename T, typename Acc, int KK, int PP>
__device__ __forceinline__ void simt_d_unit(const Acc (&w)[KK][PP], const Pack16<T> (&x)[SimtD<T, KK, PP>::NV], T* cp) {
  using G = SimtD<T, KK, PP>;
  constexpr int VE = G::VE, R = G::R, OE = G::OE, OB = G::OB;
  struct alignas(OB >= 16 ? 16 : OB) Out { T v[OE]; };
  Out o;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    Acc acc[PP];
#pragma unroll
    for (int j = 0; j < PP; ++j) acc[j] = acc_zero((Acc*)nullptr);
#pragma unroll
    for (int k = 0; k < KK; ++k) {
      const int e = r * KK + k;
      const Acc xv = to_acc(x[e / VE].v[e % VE]);
#pragma unroll
      for (int j = 0; j < PP; ++j) fma_acc(acc[j], xv, w[k][j]);
    }
#pragma unroll
    for (int j = 0; j < PP; ++j) o.v[r * PP + j] = FromAcc<T, Acc>::f(acc[j]);
  }
  if constexpr (OB >= 16) {
#pragma unroll
    for (int v = 0; v < OB / 16; ++v) reinterpret_cast<uint4*>(cp)[v] = reinterpret_cast<uint4*>(&o)[v];
  } else if constexpr (OB == 8) {
    *reinterpret_cast<uint2*>(cp) = *reinterpret_cast<uint2*>(&o);
  } else if constexpr (OB == 4) {
    *reinterpret_cast<uint32_t*>(cp) = *reinterpret_cast<uint32_t*>(&o);
  } else {
#pragma unroll
    for (int v = 0; v < OE; ++v) cp[v] = o.v[v];
  }
}

template <typename T, typename Acc, int KK, int PP>
__global__ void __launch_bounds__(256) thin_simt_d_kernel(const __grid_constant__ ThinParams p) {
  using G = SimtD<T, KK, PP>;
  constexpr int VE = G::VE, UE = G::UE, NV = G::NV, OE = G::OE;
  __shared__ Acc sS[KK][PP];
  const int64_t bb = blockIdx.y;
  const T* Xb = (const T*)p.X + bb * p.bX;
  const T* Sb = (const T*)p.S + bb * p.bS;
  T* Cb = (T*)p.C + bb * p.bC;
  if (threadIdx.x < KK * PP) {
    const int k = threadIdx.x / PP, pp = threadIdx.x % PP;
    int64_t os, oc;
    mode_offsets(p.mP, pp, os, oc);
    sS[k][pp] = to_acc(Sb[os + k * p.sSk]);
  }
  __syncthreads();
  Acc w[KK][PP];
#pragma unroll
  for (int k = 0; k < KK; ++k)
#pragma unroll
    for (int i = 0; i < PP; ++i) w[k][i] = sS[k][i];
  const int64_t nunits = p.L * KK / UE;
  constexpr int U = 4;                          // units in flight per thread
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; u0 < nunits; u0 += stride * U) {
    Pack16<T> x[U][NV];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int64_t u = u0 + i * stride;
      if (u < nunits) {
#pragma unroll
        for (int v = 0; v < NV; ++v) *reinterpret_cast<uint4*>(&x[i][v]) = ldg16(Xb + u * UE + v * VE);
      }
    }
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int64_t u = u0 + i * stride;
      if (u < nunits) simt_d_unit<T, Acc, KK, PP>(w, x[i], Cb + u * OE);
    }
  }
}

// ------------------------------------------------------------------------------------------ warp MMA
template <typename T> struct MmaOp;
template <> struct MmaOp<__nv_bfloat16> {
  __device__ static __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  __device__ static __forceinline__ uint32_t pack(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};
template <> struct MmaOp<__half> {
  __device__ static __forceinline__ void mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
  __device__ static __forceinline__ uint32_t pack(float lo, float hi) {
    __half2 v = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
  }
};

// 16-byte load: read-only global path for the per-step kernels, a plain (generic) load where the operand may sit in
// shared memory (the fused run).
template <bool GLOBAL> __device__ __forceinline__ uint4 ld16(const void* p) {
  if constexpr (GLOBAL) return ldg16(p);
  else return *reinterpret_cast<const uint4*>(p);
}
template <bool GLOBAL> __device__ __forceinline__ uint2 ld8(const void* p) {
  if constexpr (GLOBAL) return __ldg(reinterpret_cast<const uint2*>(p));
  else return *reinterpret_cast<const uint2*>(p);
}

// S staged in shared memory as [p][k] rows of PITCH = 16 KT + 8 elements, rows >= P zero.
template <int KT> struct MmaPitch { static constexpr int V = 16 * KT + 8; };

// ---- mode A: S is the mma A operand (row-major [p][k]); X[k][l] supplies B fragments.  k-step t, slot s <-> k = 16 t + s.
template <typename T, int KT, int PT>
__device__ __forceinline__ void mma_a_frags(const T* sS, uint32_t (&sa)[PT][KT][4], int g, int q) {
  constexpr int PITCH = MmaPitch<KT>::V;
#pragma unroll
  for (int mt = 0; mt < PT; ++mt)
#pragma unroll
    for (int t = 0; t < KT; ++t) {
      const T* r0 = sS + (16 * mt + g) * PITCH + 16 * t + 2 * q;
      const T* r1 = r0 + 8 * PITCH;
      sa[mt][t][0] = *reinterpret_cast<const uint32_t*>(r0);
      sa[mt][t][1] = *reinterpret_cast<const uint32_t*>(r1);
      sa[mt][t][2] = *reinterpret_cast<const uint32_t*>(r0 + 8);
      sa[mt][t][3] = *reinterpret_cast<const uint32_t*>(r1 + 8);
    }
}

// One warp, one 64-column block: C[p][l0 + c] = sum_k S[p][k] X[k][l0 + c] for p < P.  xp = X + l0 + colbase (tile
// column g of mma j <-> c = colbase + j), cb = C + l0 + 8 q; row p of C starts at cb + cOff[p].
template <typename T, int KT, int PT, bool GLOBAL>
__device__ __forceinline__ void mma_a_block(const uint32_t (&sa)[PT][KT][4], const T* xp, int64_t sXk, T* cb,
                                            const long long* cOff, int P, int g, int q) {
  uint32_t xb[KT][2][8];                 // [k-step][slot half][j]: B fragment words
#pragma unroll
  for (int t = 0; t < KT; ++t)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 16 * t + 2 * q + 8 * h;
      const uint4 a = ld16<GLOBAL>(xp + (int64_t)row * sXk);
      const uint4 b = ld16<GLOBAL>(xp + (int64_t)(row + 1) * sXk);
      xb[t][h][0] = a.x; xb[t][h][1] = b.x; xb[t][h][2] = a.y; xb[t][h][3] = b.y;
      xb[t][h][4] = a.z; xb[t][h][5] = b.z; xb[t][h][6] = a.w; xb[t][h][7] = b.w;
    }
  // interleave the two rows of every pair: word (2w, 2w+1) = (row, row+1) elements 2w / 2w+1
#pragma unroll
  for (int t = 0; t < KT; ++t)
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const uint32_t a = xb[t][h][2 * w], b = xb[t][h][2 * w + 1];
        xb[t][h][2 * w] = __byte_perm(a, b, 0x5410);
        xb[t][h][2 * w + 1] = __byte_perm(a, b, 0x7632);
      }
#pragma unroll
  for (int mt = 0; mt < PT; ++mt) {
    if (16 * mt >= P) break;
    float acc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
#pragma unroll
    for (int t = 0; t < KT; ++t)
#pragma unroll
      for (int j = 0; j < 8; ++j) MmaOp<T>::mma(acc[j], sa[mt][t], xb[t][0][j], xb[t][1][j]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 16 * mt + g + 8 * h;
      if (row < P) {
        T* cp = cb + cOff[row];
        uint4 v0, v1;
        v0.x = MmaOp<T>::pack(acc[0][2 * h], acc[1][2 * h]); v0.y = MmaOp<T>::pack(acc[2][2 * h], acc[3][2 * h]);
        v0.z = MmaOp<T>::pack(acc[4][2 * h], acc[5][2 * h]); v0.w = MmaOp<T>::pack(acc[6][2 * h], acc[7][2 * h]);
        v1.x = MmaOp<T>::pack(acc[0][2 * h + 1], acc[1][2 * h + 1]); v1.y = MmaOp<T>::pack(acc[2][2 * h + 1], acc[3][2 * h + 1]);
        v1.z = MmaOp<T>::pack(acc[4][2 * h + 1], acc[5][2 * h + 1]); v1.w = MmaOp<T>::pack(acc[6][2 * h + 1], acc[7][2 * h + 1]);
        *reinterpret_cast<uint4*>(cp) = v0;
        *reinterpret_cast<uint4*>(cp + 32) = v1;
      }
    }
  }
}

// ---- mode D: X rows are the mma A operand (k contiguous); S[k][p] supplies B fragments.  Thread q owns the k-chunk
// [4 KT q, 4 KT (q + 1)): k-step t, slot 2 q + 8 h + e <-> k = 4 KT q + 4 t + 2 h + e.
template <int PT> struct MmaD {
  static constexpr int NP8 = 2 * PT;                       // 8-column tiles of the output row
  static constexpr int PTP = NP8 < 4 ? NP8 : 4;            // tiles per 16-byte (or 8-byte) output piece
};
template <typename T, int KT, int PT>
__device__ __forceinline__ void mma_d_frags(const T* sS, uint32_t (&sb)[KT][2 * PT][2], int g, int q) {
  constexpr int PITCH = MmaPitch<KT>::V, NP8 = MmaD<PT>::NP8, PTP = MmaD<PT>::PTP;
#pragma unroll
  for (int t = 0; t < KT; ++t)
#pragma unroll
    for (int pt = 0; pt < NP8; ++pt) {
      const int pcol = (pt / PTP) * (8 * PTP) + (g >> 1) * (2 * PTP) + 2 * (pt % PTP) + (g & 1);
      const T* r = sS + pcol * PITCH + 4 * KT * q + 4 * t;
      sb[t][pt][0] = *reinterpret_cast<const uint32_t*>(r);
      sb[t][pt][1] = *reinterpret_cast<const uint32_t*>(r + 2);
    }
}

// One warp, one 64-row block: C[l0 + r][p] = sum_k X[l0 + r][k] S[k][p].  xr = X + l0 sXl, cr = C + l0 sCl.
template <typename T, int KT, int PT, bool GLOBAL>
__device__ __forceinline__ void mma_d_block(const uint32_t (&sb)[KT][2 * PT][2], const T* xr, int64_t sXl, T* cr,
                                            int64_t sCl, int g, int q) {
  constexpr int NP8 = MmaD<PT>::NP8, PTP = MmaD<PT>::PTP;
  uint32_t xa[4][2][2 * KT];
#pragma unroll
  for (int rg = 0; rg < 4; ++rg)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const T* rp = xr + (16 * rg + 8 * h + g) * sXl + 4 * KT * q;
      if constexpr (KT == 1) {
        const uint2 v = ld8<GLOBAL>(rp);
        xa[rg][h][0] = v.x; xa[rg][h][1] = v.y;
      } else {
#pragma unroll
        for (int v4 = 0; v4 < KT / 2; ++v4) {
          const uint4 v = ld16<GLOBAL>(rp + 8 * v4);
          xa[rg][h][4 * v4] = v.x; xa[rg][h][4 * v4 + 1] = v.y; xa[rg][h][4 * v4 + 2] = v.z; xa[rg][h][4 * v4 + 3] = v.w;
        }
      }
    }
#pragma unroll
  for (int rg = 0; rg < 4; ++rg) {
    float acc[NP8][4];
#pragma unroll
    for (int pt = 0; pt < NP8; ++pt) { acc[pt][0] = acc[pt][1] = acc[pt][2] = acc[pt][3] = 0.f; }
#pragma unroll
    for (int t = 0; t < KT; ++t) {
      const uint32_t a[4] = {xa[rg][0][2 * t], xa[rg][1][2 * t], xa[rg][0][2 * t + 1], xa[rg][1][2 * t + 1]};
#pragma unroll
      for (int pt = 0; pt < NP8; ++pt) MmaOp<T>::mma(acc[pt], a, sb[t][pt][0], sb[t][pt][1]);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      T* cp = cr + (16 * rg + 8 * h + g) * sCl + 2 * PTP * q;
      if constexpr (NP8 == 2) {
        uint2 v;
        v.x = MmaOp<T>::pack(acc[0][2 * h], acc[0][2 * h + 1]);
        v.y = MmaOp<T>::pack(acc[1][2 * h], acc[1][2 * h + 1]);
        *reinterpret_cast<uint2*>(cp) = v;
      } else {
#pragma unroll
        for (int piece = 0; piece < NP8 / 4; ++piece) {
          uint4 v;
          v.x = MmaOp<T>::pack(acc[4 * piece + 0][2 * h], acc[4 * piece + 0][2 * h + 1]);
          v.y = MmaOp<T>::pack(acc[4 * piece + 1][2 * h], acc[4 * piece + 1][2 * h + 1]);
          v.z = MmaOp<T>::pack(acc[4 * piece + 2][2 * h], acc[4 * piece + 2][2 * h + 1]);
          v.w = MmaOp<T>::pack(acc[4 * piece + 3][2 * h], acc[4 * piece + 3][2 * h + 1]);
          *reinterpret_cast<uint4*>(cp + 32 * piece) = v;
        }
      }
    }
  }
}

// K = 16*KT exactly; P <= 16*PT (mode A: any P, rows masked; mode D: P == 16*PT).  One warp per 64-l block.
template <typename T, int KT, int PT, int MODE>
__global__ void __launch_bounds__(256) thin_mma_kernel(const __grid_constant__ ThinParams p) {
  constexpr int KK = 16 * KT, PP = 16 * PT, PITCH = MmaPitch<KT>::V;
  __shared__ __align__(16) T sS[PP * PITCH];   // S as [p][k], zero padded rows
  __shared__ long long cOff[PP];
  const int64_t bb = blockIdx.y;
  const T* Xb = (const T*)p.X + bb * p.bX;
  const T* Sb = (const T*)p.S + bb * p.bS;
  T* Cb = (T*)p.C + bb * p.bC;
  for (int idx = threadIdx.x; idx < PP * KK; idx += blockDim.x) {
    const int pp = idx / KK, k = idx % KK;
    T v = FromAcc<T, float>::f(0.f);
    if (pp < p.P) {
      int64_t os, oc;
      mode_offsets(p.mP, pp, os, oc);
      v = Sb[os + k * p.sSk];
      if (k == 0) cOff[pp] = oc;
    }
    sS[pp * PITCH + k] = v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, q = lane & 3;
  const int64_t nblk = p.L >> 6;
  const int64_t wstride = (int64_t)gridDim.x * (blockDim.x >> 5);

  if constexpr (MODE == 0) {
    uint32_t sa[PT][KT][4];
    mma_a_frags<T, KT, PT>(sS, sa, g, q);
    const int colbase = 32 * (g & 1) + 8 * (g >> 1);   // tile column g of mma j  <->  l = l0 + colbase + j
    for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; blk < nblk; blk += wstride) {
      const int64_t l0 = blk << 6;
      mma_a_block<T, KT, PT, true>(sa, Xb + l0 + colbase, p.sXk, Cb + l0 + 8 * q, cOff, p.P, g, q);
    }
  } else {
    uint32_t sb[KT][2 * PT][2];
    mma_d_frags<T, KT, PT>(sS, sb, g, q);
    for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; blk < nblk; blk += wstride) {
      const int64_t l0 = blk << 6;
      mma_d_block<T, KT, PT, true>(sb, Xb + l0 * p.sXl, p.sXl, Cb + l0 * p.sCl, p.sCl, g, q);
    }
  }
}


// ------------------------------------------------------------------------------------------ warp MMA, fp32 as TF32
// Same scheme with mma.sync.m16n8k8 (tf32 inputs = the fp32 bit patterns, fp32 accumulate — the precision class of the
// wgmma tf32 path these shapes would otherwise take).  K = 8*KT8 in {16, 32, 64}; P <= 16*PT.
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int KT8, int PT, int MODE>
__global__ void __launch_bounds__(256) thin_mma32_kernel(const __grid_constant__ ThinParams p) {
  constexpr int KK = 8 * KT8, PP = 16 * PT, PITCH = KK + 4;
  __shared__ __align__(16) float sS[PP * PITCH];   // S as [p][k], zero padded rows
  __shared__ long long cOff[PP];
  const int64_t bb = blockIdx.y;
  const float* Xb = (const float*)p.X + bb * p.bX;
  const float* Sb = (const float*)p.S + bb * p.bS;
  float* Cb = (float*)p.C + bb * p.bC;
  for (int idx = threadIdx.x; idx < PP * KK; idx += blockDim.x) {
    const int pp = idx / KK, k = idx % KK;
    float v = 0.f;
    if (pp < p.P) {
      int64_t os, oc;
      mode_offsets(p.mP, pp, os, oc);
      v = Sb[os + k * p.sSk];
      if (k == 0) cOff[pp] = oc;
    }
    sS[pp * PITCH + k] = v;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, q = lane & 3;
  const int64_t wstride = (int64_t)gridDim.x * (blockDim.x >> 5);

  if constexpr (MODE == 0) {
    // ---- mode A: 32 long-indices per warp block; tile column c of mma j  <->  l = l0 + 16 (c & 1) + 4 (c >> 1) + j
    const int64_t nblk = p.L >> 5;
    const int colbase = 16 * (g & 1) + 4 * (g >> 1);
    for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; blk < nblk; blk += wstride) {
      const int64_t l0 = blk << 5;
      const float* xp = Xb + l0 + colbase;
      uint4 x[KT8][2];
#pragma unroll
      for (int t = 0; t < KT8; ++t)
#pragma unroll
        for (int h = 0; h < 2; ++h) x[t][h] = ldg16(xp + (int64_t)(8 * t + q + 4 * h) * p.sXk);
#pragma unroll
      for (int mt = 0; mt < PT; ++mt) {
        if (16 * mt >= p.P) break;
        float acc[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j) { acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f; }
#pragma unroll
        for (int t = 0; t < KT8; ++t) {
          const float* r0 = sS + (16 * mt + g) * PITCH + 8 * t + q;
          const uint32_t a[4] = {__float_as_uint(r0[0]), __float_as_uint(r0[8 * PITCH]), __float_as_uint(r0[4]),
                                 __float_as_uint(r0[8 * PITCH + 4])};
          mma_tf32(acc[0], a, x[t][0].x, x[t][1].x);
          mma_tf32(acc[1], a, x[t][0].y, x[t][1].y);
          mma_tf32(acc[2], a, x[t][0].z, x[t][1].z);
          mma_tf32(acc[3], a, x[t][0].w, x[t][1].w);
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = 16 * mt + g + 8 * h;
          if (row < p.P) {
            float* cp = Cb + cOff[row] + l0 + 4 * q;
            *reinterpret_cast<float4*>(cp) = make_float4(acc[0][2 * h], acc[1][2 * h], acc[2][2 * h], acc[3][2 * h]);
            *reinterpret_cast<float4*>(cp + 16) = make_float4(acc[0][2 * h + 1], acc[1][2 * h + 1], acc[2][2 * h + 1], acc[3][2 * h + 1]);
          }
        }
      }
    }
  } else {
    // ---- mode D: X rows are the A operand; thread q owns the contiguous k-chunk [2 KT8 q, 2 KT8 (q + 1)) of a row:
    // k-step t, slot q + 4h  <->  k = 2 KT8 q + 2 t + h.  Output column c of tile pt  <->  p = 16 (pt / 2) + 4 (c >> 1)
    // + 2 (pt % 2) + (c & 1), so a thread's two tiles of a piece are 4 consecutive floats.
    constexpr int NP8 = 2 * PT;
    constexpr int RG = KT8 == 8 ? 2 : 4;                  // 16-row groups per warp block
    const int64_t nblk = p.L / (16 * RG);
    for (int64_t blk = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp; blk < nblk; blk += wstride) {
      const int64_t l0 = blk * (16 * RG);
      uint32_t xa[RG][2][2 * KT8];
#pragma unroll
      for (int rg = 0; rg < RG; ++rg)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* rp = Xb + (l0 + 16 * rg + 8 * h + g) * p.sXl + 2 * KT8 * q;
#pragma unroll
          for (int v4 = 0; v4 < KT8 / 2; ++v4) {
            const uint4 v = ldg16(rp + 4 * v4);
            xa[rg][h][4 * v4] = v.x; xa[rg][h][4 * v4 + 1] = v.y; xa[rg][h][4 * v4 + 2] = v.z; xa[rg][h][4 * v4 + 3] = v.w;
          }
        }
#pragma unroll
      for (int rg = 0; rg < RG; ++rg) {
        float acc[NP8][4];
#pragma unroll
        for (int pt = 0; pt < NP8; ++pt) { acc[pt][0] = acc[pt][1] = acc[pt][2] = acc[pt][3] = 0.f; }
#pragma unroll
        for (int t = 0; t < KT8; ++t) {
          const uint32_t a[4] = {xa[rg][0][2 * t], xa[rg][1][2 * t], xa[rg][0][2 * t + 1], xa[rg][1][2 * t + 1]};
#pragma unroll
          for (int pt = 0; pt < NP8; ++pt) {
            const int pcol = (pt >> 1) * 16 + 4 * (g >> 1) + 2 * (pt & 1) + (g & 1);
            const float2 b = *reinterpret_cast<const float2*>(sS + pcol * PITCH + 2 * KT8 * q + 2 * t);
            mma_tf32(acc[pt], a, __float_as_uint(b.x), __float_as_uint(b.y));
          }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* cp = Cb + (l0 + 16 * rg + 8 * h + g) * p.sCl + 4 * q;
#pragma unroll
          for (int piece = 0; piece < NP8 / 2; ++piece)
            *reinterpret_cast<float4*>(cp + 16 * piece) =
                make_float4(acc[2 * piece][2 * h], acc[2 * piece][2 * h + 1], acc[2 * piece + 1][2 * h], acc[2 * piece + 1][2 * h + 1]);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ fused thin run
// A run of 2..8 thin steps of one mode in which step j+1 streams step j's result, as in the ramps of an MPS
// contraction: mode A, C_j[(k', m)][l] = X_{j+1}[k'][m L_j + l]; mode D, C_j[l][(m, k')] = X_{j+1}[l R_j + m][k'].
// Either way 64 long indices of the first step (a "slab": 64 columns in mode A, 64 rows in mode D) determine a
// fixed set of at most 4096 elements of every later operand and result, so one warp carries a slab through all
// the steps in shared memory: the first X is read from HBM once and only the last C is written.  Each step calls
// the per-step kernels' arithmetic (simt_*_unit, mma_*_block) and rounds to T where they store, so the result is
// bit-identical to launching the steps one by one.  Persistent: each CTA takes an equal share of (sample, slab).
constexpr int kRunMaxSteps = 8, kRunWarps = 8, kRunSlab = 4096;

struct ThinRunStep {
  const void* S; int64_t bS, sSk;
  int K, P, kind;         // kind: THIN_SIMT or THIN_MMA
  int W;                  // long extent of this step inside one slab (mode A: columns, mode D: rows)
  int64_t L;              // long extent of this step per sample
  int soff;               // byte offset of the staged S in shared memory
};
struct ThinRunParams {
  const void* X; void* C;
  int64_t sX, bX;         // first X: stride along k (mode A) / l (mode D), batch stride
  int64_t sC, bC;         // last C: stride along l (mode D), batch stride
  int64_t batch, nslab;
  int nsteps, smem_s;     // smem_s: bytes of staged S, followed by the C row offsets and the warps' slab buffers
  const long long* tab;   // device [nsteps][2][64]: S offset of row p; C offset of row p (inside the slab buffer for
                          // intermediate steps, in global memory for the last step; mode A only)
  ThinRunStep st[kRunMaxSteps];
};

__device__ __forceinline__ int run_pt(int P) { return (P + 15) / 16 <= 1 ? 1 : ((P + 15) / 16 <= 2 ? 2 : 4); }

// mode A: column of the last step's C (per sample) holding column n of the slab's last-step frame
__device__ __forceinline__ int64_t run_col(const ThinRunParams& p, int64_t slab, int n) {
  int64_t l = slab * 64;
  for (int j = p.nsteps - 2; j >= 0; --j) { l += (int64_t)(n / p.st[j].W) * p.st[j].L; n %= p.st[j].W; }
  return l + n;
}

template <typename T, int KT, int PT, int MODE>
__device__ __forceinline__ void run_mma(const ThinRunParams& p, int j, const unsigned char* smem, const long long* cOff,
                                        const T* x, int64_t sX, T* c, int64_t sC, bool last, int64_t slab, int g, int q) {
  const ThinRunStep& st = p.st[j];
  const T* sS = reinterpret_cast<const T*>(smem + st.soff);
  if constexpr (MODE == 0) {
    uint32_t sa[PT][KT][4];
    mma_a_frags<T, KT, PT>(sS, sa, g, q);
    const int colbase = 32 * (g & 1) + 8 * (g >> 1);
    for (int n0 = 0; n0 < st.W; n0 += 64)
      mma_a_block<T, KT, PT, false>(sa, x + n0 + colbase, sX, c + (last ? run_col(p, slab, n0) : n0) + 8 * q, cOff,
                                    st.P, g, q);
  } else {
    uint32_t sb[KT][2 * PT][2];
    mma_d_frags<T, KT, PT>(sS, sb, g, q);
    for (int n0 = 0; n0 < st.W; n0 += 64) mma_d_block<T, KT, PT, false>(sb, x + n0 * sX, sX, c + n0 * sC, sC, g, q);
  }
}

template <typename T, int KK, int PP, int MODE>
__device__ __forceinline__ void run_simt(const ThinRunParams& p, int j, const unsigned char* smem, const long long* cOff,
                                         const T* x, int64_t sX, T* c, bool last, int64_t slab, int lane) {
  using Acc = float;
  constexpr int VE = Vec16<T>::N;
  const ThinRunStep& st = p.st[j];
  const Acc* sS = reinterpret_cast<const Acc*>(smem + st.soff);
  Acc w[KK][PP];
#pragma unroll
  for (int k = 0; k < KK; ++k)
#pragma unroll
    for (int i = 0; i < PP; ++i) w[k][i] = sS[k * PP + i];
  if constexpr (MODE == 0) {
    long long co[PP];
#pragma unroll
    for (int i = 0; i < PP; ++i) co[i] = cOff[i];
    for (int u = lane; u < st.W / VE; u += 32) {
      Pack16<T> xv[KK];
#pragma unroll
      for (int k = 0; k < KK; ++k) *reinterpret_cast<uint4*>(&xv[k]) = ld16<false>(x + k * sX + u * VE);
      simt_a_unit<T, Acc, KK, PP>(w, xv, KK, PP, c + (last ? run_col(p, slab, u * VE) : u * VE), co);
    }
  } else {
    using G = SimtD<T, KK, PP>;
    for (int u = lane; u < st.W * KK / G::UE; u += 32) {   // X and C packed: sX == K, C rows of P elements
      Pack16<T> xv[G::NV];
#pragma unroll
      for (int v = 0; v < G::NV; ++v) *reinterpret_cast<uint4*>(&xv[v]) = ld16<false>(x + u * G::UE + v * VE);
      simt_d_unit<T, Acc, KK, PP>(w, xv, c + u * G::OE);
    }
  }
}

template <typename T, int MODE>
__global__ void __launch_bounds__(256, 1) thin_run_kernel(const __grid_constant__ ThinRunParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  long long* cOff = reinterpret_cast<long long*>(smem + p.smem_s);
  T* bufs = reinterpret_cast<T*>(cOff + kRunMaxSteps * 64);
  for (int i = threadIdx.x; i < p.nsteps * 64; i += blockDim.x) cOff[i] = p.tab[(i / 64) * 128 + 64 + i % 64];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, q = lane & 3;
  T* const wbuf = bufs + warp * 2 * kRunSlab;      // this warp's two slab buffers (step j writes buffer j & 1)
  const int64_t total = p.batch * p.nslab;
  const int64_t beg = total * blockIdx.x / gridDim.x, end = total * (blockIdx.x + 1) / gridDim.x;
  for (int64_t s0 = beg; s0 < end;) {
    const int64_t b = s0 / p.nslab;
    const int64_t s1 = (b + 1) * p.nslab < end ? (b + 1) * p.nslab : end;
    __syncthreads();                      // every warp is done with the previous sample's S
    for (int j = 0; j < p.nsteps; ++j) {  // stage this sample's S of every step, as the per-step kernels do
      const ThinRunStep& st = p.st[j];
      const T* Sb = (const T*)st.S + b * st.bS;
      const long long* sOff = p.tab + j * 128;
      if (st.kind == THIN_MMA) {
        T* sS = reinterpret_cast<T*>(smem + st.soff);
        const int PP = 16 * run_pt(st.P), pitch = st.K + 8;
        for (int idx = threadIdx.x; idx < PP * st.K; idx += blockDim.x) {
          const int pp = idx / st.K, k = idx % st.K;
          sS[pp * pitch + k] = pp < st.P ? Sb[sOff[pp] + k * st.sSk] : FromAcc<T, float>::f(0.f);
        }
      } else {
        float* sS = reinterpret_cast<float*>(smem + st.soff);
        for (int idx = threadIdx.x; idx < st.K * st.P; idx += blockDim.x) {
          const int k = idx / st.P, pp = idx % st.P;
          sS[idx] = to_acc(Sb[sOff[pp] + k * st.sSk]);
        }
      }
    }
    __syncthreads();
    for (int64_t it = s0 + warp; it < s1; it += kRunWarps) {
      const int64_t slab = it - b * p.nslab;
      for (int j = 0; j < p.nsteps; ++j) {
        const ThinRunStep& st = p.st[j];
        const bool first = j == 0, last = j == p.nsteps - 1;
        const T* x = first ? (const T*)p.X + b * p.bX + slab * 64 * (MODE == 0 ? 1 : p.sX) : wbuf + ((j - 1) & 1) * kRunSlab;
        const int64_t sX = first ? p.sX : (MODE == 0 ? st.W : st.K);
        T* c = last ? (T*)p.C + b * p.bC + (MODE == 0 ? 0 : slab * st.W * p.sC) : wbuf + (j & 1) * kRunSlab;
        const int64_t sC = last ? p.sC : st.P;
        const long long* co = cOff + j * 64;
        if (st.kind == THIN_MMA) {
          const int kt = st.K / 16, pt = run_pt(st.P);
#define TNB_RUN_M(KT, PT) \
  if (kt == KT && pt == PT) run_mma<T, KT, PT, MODE>(p, j, smem, co, x, sX, c, sC, last, slab, g, q); else
          TNB_RUN_M(1, 1) TNB_RUN_M(1, 2) TNB_RUN_M(1, 4) TNB_RUN_M(2, 1) TNB_RUN_M(2, 2) TNB_RUN_M(2, 4)
          TNB_RUN_M(4, 1) TNB_RUN_M(4, 2) TNB_RUN_M(4, 4) {}
#undef TNB_RUN_M
        } else {
#define TNB_RUN_S(KK, PP) \
  if (st.K == KK && st.P == PP) run_simt<T, KK, PP, MODE>(p, j, smem, co, x, sX, c, last, slab, lane); else
          TNB_RUN_S(2, 2) TNB_RUN_S(2, 4) TNB_RUN_S(2, 8) TNB_RUN_S(4, 2) TNB_RUN_S(4, 4) TNB_RUN_S(4, 8)
          TNB_RUN_S(8, 2) TNB_RUN_S(8, 4) TNB_RUN_S(8, 8) {}
#undef TNB_RUN_S
        }
        __syncwarp();                     // this step's result is the next step's operand (or buffer to overwrite)
      }
    }
    s0 = s1;
  }
}

// ------------------------------------------------------------------------------------------ host side
static inline unsigned thin_grid_x(int64_t work_items, int64_t batch, int ctas_per_sm) {
  int64_t want = ((int64_t)num_sms() * ctas_per_sm + batch - 1) / batch;
  int64_t cap = (work_items + 255) / 256;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  return (unsigned)want;
}

template <int DT>
static int launch_simt(int mode, const ThinParams& p, cudaStream_t st) {
  using T = typename DType<DT>::T;
  using Acc = typename DType<DT>::Acc;
  constexpr int VE = 16 / (int)sizeof(T);
  if (mode == 0) {
    const int kk = p.K <= 2 ? 2 : (p.K <= 4 ? 4 : 8), pp = p.P <= 2 ? 2 : (p.P <= 4 ? 4 : 8);
    dim3 grid(thin_grid_x(p.L / VE, p.batch, 8), (unsigned)p.batch);
#define TNB_THIN_A(KK, PP) if (kk == KK && pp == PP) thin_simt_a_kernel<T, Acc, KK, PP><<<grid, 256, 0, st>>>(p);
    TNB_THIN_A(2, 2) TNB_THIN_A(2, 4) TNB_THIN_A(2, 8)
    TNB_THIN_A(4, 2) TNB_THIN_A(4, 4) TNB_THIN_A(4, 8)
    TNB_THIN_A(8, 2) TNB_THIN_A(8, 4) TNB_THIN_A(8, 8)
#undef TNB_THIN_A
    TNB_LAUNCH_CHECK();
    count_launch();
    set_kernel_name("thin_simt_a");
    return 0;
  }
#define TNB_THIN_D(KK, PP)                                                                         \
  if (p.K == KK && p.P == PP) {                                                                    \
    constexpr int UE = VE > KK ? VE : KK;                                                          \
    dim3 grid(thin_grid_x(p.L * KK / UE / 4, p.batch, 8), (unsigned)p.batch);                      \
    thin_simt_d_kernel<T, Acc, KK, PP><<<grid, 256, 0, st>>>(p);                                   \
    TNB_LAUNCH_CHECK();                                                                            \
    count_launch();                                                                                \
    set_kernel_name("thin_simt_d");                                                                \
    return 0;                                                                                      \
  }
  TNB_THIN_D(2, 2) TNB_THIN_D(2, 4) TNB_THIN_D(2, 8)
  TNB_THIN_D(4, 2) TNB_THIN_D(4, 4) TNB_THIN_D(4, 8)
  TNB_THIN_D(8, 2) TNB_THIN_D(8, 4) TNB_THIN_D(8, 8)
#undef TNB_THIN_D
  return TNB200_ERR_UNSUPPORTED;
}

template <int DT, int KT, int PT>
static int launch_mma_kp(int mode, const ThinParams& p, cudaStream_t st) {
  using T = typename DType<DT>::T;
  // registers: ~50 (16x16) .. ~190 (64x64) per thread -> 1..4 CTAs of 256 threads per SM
  const int ctas = (KT * PT >= 8) ? 1 : (KT * PT >= 4 ? 2 : 4);
  int64_t want = ((int64_t)num_sms() * ctas + p.batch - 1) / p.batch;
  const int64_t cap = ((p.L >> 6) + 7) / 8;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  dim3 grid((unsigned)want, (unsigned)p.batch);
  if (mode == 0) thin_mma_kernel<T, KT, PT, 0><<<grid, 256, 0, st>>>(p);
  else thin_mma_kernel<T, KT, PT, 1><<<grid, 256, 0, st>>>(p);
  TNB_LAUNCH_CHECK();
  count_launch();
  set_kernel_name(mode == 0 ? "thin_mma_a" : "thin_mma_d");
  return 0;
}
template <int DT>
static int launch_mma(int mode, const ThinParams& p, cudaStream_t st) {
  const int kt = p.K / 16, pt = (p.P + 15) / 16 <= 1 ? 1 : ((p.P + 15) / 16 <= 2 ? 2 : 4);
#define TNB_THIN_M(KT, PT) if (kt == KT && pt == PT) return launch_mma_kp<DT, KT, PT>(mode, p, st);
  TNB_THIN_M(1, 1) TNB_THIN_M(1, 2) TNB_THIN_M(1, 4)
  TNB_THIN_M(2, 1) TNB_THIN_M(2, 2) TNB_THIN_M(2, 4)
  TNB_THIN_M(4, 1) TNB_THIN_M(4, 2) TNB_THIN_M(4, 4)
#undef TNB_THIN_M
  return TNB200_ERR_UNSUPPORTED;
}

template <int KT8, int PT>
static int launch_mma32_kp(int mode, const ThinParams& p, cudaStream_t st) {
  const int ctas = (KT8 * PT >= 16) ? 2 : 4;
  const int64_t nblk = mode == 0 ? (p.L >> 5) : p.L / (16 * (KT8 == 8 ? 2 : 4));
  int64_t want = ((int64_t)num_sms() * ctas + p.batch - 1) / p.batch;
  const int64_t cap = (nblk + 7) / 8;
  if (want > cap) want = cap;
  if (want < 1) want = 1;
  dim3 grid((unsigned)want, (unsigned)p.batch);
  if (mode == 0) thin_mma32_kernel<KT8, PT, 0><<<grid, 256, 0, st>>>(p);
  else thin_mma32_kernel<KT8, PT, 1><<<grid, 256, 0, st>>>(p);
  TNB_LAUNCH_CHECK();
  count_launch();
  set_kernel_name(mode == 0 ? "thin_mma_tf32_a" : "thin_mma_tf32_d");
  return 0;
}
static int launch_mma32(int mode, const ThinParams& p, cudaStream_t st) {
  const int kt = p.K / 8, pt = (p.P + 15) / 16 <= 1 ? 1 : ((p.P + 15) / 16 <= 2 ? 2 : 4);
#define TNB_THIN_M32(KT8, PT) if (kt == KT8 && pt == PT) return launch_mma32_kp<KT8, PT>(mode, p, st);
  TNB_THIN_M32(2, 1) TNB_THIN_M32(2, 2) TNB_THIN_M32(2, 4)
  TNB_THIN_M32(4, 1) TNB_THIN_M32(4, 2) TNB_THIN_M32(4, 4)
  TNB_THIN_M32(8, 1) TNB_THIN_M32(8, 2) TNB_THIN_M32(8, 4)
#undef TNB_THIN_M32
  return TNB200_ERR_UNSUPPORTED;
}

static inline bool al16(const void* p) { return ((uintptr_t)p & 15) == 0; }

// The thin layout of one contraction (mode-list conventions of tensordot.cu: mB s0 A, s1 B, s2 C; mM s0 A, s1 C;
// mN s0 B, s1 C; mK s0 A, s1 B; all lists merged): its parameters, mode (0 = A, 1 = D) and kernel family.
// Returns TNB200_ERR_UNSUPPORTED when the shape / layout is not thin.
static int plan_thin(int dt, const void* A, const void* B, void* C, const ModeList& mB, const ModeList& mM,
                     const ModeList& mN, const ModeList& mK, bool allow_tf32, ThinParams& p, int& mode, int& kind) {
  if (dt != TNB200_F64 && dt != TNB200_F32 && dt != TNB200_F16 && dt != TNB200_BF16) return TNB200_ERR_UNSUPPORTED;
  if (mB.n > 1 || mK.n != 1) return TNB200_ERR_UNSUPPORTED;
  const int64_t M = mM.total(), N = mN.total(), K = mK.total(), batch = mB.total();
  if (K > 64 || batch > 65535) return TNB200_ERR_UNSUPPORTED;
  const int64_t ve = 16 / dtype_size(dt);
  const bool half_t = dt == TNB200_F16 || dt == TNB200_BF16;
  memset(&p, 0, sizeof(p));
  p.K = (int)K; p.batch = batch;
  mode = -1;
  // ---- mode A: a is the small matrix S[p][k]; b = X[k][l] with l contiguous in b and in c
  if (M <= 64 && mN.n == 1 && mN.s0[0] == 1 && mN.s1[0] == 1 && N >= 2048) {
    mode = 0;
    p.X = B; p.S = A; p.C = C; p.L = N; p.P = (int)M;
    p.sXl = 1; p.sXk = mK.s1[0]; p.sSk = mK.s0[0]; p.sCl = 1;
    p.bX = mB.n ? mB.s1[0] : 0; p.bS = mB.n ? mB.s0[0] : 0; p.bC = mB.n ? mB.s2[0] : 0;
    ModeList sp;
    for (int i = 0; i < mM.n; ++i) sp.push(mM.ext[i], mM.s0[i], mM.s1[i]);
    if (!to_dev(sp, p.mP)) return TNB200_ERR_UNSUPPORTED;
    bool ok = al16(B) && al16(C) && p.sXk % ve == 0 && p.bX % ve == 0 && p.bC % ve == 0;
    for (int i = 0; i < mM.n && ok; ++i) ok = mM.s1[i] % ve == 0;
    if (!ok) return TNB200_ERR_UNSUPPORTED;
  } else if (N <= 64 && mM.n == 1 && mK.s0[0] == 1 && M >= 2048) {
    // ---- mode D: b is the small matrix S[k][p]; a = X[l][k] with k contiguous; c rows contiguous along p
    int64_t run = 1;
    for (int i = mN.n - 1; i >= 0; --i) { if (mN.s1[i] != run) return TNB200_ERR_UNSUPPORTED; run *= mN.ext[i]; }
    mode = 1;
    p.X = A; p.S = B; p.C = C; p.L = M; p.P = (int)N;
    p.sXl = mM.s0[0]; p.sXk = 1; p.sSk = mK.s1[0]; p.sCl = mM.s1[0];
    p.bX = mB.n ? mB.s0[0] : 0; p.bS = mB.n ? mB.s1[0] : 0; p.bC = mB.n ? mB.s2[0] : 0;
    ModeList sp;
    for (int i = 0; i < mN.n; ++i) sp.push(mN.ext[i], mN.s0[i], mN.s1[i]);
    if (!to_dev(sp, p.mP)) return TNB200_ERR_UNSUPPORTED;
    if (!(al16(A) && al16(C) && p.bX % ve == 0 && p.bC % ve == 0)) return TNB200_ERR_UNSUPPORTED;
  } else {
    return TNB200_ERR_UNSUPPORTED;
  }
  if (p.L * batch < 65536) return TNB200_ERR_UNSUPPORTED;
  // ---- CUDA-core family
  if (K <= 8 && p.P <= 8) {
    if (mode == 0) {
      if (p.L % ve) return TNB200_ERR_UNSUPPORTED;
    } else {
      const int64_t ue = ve > K ? ve : K;
      if (p.sXl != K || p.sCl != p.P || (p.L * K) % ue) return TNB200_ERR_UNSUPPORTED;
      if (!((K == 2 || K == 4 || K == 8) && (p.P == 2 || p.P == 4 || p.P == 8))) return TNB200_ERR_UNSUPPORTED;
    }
    kind = THIN_SIMT;
    return 0;
  }
  // ---- warp-MMA family (16-bit types)
  if (half_t && (K == 16 || K == 32 || K == 64) && p.P > 8 && p.L % 64 == 0) {
    if (mode == 1) {
      if (!(p.P == 16 || p.P == 32 || p.P == 64)) return TNB200_ERR_UNSUPPORTED;
      if (p.sXl % 8 || p.sCl % 8) return TNB200_ERR_UNSUPPORTED;
    }
    kind = THIN_MMA;
    return 0;
  }
  // ---- warp-MMA family, fp32 as TF32 (not under TNB200_MATH_STRICT: the planner routes strict fp32 elsewhere)
  if (dt == TNB200_F32 && allow_tf32 && (K == 16 || K == 32 || K == 64) && p.P > 8) {
    if (mode == 0) {
      if (p.L % 32) return TNB200_ERR_UNSUPPORTED;
    } else {
      if (!(p.P == 16 || p.P == 32 || p.P == 64)) return TNB200_ERR_UNSUPPORTED;
      if (p.sXl % 4 || p.sCl % 4 || p.L % 64) return TNB200_ERR_UNSUPPORTED;
    }
    kind = THIN_MMA_TF32;
    return 0;
  }
  return TNB200_ERR_UNSUPPORTED;
}

// Planner entry: launches the thin kernel for one contraction, or returns TNB200_ERR_UNSUPPORTED.
int tensordot_thin(int dt, const void* A, const void* B, void* C, const ModeList& mB, const ModeList& mM,
                   const ModeList& mN, const ModeList& mK, bool allow_tf32, cudaStream_t st) {
  ThinParams p;
  int mode, kind;
  const int rc = plan_thin(dt, A, B, C, mB, mM, mN, mK, allow_tf32, p, mode, kind);
  if (rc) return rc;
  if (kind == THIN_MMA_TF32) return launch_mma32(mode, p, st);
  if (kind == THIN_MMA) return dt == TNB200_F16 ? launch_mma<TNB200_F16>(mode, p, st) : launch_mma<TNB200_BF16>(mode, p, st);
  switch (dt) {
    case TNB200_F64: return launch_simt<TNB200_F64>(mode, p, st);
    case TNB200_F32: return launch_simt<TNB200_F32>(mode, p, st);
    case TNB200_F16: return launch_simt<TNB200_F16>(mode, p, st);
    default: return launch_simt<TNB200_BF16>(mode, p, st);
  }
}

// ------------------------------------------------------------------------------------------ fused thin run, host side
struct ThinRun {
  int dt, mode;
  ThinParams first, last;
  ThinRunParams rp;
  size_t smem;
  int grid;
};

static void host_mode_offsets(const DevModes& m, int64_t lin, int64_t& o0, int64_t& o1) {
  o0 = 0; o1 = 0;
  for (int i = m.n - 1; i > 0; --i) {
    const int64_t q = lin / m.ext[i], r = lin - q * m.ext[i];
    o0 += r * m.s0[i]; o1 += r * m.s1[i];
    lin = q;
  }
  if (m.n > 0) { o0 += lin * m.s0[0]; o1 += lin * m.s1[0]; }
}

template <typename T, int MODE> static void* thin_run_fn() { return (void*)thin_run_kernel<T, MODE>; }
static void* thin_run_kernel_ptr(int dt, int mode) {
  if (dt == TNB200_F16) return mode == 0 ? thin_run_fn<__half, 0>() : thin_run_fn<__half, 1>();
  return mode == 0 ? thin_run_fn<__nv_bfloat16, 0>() : thin_run_fn<__nv_bfloat16, 1>();
}

// Steps are given as in tnb200_tensordot (merged mode lists).  Step j + 1's X operand must be step j's C (dep_a / dep_b
// name the producing step, -1 for an operand that exists before the launch); the address of an intermediate C is not
// used, since the fused run keeps it on chip.  A step that cannot join the run: TNB200_ERR_UNSUPPORTED, *bad = its index
// (-1 when the run is declined as a whole).
int thin_run_create(int dt, int nsteps, const ModeList* mB, const ModeList* mM, const ModeList* mN, const ModeList* mK,
                    const void* const* A, const void* const* B, void* const* C, const int* dep_a, const int* dep_b,
                    int* bad, void** handle) {
  *bad = -1;
  if (nsteps < 2 || nsteps > kRunMaxSteps) return TNB200_ERR_UNSUPPORTED;
  if (dt != TNB200_F16 && dt != TNB200_BF16) { *bad = 0; return TNB200_ERR_UNSUPPORTED; }
  std::vector<ThinParams> ps((size_t)nsteps);
  std::vector<long long> tab((size_t)nsteps * 128, 0);
  ThinRun* r = new ThinRun();
  memset(&r->rp, 0, sizeof(r->rp));
  r->dt = dt;
  int W = 64, soff = 0;
  auto fail = [&](int j) { *bad = j; delete r; return TNB200_ERR_UNSUPPORTED; };
  for (int j = 0; j < nsteps; ++j) {
    ThinParams& p = ps[j];
    int mode, kind;
    if (plan_thin(dt, A[j], B[j], C[j], mB[j], mM[j], mN[j], mK[j], false, p, mode, kind)) return fail(j);
    if (j == 0) r->mode = mode;
    if (mode != r->mode || (kind != THIN_SIMT && kind != THIN_MMA)) return fail(j);
    const int dep_x = mode == 0 ? dep_b[j] : dep_a[j], dep_s = mode == 0 ? dep_a[j] : dep_b[j];
    if (dep_s >= 0 || dep_x != j - 1) return fail(j);       // X streams from the previous step, S exists beforehand
    if (kind == THIN_SIMT && !((p.K == 2 || p.K == 4 || p.K == 8) && (p.P == 2 || p.P == 4 || p.P == 8))) return fail(j);
    if (j == 0 && p.L % 64) return fail(0);
    if (j > 0) {
      // locality: step j's X is step j-1's C with the previous long axis innermost (mode A) / outermost (mode D)
      const ThinParams& pv = ps[j - 1];
      if (p.batch != pv.batch || p.L % pv.L) return fail(j);
      const int64_t R = p.L / pv.L;
      if ((int64_t)pv.P != p.K * R) return fail(j);
      if (r->mode == 0) {
        if (p.sXk < p.L) return fail(j);
        std::vector<char> seen((size_t)pv.P, 0);
        for (int pp = 0; pp < pv.P; ++pp) {
          int64_t os, oc;
          host_mode_offsets(pv.mP, pp, os, oc);
          const int64_t k = oc / p.sXk, rem = oc % p.sXk;
          if (rem % pv.L || rem / pv.L >= R || seen[k * R + rem / pv.L]) return fail(j);
          seen[k * R + rem / pv.L] = 1;
          tab[(size_t)(j - 1) * 128 + 64 + pp] = k * (W * R) + (rem / pv.L) * W;
        }
      } else if (p.sXl != p.K || pv.sCl != pv.P) {
        return fail(j);
      }
      W *= (int)R;
    }
    if ((int64_t)p.K * W > kRunSlab || (int64_t)p.P * W > kRunSlab) return fail(j);
    for (int pp = 0; pp < p.P; ++pp) {
      int64_t os, oc;
      host_mode_offsets(p.mP, pp, os, oc);
      tab[(size_t)j * 128 + pp] = os;
      if (j == nsteps - 1) tab[(size_t)j * 128 + 64 + pp] = oc;
    }
    ThinRunStep& st = r->rp.st[j];
    st.S = p.S; st.bS = p.bS; st.sSk = p.sSk; st.K = p.K; st.P = p.P; st.kind = kind; st.W = W; st.L = p.L;
    st.soff = soff;
    const int pt = (p.P + 15) / 16 <= 1 ? 1 : ((p.P + 15) / 16 <= 2 ? 2 : 4);
    soff += kind == THIN_MMA ? 16 * pt * (p.K + 8) * 2 : p.K * p.P * 4;
    soff = (soff + 15) / 16 * 16;
  }
  const ThinParams &p0 = ps[0], &pl = ps[nsteps - 1];
  ThinRunParams& rp = r->rp;
  rp.X = p0.X; rp.C = pl.C;
  rp.sX = r->mode == 0 ? p0.sXk : p0.sXl; rp.bX = p0.bX;
  rp.sC = pl.sCl; rp.bC = pl.bC;
  rp.batch = p0.batch; rp.nslab = p0.L / 64;
  rp.nsteps = nsteps; rp.smem_s = soff;
  r->smem = (size_t)soff + kRunMaxSteps * 64 * sizeof(long long) + (size_t)kRunWarps * 2 * kRunSlab * 2;
  void* fn = thin_run_kernel_ptr(dt, r->mode);
  int blocks = 0;
  // the attribute is per kernel, not per run: set the bound of any run, so that creating a smaller run of the same
  // kernel does not invalidate the launches of a larger one
  constexpr int kRunSmemMax = kRunMaxSteps * 64 * (64 + 8) * 2 + kRunMaxSteps * 64 * (int)sizeof(long long) +
                              kRunWarps * 2 * kRunSlab * 2;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kRunSmemMax) != cudaSuccess ||
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, fn, 256, r->smem) != cudaSuccess || blocks < 1) {
    cudaGetLastError();
    delete r;
    return TNB200_ERR_UNSUPPORTED;
  }
  const int64_t items = (rp.batch * rp.nslab + kRunWarps - 1) / kRunWarps;
  r->grid = (int)std::min<int64_t>((int64_t)blocks * num_sms(), items);
  long long* dtab = nullptr;
  if (cudaMalloc(&dtab, tab.size() * sizeof(long long)) != cudaSuccess ||
      cudaMemcpy(dtab, tab.data(), tab.size() * sizeof(long long), cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaGetLastError();
    if (dtab) cudaFree(dtab);
    delete r;
    return TNB200_ERR_CUDA;
  }
  rp.tab = dtab;
  *handle = r;
  return 0;
}

int thin_run_launch(void* handle, cudaStream_t st) {
  const ThinRun* r = (const ThinRun*)handle;
  if (r->dt == TNB200_F16) {
    if (r->mode == 0) thin_run_kernel<__half, 0><<<r->grid, 256, r->smem, st>>>(r->rp);
    else thin_run_kernel<__half, 1><<<r->grid, 256, r->smem, st>>>(r->rp);
  } else {
    if (r->mode == 0) thin_run_kernel<__nv_bfloat16, 0><<<r->grid, 256, r->smem, st>>>(r->rp);
    else thin_run_kernel<__nv_bfloat16, 1><<<r->grid, 256, r->smem, st>>>(r->rp);
  }
  TNB_LAUNCH_CHECK();
  count_launch();
  set_kernel_name("thin_run");
  return 0;
}

int thin_run_destroy(void* handle) {
  ThinRun* r = (ThinRun*)handle;
  if (!r) return 0;
  cudaFree((void*)r->rp.tab);
  delete r;
  return 0;
}

}  // namespace tnb
