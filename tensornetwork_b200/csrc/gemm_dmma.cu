// gemm_dmma.cu — the fp64 path of tnb200_tensordot.
//
// wgmma has no f64 kind, so double precision runs on the FP64 tensor pipe through
// mma.sync.aligned.m8n8k4.f64 (DMMA).  H100's FP64 tensor rate is 128 FMA/clk/SM, i.e.
// a 128 x BN x 16 k-block costs >= 1024 cycles of DMMA, which leaves ample room to stage the
// operands with plain 8-byte cp.async (LDGSTS): the kernel is FP64-pipe bound by construction.
// Both operands are arbitrary 2-stride matrices (the tensordot's transposes are folded into
// the cp.async address computation); shared-memory tiles use the majorness of the global
// operand with a +4-double row pad, which makes every DMMA fragment load conflict-free.
#include "gemm.cuh"

namespace tnb {

constexpr int DBM = 128, DBK = 16, DSTAGES = 3, DTHREADS = 256;

__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, bool valid) {
  int sz = valid ? 8 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

struct DmmaParams {
  const double* A; const double* B; double* C;
  int64_t M, N, K, batch;
  int64_t a_sm, a_sk, a_sb, b_sk, b_sn, b_sb, c_sm, c_sb;
  int64_t tiles_m, tiles_n;
  int vec_ok;
  int ksplit;                 // > 1: the K range is cut into ksplit slices, slice s of a tile writes its partial product to
  int64_t k_per;              //       ws[s][batch][M][N] (row-major); dmma_splitk_reduce_kernel sums them in slice order
  double* ws;
};

// A_K: A tile stored [m][k] (K-major global operand) else [k][m]; B_K likewise ([n][k] / [k][n]).
template <int BN, bool A_K, bool B_K>
__global__ void __launch_bounds__(DTHREADS, 1) gemm_dmma_kernel(const __grid_constant__ DmmaParams p) {
  constexpr int A_LD = A_K ? DBK + 4 : DBM + 4;
  constexpr int A_ELEMS = A_K ? DBM * A_LD : DBK * A_LD;
  constexpr int B_LD = B_K ? DBK + 4 : BN + 4;
  constexpr int B_ELEMS = B_K ? BN * B_LD : DBK * B_LD;
  constexpr int WN = BN / 4;          // warp tile: 64 x WN, warps arranged 2 (M) x 4 (N)
  constexpr int NT = WN / 8;          // n8 tiles per warp
  extern __shared__ __align__(16) double dsm[];
  double* As = dsm;
  double* Bs = dsm + DSTAGES * A_ELEMS;

  int64_t bid = blockIdx.x;
  const int ks = p.ksplit > 1 ? (int)(bid % p.ksplit) : 0;
  if (p.ksplit > 1) bid /= p.ksplit;
  const int64_t tn = bid % p.tiles_n; bid /= p.tiles_n;
  const int64_t tm = bid % p.tiles_m;
  const int64_t bb = bid / p.tiles_m;
  const int64_t m0 = tm * DBM, n0 = tn * BN;
  const double* Ag = p.A + bb * p.a_sb;
  const double* Bg = p.B + bb * p.b_sb;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = (warp >> 2) * 64, wn = (warp & 3) * WN;
  const int64_t kbeg = p.ksplit > 1 ? (int64_t)ks * p.k_per : 0;
  const int64_t kend = p.ksplit > 1 ? (kbeg + p.k_per < p.K ? kbeg + p.k_per : p.K) : p.K;
  const int num_kb = kend > kbeg ? (int)((kend - kbeg + DBK - 1) / DBK) : 0;

  // Per-thread copy pattern, hoisted out of the k loop: element i of a stage differs from element 0 by a constant stride
  // (rows 16 apart for a K-major tile, k-rows 2 apart for an MN-major one), so a stage costs one 64-bit add per cp.async
  // instead of a multiply-add pair per element.
  const int a_k = A_K ? tid % DBK : tid / DBM, a_m = A_K ? tid / DBK : tid % DBM;
  const int b_k = B_K ? tid % DBK : tid / BN, b_n = B_K ? tid / DBK : tid % BN;
  constexpr int A_IT = DBM * DBK / DTHREADS, B_IT = BN * DBK / DTHREADS;
  constexpr int A_STEP = A_K ? DTHREADS / DBK : DTHREADS / DBM;     // rows (A_K) or k-rows (else) between consecutive elements
  constexpr int B_STEP = B_K ? DTHREADS / DBK : DTHREADS / BN;
  const double* pA0 = Ag + (m0 + a_m) * p.a_sm + (kbeg + a_k) * p.a_sk;
  const double* pB0 = Bg + (n0 + b_n) * p.b_sn + (kbeg + b_k) * p.b_sk;
  const int64_t a_inc = A_K ? (int64_t)A_STEP * p.a_sm : (int64_t)A_STEP * p.a_sk;
  const int64_t b_inc = B_K ? (int64_t)B_STEP * p.b_sn : (int64_t)B_STEP * p.b_sk;
  const int64_t a_mrem = p.M - m0 - a_m, b_nrem = p.N - n0 - b_n;    // > 0 iff this thread's (first) row / column exists
  const uint32_t a_dst0 = (uint32_t)__cvta_generic_to_shared(A_K ? As + a_m * A_LD + a_k : As + a_k * A_LD + a_m);
  const uint32_t b_dst0 = (uint32_t)__cvta_generic_to_shared(B_K ? Bs + b_n * B_LD + b_k : Bs + b_k * B_LD + b_n);
  constexpr uint32_t A_DSTEP = (A_K ? A_STEP * A_LD : A_STEP * A_LD) * 8, B_DSTEP = (B_K ? B_STEP * B_LD : B_STEP * B_LD) * 8;

  auto load_stage = [&](int stage, int kb) {
    const int64_t k0 = kbeg + (int64_t)kb * DBK;
    const int64_t krem_a = kend - k0 - a_k, krem_b = kend - k0 - b_k;
    const double* pa = pA0 + (int64_t)kb * DBK * p.a_sk;
    const double* pb = pB0 + (int64_t)kb * DBK * p.b_sk;
    uint32_t da = a_dst0 + (uint32_t)(stage * A_ELEMS * 8), db = b_dst0 + (uint32_t)(stage * B_ELEMS * 8);
#pragma unroll
    for (int i = 0; i < A_IT; ++i) {
      const bool ok = A_K ? (a_mrem > (int64_t)i * A_STEP && krem_a > 0) : (a_mrem > 0 && krem_a > (int64_t)i * A_STEP);
      cp_async8(da, ok ? pa : Ag, ok);
      pa += a_inc; da += A_DSTEP;
    }
#pragma unroll
    for (int i = 0; i < B_IT; ++i) {
      const bool ok = B_K ? (b_nrem > (int64_t)i * B_STEP && krem_b > 0) : (b_nrem > 0 && krem_b > (int64_t)i * B_STEP);
      cp_async8(db, ok ? pb : Bg, ok);
      pb += b_inc; db += B_DSTEP;
    }
  };

  double acc[8][NT][2];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }

#pragma unroll
  for (int s = 0; s < DSTAGES - 1; ++s) {
    if (s < num_kb) load_stage(s, s);
    cp_async_commit();
  }
  const int fr = lane >> 2, fk = lane & 3;   // fragment row / k index of this lane
  for (int kb = 0; kb < num_kb; ++kb) {
    cp_async_wait<DSTAGES - 2>();
    __syncthreads();
    {
      int nk = kb + DSTAGES - 1;
      if (nk < num_kb) load_stage(nk % DSTAGES, nk);
      cp_async_commit();
    }
    const double* as = As + (kb % DSTAGES) * A_ELEMS;
    const double* bs = Bs + (kb % DSTAGES) * B_ELEMS;
#pragma unroll
    for (int k4 = 0; k4 < DBK; k4 += 4) {
      double af[8], bf[NT];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        int m = wm + i * 8 + fr, k = k4 + fk;
        af[i] = A_K ? as[m * A_LD + k] : as[k * A_LD + m];
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        int n = wn + j * 8 + fr, k = k4 + fk;
        bf[j] = B_K ? bs[n * B_LD + k] : bs[k * B_LD + n];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j) dmma(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
    }
  }
  cp_async_wait<0>();

  if (p.ksplit > 1) {                      // partial product of this K slice: plain row-major [M][N] in the workspace
    double* Wg = p.ws + (((int64_t)ks * p.batch + bb) * p.M) * p.N;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int64_t m = m0 + wm + i * 8 + fr;
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        int64_t n = n0 + wn + j * 8 + 2 * fk;
        if (n < p.N) Wg[m * p.N + n] = acc[i][j][0];
        if (n + 1 < p.N) Wg[m * p.N + n + 1] = acc[i][j][1];
      }
    }
    return;
  }
  double* Cg = p.C + bb * p.c_sb;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int64_t m = m0 + wm + i * 8 + fr;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      int64_t n = n0 + wn + j * 8 + 2 * fk;
      if (n >= p.N) continue;
      double* dst = Cg + m * p.c_sm + n;
      if (p.vec_ok && n + 1 < p.N) *(double2*)dst = make_double2(acc[i][j][0], acc[i][j][1]);
      else { dst[0] = acc[i][j][0]; if (n + 1 < p.N) dst[1] = acc[i][j][1]; }
    }
  }
}

// C[b][m][n] = sum over slices (in slice order: deterministic) of ws[s][b][m][n]
__global__ void dmma_splitk_reduce_kernel(const double* __restrict__ ws, int ksplit, int64_t batch, int64_t M, int64_t N,
                                          double* __restrict__ C, int64_t c_sm, int64_t c_sb) {
  const int64_t total = batch * M * N;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (int s = 0; s < ksplit; ++s) acc += ws[(int64_t)s * total + idx];
    const int64_t n = idx % N, m = (idx / N) % M, b = idx / (N * M);
    C[b * c_sb + m * c_sm + n] = acc;
  }
}

template <int BN, bool A_K, bool B_K>
static int launch_dmma(const DmmaParams& p, int64_t tiles, cudaStream_t st) {
  constexpr int A_LD = A_K ? DBK + 4 : DBM + 4;
  constexpr int A_ELEMS = A_K ? DBM * A_LD : DBK * A_LD;
  constexpr int B_LD = B_K ? DBK + 4 : BN + 4;
  constexpr int B_ELEMS = B_K ? BN * B_LD : DBK * B_LD;
  const size_t smem = (size_t)DSTAGES * (A_ELEMS + B_ELEMS) * sizeof(double);
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(gemm_dmma_kernel<BN, A_K, B_K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) { set_error("dmma: cannot raise dynamic smem: %s", cudaGetErrorString(e)); return TNB200_ERR_CUDA; }
    attr = true;
  }
  gemm_dmma_kernel<BN, A_K, B_K><<<(unsigned)(tiles * (p.ksplit > 1 ? p.ksplit : 1)), DTHREADS, smem, st>>>(p);
  TNB_LAUNCH_CHECK();
  count_launch();
  return 0;
}

int gemm_dmma_f64(const GemmProblem& g, cudaStream_t st) {
  if (g.dtype != TNB200_F64 || g.conjA || g.conjB) return TNB200_ERR_UNSUPPORTED;
  if (g.c_sn != 1 && g.N > 1) return TNB200_ERR_UNSUPPORTED;
  if (!g.A.simple() || !g.B.simple()) return TNB200_ERR_UNSUPPORTED;
  DmmaParams p;
  p.A = (const double*)g.A.ptr; p.B = (const double*)g.B.ptr; p.C = (double*)g.C;
  p.M = g.M; p.N = g.N; p.K = g.K; p.batch = g.batch;
  p.a_sm = g.A.f_stride(); p.a_sk = g.A.k_stride(); p.a_sb = g.A.sb;
  p.b_sk = g.B.k_stride(); p.b_sn = g.B.f_stride(); p.b_sb = g.B.sb;
  p.c_sm = g.c_sm; p.c_sb = g.c_sb;
  p.vec_ok = (((uintptr_t)g.C) % 16 == 0) && (g.c_sm % 2 == 0) && (g.c_sb % 2 == 0);
  p.tiles_m = (g.M + DBM - 1) / DBM;
  const int sms = num_sms();
  int BN = 128;
  if (p.tiles_m * ((g.N + 127) / 128) * g.batch < sms || g.N <= 64) BN = 64;
  p.tiles_n = (g.N + BN - 1) / BN;
  const int64_t tiles = p.tiles_m * p.tiles_n * g.batch;
  if (tiles >= (1LL << 31)) return TNB200_ERR_UNSUPPORTED;
  // split-K: a small output under a long contraction (e.g. 64 x 64 over K = 65536, the closing step of a tree-network
  // branch) would otherwise run on one SM.  Slices write partial products to a workspace, a second kernel sums them in
  // slice order (deterministic, unlike atomics).
  p.ksplit = 1; p.k_per = g.K; p.ws = nullptr;
  if (tiles * 2 <= sms && g.K >= 2048) {
    int64_t want = sms / tiles;
    int64_t maxs = g.K / 512;                         // at least 512 of K per slice
    if (want > maxs) want = maxs;
    if (want > 1) {
      p.k_per = ((g.K + want - 1) / want + DBK - 1) / DBK * DBK;
      p.ksplit = (int)((g.K + p.k_per - 1) / p.k_per);
      if (p.ksplit > 1) {
        int rc = ws_alloc((void**)&p.ws, sizeof(double) * (size_t)p.ksplit * (size_t)g.batch * (size_t)g.M * (size_t)g.N, st);
        if (rc) return rc;
      } else { p.ksplit = 1; p.k_per = g.K; }
    }
  }
  // an operand is loaded "K-major" when its contracted stride is the smaller one
  const bool a_k = llabs(p.a_sk) <= llabs(p.a_sm) || g.M == 1;
  const bool b_k = llabs(p.b_sk) <= llabs(p.b_sn) || g.N == 1;
  set_kernel_name(p.ksplit > 1 ? "dmma_f64_splitk" : "dmma_f64");
  int rc;
#define TNB_DMMA(BNV)                                                           \
  if (a_k && b_k) rc = launch_dmma<BNV, true, true>(p, tiles, st);              \
  else if (a_k && !b_k) rc = launch_dmma<BNV, true, false>(p, tiles, st);       \
  else if (!a_k && b_k) rc = launch_dmma<BNV, false, true>(p, tiles, st);       \
  else rc = launch_dmma<BNV, false, false>(p, tiles, st);
  if (BN == 128) { TNB_DMMA(128) } else { TNB_DMMA(64) }
#undef TNB_DMMA
  if (rc == 0 && p.ksplit > 1) {
    const int64_t total = g.batch * g.M * g.N;
    int64_t blocks = (total + 255) / 256;
    if (blocks > (int64_t)sms * 8) blocks = (int64_t)sms * 8;
    dmma_splitk_reduce_kernel<<<(unsigned)blocks, 256, 0, st>>>(p.ws, p.ksplit, g.batch, g.M, g.N, p.C, p.c_sm, p.c_sb);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("dmma split-K reduce launch failed: %s", cudaGetErrorString(e)); rc = TNB200_ERR_CUDA; }
    count_launch();
  }
  if (p.ws) ws_free(p.ws, st);
  return rc;
}

}  // namespace tnb
