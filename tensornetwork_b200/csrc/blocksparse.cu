// blocksparse.cu — tnb200_blocksparse_tensordot: every charge sector of a block-sparse
// tensordot in ONE launch (block_sparse/blocksparsetensor.py:1094-1101 runs a Python loop of
// fancy-index gather -> np.matmul -> scatter per sector).
//
// grid = (tiles over the largest sector, sector).  A CTA gathers its A/B tile through the int64
// element maps straight into shared memory (map reads are coalesced, data reads are the
// unavoidable gather), multiplies, and scatters C through its map.  Sectors at the BASELINE
// sizes are tiny (2..66 rows), so this is latency/HBM-bound: no tensor cores, 32x32 tiles.
#include "common.cuh"

namespace tnb {

constexpr int GT = 32, GK = 16;

template <typename T, typename Acc>
__global__ void __launch_bounds__(256) blocksparse_kernel(const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C,
                                                          const long long* __restrict__ dims,
                                                          const long long* __restrict__ amap, const long long* __restrict__ aoff,
                                                          const long long* __restrict__ bmap, const long long* __restrict__ boff,
                                                          const long long* __restrict__ cmap, const long long* __restrict__ coff,
                                                          int tiles_n, int conj_b) {
  __shared__ Acc As[GK][GT + 1];
  __shared__ Acc Bs[GK][GT + 1];
  const int q = blockIdx.y;
  const long long m = dims[3 * q], k = dims[3 * q + 1], n = dims[3 * q + 2];
  const int tm = blockIdx.x / tiles_n, tn = blockIdx.x % tiles_n;
  const long long m0 = (long long)tm * GT, n0 = (long long)tn * GT;
  if (m0 >= m || n0 >= n) return;
  const long long* am = amap + aoff[q];
  const long long* bm = bmap + boff[q];
  const long long* cm = cmap + coff[q];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;   // 16 x 16 threads, 2 x 2 outputs each
  Acc acc[2][2];
  acc[0][0] = acc[0][1] = acc[1][0] = acc[1][1] = acc_zero((Acc*)nullptr);
  for (long long k0 = 0; k0 < k; k0 += GK) {
    // A tile: GT rows x GK k (k contiguous in the map)
    for (int idx = t; idx < GT * GK; idx += 256) {
      int r = idx / GK, kk = idx % GK;
      Acc v = acc_zero((Acc*)nullptr);
      if (m0 + r < m && k0 + kk < k) v = to_acc(A[am[(m0 + r) * k + k0 + kk]]);
      As[kk][r] = v;
    }
    // B tile: GK k x GT cols (cols contiguous in the map)
    for (int idx = t; idx < GT * GK; idx += 256) {
      int kk = idx / GT, c = idx % GT;
      Acc v = acc_zero((Acc*)nullptr);
      if (n0 + c < n && k0 + kk < k) { v = to_acc(B[bm[(k0 + kk) * n + n0 + c]]); if (conj_b) v = conj_acc(v); }
      Bs[kk][c] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GK; ++kk) {
      Acc a0 = As[kk][ty], a1 = As[kk][ty + 16], b0 = Bs[kk][tx], b1 = Bs[kk][tx + 16];
      fma_acc(acc[0][0], a0, b0); fma_acc(acc[0][1], a0, b1);
      fma_acc(acc[1][0], a1, b0); fma_acc(acc[1][1], a1, b1);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      long long r = m0 + ty + 16 * i, c = n0 + tx + 16 * j;
      if (r < m && c < n) C[cm[r * n + c]] = FromAcc<T, Acc>::f(acc[i][j]);
    }
}

// ---- fp64 sectors large enough for the tensor pipe: 64 x 64 output tiles, DMMA (mma.sync.m8n8k4.f64), operands gathered
// through the element maps into K-major shared-memory tiles (register-prefetched: the next chunk's map entries and data are
// in flight while the current chunk multiplies).  Same grouped launch shape: grid = (tiles of the largest sector, sector).
constexpr int DT_ = 64, DK_ = 16, DLD_ = DK_ + 4;

__device__ __forceinline__ void bs_dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__global__ void __launch_bounds__(256) blocksparse_dmma_kernel(const double* __restrict__ A, const double* __restrict__ B, double* __restrict__ C,
                                                               const long long* __restrict__ dims,
                                                               const long long* __restrict__ amap, const long long* __restrict__ aoff,
                                                               const long long* __restrict__ bmap, const long long* __restrict__ boff,
                                                               const long long* __restrict__ cmap, const long long* __restrict__ coff,
                                                               int tiles_n) {
  __shared__ double As[2][DT_ * DLD_];
  __shared__ double Bs[2][DT_ * DLD_];
  const int q = blockIdx.y;
  const long long m = dims[3 * q], k = dims[3 * q + 1], n = dims[3 * q + 2];
  const int tm = blockIdx.x / tiles_n, tn = blockIdx.x % tiles_n;
  const long long m0 = (long long)tm * DT_, n0 = (long long)tn * DT_;
  if (m0 >= m || n0 >= n) return;
  const long long* am = amap + aoff[q];
  const long long* bm = bmap + boff[q];
  const long long* cm = cmap + coff[q];
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31, fr = lane >> 2, fk = lane & 3;
  const int wm = (warp >> 1) * 16, wn = (warp & 1) * 32;
  // this thread's 4 A elements (row ar[i], k-offset ak) and 4 B elements (k-offset bk[i], column bc) of every chunk
  const int ak = t & 15, ar0 = t >> 4;               // rows ar0 + 16 i
  const int bc = t & 63, bk0 = t >> 6;               // k-offsets bk0 + 4 i
  // the gather is a double indirection (map entry -> data): map entries are fetched TWO chunks ahead, data ONE chunk ahead,
  // so each iteration exposes one memory round trip instead of two
  double pa[4], pb[4];
  long long ia[4], ib[4];
  auto fetch_idx = [&](long long k0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const long long r = m0 + ar0 + 16 * i, kk = k0 + ak;
      ia[i] = (r < m && kk < k) ? am[r * k + kk] : -1;
      const long long kb = k0 + bk0 + 4 * i, c = n0 + bc;
      ib[i] = (kb < k && c < n) ? bm[kb * n + c] : -1;
    }
  };
  auto fetch_data = [&]() {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      pa[i] = ia[i] >= 0 ? A[ia[i]] : 0.0;
      pb[i] = ib[i] >= 0 ? B[ib[i]] : 0.0;
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      As[buf][(ar0 + 16 * i) * DLD_ + ak] = pa[i];
      Bs[buf][bc * DLD_ + bk0 + 4 * i] = pb[i];
    }
  };
  double acc[2][4][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[i][j][0] = 0.0; acc[i][j][1] = 0.0; }
  fetch_idx(0);
  fetch_data();
  stash(0);
  fetch_idx(DK_);                       // (out of range -> -1: harmless)
  __syncthreads();
  int buf = 0;
  for (long long k0 = 0; k0 < k; k0 += DK_) {
    const bool more = k0 + DK_ < k;
    if (more) { fetch_data(); fetch_idx(k0 + 2 * DK_); }
    const double* as = As[buf];
    const double* bs = Bs[buf];
#pragma unroll
    for (int k4 = 0; k4 < DK_; k4 += 4) {
      double af[2], bf[4];
#pragma unroll
      for (int i = 0; i < 2; ++i) af[i] = as[(wm + i * 8 + fr) * DLD_ + k4 + fk];
#pragma unroll
      for (int j = 0; j < 4; ++j) bf[j] = bs[(wn + j * 8 + fr) * DLD_ + k4 + fk];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) bs_dmma(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
    }
    if (more) stash(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long r = m0 + wm + i * 8 + fr, c = n0 + wn + j * 8 + 2 * fk;
      if (r < m) {
        if (c < n) C[cm[r * n + c]] = acc[i][j][0];
        if (c + 1 < n) C[cm[r * n + c + 1]] = acc[i][j][1];
      }
    }
}

template <int DT>
static int launch_bs(const void* a, const void* b, void* c, int nsect, const int64_t* dims, const int64_t* am, const int64_t* ao,
                     const int64_t* bm, const int64_t* bo, const int64_t* cm, const int64_t* co, int64_t max_m, int64_t max_n,
                     int conj_b, cudaStream_t st) {
  using T = typename DType<DT>::T;
  using Acc = typename DType<DT>::Acc;
  const int tiles_m = (int)((max_m + GT - 1) / GT), tiles_n = (int)((max_n + GT - 1) / GT);
  dim3 grid((unsigned)(tiles_m * tiles_n), (unsigned)nsect);
  blocksparse_kernel<T, Acc><<<grid, 256, 0, st>>>((const T*)a, (const T*)b, (T*)c, (const long long*)dims, (const long long*)am,
                                                   (const long long*)ao, (const long long*)bm, (const long long*)bo,
                                                   (const long long*)cm, (const long long*)co, tiles_n, conj_b);
  TNB_LAUNCH_CHECK();
  count_launch();
  return 0;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_blocksparse_tensordot(const void* a_data, const void* b_data, void* c_data, int32_t dtype, int32_t nsect,
                                                const int64_t* dims_dev, const int64_t* a_map_dev, const int64_t* a_off_dev,
                                                const int64_t* b_map_dev, const int64_t* b_off_dev, const int64_t* c_map_dev,
                                                const int64_t* c_off_dev, int64_t max_m, int64_t max_n, int32_t conj_b, void* stream) {
  TNB_REQUIRE(nsect >= 0 && max_m >= 0 && max_n >= 0, TNB200_ERR_INVALID, "blocksparse: bad sizes");
  if (nsect == 0 || max_m == 0 || max_n == 0) return 0;
  TNB_REQUIRE(nsect <= 65535, TNB200_ERR_UNSUPPORTED, "blocksparse: more than 65535 sectors");
  TNB_REQUIRE(a_data && b_data && c_data && dims_dev && a_map_dev && b_map_dev && c_map_dev, TNB200_ERR_INVALID, "blocksparse: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  set_kernel_name("blocksparse_grouped");
  const bool cj = conj_b && dtype_is_complex(dtype);
  if (dtype == TNB200_F64 && max_m >= 48 && max_n >= 48) {
    const int tiles_m = (int)((max_m + DT_ - 1) / DT_), tiles_n = (int)((max_n + DT_ - 1) / DT_);
    blocksparse_dmma_kernel<<<dim3((unsigned)(tiles_m * tiles_n), (unsigned)nsect), 256, 0, st>>>(
        (const double*)a_data, (const double*)b_data, (double*)c_data, (const long long*)dims_dev, (const long long*)a_map_dev,
        (const long long*)a_off_dev, (const long long*)b_map_dev, (const long long*)b_off_dev, (const long long*)c_map_dev,
        (const long long*)c_off_dev, tiles_n);
    TNB_LAUNCH_CHECK();
    count_launch();
    set_kernel_name("blocksparse_grouped_dmma");
    return 0;
  }
  switch (dtype) {
    case TNB200_F64: return launch_bs<TNB200_F64>(a_data, b_data, c_data, nsect, dims_dev, a_map_dev, a_off_dev, b_map_dev, b_off_dev, c_map_dev, c_off_dev, max_m, max_n, 0, st);
    case TNB200_F32: return launch_bs<TNB200_F32>(a_data, b_data, c_data, nsect, dims_dev, a_map_dev, a_off_dev, b_map_dev, b_off_dev, c_map_dev, c_off_dev, max_m, max_n, 0, st);
    case TNB200_C64: return launch_bs<TNB200_C64>(a_data, b_data, c_data, nsect, dims_dev, a_map_dev, a_off_dev, b_map_dev, b_off_dev, c_map_dev, c_off_dev, max_m, max_n, cj, st);
    case TNB200_C128: return launch_bs<TNB200_C128>(a_data, b_data, c_data, nsect, dims_dev, a_map_dev, a_off_dev, b_map_dev, b_off_dev, c_map_dev, c_off_dev, max_m, max_n, cj, st);
  }
  set_error("blocksparse: dtype %s is not supported (f32/f64/c64/c128)", dtype_name(dtype));
  return TNB200_ERR_DTYPE;
}
