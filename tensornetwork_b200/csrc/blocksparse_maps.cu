// blocksparse_maps.cu — tnb200_blocksparse_maps(_nsym): the int64 element maps of a block-sparse matrix view, built ON THE
// DEVICE, for legs carrying one charge or a product of nsym U(1) / Z_N charges.
//
// Reference: block_sparse/blocksparse_utils.py:330-634 (`_find_diagonal_sparse_blocks`, `_find_transposed_diagonal_sparse_
// blocks`, `reduce_charges`) — numpy unique / intersect / fancy indexing on the host, recomputed per call unless the opt-in
// cache (caching.py:22-88) is on.  Here it is pure integer work on the GPU, bit-identical to the host construction
// (tests/test_gpu_blocksparse.py compares with the golden maps of the real reference):
//
//   data vector   = the elements of the dense tensor (stored leg order, row-major) whose total signed charge is zero,
//                   in ascending flat position.  The stored legs are cut into a LEFT and a RIGHT group; element e is
//                   the j-th partner of left state l: r = bucket[ -q_l ][ j ]   (right states bucketed by charge, ascending)
//   matrix view   = rows: legs order[0..partition), columns: the rest.  Sector of charge q holds the rows with fused
//                   charge q (ascending row index) x the columns with charge -q (ascending column index), row-major.
//   map[ sect_off[q] + rowrank(R) * ncols[q] + colrank(C) ] = e
//
// A charge is a vector of nsym components; its BIN is a mixed-radix number over the per-component bins (component 0 most
// significant): U(1) component k: q_k + shift_k in radix 2 shift_k + 1, Z_N component k: q_k mod N_k in radix N_k.
//
// Kernels: fuse (mixed-radix decode -> charge bin of every state of a leg group), rank (position of a state among the
// states of equal bin), scan (first element of every left state), bucket, element (binary search e -> (l, j), decode,
// scatter).  Rank has two forms, chosen by the bin count: up to BM_PERBIN_MAX_BINS bins one CTA per bin scans all states
// (ballot prefix sums; the fewest launches), above it a stable counting sort whose work is O(states + bins): per-tile
// ranks and (bin, tile) counts, one exclusive scan over (bin, tile), then rank = scanned offset + rank in the tile.  The
// small per-charge tables (counts, offsets) are charge-degeneracy arithmetic done by the caller on the host (histogram
// convolutions of the legs).
#include "common.cuh"
#include "../../include/tnb200_symmetry.h"

namespace tnb {

constexpr int BM_MAXLEGS = TNB200_MAX_NDIM;
constexpr int BM_MAXSYM = TNB200_BLOCKSPARSE_MAX_NSYM;
constexpr int BM_PERBIN_MAX_BINS = 256;        // one CTA per bin at or below, counting sort above
constexpr long long BM_TILE_BUDGET = 1 << 22;  // (bin, tile) counters of the counting sort: ntiles = budget / nbins
constexpr int BM_TILE_THREADS = 256;
constexpr int BM_SCAN_THREADS = 1024, BM_SCAN_PER_THREAD = 4, BM_SCAN_CHUNK = BM_SCAN_THREADS * BM_SCAN_PER_THREAD;

struct LegGroup {                      // an ordered group of stored legs forming one product space
  int n;
  int leg[BM_MAXLEGS];                 // stored leg ids, most significant first
  long long dim[BM_MAXLEGS];
  long long coff[BM_MAXLEGS];          // state offset of the leg's signed charges in the charge table
};

struct Sym {                           // the charge components and their bins
  int n;
  long long mod[BM_MAXSYM];            // N for Z_N, 0 for U(1)
  long long shift[BM_MAXSYM];          // U(1): sum over the legs of max |charge|
  long long radix[BM_MAXSYM];          // 2 shift + 1 or N
};

// bin of the charge q[0..n): the mixed-radix number of the per-component bins
__device__ __forceinline__ int bm_bin(const long long (&q)[BM_MAXSYM], const Sym& s) {
  long long b = 0;
#pragma unroll
  for (int k = 0; k < BM_MAXSYM; ++k) {
    if (k < s.n) {
      long long c;
      if (s.mod[k] > 0) { c = q[k] % s.mod[k]; if (c < 0) c += s.mod[k]; } else { c = q[k] + s.shift[k]; }
      b = b * s.radix[k] + c;
    }
  }
  return (int)b;
}

// bin of the charge -q, q the charge of bin b: per component 2 shift - c (U(1)) or (N - c) mod N (Z_N)
__device__ __forceinline__ long long bm_partner(int b, const Sym& s) {
  long long rem = b, p = 0, mul = 1;
#pragma unroll
  for (int kk = 0; kk < BM_MAXSYM; ++kk) {
    const int k = BM_MAXSYM - 1 - kk;
    if (k < s.n) {
      const long long c = rem % s.radix[k];
      rem /= s.radix[k];
      p += (s.mod[k] > 0 ? (s.mod[k] - c) % s.mod[k] : 2 * s.shift[k] - c) * mul;
      mul *= s.radix[k];
    }
  }
  return p;
}

// adds the nsym components of the charge table row of state `row` to q
__device__ __forceinline__ void bm_add(long long (&q)[BM_MAXSYM], const long long* __restrict__ charges, long long row, const Sym& s) {
  const long long* c = charges + row * s.n;
#pragma unroll
  for (int k = 0; k < BM_MAXSYM; ++k)
    if (k < s.n) q[k] += c[k];
}

__global__ void bm_fuse_kernel(LegGroup g, Sym sy, const long long* __restrict__ charges, long long N, int* __restrict__ bin) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= N) return;
  long long rem = s, q[BM_MAXSYM];
#pragma unroll
  for (int k = 0; k < BM_MAXSYM; ++k) q[k] = 0;
#pragma unroll 1
  for (int i = g.n - 1; i >= 0; --i) {
    const long long d = rem % g.dim[i];
    rem /= g.dim[i];
    bm_add(q, charges, g.coff[i] + d, sy);
  }
  bin[s] = bm_bin(q, sy);
}

// rank[s] = number of states s' < s with bin[s'] == bin[s]; cnt[b] = number of states in bin b.  One CTA per bin.
__global__ void __launch_bounds__(1024) bm_rank_kernel(const int* __restrict__ bin, long long N, int* __restrict__ rank,
                                                       long long* __restrict__ cnt) {
  __shared__ int wsum[32];
  __shared__ int running_s;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) running_s = 0;
  __syncthreads();
  for (long long base = 0; base < N; base += 1024) {
    const long long i = base + tid;
    const bool f = i < N && bin[i] == b;
    const unsigned m = __ballot_sync(0xffffffffu, f);
    const int pre = __popc(m & ((1u << lane) - 1u));
    if (lane == 0) wsum[warp] = __popc(m);
    __syncthreads();
    int off = 0, tot = 0;
    for (int w = 0; w < 32; ++w) { const int v = wsum[w]; if (w < warp) off += v; tot += v; }
    const int run = running_s;
    if (f) rank[i] = run + off + pre;
    __syncthreads();
    if (tid == 0) running_s = run + tot;
    __syncthreads();
  }
  if (tid == 0) cnt[b] = running_s;
}

// Counting sort, step 1.  CTA t owns the states [t T, min(N, (t + 1) T)) and the counters tcnt[b * ntiles + t] (zeroed by
// the caller).  It walks its tile in chunks of BM_TILE_THREADS states; a state's rank in the tile = the counter of its bin
// before the chunk + the states of the same bin earlier in the chunk; the last state of a bin in the chunk advances the
// counter.  trank[s] = rank of s among the states of its bin in its tile.
__global__ void __launch_bounds__(BM_TILE_THREADS) bm_tile_rank_kernel(const int* __restrict__ bin, long long N, long long T, int ntiles,
                                                                       int* __restrict__ trank, int* __restrict__ tcnt) {
  __shared__ int sb[BM_TILE_THREADS];
  const int t = blockIdx.x, tid = threadIdx.x;
  const long long lo = t * T, hi = min(N, lo + T);
  for (long long base = lo; base < hi; base += BM_TILE_THREADS) {
    const long long i = base + tid;
    const int b = i < hi ? bin[i] : -1;
    sb[tid] = b;
    __syncthreads();
    int before = 0;
    bool last = true;
    if (b >= 0) {
#pragma unroll 8
      for (int j = 0; j < BM_TILE_THREADS; ++j) {
        const int o = sb[j];
        before += (o == b) & (j < tid);
        last &= !((o == b) & (j > tid));
      }
    }
    int* c = tcnt + (long long)(b < 0 ? 0 : b) * ntiles + t;
    const int run = b >= 0 ? *c : 0;
    __syncthreads();                           // every read of this chunk's counters precedes the first write
    if (b >= 0) {
      trank[i] = run + before;
      if (last) *c = run + before + 1;
    }
    __syncthreads();
  }
}

// Exclusive scan of x[0..M) in place, per chunk of BM_SCAN_CHUNK elements (one CTA each); the chunk's total goes to
// totals[blockIdx.x].  Run once over the data and once, as a single CTA, over the chunk totals; bm_scan_add_kernel then
// adds the scanned totals.
__global__ void __launch_bounds__(BM_SCAN_THREADS) bm_scan_chunk_kernel(int* __restrict__ x, long long M, int* __restrict__ totals) {
  __shared__ int wsum[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long base = blockIdx.x * (long long)BM_SCAN_CHUNK + (long long)tid * BM_SCAN_PER_THREAD;
  int v[BM_SCAN_PER_THREAD], sum = 0;
#pragma unroll
  for (int j = 0; j < BM_SCAN_PER_THREAD; ++j) { v[j] = base + j < M ? x[base + j] : 0; sum += v[j]; }
  int incl = sum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += y; }
  if (lane == 31) wsum[warp] = incl;
  __syncthreads();
  int off = 0, tot = 0;
  for (int w = 0; w < 32; ++w) { const int t = wsum[w]; if (w < warp) off += t; tot += t; }
  int run = off + incl - sum;
#pragma unroll
  for (int j = 0; j < BM_SCAN_PER_THREAD; ++j) { if (base + j < M) x[base + j] = run; run += v[j]; }
  if (tid == 0) totals[blockIdx.x] = tot;
}

__global__ void bm_scan_add_kernel(int* __restrict__ x, long long M, const int* __restrict__ chunk_off) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < M) x[i] += chunk_off[i / BM_SCAN_CHUNK];
}

// Counting sort, step 3: off = the exclusive scan of tcnt (bin-major, so off[b * ntiles] is the first sorted position of
// bin b and off[nbins * ntiles] = N).  rank[s] = off[b * ntiles + tile] - off[b * ntiles] + trank[s] (in place over trank);
// cnt[b] = off[(b + 1) * ntiles] - off[b * ntiles].
__global__ void bm_rank_finish_kernel(const int* __restrict__ bin, long long N, long long T, int ntiles, const int* __restrict__ off,
                                      int* __restrict__ rank, int nbins, long long* __restrict__ cnt) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < N) {
    const long long b0 = (long long)bin[i] * ntiles;
    rank[i] += off[b0 + i / T] - off[b0];
  }
  if (i < nbins) cnt[i] = off[(i + 1) * ntiles] - off[i * ntiles];
}

// first[l] = sum over l' < l of cnt_right[ partner bin of l' ]   (exclusive scan, one CTA; first[NL] = nnz)
__global__ void __launch_bounds__(1024) bm_first_kernel(const int* __restrict__ bin_left, long long NL, const long long* __restrict__ cnt_right,
                                                        Sym sy, long long* __restrict__ first) {
  __shared__ long long wsum[32];
  __shared__ long long running_s;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) running_s = 0;
  __syncthreads();
  for (long long base = 0; base < NL; base += 1024) {
    const long long i = base + tid;
    long long v = 0;
    if (i < NL) v = cnt_right[bm_partner(bin_left[i], sy)];               // states of the charge -q
    long long x = v;                                                       // inclusive warp scan
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    long long off = 0, tot = 0;
    for (int w = 0; w < 32; ++w) { const long long t = wsum[w]; if (w < warp) off += t; tot += t; }
    const long long run = running_s;
    if (i < NL) first[i] = run + off + x - v;
    __syncthreads();
    if (tid == 0) running_s = run + tot;
    __syncthreads();
  }
  if (tid == 0) first[NL] = running_s;
}

// bucket[start[bin[r]] + rank[r]] = r
__global__ void bm_bucket_kernel(const int* __restrict__ bin, const int* __restrict__ rank, long long N,
                                 const long long* __restrict__ start, long long* __restrict__ bucket) {
  const long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (r < N) bucket[start[bin[r]] + rank[r]] = r;
}

struct ElemParams {
  LegGroup left, right;                       // the two stored halves
  long long row_mul[BM_MAXLEGS], col_mul[BM_MAXLEGS];   // per STORED leg: multiplier in the row / column index (0 if absent)
  int is_row[BM_MAXLEGS];
  long long coff[BM_MAXLEGS];                 // per stored leg: state offset of its charges
  long long NL, NR, nnz;
  Sym sym;
};

__global__ void bm_element_kernel(ElemParams p, const long long* __restrict__ charges, const int* __restrict__ bin_left,
                                  const long long* __restrict__ first, const long long* __restrict__ start_right,
                                  const long long* __restrict__ bucket, const int* __restrict__ row_rank, const int* __restrict__ col_rank,
                                  const long long* __restrict__ sect_off, const long long* __restrict__ ncols,
                                  long long* __restrict__ map) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= p.nnz) return;
  // l = last left state with first[l] <= e
  long long lo = 0, hi = p.NL;                // first[NL] = nnz > e
  while (hi - lo > 1) { const long long mid = (lo + hi) >> 1; if (first[mid] <= e) lo = mid; else hi = mid; }
  const long long l = lo, j = e - first[l];
  const long long r = bucket[start_right[bm_partner(bin_left[l], p.sym)] + j];
  long long R = 0, C = 0, rq[BM_MAXSYM];
#pragma unroll
  for (int k = 0; k < BM_MAXSYM; ++k) rq[k] = 0;
  long long rem = l;
#pragma unroll 1
  for (int i = p.left.n - 1; i >= 0; --i) {
    const long long d = rem % p.left.dim[i];
    rem /= p.left.dim[i];
    const int t = p.left.leg[i];
    R += d * p.row_mul[t]; C += d * p.col_mul[t];
    if (p.is_row[t]) bm_add(rq, charges, p.coff[t] + d, p.sym);
  }
  rem = r;
#pragma unroll 1
  for (int i = p.right.n - 1; i >= 0; --i) {
    const long long d = rem % p.right.dim[i];
    rem /= p.right.dim[i];
    const int t = p.right.leg[i];
    R += d * p.row_mul[t]; C += d * p.col_mul[t];
    if (p.is_row[t]) bm_add(rq, charges, p.coff[t] + d, p.sym);
  }
  const int qb = bm_bin(rq, p.sym);
  map[sect_off[qb] + (long long)row_rank[R] * ncols[qb] + col_rank[C]] = e;
}

// rank[] and cnt[] of the N bins in bin[]; returns the launch count or a negative status
int bm_rank(const int* bin, long long N, int nbins, int* rank, long long* cnt, cudaStream_t st) {
  if (nbins <= BM_PERBIN_MAX_BINS) {
    bm_rank_kernel<<<nbins, 1024, 0, st>>>(bin, N, rank, cnt);
    return 1;
  }
  const long long want = (N + BM_TILE_THREADS - 1) / BM_TILE_THREADS;
  const long long fit = BM_TILE_BUDGET / nbins;
  long long ntiles = fit < want ? fit : want;
  if (ntiles < 1) ntiles = 1;
  const long long T = (N + ntiles - 1) / ntiles;
  ntiles = (N + T - 1) / T;
  const long long M = (long long)nbins * ntiles;
  const long long nchunks = (M + BM_SCAN_CHUNK - 1) / BM_SCAN_CHUNK;    // <= BM_SCAN_CHUNK: M <= max(budget, max bins)
  int *tcnt = nullptr, *part = nullptr;
  int rc;
  if ((rc = ws_alloc((void**)&tcnt, sizeof(int) * (size_t)(M + 1), st))) return rc;
  if ((rc = ws_alloc((void**)&part, sizeof(int) * (size_t)nchunks, st))) return rc;
  TNB_CHECK_CUDA(cudaMemsetAsync(tcnt, 0, sizeof(int) * (size_t)(M + 1), st));
  bm_tile_rank_kernel<<<(unsigned)ntiles, BM_TILE_THREADS, 0, st>>>(bin, N, T, (int)ntiles, rank, tcnt);
  bm_scan_chunk_kernel<<<(unsigned)nchunks, BM_SCAN_THREADS, 0, st>>>(tcnt, M, part);
  bm_scan_chunk_kernel<<<1, BM_SCAN_THREADS, 0, st>>>(part, nchunks, tcnt + M);       // tcnt[M] = N
  bm_scan_add_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(tcnt, M, part);
  const long long n_fin = N > nbins ? N : nbins;
  bm_rank_finish_kernel<<<(unsigned)((n_fin + 255) / 256), 256, 0, st>>>(bin, N, T, (int)ntiles, tcnt, rank, nbins, cnt);
  ws_free(tcnt, st); ws_free(part, st);
  return 5;
}

int bm_maps(int nlegs, int nsym, const int64_t* dims, const int64_t* charges_dev, const int64_t* leg_off, const int32_t* order,
            int partition, int split, const int64_t* moduli, const int64_t* shifts, int nbins, const int64_t* tables_dev,
            int64_t nnz, int64_t* map_dev, void* stream) {
  TNB_REQUIRE(nlegs >= 1 && nlegs <= BM_MAXLEGS && partition >= 0 && partition <= nlegs && split >= 0 && split <= nlegs, TNB200_ERR_INVALID,
              "blocksparse_maps: bad leg counts");
  TNB_REQUIRE(nsym >= 1 && nsym <= BM_MAXSYM, TNB200_ERR_INVALID, "blocksparse_maps: nsym = %d outside [1, %d]", nsym, BM_MAXSYM);
  TNB_REQUIRE(dims && charges_dev && leg_off && order && moduli && shifts && tables_dev && (map_dev || nnz == 0) && nbins >= 1,
              TNB200_ERR_INVALID, "blocksparse_maps: null pointer");
  Sym sy;
  sy.n = nsym;
  long long bins = 1;
  for (int k = 0; k < BM_MAXSYM; ++k) { sy.mod[k] = 0; sy.shift[k] = 0; sy.radix[k] = 1; }
  for (int k = 0; k < nsym; ++k) {
    TNB_REQUIRE(moduli[k] >= 0 && shifts[k] >= 0, TNB200_ERR_INVALID, "blocksparse_maps: negative modulus or shift of component %d", k);
    sy.mod[k] = moduli[k];
    sy.shift[k] = moduli[k] > 0 ? 0 : shifts[k];
    sy.radix[k] = moduli[k] > 0 ? moduli[k] : 2 * shifts[k] + 1;
    bins = bins * sy.radix[k] > TNB200_BLOCKSPARSE_MAX_BINS ? TNB200_BLOCKSPARSE_MAX_BINS + 1LL : bins * sy.radix[k];
  }
  TNB_REQUIRE(bins <= TNB200_BLOCKSPARSE_MAX_BINS && nbins <= TNB200_BLOCKSPARSE_MAX_BINS, TNB200_ERR_UNSUPPORTED,
              "blocksparse_maps: the charges span more than TNB200_BLOCKSPARSE_MAX_BINS = %d bins", TNB200_BLOCKSPARSE_MAX_BINS);
  TNB_REQUIRE(bins == nbins, TNB200_ERR_INVALID, "blocksparse_maps: nbins = %d, the moduli and shifts give %lld", nbins, bins);
  if (nnz == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  // tables_dev (int64, uploaded by the caller): [start_right (nbins)] [sect_off (nbins)] [ncols (nbins)]
  const long long* start_right = (const long long*)tables_dev;
  const long long* sect_off = start_right + nbins;
  const long long* ncols = sect_off + nbins;
  auto group = [&](const int* legs, int n) {
    LegGroup g; g.n = n;
    for (int i = 0; i < BM_MAXLEGS; ++i) { g.leg[i] = 0; g.dim[i] = 1; g.coff[i] = 0; }
    for (int i = 0; i < n; ++i) { g.leg[i] = legs[i]; g.dim[i] = dims[legs[i]]; g.coff[i] = leg_off[legs[i]]; }
    return g;
  };
  auto total = [&](const LegGroup& g) { long long t = 1; for (int i = 0; i < g.n; ++i) t *= g.dim[i]; return t; };
  int stored[BM_MAXLEGS];
  for (int i = 0; i < nlegs; ++i) stored[i] = i;
  const LegGroup gl = group(stored, split), gr = group(stored + split, nlegs - split);
  const LegGroup grow = group(order, partition), gcol = group(order + partition, nlegs - partition);
  const long long NL = total(gl), NR = total(gr), NRo = total(grow), NCo = total(gcol);
  TNB_REQUIRE(NL < (1LL << 31) && NR < (1LL << 31) && NRo < (1LL << 31) && NCo < (1LL << 31), TNB200_ERR_UNSUPPORTED,
              "blocksparse_maps: a leg group has more than 2^31 states");
  int *bin_l = nullptr, *bin_r = nullptr, *bin_ro = nullptr, *bin_co = nullptr, *rank_r = nullptr, *rank_ro = nullptr, *rank_co = nullptr;
  long long *cnt = nullptr, *first = nullptr, *bucket = nullptr;
  int rc;
  if ((rc = ws_alloc((void**)&bin_l, sizeof(int) * (size_t)NL, st))) return rc;
  if ((rc = ws_alloc((void**)&bin_r, sizeof(int) * (size_t)NR, st))) return rc;
  if ((rc = ws_alloc((void**)&bin_ro, sizeof(int) * (size_t)NRo, st))) return rc;
  if ((rc = ws_alloc((void**)&bin_co, sizeof(int) * (size_t)NCo, st))) return rc;
  if ((rc = ws_alloc((void**)&rank_r, sizeof(int) * (size_t)NR, st))) return rc;
  if ((rc = ws_alloc((void**)&rank_ro, sizeof(int) * (size_t)NRo, st))) return rc;
  if ((rc = ws_alloc((void**)&rank_co, sizeof(int) * (size_t)NCo, st))) return rc;
  if ((rc = ws_alloc((void**)&cnt, sizeof(long long) * (size_t)nbins * 3, st))) return rc;
  if ((rc = ws_alloc((void**)&first, sizeof(long long) * (size_t)(NL + 1), st))) return rc;
  if ((rc = ws_alloc((void**)&bucket, sizeof(long long) * (size_t)NR, st))) return rc;
  const long long* ch = (const long long*)charges_dev;
  auto blocks = [](long long n) { return (unsigned)((n + 255) / 256); };
  bm_fuse_kernel<<<blocks(NL), 256, 0, st>>>(gl, sy, ch, NL, bin_l);
  bm_fuse_kernel<<<blocks(NR), 256, 0, st>>>(gr, sy, ch, NR, bin_r);
  bm_fuse_kernel<<<blocks(NRo), 256, 0, st>>>(grow, sy, ch, NRo, bin_ro);
  bm_fuse_kernel<<<blocks(NCo), 256, 0, st>>>(gcol, sy, ch, NCo, bin_co);
  int launches = 7;
  if ((rc = bm_rank(bin_r, NR, nbins, rank_r, cnt, st)) < 0) return rc;
  launches += rc;
  if ((rc = bm_rank(bin_ro, NRo, nbins, rank_ro, cnt + nbins, st)) < 0) return rc;
  launches += rc;
  if ((rc = bm_rank(bin_co, NCo, nbins, rank_co, cnt + 2 * nbins, st)) < 0) return rc;
  launches += rc;
  bm_first_kernel<<<1, 1024, 0, st>>>(bin_l, NL, cnt, sy, first);
  bm_bucket_kernel<<<blocks(NR), 256, 0, st>>>(bin_r, rank_r, NR, start_right, bucket);
  ElemParams p;
  p.left = gl; p.right = gr; p.NL = NL; p.NR = NR; p.nnz = nnz; p.sym = sy;
  for (int t = 0; t < BM_MAXLEGS; ++t) { p.row_mul[t] = 0; p.col_mul[t] = 0; p.is_row[t] = 0; p.coff[t] = 0; }
  for (int t = 0; t < nlegs; ++t) p.coff[t] = leg_off[t];
  { long long m = 1; for (int i = partition - 1; i >= 0; --i) { p.row_mul[order[i]] = m; p.is_row[order[i]] = 1; m *= dims[order[i]]; } }
  { long long m = 1; for (int i = nlegs - 1; i >= partition; --i) { p.col_mul[order[i]] = m; m *= dims[order[i]]; } }
  bm_element_kernel<<<blocks(nnz), 256, 0, st>>>(p, ch, bin_l, first, start_right, bucket, rank_ro, rank_co, sect_off, ncols, (long long*)map_dev);
  TNB_LAUNCH_CHECK();
  count_launch(launches);
  set_kernel_name("blocksparse_maps");
  ws_free(bin_l, st); ws_free(bin_r, st); ws_free(bin_ro, st); ws_free(bin_co, st); ws_free(rank_r, st); ws_free(rank_ro, st);
  ws_free(rank_co, st); ws_free(cnt, st); ws_free(first, st); ws_free(bucket, st);
  return 0;
}

}  // namespace tnb

using namespace tnb;

extern "C" int32_t tnb200_blocksparse_maps_nsym(int32_t nlegs, int32_t nsym, const int64_t* dims, const int64_t* charges_dev,
                                                const int64_t* leg_off, const int32_t* order, int32_t partition, int32_t split,
                                                const int64_t* moduli, const int64_t* shifts, int32_t nbins, const int64_t* tables_dev,
                                                int64_t nnz, int64_t* map_dev, void* stream) {
  return bm_maps(nlegs, nsym, dims, charges_dev, leg_off, order, partition, split, moduli, shifts, nbins, tables_dev, nnz, map_dev, stream);
}

extern "C" int32_t tnb200_blocksparse_maps(int32_t nlegs, const int64_t* dims, const int64_t* charges_dev, const int64_t* leg_off,
                                           const int32_t* order, int32_t partition, int32_t split, int64_t modulus, int64_t shift,
                                           int32_t nbins, const int64_t* tables_dev, int64_t nnz, int64_t* map_dev, void* stream) {
  return bm_maps(nlegs, 1, dims, charges_dev, leg_off, order, partition, split, &modulus, &shift, nbins, tables_dev, nnz, map_dev, stream);
}
