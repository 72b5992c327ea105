// gemm_wgmma.cu — the tensor-core path of tnb200_tensordot for bf16 / f16 / f32(tf32).
//
// One persistent, warp-specialised kernel per launch (H100, sm_90a), 384 threads:
//   warpgroup 0, warp 0 : TMA producer — cp.async.bulk.tensor (5-D tiled maps built over the *strided
//                         operand views*, so the tensordot's transpose is performed by the TMA engine),
//                         SWIZZLE_128B tiles into an S-stage shared-memory ring, mbarrier complete_tx.
//   warpgroups 1, 2     : consumers — each owns 64 rows of the 128 x BN output tile, issues
//                         wgmma.mma_async (m64 nBN, K = 32 bytes per instruction) from shared-memory
//                         descriptors into f32 register accumulators, releases ring slots once the
//                         MMAs that read them have retired, then stores the tile (converted) to C.
// 16-bit operands may be K-major (unit stride along the contracted mode) or MN-major (unit stride
// along the free mode): both are native wgmma layouts (transpose bit).  wgmma reads tf32 operands
// K-major only, so an MN-major f32 operand is loaded by TMA into a staging slot of the stage and
// transposed into the K-major layout in shared memory by the consumers — never repacked in HBM.
// Ragged edges in M, N, K are handled by TMA out-of-bounds zero fill + predicated stores.
//
// The chained variant runs a sequence of dependent GEMMs as tiles of the same kernel (see below); its
// consumers hand the tile to warp 1, which stores it with TMA while they start the next tile.
#include "gemm.cuh"
#include "wgmma.cuh"
#include <cuda.h>
#include <mutex>
#include <vector>

namespace tnb {

// ------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded wait: a protocol bug traps (visible as a CUDA error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
#pragma unroll 1
  for (uint32_t it = 0; it < (1u << 28); ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) return;
  }
  __trap();
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
// The same load issued to both CTAs of a 2-CTA cluster (mask 0b11): the box lands at the same shared-memory offset in
// each and signals the mbarrier at the same offset in each.
__device__ __forceinline__ void tma_load_5d_pair(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                                 int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2], %8;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "h"((uint16_t)0x3) : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// Arrive on the mbarrier at the same shared-memory offset as `bar` in CTA `cta` of the cluster.  Default semantics
// (release at CTA scope): the arrive only has to follow the wgmma reads of the slot, which wgmma.wait_group has
// retired.  .release.cluster puts a MEMBAR.ALL.GPU before every arrive: the chain's k loop took 1.6x as long with
// it in one measurement (bench cfg2, H100 SXM, 400 W).
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t}"
      ::"r"(bar), "r"(cta) : "memory");
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// wgmma shared-memory matrix descriptor, 128-byte swizzle.  K-major: rows of 128 bytes, 8-row groups
// SBO = 1024 B apart (LBO unused).  MN-major: 64-element MN chunks LBO apart, 8-row K groups SBO apart.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

struct TcParams {
  int64_t M, N, K, batch;
  int BN, num_kb, stages, out_kind;   // out_kind: 0 bf16, 1 f16, 2 f32
  int64_t tiles_m, tiles_n, num_tiles;
  int a_mn, b_mn;                     // operand is MN-major
  // multi-mode operands: extent of the INNER free / contracted mode (0 = the group is one mode).
  // TMA dims are always (K-major)  [k_in, f_in, f_out, k_out, batch]
  //                     (MN-major) [f_in, k_in, k_out, f_out, batch]
  uint32_t a_fe, a_ke, b_fe, b_ke;
  void* C; int64_t c_sm, c_sb;        // row stride / batch stride of the output tile rows
  int64_t c_cs;                       // column stride: 1 (normal) or the original row stride (swap-AB: the
                                      // kernel computes C^T tiles and stores them transposed)
  int vec_ok;
};

constexpr int kBM = 128;
constexpr int kRowBytes = 128;        // one swizzle row = BK elements
constexpr int kThreads = 384;

// ---------------------------------------------------------------------------------------------
// Chained GEMMs in ONE persistent launch.
//
// A contraction path often contains long runs of dependent GEMMs (the MPS "zipper": E' = A^T (E A) per site).
// Launched one by one, every step pays the persistent kernel's prologue + drain, and every intermediate makes
// a round trip through HBM.  Here all steps of such a run are tiles of ONE kernel: the tile sequence is ordered
// so that a small group of samples is carried through the whole run of steps before the next group starts
// (intermediates are produced and consumed while still in L2), and inter-step dependencies are tracked per
// (step, sample) with release/acquire counters in global memory: once the TMA stores of an output tile have
// completed, the CTA's store warp publishes the tile with red.release, the TMA producer of a dependent tile spins
// with ld.acquire + fence.proxy.async before its first load.
//
// The unit of the sequence is a *pair* of tiles: the same step, sample and N tile, M tiles 2j and 2j + 1, run by
// the two CTAs of a 2-CTA cluster (rank r takes M tile 2j + r).  The pair shares its B tile: each CTA loads its own
// A tile and one half of B, multicast into both CTAs, so a pair reads 2 x 128 + 256 operand rows per k block instead
// of 2 x (128 + 256), a third less L2 -> SM traffic (a 128 x 256 tile alone reads 85 flop per operand byte).  A
// ring slot is refilled only when the consumers of BOTH CTAs have released it: the empty barrier counts the
// consumer warps of the pair, each of which arrives in its own CTA and in the partner.  Both
// producers of a pair wait on the same dependency counters and walk the ring in the same order, which keeps the two
// CTAs in step.  When tiles_m is odd the partner of the last M tile has no tile: it still loads and multicasts its
// half of B and releases its slots, but issues no MMAs and stores and publishes nothing.  Each CTA publishes its own
// tile, so the counters still count tiles.  Pairs are assigned to clusters round-robin in sequence order and all
// clusters are co-resident (grid <= resident clusters), so a pair only ever waits for pairs that are earlier in the
// sequence: no deadlock.
//
// The chain's epilogue overlaps the next tile's k loop: the consumers convert the accumulators into a shared-memory
// staging buffer (128-byte swizzled 64-row x 128-byte boxes: conflict-free stores) and go on to the next tile; warp
// 1 writes the buffer out with TMA stores through a per-step tensor map of C, frees it once the TMA engine has
// read it, and publishes the tile once the stores are complete.  16-bit chains run 128 x 256 tiles, tf32 chains
// 128 x 128 (their MN-major transpose slot doubles a stage).  Either way a consumer warpgroup's 32 KB half of the
// output tile is staged in two 16 KB passes, so that the ring gets 4 stages of 48 KB (16-bit) or 3 of 64 KB (tf32).
//
// Measured on the bench's cfg2 chain (H100 SXM, 700 W; tools/chain_phases.py, one run per build): the 16-bit k loop
// waits on load latency more than on L2 bandwidth.  A stage is about 0.55 us of MMAs at 128 x 256.
//   3 stages, no pairs: launch 7.22 ms, consumers' wait for a stage 3.56 ms per CTA
//   pairs, 3 stages:    launch 7.19 ms, wait 3.57 ms (a run of its own against 7.16 / 3.58 ms without pairs)
//   4 stages, no pairs: launch 6.58 ms, wait 1.99 ms
//   pairs, 4 stages:    launch 6.85 ms, wait 1.93 ms
// So the 4th stage (room made by the two-pass epilogue) is what shortens the wait.  A third less L2 traffic does
// not, and a refill that waits for the slower CTA of the pair costs launch time.  Over three alternated bench runs
// the step took 10.28-10.45 ms (3 stages, no pairs), 9.96-10.08 ms (4 stages, no pairs) and 10.01-10.12 ms (pairs,
// 4 stages).
struct alignas(64) ChainStepDev {
  CUtensorMap tmA, tmB, tmC;
  TcParams p;
  int dep_a, dep_b;               // chain step that produces operand a / b (-1: available before the launch)
  uint32_t need_a, need_b;        // counter value of that step's (sample) entry when it is complete: its tiles
  int tiles_per_sample;
};
struct ChainSeg { long long tile0; int step, sample0, nsamples, pad; };   // tile0: first pair of the segment
struct ChainParams {
  const ChainStepDev* steps;
  const ChainSeg* segs;
  uint32_t* done;                 // [nsteps][batch] completion counters (zeroed before every launch)
  long long num_tiles;            // pairs
  int nsegs, batch, stages, stage_bytes;
};
constexpr int kConsumerWarps = 8;     // consumer warps per CTA: each releases ring slots
// Chain epilogue staging, per consumer warpgroup: 64 rows x 512 bytes of output = four 8 KB boxes, two per pass.
constexpr int kChainBN16 = 256, kChainBN32 = 128;
constexpr int kBoxBytes = 64 * 128;
constexpr int kChainStageHalf = 2 * kBoxBytes;

// Everything one launch needs: a single GEMM (tile params + maps) or a chain.
struct KernelArgs {
  CUtensorMap tmA, tmB;
  TcParams p;
  ChainParams cp;
  int stage_bytes;
};

__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_add_u32(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
#ifdef TNB200_CHAIN_PHASES
// Diagnostic build only (tools/chain_phases.py; never part of the library): per CTA, nanoseconds of %globaltimer
// spent in each phase of the chained kernel, accumulated over launches.  Each slot has a single writer thread.
constexpr int kPhases = 6;        // producer chain_wait, consumer full-barrier wait, k loop, epilogue, CTA lifetime, tiles
constexpr int kPhaseCtas = 1024;
__device__ unsigned long long g_chain_phase[kPhaseCtas * kPhases];
__device__ __forceinline__ unsigned long long phase_clock() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
  return t;
}
#define TNB_PHASE(...) __VA_ARGS__
#define TNB_PHASE_ADD(slot, v) (g_chain_phase[blockIdx.x * kPhases + (slot)] += (v))
#else
#define TNB_PHASE(...)
#endif

// bounded spin on a dependency counter (a scheduling bug traps instead of hanging the GPU)
__device__ __forceinline__ void chain_wait(const uint32_t* ctr, uint32_t need) {
#pragma unroll 1
  for (uint32_t it = 0; it < (1u << 24); ++it) {
    if (ld_acquire_u32(ctr) >= need) return;
    __nanosleep(64);
  }
  __trap();
}

struct Tile {
  const TcParams* p;
  const CUtensorMap *ma, *mb;
  const ChainStepDev* sd;         // chain step (nullptr for a single GEMM)
  int bi, mi, ni, step;
  bool live;                      // false: the partner of the last M tile when tiles_m is odd (chain only)
};
// Single GEMM: `tile` is a tile.  Chain: `tile` is a pair and `rank` the CTA's rank in the cluster.
template <bool CHAIN>
__device__ __forceinline__ void decode_tile(const KernelArgs& a, long long tile, int rank, int& cursor, Tile& t) {
  if (!CHAIN) {
    uint32_t x = (uint32_t)tile;
    const uint32_t tn = (uint32_t)a.p.tiles_n, tm = (uint32_t)a.p.tiles_m;
    t.ni = (int)(x % tn); x /= tn;
    t.mi = (int)(x % tm);
    t.bi = (int)(x / tm);
    t.p = &a.p; t.ma = &a.tmA; t.mb = &a.tmB; t.sd = nullptr; t.step = 0;
    t.live = true;
  } else {
    const ChainParams& cp = a.cp;
    while (cursor + 1 < cp.nsegs && tile >= cp.segs[cursor + 1].tile0) ++cursor;
    const ChainSeg sg = cp.segs[cursor];
    const ChainStepDev* sd = cp.steps + sg.step;
    uint32_t local = (uint32_t)(tile - sg.tile0);
    const uint32_t tn = (uint32_t)sd->p.tiles_n, tm = (uint32_t)sd->p.tiles_m, pm = (tm + 1) / 2;
    t.ni = (int)(local % tn); local /= tn;
    t.mi = 2 * (int)(local % pm) + rank;
    t.bi = sg.sample0 + (int)(local / pm);
    t.step = sg.step;
    t.p = &sd->p; t.ma = &sd->tmA; t.mb = &sd->tmB; t.sd = sd;
    t.live = (uint32_t)t.mi < tm;
  }
}

// Transpose the MN-major f32 staging tiles of one stage (TMA layout: chunks of 32 MN elements x 32 K rows,
// 128-byte rows, 128B swizzle) into the K-major 128B-swizzled rows wgmma reads.  All 256 consumer threads;
// a warp covers 32 consecutive MN rows of one 16-byte K group: conflict-free reads, 8 rows per store wave.
__device__ __forceinline__ void transpose_stage_tf32(uint32_t stage, int a_mn, int b_mn, int BN, int ctid) {
  const uint32_t a_bytes = kBM * kRowBytes, b_bytes = (uint32_t)BN * kRowBytes;
  const uint32_t staging = stage + a_bytes + b_bytes;
  const int rows_a = a_mn ? kBM : 0, rows = rows_a + (b_mn ? BN : 0);
#pragma unroll 1
  for (int idx = ctid; idx < rows * 8; idx += 256) {
    const int m = idx & 31, rest = idx >> 5, kc = rest & 7;
    const int r = (rest >> 3) * 32 + m;                       // row across A rows then B rows
    const bool is_a = r < rows_a;
    const int rr = is_a ? r : r - rows_a;
    const uint32_t src = staging + (is_a ? 0u : a_bytes) + (uint32_t)(rr >> 5) * 4096u;
    const uint32_t dst = stage + (is_a ? 0u : a_bytes) + (uint32_t)rr * 128u + (uint32_t)((kc ^ (rr & 7)) << 4);
    uint32_t v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int k = kc * 4 + i;
      const uint32_t addr = src + (uint32_t)k * 128u + (uint32_t)((((m >> 2) ^ (k & 7)) << 4) | ((m & 3) << 2));
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v[i]) : "r"(addr) : "memory");
    }
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3]) : "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma (async proxy) reads
}

template <int KIND, int BN, int TA, int TB>
__device__ __forceinline__ void mma_k(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (KIND == 2) {
    if constexpr (BN == 64) wgmma_n64_tf32(d, a, b, acc);
    else if constexpr (BN == 128) wgmma_n128_tf32(d, a, b, acc);
    else wgmma_n256_tf32(d, a, b, acc);
  } else if constexpr (KIND == 0) {
    if constexpr (BN == 64) wgmma_n64_bf16<TA, TB>(d, a, b, acc);
    else if constexpr (BN == 128) wgmma_n128_bf16<TA, TB>(d, a, b, acc);
    else wgmma_n256_bf16<TA, TB>(d, a, b, acc);
  } else {
    if constexpr (BN == 64) wgmma_n64_f16<TA, TB>(d, a, b, acc);
    else if constexpr (BN == 128) wgmma_n128_f16<TA, TB>(d, a, b, acc);
    else wgmma_n256_f16<TA, TB>(d, a, b, acc);
  }
}

// Release ring slot `bar` (its empty barrier) from one consumer warp: in the chain, to the producers of both CTAs of
// the pair, since either may refill the slot's B half in both.
template <bool PAIR>
__device__ __forceinline__ void release_slot(uint32_t bar) {
  if constexpr (PAIR) { mbar_arrive_cluster(bar, 0); mbar_arrive_cluster(bar, 1); }
  else mbar_arrive(bar);
}

// The k loop of the partner that has no tile: it takes every stage as the live CTA does (so that the partner's
// multicast has landed before the slot is released) and releases it at once.
__device__ __forceinline__ void drainloop(int S, uint32_t bar_base, int num_kb, int lane, int& s, uint32_t& ph) {
#pragma unroll 1
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(bar_base + 8u * s, ph);
    __syncwarp();
    if (lane == 0) release_slot<true>(bar_base + 8u * (S + s));
    if (++s == S) { s = 0; ph ^= 1; }
  }
}

// The k loop of one tile for one consumer warpgroup.  The operand majorness is a template parameter so that
// the wgmma sequence is straight-line code.  Descriptor fields: a K-major operand advances 32 bytes per MMA,
// an MN-major one 16 K rows (2 KB); MN chunks of 64 elements are BK rows x 128 B apart.
template <int KIND, int BN, int TA, int TB, bool PAIR>
__device__ __forceinline__ void mainloop(float* d, uint8_t* smem, int stage_bytes, int S, uint32_t bar_base, int num_kb,
                                         int a_mn, int b_mn, int wg, int ctid, int lane, int& s, uint32_t& ph) {
  constexpr int BK = kRowBytes / (KIND == 2 ? 4 : 2);
  constexpr uint32_t a_lbo = TA ? BK * kRowBytes : 16u, b_lbo = TB ? BK * kRowBytes : 16u;
  constexpr uint32_t a_kstep = TA ? 16u * kRowBytes : 32u, b_kstep = TB ? 16u * kRowBytes : 32u;
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    TNB_PHASE(const unsigned long long tw = phase_clock();)
    mbar_wait(bar_base + 8u * s, ph);
    TNB_PHASE(if (ctid == 0) TNB_PHASE_ADD(1, phase_clock() - tw);)
    const uint32_t sa = smem_u32(smem + (size_t)s * stage_bytes);
    if (KIND == 2 && (a_mn || b_mn)) {
      transpose_stage_tf32(sa, a_mn, b_mn, BN, ctid);
      consumers_sync();
    }
    const uint32_t sa_wg = sa + (uint32_t)wg * 64u * kRowBytes;   // 64 rows (K-major) = one 64-element chunk (MN-major)
    const uint32_t sb = sa + kBM * kRowBytes;
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      mma_k<KIND, BN, TA, TB>(d, gmma_desc(sa_wg + k * a_kstep, a_lbo, 1024u), gmma_desc(sb + k * b_kstep, b_lbo, 1024u),
                              (kb > 0 || k > 0) ? 1u : 0u);
    wg_commit();
    if (prev >= 0) {
      wg_wait<1>();                                            // the MMAs of the previous stage have retired
      __syncwarp();
      if (lane == 0) release_slot<PAIR>(bar_base + 8u * (S + prev));
    }
    prev = s;
    if (++s == S) { s = 0; ph ^= 1; }
  }
  wg_wait<0>();
  __syncwarp();
  if (lane == 0) release_slot<PAIR>(bar_base + 8u * (S + prev));
}

__device__ __forceinline__ void store_one(const TcParams& p, int64_t off, float v) {
  if (p.out_kind == 2) ((float*)p.C)[off] = v;
  else if (p.out_kind == 0) ((__nv_bfloat16*)p.C)[off] = __float2bfloat16_rn(v);
  else ((__half*)p.C)[off] = __float2half_rn(v);
}
__device__ __forceinline__ void store_pair(const TcParams& p, int64_t off, float v0, float v1) {
  if (p.out_kind == 2) *(float2*)((float*)p.C + off) = make_float2(v0, v1);
  else if (p.out_kind == 0) *(__nv_bfloat162*)((__nv_bfloat16*)p.C + off) = __floats2bfloat162_rn(v0, v1);
  else *(__half2*)((__half*)p.C + off) = __floats2half2_rn(v0, v1);
}

template <int KIND, int BN, bool CHAIN>
__global__ void __launch_bounds__(kThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ KernelArgs args) {
  constexpr int ES = KIND == 2 ? 4 : 2;          // operand element bytes
  constexpr int BK = kRowBytes / ES;             // 64 (16-bit) or 32 (tf32) elements per k-block
  constexpr int CHUNK = kRowBytes / ES;          // MN elements per 128-byte row of an MN-major tile
  constexpr int A_BYTES = kBM * kRowBytes;       // 16 KB per stage
  constexpr int B_BYTES = BN * kRowBytes;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  const int STAGE_BYTES = args.stage_bytes;
  const int S = CHAIN ? args.cp.stages : args.p.stages;
  const long long num_tiles = CHAIN ? args.cp.num_tiles : args.p.num_tiles;
  // chain: the epilogue staging buffer (one half per consumer warpgroup) follows the ring
  constexpr int STAGE_HALF = kChainStageHalf;
  const uint32_t staging = smem_u32(smem + (size_t)S * STAGE_BYTES);
  uint64_t* bars = (uint64_t*)(smem + (size_t)S * STAGE_BYTES + (CHAIN ? 2 * STAGE_HALF : 0));
  const uint32_t bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };       // bars: full[S], empty[S], staged[2], freed[2]
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };
  auto staged_bar = [&](int wg) { return bar_base + 8u * (2 * S + wg); };
  auto freed_bar = [&](int wg) { return bar_base + 8u * (2 * S + 2 + wg); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  TNB_PHASE(const unsigned long long t_start = phase_clock();)
  if (threadIdx.x == 0) {
    if (!CHAIN) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&args.tmA) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&args.tmB) : "memory");
    }
    // chain: the consumer warps of both CTAs of the pair release a slot
    for (int s = 0; s < S; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), (CHAIN ? 2 : 1) * kConsumerWarps);
    }
    if (CHAIN)
      for (int wg = 0; wg < 2; ++wg) { mbar_init(staged_bar(wg), 4); mbar_init(freed_bar(wg), 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // chain: the partner's multicast loads and remote arrives target this CTA's barriers from the start
  if constexpr (CHAIN) cluster_sync();
  else __syncthreads();
  // chain: cluster c runs pairs c, c + clusters, ...; its CTA of rank r takes M tile 2j + r of each
  const int rank = CHAIN ? (int)cluster_ctarank() : 0;
  const long long first = CHAIN ? blockIdx.x / 2 : blockIdx.x, step = CHAIN ? gridDim.x / 2 : gridDim.x;

  if (warp == 0) {
    // ===================================================== TMA producer (whole warp)
    // lane l owns "load slot" l of a stage: one box of A (slots 0..nA-1) or of B (nA..nA+nB-1), so the boxes of a
    // stage are issued in parallel; inside the k loop a lane only advances its contracted-mode coordinates
    // incrementally.  A box covers 128 bytes of an MN-major operand's free mode, or all kBM rows of a K-major A and
    // BN / B_SPLIT rows of a K-major B.  In the chain each CTA loads B half `rank` and multicasts it to the pair.
    constexpr int B_SPLIT = CHAIN ? 2 : 1;
    int s = 0; uint32_t ph = 0;
    int cursor = 0;
    for (long long tile = first; tile < num_tiles; tile += step) {
      Tile t;
      decode_tile<CHAIN>(args, tile, rank, cursor, t);
      const TcParams& p = *t.p;
      const int a_mn = p.a_mn, b_mn = p.b_mn;
      const int nA = t.live ? (a_mn ? kBM / CHUNK : 1) : 0;
      const int nB = b_mn ? BN / CHUNK / B_SPLIT : 1;
      const bool mine = lane < nA + nB;
      const bool is_a = lane < nA;
      const bool mn = is_a ? (a_mn != 0) : (b_mn != 0);
      const int c = is_a ? lane : rank * nB + lane - nA;          // box index inside the operand tile
      const int fbox = mn ? CHUNK : (is_a ? kBM : BN / B_SPLIT);  // free elements of one box (BK = CHUNK K rows)
      const uint32_t fe = is_a ? p.a_fe : p.b_fe, ke = is_a ? p.a_ke : p.b_ke;
      const CUtensorMap* map = is_a ? t.ma : t.mb;
      uint32_t dst_off = (is_a ? 0u : (uint32_t)A_BYTES) + (uint32_t)(c * fbox * kRowBytes);
      if (KIND == 2 && mn) dst_off += A_BYTES + B_BYTES;          // f32 MN-major: staging slot, transposed by the consumers
      const int f = (is_a ? t.mi * kBM : t.ni * BN) + c * fbox;
      const int f_in = fe ? (int)((uint32_t)f % fe) : f, f_out = fe ? (int)((uint32_t)f / fe) : 0;
      const uint32_t tx_bytes = (t.live ? A_BYTES : 0) + B_BYTES;  // B: both halves land here
      const int num_kb = p.num_kb;
      if (CHAIN) {
        // operands produced by earlier steps of this launch: wait until every tile of (that step, this sample) is out
        if (lane == 0) {
          TNB_PHASE(const unsigned long long tw = phase_clock();)
          const ChainStepDev* sd = t.sd;
          if (sd->dep_a >= 0) chain_wait(args.cp.done + (size_t)sd->dep_a * args.cp.batch + t.bi, sd->need_a);
          if (sd->dep_b >= 0) chain_wait(args.cp.done + (size_t)sd->dep_b * args.cp.batch + t.bi, sd->need_b);
          TNB_PHASE(TNB_PHASE_ADD(0, phase_clock() - tw);)
        }
        __syncwarp();
        asm volatile("fence.proxy.async;" ::: "memory");     // generic-proxy writes (other SMs' epilogues) -> our TMA reads
      }
      int k_in = 0, k_out = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(empty_bar(s), ph ^ 1);                          // slot free (every lane observes it)
        const uint32_t full = full_bar(s);
        if (lane == 0) mbar_expect_tx(full, tx_bytes);
        __syncwarp();
        if (mine) {
          const uint32_t dst = smem_u32(smem + (size_t)s * STAGE_BYTES) + dst_off;
          const int x0 = mn ? f_in : k_in, x1 = mn ? k_in : f_in, x2 = mn ? k_out : f_out, x3 = mn ? f_out : k_out;
          if (CHAIN && !is_a) tma_load_5d_pair(dst, map, full, x0, x1, x2, x3, t.bi);
          else                tma_load_5d(dst, map, full, x0, x1, x2, x3, t.bi);
        }
        k_in += BK;
        if (ke && (uint32_t)k_in >= ke) { k_in = 0; ++k_out; }
        if (++s == S) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================================================== consumers: MMA + epilogue
    const int ctid = threadIdx.x - 128;                           // 0..255
    const int wg = ctid >> 7;                                     // rows 64 wg .. 64 wg + 63 of the tile
    const int wt = ctid & 127;
    int s = 0; uint32_t ph = 0;
    uint32_t eph = 0;                                             // chain: staging-buffer phase
    int cursor = 0;
    float d[BN / 2];
    for (long long tile = first; tile < num_tiles; tile += step) {
      Tile t;
      decode_tile<CHAIN>(args, tile, rank, cursor, t);
      const TcParams& p = *t.p;
      const int a_mn = p.a_mn, b_mn = p.b_mn, num_kb = p.num_kb;
      if (CHAIN && !t.live) {
        drainloop(S, bar_base, num_kb, lane, s, ph);
        continue;
      }
      TNB_PHASE(const unsigned long long tk = phase_clock();)
      if constexpr (KIND == 2) {
        mainloop<KIND, BN, 0, 0, CHAIN>(d, smem, STAGE_BYTES, S, bar_base, num_kb, a_mn, b_mn, wg, ctid, lane, s, ph);
      } else {
        if (a_mn && b_mn) mainloop<KIND, BN, 1, 1, CHAIN>(d, smem, STAGE_BYTES, S, bar_base, num_kb, a_mn, b_mn, wg, ctid, lane, s, ph);
        else if (a_mn) mainloop<KIND, BN, 1, 0, CHAIN>(d, smem, STAGE_BYTES, S, bar_base, num_kb, a_mn, b_mn, wg, ctid, lane, s, ph);
        else if (b_mn) mainloop<KIND, BN, 0, 1, CHAIN>(d, smem, STAGE_BYTES, S, bar_base, num_kb, a_mn, b_mn, wg, ctid, lane, s, ph);
        else mainloop<KIND, BN, 0, 0, CHAIN>(d, smem, STAGE_BYTES, S, bar_base, num_kb, a_mn, b_mn, wg, ctid, lane, s, ph);
      }
      TNB_PHASE(const unsigned long long te = phase_clock(); if (ctid == 0) TNB_PHASE_ADD(2, te - tk);)
      const int r0 = (wt >> 5) * 16 + (lane >> 2);
      if constexpr (CHAIN) {
        // ---- epilogue into the staging buffer; warp 1 stores it.  Accumulator d[4j + 2h + e] is row r0 + 8h,
        // column 8j + 2(lane & 3) + e; a box holds 128 bytes of 64 rows, its 16-byte chunk c of row r at c ^ (r & 7).
        constexpr int J_PER_PASS = BN / 8 * STAGE_HALF / (4 * kBoxBytes);
        const uint32_t half = staging + (uint32_t)wg * STAGE_HALF;
#pragma unroll
        for (int pass = 0; pass < 4 * kBoxBytes / STAGE_HALF; ++pass) {
          mbar_wait(freed_bar(wg), eph ^ 1);                       // the store warp has read the previous contents
#pragma unroll
          for (int jj = 0; jj < J_PER_PASS; ++jj) {
            const int j = pass * J_PER_PASS + jj;
            const uint32_t colb = (uint32_t)(8 * j + 2 * (lane & 3)) * ES - (uint32_t)pass * STAGE_HALF / 64;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t r = (uint32_t)(r0 + 8 * h);
              const uint32_t addr = half + (colb >> 7) * kBoxBytes + r * 128u + ((((colb >> 4) & 7) ^ (r & 7)) << 4) + (colb & 15);
              const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
              if constexpr (KIND == 2) {
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
              } else {
                uint32_t u;
                if constexpr (KIND == 0) { __nv_bfloat162 x = __floats2bfloat162_rn(v0, v1); u = *(uint32_t*)&x; }
                else { __half2 x = __floats2half2_rn(v0, v1); u = *(uint32_t*)&x; }
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(u) : "memory");
              }
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic writes -> TMA (async proxy) reads
          __syncwarp();
          if (lane == 0) mbar_arrive(staged_bar(wg));
          eph ^= 1;
        }
        TNB_PHASE(if (ctid == 0) { TNB_PHASE_ADD(3, phase_clock() - te); TNB_PHASE_ADD(5, 1); })
        continue;
      }
      // ---- epilogue straight from the accumulator registers
      const int64_t row0 = (int64_t)t.mi * kBM + wg * 64 + r0;
      const int64_t n0 = (int64_t)t.ni * BN + 2 * (lane & 3);
      const int64_t cb = (int64_t)t.bi * p.c_sb;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = row0 + 8 * h;
        if (row < p.M) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int64_t col = n0 + 8 * j;
            const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
            if (p.c_cs == 1) {
              const int64_t off = cb + row * p.c_sm + col;
              if (p.vec_ok && col + 1 < p.N) store_pair(p, off, v0, v1);
              else {
                if (col < p.N) store_one(p, off, v0);
                if (col + 1 < p.N) store_one(p, off + 1, v1);
              }
            } else {
              const int64_t off = cb + row * p.c_sm + col * p.c_cs;
              if (col < p.N) store_one(p, off, v0);
              if (col + 1 < p.N) store_one(p, off + p.c_cs, v1);
            }
          }
        }
      }
    }
    TNB_PHASE(if (ctid == 0) TNB_PHASE_ADD(4, phase_clock() - t_start);)
  } else if (CHAIN && warp == 1 && lane == 0) {
    // ===================================================== chain: store warp
    int cursor = 0;
    uint32_t sph = 0;
    for (long long tile = first; tile < num_tiles; tile += step) {
      Tile t;
      decode_tile<CHAIN>(args, tile, rank, cursor, t);
      if (!t.live) continue;
      const CUtensorMap* mc = &t.sd->tmC;
#pragma unroll 1
      for (int pass = 0; pass < 4 * kBoxBytes / STAGE_HALF; ++pass) {
#pragma unroll 1
        for (int wg = 0; wg < 2; ++wg) {
          mbar_wait(staged_bar(wg), sph);
          for (int b = 0; b < STAGE_HALF / kBoxBytes; ++b) {
            const int box = pass * (STAGE_HALF / kBoxBytes) + b;
            tma_store_3d(mc, staging + (uint32_t)(wg * STAGE_HALF + b * kBoxBytes), t.ni * BN + box * (128 / ES),
                         t.mi * kBM + wg * 64, t.bi);
          }
          bulk_commit();
          bulk_wait_read_all();
          mbar_arrive(freed_bar(wg));
        }
        sph ^= 1;
      }
      // Publish the tile.  wait_group (without .read) returns once the bulk stores are complete, i.e. their writes
      // to global memory have been performed.  Those writes belong to the async proxy; fence.proxy.async orders them
      // with this thread's generic-proxy accesses, so the red.release that follows publishes them at gpu scope.  A
      // dependent producer pairs it with ld.acquire and its own fence.proxy.async before its TMA (async-proxy) loads.
      bulk_wait_all();
      asm volatile("fence.proxy.async.global;" ::: "memory");
      red_release_add_u32(args.cp.done + (size_t)t.step * args.cp.batch + t.bi, 1u);
    }
  }
  // chain: neither CTA exits while its partner can still arrive on its barriers
  if constexpr (CHAIN) cluster_sync();
}

// ------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  });
  return fn;
}

static int es_of(int dt) { return dt == TNB200_F32 ? 4 : 2; }
static int kind_of(int dt) { return dt == TNB200_BF16 ? 0 : (dt == TNB200_F16 ? 1 : 2); }

// Which operand majorness can serve this view?  0: K-major, 1: MN-major, -1: neither (needs a repack).
// Conditions (es = element bytes, R = 128/es elements per swizzle row):
//   * unit stride on the innermost contracted mode (K-major) or innermost free mode (MN-major);
//   * every other stride and the base pointer 16-byte aligned; rank <= 5 (<= 2 modes per group);
//   * two contracted modes: inner extent % R == 0 (a k-block never straddles the mode boundary);
//   * two free modes: MN-major: inner extent % R == 0;  K-major: inner extent % 256 == 0, or a
//     power of two <= 64 (so every tile size 64/128/256 either divides it or is a multiple of it).
static int view_major(int dtype, const OperandView& v, int64_t ext_f, int64_t ext_k, int64_t batch) {
  if (dtype != TNB200_F32 && dtype != TNB200_F16 && dtype != TNB200_BF16) return -1;
  const int es = es_of(dtype);
  const int64_t R = kRowBytes / es;
  if (((uintptr_t)v.ptr) & 15) return -1;
  if (v.nF > 2 || v.nK > 2) return -1;
  if (ext_f >= (1LL << 31) || ext_k >= (1LL << 31) || batch >= (1LL << 31)) return -1;
  auto ok16 = [&](int64_t s) { return s > 0 && (s * es) % 16 == 0 && s * es < (1LL << 40); };
  if (batch > 1 && !ok16(v.sb)) return -1;
  if (v.nK == 2 && v.ke[1] % R != 0) return -1;
  const bool k_unit = ext_k == 1 || v.nK == 0 || v.ks[v.nK - 1] == 1;
  const bool f_unit = ext_f == 1 || v.nF == 0 || v.fs[v.nF - 1] == 1;
  if (k_unit) {  // K-major candidate: all free strides + outer K stride must be 16B multiples
    bool ok = true;
    for (int i = 0; i < v.nF; ++i) ok = ok && (v.fe[i] == 1 || ok16(v.fs[i]));
    if (v.nK == 2) ok = ok && ok16(v.ks[0]);
    if (v.nF == 2) { int64_t e = v.fe[1]; ok = ok && (e % 256 == 0 || (e <= 64 && (e & (e - 1)) == 0)); }
    if (ok) return 0;
  }
  if (f_unit) {
    bool ok = true;
    for (int i = 0; i < v.nK; ++i) ok = ok && (v.ke[i] == 1 || ok16(v.ks[i]));
    if (v.nF == 2) ok = ok && ok16(v.fs[0]) && (v.fe[1] % R == 0);
    if (ok) return 1;
  }
  return -1;
}

bool tma_view_ok(int dtype, const OperandView& v, int64_t ext_f, int64_t ext_k, int64_t batch) {
  return view_major(dtype, v, ext_f, ext_k, batch) >= 0;
}

// Build the rank-5 tensor map of one operand for tiles of `tile` free rows.
static int encode_operand(CUtensorMap* map, int dtype, const OperandView& v, int64_t ext_f, int64_t ext_k, int64_t batch,
                          int tile, bool& mn_major, uint32_t& fe_in, uint32_t& ke_in) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return TNB200_ERR_UNSUPPORTED;
  const int major = view_major(dtype, v, ext_f, ext_k, batch);
  if (major < 0) return TNB200_ERR_UNSUPPORTED;
  mn_major = major == 1;
  const int es = es_of(dtype);
  const int R = kRowBytes / es;
  CUtensorMapDataType cdt = dtype == TNB200_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                            : (dtype == TNB200_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  // (extent, stride) of inner / outer mode of each group; missing modes are extent 1
  int64_t f_in_e = v.nF ? v.fe[v.nF - 1] : 1, f_in_s = v.nF ? v.fs[v.nF - 1] : 0;
  int64_t f_out_e = v.nF == 2 ? v.fe[0] : 1, f_out_s = v.nF == 2 ? v.fs[0] : 0;
  int64_t k_in_e = v.nK ? v.ke[v.nK - 1] : 1, k_in_s = v.nK ? v.ks[v.nK - 1] : 0;
  int64_t k_out_e = v.nK == 2 ? v.ke[0] : 1, k_out_s = v.nK == 2 ? v.ks[0] : 0;
  fe_in = v.nF == 2 ? (uint32_t)f_in_e : 0u;
  ke_in = v.nK == 2 ? (uint32_t)k_in_e : 0u;
  int64_t de[5], ds[5];   // extents, element strides (ds[0] is the unit-stride dim)
  cuuint32_t box[5] = {1, 1, 1, 1, 1}, estr[5] = {1, 1, 1, 1, 1};
  if (!mn_major) {
    de[0] = k_in_e; ds[0] = 1;
    de[1] = f_in_e; ds[1] = f_in_s; de[2] = f_out_e; ds[2] = f_out_s;
    de[3] = k_out_e; ds[3] = k_out_s; de[4] = batch; ds[4] = v.sb;
    box[0] = R;
    if (v.nF == 2 && f_in_e < tile) {
      if (tile % f_in_e) return TNB200_ERR_UNSUPPORTED;
      box[1] = (cuuint32_t)f_in_e; box[2] = (cuuint32_t)(tile / f_in_e);
    } else {
      if (v.nF == 2 && f_in_e % tile) return TNB200_ERR_UNSUPPORTED;
      box[1] = tile;
    }
  } else {
    de[0] = f_in_e; ds[0] = 1;
    de[1] = k_in_e; ds[1] = k_in_s; de[2] = k_out_e; ds[2] = k_out_s;
    de[3] = f_out_e; ds[3] = f_out_s; de[4] = batch; ds[4] = v.sb;
    box[0] = R; box[1] = R;   // R elements of the free mode (128 B) x BK = R contracted rows
  }
  cuuint64_t dims[5], strides[4];
  int64_t natural = 16;   // bytes: a packed stride for extent-1 (never addressed) dims
  for (int d = 0; d < 5; ++d) {
    dims[d] = (cuuint64_t)(de[d] < 1 ? 1 : de[d]);
    int64_t bytes = es;
    if (d > 0) {
      bytes = ds[d] * es;
      if (de[d] <= 1) bytes = (natural + 15) / 16 * 16;
      else if (bytes <= 0 || bytes % 16) return TNB200_ERR_UNSUPPORTED;
      strides[d - 1] = (cuuint64_t)bytes;
    }
    if ((int64_t)dims[d] * bytes > natural) natural = (int64_t)dims[d] * bytes;
  }
  CUresult r = enc(map, cdt, 5, const_cast<void*>(v.ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return TNB200_ERR_UNSUPPORTED;
  return 0;
}

// Tensor map of a chain step's output C = [batch][M rows at c_sm][N contiguous] for the TMA-store epilogue:
// boxes of 64 rows x 128 bytes in the 128-byte swizzle the consumers stage them in.  TMA clips ragged edges.
static int encode_output(CUtensorMap* map, const GemmProblem& g) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return TNB200_ERR_UNSUPPORTED;
  const int64_t es = es_of(g.dtype);
  if (((uintptr_t)g.C) & 15 || g.c_sm <= 0 || (g.c_sm * es) % 16) return TNB200_ERR_UNSUPPORTED;
  if (g.batch > 1 && (g.c_sb <= 0 || (g.c_sb * es) % 16)) return TNB200_ERR_UNSUPPORTED;
  const CUtensorMapDataType cdt = g.dtype == TNB200_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                  : (g.dtype == TNB200_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
  cuuint64_t dims[3] = {(cuuint64_t)g.N, (cuuint64_t)g.M, (cuuint64_t)g.batch};
  cuuint64_t strides[2] = {(cuuint64_t)(g.c_sm * es), (cuuint64_t)((g.batch > 1 ? g.c_sb : g.M * g.c_sm) * es)};
  cuuint32_t box[3] = {(cuuint32_t)(kRowBytes / es), 64, 1}, estr[3] = {1, 1, 1};
  CUresult r = enc(map, cdt, 3, g.C, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : TNB200_ERR_UNSUPPORTED;
}

// bytes of one ring stage: A and B tiles, plus the staging slots of f32 MN-major operands
static int stage_bytes_of(int dtype, int BN, bool a_mn, bool b_mn) {
  const int kmajor = kBM * kRowBytes + BN * kRowBytes;
  return (dtype == TNB200_F32 && (a_mn || b_mn)) ? 2 * kmajor : kmajor;
}
constexpr int kRingBudget = 200 * 1024;

struct TcPrep {
  TcParams p;
  CUtensorMap tmA, tmB;
  int stage_bytes;
};

// Tile selection and tensor maps of one GEMM.  chain_mode: the problem is one step of a chained launch, whose
// steps share one kernel instance: 128 x 256 tiles (16-bit) or 128 x 128 (tf32).
static int tc_prepare(const GemmProblem& g, bool chain_mode, TcPrep& o) {
  TcParams& p = o.p;
  const int es = es_of(g.dtype);
  const int sms = num_sms();
  const int64_t tiles_m = (g.M + kBM - 1) / kBM;
  int BN = 64;   // multiples of 64 so that an MN-major B tile is a whole number of 128-byte chunks
  if (chain_mode) {
    BN = g.dtype == TNB200_F32 ? kChainBN32 : kChainBN16;
  } else if (!g.swapped) {
    const int cands[3] = {256, 128, 64};
    for (int i = 0; i < 3; ++i) {
      int bn = cands[i];
      if (bn > 64 && bn / 2 >= g.N) continue;          // tile mostly empty
      int64_t tiles = tiles_m * ((g.N + bn - 1) / bn) * g.batch;
      if (tiles >= sms || bn == 64) { BN = bn; break; }
    }
  }
  p.M = g.M; p.N = g.N; p.K = g.K; p.batch = g.batch;
  p.BN = BN;
  const int bk = kRowBytes / es;
  p.num_kb = (int)((g.K + bk - 1) / bk);
  p.tiles_m = tiles_m;
  p.tiles_n = (g.N + BN - 1) / BN;
  p.num_tiles = p.tiles_m * p.tiles_n * g.batch;
  p.out_kind = g.dtype == TNB200_BF16 ? 0 : (g.dtype == TNB200_F16 ? 1 : 2);
  p.C = g.C; p.c_sm = g.c_sm; p.c_sb = g.c_sb; p.c_cs = g.swapped ? g.c_sn : 1;
  if (g.swapped && p.c_cs == 1) p.c_cs = 2;   // degenerate (M == 1): force the transposed-store path; stride unused
  p.vec_ok = !g.swapped && (((uintptr_t)g.C) % 16 == 0) && ((g.c_sm * es) % 16 == 0) && ((g.c_sb * es) % 16 == 0);
  bool a_mn = false, b_mn = false;
  int rc = encode_operand(&o.tmA, g.dtype, g.A, g.M, g.K, g.batch, kBM, a_mn, p.a_fe, p.a_ke);
  if (rc) return rc;
  // chain: each CTA of a pair loads half of the B tile (a K-major box of BN / 2 rows)
  rc = encode_operand(&o.tmB, g.dtype, g.B, g.N, g.K, g.batch, chain_mode ? BN / 2 : BN, b_mn, p.b_fe, p.b_ke);
  if (rc) return rc;
  p.a_mn = a_mn; p.b_mn = b_mn;
  o.stage_bytes = stage_bytes_of(g.dtype, BN, a_mn, b_mn);
  int stages = kRingBudget / o.stage_bytes;
  if (stages > 8) stages = 8;
  if (stages > p.num_kb + 1 && p.num_tiles <= sms) stages = p.num_kb + 1 > 2 ? p.num_kb + 1 : 2;
  p.stages = stages;
  return 0;
}

typedef void (*KernelFn)(KernelArgs);
static KernelFn kernel_of(int kind, int BN, bool chain) {
#define TNB_K(K) (chain ? (KernelFn)gemm_wgmma_kernel<K, (K == 2 ? kChainBN32 : kChainBN16), true>        \
                        : (BN == 64 ? (KernelFn)gemm_wgmma_kernel<K, 64, false>                      \
                                    : (BN == 128 ? (KernelFn)gemm_wgmma_kernel<K, 128, false>        \
                                                 : (KernelFn)gemm_wgmma_kernel<K, 256, false>)))
  return kind == 0 ? TNB_K(0) : (kind == 1 ? TNB_K(1) : TNB_K(2));
#undef TNB_K
}
static size_t smem_of(int stages, int stage_bytes) { return (size_t)stages * stage_bytes + 2 * stages * 8 + 1024; }
static int raise_smem(KernelFn fn) {
  cudaError_t e = cudaFuncSetAttribute((const void*)fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) { set_error("wgmma: cannot raise dynamic smem: %s", cudaGetErrorString(e)); return TNB200_ERR_CUDA; }
  return 0;
}

int gemm_wgmma(const GemmProblem& g, cudaStream_t st) {
  if (g.dtype != TNB200_F32 && g.dtype != TNB200_F16 && g.dtype != TNB200_BF16) return TNB200_ERR_UNSUPPORTED;
  if (g.conjA || g.conjB) return TNB200_ERR_UNSUPPORTED;
  if (!g.swapped && g.c_sn != 1 && g.N > 1) return TNB200_ERR_UNSUPPORTED;
  if (g.swapped && g.c_sm != 1 && g.M > 1) return TNB200_ERR_UNSUPPORTED;
  if (g.M >= (1LL << 31) || g.N >= (1LL << 31) || g.K >= (1LL << 31)) return TNB200_ERR_UNSUPPORTED;
  if (!tma_view_ok(g.dtype, g.A, g.M, g.K, g.batch) || !tma_view_ok(g.dtype, g.B, g.N, g.K, g.batch))
    return TNB200_ERR_UNSUPPORTED;
  // swap-AB: a tiny M under a large N would waste the 128-row tile; compute C^T = B^T A^T instead
  // (the big free dimension rides the 128 tile rows, the tiny one a 64-column tile) and let the
  // epilogue store the tile transposed.
  if (g.M <= 64 && g.N >= 128 && !g.swapped) {
    GemmProblem t = g;
    t.swapped = true;
    t.M = g.N; t.N = g.M; t.A = g.B; t.B = g.A;
    t.c_sm = g.c_sn; t.c_sn = g.c_sm;          // row stride of C^T = column stride of C (1)
    return gemm_wgmma(t, st);
  }
  KernelArgs args;
  memset(&args, 0, sizeof(args));
  {
    TcPrep prep;
    int rc = tc_prepare(g, false, prep);
    if (rc) return rc;
    args.tmA = prep.tmA; args.tmB = prep.tmB; args.p = prep.p; args.stage_bytes = prep.stage_bytes;
  }
  const int kind = kind_of(g.dtype);
  KernelFn fn = kernel_of(kind, args.p.BN, false);
  static bool attr_set[3][3] = {};
  const int bi = args.p.BN == 64 ? 0 : (args.p.BN == 128 ? 1 : 2);
  if (!attr_set[kind][bi]) {
    int rc = raise_smem(fn);
    if (rc) return rc;
    attr_set[kind][bi] = true;
  }
  const int64_t sms = num_sms();
  const int64_t grid = args.p.num_tiles < sms ? args.p.num_tiles : sms;
  fn<<<(unsigned)grid, kThreads, smem_of(args.p.stages, args.stage_bytes), st>>>(args);
  TNB_LAUNCH_CHECK();
  count_launch();
  set_kernel_name(kind == 0 ? "wgmma_bf16" : (kind == 1 ? "wgmma_f16" : "wgmma_tf32"));
  return 0;
}

// ------------------------------------------------------------------------------- chain: host side
struct ChainHandle {
  ChainStepDev* d_steps = nullptr;
  ChainSeg* d_segs = nullptr;
  uint32_t* d_done = nullptr;
  KernelArgs args;
  int kind = 0, nsteps = 0;
  size_t smem = 0, done_bytes = 0;
  unsigned grid = 0;
};

// Launch configuration of the chained kernel: 2-CTA clusters along x (the pairs).
struct PairLaunch {
  cudaLaunchAttribute attr;
  cudaLaunchConfig_t cfg;
  PairLaunch(unsigned grid, size_t smem, cudaStream_t st) {
    memset(&attr, 0, sizeof(attr));
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cfg.attrs = &attr; cfg.numAttrs = 1;
  }
  PairLaunch(const PairLaunch&) = delete;
};

int gemm_chain_create(int nsteps, const GemmProblem* probs, const int* dep_a, const int* dep_b, int* first_unsupported,
                      void** handle) {
  *handle = nullptr;
  if (nsteps < 1) return TNB200_ERR_INVALID;
  // A step the kernel cannot take is named in *first_unsupported, so that the caller can split the run around it.
  // Rejections of the chain as a whole (too few tiles, shared memory) leave it at -1.
  auto reject = [&](int i, int rc) { if (first_unsupported) *first_unsupported = i; return rc; };
  // every step runs in the shared kernel's tiles (M and N of at least 128) over the same samples and dtype
  for (int i = 0; i < nsteps; ++i) {
    const GemmProblem& g = probs[i];
    if (g.M < 128 || g.N < 128 || g.batch != probs[0].batch || g.dtype != probs[0].dtype)
      return reject(i, TNB200_ERR_UNSUPPORTED);
  }
  const int dtype = probs[0].dtype;
  const int64_t batch = probs[0].batch;
  std::vector<ChainStepDev> steps(nsteps);
  int max_stage = 0;
  std::vector<int64_t> step_bytes(nsteps), out_bytes(nsteps);   // per sample: operands + result, result
  for (int i = 0; i < nsteps; ++i) {
    const GemmProblem& g = probs[i];
    if (g.conjA || g.conjB || g.swapped) return reject(i, TNB200_ERR_UNSUPPORTED);
    if (g.dtype != TNB200_F32 && g.dtype != TNB200_F16 && g.dtype != TNB200_BF16) return reject(i, TNB200_ERR_UNSUPPORTED);
    if (g.c_sn != 1 || g.M >= (1LL << 31) || g.N >= (1LL << 31) || g.K >= (1LL << 31)) return reject(i, TNB200_ERR_UNSUPPORTED);
    if (dep_a[i] >= i || dep_b[i] >= i) return TNB200_ERR_INVALID;
    TcPrep prep;
    int rc = tc_prepare(g, true, prep);
    if (rc) return reject(i, rc);
    ChainStepDev& sd = steps[i];
    memset(&sd, 0, sizeof(sd));
    rc = encode_output(&sd.tmC, g);
    if (rc) return reject(i, rc);
    sd.tmA = prep.tmA; sd.tmB = prep.tmB; sd.p = prep.p;
    sd.dep_a = dep_a[i]; sd.dep_b = dep_b[i];
    sd.tiles_per_sample = (int)(prep.p.tiles_m * prep.p.tiles_n);
    if (prep.stage_bytes > max_stage) max_stage = prep.stage_bytes;
    step_bytes[i] = (g.M * g.K + g.N * g.K + g.M * g.N) * es_of(dtype);
    out_bytes[i] = g.M * g.N * es_of(dtype);
  }
  for (int i = 0; i < nsteps; ++i) {
    if (steps[i].dep_a >= 0) steps[i].need_a = (uint32_t)steps[steps[i].dep_a].tiles_per_sample;
    if (steps[i].dep_b >= 0) steps[i].need_b = (uint32_t)steps[steps[i].dep_b].tiles_per_sample;
  }
  const int kind = kind_of(dtype);
  KernelFn fn = kernel_of(kind, 0, true);
  {
    static bool attr_set[3] = {};
    if (!attr_set[kind]) {
      int rc = raise_smem(fn);
      if (rc) return rc;
      attr_set[kind] = true;
    }
  }
  // the ring gets what the 227 KB of shared memory leave beside the epilogue staging and the barriers
  const int staging = 2 * kChainStageHalf;
  int stages = (227 * 1024 - 1024 - staging - 256) / max_stage;
  if (stages > 8) stages = 8;
  if (stages < 2) return TNB200_ERR_UNSUPPORTED;
  const size_t smem = smem_of(stages, max_stage) + staging + 4 * 8;
  // every cluster of the launch must be resident (pairs wait on earlier pairs): ask the runtime how many fit
  int clusters = 0;
  {
    PairLaunch pl(2 * num_sms(), smem, nullptr);
    if (cudaOccupancyMaxActiveClusters(&clusters, (void*)fn, &pl.cfg) != cudaSuccess) {
      cudaGetLastError();
      clusters = 0;
    }
  }
  if (clusters < 1) return TNB200_ERR_UNSUPPORTED;
  // pairs per sample of each step: N tiles x M tile pairs
  std::vector<int> pps(nsteps);
  for (int i = 0; i < nsteps; ++i) pps[i] = (int)(steps[i].p.tiles_n * ((steps[i].p.tiles_m + 1) / 2));
  // ---- pair sequence.  The batch is cut into rounds of about G samples and every round is carried through ALL
  // steps, in step order, before the next one starts, so a step's results are consumed soon after they are produced.
  // G follows from the dependencies.  A round must be wide enough that the segment of a step starts at least one
  // full wave of pairs after the segment of each step it reads: in a run that is the segment just before it, in a
  // group of independent runs (the heads of the four MPS ramps) it lies several segments back.  And a round should
  // be as wide as the L2 allows: per sample it keeps live the results that a later step of the round has yet to read,
  // besides the operands and result of the step that runs.  In a run the only such result is the running step's
  // operand, so the bound is the largest step alone.
  auto env_int = [](const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; };
  int min_pps = pps[0];
  for (int i = 1; i < nsteps; ++i) if (pps[i] < min_pps) min_pps = pps[i];
  if (batch * min_pps < clusters && !env_int("TNB200_CHAIN_FORCE", 0))
    return TNB200_ERR_UNSUPPORTED;  // too few pairs per step to hide the producer->consumer latency: go step by step
  int l2 = 0;
  {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) != cudaSuccess) {
      cudaGetLastError();
      l2 = 0;
    }
  }
  int g_wave = 1;
  std::vector<int> last_reader(nsteps, -1);
  for (int i = 0; i < nsteps; ++i) {
    for (const int d : {dep_a[i], dep_b[i]}) {
      if (d < 0) continue;
      last_reader[d] = i;
      int64_t gap = 0;                // pairs per sample from the start of step d's segment to the start of step i's
      for (int j = d; j < i; ++j) gap += pps[j];
      const int g = (int)((clusters + gap - 1) / gap);
      if (g > g_wave) g_wave = g;
    }
  }
  int64_t live_bytes = 0;
  for (int i = 0; i < nsteps; ++i) {
    int64_t live = step_bytes[i];
    for (int j = 0; j < i; ++j)
      if (last_reader[j] > i && dep_a[i] != j && dep_b[i] != j) live += out_bytes[j];
    if (live > live_bytes) live_bytes = live;
  }
  const int g_l2 = (int)(l2 / live_bytes);
  int G = env_int("TNB200_CHAIN_G", g_wave > g_l2 ? g_wave : g_l2);
  if (G < 1) G = 1;
  // balanced rounds: ceil(batch / G) of them, sizes differing by at most one sample
  const int64_t rounds = (batch + G - 1) / G;
  std::vector<ChainSeg> segs;
  long long tile0 = 0;
  for (int64_t r = 0; r < rounds; ++r) {
    const int64_t r0 = batch * r / rounds, r1 = batch * (r + 1) / rounds;
    for (int i = 0; i < nsteps; ++i) {
      ChainSeg sg;
      sg.tile0 = tile0; sg.step = i; sg.sample0 = (int)r0; sg.nsamples = (int)(r1 - r0); sg.pad = 0;
      segs.push_back(sg);
      tile0 += (long long)(r1 - r0) * pps[i];
    }
  }
  ChainHandle* h = new ChainHandle();
  h->kind = kind;
  h->nsteps = nsteps;
  h->done_bytes = sizeof(uint32_t) * (size_t)nsteps * (size_t)batch;
  cudaError_t e = cudaMalloc(&h->d_steps, sizeof(ChainStepDev) * steps.size());
  if (e == cudaSuccess) e = cudaMalloc(&h->d_segs, sizeof(ChainSeg) * segs.size());
  if (e == cudaSuccess) e = cudaMalloc(&h->d_done, h->done_bytes);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_steps, steps.data(), sizeof(ChainStepDev) * steps.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_segs, segs.data(), sizeof(ChainSeg) * segs.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    set_error("chain: device table allocation failed: %s", cudaGetErrorString(e));
    cudaFree(h->d_steps); cudaFree(h->d_segs); cudaFree(h->d_done);
    delete h;
    return TNB200_ERR_CUDA;
  }
  memset(&h->args, 0, sizeof(h->args));
  ChainParams& cp = h->args.cp;
  cp.steps = h->d_steps; cp.segs = h->d_segs; cp.done = h->d_done;
  cp.num_tiles = tile0; cp.nsegs = (int)segs.size(); cp.batch = (int)batch;
  cp.stages = stages; cp.stage_bytes = max_stage;
  h->args.stage_bytes = max_stage;
  h->smem = smem;
  h->grid = (unsigned)(2 * (tile0 < clusters ? tile0 : clusters));
  *handle = h;
  return 0;
}

int gemm_chain_launch(void* handle, cudaStream_t st) {
  ChainHandle* h = (ChainHandle*)handle;
  if (!h) return TNB200_ERR_INVALID;
  TNB_CHECK_CUDA(cudaMemsetAsync(h->d_done, 0, h->done_bytes, st));
  PairLaunch pl(h->grid, h->smem, st);
  TNB_CHECK_CUDA(cudaLaunchKernelEx(&pl.cfg, kernel_of(h->kind, 0, true), h->args));
  count_launch();
  set_kernel_name(h->kind == 2 ? "wgmma_chain_tf32" : "wgmma_chain_16");
  return 0;
}

int gemm_chain_destroy(void* handle) {
  ChainHandle* h = (ChainHandle*)handle;
  if (!h) return 0;
  cudaFree(h->d_steps); cudaFree(h->d_segs); cudaFree(h->d_done);
  delete h;
  return 0;
}

}  // namespace tnb

#ifdef TNB200_CHAIN_PHASES
// Copy the per-CTA phase accumulators ([kPhaseCtas][kPhases] u64) to host memory, then zero them if `reset`.
extern "C" TNB200_API int32_t tnb200_chain_phases(unsigned long long* out, int32_t reset) {
  if (cudaMemcpyFromSymbol(out, tnb::g_chain_phase, sizeof(tnb::g_chain_phase)) != cudaSuccess) return TNB200_ERR_CUDA;
  if (reset) {
    void* p = nullptr;
    if (cudaGetSymbolAddress(&p, tnb::g_chain_phase) != cudaSuccess || cudaMemset(p, 0, sizeof(tnb::g_chain_phase)) != cudaSuccess)
      return TNB200_ERR_CUDA;
  }
  return 0;
}
#endif
