// gemm.cuh — the canonical (batched, strided, multi-mode) GEMM problem the tensordot planner lowers to.
#pragma once
#include "common.cuh"

namespace tnb {

// One operand as a (batch, free modes, contracted modes) view.  Modes are listed outer -> inner
// (row-major linearisation of the group), strides in elements.  A group with one mode is a
// plain matrix dimension; up to two modes per group can be addressed directly by the TMA path.
struct OperandView {
  const void* ptr = nullptr;
  int nF = 0, nK = 0;
  int64_t fe[4] = {1, 1, 1, 1}, fs[4] = {0, 0, 0, 0};
  int64_t ke[4] = {1, 1, 1, 1}, ks[4] = {0, 0, 0, 0};
  int64_t sb = 0;  // batch stride
  bool simple() const { return nF <= 1 && nK <= 1; }
  int64_t f_stride() const { return nF ? fs[nF - 1] : 0; }   // innermost free stride
  int64_t k_stride() const { return nK ? ks[nK - 1] : 0; }   // innermost contracted stride
};

// C[b, m, n] = sum_k A[b, m, k] * B[b, k, n]; C is a 2-stride matrix per batch entry.
struct GemmProblem {
  int dtype = 0;
  int64_t M = 0, N = 0, K = 0, batch = 1;
  OperandView A, B;
  void* C = nullptr; int64_t c_sm = 0, c_sn = 0, c_sb = 0;
  bool conjA = false, conjB = false;
  int math = 0;  // TNB200_MATH_* >> 4
  bool swapped = false;   // internal: operands exchanged by gemm_wgmma (C is written transposed)
};

// Each returns TNB200_ERR_UNSUPPORTED (without setting an error) when the problem does not
// meet the kernel's layout/alignment constraints; the planner then repacks or falls back.
int gemm_wgmma(const GemmProblem& p, cudaStream_t st);     // bf16 / f16 / f32(tf32)
int gemm_dmma_f64(const GemmProblem& p, cudaStream_t st);  // f64 via mma.sync DMMA
// Chained GEMMs in one persistent launch (gemm_wgmma.cu): dep_a[i] / dep_b[i] = index of the chain step whose
// output is step i's operand A / B (or -1).  create() allocates device tables (call it outside stream capture).
// A step the kernel cannot take (below its 128 x 128 tile, another batch or dtype than step 0, a C that is not
// row-major with 16-byte aligned rows, operands its tensor maps cannot address) is reported in *first_unsupported
// (when not null) with TNB200_ERR_UNSUPPORTED; a rejection of the chain as a whole leaves it at -1.
int gemm_chain_create(int nsteps, const GemmProblem* probs, const int* dep_a, const int* dep_b, int* first_unsupported,
                      void** handle);
int gemm_chain_launch(void* handle, cudaStream_t st);
int gemm_chain_destroy(void* handle);
// can the TMA/wgmma path address this operand view in place?  (tile-size independent check)
bool tma_view_ok(int dtype, const OperandView& v, int64_t ext_f, int64_t ext_k, int64_t batch);

}  // namespace tnb
