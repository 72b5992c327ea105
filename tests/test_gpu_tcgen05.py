"""GPU parity of the wgmma/TMA tensor-core path (bf16 / f16 / tf32) against float64 numpy on
identically rounded inputs.  Tolerances: bf16 4e-3 (output rounding 2^-9), f16 1e-3, tf32 1e-3
(10-bit mantissa inputs, fp32 accumulate), all relative Frobenius."""
import numpy as np
import pytest
from util import assert_close, get_backend, rel_err

pytestmark = pytest.mark.gpu
TOLS = {"bfloat16": 4e-3, "float16": 1e-3, "float32": 1e-3}


def _mk(be, rng, shape, dtype):
  x = rng.standard_normal(shape).astype(np.float32)
  if dtype == "float32":
    t = be.convert_to_tensor(x)
  else:
    t = be.astype(be.convert_to_tensor(x), dtype)
  return t, t.to_host().astype(np.float64)


@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32"])
@pytest.mark.parametrize("axes", [([2], [0]), ([0], [2]), ([2], [2]), ([0], [0]), ([0, 1], [0, 1]), ([1, 2], [1, 2])])
def test_two_site_all_majors(dtype, axes):
  """A,B (256,2,256): every combination of K-major / MN-major operands (fused transposes)."""
  be = get_backend()
  rng = np.random.default_rng(21)
  A, a = _mk(be, rng, (256, 2, 256), dtype)
  B, b = _mk(be, rng, (256, 2, 256), dtype)
  out = be.tensordot(A, B, axes)
  kern = be.lib.tnb200_last_kernel().decode()
  assert kern.startswith("wgmma"), kern
  ref = np.tensordot(a, b, axes)
  e = rel_err(out.to_host(), ref)
  assert e < TOLS[dtype], "%s %s via %s: %.3e" % (dtype, axes, kern, e)


@pytest.mark.parametrize("dtype", ["bfloat16", "float32"])
@pytest.mark.parametrize("mkn", [(128, 64, 64), (130, 72, 136), (1000, 520, 264), (64, 1024, 8), (8, 64, 520),
                                 (512, 512, 1024), (2048, 40, 2048), (136, 8, 72)])
def test_ragged_sizes(dtype, mkn):
  be = get_backend()
  rng = np.random.default_rng(22)
  m, k, n = mkn
  A, a = _mk(be, rng, (m, k), dtype)
  B, b = _mk(be, rng, (k, n), dtype)
  out = be.tensordot(A, B, 1)
  kern = be.lib.tnb200_last_kernel().decode()
  assert rel_err(out.to_host(), a @ b) < TOLS[dtype], (kern, mkn)
  # transposed operands: (k,m)^T x (n,k)^T
  At, at = _mk(be, rng, (k, m), dtype)
  Bt, bt = _mk(be, rng, (n, k), dtype)
  out2 = be.tensordot(be.transpose(At), be.transpose(Bt), 1)
  assert rel_err(out2.to_host(), at.T @ bt.T) < TOLS[dtype], (be.lib.tnb200_last_kernel().decode(), mkn)


@pytest.mark.parametrize("dtype", ["bfloat16", "float32"])
def test_batched(dtype):
  be = get_backend()
  rng = np.random.default_rng(23)
  A, a = _mk(be, rng, (6, 256, 128), dtype)
  B, b = _mk(be, rng, (6, 128, 192), dtype)
  out = be.matmul(A, B)
  assert be.lib.tnb200_last_kernel().decode().startswith("wgmma")
  assert rel_err(out.to_host(), np.matmul(a, b)) < TOLS[dtype]


# (dtype, shape of A, slice of A, shape of B, contracted axes, transposed output, kernel, launches including repacks)
REPACK_CASES = {
    # odd leading dimension -> not addressable in place -> one strided-copy repack, then the tensor-core GEMM
    "a_packed": ("bfloat16", (256, 131), None, (131, 256), ([1], [0]), False, "wgmma_bf16", 2),
    "b_packed": ("bfloat16", (256, 128), None, (128, 131), ([1], [0]), False, "wgmma_bf16", 2),
    "both_packed": ("bfloat16", (256, 131), None, (131, 260), ([1], [0]), False, "wgmma_bf16", 3),
    # A keeps two K modes in place (the slice breaks mergeability); the packed B walks K in the same two modes
    "k_split": ("bfloat16", (256, 2, 128), np.s_[:, :, :64], (2, 64, 129), ([1, 2], [0, 1]), False, "wgmma_bf16", 2),
    # DMMA addresses only one mode per group: a two-mode free group is repacked, a two-mode K group repacks both
    "f64_free_modes": ("float64", (4, 64, 128), np.s_[:, :32, :], (128, 128), ([2], [0]), False, "dmma_f64", 2),
    "f64_k_modes": ("float64", (128, 4, 64), np.s_[:, :, :32], (4, 32, 128), ([1, 2], [0, 1]), False, "dmma_f64", 3),
    # the GEMM rejects a column-strided C after A was repacked: B is repacked too (A's copy is reused), then SIMT
    "rejected_retry": ("bfloat16", (256, 131), None, (131, 256), ([1], [0]), True, "simt", 3),
}


def test_unaligned_operand_falls_back_to_repack():
  """operands the GEMM cannot address in place are repacked; the kernel, the launch count and the result are pinned."""
  be = get_backend()
  for case, (dtype, sa, sl, sb, axes, c_transposed, kern, launches) in REPACK_CASES.items():
    rng = np.random.default_rng(24)
    A, a = _mk(be, rng, sa, dtype)
    B, b = _mk(be, rng, sb, dtype)
    if sl is not None:
      A, a = A[sl], a[sl]
    ref = np.tensordot(a, b, axes)
    out = None
    if c_transposed:
      out = be.transpose(be._new(ref.shape[::-1], A.code))  # pylint: disable=protected-access
    l0 = _launches(be)
    out = be._contract(A, B, axes[0], axes[1], [], [], out=out)  # pylint: disable=protected-access
    assert (be.lib.tnb200_last_kernel().decode(), _launches(be) - l0) == (kern, launches), case
    assert rel_err(out.to_host(), ref) < TOLS.get(dtype, 1e-12), case


def test_linearity_at_flagship_size():
  """size-independent property at the flagship shape: T(a1 + a2, b) == T(a1, b) + T(a2, b)."""
  be = get_backend()
  rng = np.random.default_rng(25)
  A1, a1 = _mk(be, rng, (512, 2, 512), "float32")
  A2, a2 = _mk(be, rng, (512, 2, 512), "float32")
  B, b = _mk(be, rng, (512, 2, 512), "float32")
  lhs = be.tensordot(be.addition(A1, A2), B, ([2], [0]))
  rhs = be.addition(be.tensordot(A1, B, ([2], [0])), be.tensordot(A2, B, ([2], [0])))
  assert rel_err(lhs.to_host(), rhs.to_host()) < 2e-3


def _launches(be):
  return be.lib.tnb200_launch_count()


@pytest.mark.parametrize("dtype", ["bfloat16", "float32"])
def test_multimode_operands_are_fused_not_repacked(dtype):
  """Operands whose free / contracted group is two non-mergeable modes are addressed in place by
  rank-5 TMA maps: exactly ONE kernel launch (no strided-copy repack), results within tolerance."""
  be = get_backend()
  rng = np.random.default_rng(26)
  # (b) of the cfg-2 zipper: A(512,2,512) x T(2,512,512) over A axes (0,1) <-> T axes (2,0)
  A, a = _mk(be, rng, (512, 2, 512), dtype)
  Tt, t = _mk(be, rng, (2, 512, 512), dtype)
  l0 = _launches(be)
  out = be.tensordot(A, Tt, ([0, 1], [2, 0]))
  assert _launches(be) - l0 == 1, "repacked: %d launches" % (_launches(be) - l0)
  assert be.lib.tnb200_last_kernel().decode().startswith("wgmma")
  assert rel_err(out.to_host(), np.tensordot(a, t, ([0, 1], [2, 0]))) < TOLS[dtype]
  # free group = two modes around the contracted physical leg (MN-major, inner extent % 64 == 0)
  X, x = _mk(be, rng, (256, 4, 128), dtype)
  Y, y = _mk(be, rng, (4, 192), dtype)
  l0 = _launches(be)
  out = be.tensordot(X, Y, ([1], [0]))
  assert _launches(be) - l0 == 1
  assert rel_err(out.to_host(), np.tensordot(x, y, ([1], [0]))) < TOLS[dtype]
  # K-major operand with two free modes (a slice breaks mergeability), power-of-two inner extent
  Z, z = _mk(be, rng, (8, 64, 256), dtype)
  Zs = Z[:, :32, :]
  W, w = _mk(be, rng, (256, 64), dtype)
  l0 = _launches(be)
  out = be.tensordot(Zs, W, ([2], [0]))
  assert _launches(be) - l0 == 1
  assert rel_err(out.to_host(), np.tensordot(z[:, :32, :], w, ([2], [0]))) < TOLS[dtype]
  # batched + multi-mode
  Ab, ab = _mk(be, rng, (3, 256, 2, 128), dtype)
  Bb, bb = _mk(be, rng, (3, 2, 64, 256), dtype)
  out = be._contract(Ab, Bb, [1, 2], [3, 1], [0], [0])
  ref = np.einsum("bimk,bmji->bkj", ab, bb)
  assert rel_err(out.to_host(), ref) < TOLS[dtype]


@pytest.mark.parametrize("dtype", ["bfloat16", "float32"])
def test_swap_ab_tiny_m(dtype):
  """tiny M under a huge N (the ramp-up steps of the cfg-2 path): computed as C^T tiles, stored transposed."""
  be = get_backend()
  rng = np.random.default_rng(27)
  for (m, k, n) in [(4, 4, 4096), (8, 8, 2048), (16, 16, 1024), (33, 40, 640), (64, 64, 512), (1, 128, 256), (2, 512, 128)]:
    A, a = _mk(be, rng, (m, k), dtype)
    B, b = _mk(be, rng, (k, n), dtype)
    out = be.tensordot(A, B, 1)
    kern = be.lib.tnb200_last_kernel().decode()     # short K + tiny M streams through the CUDA-core kernel
    assert kern.startswith("wgmma") or kern == "skinny_outer", (m, k, n, kern)
    assert rel_err(out.to_host(), a @ b) < TOLS[dtype], (m, k, n)
    Bt, bt = _mk(be, rng, (n, k), dtype)          # K-major big operand
    out = be.tensordot(A, be.transpose(Bt), 1)
    assert rel_err(out.to_host(), a @ bt.T) < TOLS[dtype], (m, k, n)
  # batched ramp-up step with many small legs: (nb, 4, 2, 2) . (nb, 2, 4, 2, 2, 2, 64, 2, 2) over A[1] <-> B[2]... cfg-2 style
  Ab, ab = _mk(be, rng, (3, 8, 2, 4), dtype)
  Bb, bb = _mk(be, rng, (3, 2, 8, 2, 2, 2, 2, 64, 2, 2), dtype)
  out = be._contract(Ab, Bb, [1], [2], [0], [0])
  ref = np.einsum("bkpq,bxkcdefghi->bpqxcdefghi", ab, bb)
  assert rel_err(out.to_host(), ref) < TOLS[dtype]


def test_chain_names_first_step_below_its_tile():
  """The chained kernel takes steps of at least 128 x 128: create() reports the first smaller step and makes no handle."""
  import ctypes
  from tensornetwork_b200 import _lib as L
  be = get_backend()
  rng = np.random.default_rng(28)
  A0, _ = _mk(be, rng, (256, 256), "bfloat16")
  B0, _ = _mk(be, rng, (256, 256), "bfloat16")
  A1, _ = _mk(be, rng, (64, 256), "bfloat16")
  A2, _ = _mk(be, rng, (128, 64), "bfloat16")
  C0, C1, C2 = (be._new(s, L.BF16) for s in ((256, 256), (64, 256), (128, 256)))  # pylint: disable=protected-access
  # C0 = A0 B0, C1 = A1 C0 (M = 64), C2 = A2 C1: every step is addressable in place, only step 1 is below the tile
  steps = [(A0, B0, C0, -1), (A1, C0, C1, 0), (A2, C1, C2, 1)]
  arr = (L.ChainStep * len(steps))()
  for cs, (a, b, c, dep_b) in zip(arr, steps):
    cs.a, cs.b, cs.c = a.desc(), b.desc(), c.desc()
    cs.naxes, cs.nbatch = 1, 0
    cs.axes_a[0], cs.axes_b[0] = 1, 0
    cs.dep_a, cs.dep_b = -1, dep_b
  bad, handle = ctypes.c_int32(-1), ctypes.c_void_p()
  rc = be.lib.tnb200_chain_create(len(steps), arr, ctypes.byref(bad), ctypes.byref(handle))
  assert (rc, bad.value, handle.value) == (L.ERR_UNSUPPORTED, 1, None)


# ------------------------------------------------------------------------------------------------
# thin contractions (tensordot_thin.cu): small matrix x long tensor, the ramp-up steps of the cfg-2 path
@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32", "float64"])
@pytest.mark.parametrize("kp", [(2, 2), (4, 4), (8, 8), (4, 8), (8, 2), (3, 5)])
def test_thin_simt_both_layouts(dtype, kp):
  be = get_backend()
  rng = np.random.default_rng(31)
  k, p = kp
  nb, L = 3, 32768
  tol = {"float32": 2e-5, "float64": 1e-12}.get(dtype) or TOLS[dtype]
  # mode A: S[b, p1, 2, k] . X[b, k, (2, 2, L/4)] -> C[b, p1, 2, 2, 2, L/4]  (many-leg operands, merged by the planner)
  if p % 2 == 0:
    S, s = _mk(be, rng, (nb, p // 2, 2, k), dtype)
    X, x = _mk(be, rng, (nb, k, 2, 2, L // 4), dtype)
    out = be._contract(S, X, [3], [1], [0], [0])
    assert be.lib.tnb200_last_kernel().decode() == "thin_simt_a"
    e = rel_err(out.to_host(), np.einsum("bpqk,bkxyl->bpqxyl", s, x))
    assert e < tol, (dtype, kp, "A", e)
  else:
    S, s = _mk(be, rng, (nb, p, k), dtype)
    X, x = _mk(be, rng, (nb, k, L), dtype)
    out = be._contract(S, X, [2], [1], [0], [0])
    assert be.lib.tnb200_last_kernel().decode() == "thin_simt_a"
    assert rel_err(out.to_host(), np.einsum("bpk,bkl->bpl", s, x)) < tol, (dtype, kp, "A")
  # mode D: X[b, L, k] . S[b, k, p] -> C[b, L, p]   (power-of-two K, P only; others take the generic paths)
  X, x = _mk(be, rng, (nb, L // 2, 2, k), dtype)
  S, s = _mk(be, rng, (nb, k, p), dtype)
  out = be._contract(X, S, [3], [1], [0], [0])
  kern = be.lib.tnb200_last_kernel().decode()
  if k in (2, 4, 8) and p in (2, 4, 8):
    assert kern == "thin_simt_d", kern
  e = rel_err(out.to_host(), np.einsum("bxyk,bkp->bxyp", x, s))
  assert e < tol, (dtype, kp, "D", kern, e)


@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32"])
@pytest.mark.parametrize("kp", [(16, 16), (32, 32), (64, 64), (16, 64), (64, 16), (32, 64), (64, 32), (16, 32), (32, 16)])
def test_thin_mma_both_layouts(dtype, kp):
  be = get_backend()
  rng = np.random.default_rng(32)
  k, p = kp
  nb, L = 5, 16384
  sfx = "_tf32" if dtype == "float32" else ""
  # mode A with a two-leg S (site tensor (p/2, 2, k)) and batch
  S, s = _mk(be, rng, (nb, p // 2, 2, k), dtype)
  X, x = _mk(be, rng, (nb, k, 2, L // 2), dtype)
  out = be._contract(S, X, [3], [1], [0], [0])
  assert be.lib.tnb200_last_kernel().decode() == "thin_mma" + sfx + "_a"
  e = rel_err(out.to_host(), np.einsum("bpqk,bkxl->bpqxl", s, x))
  assert e < TOLS[dtype], (dtype, kp, "A", e)
  # mode D with a two-leg S (site tensor (k, 2, p/2))
  X, x = _mk(be, rng, (nb, L, k), dtype)
  S, s = _mk(be, rng, (nb, k, 2, p // 2), dtype)
  out = be._contract(X, S, [2], [1], [0], [0])
  assert be.lib.tnb200_last_kernel().decode() == "thin_mma" + sfx + "_d"
  e = rel_err(out.to_host(), np.einsum("blk,bkqp->blqp", x, s))
  assert e < TOLS[dtype], (dtype, kp, "D", e)


def test_thin_mma_masked_rows_and_unbatched():
  """P not a multiple of 16 (mode A masks rows), no batch axis, transposed S view."""
  be = get_backend()
  rng = np.random.default_rng(33)
  S, s = _mk(be, rng, (32, 24), "bfloat16")          # stored [k][p]; used as S^T
  X, x = _mk(be, rng, (32, 131072), "bfloat16")
  out = be.tensordot(be.transpose(S), X, 1)
  assert be.lib.tnb200_last_kernel().decode() == "thin_mma_a"
  assert rel_err(out.to_host(), s.T @ x) < TOLS["bfloat16"]


def test_thin_fp32_strict_mode_stays_fp32():
  """TNB200_MATH_STRICT: the thin fp32 shapes must not take the TF32 warp-MMA kernel (true fp32 accuracy 2e-5)."""
  from tensornetwork_b200 import _lib as L
  be = get_backend()
  rng = np.random.default_rng(34)
  S, s = _mk(be, rng, (3, 32, 32), "float32")
  X, x = _mk(be, rng, (3, 32, 32768), "float32")
  old = be.math_mode
  be.math_mode = L.MATH_STRICT
  try:
    out = be._contract(S, X, [2], [1], [0], [0])
    kern = be.lib.tnb200_last_kernel().decode()
  finally:
    be.math_mode = old
  assert "tf32" not in kern and not kern.startswith("wgmma"), kern
  assert rel_err(out.to_host(), np.einsum("bpk,bkl->bpl", s, x)) < 2e-5
