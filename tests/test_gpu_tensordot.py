"""GPU parity: tnb200_tensordot (through the backend class) vs golden vectors of the real
reference and vs the numpy oracle on seeded inputs."""
import numpy as np
import pytest
from conftest import load_golden
from util import assert_close, get_backend, rel_err, TOL
from oracle import np_backend as nb

pytestmark = pytest.mark.gpu


def test_golden_tensordot():
  be = get_backend()
  meta, z = load_golden("tensordot")
  for i, m in enumerate(meta):
    a, b = be.convert_to_tensor(z["a%d" % i]), be.convert_to_tensor(z["b%d" % i])
    if m["perm_a"] is not None:
      a = be.transpose(a, m["perm_a"])
    if m["perm_b"] is not None:
      b = be.transpose(b, m["perm_b"])
    out = be.tensordot(a, b, m["axes"])
    assert out.dtype == z["out%d" % i].dtype
    kern = be.lib.tnb200_last_kernel().decode()
    # float32 on the tensor cores is TF32 (10-bit mantissa): stated tolerance 2e-3
    tol = TOL["tf32"] if kern.startswith("wgmma") else None
    assert_close(out, z["out%d" % i], tol=tol, what="golden tensordot case %d via %s" % (i, kern))


@pytest.mark.parametrize("dtype", ["float64", "float32", "complex128", "complex64", "float16", "int64", "int32"])
@pytest.mark.parametrize("case", [
    ((7, 5, 3), (3, 5, 4), ([1, 2], [1, 0])),
    ((33, 65), (65, 17), ([1], [0])),
    ((4, 3, 2, 5), (5, 2, 6), ([3, 2], [0, 1])),
    ((6,), (6,), ([0], [0])),
    ((3, 4), (5, 6), 0),
    ((100, 70), (70, 90), 1),
])
def test_oracle_random(dtype, case):
  be = get_backend()
  sa, sb, axes = case
  rng = np.random.default_rng(7)

  def mk(shape):
    if dtype.startswith("int"):
      return rng.integers(-4, 5, size=shape).astype(dtype)
    x = rng.standard_normal(shape)
    if dtype.startswith("complex"):
      x = x + 1j * rng.standard_normal(shape)
    return x.astype(dtype)
  a, b = mk(sa), mk(sb)
  ref = nb.tensordot(a.astype("float32") if dtype == "float16" else a,
                     b.astype("float32") if dtype == "float16" else b, axes)
  out = be.tensordot(be.convert_to_tensor(a), be.convert_to_tensor(b), axes)
  assert out.shape == ref.shape
  kern = be.lib.tnb200_last_kernel().decode()
  tol = TOL["tf32"] if (dtype == "float32" and kern.startswith("wgmma")) else None   # fp32 on tensor cores = TF32
  assert_close(out, ref.astype(dtype) if dtype.startswith("int") else ref, dtype=dtype, tol=tol)


def test_strided_views_and_permutes():
  """transposed / sliced views are consumed in place (fused transpose)."""
  be = get_backend()
  rng = np.random.default_rng(8)
  a = rng.standard_normal((6, 10, 8, 4))
  b = rng.standard_normal((8, 12, 10))
  A, B = be.convert_to_tensor(a), be.convert_to_tensor(b)
  av = be.transpose(A, (3, 1, 0, 2))[1:4]       # shape (3, 10, 6, 8), offset view
  bv = be.transpose(B, (2, 0, 1))               # (10, 8, 12)
  ref = np.tensordot(np.transpose(a, (3, 1, 0, 2))[1:4], np.transpose(b, (2, 0, 1)), ([1, 3], [0, 1]))
  assert_close(be.tensordot(av, bv, ([1, 3], [0, 1])), ref)


def test_batched_matmul():
  """ncon_interface_test.py:472-490 shapes: (10,11,100) x (11,100,12) style batch."""
  be = get_backend()
  rng = np.random.default_rng(9)
  a = rng.standard_normal((5, 7, 11))
  b = rng.standard_normal((5, 11, 3))
  assert_close(be.matmul(be.convert_to_tensor(a), be.convert_to_tensor(b)), np.matmul(a, b))
  a4 = rng.standard_normal((2, 3, 4, 6))
  b4 = rng.standard_normal((2, 3, 6, 5))
  assert_close(be.matmul(be.convert_to_tensor(a4), be.convert_to_tensor(b4)), np.matmul(a4, b4))
  with pytest.raises(ValueError):
    be.matmul(be.convert_to_tensor(rng.standard_normal(3)), be.convert_to_tensor(rng.standard_normal(3)))


def test_errors_match_reference():
  be = get_backend()
  a = be.convert_to_tensor(np.ones((2, 3)))
  b = be.convert_to_tensor(np.ones((4, 5)))
  with pytest.raises(ValueError):
    be.tensordot(a, b, ([1], [0]))
  with pytest.raises(TypeError):
    be.tensordot(np.ones((2, 3)), b, 0)
  with pytest.raises(TypeError):
    be.convert_to_tensor([1, 2, 3])


def test_empty_and_scalar_results():
  be = get_backend()
  a = be.convert_to_tensor(np.zeros((0, 4)))
  b = be.convert_to_tensor(np.ones((4, 3)))
  assert be.tensordot(a, b, ([1], [0])).shape == (0, 3)
  # numpy_backend_test.py:12-28: ones(2,3,4) . ones(2,3,4) over all axes -> 24.0
  x = be.convert_to_tensor(2 * np.ones((2, 3, 4)))
  y = be.convert_to_tensor(np.ones((2, 3, 4)))
  out = be.tensordot(x, y, ((1, 2), (1, 2)))
  np.testing.assert_allclose(out.to_host(), np.full((2, 2), 24.0))
  full = be.tensordot(x, y, ((0, 1, 2), (0, 1, 2)))
  assert full.shape == () and full.item() == 48.0
  k0 = be.tensordot(be.convert_to_tensor(np.ones((3, 0))), be.convert_to_tensor(np.ones((0, 2))), 1)
  np.testing.assert_array_equal(k0.to_host(), np.zeros((3, 2)))


@pytest.mark.parametrize("dtype,tolkey", [("float64", "float64"), ("float32", "tf32")])
@pytest.mark.parametrize("axes", [([2], [0]), ([0], [2]), ([2], [2]), ([0], [0])])
def test_flagship_two_site_shapes(dtype, tolkey, axes):
  """SURVEY 8(d) flagship: A,B (512,2,512) over the shared bond, 4 axis variants, full size."""
  be = get_backend()
  rng = np.random.default_rng(2)
  a = (rng.standard_normal((512, 2, 512)) / np.sqrt(512)).astype(dtype)
  b = (rng.standard_normal((512, 2, 512)) / np.sqrt(512)).astype(dtype)
  out = be.tensordot(be.convert_to_tensor(a), be.convert_to_tensor(b), axes)
  ref = np.tensordot(a.astype("float64"), b.astype("float64"), axes)
  assert_close(out, ref, tol=TOL[tolkey], what="flagship %s %s" % (dtype, axes))


def test_strict_fp32_mode_is_true_fp32():
  """TNB200_MATH_STRICT: float32 never drops to TF32 (CUDA-core fp32 FMA kernel), tol 2e-5."""
  from tensornetwork_b200 import _lib as L
  be = get_backend()
  rng = np.random.default_rng(5)
  a = rng.standard_normal((256, 2, 256)).astype(np.float32)
  b = rng.standard_normal((256, 2, 256)).astype(np.float32)
  old = be.math_mode
  try:
    be.math_mode = L.MATH_STRICT
    out = be.tensordot(be.convert_to_tensor(a), be.convert_to_tensor(b), ([2], [0]))
    assert be.lib.tnb200_last_kernel().decode() == "simt"
  finally:
    be.math_mode = old
  assert_close(out, np.tensordot(a.astype(np.float64), b.astype(np.float64), ([2], [0])), tol=2e-5)


def test_skinny_long_k_uses_split_k():
  """(M, N tiny; K huge) — the closing step of the cfg-2 greedy path is (2 x 262144) . (262144 x 2)."""
  be = get_backend()
  rng = np.random.default_rng(6)
  for dtype, tol in (("float64", 1e-10), ("float32", 2e-5)):
    a = rng.standard_normal((2, 262144)).astype(dtype)
    b = rng.standard_normal((262144, 2)).astype(dtype)
    out = be.tensordot(be.convert_to_tensor(a), be.convert_to_tensor(b), 1)
    assert be.lib.tnb200_last_kernel().decode() == "skinny_dot"
    assert_close(out, a.astype(np.float64) @ b.astype(np.float64), tol=tol)
  x = rng.standard_normal((3, 5, 40000))
  y = rng.standard_normal((40000, 5, 7))
  assert_close(be.tensordot(be.convert_to_tensor(x), be.convert_to_tensor(y), ([2, 1], [0, 1])),
               np.tensordot(x, y, ([2, 1], [0, 1])), tol=1e-10)


@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_skinny_outer_family(dtype):
  """one side tiny + short K, other side long (cfg-2 ramp-up steps), incl. many-leg operands and batch."""
  be = get_backend()
  rng = np.random.default_rng(7)
  tol = 1e-10 if dtype == "float64" else 2e-5
  a = rng.standard_normal((2, 2, 4)).astype(dtype)
  b = rng.standard_normal((4, 2, 2, 2, 2, 2, 64, 2, 2)).astype(dtype)
  out = be.tensordot(be.convert_to_tensor(a), be.convert_to_tensor(b), ([2], [0]))
  assert be.lib.tnb200_last_kernel().decode() == "skinny_outer"
  assert_close(out, np.tensordot(a.astype(np.float64), b.astype(np.float64), ([2], [0])), tol=tol)
  # mirrored: the long operand first, contracted over an inner axis of both
  c = rng.standard_normal((2, 2, 2, 2, 512, 2, 2)).astype(dtype)
  d = rng.standard_normal((2, 2)).astype(dtype)
  out = be.tensordot(be.convert_to_tensor(c), be.convert_to_tensor(d), ([0], [0]))
  assert be.lib.tnb200_last_kernel().decode() == "skinny_outer"
  assert_close(out, np.tensordot(c.astype(np.float64), d.astype(np.float64), ([0], [0])), tol=tol)
  # batched + transposed view of the long operand
  A = rng.standard_normal((5, 3, 6)).astype(dtype)
  B = rng.standard_normal((5, 2048, 6)).astype(dtype)
  out = be._contract(be.convert_to_tensor(A), be.convert_to_tensor(B), [2], [2], [0], [0])
  assert be.lib.tnb200_last_kernel().decode() == "skinny_outer"
  assert_close(out, np.einsum("bmk,bnk->bmn", A.astype(np.float64), B.astype(np.float64)), tol=tol)


@pytest.mark.parametrize("shape_a,shape_b,axes", [
    ((16, 16, 64, 16, 16), (16, 16, 48, 16, 16), ([0, 1, 3, 4], [0, 1, 3, 4])),     # 64 x 48 output over K = 65536
    ((40000, 24), (40000, 8), ([0], [0])),                                          # tall operands, tiny output
    ((3, 20, 9000), (3, 9000, 12), None),                                           # batched matmul with long K
    ((32768, 96), (32768, 160), ([0], [0])),                                        # 96 x 160 output: two DMMA tiles, K cut into slices
])
def test_fp64_split_k(shape_a, shape_b, axes):
  """fp64, a small output under a long contraction: K is cut into slices whose partial products are summed in slice order by a
  second kernel (deterministic) — the SIMT split-K kernel for outputs up to 64 x 64, the DMMA kernel with split-K above;
  result against numpy at 1e-12; the DMMA path bit-identical between two runs."""
  be = get_backend()
  rng = np.random.default_rng(12)
  a, b = rng.standard_normal(shape_a), rng.standard_normal(shape_b)
  A, B = be.convert_to_tensor(a), be.convert_to_tensor(b)
  if axes is None:
    got1, got2, ref = be.matmul(A, B).to_host(), be.matmul(A, B).to_host(), np.matmul(a, b)
  else:
    got1, got2 = be.tensordot(A, B, axes).to_host(), be.tensordot(A, B, axes).to_host()
    ref = np.tensordot(a, b, axes)
  kern = be.lib.tnb200_last_kernel().decode()
  assert kern == ("dmma_f64_splitk" if min(ref.shape[-2:]) > 64 else "simt_splitk"), kern
  assert rel_err(got1, ref) < 1e-12 and rel_err(got2, ref) < 1e-12
  if kern == "dmma_f64_splitk":                 # (the SIMT split-K kernel accumulates its slices with atomics)
    np.testing.assert_array_equal(got1, got2)
