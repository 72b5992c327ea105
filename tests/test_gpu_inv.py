"""GPU: LU with partial pivoting (tnb200_lu_factor) against scipy.linalg.lu_factor, and CudaB200Backend.inv
(tnb200_inv) against np.linalg.inv.  Pivots are compared exactly; factors and inverses through residuals."""
import numpy as np
import pytest
import scipy.linalg
import torch
from util import get_backend

pytestmark = pytest.mark.gpu

# the largest panel the 8-CTA cluster holds in shared memory is about 6900 rows in f64; this size exceeds it, so its
# first panels run from global memory
ABOVE_CLUSTER_LIMIT = 7000


def _random(rng, shape, dtype):
  x = rng.standard_normal(shape)
  if np.dtype(dtype).kind == "c":
    x = x + 1j * rng.standard_normal(shape)
  return x.astype(dtype)


def _lu_factor(be, a):
  """tnb200_lu_factor through the C ABI -> (lu, piv, info) on the host"""
  from tensornetwork_b200 import _lib as L
  n = a.shape[0]
  lu = be._new((n, n), a.code)
  piv = torch.full((max(n, 1),), -1, dtype=torch.int32, device=be.device)
  info = torch.full((1,), -1, dtype=torch.int32, device=be.device)
  L.check(be.lib.tnb200_lu_factor(a.ref(), lu.ref(), piv.data_ptr(), info.data_ptr(), be._stream()))
  return lu.to_host(), piv.cpu().numpy()[:n], int(info.item())


def _permute(a, piv):
  pa = a.copy()
  for i, p in enumerate(piv):
    pa[[i, p]] = pa[[p, i]]
  return pa


def _check_lu(a, lu, piv):
  n = a.shape[0]
  ref_lu, ref_piv = scipy.linalg.lu_factor(a, check_finite=False)
  np.testing.assert_array_equal(piv, ref_piv)
  l = np.tril(lu, -1) + np.eye(n)
  u = np.triu(lu)
  eps = np.finfo(a.real.dtype).eps
  res = np.linalg.norm(_permute(a, piv) - l @ u) / np.linalg.norm(a)
  assert res <= 50 * n * eps, res
  assert np.linalg.norm(lu - ref_lu) <= 1e3 * n * eps * np.linalg.norm(ref_lu)


@pytest.mark.parametrize("n", [0, 1, 2, 31, 32, 33, 63, 64, 65, 100, 257, 1000, 2048])
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_lu_factor(dtype, n):
  be = get_backend()
  a = _random(np.random.default_rng(n), (n, n), dtype)
  lu, piv, info = _lu_factor(be, be.convert_to_tensor(a))
  assert info == 0 and lu.dtype == np.dtype(dtype)
  if n:
    _check_lu(a, lu, piv)


def test_lu_factor_above_cluster_panel_limit():
  be = get_backend()
  n = ABOVE_CLUSTER_LIMIT
  a = _random(np.random.default_rng(5), (n, n), "float64")
  lu, piv, info = _lu_factor(be, be.convert_to_tensor(a))
  assert info == 0
  _check_lu(a, lu, piv)


def test_lu_factor_c128_above_cluster_panel_limit():
  """c128 panels (16-byte elements) leave shared memory above about 3300 rows"""
  be = get_backend()
  n = 3400
  a = _random(np.random.default_rng(6), (n, n), "complex128")
  lu, piv, info = _lu_factor(be, be.convert_to_tensor(a))
  assert info == 0
  _check_lu(a, lu, piv)


def test_nan_and_inf_input():
  """NaN never makes a pivot index out of range: reference BLAS idamax keeps a NaN on the diagonal as the pivot and never
  picks a NaN below it; the NaNs then run through the factors and the inverse, and nothing raises"""
  be = get_backend()
  rng = np.random.default_rng(12)
  nan_diag = np.array([[np.nan, 1.0], [1.0, 1.0]])              # the second column is NaN after one step
  inf_case = np.array([[np.inf, np.inf], [1.0, 1.0]])           # the same through inf - inf
  mid = np.array([[1.0, 2.0, 3.0], [4.0, np.nan, 6.0], [7.0, 8.0, 10.0]])
  nan_col = rng.standard_normal((300, 300))
  nan_col[:, 40] = np.nan                                       # a whole column of NaN, spread over every CTA
  nan_below = rng.standard_normal((300, 300))
  nan_below[250, 0] = np.nan                                    # a NaN below the diagonal is never the pivot
  for m in (nan_diag, inf_case, mid, nan_col, nan_below):
    n = m.shape[0]
    lu, piv, info = _lu_factor(be, be.convert_to_tensor(m))
    assert np.all(piv >= np.arange(n)) and np.all(piv < n), piv
    assert info == 0
    x = be.inv(be.convert_to_tensor(m)).to_host()
    assert x.shape == (n, n) and np.isnan(x).any()
  assert _lu_factor(be, be.convert_to_tensor(nan_diag))[1][0] == 0
  assert _lu_factor(be, be.convert_to_tensor(nan_below))[1][0] != 250
  np.testing.assert_array_equal(_lu_factor(be, be.convert_to_tensor(mid))[1], [2, 1, 2])
  assert np.isnan(be.inv(be.convert_to_tensor(inf_case)).to_host()).all() and np.isnan(np.linalg.inv(inf_case)).all()
  c = nan_col.astype(np.complex128) * (1 + 1j)
  _, piv, info = _lu_factor(be, be.convert_to_tensor(c))
  assert info == 0 and np.all(piv >= np.arange(300)) and np.all(piv < 300)


def test_complex_pivots_at_the_ends_of_the_double_range():
  """|pivot|^2 is never formed, so a well-conditioned complex matrix scaled by 1e200 or 1e-200 still inverts"""
  be = get_backend()
  a = _random(np.random.default_rng(13), (64, 64), "complex128")
  ref = np.linalg.inv(a)
  for s in (1e200, 1e-200):
    x = be.inv(be.convert_to_tensor(a * s)).to_host()
    assert np.all(np.isfinite(x))
    np.testing.assert_allclose(x * s, ref, rtol=0, atol=1e-10 * np.abs(ref).max())


def test_lu_factor_single_precision_and_strided():
  be = get_backend()
  rng = np.random.default_rng(2)
  for dtype in ("float32", "complex64"):
    a = _random(rng, (300, 300), dtype)
    lu, piv, info = _lu_factor(be, be.convert_to_tensor(a))
    assert info == 0 and lu.dtype == np.dtype(dtype)
    wide = a.astype(np.complex128 if dtype == "complex64" else np.float64)
    l, u = np.tril(lu, -1) + np.eye(300), np.triu(lu)
    assert np.linalg.norm(_permute(wide, piv) - l @ u) / np.linalg.norm(wide) <= 50 * 300 * np.finfo(dtype).eps
  big = _random(rng, (400, 300), "float64")
  view = be.transpose(be.convert_to_tensor(big)[::2, :200])          # a strided, transposed 200 x 200 view
  lu, piv, info = _lu_factor(be, view)
  _check_lu(big[::2, :200].T.copy(), lu, piv)


def test_pivot_ties_take_the_first_index():
  be = get_backend()
  a = np.array([[1.0, 2.0, 0.5, 1.0], [-3.0, 1.0, 2.0, 0.0], [3.0, 0.5, 1.0, 2.0], [2.0, 4.0, -4.0, 1.0]])
  lu, piv, info = _lu_factor(be, be.convert_to_tensor(a))
  assert piv[0] == 1                                   # |-3| == |3|: the first of the two rows
  np.testing.assert_array_equal(piv, scipy.linalg.lu_factor(a)[1])
  ac = np.array([[1.0, 1.0], [1 + 1j, 0.0], [-2.0, 1.0], [0.0, 3.0]])    # |re| + |im|: 2, 2 -> row 1
  c = np.zeros((4, 4), np.complex128)
  c[:, :2] = ac
  c[:, 2:] = np.eye(4)[:, :2] + 0.5
  lu, piv, info = _lu_factor(be, be.convert_to_tensor(c))
  assert piv[0] == 1
  np.testing.assert_array_equal(piv, scipy.linalg.lu_factor(c)[1])


def _inv_case(rng, n, dtype):
  if np.dtype(dtype).kind == "i":
    return (rng.integers(-5, 6, (n, n)) + 20 * np.eye(n, dtype=np.int64)).astype(dtype)
  return _random(rng, (n, n), dtype)


@pytest.mark.parametrize("n", [1, 5, 33, 100, 513])
@pytest.mark.parametrize("dtype", ["float64", "complex128", "float32", "complex64", "int64"])
def test_inv(dtype, n):
  be = get_backend()
  rng = np.random.default_rng(n + 17)
  a = _inv_case(rng, n, dtype)
  x = be.inv(be.convert_to_tensor(a))
  out_dtype = np.float64 if np.dtype(dtype).kind == "i" else np.dtype(dtype)
  assert x.dtype == out_dtype and x.shape == (n, n)
  xh = x.to_host()
  wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
  eps = np.finfo(out_dtype).eps
  aw, xw = a.astype(wide), xh.astype(wide)
  res = np.linalg.norm(aw @ xw - np.eye(n)) / (np.linalg.norm(aw) * np.linalg.norm(xw))
  assert res <= 50 * n * eps, res
  ref = np.linalg.inv(aw)
  assert np.linalg.norm(xw - ref) <= 50 * n * eps * np.linalg.cond(aw) * np.linalg.norm(ref)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_inv_strided_and_transposed_views(dtype):
  be = get_backend()
  rng = np.random.default_rng(4)
  big = _random(rng, (260, 390), dtype)
  base = be.convert_to_tensor(big)
  for view, host in ((base[::2, 1:261:2], big[::2, 1:261:2]), (be.transpose(base[:, :260]), big[:, :260].T)):
    x = be.inv(view)
    n = host.shape[0]
    res = np.linalg.norm(host @ x.to_host() - np.eye(n)) / (np.linalg.norm(host) * np.linalg.norm(x.to_host()))
    assert res <= 50 * n * np.finfo(dtype).eps, res
  out = be.transpose(be._new((130, 130), base.code))                  # a preallocated, transposed output
  from tensornetwork_b200 import _lib as L
  info = torch.zeros(1, dtype=torch.int32, device=be.device)
  L.check(be.lib.tnb200_inv(base[::2, 1:261:2].ref(), out.ref(), info.data_ptr(), be._stream()))
  assert int(info.item()) == 0
  np.testing.assert_allclose(out.to_host(), np.linalg.inv(big[::2, 1:261:2]), rtol=0,
                             atol=1e-9 * np.abs(np.linalg.inv(big[::2, 1:261:2])).max())


def test_singular_input_raises():
  be = get_backend()
  rng = np.random.default_rng(8)
  zero = np.zeros((6, 6))
  zcol = rng.standard_normal((50, 50))
  zcol[:, 17] = 0.0
  same = np.array([[1.0, 2.0, 3.0, 1.0], [4.0, 5.0, 6.0, 2.0], [2.0, 0.0, 1.0, 1.0], [4.0, 5.0, 6.0, 2.0]])
  # (rows 1 and 3 agree and every step of the elimination is exact, so a pivot is exactly zero; larger random rows
  # can leave a pivot of rounding size instead, and then neither numpy nor LAPACK reports a singular matrix)
  for m in (zero, zcol, same):
    with pytest.raises(np.linalg.LinAlgError):
      np.linalg.inv(m)
    with pytest.raises(np.linalg.LinAlgError, match="Singular"):
      be.inv(be.convert_to_tensor(m))
  _, _, info = _lu_factor(be, be.convert_to_tensor(zcol))
  assert info == 18                                    # 1 + the first zero pivot, LAPACK's info
  assert info == scipy.linalg.lapack.dgetrf(zcol)[2]


def test_errors():
  be = get_backend()
  with pytest.raises(ValueError):
    be.inv(be.convert_to_tensor(np.ones((2, 2, 2))))
  with pytest.raises(np.linalg.LinAlgError):
    be.inv(be.convert_to_tensor(np.ones(3)))
  with pytest.raises(np.linalg.LinAlgError):
    be.inv(be.convert_to_tensor(np.ones((2, 3))))
  with pytest.raises(TypeError):
    be.inv(be.convert_to_tensor(np.eye(3, dtype=np.float16)))
  with pytest.raises(TypeError):
    be.inv(be.astype(be.convert_to_tensor(np.eye(3)), "bfloat16"))
  with pytest.raises(ValueError):
    _lu_factor(be, be.convert_to_tensor(np.ones((2, 3))))
  with pytest.raises(TypeError):
    _lu_factor(be, be.convert_to_tensor(np.eye(3, dtype=np.int64)))
  assert be.inv(be.convert_to_tensor(np.zeros((0, 0)))).shape == (0, 0)


def test_jit_falls_back_to_eager():
  be = get_backend()
  a = _random(np.random.default_rng(6), (64, 64), "float64")
  ad = be.convert_to_tensor(a)
  f = be.jit(lambda x: be.inv(x), static_argnums=())
  fails0 = be.jit_stats["capture_failures"]
  for _ in range(3):
    np.testing.assert_allclose(f(ad).to_host(), np.linalg.inv(a), rtol=0, atol=1e-10 * np.abs(np.linalg.inv(a)).max())
  assert be.jit_stats["capture_failures"] - fails0 == 1


def test_launch_count_scales_with_panels():
  """one n = 2048 f64 inversion: at most 8 ceil(n / 32) + 8 launches (four per panel for the factorisation, two per
  32-row step of each substitution), not O(n)"""
  be = get_backend()
  n = 2048
  ad = be.convert_to_tensor(_random(np.random.default_rng(7), (n, n), "float64"))
  be.synchronize()
  c0 = be.lib.tnb200_launch_count()
  be.inv(ad)
  launches = be.lib.tnb200_launch_count() - c0
  assert launches <= 8 * (n // 32) + 8, launches
  assert launches >= 4 * (n // 32), launches
