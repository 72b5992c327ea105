"""GPU: the matrix exponential (tnb200_expm behind CudaB200Backend.expm) against scipy.linalg.expm, its degree and
squaring choice against the restatement of scipy's rule in expm_rule.py, known answers, non-finite input, graph
capture, and tnb200_lu_solve against scipy.linalg.lu_solve."""
import numpy as np
import pytest
import scipy.linalg
import torch
from util import get_backend
import expm_rule

pytestmark = pytest.mark.gpu


def _lib():
  from tensornetwork_b200 import _lib as L
  return L


F = 48      # _lib.EXPM_FUSED_MAX_N, checked below


def _random(rng, shape, dtype):
  x = rng.standard_normal(shape)
  if np.dtype(dtype).kind == "c":
    x = x + 1j * rng.standard_normal(shape)
  return x.astype(dtype)


def _expm_info(be, a):
  """tnb200_expm through the C ABI -> (x on the host, info [m, s, path, lu_info])"""
  L = _lib()
  x = be._new(a.shape, a.code)
  info = torch.full((4,), -7, dtype=torch.int32, device=be.device)
  L.check(be.lib.tnb200_expm(a.ref(), x.ref(), info.data_ptr(), be._stream()))
  return x.to_host(), info.cpu().numpy()


def _tol(n, a, dtype):
  eps = np.finfo(np.dtype(dtype)).eps
  return 100 * n * eps * max(1.0, expm_rule.onenorm(a))


def _rel(x, ref):
  return np.linalg.norm(x - ref) / np.linalg.norm(ref)


def test_fused_limit_matches_header():
  assert _lib().EXPM_FUSED_MAX_N == F


@pytest.mark.parametrize("n", [2, 3, 4, 9, 16, 31, 32, 33, F - 1, F, F + 1, 100, 256, 1000])
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_parity_with_scipy(dtype, n):
  be = get_backend()
  rng = np.random.default_rng(n)
  a = _random(rng, (n, n), dtype)
  a /= expm_rule.onenorm(a)                      # ||A||_1 = 1
  x, info = _expm_info(be, be.convert_to_tensor(a))
  ref = scipy.linalg.expm(a)
  assert x.dtype == np.dtype(dtype)
  assert _rel(x, ref) <= _tol(n, a, dtype)
  assert tuple(info[:2]) == expm_rule.select(a)
  assert info[2] == (0 if n <= F else 1) and info[3] == 0


def test_path_flips_at_the_fused_limit():
  be = get_backend()
  for n, path in ((F, 0), (F + 1, 1)):
    a = _random(np.random.default_rng(3), (n, n), "complex128") * 0.1
    _, info = _expm_info(be, be.convert_to_tensor(a))
    assert info[2] == path


def test_size_one_and_zero():
  be = get_backend()
  np.testing.assert_allclose(be.expm(be.convert_to_tensor(np.array([[0.5]]))).to_host(), [[np.exp(0.5)]], rtol=1e-15)
  z = be.expm(be.convert_to_tensor(np.zeros((0, 0), dtype=np.complex64)))
  assert z.shape == (0, 0) and z.dtype == np.complex64


@pytest.mark.parametrize("dtype,out", [("float32", "float32"), ("complex64", "complex64"), ("int64", "float64"),
                                       ("int32", "float64"), ("bool", "float64")])
@pytest.mark.parametrize("n", [3, F, F + 1, 100])
def test_other_dtypes(dtype, out, n):
  be = get_backend()
  rng = np.random.default_rng(n + 1)
  if dtype in ("int64", "int32"):
    a = rng.integers(-2, 3, (n, n)).astype(dtype)
    scale = 1
  elif dtype == "bool":
    a = rng.random((n, n)) < 1.0 / n
    scale = 1
  else:
    a = _random(rng, (n, n), dtype)
    scale = expm_rule.onenorm(a)
    a = (a / scale).astype(dtype)
  r = be.expm(be.convert_to_tensor(a))
  assert r.dtype == np.dtype(out)
  a64 = a.astype(np.complex128 if np.dtype(dtype).kind == "c" else np.float64)
  ref = scipy.linalg.expm(a64)
  assert _rel(r.to_host(), ref) <= _tol(n, a64, out)


@pytest.mark.parametrize("n", [4, F + 1])
def test_bf16_gives_float32(n):
  be = get_backend()
  a = np.random.default_rng(2).standard_normal((n, n)) / n
  t = be.astype(be.convert_to_tensor(a), _lib().BF16)
  r = be.expm(t)
  assert r.dtype == np.float32
  a16 = be.astype(t, _lib().F64).to_host()
  assert _rel(r.to_host(), scipy.linalg.expm(a16)) <= _tol(n, a16, "float32")


# matrices scaled into each degree and into s = 0, 1 and >= 8, kept away from the selection boundaries
@pytest.mark.parametrize("n", [8, F + 8])
@pytest.mark.parametrize("target", [(3, 0), (5, 0), (7, 0), (9, 0), (13, 0), (13, 1), (13, 9)])
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_each_degree_and_squaring(dtype, target, n):
  be = get_backend()
  rng = np.random.default_rng(11)
  h = _random(rng, (n, n), dtype)
  h = h / expm_rule.onenorm(h)
  scale = {(3, 0): 0.005, (5, 0): 0.1, (7, 0): 0.5, (9, 0): 1.8, (13, 0): 4.5, (13, 1): 11.0, (13, 9): 1500.0}[target]
  if target == (13, 9):                          # skew-Hermitian, so that exp(A) stays bounded at this norm
    h = (h - h.conj().T) / expm_rule.onenorm(h - h.conj().T)
  a = h * scale
  sel = expm_rule.select(a)
  assert sel[0] == target[0] and (sel[1] == target[1] or (target[1] >= 8 and sel[1] >= 8)), sel
  x, info = _expm_info(be, be.convert_to_tensor(a))
  assert tuple(info[:2]) == sel
  ref = scipy.linalg.expm(a)
  assert _rel(x, ref) <= _tol(n, a, dtype)


@pytest.mark.parametrize("n", [5, F + 3])
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_known_answers(dtype, n):
  be = get_backend()
  E = lambda a: be.expm(be.convert_to_tensor(a)).to_host()   # noqa: E731
  eps = np.finfo(np.dtype(dtype)).eps
  np.testing.assert_array_equal(E(np.zeros((n, n), dtype)), np.eye(n))
  d = np.linspace(-2, 1.5, n).astype(dtype)
  np.testing.assert_allclose(E(np.diag(d)), np.diag(np.exp(d)), rtol=100 * n * eps, atol=100 * n * eps)
  N = np.triu(_random(np.random.default_rng(1), (n, n), dtype), 1)
  series, term = np.eye(n, dtype=dtype), np.eye(n, dtype=dtype)
  for k in range(1, n):
    term = term @ N / k
    series = series + term
  assert _rel(E(N), series) <= _tol(n, N, dtype) * 10
  t = 0.7
  rot = E(np.array([[0, -t], [t, 0]], dtype))
  np.testing.assert_allclose(rot, [[np.cos(t), -np.sin(t)], [np.sin(t), np.cos(t)]], atol=1e-15)
  a = _random(np.random.default_rng(2), (n, n), dtype)
  a = a / expm_rule.onenorm(a)
  c = 0.3
  assert _rel(E(a + c * np.eye(n)), np.exp(c) * E(a)) <= _tol(n, a, dtype)
  prod = E(2 * a) @ E(-2 * a)
  assert np.abs(prod - np.eye(n)).max() <= _tol(n, 2 * a, dtype) * 10


@pytest.mark.parametrize("n", [4, 16, F + 1, 64])
def test_unitary_evolution(n):
  be = get_backend()
  h = _random(np.random.default_rng(n), (n, n), "complex128")
  h = (h + h.conj().T) / 2
  u = be.expm(be.convert_to_tensor(-1j * 0.3 * h)).to_host()
  assert np.linalg.norm(u.conj().T @ u - np.eye(n)) <= 50 * n * np.finfo(float).eps
  assert _rel(u, scipy.linalg.expm(-1j * 0.3 * h)) <= _tol(n, 0.3 * h, "complex128")


@pytest.mark.parametrize("n", [6, F + 6])
def test_views_equal_contiguous(n):
  be = get_backend()
  big = _random(np.random.default_rng(4), (2 * n, 2 * n), "complex128") / n
  t = be.convert_to_tensor(big)
  ref = be.expm(be.convert_to_tensor(np.ascontiguousarray(big[1:2 * n:2, :n]))).to_host()
  view = be.slice(t, (1, 0), (2 * n - 1, n))
  from tensornetwork_b200.tensor import B200Tensor
  view = B200Tensor(view.t[::2], view.code)
  np.testing.assert_array_equal(be.expm(view).to_host(), ref)
  reft = be.expm(be.convert_to_tensor(np.ascontiguousarray(big[:n, :n].T))).to_host()
  np.testing.assert_array_equal(be.expm(be.transpose(be.slice(t, (0, 0), (n, n)))).to_host(), reft)


@pytest.mark.parametrize("n", [5, F + 5])
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_gives_nan(bad, n):
  be = get_backend()
  a = np.random.default_rng(1).standard_normal((n, n))
  a[n // 2, 1] = bad
  x, info = _expm_info(be, be.convert_to_tensor(a))
  assert np.isnan(x).all()
  assert np.isnan(be.expm(be.convert_to_tensor(a.astype(np.complex64))).to_host()).all()


def test_graph_capture_small():
  be = get_backend()
  rng = np.random.default_rng(5)
  tau = be.convert_to_tensor(np.array(-0.1j))

  def gates(h):
    return be.expm(be.multiply(h, tau))
  jf = be.jit(gates, static_argnums=())
  st0 = dict(be.jit_stats)
  for _ in range(4):
    h = _random(rng, (16, 16), "complex128")
    h = be.convert_to_tensor(h + h.conj().T)
    out = jf(h).to_host()
    eager = gates(h).to_host()
    np.testing.assert_array_equal(out, eager)
  assert be.jit_stats["captures"] - st0["captures"] == 1
  assert be.jit_stats["capture_failures"] == st0["capture_failures"]


def test_graph_capture_large_runs_eagerly():
  be = get_backend()
  rng = np.random.default_rng(6)
  jf = be.jit(lambda h: be.expm(h), static_argnums=())
  st0 = dict(be.jit_stats)
  for _ in range(3):
    h = be.convert_to_tensor(_random(rng, (F + 1, F + 1), "float64") / F)
    np.testing.assert_array_equal(jf(h).to_host(), be.expm(h).to_host())
  assert be.jit_stats["captures"] == st0["captures"]


@pytest.mark.parametrize("n", [1, 31, 32, 33, 100, 1000])
@pytest.mark.parametrize("k", ["1", "7", "n"])
@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_lu_solve(dtype, k, n):
  be = get_backend()
  L = _lib()
  kk = {"1": 1, "7": 7, "n": n}[k]
  rng = np.random.default_rng(n * 10 + kk)
  a = _random(rng, (n, n), dtype)
  b = _random(rng, (kk, n), dtype).T                 # a strided (column-major) right-hand side
  ad = be.convert_to_tensor(a)
  lu = be._new((n, n), ad.code)
  piv = torch.empty(n, dtype=torch.int32, device=be.device)
  info = torch.empty(1, dtype=torch.int32, device=be.device)
  L.check(be.lib.tnb200_lu_factor(ad.ref(), lu.ref(), piv.data_ptr(), info.data_ptr(), be._stream()))
  bd = be.transpose(be.convert_to_tensor(np.ascontiguousarray(b.T)))
  x = be._new((n, kk), ad.code)
  L.check(be.lib.tnb200_lu_solve(lu.ref(), piv.data_ptr(), bd.ref(), x.ref(), be._stream()))
  xh = x.to_host()
  eps = np.finfo(np.dtype(dtype)).eps
  res = np.linalg.norm(a @ xh - b) / (np.linalg.norm(a) * np.linalg.norm(xh))
  assert res <= 50 * n * eps, res
  ref = scipy.linalg.lu_solve(scipy.linalg.lu_factor(a), b)
  assert _rel(xh, ref) <= 1e4 * n * eps * np.linalg.cond(a)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_reference_entry_point(tn, dtype):
  rng = np.random.default_rng(7)
  a = _random(rng, (8, 8), dtype) / 4
  ours = tn.linalg.linalg.expm(tn.Tensor(get_backend().convert_to_tensor(a), backend="cuda_b200"))
  theirs = tn.linalg.linalg.expm(tn.Tensor(a, backend="numpy"))
  assert _rel(ours.array.to_host(), theirs.array) <= _tol(8, a, dtype)
  eye = tn.eye(6, backend="cuda_b200", dtype=np.dtype(dtype))
  np.testing.assert_allclose(tn.linalg.linalg.expm(eye).array.to_host(),
                             tn.linalg.linalg.expm(tn.eye(6, backend="numpy", dtype=np.dtype(dtype))).array)


def test_ell_terms_drive_the_degree():
  """A^2 = 0 but |A| is not nilpotent: the theta tests all pass and the _ell terms alone choose degree 9"""
  be = get_backend()
  a = np.array([[1.0, 1.0], [-1.0, -1.0]])
  x, info = _expm_info(be, be.convert_to_tensor(a))
  assert tuple(info[:2]) == expm_rule.select(a) == (9, 0)
  np.testing.assert_allclose(x, np.eye(2) + a, rtol=0, atol=1e-15)
