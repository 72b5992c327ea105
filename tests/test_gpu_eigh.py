"""GPU: Hermitian eigendecomposition (CudaB200Backend.eigh -> tnb200_eigh, block Jacobi) against np.linalg.eigh in
float64.  Eigenvalues are compared directly (1e-10 of the largest |w| in f64/c128, 2e-5 in f32/c64); eigenvectors
never element by element, only through the residual ||A V - V diag(w)|| and the orthonormality of V."""
import numpy as np
import pytest
import torch
from util import get_backend

pytestmark = pytest.mark.gpu

DTYPES = ["float64", "complex128", "float32", "complex64"]


def _tol(dtype):
  return 1e-10 if np.dtype(dtype) in (np.float64, np.complex128) else 2e-5


def _wide(dtype):
  return np.complex128 if np.dtype(dtype).kind == "c" else np.float64


def _random(rng, shape, dtype):
  x = rng.standard_normal(shape)
  if np.dtype(dtype).kind == "c":
    x = x + 1j * rng.standard_normal(shape)
  return x


def _unitary(rng, n, dtype):
  return np.linalg.qr(_random(rng, (n, n), dtype))[0]


def _hermitian(rng, n, dtype):
  x = _random(rng, (n, n), dtype)
  return ((x + x.conj().T) / 2).astype(dtype)


def _from_spectrum(rng, lam, dtype):
  q = _unitary(rng, len(lam), dtype)
  return ((q * lam[None, :]) @ q.conj().T).astype(dtype)


def _lower_hermitian(x):
  """The matrix LAPACK's UPLO='L' sees: the lower triangle, its conjugate above, the real part of the diagonal."""
  x = x.astype(_wide(x.dtype))
  low = np.tril(x, -1)
  return low + low.conj().T + np.diag(np.diag(x).real)


def _check(x, w, v, ref_w=None):
  """w, v: the device results for the host matrix x (only x's lower triangle counts)."""
  n = x.shape[0]
  tol = _tol(x.dtype)
  real = np.float32 if np.dtype(x.dtype) in (np.float32, np.complex64) else np.float64
  assert w.shape == (n,) and v.shape == (n, n)
  assert w.dtype == real and v.dtype == x.dtype
  h = _lower_hermitian(x)
  if ref_w is None:
    ref_w = np.linalg.eigh(h)[0]
  wh, vh = w.to_host().astype(np.float64), v.to_host().astype(_wide(x.dtype))
  scale = max(float(np.abs(ref_w).max()), 1e-300)
  np.testing.assert_allclose(wh, ref_w, rtol=0, atol=tol * scale)
  assert np.all(np.diff(wh) >= 0)
  res = np.linalg.norm(h @ vh - vh * wh[None, :]) / max(np.linalg.norm(h), 1e-300)
  assert res <= 50 * tol, res
  np.testing.assert_allclose(vh.conj().T @ vh, np.eye(n), rtol=0, atol=200 * tol)
  return wh, vh


def _eigh_info(be, a):
  """tnb200_eigh through the C ABI, returning (w, v, sweeps, converged)."""
  from tensornetwork_b200 import _lib as L
  from tensornetwork_b200 import tensor as T
  n = a.shape[0]
  w = be._new((n,), T.real_code(a.code))
  v = be._new((n, n), a.code)
  info = torch.zeros(4, dtype=torch.int32, device=be.device)
  L.check(be.lib.tnb200_eigh(a.ref(), w.ref(), v.ref(), info.data_ptr(), be._stream()))
  return w, v, int(info[0]), int(info[1])


@pytest.mark.parametrize("n", [1, 2, 15, 16, 17, 31, 32, 33, 100, 257, 1000])
@pytest.mark.parametrize("dtype", DTYPES)
def test_random_hermitian(dtype, n):
  """Partial pads (n not a multiple of 32), one block pair (n <= 32) and many rounds."""
  be = get_backend()
  rng = np.random.default_rng(1000 + n)
  x = _hermitian(rng, n, dtype)
  w, v = be.eigh(be.convert_to_tensor(x))
  assert be.lib.tnb200_last_kernel().decode() == "eigh_block_jacobi"
  _check(x, w, v)


@pytest.mark.parametrize("dtype", DTYPES)
def test_empty(dtype):
  be = get_backend()
  w, v = be.eigh(be.convert_to_tensor(np.zeros((0, 0), dtype)))
  ref_w, ref_v = np.linalg.eigh(np.zeros((0, 0), dtype))
  assert w.shape == ref_w.shape == (0,) and v.shape == ref_v.shape == (0, 0)
  assert w.dtype == ref_w.dtype and v.dtype == ref_v.dtype


@pytest.mark.parametrize("dtype", DTYPES)
def test_plus_minus_pairs(dtype):
  """+-lambda pairs: the same singular values, which a one-sided method cannot tell apart."""
  be = get_backend()
  rng = np.random.default_rng(2)
  mags = np.repeat(np.arange(1.0, 36.0), 2)
  lam = mags * np.tile([1.0, -1.0], 35)
  x = _from_spectrum(rng, lam, dtype)
  w, v = be.eigh(be.convert_to_tensor(x))
  wh, _ = _check(x, w, v)
  np.testing.assert_allclose(wh, np.sort(lam), rtol=0, atol=_tol(dtype) * 35 * 10)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rank_deficient(dtype):
  """Many exact zero eigenvalues: the finalize step must take the matrix's indices, not look for zeros."""
  be = get_backend()
  rng = np.random.default_rng(3)
  lam = np.concatenate([np.zeros(40), rng.uniform(-3.0, 3.0, 30)])
  x = _from_spectrum(rng, lam, dtype)
  w, v = be.eigh(be.convert_to_tensor(x))
  wh, _ = _check(x, w, v)
  np.testing.assert_allclose(wh, np.sort(lam), rtol=0, atol=_tol(dtype) * 30)
  z = np.zeros((50, 50), dtype)
  w, v = be.eigh(be.convert_to_tensor(z))
  np.testing.assert_array_equal(w.to_host(), np.zeros(50))
  np.testing.assert_array_equal(v.to_host(), np.eye(50))


@pytest.mark.parametrize("dtype", DTYPES)
def test_degenerate(dtype):
  """The identity and c * I (already diagonal: V = I), and a fully degenerate spectrum in a rotated basis."""
  be = get_backend()
  for c in (1.0, -2.5):
    x = (c * np.eye(45)).astype(dtype)
    w, v, sweeps, conv = _eigh_info(be, be.convert_to_tensor(x))
    np.testing.assert_array_equal(w.to_host(), np.full(45, c))
    np.testing.assert_array_equal(v.to_host(), np.eye(45))
    assert (sweeps, conv) == (1, 1)
  rng = np.random.default_rng(4)
  x = _from_spectrum(rng, np.full(70, 3.0), dtype)
  w, v = be.eigh(be.convert_to_tensor(x))
  _check(x, w, v)


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_wide_spread(dtype):
  """Eigenvalues of both signs spread over 1e-8 .. 1e8."""
  be = get_backend()
  rng = np.random.default_rng(5)
  lam = np.logspace(-8, 8, 150) * rng.choice([-1.0, 1.0], 150)
  x = _from_spectrum(rng, lam, dtype)
  w, v = be.eigh(be.convert_to_tensor(x))
  wh, _ = _check(x, w, v)
  np.testing.assert_allclose(wh, np.sort(lam), rtol=0, atol=_tol(dtype) * 1e8)


@pytest.mark.parametrize("dtype", DTYPES)
def test_diagonal_converges_in_one_sweep(dtype):
  be = get_backend()
  rng = np.random.default_rng(6)
  d = rng.standard_normal(77)
  w, v, sweeps, conv = _eigh_info(be, be.convert_to_tensor(np.diag(d).astype(dtype)))
  assert (sweeps, conv) == (1, 1)
  order = np.argsort(d, kind="stable")
  np.testing.assert_array_equal(w.to_host(), d[order].astype(w.dtype))
  np.testing.assert_array_equal(v.to_host(), np.eye(77, dtype=dtype)[:, order])


@pytest.mark.parametrize("dtype", DTYPES)
def test_reads_lower_triangle_only(dtype):
  """A non-Hermitian input (and for complex, an imaginary diagonal) gives what np.linalg.eigh gives on the same array;
  garbage in the upper triangle changes nothing, bit for bit."""
  be = get_backend()
  rng = np.random.default_rng(7)
  x = _random(rng, (90, 90), dtype).astype(dtype)
  if np.dtype(dtype).kind == "c":
    x[np.diag_indices(90)] += 1j * rng.standard_normal(90).astype(dtype)
  w, v = be.eigh(be.convert_to_tensor(x))
  _check(x, w, v, ref_w=np.linalg.eigh(x.astype(_wide(dtype)))[0])
  g = x.copy()
  iu = np.triu_indices(90, 1)
  g[iu] = np.nan
  w2, v2 = be.eigh(be.convert_to_tensor(g))
  np.testing.assert_array_equal(w2.to_host(), w.to_host())
  np.testing.assert_array_equal(v2.to_host(), v.to_host())
  g[iu] = 1e30 * rng.standard_normal(len(iu[0]))
  w3, v3 = be.eigh(be.convert_to_tensor(g))
  np.testing.assert_array_equal(w3.to_host(), w.to_host())
  np.testing.assert_array_equal(v3.to_host(), v.to_host())


@pytest.mark.parametrize("dtype", DTYPES)
def test_strided_input(dtype):
  be = get_backend()
  rng = np.random.default_rng(8)
  x = _random(rng, (70, 70), dtype).astype(dtype)
  t = be.transpose(be.convert_to_tensor(x))            # a transposed view: its lower triangle is x's upper one
  assert not t.t.is_contiguous()
  w, v = be.eigh(t)
  _check(np.ascontiguousarray(x.T), w, v)
  big = _random(rng, (120, 150), dtype).astype(dtype)
  s = be.convert_to_tensor(big)[5:105:2, 7:107:2]     # non-contiguous slice with steps in both axes
  assert not s.t.is_contiguous()
  w, v = be.eigh(s)
  _check(np.ascontiguousarray(big[5:105:2, 7:107:2]), w, v)


def test_errors_match_numpy():
  be = get_backend()
  with pytest.raises(TypeError):
    be.eigh(be.convert_to_tensor(np.eye(4, dtype=np.int32)))
  with pytest.raises(TypeError):
    be.eigh(be.astype(be.convert_to_tensor(np.eye(4, dtype=np.float32)), "bfloat16"))
  with pytest.raises(TypeError):                       # numpy has no 16-bit linalg either
    np.linalg.eigh(np.eye(4, dtype=np.float16))
  with pytest.raises(ValueError):
    be.eigh(be.convert_to_tensor(np.ones((3, 4))))
  with pytest.raises(ValueError):                      # LinAlgError is a ValueError
    np.linalg.eigh(np.ones((3, 4)))
  with pytest.raises(NotImplementedError):
    be.eigh(be.convert_to_tensor(np.ones((2, 3, 3))))


def test_jit_falls_back_to_eager():
  """eigh reads a convergence flag on the host once per sweep, so it cannot be captured in a CUDA graph: the jitted
  function falls back to eager execution and stays correct."""
  be = get_backend()
  rng = np.random.default_rng(9)
  f = be.jit(lambda t: be.eigh(t)[0], static_argnums=())
  fails0 = be.jit_stats["capture_failures"]
  for _ in range(3):
    x = _hermitian(rng, 40, "float64")
    np.testing.assert_allclose(f(be.convert_to_tensor(x)).to_host(), np.linalg.eigh(x)[0], rtol=0, atol=1e-10 * 10)
  assert be.jit_stats["capture_failures"] - fails0 == 1


@pytest.mark.parametrize("dtype", DTYPES)
def test_reference_tn_eigh(tn, dtype):
  """The reference's own caller: linalg.eigh (linalg/linalg.py:178-191) on backend="cuda_b200" against the same call on
  the numpy backend; v compared through v diag(w) v^H, which does not depend on the phase of each column."""
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import  (registers "cuda_b200")
  rng = np.random.default_rng(10)
  x = _hermitian(rng, 60, dtype)
  w, v = tn.eigh(tn.Tensor(x, backend="cuda_b200"))
  rw, rv = tn.eigh(tn.Tensor(x, backend="numpy"))
  assert w.backend.name == "cuda_b200" and v.backend.name == "cuda_b200"
  tol = _tol(dtype)
  rw, rv = np.asarray(rw.array), np.asarray(rv.array)
  wh, vh = np.asarray(w.array), np.asarray(v.array)
  scale = float(np.abs(rw).max())
  np.testing.assert_allclose(wh, rw, rtol=0, atol=tol * scale)
  rec, ref_rec = (vh * wh[None, :]) @ vh.conj().T, (rv * rw[None, :]) @ rv.conj().T
  assert np.linalg.norm(rec - ref_rec) <= 50 * tol * np.linalg.norm(ref_rec)
