"""GPU: the non-Hermitian eigensolver (CudaB200Backend.eigs: implicitly restarted Arnoldi, tnb200_arnoldi_orth) against
numpy in float64.  Eigenvectors are never compared element by element: only through residuals, or up to a scalar."""
import numpy as np
import pytest
import torch
from util import get_backend

pytestmark = pytest.mark.gpu

DTYPES = ["float64", "complex128", "float32", "complex64"]
WHICH = ["LM", "SM", "LR", "SR"]


def _single(dtype):
  return np.dtype(dtype) in (np.float32, np.complex64)


def _tols(dtype):
  return (1e-5, 1e-4) if _single(dtype) else (1e-12, 1e-9)


def _acc(dtype):
  return np.complex128 if np.dtype(dtype).kind == "c" else np.float64


# ---------------------------------------------------------------- 1. the kernel through the C ABI
def _orthonormal_rows(rng, k, n, dtype):
  """k orthonormal rows of length n (k <= n): QR for moderate n, signed Fourier rows for long ones"""
  cplx = np.dtype(dtype).kind == "c"
  if n <= 5000:
    x = rng.standard_normal((n, k)) + (1j * rng.standard_normal((n, k)) if cplx else 0)
    return np.linalg.qr(x)[0].T.copy()
  e = np.arange(n)
  s = rng.choice([-1.0, 1.0], n)
  f = np.arange(1, k + 1)[:, None]
  if cplx:
    return np.exp(2j * np.pi * f * e[None, :] / n) * s / np.sqrt(n)
  return np.sqrt(2.0 / n) * np.cos(2 * np.pi * f * e[None, :] / n) * s        # n odd: orthogonal for f < n / 2


def _cgs2(V, w):
  h1 = V.conj() @ w
  u = w - V.T @ h1
  h2 = V.conj() @ u
  r = u - V.T @ h2
  return h1 + h2, r


def _orth(be, Vd, j, wd):
  from tensornetwork_b200 import _lib as L
  acc = torch.complex128 if Vd.t.is_complex() else torch.float64
  h = torch.zeros(j + 2, dtype=acc, device=be.device)
  L.check(be.lib.tnb200_arnoldi_orth(Vd.ref(), j, wd.ref(), h.data_ptr(), be._stream()))
  return h


@pytest.mark.parametrize("n", [1, 3, 31, 32, 33, 1000, 4097, 2**20 + 7])
@pytest.mark.parametrize("dtype", DTYPES)
def test_orth_kernel(dtype, n):
  be = get_backend()
  rng = np.random.default_rng(n)
  single = _single(dtype)
  for j in (0, 1, 63, 64, 65, 255):
    k = j + 1
    if n >= 2**20 and j > 65:
      continue                                           # n = 4097 covers j = 255; this keeps host memory modest
    cplx = np.dtype(dtype).kind == "c"
    ortho = k < n and (n <= 5000 or k < n // 2)
    if ortho:
      V = _orthonormal_rows(rng, k, n, dtype)
    else:                                                # more rows than n: any rows, CGS2 arithmetic only
      V = rng.standard_normal((k, n)) + (1j * rng.standard_normal((k, n)) if cplx else 0)
    Vs = np.zeros((k + 1, n), dtype)
    Vs[:k] = V
    w = (rng.standard_normal(n) + (1j * rng.standard_normal(n) if cplx else 0)).astype(dtype)
    Vd, wd = be.convert_to_tensor(Vs), be.convert_to_tensor(w)
    n0 = be.lib.tnb200_launch_count()
    h = _orth(be, Vd, j, wd).cpu().numpy()
    assert be.lib.tnb200_launch_count() - n0 == 4          # the constant in arnoldi.cu's comment
    assert be.lib.tnb200_last_kernel().decode() == "arnoldi_cgs2"
    np.testing.assert_array_equal(wd.to_host(), w)         # w is only read
    out = Vd.to_host().astype(_acc(dtype))
    Vh = Vs[:k].astype(_acc(dtype))
    ref_h, r = _cgs2(Vh, w.astype(_acc(dtype)))
    tol = 1e-5 if single else 1e-12
    scale = np.linalg.norm(w) * (1 + np.abs(Vh).max() * np.sqrt(n) if not ortho else 1)
    if not ortho:
      assert np.all(np.isfinite(h))
      continue
    np.testing.assert_allclose(h[:k], ref_h, rtol=0, atol=tol * scale)
    beta = h[k].real
    np.testing.assert_allclose(beta, np.linalg.norm(r), rtol=0, atol=tol * scale)
    assert h[k].imag == 0
    np.testing.assert_array_equal(out[:k], Vh)             # rows 0..j untouched
    if beta > 0:
      otol = 1e-5 if single else 1e-13 * max(1.0, np.sqrt(n) / 100)     # host rows of 2^20 elements: 1e-12
      assert abs(np.linalg.norm(out[k]) - 1) < otol
      assert np.abs(Vh.conj() @ out[k]).max() < otol


@pytest.mark.parametrize("dtype", DTYPES)
def test_orth_in_span_is_breakdown(dtype):
  be = get_backend()
  rng = np.random.default_rng(5)
  k, n = 20, 3000
  V = _orthonormal_rows(rng, k, n, dtype)
  Vs = np.zeros((k + 1, n), dtype)
  Vs[:k] = V
  w = (rng.standard_normal(k) @ V).astype(dtype)
  Vd = be.convert_to_tensor(Vs)
  h = _orth(be, Vd, k - 1, be.convert_to_tensor(w)).cpu().numpy()
  assert h[k] == 0
  assert np.all(Vd.to_host()[k] == 0)


# ---------------------------------------------------------------- 2. dense operators
def _unitary(rng, n, dtype):
  cplx = np.dtype(dtype).kind == "c"
  x = rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cplx else 0)
  return np.linalg.qr(x)[0]


def _from_spectrum(rng, lam, dtype, normal, q=None):
  n = len(lam)
  q = _unitary(rng, n, dtype) if q is None else q
  t = np.diag(lam).astype(_acc(dtype))
  if not normal:                                         # Schur form with a random unitary
    t = t + np.triu(rng.standard_normal((n, n)), 1) * (0.5 / np.sqrt(n))
  return (q @ t @ q.conj().T).astype(dtype)


def _key(vals, which):
  k = {"LM": -np.abs(vals), "SM": np.abs(vals), "LR": -vals.real, "SR": vals.real}[which]
  return np.lexsort((-vals.imag, np.round(k / np.abs(vals).max(), 10)))


def _spectrum(rng, n, which):
  """the six best under `which` stand apart from each other and from the rest"""
  if which == "SM":
    head = [0.01, 0.02, -0.03, 0.045, 0.06, 0.075, -0.09]
    return np.concatenate([head, rng.uniform(1.0, 3.0, n - len(head))])
  head = [10.0, 9.0, 8.2, 7.5, 7.0, 6.6, -10.5, -9.3, -8.4, -7.6, -7.1, -6.5]
  return np.concatenate([head, rng.uniform(-3.0, 3.0, n - len(head))])


class _strict_matvecs:
  """the tests' own matvecs in the input precision (f32 tensordots would otherwise take TF32 at these sizes)"""

  def __init__(self, be):
    self.be = be

  def __enter__(self):
    from tensornetwork_b200 import _lib as L
    self.mode, self.be.math_mode = self.be.math_mode, L.MATH_STRICT

  def __exit__(self, *exc):
    self.be.math_mode = self.mode


def _dense_case(be, M, which, numeig, ncv, dtype, spectrum=None, x0=None):
  """spectrum: M's eigenvalues when known (else np.linalg.eig)"""
  from tensornetwork_b200 import arnoldi
  tol, rtol = _tols(dtype)
  Md = be.convert_to_tensor(M)
  n = M.shape[0]
  if x0 is None:
    x0 = np.random.default_rng(0).standard_normal(n).astype(dtype)
  x0d = be.convert_to_tensor(x0)
  seen = set()

  def mv(x):
    seen.add(x.code)
    return be.tensordot(Md, x, ([1], [0]))
  with _strict_matvecs(be):
    eta, vecs, info = arnoldi.eigs(be, mv, [], x0d, None, None, ncv, numeig, tol, which, None, return_info=True)
  assert seen == {x0d.code}
  np.testing.assert_array_equal(x0d.to_host(), x0)
  assert eta.shape == (numeig,) and eta.dtype == (np.complex64 if _single(dtype) else np.complex128)
  assert len(vecs) == numeig and all(v.shape == (n,) and v.dtype == eta.dtype for v in vecs)
  lam = eta.to_host().astype(np.complex128)
  ref = np.linalg.eig(M.astype(np.complex128))[0] if spectrum is None else np.asarray(spectrum, np.complex128)
  scale = np.abs(ref).max()
  ref = ref[_key(ref, which)][:numeig]
  np.testing.assert_allclose(lam, ref, rtol=0, atol=rtol * scale)
  for l, v in zip(lam, vecs):
    x = v.to_host().astype(np.complex128)
    assert abs(np.linalg.norm(x) - 1) < 10 * rtol
    assert np.linalg.norm(M @ x - l * x) <= 50 * rtol * scale
  return lam, vecs, info


@pytest.mark.parametrize("n", [20, 100, 1000, 4096])
@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_operators(dtype, n):
  be = get_backend()
  rng = np.random.default_rng(n)
  q = _unitary(rng, n, dtype)
  for which in WHICH:
    for normal in (True, False):
      lam = _spectrum(rng, n, which)
      M = _from_spectrum(rng, lam, dtype, normal, q)
      for numeig in (1, 3, 6):
        ncv = min(n, 60 if which == "SM" else 24)
        _dense_case(be, M, which, numeig, ncv, dtype, spectrum=lam)


# ---------------------------------------------------------------- 3. real operators with complex spectra
@pytest.mark.parametrize("numeig", [1, 2])
def test_real_operator_conjugate_pair(numeig):
  be = get_backend()
  rng = np.random.default_rng(3)
  n = 300
  d = np.zeros((n, n))
  for b, (r, im) in enumerate([(2.0, 1.0), (1.5, 0.5), (0.5, 0.2)]):
    d[2 * b:2 * b + 2, 2 * b:2 * b + 2] = [[r, -im], [im, r]]
  d[6:, 6:] = np.diag(rng.uniform(-0.5, 0.5, n - 6))
  q = np.linalg.qr(rng.standard_normal((n, n)))[0]
  M = q @ d @ q.T
  lam, _, _ = _dense_case(be, M, "LM", numeig, 20, "float64")
  np.testing.assert_allclose(lam[0], 2.0 + 1.0j, atol=1e-9)
  if numeig == 2:
    assert lam[1] == np.conj(lam[0])


def test_real_dominant_eigenvalue_is_exactly_real():
  be = get_backend()
  rng = np.random.default_rng(4)
  M = _from_spectrum(rng, np.concatenate([[5.0], rng.uniform(-1, 1, 399)]), "float64", normal=False)
  lam, vecs, _ = _dense_case(be, M, "LR", 1, 20, "float64", spectrum=None)
  assert lam[0].imag == 0.0
  assert np.all(vecs[0].to_host().imag == 0.0)


# ---------------------------------------------------------------- 4. breakdown
@pytest.mark.parametrize("dtype", DTYPES)
def test_breakdown_invariant_subspace(dtype):
  be = get_backend()
  M = np.diag(np.arange(1.0, 201.0)).astype(dtype)
  x0 = np.zeros(200, dtype)
  x0[[3, 17, 130]] = 1.0
  Md = be.convert_to_tensor(M)
  with _strict_matvecs(be):
    eta, vecs = be.eigs(lambda x: be.tensordot(Md, x, ([1], [0])), initial_state=be.convert_to_tensor(x0),
                        num_krylov_vecs=10, numeig=2, tol=_tols(dtype)[0])
  lam = eta.to_host()
  assert np.all(np.isfinite(lam))
  np.testing.assert_allclose(lam, [131.0, 18.0], rtol=_tols(dtype)[1])
  for l, v in zip(lam, vecs):
    x = v.to_host().astype(np.complex128)
    assert np.all(np.isfinite(x))
    assert np.linalg.norm(M @ x - l * x) <= _tols(dtype)[1] * 200


# ---------------------------------------------------------------- 5. the reference's callers
@pytest.mark.parametrize("D", [10, 128])
@pytest.mark.parametrize("direction", ["l", "r"])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_transfer_matrix_eigs(tn, dtype, direction, D):
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import  (registers "cuda_b200")
  from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS
  np.random.seed(7)
  ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=dtype, backend="numpy")
  mps = InfiniteMPS(tensors=[np.asarray(t) for t in ref.tensors], center_position=0, backend="cuda_b200")
  eta, l = mps.transfer_matrix_eigs(direction)
  reta, rl = ref.transfer_matrix_eigs(direction)
  assert eta.dtype == np.complex128 and l.dtype == np.complex128
  l2 = mps.unit_cell_transfer_operator(direction, l)
  e, lh, l2h = complex(eta.item()), l.to_host(), l2.to_host()
  assert np.linalg.norm(l2h - e * lh) <= 1e-9 * abs(e) * np.linalg.norm(lh)
  assert abs(e - complex(reta)) <= 1e-9 * abs(complex(reta))
  rlh = np.asarray(rl).ravel()
  c = np.vdot(rlh, lh.ravel()) / np.vdot(rlh, rlh)
  assert np.linalg.norm(lh.ravel() - c * rlh) <= 1e-8 * np.linalg.norm(lh)
  s = mps.backend.sqrt(mps.backend.abs(eta))                  # the way canonicalize uses eta
  assert s.shape == () and abs(float(s.item()) - np.sqrt(abs(e))) < 1e-12 * np.sqrt(abs(e))


def test_krylov_eigs_with_args(tn):
  """linalg/tests/test_krylov.py::test_eigs_with_args on backend="cuda_b200": the matvec with and without `args` gives
  the same eigenvalue (4: x0 is an eigenvector, so the Krylov space breaks down after one step), and
  matvec(R) / r = R.  (Its numpy arm cannot run here: scipy refuses the (4, 4) x0 as v0.)"""
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import
  from tensornetwork.linalg import initialization, krylov
  shape = (4, 4)
  tensor = initialization.ones(shape, backend="cuda_b200", dtype=np.float64)
  x0 = initialization.ones(shape, backend="cuda_b200", dtype=np.float64)

  def matvec(B):
    return tensor @ B

  def test_matvec(B, A):
    return A @ B
  rev, _ = krylov.eigs(matvec, backend="cuda_b200", x0=x0, num_krylov_vecs=3, numeig=1)
  tev, teV = krylov.eigs(test_matvec, x0=x0, num_krylov_vecs=3, numeig=1, args=[tensor])
  for r, t, R in zip(rev.to_host(), tev.to_host(), teV):
    np.testing.assert_allclose(r, t)
    np.testing.assert_allclose(t, 4.0, rtol=1e-12)
    np.testing.assert_allclose(np.asarray((matvec(R) / t).array), np.asarray(R.array), rtol=1e-5)


# ---------------------------------------------------------------- 6. errors and limits
def test_errors_and_limits():
  be = get_backend()
  x = be.convert_to_tensor(np.ones(30))
  mv = lambda v: v  # noqa: E731
  with pytest.raises(ValueError):
    be.eigs(mv, initial_state=x, which="LI")
  with pytest.raises(ValueError):
    be.eigs(mv, initial_state=x, which="SI")
  with pytest.raises(ValueError):
    be.eigs(mv, initial_state=x, numeig=5, num_krylov_vecs=6)
  with pytest.raises(ValueError):
    be.eigs(mv)
  with pytest.raises(ValueError):
    be.eigs(mv, initial_state=x, numeig=2, num_krylov_vecs=31)
  with pytest.raises(TypeError):
    be.eigs(mv, initial_state=x, numeig=29, num_krylov_vecs=31)
  with pytest.raises(TypeError):
    be.eigs(mv, initial_state=np.ones(30), num_krylov_vecs=10)
  with pytest.raises(TypeError):
    be.eigs(mv, initial_state=be.convert_to_tensor(np.ones(30, np.int32)), num_krylov_vecs=10, numeig=1)
  with pytest.raises(TypeError):
    be.eigs(mv, initial_state=be.astype(x, "bfloat16"), num_krylov_vecs=10, numeig=1)
  with pytest.raises(ValueError):
    be.eigs(lambda v: be.reshape(v, (5, 6)), initial_state=x, numeig=1, num_krylov_vecs=10)
  with pytest.raises(ValueError):
    be.eigs(mv, initial_state=be.convert_to_tensor(np.zeros(30)), numeig=1, num_krylov_vecs=10)
  # a slowly converging case: maxiter=1 is a soft RuntimeError, and the initial state is left alone
  rng = np.random.default_rng(9)
  M = _from_spectrum(rng, np.concatenate([[1.0, 0.99], rng.uniform(-0.9, 0.9, 998)]), "float64", True)
  Md = be.convert_to_tensor(M)
  x0 = rng.standard_normal(1000)
  x0d = be.convert_to_tensor(x0)
  with pytest.raises(RuntimeError, match="converged"):
    be.eigs(lambda v: be.tensordot(Md, v, ([1], [0])), initial_state=x0d, numeig=1, num_krylov_vecs=8, maxiter=1,
            tol=1e-12)
  np.testing.assert_array_equal(x0d.to_host(), x0)
  eta, _ = be.eigs(lambda v: be.tensordot(Md, v, ([1], [0])), initial_state=x0d, numeig=1, num_krylov_vecs=8,
                   tol=1e-12)
  assert abs(eta.to_host()[0] - 1.0) < 1e-9


def test_jit_falls_back_to_eager():
  be = get_backend()
  rng = np.random.default_rng(11)
  M = _from_spectrum(rng, np.concatenate([[4.0, 3.0], rng.uniform(-1, 1, 98)]), "float64", False)
  Md = be.convert_to_tensor(M)
  x0 = be.convert_to_tensor(rng.standard_normal(100))
  f = be.jit(lambda x: be.eigs(lambda v: be.tensordot(Md, v, ([1], [0])), initial_state=x, numeig=1,
                               num_krylov_vecs=20, tol=1e-12)[0], static_argnums=())
  fails0 = be.jit_stats["capture_failures"]
  for _ in range(3):
    assert abs(f(x0).to_host()[0] - 4.0) < 1e-9
  assert be.jit_stats["capture_failures"] - fails0 == 1
