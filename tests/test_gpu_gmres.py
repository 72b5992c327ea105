"""GPU: restarted GMRES (CudaB200Backend.gmres: tensornetwork_b200/gmres.py on tnb200_arnoldi_orth) against
scipy.sparse.linalg.gmres on the host in float64: info, the matvec count, the true residual and x."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla
from util import get_backend

pytestmark = pytest.mark.gpu

DTYPES = ["float64", "complex128", "float32", "complex64"]


def _single(dtype):
  return np.dtype(dtype) in (np.float32, np.complex64)


def _wide(dtype):
  return np.complex128 if np.dtype(dtype).kind == "c" else np.float64


def _rand(rng, shape, dtype):
  x = rng.standard_normal(shape) + (1j * rng.standard_normal(shape) if np.dtype(dtype).kind == "c" else 0)
  return x.astype(dtype)


class _strict_matvecs:
  """the tests' own matvecs in the input precision (f32 tensordots would otherwise take TF32 at these sizes)"""

  def __init__(self, be):
    self.be = be

  def __enter__(self):
    from tensornetwork_b200 import _lib as L
    self.mode, self.be.math_mode = self.be.math_mode, L.MATH_STRICT

  def __exit__(self, *exc):
    self.be.math_mode = self.mode


def _scipy(matvec, b, x0, tol, atol, m, maxiter):
  """scipy's gmres on the host in double precision, with its matvec count"""
  count = [0]

  def mv(v):
    count[0] += 1
    return matvec(v)
  op = spla.LinearOperator((b.size, b.size), matvec=mv, dtype=b.dtype)
  x, info = spla.gmres(op, b, x0=x0, rtol=tol, atol=atol, restart=m, maxiter=maxiter)
  return x, info, count[0]


def _dense_case(be, A, b, tol, m, maxiter=None, x0=None, atol=None):
  """our gmres on the device and scipy's on the float64 form of the same (stored) A, b and x0"""
  from tensornetwork_b200 import gmres
  Ad, bd = be.convert_to_tensor(A), be.convert_to_tensor(b)
  x0d = None if x0 is None else be.convert_to_tensor(x0)
  seen = set()

  def mv(v):
    seen.add(v.code)
    return be.tensordot(Ad, v, ([1], [0]))
  with _strict_matvecs(be):
    x, info, st = gmres.gmres(be, mv, bd, None, None, x0d, tol, atol, m, maxiter, None, return_info=True)
  assert seen <= {bd.code} and x.dtype == b.dtype and x.shape == b.shape
  np.testing.assert_array_equal(bd.to_host(), b)
  if x0 is not None:
    np.testing.assert_array_equal(x0d.to_host(), x0)
  Aw, bw = A.astype(_wide(A.dtype)), b.astype(_wide(A.dtype))
  x0w = None if x0 is None else x0.astype(_wide(A.dtype))
  xs, sinfo, smv = _scipy(lambda v: Aw @ v, bw, x0w, tol, tol if atol is None else atol, m, maxiter)
  assert info == sinfo, (info, sinfo, st)
  assert st["matvecs"] == smv, (st, smv)
  xh = x.to_host().astype(Aw.dtype)
  bn = np.linalg.norm(bw)
  if info == 0:
    goal = max(tol if atol is None else atol, tol * bn)
    slack = 10 * np.finfo(b.dtype).eps * np.linalg.norm(Aw) * np.linalg.norm(xh)       # the residual of a rounded x
    assert np.linalg.norm(bw - Aw @ xh) <= goal * 1.0001 + slack
  return xh, xs, info, st


def _shifted(rng, n, dtype):
  """3 I + G / sqrt(n): nonsymmetric, eigenvalues in the unit disc around 3"""
  g = _rand(rng, (n, n), dtype) / np.sqrt(n * (2 if np.dtype(dtype).kind == "c" else 1))
  return (3.0 * np.eye(n) + g).astype(dtype)


def _indefinite(rng, n, dtype):
  """eigenvalues in [-3, -1] and [1, 3], non-normal"""
  lam = np.concatenate([-rng.uniform(1, 3, n // 2), rng.uniform(1, 3, n - n // 2)])
  q = np.linalg.qr(_rand(rng, (n, n), _wide(dtype)))[0]
  t = np.diag(lam) + np.triu(_rand(rng, (n, n), _wide(dtype)), 1) * (0.3 / np.sqrt(n))
  return (q @ t @ q.conj().T).astype(dtype)


@pytest.mark.parametrize("m", [20, 50])
@pytest.mark.parametrize("n", [100, 1000, 4096])
@pytest.mark.parametrize("dtype", DTYPES)
def test_dense_operators(dtype, n, m):
  be = get_backend()
  rng = np.random.default_rng(n + m)
  tol = 1e-5 if _single(dtype) else 1e-10
  b = _rand(rng, n, dtype)
  mats = [_shifted(rng, n, dtype)] + ([_indefinite(rng, n, dtype)] if n <= 1000 else [])
  for A in mats:
    xh, xs, info, st = _dense_case(be, A, b, tol, m, maxiter=500)
    assert info == 0, st
    cond = np.linalg.cond(A.astype(_wide(dtype)), 1)
    assert np.linalg.norm(xh - xs) <= 10 * tol * cond * np.linalg.norm(xs)


@pytest.mark.parametrize("dtype", DTYPES)
def test_breakdown_gives_the_exact_solution(dtype):
  """b in an invariant subspace of dimension 3 < m: the kernel reports beta = 0 at the third step"""
  be = get_backend()
  d = np.arange(1.0, 201.0)
  A = np.diag(d).astype(dtype)
  b = np.zeros(200, dtype)
  b[[3, 17, 130]] = [1.0, -2.0, 0.5]
  xh, _, info, st = _dense_case(be, A, b, 1e-5 if _single(dtype) else 1e-14, 10, maxiter=5, atol=0.0)
  assert info == 0 and st["cycles"] == 1 and st["matvecs"] == 4, st
  np.testing.assert_allclose(xh, b / d, rtol=0, atol=(1e-6 if _single(dtype) else 1e-14))


@pytest.mark.parametrize("dtype", DTYPES)
def test_maxiter_and_x0(dtype):
  be = get_backend()
  rng = np.random.default_rng(2)
  n = 500
  tol = 1e-5 if _single(dtype) else 1e-10
  A = _shifted(rng, n, dtype)
  b = _rand(rng, n, dtype)
  _, _, info, st = _dense_case(be, A, b, tol, 3, maxiter=2)             # stops at maxiter
  assert info == 2 and st["cycles"] == 2 and st["matvecs"] == 8, st
  x0 = _rand(rng, n, dtype)
  _, _, info, st = _dense_case(be, A, b, tol, 20, maxiter=50, x0=x0)     # a nonzero x0: one more matvec
  assert info == 0 and st["matvecs"] > 1, st
  xe = np.linalg.solve(A.astype(_wide(dtype)), b.astype(_wide(dtype))).astype(dtype)
  xh, _, info, st = _dense_case(be, A, b, 1e-3 if _single(dtype) else 1e-10, 20, x0=xe)   # already exact
  assert info == 0 and st["matvecs"] == 1 and st["cycles"] == 0, st
  np.testing.assert_array_equal(xh, xe.astype(xh.dtype))
  xh, _, info, st = _dense_case(be, A, np.zeros(n, dtype), tol, 20, x0=x0)                # b = 0
  assert info == 0 and st["matvecs"] == 0 and not xh.any()
  bn = np.linalg.norm(b.astype(_wide(dtype)))
  xh, _, info, st = _dense_case(be, A, b, 1e-12 if not _single(dtype) else 1e-6, 10, maxiter=50, atol=1e-3 * bn)
  assert info == 0 and st["cycles"] == 1, st                            # atol dominates tol


# ---------------------------------------------------------------- the reference's callers
@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, np.complex128])
def test_krylov_gmres(tn, dtype):
  """linalg/tests/test_krylov.py::test_gmres and ::test_gmres_with_args on backend="cuda_b200": the backend method,
  krylov.gmres, and krylov.gmres with the operator passed in A_args agree, and solve the 2 x 2 system.  (Their numpy
  arm cannot run here: the reference's NumPyBackend.gmres passes `tol=` to scipy.sparse.linalg.gmres, which SciPy
  1.14 removed.)"""
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import  (registers "cuda_b200")
  from tensornetwork.linalg import krylov
  be = get_backend()
  Adat = np.array(([[1, 1], [3, -4]]), dtype=dtype)
  A = tn.Tensor(be.convert_to_tensor(Adat), backend="cuda_b200")
  bdat = np.array([3, 2], dtype=dtype).reshape((2, 1))
  b = tn.Tensor(be.convert_to_tensor(bdat), backend="cuda_b200")
  x0 = tn.Tensor(be.convert_to_tensor(np.ones((2, 1), dtype=dtype)), backend="cuda_b200")

  def A_mv(y):
    return A @ y

  def A_mv_arr(y):
    return A.array @ y

  def A_mv_test(y, A):
    return A @ y
  with _strict_matvecs(be):
    x, info = A.backend.gmres(A_mv_arr, b.array, x0=x0.array, num_krylov_vectors=2)
    xT, infoT = krylov.gmres(A_mv, b, x0=x0, num_krylov_vectors=2)
    xA, infoA = krylov.gmres(A_mv_test, b, x0=x0, num_krylov_vectors=2, A_args=[A])
  assert info == infoT == infoA == 0
  np.testing.assert_allclose(x.to_host(), xT.array.to_host())
  np.testing.assert_allclose(xT.array.to_host(), xA.array.to_host())
  exact = np.linalg.solve(Adat.astype(np.complex128), bdat.astype(np.complex128))
  np.testing.assert_allclose(x.to_host(), exact, rtol=1e-5 if dtype in (np.float32, np.complex64) else 1e-12)


def test_krylov_gmres_raises(tn):
  """linalg/tests/test_krylov.py::test_gmres_raises with the jax arm replaced by cuda_b200"""
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import
  from tensornetwork.linalg import initialization, krylov
  tensor = initialization.ones((2, 1), backend="cuda_b200", dtype=np.float64)
  tensornp = initialization.ones((2, 1), backend="numpy", dtype=np.float64)

  def matvec(B):
    return tensor @ B
  with pytest.raises(ValueError):
    krylov.gmres(matvec, tensor, x0=tensornp)
  with pytest.raises(ValueError):
    krylov.gmres(matvec, tensornp, x0=tensor)
  with pytest.raises(TypeError):
    krylov.gmres(matvec, tensor.array)
  with pytest.raises(TypeError):
    krylov.gmres(matvec, tensor, x0=tensor.array)
  with pytest.raises(TypeError):
    krylov.gmres(matvec, tensor, A_args=[tensor.array])


# ---------------------------------------------------------------- the infinite-MPS environment equation
def _real_part(v):
  """a complex eigenvector of a real operator's real eigenvalue, rotated to be real, as a real array"""
  i = np.argmax(np.abs(v))
  v = v * (abs(v.flat[i]) / v.flat[i])
  assert np.abs(v.imag).max() <= 1e-10 * np.abs(v).max()
  return v.real


def environment_problem(D, dtype, seed):
  """A random InfiniteMPS (d = 2, two-site unit cell) on cuda_b200 and the operator x - T(x) / eta + tr(x r) l of
  its unit-cell transfer operator T, with eta, l and r the dominant eigenvalue and eigenvectors from
  transfer_matrix_eigs("l") and ("r"), normalised so that tr(l r) = 1.  The state is not canonicalised: for a real
  state, canonicalize returns complex tensors (its eigh gauge carries phases), which would make T complex; dividing T
  by eta poses the same equation.  Returns (device matvec, host matvec on numpy arrays, device mps)."""
  from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS
  np.random.seed(seed)
  ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=dtype, backend="numpy")
  mps = InfiniteMPS(tensors=[np.asarray(t) for t in ref.tensors], center_position=0, backend="cuda_b200")
  be = mps.backend
  eta, l = mps.transfer_matrix_eigs("l")
  _, r = mps.transfer_matrix_eigs("r")
  eta = complex(eta.item())
  lh, rh = l.to_host(), r.to_host()
  if np.dtype(dtype).kind != "c":
    assert abs(eta.imag) <= 1e-12 * abs(eta)
    eta, lh, rh = eta.real, _real_part(lh), _real_part(rh)
  lh = lh / np.linalg.norm(lh)
  rh = rh / np.trace(lh @ rh)
  lh, rh = lh.astype(dtype), rh.astype(dtype)
  ld, rd = be.convert_to_tensor(lh), be.convert_to_tensor(rh)
  host = InfiniteMPS(tensors=[np.asarray(t) for t in mps.tensors], center_position=0, backend="numpy")

  def dev(x):
    tx = mps.unit_cell_transfer_operator("l", x)
    return x - tx * (1.0 / eta) + be.tensordot(x, rd, ([0, 1], [1, 0])) * ld

  def hostmv(v):
    x = v.reshape(D, D)
    tx = np.asarray(host.unit_cell_transfer_operator("l", x))
    return (x - tx / eta + np.trace(x @ rh) * lh).ravel()
  return dev, hostmv, mps


@pytest.mark.parametrize("D", [10, 128])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_environment_equation(tn, dtype, D):
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import
  from tensornetwork_b200 import gmres
  dev, hostmv, mps = environment_problem(D, dtype, seed=D)
  be = mps.backend
  rng = np.random.default_rng(D)
  b = _rand(rng, (D, D), dtype)
  bd = be.convert_to_tensor(b)
  x, info, st = gmres.gmres(be, dev, bd, None, None, None, 1e-10, 0.0, 30, 100, None, return_info=True)
  np.testing.assert_array_equal(bd.to_host(), b)
  xs, sinfo, _ = _scipy(hostmv, b.ravel(), None, 1e-10, 0.0, 30, 100)
  assert info == sinfo == 0, (info, sinfo, st)
  xh = x.to_host()
  assert x.shape == (D, D) and xh.dtype == np.dtype(dtype)
  assert np.linalg.norm(b.ravel() - hostmv(xh.ravel())) <= (1e-10 + 1e-14) * np.linalg.norm(b)
  assert np.linalg.norm(xh.ravel() - xs) <= 1e-8 * np.linalg.norm(xs)


# ---------------------------------------------------------------- errors, jit
def test_errors():
  be = get_backend()
  x = be.convert_to_tensor(np.ones(30))
  mv = lambda v: v  # noqa: E731
  with pytest.raises(NotImplementedError):
    be.gmres(mv, x, M=lambda v: v)
  with pytest.raises(NotImplementedError):
    be.gmres(mv, be.convert_to_tensor(np.ones(2000)), num_krylov_vectors=1025)
  with pytest.raises(NotImplementedError):
    be.gmres(mv, be.convert_to_tensor(np.ones(2000)), num_krylov_vectors=None)
  with pytest.raises(TypeError):
    be.gmres(lambda v: be.astype(v, np.complex128), x)
  with pytest.raises(ValueError):
    be.gmres(lambda v: be.reshape(v, (5, 6)), x)
  with pytest.raises(ValueError):
    be.gmres(mv, x, x0=be.convert_to_tensor(np.ones(31)))
  with pytest.raises(TypeError):
    be.gmres(mv, x, x0=be.convert_to_tensor(np.ones(30, np.float32)))
  with pytest.raises(ValueError):
    be.gmres(mv, x, num_krylov_vectors=0)
  with pytest.raises(ValueError):
    be.gmres(mv, x, tol=-1.0)
  with pytest.raises(ValueError):
    be.gmres(mv, x, atol=-1.0)
  with pytest.raises(TypeError):
    be.gmres(mv, be.convert_to_tensor(np.ones(30, np.int32)))
  with pytest.raises(TypeError):
    be.gmres(mv, be.astype(x, "bfloat16"))


def test_jit_falls_back_to_eager():
  be = get_backend()
  rng = np.random.default_rng(11)
  A = _shifted(rng, 100, "float64")
  Ad = be.convert_to_tensor(A)
  b = rng.standard_normal(100)
  f = be.jit(lambda v: be.gmres(lambda y: be.tensordot(Ad, y, ([1], [0])), v, tol=1e-10, maxiter=10)[0],
             static_argnums=())
  fails0 = be.jit_stats["capture_failures"]
  for _ in range(3):
    x = f(be.convert_to_tensor(b)).to_host()
    assert np.linalg.norm(A @ x - b) <= 1e-10 * np.linalg.norm(b)
  assert be.jit_stats["capture_failures"] - fails0 == 1
