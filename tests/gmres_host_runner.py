"""Runs in a subprocess (build container only): the host driver of CudaB200Backend.gmres (tensornetwork_b200/gmres.py)
on a stand-in library whose tnb200_arnoldi_orth is a plain numpy CGS2 on host memory.  Compares info, the matvec count
and x with scipy.sparse.linalg.gmres on dense problems, and checks breakdown, x0, b = 0, atol and the errors; the
kernel itself is checked by tests/test_gpu_eigs.py."""
import numpy as np
import scipy.sparse.linalg as spla
import hostrun
from hostrun import raises
_, lib = hostrun.install()
from tensornetwork_b200 import backend as tb_backend, gmres as tb_gmres  # noqa: E402

be = tb_backend.CudaB200Backend()
rng = np.random.default_rng(1)


def rand(shape, dtype):
  x = rng.standard_normal(shape) + (1j * rng.standard_normal(shape) if np.dtype(dtype).kind == "c" else 0)
  return x.astype(dtype)


def scipy_gmres(A, b, x0, tol, atol, m, maxiter):
  count = [0]

  def mv(v):
    count[0] += 1
    return A @ v
  op = spla.LinearOperator(A.shape, matvec=mv, dtype=A.dtype)
  x, info = spla.gmres(op, b, x0=x0, rtol=tol, atol=atol, restart=m, maxiter=maxiter)
  return x, info, count[0]


def run(A, b, x0=None, tol=1e-10, atol=None, m=20, maxiter=None, shape=None):
  """ours (through the driver, with its counts) and scipy's on the same problem; asserts what must agree"""
  shape = shape or b.shape
  Ad = be.convert_to_tensor(A)
  bd = be.convert_to_tensor(b.reshape(shape))
  x0d = None if x0 is None else be.convert_to_tensor(x0.reshape(shape))
  seen = set()

  def mv(x):
    seen.add(x.code)
    assert tuple(x.shape) == shape
    return be.reshape(be.tensordot(Ad, be.reshape(x, (A.shape[0],)), ([1], [0])), shape)
  x, info, st = tb_gmres.gmres(be, mv, bd, None, None, x0d, tol, atol, m, maxiter, None, return_info=True)
  assert seen <= {bd.code} and x.dtype == b.dtype and tuple(x.shape) == shape
  np.testing.assert_array_equal(bd.to_host(), b.reshape(shape))                # b untouched
  if x0 is not None:
    np.testing.assert_array_equal(x0d.to_host(), x0.reshape(shape))            # x0 untouched
  xs, sinfo, smv = scipy_gmres(A, b, x0, tol, tol if atol is None else atol, m, maxiter)
  xh = x.to_host().reshape(-1)
  assert info == sinfo, (info, sinfo, st)
  assert st["matvecs"] == smv, (st, smv)
  bn = np.linalg.norm(b)
  goal = max(tol if atol is None else atol, tol * bn)
  if info == 0:
    assert np.linalg.norm(b - A @ xh.astype(A.dtype)) <= goal * 1.0001 + 10 * np.finfo(b.dtype).eps * bn
  if bn > 0:
    cond = np.linalg.cond(A.astype(np.complex128))
    rel = np.linalg.norm(xh - xs) / max(np.linalg.norm(xs), np.finfo(b.dtype).tiny)
    assert rel <= 10 * max(tol, np.finfo(b.dtype).eps) * cond, (rel, cond)
  return xh, info, st


def shifted(n, dtype, shift=3.0):
  """shift I + G / sqrt(n): nonsymmetric, eigenvalues in the unit disc around `shift`"""
  return (shift * np.eye(n) + rand((n, n), dtype) / np.sqrt(2 * n if np.dtype(dtype).kind == "c" else n)).astype(dtype)


def indefinite(n, dtype):
  """eigenvalues in [-3, -1] and [1, 3], non-normal"""
  lam = np.concatenate([-rng.uniform(1, 3, n // 2), rng.uniform(1, 3, n - n // 2)])
  q = np.linalg.qr(rand((n, n), dtype))[0]
  t = np.diag(lam) + np.triu(rand((n, n), dtype), 1) * (0.3 / np.sqrt(n))
  return (q @ t @ q.conj().T).astype(dtype)


for dtype, tol in (("float64", 1e-10), ("complex128", 1e-10), ("float32", 1e-5), ("complex64", 1e-5)):
  n = 200
  A = shifted(n, dtype)
  b = rand(n, dtype)
  _, info, st = run(A, b, tol=tol, m=50)                          # one cycle
  assert info == 0 and st["cycles"] == 1, st
  _, info, st = run(A, b, tol=tol, m=4)                           # several restarts
  assert info == 0 and st["cycles"] >= 3, st
  _, info, st = run(A, b, tol=tol, m=3, maxiter=2)                # stops at maxiter
  assert info == 2 and st["cycles"] == 2, st
  Ai = indefinite(n, dtype)
  _, info, st = run(Ai, b, tol=tol, m=30, maxiter=200)            # indefinite: restarts
  assert info == 0, st
  _, info, st = run(A, b, tol=tol, m=20, shape=(10, 20))        # a tensor-shaped b
  assert info == 0
  print("dense", dtype, "ok")

# breakdown: b in an invariant subspace of dimension 3 < m: the exact solution after three steps
for dtype in ("float64", "complex128"):
  A = np.diag(np.arange(1.0, 41.0)).astype(dtype)
  b = np.zeros(40, dtype)
  b[[3, 17, 30]] = [1.0, -2.0, 0.5]
  x, info, st = run(A, b, tol=1e-14, atol=0.0, m=10, maxiter=5)
  assert info == 0 and st["cycles"] == 1 and st["matvecs"] == 4, st
  np.testing.assert_allclose(x, b / np.arange(1.0, 41.0), rtol=0, atol=1e-14)
print("breakdown ok")

# x0 given, x0 exact, b = 0, atol dominating tol
A = shifted(100, "float64")
b = rand(100, "float64")
x0 = rand(100, "float64")
_, info, st = run(A, b, x0=x0, m=10)
assert info == 0 and st["matvecs"] > 1, st
xe = np.linalg.solve(A, b)
x, info, st = run(A, b, x0=xe, m=10)
assert info == 0 and st["matvecs"] == 1 and st["cycles"] == 0, st
np.testing.assert_array_equal(x, xe)
x, info, st = run(A, np.zeros(100), x0=x0, m=10)
assert info == 0 and st["matvecs"] == 0 and not x.any(), st
x, info, st = run(A, b, tol=1e-12, atol=1e-3 * np.linalg.norm(b), m=10)
assert info == 0 and np.linalg.norm(b - A @ x) <= 1e-3 * np.linalg.norm(b)
_, info2, st2 = run(A, b, tol=1e-12, atol=0.0, m=10)
assert info2 == 0 and st2["matvecs"] > st["matvecs"], (st, st2)
print("x0 / b = 0 / atol ok")

# the backend method: defaults (num_krylov_vectors=20, maxiter=1), None meaning b.size, and A_args / A_kwargs
Ad = be.convert_to_tensor(A)
bd = be.convert_to_tensor(b)
x, info = be.gmres(lambda v, M, s=1.0: be.tensordot(M, v, ([1], [0])) * s, bd, A_args=[Ad], A_kwargs={"s": 1.0},
                   num_krylov_vectors=None)
assert isinstance(info, int) and info == 0
assert np.linalg.norm(b - A @ x.to_host()) <= 1e-5 * np.linalg.norm(b)
xs, sinfo, _ = scipy_gmres(A, b, None, 1e-5, 1e-5, 20, 1)
x, info = be.gmres(lambda v: be.tensordot(Ad, v, ([1], [0])), bd)
assert info == sinfo and isinstance(info, int)
np.testing.assert_allclose(x.to_host(), xs, rtol=0, atol=1e-8 * np.linalg.norm(xs))
print("backend method ok")


# errors
x = be.convert_to_tensor(np.ones(30))
mv = lambda v: v  # noqa: E731
raises(ValueError, lambda: be.gmres(mv, x, x0=be.convert_to_tensor(np.ones(31))))
raises(ValueError, lambda: be.gmres(mv, x, x0=be.convert_to_tensor(np.ones((5, 6)))))
raises(TypeError, lambda: be.gmres(mv, x, x0=be.convert_to_tensor(np.ones(30, np.float32))))
raises(ValueError, lambda: be.gmres(mv, x, num_krylov_vectors=0))
raises(ValueError, lambda: be.gmres(mv, x, num_krylov_vectors=-3))
raises(ValueError, lambda: be.gmres(mv, x, tol=-1e-5))
raises(ValueError, lambda: be.gmres(mv, x, atol=-1e-5))
raises(ValueError, lambda: be.gmres(mv, x, maxiter=0))
raises(NotImplementedError, lambda: be.gmres(mv, x, M=lambda v: v))
raises(NotImplementedError, lambda: be.gmres(mv, be.convert_to_tensor(np.ones(2000)), num_krylov_vectors=1025))
raises(NotImplementedError, lambda: be.gmres(mv, be.convert_to_tensor(np.ones(2000)), num_krylov_vectors=None))
raises(TypeError, lambda: be.gmres(mv, be.convert_to_tensor(np.ones(30, np.int64))))
raises(TypeError, lambda: be.gmres(mv, np.ones(30)))
raises(TypeError, lambda: be.gmres(lambda v: be.astype(v, np.complex128), x))
raises(TypeError, lambda: be.gmres(lambda v: v.to_host(), x))
raises(ValueError, lambda: be.gmres(lambda v: be.reshape(v, (5, 6)), x))
# clipped to b.size: 40 vectors on a 30-vector problem is a full Krylov space, converged in one cycle
y, info = be.gmres(lambda v: v * 2.0, x, num_krylov_vectors=40)
assert info == 0 and np.allclose(y.to_host(), 0.5)
print("errors ok")
hostrun.done(lib)
