"""Runs in a subprocess (build container only): the host driver of CudaB200Backend.eigs (tensornetwork_b200/arnoldi.py)
on a stand-in library whose tnb200_arnoldi_orth is a plain numpy CGS2 on host memory.  Checks restarts, conjugate
pairs, breakdown, every `which`, the errors and the statistics against np.linalg.eig; the kernel itself is checked by
tests/test_gpu_eigs.py."""
import numpy as np
import hostrun
from hostrun import raises
_, lib = hostrun.install()
from tensornetwork_b200 import backend as tb_backend, arnoldi  # noqa: E402

be = tb_backend.CudaB200Backend()

WHICH = ("LM", "SM", "LR", "SR")


def key(vals, which):
  """best first; members of a conjugate pair tie (their keys agree to rounding), and Im > 0 comes first"""
  k = {"LM": -np.abs(vals), "SM": np.abs(vals), "LR": -vals.real, "SR": vals.real}[which]
  return np.lexsort((-vals.imag, np.round(k / np.abs(vals).max(), 10)))


def from_spectrum(rng, lam, dtype, normal=True):
  """a matrix with eigenvalues lam: Q diag Q^H (normal) or Q (diag + strict upper triangle) Q^H (non-normal)"""
  n = len(lam)
  cplx = np.dtype(dtype).kind == "c"
  x = rng.standard_normal((n, n)) + (1j * rng.standard_normal((n, n)) if cplx else 0)
  q = np.linalg.qr(x)[0]
  t = np.diag(lam).astype(np.complex128 if cplx else np.float64)
  if not normal:
    t = t + np.triu(rng.standard_normal((n, n)), 1) * (0.5 / np.sqrt(n))     # well-conditioned eigenvalues
  return (q @ t @ q.conj().T).astype(dtype)


def run(M, which, numeig, ncv, tol, x0=None, maxiter=None, seed=0):
  Md = be.convert_to_tensor(M)
  seen = []

  def mv(x):
    seen.append(x.code)
    return be.tensordot(Md, x, ([1], [0]))
  if x0 is None:
    x0 = np.random.default_rng(seed).standard_normal(M.shape[0]).astype(M.dtype)
  x0d = be.convert_to_tensor(x0)
  eta, vecs, info = arnoldi.eigs(be, mv, [], x0d, None, None, ncv, numeig, tol, which, maxiter, return_info=True)
  np.testing.assert_array_equal(x0d.to_host(), x0)              # initial_state untouched
  assert all(c == x0d.code for c in seen)                      # the matvec never sees another dtype
  return eta.to_host(), [v.to_host() for v in vecs], info


def check(M, which, numeig, ncv=None, tol=1e-12, rtol=1e-9, **kw):
  n = M.shape[0]
  ncv = ncv or min(n, max(2 * numeig + 10, 20))
  lam, vecs, info = run(M, which, numeig, ncv, tol, **kw)
  single = M.dtype in (np.float32, np.complex64)
  assert lam.dtype == (np.complex64 if single else np.complex128), lam.dtype
  ref = np.linalg.eig(M.astype(np.complex128))[0]
  ref = ref[key(ref, which)][:numeig]
  scale = np.abs(ref).max()
  np.testing.assert_allclose(lam, ref, rtol=0, atol=rtol * scale)
  for l, v in zip(lam, vecs):
    assert v.shape == (n,) and v.dtype == lam.dtype
    v = v.astype(np.complex128)
    assert abs(np.linalg.norm(v) - 1) < 10 * rtol
    assert np.linalg.norm(M @ v - l * v) <= 100 * rtol * scale, np.linalg.norm(M @ v - l * v)
  assert info["nconv"] >= numeig and info["matvecs"] >= ncv
  return lam, vecs, info


rng = np.random.default_rng(1)
n = 200
gaps = np.concatenate([[10.0, 9.0, -8.5, 8.0, 7.0, 6.0 + 0j, -6.8], rng.uniform(-3, 3, n - 7)])
for dtype, tol, rtol in (("float64", 1e-12, 1e-9), ("complex128", 1e-12, 1e-9), ("float32", 1e-5, 1e-4), ("complex64", 1e-5, 1e-4)):
  for normal in (True, False):
    M = from_spectrum(rng, gaps.real, dtype, normal)
    for which in WHICH:
      for numeig in (1, 3, 6):
        if which == "SM":                                      # the small end: spread it so it converges
          lam = np.concatenate([[0.01, 0.02, -0.03, 0.045, 0.06, 0.075, -0.09], rng.uniform(1.0, 3.0, n - 7)])
          Ms = from_spectrum(rng, lam, dtype, normal)
          check(Ms, which, numeig, ncv=60, tol=tol, rtol=rtol)
        else:
          check(M, which, numeig, tol=tol, rtol=rtol)
  print("dense", dtype, "ok")

# restarts actually happen on a slowly converging case; maxiter=1 there is a RuntimeError naming nconv
M = from_spectrum(rng, np.concatenate([[1.0, 0.99], rng.uniform(-0.9, 0.9, 498)]), "float64")
_, _, info = check(M, "LR", 1, ncv=8)
assert info["restarts"] >= 2, info
assert info["host_reads"] >= info["matvecs"], info
raises(RuntimeError, lambda: run(M, "LR", 1, 8, 1e-12, maxiter=1), match="converged")
print("restarts ok", info)

# a real operator with complex eigenvalues: rotation blocks in a random real basis
for numeig in (1, 2):
  blocks = [(2.0, 1.0), (1.5, 0.5), (0.5, 0.2)]
  d = np.zeros((60, 60))
  for b, (r, im) in enumerate(blocks):
    d[2 * b:2 * b + 2, 2 * b:2 * b + 2] = [[r, -im], [im, r]]
  d[6:, 6:] = np.diag(rng.uniform(-0.5, 0.5, 54))
  q = np.linalg.qr(rng.standard_normal((60, 60)))[0]
  M = q @ d @ q.T
  lam, vecs, _ = check(M, "LM", numeig, ncv=20)
  assert lam[0].imag > 0
  if numeig == 2:
    assert lam[1] == np.conj(lam[0])
# a real dominant eigenvalue of a real operator: exactly real value and vector
M = from_spectrum(rng, np.concatenate([[5.0], rng.uniform(-1, 1, 79)]), "float64", normal=False)
lam, vecs, _ = check(M, "LR", 1, ncv=20)
assert lam[0].imag == 0.0 and np.all(vecs[0].imag == 0.0)
print("real operators ok")

# breakdown: an invariant subspace (three nonzero entries of a diagonal operator) smaller than num_krylov_vecs
for dtype in ("float64", "complex128"):
  M = np.diag(np.arange(1.0, 41.0)).astype(dtype)
  x0 = np.zeros(40, dtype)
  x0[[3, 17, 30]] = 1.0
  lam, vecs, info = run(M, "LR", 2, 10, 1e-12, x0=x0)
  assert np.all(np.isfinite(lam)) and all(np.all(np.isfinite(v)) for v in vecs)
  np.testing.assert_allclose(lam, [31.0, 18.0], rtol=1e-12)          # the invariant subspace's eigenpairs
  for l, v in zip(lam, vecs):
    assert np.linalg.norm(M @ v - l * v) < 1e-10
  assert info["matvecs"] == 3 and info["restarts"] == 0, info
  # more eigenpairs than the invariant subspace holds: continues from a random vector, still exact eigenpairs
  lam, vecs, info = run(M, "LR", 5, 30, 1e-12, x0=x0)
  assert np.all(np.isfinite(lam))
  for l, v in zip(lam, vecs):
    assert np.linalg.norm(M @ v - l * v) < 1e-9 * 40
print("breakdown ok")

# errors (numpy backend / scipy conventions)
x = be.convert_to_tensor(np.ones(30))
mv = lambda v: v  # noqa: E731

raises(ValueError, lambda: be.eigs(mv, initial_state=x, which="LI"))
raises(ValueError, lambda: be.eigs(mv, initial_state=x, which="SI"))
raises(ValueError, lambda: be.eigs(mv, initial_state=x, numeig=5, num_krylov_vecs=6))
raises(ValueError, lambda: be.eigs(mv))
raises(ValueError, lambda: be.eigs(mv, initial_state=x, numeig=2, num_krylov_vecs=31))
raises(TypeError, lambda: be.eigs(mv, initial_state=x, numeig=29, num_krylov_vecs=31))
raises(TypeError, lambda: be.eigs(mv, initial_state=np.ones(30), num_krylov_vecs=10))
raises(TypeError, lambda: be.eigs(mv, initial_state=be.convert_to_tensor(np.ones(30, np.int64)), num_krylov_vecs=10))
raises(ValueError, lambda: be.eigs(lambda v: be.reshape(v, (5, 6)), initial_state=x, numeig=1, num_krylov_vecs=10))
raises(ValueError, lambda: be.eigs(mv, initial_state=be.convert_to_tensor(np.zeros(30)), numeig=1, num_krylov_vecs=10))
# shape / dtype instead of initial_state
eta, vecs = be.eigs(lambda v: v * 2.0, shape=(6, 5), dtype=np.float64, numeig=1, num_krylov_vecs=10)
assert vecs[0].shape == (6, 5) and abs(eta.to_host()[0] - 2.0) < 1e-12
print("errors ok")
hostrun.done(lib)
