"""Runs in a subprocess (build container only): CudaB200Backend.expm on a stand-in library whose tnb200_expm and
tnb200_lu_solve are scipy.linalg.expm and scipy.linalg.lu_solve on host memory, with the contracts of include/tnb200.h.
Checks the adapter: the numpy backend's errors, scipy's result dtypes, 0 x 0 and 1 x 1, strided views, and the
reference's tn.linalg.expm on backend="cuda_b200" against backend="numpy".  The kernels are checked by
tests/test_gpu_expm.py."""
import ctypes
import os
import sys
import numpy as np
import scipy.linalg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from baseline import refenv  # noqa: E402
tn = refenv.try_load()
from tensornetwork_b200 import _lib, backend as tb_backend  # noqa: E402
import fake_lib  # noqa: E402
import expm_rule  # noqa: E402


class ExpmFakeLib(fake_lib.FakeLib):
  """FakeLib plus tnb200_expm and tnb200_lu_solve."""

  def __init__(self):
    super().__init__()
    self.expm_calls = 0

  def tnb200_expm(self, a, x, info_ptr, stream):
    A, X = fake_lib._view(a), fake_lib._view(x)
    if A.ndim != 2 or A.shape[0] != A.shape[1]:
      return self._fail(_lib.ERR_INVALID, "expm: the matrix must be square")
    if A.dtype not in (np.float64, np.float32, np.complex64, np.complex128):
      return self._fail(_lib.ERR_DTYPE, "expm: dtype not supported")
    self.expm_calls += 1
    n = A.shape[0]
    if n == 0:
      return 0
    wide = A.astype(np.complex128 if np.iscomplexobj(A) else np.float64)
    finite = np.isfinite(wide).all()
    X[...] = scipy.linalg.expm(wide) if finite else np.nan
    if info_ptr:
      m, s = expm_rule.select(wide) if finite and n > 1 else (0, 0)
      info = np.ndarray((4,), dtype=np.int32, buffer=(ctypes.c_char * 16).from_address(info_ptr))
      info[...] = (m, s, 0 if n <= _lib.EXPM_FUSED_MAX_N else 1, 0)
    self._launches += 1
    return 0

  def tnb200_lu_solve(self, lu, piv_ptr, b, x, stream):
    LU, B, X = fake_lib._view(lu), fake_lib._view(b), fake_lib._view(x)
    n = LU.shape[0]
    piv = np.ndarray((n,), dtype=np.int32, buffer=(ctypes.c_char * (4 * max(n, 1))).from_address(piv_ptr))
    X[...] = scipy.linalg.lu_solve((LU, piv), B)
    return 0


lib = ExpmFakeLib()
_lib.set_lib(lib)
tb_backend._CONFIG["device"] = "cpu"
be = tb_backend.CudaB200Backend()
if tn is not None:
  tb_backend.register()
rng = np.random.default_rng(3)


def expect_raises(exc, match, f, *args):
  try:
    f(*args)
  except exc as e:
    assert match in str(e), str(e)
    return
  raise AssertionError("no {} raised".format(exc.__name__))


# errors: the numpy backend's ValueErrors and messages
expect_raises(ValueError, "Only matrices are supported", be.expm, be.convert_to_tensor(np.ones((2, 2, 2))))
expect_raises(ValueError, "Only matrices are supported", be.expm, be.convert_to_tensor(np.ones(3)))
expect_raises(ValueError, "N*N matrix, 4*3 matrix is given", be.expm, be.convert_to_tensor(np.ones((4, 3))))

# result dtypes, as scipy.linalg.expm returns them (bool via the index_update mask path needs the device: not here)
for dt, out in ((np.float64, np.float64), (np.float32, np.float32), (np.complex64, np.complex64),
                (np.complex128, np.complex128), (np.int32, np.float64), (np.int64, np.float64),
                (np.float16, np.float32)):
  for n in (1, 2, 5, _lib.EXPM_FUSED_MAX_N + 1):
    a = (rng.standard_normal((n, n)) * 2).astype(dt) if np.dtype(dt).kind != "c" else \
        (rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))).astype(dt)
    r = be.expm(be.convert_to_tensor(a))
    assert r.dtype == np.dtype(out), (dt, n, r.dtype)
    ref = scipy.linalg.expm(a.astype(np.complex128 if np.dtype(dt).kind == "c" else np.float64))
    tol = 1e-12 if np.dtype(out).itemsize >= 8 and out != np.complex64 else 1e-5
    assert np.linalg.norm(r.to_host() - ref) <= tol * np.linalg.norm(ref), (dt, n)

# 0 x 0 keeps the dtype and calls nothing; 1 x 1 is the elementwise exp
c0 = lib.expm_calls
z = be.expm(be.convert_to_tensor(np.zeros((0, 0), dtype=np.int64)))
assert z.shape == (0, 0) and z.dtype == np.int64
one = be.expm(be.convert_to_tensor(np.array([[0.25]])))
assert lib.expm_calls == c0 and np.allclose(one.to_host(), [[np.exp(0.25)]])

# strided views: transposed and sliced
big = rng.standard_normal((12, 12))
t = be.convert_to_tensor(big)
np.testing.assert_allclose(be.expm(be.transpose(t)).to_host(), scipy.linalg.expm(big.T), rtol=1e-13)
np.testing.assert_allclose(be.expm(be.slice(t, (2, 3), (5, 5))).to_host(), scipy.linalg.expm(big[2:7, 3:8]),
                           rtol=1e-13)

# non-finite input: all NaN
bad = np.eye(3)
bad[1, 2] = np.inf
assert np.isnan(be.expm(be.convert_to_tensor(bad)).to_host()).all()

# the reference's entry point on backend="cuda_b200" against backend="numpy"
if tn is not None:
  for dt in (np.float64, np.complex128):
    a = rng.standard_normal((6, 6)).astype(dt) / 3
    ours = tn.linalg.linalg.expm(tn.Tensor(be.convert_to_tensor(a), backend="cuda_b200"))
    theirs = tn.linalg.linalg.expm(tn.Tensor(a, backend="numpy"))
    np.testing.assert_allclose(ours.array.to_host(), theirs.array, rtol=1e-13)
    eye = tn.eye(6, backend="cuda_b200", dtype=dt)
    np.testing.assert_allclose(tn.linalg.linalg.expm(eye).array.to_host(),
                               tn.linalg.linalg.expm(tn.eye(6, backend="numpy", dtype=dt)).array)
print("EXPM HOST OK")
