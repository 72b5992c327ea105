"""Runs in a subprocess (build container only): CudaB200Backend.expm on a stand-in library whose tnb200_expm and
tnb200_lu_solve are scipy.linalg.expm and scipy.linalg.lu_solve on host memory, with the contracts of include/tnb200.h.
Checks the adapter: the numpy backend's errors, scipy's result dtypes, 0 x 0 and 1 x 1, strided views, and the
reference's tn.linalg.expm on backend="cuda_b200" against backend="numpy".  The kernels are checked by
tests/test_gpu_expm.py."""
import numpy as np
import scipy.linalg
import hostrun
from hostrun import raises
tn, lib = hostrun.install(reference=None)
from tensornetwork_b200 import _lib, backend as tb_backend  # noqa: E402
be = tb_backend.CudaB200Backend()
rng = np.random.default_rng(3)


# errors: the numpy backend's ValueErrors and messages
raises(ValueError, be.expm, be.convert_to_tensor(np.ones((2, 2, 2))), match="Only matrices are supported")
raises(ValueError, be.expm, be.convert_to_tensor(np.ones(3)), match="Only matrices are supported")
raises(ValueError, be.expm, be.convert_to_tensor(np.ones((4, 3))), match="N*N matrix, 4*3 matrix is given")

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
c0 = lib.calls["tnb200_expm"]
z = be.expm(be.convert_to_tensor(np.zeros((0, 0), dtype=np.int64)))
assert z.shape == (0, 0) and z.dtype == np.int64
one = be.expm(be.convert_to_tensor(np.array([[0.25]])))
assert lib.calls["tnb200_expm"] == c0 and np.allclose(one.to_host(), [[np.exp(0.25)]])

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
hostrun.done(lib)
