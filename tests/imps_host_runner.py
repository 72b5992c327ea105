"""Runs in a subprocess (build container only): the reference's own InfiniteMPS.canonicalize on backend="cuda_b200",
on the stand-in library tests/fake_lib.FakeLib, whose tnb200_eigh, tnb200_arnoldi_orth, tnb200_compare,
tnb200_index_update, tnb200_lu_factor and tnb200_inv are numpy versions with the contracts of include/tnb200.h.  Checks
the adapter's host logic against backend="numpy": canonicalize's results, the comparison / index_update semantics and
inv's errors.  The kernels themselves are checked by tests/test_gpu_inv.py and tests/test_gpu_canonicalize.py."""
import numpy as np
import hostrun
from hostrun import raises
tn, lib = hostrun.install(reference=True)
from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS  # noqa: E402
from tensornetwork_b200 import backend as tb_backend  # noqa: E402
from tensornetwork_b200.tensor import B200Tensor  # noqa: E402
be = tb_backend.get_instance()


def schmidt(connector):
  return np.sort(np.abs(np.diag(np.linalg.inv(np.asarray(connector)))))


# ---------------------------------------------------------------- 1. canonicalize against the numpy backend
for dtype in (np.float64, np.complex128):
  for D in (1, 8, 16):
    np.random.seed(D)
    ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=dtype, backend="numpy")
    mps = InfiniteMPS(tensors=[np.asarray(t) for t in ref.tensors], center_position=0, backend="cuda_b200")
    a = ref.canonicalize()
    b = mps.canonicalize()
    assert isinstance(b, B200Tensor) and b.shape == (), b
    assert abs(complex(b.item()) - complex(a)) <= 1e-12 * abs(complex(a)), (a, b.item())
    sa, sb = schmidt(ref.connector_matrix), schmidt(mps.connector_matrix)
    assert sa.shape == sb.shape and np.max(np.abs(sa - sb)) <= 1e-12 * np.max(sa), (sa, sb)
    assert [np.asarray(t).dtype for t in mps.tensors] == [np.asarray(t).dtype for t in ref.tensors]
    assert mps.connector_matrix.dtype == np.asarray(ref.connector_matrix).dtype
    assert b.dtype == np.asarray(a).dtype, (b.dtype, np.asarray(a).dtype)
    print("canonicalize", dtype.__name__, D, "ok")

# ---------------------------------------------------------------- 2. comparisons
x = be.convert_to_tensor(np.array([0.5, -1.0, 2.0, np.nan]))
one = be.convert_to_tensor(np.array([0.25]))
r = one <= 0.3                                                 # one element vs a host scalar: a host bool, as before
assert r is True
assert (one < be.convert_to_tensor(np.array(0.5))) is True
r = be.convert_to_tensor(np.array(3.0)) >= np.float64(3.0)
assert isinstance(r, (bool, np.bool_)) and r
for op, ref_op in ((x.__lt__, np.less), (x.__le__, np.less_equal), (x.__gt__, np.greater), (x.__ge__, np.greater_equal)):
  m = op(0.5)
  assert isinstance(m, B200Tensor) and m.dtype == np.dtype(bool) and m.shape == (4,)
  with np.errstate(invalid="ignore"):
    np.testing.assert_array_equal(np.asarray(m), ref_op(np.array([0.5, -1.0, 2.0, np.nan]), 0.5))
# broadcasting against a tensor, and a one-element tensor against a larger one compares on the device
col = be.convert_to_tensor(np.arange(3.0).reshape(3, 1))
row = be.convert_to_tensor(np.arange(4.0).reshape(1, 4))
np.testing.assert_array_equal(np.asarray(col < row), np.arange(3.0).reshape(3, 1) < np.arange(4.0).reshape(1, 4))
np.testing.assert_array_equal(np.asarray(one < x), 0.25 < np.array([0.5, -1.0, 2.0, np.nan]))
# promotion: an integer tensor against a float scalar compares in float
xi = be.convert_to_tensor(np.array([1, 2, 3], np.int64))
np.testing.assert_array_equal(np.asarray(xi > 1.5), [False, True, True])
raises(TypeError, lambda: be.convert_to_tensor(np.array([1j, 2.0])) < 1.0)
# a host bool array round-trips
hb = be.convert_to_tensor(np.array([True, False, True]))
assert hb.dtype == np.dtype(bool)
np.testing.assert_array_equal(np.asarray(hb), [True, False, True])
print("compare ok")

# ---------------------------------------------------------------- 3. index_update
h = np.arange(12.0).reshape(3, 4) - 5.0
t = be.convert_to_tensor(h)


def np_update(arr, mask, v):
  out = np.copy(arr)
  out[mask] = v
  return out


for mask in (True, False, np.bool_(True), np.bool_(False), np.array(True),
             h > 0, np.array([True, False, True]), np.array([[True] * 4, [False] * 4, [True, False] * 2])):
  out = be.index_update(t, mask, 7.5)
  assert out is not t and out.shape == t.shape and out.dtype == t.dtype
  np.testing.assert_array_equal(np.asarray(out), np_update(h, mask, 7.5))
np.testing.assert_array_equal(np.asarray(t), h)                # the input is untouched
dmask = t > 0.0                                                # a device mask, and a device prefix mask
np.testing.assert_array_equal(np.asarray(be.index_update(t, dmask, -1.0)), np_update(h, h > 0, -1.0))
pmask = be.convert_to_tensor(np.array([1.0, -1.0, 1.0])) > 0.0
np.testing.assert_array_equal(np.asarray(be.index_update(t, pmask, 0.0)), np_update(h, np.array([True, False, True]), 0.0))
# assignee forms and casting
dev = be.convert_to_tensor(np.array(3.25))
np.testing.assert_array_equal(np.asarray(be.index_update(t, h > 0, dev)), np_update(h, h > 0, 3.25))
np.testing.assert_array_equal(np.asarray(be.index_update(t, h > 0, np.float32(2.5))), np_update(h, h > 0, 2.5))
ti = be.convert_to_tensor(np.arange(6, dtype=np.int64))
mi = np.array([True, False, True, False, True, False])
for v in (2.7, -2.7, np.float64(9.9), 4, True):
  out = be.index_update(ti, mi, v)
  assert out.dtype == np.int64
  np.testing.assert_array_equal(np.asarray(out), np_update(np.arange(6, dtype=np.int64), mi, v))
np.testing.assert_array_equal(np.asarray(be.index_update(ti, mi, be.convert_to_tensor(np.array(-3.9)))),
                              np_update(np.arange(6, dtype=np.int64), mi, -3.9))
tc = be.convert_to_tensor(h.astype(np.complex128))
np.testing.assert_array_equal(np.asarray(be.index_update(tc, h > 0, 1 + 2j)), np_update(h.astype(np.complex128), h > 0, 1 + 2j))
raises(TypeError, lambda: be.index_update(t, h > 0, 1j))
raises(TypeError, lambda: be.index_update(t, h > 0, be.convert_to_tensor(np.array(1j))))
raises(IndexError, lambda: be.index_update(t, np.array([True, False]), 0.0))
raises(IndexError, lambda: be.index_update(t, np.ones((4, 3), bool), 0.0))
raises(IndexError, lambda: be.index_update(t, np.array([0, 1]), 0.0))
raises(IndexError, lambda: be.index_update(t, t, 0.0))
raises(NotImplementedError, lambda: be.index_update(t, h > 0, np.arange(5.0)))
for v in (2**62 + 1, -(2**62) - 3, np.int64(2**60 + 7)):               # integers beyond 2^53 stay exact
  np.testing.assert_array_equal(np.asarray(be.index_update(ti, mi, v)), np_update(np.arange(6, dtype=np.int64), mi, v))
t32 = be.convert_to_tensor(np.arange(6, dtype=np.int32))
raises(OverflowError, lambda: be.index_update(t32, mi, 2**40))
np.testing.assert_array_equal(np.asarray(be.index_update(t32, mi, np.int64(2**40 + 5))),
                              np_update(np.arange(6, dtype=np.int32), mi, np.int64(2**40 + 5)))
raises(NotImplementedError, lambda: be.index_update(t, h > 0, be.convert_to_tensor(np.arange(5.0))))
print("index_update ok")

# ---------------------------------------------------------------- 4. inv
rng = np.random.default_rng(3)
for dtype in (np.float64, np.complex128, np.float32, np.complex64):
  m = rng.standard_normal((6, 6)) + (1j * rng.standard_normal((6, 6)) if np.dtype(dtype).kind == "c" else 0)
  m = m.astype(dtype)
  xi = be.inv(be.convert_to_tensor(m))
  assert xi.dtype == np.dtype(dtype)
  np.testing.assert_allclose(np.asarray(xi), np.linalg.inv(m), rtol=1e-4 if dtype in (np.float32, np.complex64) else 1e-10)
xi = be.inv(be.convert_to_tensor(np.array([[2, 1], [1, 1]], np.int64)))
assert xi.dtype == np.float64
np.testing.assert_allclose(np.asarray(xi), [[1, -1], [-1, 2]])
assert be.inv(be.convert_to_tensor(np.zeros((0, 0)))).shape == (0, 0)
raises(ValueError, lambda: be.inv(be.convert_to_tensor(np.ones((2, 2, 2)))))
raises(np.linalg.LinAlgError, lambda: be.inv(be.convert_to_tensor(np.ones(3))))
raises(np.linalg.LinAlgError, lambda: be.inv(be.convert_to_tensor(np.ones((2, 3)))))
raises(TypeError, lambda: be.inv(be.convert_to_tensor(np.eye(2, dtype=np.float16))))
raises(np.linalg.LinAlgError, lambda: be.inv(be.convert_to_tensor(np.ones((3, 3)))))
# tn.linalg.inv on a tn.Tensor
from tensornetwork.linalg import linalg as tn_linalg  # noqa: E402
m = rng.standard_normal((5, 5))
out = tn_linalg.inv(tn.Tensor(be.convert_to_tensor(m), backend="cuda_b200"))
np.testing.assert_allclose(np.asarray(out.array), np.linalg.inv(m), rtol=1e-10)
print("inv ok")
hostrun.done(lib)
