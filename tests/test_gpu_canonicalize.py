"""GPU: the pieces InfiniteMPS.canonicalize needs beyond the eigensolvers — comparison masks (tnb200_compare),
index_update (tnb200_index_update), inv — and the reference's own canonicalize against its numpy backend."""
import numpy as np
import pytest
from util import get_backend

pytestmark = pytest.mark.gpu

OPS = {"lt": np.less, "le": np.less_equal, "gt": np.greater, "ge": np.greater_equal}
CMP_DTYPES = ["float64", "float32", "float16", "bfloat16", "int32", "int64"]


def _dev(be, host, dtype):
  if dtype == "bfloat16":
    return be.astype(be.convert_to_tensor(host.astype(np.float32)), "bfloat16")
  return be.convert_to_tensor(host.astype(dtype))


@pytest.mark.parametrize("op", sorted(OPS))
@pytest.mark.parametrize("dtype", CMP_DTYPES)
def test_compare(dtype, op):
  from tensornetwork_b200 import _lib as L
  be = get_backend()
  code = {"lt": L.LT, "le": L.LE, "gt": L.GT, "ge": L.GE}[op]
  rng = np.random.default_rng(1)
  a = rng.integers(-3, 4, (5, 1, 7)).astype(np.float64)
  b = rng.integers(-3, 4, (1, 6, 7)).astype(np.float64)
  if dtype not in ("int32", "int64"):
    a = a + 0.5 * rng.integers(0, 2, a.shape)
    a[0, 0, :3] = np.nan
    b[0, 1, 2] = np.nan
  ad, bd = _dev(be, a, dtype), _dev(be, b, dtype)
  ah, bh = ad.to_host().astype(np.float64), bd.to_host().astype(np.float64)   # the values as stored
  m = be.compare(code, ad, bd)                                               # broadcast (5,1,7) x (1,6,7)
  assert m.shape == (5, 6, 7) and m.dtype == np.dtype(bool)
  with np.errstate(invalid="ignore"):
    np.testing.assert_array_equal(m.to_host(), OPS[op](ah, bh))
    # the operators: a multi-element tensor against a scalar, and a transposed (strided) view
    m = getattr(ad, "__{}__".format(op))(0.5 if dtype not in ("int32", "int64") else 1)
    np.testing.assert_array_equal(m.to_host(), OPS[op](ah, 0.5 if dtype not in ("int32", "int64") else 1))
    t = be.transpose(ad, (2, 1, 0))
    np.testing.assert_array_equal(np.asarray(be.compare(code, t, t)), OPS[op](ah.transpose(2, 1, 0), ah.transpose(2, 1, 0)))


def test_compare_int64_is_exact_and_complex_refused():
  from tensornetwork_b200 import _lib as L
  be = get_backend()
  big = np.array([2**62, 2**62 + 1, -2**62], np.int64)
  x, y = be.convert_to_tensor(big), be.convert_to_tensor(np.array([2**62 + 1] * 3, np.int64))
  np.testing.assert_array_equal(be.compare(L.LT, x, y).to_host(), big < 2**62 + 1)
  with pytest.raises(TypeError):
    be.convert_to_tensor(np.array([1j, 2.0])) < 1.0
  one = be.convert_to_tensor(np.array([0.25]))
  assert (one < 0.5) is True                      # the one-element host comparison is unchanged


IU_DTYPES = ["float64", "float32", "float16", "bfloat16", "complex64", "complex128", "int32", "int64"]


@pytest.mark.parametrize("dtype", IU_DTYPES)
def test_index_update(dtype):
  be = get_backend()
  rng = np.random.default_rng(2)
  h = rng.integers(-5, 6, (4, 3, 5)).astype(np.float64)
  t = _dev(be, h, dtype)
  hv = t.to_host()
  masks = [True, False, np.bool_(True), h[:, :, 0] > 0, h > 0, np.array([True, False, True, False])]
  for mask in masks:
    out = be.index_update(t, mask, 2.75)
    ref = np.copy(hv)
    ref[mask] = 2.75 if dtype not in ("int32", "int64") else 2
    assert out.shape == t.shape and out.dtype == t.dtype
    np.testing.assert_array_equal(out.to_host(), ref)
  np.testing.assert_array_equal(t.to_host(), hv)                   # untouched
  dmask = be.convert_to_tensor(h) > 0.0                             # a device mask and a device-scalar assignee
  val = be.convert_to_tensor(np.array(-1.5))
  ref = np.copy(hv)
  ref[h > 0] = -1.5 if dtype not in ("int32", "int64") else -1
  np.testing.assert_array_equal(be.index_update(t, dmask, val).to_host(), ref)
  if np.dtype(dtype if dtype != "bfloat16" else "float32").kind != "c":
    with pytest.raises(TypeError):
      be.index_update(t, dmask, 1j)
  else:
    ref = np.copy(hv)
    ref[h > 0] = 1 - 2j
    np.testing.assert_array_equal(be.index_update(t, dmask, be.convert_to_tensor(np.array(1 - 2j))).to_host(), ref)
  with pytest.raises(IndexError):
    be.index_update(t, np.ones((3, 4), bool), 0.0)
  with pytest.raises(NotImplementedError):
    be.index_update(t, dmask, np.arange(3.0))


def test_index_update_integers_are_exact():
  """integers beyond 2^53 (which a double rounds) are stored exactly, as numpy stores them"""
  be = get_backend()
  h = np.arange(4, dtype=np.int64)
  m = np.array([True, False, True, False])
  t = be.convert_to_tensor(h)
  for v in (2**62 + 1, -(2**62) - 3, np.int64(2**60 + 7), 2**53 + 1):
    ref = np.copy(h)
    ref[m] = v
    np.testing.assert_array_equal(be.index_update(t, m, v).to_host(), ref)
  dv = be.convert_to_tensor(np.array(2**62 + 1, np.int64))                   # a device int64 scalar, too
  ref = np.copy(h)
  ref[m] = 2**62 + 1
  np.testing.assert_array_equal(be.index_update(t, m, dv).to_host(), ref)
  t32 = be.convert_to_tensor(h.astype(np.int32))
  with pytest.raises(OverflowError):
    be.index_update(t32, m, 2**40)
  ref = h.astype(np.int32)
  ref[m] = np.int64(2**40 + 5)                                                # a numpy integer wraps, as in numpy
  np.testing.assert_array_equal(be.index_update(t32, m, np.int64(2**40 + 5)).to_host(), ref)


def test_mask_and_index_update_replay_in_a_captured_graph():
  """mask made on the device, index_update with a device-scalar assignee: no host sync, so jit captures and replays"""
  be = get_backend()
  rng = np.random.default_rng(3)
  x = be.convert_to_tensor(rng.standard_normal(1000))
  s = be.convert_to_tensor(np.array(9.0))

  def f(v, val):
    mask = v <= 0.0
    w = be.index_update(v, mask, val)
    return be.index_update(1.0 / w, mask, 0.0)
  jf = be.jit(f, static_argnums=())
  st0 = dict(be.jit_stats)
  for _ in range(4):
    xh = rng.standard_normal(1000)
    x = be.convert_to_tensor(xh)
    out = jf(x, s).to_host()
    ref = np.where(xh <= 0.0, 0.0, 1.0 / np.where(xh <= 0.0, 9.0, xh))
    np.testing.assert_allclose(out, ref, rtol=1e-15)
  assert be.jit_stats["captures"] - st0["captures"] == 1
  assert be.jit_stats["replays"] - st0["replays"] >= 2
  assert be.jit_stats["capture_failures"] == st0["capture_failures"]


# ---------------------------------------------------------------- the reference's canonicalize
def _schmidt(c):
  return np.sort(np.abs(np.diag(np.linalg.inv(np.asarray(c)))))


def _check_canonical(mps, ref, lam, ref_lam, tol=1e-9):
  assert abs(complex(lam.item()) - complex(ref_lam)) <= tol * abs(complex(ref_lam))
  sa, sb = _schmidt(ref.connector_matrix), _schmidt(mps.connector_matrix)
  assert sa.shape == sb.shape, (sa.shape, sb.shape)
  assert np.max(np.abs(sa - sb)) <= tol * np.max(sa)
  for i, t in enumerate(mps.tensors):
    if i == mps.center_position:
      continue
    a = np.asarray(t)
    g = np.einsum("lsr,lsq->rq", a.conj(), a)
    assert np.max(np.abs(g - np.eye(g.shape[0]))) <= 1e-10, i
  # the dominant eigenvalue of the canonical state's unit-cell transfer matrix.  The reference leaves lam_norm in the
  # state (canonicalize returns it instead of dividing it out), so the value is not 1: it is compared with the value
  # the numpy backend finds for its own canonical state.
  d = np.asarray(mps.connector_matrix).shape[0]
  ncv = min(30, d * d)
  eta, _ = mps.transfer_matrix_eigs("l", num_krylov_vecs=ncv)
  ref_eta, _ = ref.transfer_matrix_eigs("l", num_krylov_vecs=ncv)
  assert abs(complex(eta.item()) - complex(ref_eta)) <= tol * abs(complex(ref_eta))


@pytest.mark.parametrize("D", [1, 8, 64, 256])
@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_canonicalize(tn, dtype, D):
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import  (registers "cuda_b200")
  from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS
  np.random.seed(D)
  ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=dtype, backend="numpy")
  mps = InfiniteMPS(tensors=[np.asarray(t) for t in ref.tensors], center_position=0, backend="cuda_b200")
  ref_lam = ref.canonicalize(precision=1e-10)
  lam = mps.canonicalize(precision=1e-10)
  assert [t.dtype for t in mps.tensors] == [np.asarray(t).dtype for t in ref.tensors]
  _check_canonical(mps, ref, lam, ref_lam)


def test_canonicalize_rank_deficient(tn):
  """D = 8 tensors that are D = 4 tensors padded with zeros: the masks select entries and the boundary truncation
  keeps the same bond dimension as numpy"""
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import
  from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS
  np.random.seed(4)
  small = InfiniteMPS.random(d=[2, 2], D=[4] * 3, dtype=np.float64, backend="numpy")
  padded = []
  for t in small.tensors:
    p = np.zeros((8, 2, 8))
    p[:4, :, :4] = np.asarray(t)
    padded.append(p)
  ref = InfiniteMPS(tensors=[p.copy() for p in padded], center_position=0, backend="numpy")
  mps = InfiniteMPS(tensors=[p.copy() for p in padded], center_position=0, backend="cuda_b200")
  ref_lam = ref.canonicalize(precision=1e-10)
  lam = mps.canonicalize(precision=1e-10)
  assert np.asarray(mps.connector_matrix).shape == np.asarray(ref.connector_matrix).shape
  assert np.asarray(ref.connector_matrix).shape[0] < 8                     # the truncation did cut
  assert [tuple(t.shape) for t in mps.tensors] == [np.asarray(t).shape for t in ref.tensors]
  _check_canonical(mps, ref, lam, ref_lam)


def test_tn_linalg_inv(tn):
  import tensornetwork_b200  # noqa: F401  pylint: disable=unused-import
  from tensornetwork.linalg import linalg as tn_linalg
  rng = np.random.default_rng(5)
  m = rng.standard_normal((40, 40)) + 1j * rng.standard_normal((40, 40))
  be = get_backend()
  out = tn_linalg.inv(tn.Tensor(be.convert_to_tensor(m), backend="cuda_b200"))
  ref = tn_linalg.inv(tn.Tensor(m, backend="numpy"))
  np.testing.assert_allclose(out.array.to_host(), np.asarray(ref.array), rtol=0, atol=1e-12 * np.abs(ref.array).max())
