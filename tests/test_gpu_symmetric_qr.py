"""Block-sparse qr / rq on backend="symmetric_b200" (tensornetwork_b200/symmetric.py -> blocksparse.qr / rq ->
tnb200_qr_batched, with tnb200_qr for sectors over the batched kernel's limit): parity with the reference's
backend="symmetric" where it runs, per-sector checks against np.linalg.qr on the dimension-1 boundary legs where it
does not, and the reference's FiniteMPS canonicalisation and split_node_qr / split_node_rq on top."""
import numpy as np
import pytest
from oracle import np_blocksparse as npb

pytestmark = pytest.mark.gpu


def _backends():
  import tensornetwork_b200  # noqa: F401  (registers "symmetric_b200")
  from tensornetwork.backends import backend_factory
  return backend_factory.get_backend("symmetric_b200"), backend_factory.get_backend("symmetric")


def _tol(dtype, a):
  scale = max(1.0, float(np.abs(a).max())) if np.size(a) else 1.0
  return (1e-12 if np.dtype(dtype) in (np.float64, np.complex128) else 1e-5) * scale


def _dense(t):
  return np.asarray(t.todense())


def _random(tn, legs, dtype, seed):
  np.random.seed(seed)
  t = tn.BlockSparseTensor.random(legs, dtype=dtype)
  if np.dtype(dtype).kind == "c":
    t.data = (np.random.uniform(-1, 1, t.data.shape) + 1j * np.random.uniform(-1, 1, t.data.shape)).astype(dtype)
  return t


def _legs(tn, charge, seed, dims, flows):
  np.random.seed(seed)
  if charge == "U1":
    return [tn.Index(tn.U1Charge.random(d, -2, 2), f) for d, f in zip(dims, flows)]
  z3 = tn.ZNCharge(3)
  return [tn.Index(z3.random(d, 0, 2), f) for d, f in zip(dims, flows)]


def _same(got, want, tol):
  """the reference's shapes, elementary charges, flows, leg grouping and dense values"""
  assert got.shape == want.shape
  assert [list(o) for o in got._order] == [list(o) for o in want._order]
  assert list(got.flat_flows) == list(want.flat_flows)
  for cg, cw in zip(got.flat_charges, want.flat_charges):
    np.testing.assert_array_equal(np.asarray(cg.charges), np.asarray(cw.charges))
  np.testing.assert_allclose(_dense(got), _dense(want), rtol=0, atol=tol)


def _sector_dims(be, t, pivot):
  from tensornetwork_b200 import blocksparse as bsp, symmetric as sym
  dt, groups = sym._to_device(t, be.device_backend)
  nl = sum(len(g) for g in groups[:pivot])
  return bsp._sector_maps(dt.indices, dt.order, nl)[1]


def _parity(t, pivots):
  be, ref = _backends()
  tol = _tol(t.dtype, t.data)
  for p in pivots:
    q, r = be.qr(t, p)
    rq_, rr = ref.qr(t, p)
    _same(q, rq_, tol)
    _same(r, rr, tol)
    r2, q2 = be.rq(t, p)
    rr2, rq2 = ref.rq(t, p)
    _same(r2, rr2, tol)
    _same(q2, rq2, tol)


@pytest.mark.parametrize("dtype", [np.float64, np.complex128, np.float32, np.complex64])
@pytest.mark.parametrize("charge", ["U1", "Z3"])
@pytest.mark.parametrize("ndim", [3, 4])
def test_qr_rq_match_reference(tn, charge, ndim, dtype):
  dims, flows = ((6, 5, 9), (False, True, True)) if ndim == 3 else ((5, 4, 6, 7), (False, True, False, True))
  t = _random(tn, _legs(tn, charge, 11 + ndim, dims, flows), dtype, 3)
  _parity(t, range(1, ndim))


def test_tall_and_wide_sectors_in_one_tensor(tn):
  be, _ = _backends()
  t = _random(tn, _legs(tn, "U1", 21, (3, 4, 10), (False, False, True)), np.float64, 5)
  d = _sector_dims(be, t, 2)
  assert (d[:, 0] > d[:, 1]).any() and (d[:, 0] < d[:, 1]).any(), d
  _parity(t, [1, 2])


def test_fused_and_transposed_inputs(tn):
  _, ref = _backends()
  t = _random(tn, _legs(tn, "U1", 31, (4, 5, 6, 3), (False, True, False, True)), np.float64, 7)
  tt = ref.transpose(t, (2, 0, 3, 1))
  _parity(tt, [1, 2, 3])
  fused = ref.reshape(tt, (tt.shape[0] * tt.shape[1], tt.shape[2], tt.shape[3]))
  _parity(fused, [1, 2])


@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_sectors_over_the_batched_limit_fall_back(tn, dtype):
  from tensornetwork_b200 import _lib
  be, _ = _backends()
  np.random.seed(41)
  c0 = np.concatenate([np.zeros(150, dtype=np.int16), np.random.randint(-2, 3, 30).astype(np.int16)])
  legs = [tn.Index(tn.U1Charge(c0), False), tn.Index(tn.U1Charge(np.array([0, 0, 1])), False),
          tn.Index(tn.U1Charge(np.concatenate([np.zeros(120, dtype=np.int16), np.arange(-2, 4, dtype=np.int16)])), True)]
  t = _random(tn, legs, dtype, 9)
  d = _sector_dims(be, t, 2)
  wide = 16 if np.dtype(dtype).kind == "c" else 8
  big = d[:, 0] * d[:, 1] * wide > _lib.QR_BATCHED_MAX_BYTES
  assert big.any() and (~big & (d[:, 0] * d[:, 1] > 0)).any(), d
  _parity(t, [2])


def _sectors_against_numpy(t, q, r, pivot, tol):
  """every sector of q (.. x k) and r (k x ..) is np.linalg.qr of the same sector of t (identity order)"""
  charges = [np.asarray(c.charges)[:, 0].astype(np.int64) for c in t.flat_charges]
  flows = list(t.flat_flows)
  maps, dims = npb.diagonal_blocks(charges, flows, pivot)
  rows_q = npb.fuse(charges[:pivot], flows[:pivot])
  cols_q = npb.fuse(charges[pivot:], [not f for f in flows[pivot:]])
  bond = np.asarray(q.flat_charges[-1].charges)[:, 0]
  qd = _dense(q).reshape(-1, bond.shape[0])
  rd = _dense(r).reshape(bond.shape[0], -1)
  assert sorted(maps) == sorted(set(bond.tolist()))
  for c, pos in maps.items():
    a = t.data[pos].reshape(dims[c])
    wq, wr = np.linalg.qr(a)
    rows, cols, b = rows_q == c, cols_q == c, bond == c
    np.testing.assert_allclose(qd[rows][:, b], wq, rtol=0, atol=tol)
    np.testing.assert_allclose(rd[b][:, cols], wr, rtol=0, atol=tol)


def _isometry_and_product(a, left, right, tol):
  """left^H left = I and left right = a for matrices (dense)"""
  np.testing.assert_allclose(left.conj().T @ left, np.eye(left.shape[1]), rtol=0, atol=tol)
  np.testing.assert_allclose(left @ right, a, rtol=0, atol=tol)


@pytest.mark.parametrize("dtype", [np.float64, np.complex128])
def test_dimension_one_legs_against_numpy(tn, dtype):
  be, _ = _backends()
  I = tn.Index
  cp = tn.U1Charge(np.array([0, 1]))
  np.random.seed(51)
  cD = tn.U1Charge(np.sort(np.random.randint(0, 2, 16)))
  first = _random(tn, [I(tn.U1Charge(np.array([0])), False), I(cp, False), I(cD, True)], dtype, 1)
  last = _random(tn, [I(cD, False), I(cp, False), I(tn.U1Charge(np.array([1])), True)], dtype, 2)
  tol = _tol(dtype, first.data)
  q, r = be.qr(first, 2)
  assert q.shape[:2] == (1, 2) and r.shape[1] == 16
  _sectors_against_numpy(first, q, r, 2, tol)
  a = _dense(first).reshape(2, 16)
  _isometry_and_product(a, _dense(q).reshape(2, -1), _dense(r).reshape(-1, 16), tol)
  r2, q2 = be.rq(last, 1)
  a = _dense(last).reshape(16, 2)
  k = q2.shape[0]
  _isometry_and_product(a.conj().T, _dense(q2).reshape(k, 2).conj().T, _dense(r2).reshape(16, k).conj().T, tol)


def test_rank_deficient_sector(tn):
  be, _ = _backends()
  I = tn.Index
  legs = [I(tn.U1Charge(np.array([0, 0, 0, 0, 1, 1])), False), I(tn.U1Charge(np.array([0, 1])), False),
          I(tn.U1Charge(np.array([0, 0, 0, 1, 1, 2])), True)]
  t = _random(tn, legs, np.float64, 61)
  d = _dense(t).reshape(12, 6)
  d[:, 1] = 0.0                                  # a zero column inside the charge-0 sector
  t = tn.BlockSparseTensor.fromdense(legs, d.reshape(6, 2, 6))
  tol = _tol(np.float64, t.data)
  q, r = be.qr(t, 2)
  _isometry_and_product(d, _dense(q).reshape(12, -1), _dense(r).reshape(-1, 6), tol)
  r2, q2 = be.rq(t, 2)
  k = q2.shape[0]
  qd = _dense(q2).reshape(k, 6)
  np.testing.assert_allclose(qd @ qd.conj().T, np.eye(k), rtol=0, atol=tol)
  np.testing.assert_allclose(_dense(r2).reshape(12, k) @ qd, d, rtol=0, atol=tol)


def _mps_tensors(tn, N, D, seed):
  I = tn.Index
  np.random.seed(seed)
  cp = tn.U1Charge(np.array([0, 1]))
  def bond(n):                                  # particle numbers reachable after n sites with N / 2 in total
    lo, hi = max(0, N // 2 - (N - n)), min(n, N // 2)
    return tn.U1Charge(np.sort(np.random.randint(lo, hi + 1, D)))
  bonds = [tn.U1Charge(np.array([0]))] + [bond(n) for n in range(1, N)] + [tn.U1Charge(np.array([N // 2]))]
  return [tn.BlockSparseTensor.random([I(bonds[n], False), I(cp, False), I(bonds[n + 1], True)], dtype=np.float64)
          for n in range(N)]


def _state(ts):
  psi = np.ones((1, 1))
  for t in ts:
    psi = np.tensordot(psi, t, ([psi.ndim - 1], [0]))
  return psi.ravel()


def _check_canonical(mps, psi):
  tol = 1e-12
  ts = [_dense(t) for t in mps.tensors]
  for n, t in enumerate(ts):
    if n < mps.center_position:
      g = np.einsum("abc,abd->cd", t.conj(), t)
    elif n > mps.center_position:
      g = np.einsum("abc,dbc->ad", t, t.conj())
    else:
      continue
    np.testing.assert_allclose(g, np.eye(g.shape[0]), rtol=0, atol=tol)
  np.testing.assert_allclose(_state(ts), psi / np.linalg.norm(psi), rtol=0, atol=tol)


def test_finite_mps_canonicalises_on_device(tn):
  ts = _mps_tensors(tn, 8, 16, 71)
  psi = _state([_dense(t) for t in ts])
  host_qr = np.linalg.qr

  def refuse(*args, **kwargs):
    raise AssertionError("np.linalg.qr ran on the host")
  np.linalg.qr = refuse
  try:
    mps = tn.FiniteMPS(ts, canonicalize=True, backend="symmetric_b200")
    assert mps.center_position == 0
    _check_canonical(mps, psi)
    mps.position(5)
    assert mps.center_position == 5
    _check_canonical(mps, psi)
    mps.position(2)
    _check_canonical(mps, psi)
  finally:
    np.linalg.qr = host_qr


def test_split_node_qr_and_rq(tn):
  t = _random(tn, _legs(tn, "U1", 81, (6, 5, 7, 4), (False, True, False, True)), np.float64, 13)
  out = {}
  for backend in ("symmetric", "symmetric_b200"):
    res = []
    for split in (tn.split_node_qr, tn.split_node_rq):
      node = tn.Node(t, backend=backend)
      left, right = split(node, [node[0], node[1]], [node[2], node[3]])
      res.append((left.tensor, right.tensor))
    out[backend] = res
  for (gl, gr), (wl, wr) in zip(out["symmetric_b200"], out["symmetric"]):
    _same(gl, wl, 1e-12)
    _same(gr, wr, 1e-12)
