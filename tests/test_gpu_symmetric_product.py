"""Product charges (U(1) x U(1), U(1) x Z_2, ...) on the device: tnb200_blocksparse_maps_nsym against the host sector maps,
and backend="symmetric_b200" against the reference's backend="symmetric" for tensordot, svd, qr and rq, the DMRG two-site
matvec network and FiniteMPS canonicalisation."""
import itertools
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MODS = {"U1xU1": (None, None), "U1xZ2": (None, 2), "Z2xZ3": (2, 3), "U1x3": (None, None, None), "U1xZ2xU1xZ3": (None, 2, None, 3),
        "5comp": (None, 2, None, None, 3)}


def _backends():
  import tensornetwork_b200  # noqa: F401  (registers "symmetric_b200")
  from tensornetwork.backends import backend_factory
  return backend_factory.get_backend("symmetric_b200"), backend_factory.get_backend("symmetric")


def _charge(tn, q, mods):
  from tensornetwork.block_sparse.charge import BaseCharge
  types = [tn.U1Charge if m is None else tn.Z2Charge if m == 2 else tn.ZNCharge(m) for m in mods]
  return BaseCharge(np.asarray(q, dtype=np.int16), charge_types=types)


def _random_charges(rng, mods, d, lo=-2, hi=2):
  return np.stack([rng.integers(lo, hi + 1, d) if m is None else rng.integers(0, m, d) for m in mods], axis=1)


def _maps_equal(be, idx, order, part):
  from tensornetwork_b200 import blocksparse as bs
  bs._MAP_CACHE.clear()
  q1, d1, m1 = bs._sector_maps(idx, order, part)
  q2, d2, dm, off = bs._device_sector_maps(be, idx, order, part)
  flat = np.concatenate(m1) if m1 else np.zeros(0, dtype=np.int64)
  np.testing.assert_array_equal(q1, q2)
  np.testing.assert_array_equal(d1, d2)
  np.testing.assert_array_equal(flat, dm.cpu().numpy()[:flat.shape[0]])
  np.testing.assert_array_equal(off[:-1], np.cumsum(d1[:, 0] * d1[:, 1]) - d1[:, 0] * d1[:, 1])


@pytest.mark.parametrize("sym", list(MODS))
def test_device_maps_equal_host_maps(tn, sym):
  import tensornetwork_b200 as tb
  from tensornetwork_b200 import blocksparse as bs
  be, mods = tb.get_backend(), MODS[sym]
  rng = np.random.default_rng(sum(map(ord, sym)))
  for trial in range(6):
    n = int(rng.integers(2, 5))
    idx = [bs.Index(_random_charges(rng, mods, int(rng.integers(1, 7))), bool(rng.integers(0, 2)), mods) for _ in range(n)]
    for order in itertools.permutations(range(n)):
      for part in range(n + 1):
        _maps_equal(be, idx, list(order), part)


def test_device_maps_with_many_bins(tn):
  """U(1) x U(1) spread over 125^2 = 15625 bins, row groups of 120000 states: the counting-sort rank stage"""
  import tensornetwork_b200 as tb
  from tensornetwork_b200 import blocksparse as bs
  be, mods = tb.get_backend(), (None, None)
  rng = np.random.default_rng(5)
  idx = [bs.Index(_random_charges(rng, mods, d, lo, hi), f, mods)
         for d, (lo, hi), f in zip((400, 300, 8), ((-30, 30), (-30, 30), (-2, 2)), (False, True, False))]
  shifts = bs._shifts(idx, mods)
  assert (2 * shifts[0] + 1) * (2 * shifts[1] + 1) >= 10 ** 4
  for order, part in (([0, 1, 2], 2), ([1, 0, 2], 2), ([2, 0, 1], 1), ([2, 1, 0], 1)):
    assert np.prod([idx[t].dim for t in order[:part]]) >= 10 ** 5 or np.prod([idx[t].dim for t in order[part:]]) >= 10 ** 5
    _maps_equal(be, idx, order, part)


def _tol(dtype, a):
  scale = max(1.0, float(np.abs(a).max())) if np.size(a) else 1.0
  return (1e-12 if np.dtype(dtype) in (np.float64, np.complex128) else 2e-5) * scale


def _dense(t):
  return np.asarray(t.todense())


def _same(got, want, tol):
  """the reference's shapes, per-leg charges (order included), flows, leg grouping and dense values"""
  assert got.shape == want.shape
  assert [list(o) for o in got._order] == [list(o) for o in want._order]
  assert list(got.flat_flows) == list(want.flat_flows)
  for cg, cw in zip(got.flat_charges, want.flat_charges):
    np.testing.assert_array_equal(np.asarray(cg.charges), np.asarray(cw.charges))
  np.testing.assert_allclose(_dense(got), _dense(want), rtol=0, atol=tol)


def _tensor(tn, legs, dtype, seed):
  np.random.seed(seed)
  t = tn.BlockSparseTensor.random(legs, dtype=dtype)
  if np.dtype(dtype).kind == "c":
    t.data = (np.random.uniform(-1, 1, t.data.shape) + 1j * np.random.uniform(-1, 1, t.data.shape)).astype(dtype)
  return t


def _legs(tn, sym, seed, dims, flows):
  rng = np.random.default_rng(seed)
  mods = MODS[sym]
  return [tn.Index(_charge(tn, _random_charges(rng, mods, d), mods), f) for d, f in zip(dims, flows)]


@pytest.mark.parametrize("dtype", [np.float64, np.complex128, np.float32, np.complex64])
@pytest.mark.parametrize("sym", ["U1xU1", "U1xZ2"])
@pytest.mark.parametrize("ndim", [3, 4])
def test_operations_match_reference(tn, sym, ndim, dtype):
  be, ref = _backends()
  dims, flows = ((6, 5, 9), (False, True, True)) if ndim == 3 else ((5, 4, 6, 7), (False, True, False, True))
  legs = _legs(tn, sym, 11 + ndim, dims, flows)
  t = _tensor(tn, legs, dtype, 3)
  tol = _tol(dtype, t.data)
  # tensordot: plain, with a transposed operand, and with a fused operand
  other = _tensor(tn, [l.copy().flip_flow() for l in legs[1:]] + [tn.Index(legs[0].charges, True)], dtype, 4)
  axes = (list(range(1, ndim)), list(range(ndim - 1)))
  _same(be.tensordot(t, other, axes), ref.tensordot(t, other, axes), tol * 10)
  tt = ref.transpose(t, list(range(1, ndim)) + [0])
  _same(be.tensordot(tt, other, (list(range(ndim - 1)), list(range(ndim - 1)))),
        ref.tensordot(tt, other, (list(range(ndim - 1)), list(range(ndim - 1)))), tol * 10)
  d = t.shape                                  # legs 1 and 2 fused on both operands
  fused = ref.reshape(t, (d[0], d[1] * d[2]) + tuple(d[3:]))
  fo = ref.reshape(other, (d[1] * d[2],) + tuple(other.shape[2:]))
  fax = ([1], [0]) if ndim == 3 else ([1, 2], [0, 1])
  _same(be.tensordot(fused, fo, fax), ref.tensordot(fused, fo, fax), tol * 10)
  # qr / rq at every pivot, on the plain and the transposed tensor
  for x in (t, tt):
    for p in range(1, ndim):
      for op in ("qr", "rq"):
        for g, w in zip(getattr(be, op)(x, p), getattr(ref, op)(x, p)):
          _same(g, w, tol)
  # svd: singular values and their charges, the discarded values, and U S V
  for kw in ({}, {"max_singular_values": 7}, {"max_truncation_error": 0.2}, {"max_truncation_error": 0.1, "relative": True}):
    u, s, v, sd = be.svd(t, 2, **kw)
    ru, rs, rv, rsd = ref.svd(t, 2, **kw)
    assert u.shape == ru.shape and v.shape == rv.shape and s.shape == rs.shape and sd.shape == rsd.shape, kw
    np.testing.assert_allclose(s.data, rs.data, rtol=0, atol=tol)
    np.testing.assert_allclose(sd.data, rsd.data, rtol=0, atol=tol)
    np.testing.assert_array_equal(np.asarray(s._charges[0].charges), np.asarray(rs._charges[0].charges))
    np.testing.assert_array_equal(np.asarray(sd._charges[0].charges), np.asarray(rsd._charges[0].charges))
    for g, w in ((u, ru), (v, rv)):
      assert [np.asarray(c.charges).tolist() for c in g.flat_charges] == [np.asarray(c.charges).tolist() for c in w.flat_charges]
    k = s.shape[0]                               # U S V densely (the reference's diag fails on a one-element bond)
    rec = (_dense(u).reshape(-1, k) * s.data) @ _dense(v).reshape(k, -1)
    rrec = (_dense(ru).reshape(-1, k) * rs.data) @ _dense(rv).reshape(k, -1)
    np.testing.assert_allclose(rec, rrec, rtol=0, atol=tol * 10)


def test_two_site_matvec_network(tn):
  """the DMRG matvec network (L, theta, W1, W2, R) of a spinful chain: U(1) x U(1) = particle number x 2 S_z"""
  rng = np.random.default_rng(4)
  mods = MODS["U1xU1"]
  C = lambda q: _charge(tn, q, mods)
  D, w = 12, 5
  cD, cD2 = C(_random_charges(rng, mods, D)), C(_random_charges(rng, mods, D))
  cw = C(np.array([[0, 0], [1, 1], [-1, -1], [1, -1], [0, 0]]))
  cp = C(np.array([[0, 0], [1, 1], [1, -1], [2, 0]]))             # empty, up, down, doubly occupied
  I = tn.Index
  np.random.seed(4)
  L = tn.BlockSparseTensor.random([I(cw, False), I(cD, True), I(cD, False)], dtype=np.float64)
  th = tn.BlockSparseTensor.random([I(cD, True), I(cp, False), I(cp, False), I(cD2, True)], dtype=np.float64)
  M1 = tn.BlockSparseTensor.random([I(cw, True), I(cw, False), I(cp, False), I(cp, True)], dtype=np.float64)
  M2 = tn.BlockSparseTensor.random([I(cw, True), I(cw, False), I(cp, False), I(cp, True)], dtype=np.float64)
  R = tn.BlockSparseTensor.random([I(cw, True), I(cD2, True), I(cD2, False)], dtype=np.float64)
  net = [[3, -1, 1], [1, 2, 4, 6], [3, 5, -2, 2], [5, 7, -3, 4], [7, -4, 6]]
  got = tn.ncon([L, th, M1, M2, R], net, backend="symmetric_b200")
  want = tn.ncon([L, th, M1, M2, R], net, backend="symmetric")
  _same(got, want, 1e-12 * max(1.0, float(np.abs(want.data).max())))


def test_finite_mps_canonicalises_product_charges(tn):
  """U(1) x U(1) MPS with dimension-1 boundary legs: checked against todense (the reference's host qr fails on those legs)"""
  rng = np.random.default_rng(71)
  mods = MODS["U1xU1"]
  I = tn.Index
  N, D = 6, 12
  cp = _charge(tn, np.array([[0, 0], [1, 1], [1, -1], [2, 0]]), mods)
  def bond(n):                                 # (particle number, 2 S_z) reachable after n of N sites, N particles in total
    num = rng.integers(max(0, N - 2 * (N - n)), min(2 * n, N) + 1, D)
    return _charge(tn, np.stack([num, num - 2 * rng.integers(0, num + 1)], axis=1), mods)
  bonds = [_charge(tn, np.array([[0, 0]]), mods)] + [bond(n) for n in range(1, N)] + [_charge(tn, np.array([[N, 0]]), mods)]
  np.random.seed(7)
  ts = [tn.BlockSparseTensor.random([I(bonds[n], False), I(cp, False), I(bonds[n + 1], True)], dtype=np.float64) for n in range(N)]
  assert all(t.data.size for t in ts)
  def state(xs):
    psi = np.ones((1, 1))
    for x in xs:
      psi = np.tensordot(psi, x, ([psi.ndim - 1], [0]))
    return psi.ravel()
  psi = state([_dense(t) for t in ts])
  assert np.linalg.norm(psi) > 0
  mps = tn.FiniteMPS(ts, canonicalize=True, backend="symmetric_b200")
  for pos in (None, 3):
    if pos is not None:
      mps.position(pos)
    dense = [_dense(t) for t in mps.tensors]
    for n, x in enumerate(dense):
      if n < mps.center_position:
        g = np.einsum("abc,abd->cd", x.conj(), x)
      elif n > mps.center_position:
        g = np.einsum("abc,dbc->ad", x, x.conj())
      else:
        continue
      np.testing.assert_allclose(g, np.eye(g.shape[0]), rtol=0, atol=1e-12)
    np.testing.assert_allclose(state(dense), psi / np.linalg.norm(psi), rtol=0, atol=1e-12)
