"""Block-sparse DMRG with the data in HBM: device-resident BlockSparseTensors (tensornetwork_b200.symmetric) against the
reference's own tensors, `eigsh_lanczos` on backend="symmetric_b200" against backend="symmetric", what stays on the
device through a sweep, and FiniteDMRG against exact diagonalisation."""
import collections
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SYMS = {"U1": (None,), "Z3": (3,), "U1xU1": (None, None)}
TWO_SITE = [[3, 1, -1], [1, 2, 5, 6], [3, 4, -2, 2], [4, 7, -3, 5], [7, 6, -4]]     # dmrg.py two_site_matvec


def _backends():
  import tensornetwork_b200  # noqa: F401  (registers "symmetric_b200")
  from tensornetwork.backends import backend_factory
  return backend_factory.get_backend("symmetric_b200"), backend_factory.get_backend("symmetric")


def _resident_class():
  from tensornetwork_b200 import symmetric
  return symmetric.resident_class()


def _charge(tn, q, mods):
  """a reference charge of charges q ((n,) or (n, nsym)) and per-component moduli (None: U(1))"""
  from tensornetwork.block_sparse.charge import BaseCharge
  q = np.asarray(q, dtype=np.int16).reshape(len(q), -1)
  types = [tn.U1Charge if m is None else tn.ZNCharge(m) for m in mods]
  if mods == (None,):
    return tn.U1Charge(q[:, 0])
  return BaseCharge(q, charge_types=types)          # (the reference's ZNCharge class fails in its own `contiguous`)


def _random_tensor(tn, legs, dtype, seed):
  np.random.seed(seed)
  t = tn.BlockSparseTensor.random(legs, boundaries=(-1.0, 1.0), dtype=dtype)
  if np.dtype(dtype).kind == "c":
    t.data = (np.random.uniform(-1, 1, t.data.shape) + 1j * np.random.uniform(-1, 1, t.data.shape)).astype(dtype)
  return t


def _upload(tensor):
  """a resident copy of a host tensor"""
  import tensornetwork_b200 as tb
  return _resident_class()(tb.get_backend().convert_to_tensor(np.array(tensor.data)), tensor._charges, tensor._flows,
                           tensor._order)


def _is_resident(t):
  return isinstance(t, _resident_class()) and t.device_data is not None


def _same(got, want, atol, bitwise=False):
  """the reference's shapes, per-leg charges, flows and leg grouping, and its data vector"""
  assert got.shape == want.shape
  assert [[int(x) for x in o] for o in got._order] == [[int(x) for x in o] for o in want._order]
  assert list(got._flows) == list(want._flows)
  for cg, cw in zip(got._charges, want._charges):
    np.testing.assert_array_equal(np.asarray(cg.charges), np.asarray(cw.charges))
  if bitwise:
    assert got.dtype == want.dtype
    np.testing.assert_array_equal(np.asarray(got.data), np.asarray(want.data))
  else:
    np.testing.assert_allclose(np.asarray(got.todense()), np.asarray(want.todense()), rtol=0, atol=atol)


# ----------------------------------------------------------------------------------------------- resident tensors
@pytest.mark.parametrize("sym", list(SYMS))
def test_resident_operations_match_reference(tn, sym):
  be, ref = _backends()
  mods = SYMS[sym]
  rng = np.random.default_rng(sum(map(ord, sym)))
  rand_q = lambda d: np.stack([rng.integers(-2, 3, d) if m is None else rng.integers(0, m, d) for m in mods], axis=1)
  legs = [tn.Index(_charge(tn, rand_q(d), mods), f) for d, f in zip((5, 6, 4, 7), (False, True, False, True))]
  t = _random_tensor(tn, legs, np.float64, 1)
  d = _upload(t)
  tol = 1e-13 * max(1.0, float(np.abs(t.data).max()))
  # transpose / reshape, then contiguous: the reference's data vector bit for bit, with and without a permutation
  for perm in ((2, 0, 3, 1), (1, 0, 2, 3), (3, 2, 1, 0)):
    g, w = d.transpose(perm), t.transpose(perm)
    assert _is_resident(g)
    _same(g.contiguous(), w.contiguous(), 0, bitwise=True)
    _same(d.transpose(perm, shuffle=True), t.transpose(perm, shuffle=True), 0, bitwise=True)
  g = d.transpose((2, 0, 3, 1)).reshape((4 * 5, 7, 6))
  w = t.transpose((2, 0, 3, 1)).reshape((4 * 5, 7, 6))
  assert _is_resident(g)
  _same(g.contiguous(), w.contiguous(), 0, bitwise=True)
  _same(g.contiguous([3, 1, 0, 2]), w.contiguous([3, 1, 0, 2]), 0, bitwise=True)
  gi, wi = g.copy(), w.copy()                              # in place, as `_align_storage_layout` calls it
  assert gi.contiguous([1, 0, 3, 2], inplace=True) is gi and _is_resident(gi)
  wi.contiguous([1, 0, 3, 2], inplace=True)
  _same(gi, wi, 0, bitwise=True)
  with pytest.raises(ValueError):
    d.reshape((7, 11))
  with pytest.raises(ValueError):
    d.transpose((0, 1))
  # elementwise, scalar and copy
  for f in (lambda x: x.conj(), lambda x: x * 2.5, lambda x: 0.5 * x, lambda x: x / 3.0, lambda x: -x, lambda x: x.copy(),
            lambda x: x + x.transpose((0, 1, 2, 3)), lambda x: x - 2.0 * x, lambda x: x.transpose((1, 0, 3, 2)) + x.transpose((1, 0, 3, 2))):
    got, want = f(d), f(t)
    assert _is_resident(got)
    _same(got, want, tol)
  # a resident and a host operand, each with its own storage layout
  tt = t.transpose((1, 0, 3, 2)).contiguous().transpose((1, 0, 3, 2))
  _same(d + tt, t + tt, tol)
  _same(tt.copy() - d, tt - t, tol)
  for bad in (lambda: d * np.ones(2), lambda: d / np.ones(2), lambda: d + 1.0):
    with pytest.raises(TypeError):
      bad()
  assert isinstance(be.norm(d), np.float64) and abs(be.norm(d) - ref.norm(t)) <= 1e-13 * ref.norm(t)
  # tensordot: resident x resident, resident x host, host x resident
  other = _random_tensor(tn, [legs[2].copy().flip_flow(), legs[3].copy().flip_flow(), legs[0].copy()], np.float64, 2)
  want = ref.tensordot(t, other, ([2, 3], [0, 1]))
  for a, b in ((d, _upload(other)), (d, other), (t, _upload(other))):
    got = be.tensordot(a, b, ([2, 3], [0, 1]))
    assert _is_resident(got)
    _same(got, want, tol * 10)
  got = be.tensordot(t, other, ([2, 3], [0, 1]))              # host inputs: the reference's class, on the host
  assert type(got) is tn.BlockSparseTensor
  # svd, qr and rq of a resident (transposed) input: resident factors, S on the host
  for x, y in ((d, t), (d.transpose((1, 3, 0, 2)), t.transpose((1, 3, 0, 2)))):
    u, s, v, _ = be.svd(x, 2, max_singular_values=12)
    ru, rs, rv, _ = ref.svd(y, 2, max_singular_values=12)
    assert _is_resident(u) and _is_resident(v) and not _is_resident(s)
    np.testing.assert_allclose(s.data, rs.data, rtol=0, atol=tol * 10)
    k = s.shape[0]
    rec = (np.asarray(u.todense()).reshape(-1, k) * s.data) @ np.asarray(v.todense()).reshape(k, -1)
    rrec = (np.asarray(ru.todense()).reshape(-1, k) * rs.data) @ np.asarray(rv.todense()).reshape(k, -1)
    np.testing.assert_allclose(rec, rrec, rtol=0, atol=tol * 100)
    for op in ("qr", "rq"):
      for g, w in zip(getattr(be, op)(x, 2), getattr(ref, op)(y, 2)):
        assert _is_resident(g)
        _same(g, w, tol * 10)


def test_resident_data_is_read_only_and_assignment_moves_to_host(tn):
  legs = [tn.Index(tn.U1Charge(np.array([0, 1, -1, 1])), False), tn.Index(tn.U1Charge(np.array([1, 0, -1])), True)]
  t = _random_tensor(tn, legs, np.float64, 3)
  d = _upload(t)
  np.testing.assert_array_equal(d.data, t.data)
  with pytest.raises(ValueError):
    d.data[0] = 1.0
  with pytest.raises(ValueError):
    d.data *= 2.0
  d.data = np.array(t.data) * 2.0
  assert not _is_resident(d) and d.data.flags.writeable
  d.data[0] = 7.0                                          # a host-backed tensor is an ordinary reference tensor
  assert d.data[0] == 7.0 and not _is_resident(d * 2.0)
  assert d.dtype == np.float64


# ----------------------------------------------------------------------------------------------- models
def _xxz_dense(tn, N, dtype, jz=1.0):
  mpo = tn.FiniteXXZ(Jz=jz * np.ones(N - 1), Jxy=np.ones(N - 1), Bz=0.1 * np.ones(N), dtype=dtype, backend="numpy")
  return [np.asarray(w) for w in mpo.tensors]


def _spinful_dense(N, dtype, t=1.0, U=2.0, jz=0.5):
  """hard-core bosons of two species on N sites: site states empty, up, down, both; H = -t sum (b+_s b_s + h.c.) between
  neighbours + U n_up n_down + jz S^z S^z between neighbours.  Conserves both particle numbers: U(1) x U(1) = (N, 2 S_z)."""
  def op(pairs):
    m = np.zeros((4, 4))
    for o, i in pairs:
      m[o, i] = 1.0
    return m
  bu, bd = op([(1, 0), (3, 2)]), op([(2, 0), (3, 1)])          # creation
  sz = np.diag([0.0, 0.5, -0.5, 0.0])
  pairs = [(-t * bu, bu.T), (-t * bu.T, bu), (-t * bd, bd.T), (-t * bd.T, bd), (jz * sz, sz)]
  onsite = U * np.diag([0.0, 0.0, 0.0, 1.0])
  w = len(pairs) + 2
  bulk = np.zeros((w, w, 4, 4))
  bulk[0, 0] = bulk[w - 1, w - 1] = np.eye(4)
  bulk[w - 1, 0] = onsite
  for k, (a, b) in enumerate(pairs):
    bulk[k + 1, 0] = b
    bulk[w - 1, k + 1] = a
  return [bulk[w - 1:w].astype(dtype)] + [bulk.astype(dtype)] * (N - 2) + [bulk[:, :1].astype(dtype)]


def _mpo_charges(dense, cp):
  """charges of the MPO bond legs (flows True, False, False, True: W[l, r, out, in] conserves
  q_r - q_l + q[out] - q[in] = 0), from the left boundary charge 0 and the nonzero pattern of each tensor"""
  qs = [np.zeros((1, cp.shape[1]), dtype=np.int64)]
  for w in dense:
    qr = np.full((w.shape[1], cp.shape[1]), np.iinfo(np.int64).min)
    for a, b, o, i in zip(*np.nonzero(w)):
      qr[b] = qs[-1][a] - cp[o] + cp[i]
    assert (qr != np.iinfo(np.int64).min).all()
    qs.append(qr)
  return qs


def _model(tn, name, N, dtype):
  """(block-sparse MPO tensors, their dense arrays, site charges (d, nsym), moduli, target charge)"""
  if name == "xxz":
    dense, cp, mods, target = _xxz_dense(tn, N, dtype), np.array([[-1], [1]]), (None,), (0,)
  else:
    dense, cp, mods, target = _spinful_dense(N, dtype), np.array([[0, 0], [1, 1], [1, -1], [2, 0]]), (None, None), (N, 0)
  qs = _mpo_charges(dense, cp)
  I = tn.Index
  phys = _charge(tn, cp, mods)
  mpo = [tn.BlockSparseTensor.fromdense([I(_charge(tn, qs[n], mods), True), I(_charge(tn, qs[n + 1], mods), False),
                                         I(phys, False), I(phys, True)], w) for n, w in enumerate(dense)]
  for m, w in zip(mpo, dense):
    np.testing.assert_array_equal(np.asarray(m.todense()), w)         # nothing was dropped
  return mpo, dense, cp, mods, target


def _bond_charges(cp, N, target):
  """every charge of the left block of n sites that the right block can complete to `target`, with multiplicity
  min(left states, right states): bond spaces large enough for the exact ground state"""
  counts = [collections.Counter({(0,) * cp.shape[1]: 1})]
  for _ in range(N):
    c = collections.Counter()
    for q, k in counts[-1].items():
      for s in cp:
        c[tuple(int(x) for x in np.add(q, s))] += k
    counts.append(c)
  bonds = []
  for n in range(N + 1):
    rows = []
    for q, k in sorted(counts[n].items()):
      rest = tuple(int(x) for x in np.subtract(target, q))
      rows += [q] * min(k, counts[N - n].get(rest, 0))
    bonds.append(np.array(rows, dtype=np.int64))
  return bonds


def _mps(tn, cp, mods, target, N, dtype, seed, max_dim=None):
  I = tn.Index
  bonds = _bond_charges(cp, N, target)
  if max_dim is not None:
    rng = np.random.default_rng(seed)
    bonds = [b if len(b) <= max_dim else b[np.sort(rng.choice(len(b), max_dim, replace=False))] for b in bonds]
  phys = _charge(tn, cp, mods)
  return [_random_tensor(tn, [I(_charge(tn, bonds[n], mods), False), I(phys, False), I(_charge(tn, bonds[n + 1], mods), True)],
                         dtype, seed + n) for n in range(N)]


def _exact_energy(dense, cp, target):
  """lowest eigenvalue of the MPO's Hamiltonian in the sector of total charge `target`"""
  import scipy.sparse as sp
  h = [sp.csr_matrix(np.ones((1, 1)))] * dense[0].shape[0]
  q = np.zeros((1, cp.shape[1]), dtype=np.int64)
  for w in dense:
    h = [sum((sp.kron(h[a], sp.csr_matrix(w[a, b])) for a in range(w.shape[0]) if np.any(w[a, b])),
             sp.csr_matrix((h[0].shape[0] * w.shape[2],) * 2)) for b in range(w.shape[1])]
    q = (q[:, None, :] + cp[None, :, :]).reshape(-1, cp.shape[1])
  keep = np.nonzero((q == np.asarray(target)).all(axis=1))[0]
  sector = h[0].tocsr()[keep][:, keep].toarray()
  return float(np.linalg.eigvalsh(sector)[0])


def _dmrg(tn, mps_tensors, mpo_tensors, backend):
  mps = tn.FiniteMPS(mps_tensors, canonicalize=True, backend=backend)
  mpo = tn.FiniteMPO(mpo_tensors, backend=backend)
  return tn.FiniteDMRG(mps, mpo)


# ----------------------------------------------------------------------------------------------- eigsh_lanczos
def _local_problem(tn, dtype, seed=5):
  """the two-site DMRG problem at the bond (3, 4) of an XXZ chain of 8 sites: (initial state, [L, W3, W4, R]), host"""
  mpo, _, cp, mods, target = _model(tn, "xxz", 8, dtype)
  dm = _dmrg(tn, _mps(tn, cp, mods, target, 8, dtype, seed), mpo, "symmetric_b200")
  dm.mps.position(3)
  dm.compute_left_envs()
  dm.compute_right_envs()
  x = tn.ncon([dm.mps.tensors[3], dm.mps.tensors[4]], [[-1, -2, 1], [1, -3, -4]], backend="symmetric")
  return x, [dm.left_envs[3], mpo[3], mpo[4], dm.right_envs[4]]


def _matvec(tn, backend):
  """the two-site DMRG matvec (the reference's `enable_caching` needs ndarray.tostring, gone in numpy 2: it is off)"""
  return lambda x, L, W1, W2, R: tn.ncon([L, x, W1, W2, R], TWO_SITE, backend=backend)


def _rtol(dtype):
  return 1e-10 if np.dtype(dtype) in (np.float64, np.complex128) else 1e-4


def _same_up_to_phase(got, want, rtol):
  g, w = np.asarray(got.todense()).ravel(), np.asarray(want.todense()).ravel()
  ov = np.vdot(g, w)
  phase = ov / abs(ov)
  np.testing.assert_allclose(g * phase, w, rtol=0, atol=rtol * 100 * max(1.0, np.abs(w).max()))


@pytest.mark.parametrize("dtype", [np.float64, np.complex128, np.float32, np.complex64])
@pytest.mark.parametrize("mode", [(False, 1, 20), (True, 1, 20), (True, 3, 20), (False, 1, 3)])
def test_eigsh_lanczos_matches_reference(tn, dtype, mode):
  reorth, numeig, ndiag = mode
  be, ref = _backends()
  x, args = _local_problem(tn, dtype)
  kw = dict(num_krylov_vecs=24, numeig=numeig, tol=1e-12, delta=1e-10, ndiag=ndiag, reorthogonalize=reorth)
  x_before = np.array(x.data)
  eg, vg = be.eigsh_lanczos(_matvec(tn, "symmetric_b200"), args, x, **kw)
  np.testing.assert_array_equal(x.data, x_before)               # the caller's tensor is left alone
  er, vr = ref.eigsh_lanczos(_matvec(tn, "symmetric"), args, x.copy(), enable_caching=False, **kw)
  assert isinstance(eg, np.ndarray) and eg.dtype == er.dtype and eg.shape == er.shape
  np.testing.assert_allclose(eg, er, rtol=_rtol(dtype), atol=0)
  assert len(vg) == len(vr) == numeig
  if numeig == 1 or np.dtype(dtype) in (np.float64, np.complex128):
    for g, w in zip(vg[:1], vr[:1]):
      assert _is_resident(g) and g.dtype == w.dtype
      _same_up_to_phase(g, w, _rtol(dtype))


def test_eigsh_lanczos_stops_on_an_eigenvector(tn):
  """an initial state that is an eigenvector: the second Krylov vector's norm is below `delta`, one step only"""
  be, ref = _backends()
  x, args = _local_problem(tn, np.float64)
  assert x.data.size < 200                                   # so that a reorthogonalised Krylov space exhausts it
  e0, (v0,) = ref.eigsh_lanczos(_matvec(tn, "symmetric"), args, x.copy(), num_krylov_vecs=200, tol=1e-14, delta=1e-12,
                                ndiag=10, reorthogonalize=True, enable_caching=False)
  calls = []
  mv = _matvec(tn, "symmetric_b200")
  eg, (vg,) = be.eigsh_lanczos(lambda *a: calls.append(1) or mv(*a), args, _upload(v0), num_krylov_vecs=20, delta=1e-6)
  er, (vr,) = ref.eigsh_lanczos(_matvec(tn, "symmetric"), args, v0.copy(), num_krylov_vecs=20, delta=1e-6,
                                enable_caching=False)
  assert len(calls) == 1 and eg.shape == er.shape == (1,)
  np.testing.assert_allclose(eg, er, rtol=1e-10)
  np.testing.assert_allclose(eg, e0, rtol=1e-10)
  _same_up_to_phase(vg, vr, 1e-10)


def test_eigsh_lanczos_errors(tn):
  be, _ = _backends()
  x, args = _local_problem(tn, np.float64)
  mv = _matvec(tn, "symmetric_b200")
  with pytest.raises(ValueError, match="`num_krylov_vecs` >= `numeig` required!"):
    be.eigsh_lanczos(mv, args, x, num_krylov_vecs=2, numeig=3, reorthogonalize=True)
  with pytest.raises(ValueError, match="Use `reorthogonalize=True` for `numeig > 1`"):
    be.eigsh_lanczos(mv, args, x, numeig=2)
  with pytest.raises(ValueError, match="have to be provided"):
    be.eigsh_lanczos(mv, args)
  with pytest.raises(TypeError, match="Expected a `BlockSparseTensor`"):
    be.eigsh_lanczos(mv, args, np.ones(4))
  with pytest.raises(ValueError, match="charges or flows"):            # a matvec that changes the legs
    be.eigsh_lanczos(lambda v, *a: mv(v, *a).conj(), args, x)


def test_eigsh_lanczos_uploads_once(tn):
  """host -> device conversions in one call: the initial state and each block-sparse argument, for any Krylov size"""
  import tensornetwork_b200 as tb
  from tensornetwork_b200.tensor import B200Tensor
  be, _ = _backends()
  x, args = _local_problem(tn, np.float64)
  cls = type(tb.get_backend())
  original = cls.convert_to_tensor
  count = [0]
  def counting(self, tensor):
    count[0] += not isinstance(tensor, B200Tensor)
    return original(self, tensor)
  cls.convert_to_tensor = counting
  try:
    for nk in (4, 12):
      count[0] = 0
      be.eigsh_lanczos(_matvec(tn, "symmetric_b200"), args, x, num_krylov_vecs=nk, delta=1e-14, tol=1e-14)
      assert count[0] == 1 + len(args), (nk, count[0])
  finally:
    cls.convert_to_tensor = original


# ----------------------------------------------------------------------------------------------- FiniteDMRG
def test_sweep_keeps_tensors_and_environments_resident(tn):
  mpo, _, cp, mods, target = _model(tn, "xxz", 8, np.float64)
  dm = _dmrg(tn, _mps(tn, cp, mods, target, 8, np.float64, 11), mpo, "symmetric_b200")
  dm.run_two_site(max_bond_dim=16, num_sweeps=1, num_krylov_vecs=6, verbose=0)
  assert all(_is_resident(t) for t in dm.mps.tensors)
  assert all(_is_resident(e) for n, e in dm.left_envs.items() if n > 0)
  assert all(_is_resident(e) for n, e in dm.right_envs.items() if n < len(dm.mps) - 1)
  cls = _resident_class()
  original = cls._download
  downloads = [0]
  def counting(self):
    downloads[0] += 1
    return original(self)
  cls._download = counting
  try:
    dm.position(3)
    dm._optimize_2s_local(max_bond_dim=16, sweep_dir="right", num_krylov_vecs=6)
    dm._optimize_2s_local(max_bond_dim=16, sweep_dir="left", num_krylov_vecs=6)
  finally:
    cls._download = original
  assert downloads[0] == 0
  assert all(_is_resident(t) for t in dm.mps.tensors)


@pytest.mark.parametrize("case", [("xxz", 12), ("spinful", 6)])
def test_finite_dmrg_matches_exact_diagonalisation(tn, case):
  name, N = case
  mpo, dense, cp, mods, target = _model(tn, name, N, np.float64)
  exact = _exact_energy(dense, cp, target)
  kw = dict(num_sweeps=6, precision=1e-12, num_krylov_vecs=20, delta=1e-12, tol=1e-12, ndiag=10, verbose=0)
  dm = _dmrg(tn, _mps(tn, cp, mods, target, N, np.float64, 21), mpo, "symmetric_b200")
  e2 = dm.run_two_site(max_bond_dim=64, **kw)
  assert abs(e2 - exact) <= 1e-8 * abs(exact), (e2, exact)
  assert all(_is_resident(t) for t in dm.mps.tensors)
  dm1 = _dmrg(tn, _mps(tn, cp, mods, target, N, np.float64, 31), mpo, "symmetric_b200")
  e1 = dm1.run_one_site(**kw)
  assert abs(e1 - exact) <= 1e-8 * abs(exact), (e1, exact)
