"""Two-site DMRG driver on the `cuda_b200` backend (SURVEY.md 8a row a14).

With the `tensornetwork` package installed, the reference's own `FiniteDMRG.run_two_site`
(matrixproductstates/dmrg.py:445-559) runs unchanged on `backend="cuda_b200"`
(tests/test_refhost.py).  This module restates that driver — same ncon networks, same sweep
order, same Lanczos / SVD calls — without depending on the reference package, so cfg 5 can be
run and timed on a GPU machine where the reference is absent:

  two_site_matvec  <-> dmrg.py:95-100       add_left/right_layer <-> dmrg.py:102-112
  position (QR/RQ) <-> base_mps.py:139-226   _optimize_2s_local   <-> dmrg.py:251-343
  run_two_site     <-> dmrg.py:445-559       XXZ MPO              <-> mpo.py:129-220 (FiniteXXZ)

It is generic over an `ops` object exposing the backend surface (`ncon`, `conj`, `qr`, `rq`,
`svd`, `norm`, `diagflat`, `eigsh_lanczos`, `ones`, `convert_to_tensor`): the product passes the
CUDA backend; the parity tests pass a numpy adapter (oracle/np_ops.py) and golden energies from
the real reference.
"""
import numpy as np


def xxz_mpo(Jz, Jxy, Bz, dtype=np.float64):
  """FiniteXXZ (matrixproductstates/mpo.py:129-220): list of numpy MPO tensors with index order
  (left bond, right bond, physical out, physical in); entries copied value-for-value from mpo.py:158-200."""
  Jz, Jxy, Bz = np.asarray(Jz), np.asarray(Jxy), np.asarray(Bz)
  N = len(Bz)
  sz = np.array([[-0.5, 0.0], [0.0, 0.5]])
  sp = np.array([[0.0, 0.0], [1.0, 0.0]])
  sm = np.array([[0.0, 1.0], [0.0, 0.0]])
  eye = np.eye(2)
  mpo = []
  t = np.zeros((1, 5, 2, 2), dtype=dtype)
  t[0, 0] = Bz[0] * sz
  t[0, 1] = Jxy[0] / 2.0 * sm
  t[0, 2] = Jxy[0] / 2.0 * sp
  t[0, 3] = Jz[0] * sz
  t[0, 4] = eye
  mpo.append(t)
  for n in range(1, N - 1):
    t = np.zeros((5, 5, 2, 2), dtype=dtype)
    t[0, 0] = eye
    t[1, 0] = sp
    t[2, 0] = sm
    t[3, 0] = sz
    t[4, 0] = Bz[n] * sz
    t[4, 1] = Jxy[n] / 2.0 * sm
    t[4, 2] = Jxy[n] / 2.0 * sp
    t[4, 3] = Jz[n] * sz
    t[4, 4] = eye
    mpo.append(t)
  t = np.zeros((5, 1, 2, 2), dtype=dtype)
  t[0, 0] = eye
  t[1, 0] = sp
  t[2, 0] = sm
  t[3, 0] = sz
  t[4, 0] = Bz[-1] * sz
  mpo.append(t)
  return mpo


class TwoSiteDMRG:
  """mps: list of (Dl, d, Dr) tensors, mpo: list of (wl, wr, d, d) tensors (host arrays or backend
  tensors).  The MPS is brought to centre position 0 on construction (`position(0)`)."""

  def __init__(self, ops, mps, mpo, center_position=None):
    self.ops = ops
    self.mps = [ops.convert_to_tensor(t) for t in mps]
    self.mpo = [ops.convert_to_tensor(t) for t in mpo]
    n = len(self.mps)
    if len(self.mpo) != n:
      raise ValueError("len(mps) != len(mpo)")
    self.center = n - 1 if center_position is None else center_position
    dtype = self.mps[0].dtype
    self.left_envs = {0: ops.ones((self.mps[0].shape[0], self.mpo[0].shape[0], self.mps[0].shape[0]), dtype)}
    self.right_envs = {n - 1: ops.ones((self.mps[-1].shape[2], self.mpo[-1].shape[1], self.mps[-1].shape[2]), dtype)}
    self.num_matvecs = 0

  # ---- dmrg.py:90-112
  def two_site_matvec(self, bond, L, wl, wr, R):
    self.num_matvecs += 1
    return self.ops.ncon([L, bond, wl, wr, R],
                         [[3, 1, -1], [1, 2, 5, 6], [3, 4, -2, 2], [4, 7, -3, 5], [7, 6, -4]])

  def add_left_layer(self, L, a, w):
    return self.ops.ncon([L, a, w, self.ops.conj(a)], [[2, 1, 5], [1, 3, -2], [2, -1, 4, 3], [5, 4, -3]])

  def add_right_layer(self, R, a, w):
    return self.ops.ncon([R, a, w, self.ops.conj(a)], [[2, 1, 5], [-2, 3, 1], [-1, 2, 4, 3], [-3, 4, 5]])

  # ---- base_mps.py:139-226 (no truncation), dmrg.py:114-160
  def _mps_position(self, site, normalize=True):
    ops = self.ops
    if site == self.center:
      z = ops.norm(self.mps[site])
      if normalize:
        self.mps[site] /= z
      return
    if site > self.center:
      for n in range(self.center, site):
        iso, rest = ops.qr(self.mps[n], 2)
        self.mps[n] = iso
        self.mps[n + 1] = ops.ncon([rest, self.mps[n + 1]], [[-1, 1], [1, -2, -3]])
        if normalize:
          self.mps[n + 1] /= ops.norm(self.mps[n + 1])
    else:
      for n in reversed(range(site + 1, self.center + 1)):
        rest, iso = ops.rq(self.mps[n], 1)
        self.mps[n] = iso
        self.mps[n - 1] = ops.ncon([self.mps[n - 1], rest], [[-1, -2, 1], [1, -3]])
        if normalize:
          self.mps[n - 1] /= ops.norm(self.mps[n - 1])
    self.center = site

  def position(self, site):
    if site == self.center:
      return
    old = self.center
    self._mps_position(site)
    if site > old:
      for m in range(old, site):
        self.left_envs[m + 1] = self.add_left_layer(self.left_envs[m], self.mps[m], self.mpo[m])
    else:
      for m in reversed(range(site, old)):
        self.right_envs[m] = self.add_right_layer(self.right_envs[m + 1], self.mps[m + 1], self.mpo[m + 1])

  def compute_right_envs(self):
    """dmrg.py:213-222: all right environments for the current centre position."""
    n = len(self.mps)
    for m in reversed(range(self.center, n - 1)):
      self.right_envs[m] = self.add_right_layer(self.right_envs[m + 1], self.mps[m + 1], self.mpo[m + 1])

  # ---- dmrg.py:251-343
  def optimize_two_sites(self, max_bond_dim, sweep_dir, num_krylov_vecs=10, tol=1e-5, delta=1e-6, ndiag=10):
    ops = self.ops
    site = self.center
    if sweep_dir == "right":
      l, r = site, site + 1
    else:
      l, r = site - 1, site
    bond = ops.ncon([self.mps[l], self.mps[r]], [[-1, -2, 1], [1, -3, -4]])
    energies, states = ops.eigsh_lanczos(A=self.two_site_matvec,
                                         args=[self.left_envs[l], self.mpo[l], self.mpo[r], self.right_envs[r]],
                                         initial_state=bond, num_krylov_vecs=num_krylov_vecs, numeig=1, tol=tol,
                                         delta=delta, ndiag=ndiag, reorthogonalize=False)
    gs = states[0]
    energy = energies[0]
    gs /= ops.norm(gs)
    u, s, vh, _ = ops.svd(gs, 2, max_bond_dim, None, relative=True)     # base_mps.py:102-107
    s = ops.diagflat(s)
    if sweep_dir == "right":
      self.mps[l] = u
      self.center += 1
      self.mps[r] = ops.ncon([s, vh], [[-1, 1], [1, -2, -3]])
      self.left_envs[r] = self.add_left_layer(self.left_envs[l], u, self.mpo[l])
    else:
      self.mps[r] = vh
      self.center -= 1
      self.mps[l] = ops.ncon([u, s], [[-1, -2, 1], [1, -3]])
      self.right_envs[l] = self.add_right_layer(self.right_envs[r], vh, self.mpo[r])
    return energy

  # ---- dmrg.py:445-559
  def run_two_site(self, max_bond_dim, num_sweeps=4, precision=1e-6, num_krylov_vecs=10, delta=1e-6, tol=1e-6,
                   ndiag=10):
    n = len(self.mps)
    self._mps_position(0)
    self.compute_right_envs()
    final_energy = 1e100
    energy = None
    iteration = 1
    while True:
      self.position(0)
      while self.center < n - 1:
        energy = self.optimize_two_sites(max_bond_dim, "right", num_krylov_vecs, tol, delta, ndiag)
      self.position(n - 1)
      while self.center > 0:
        energy = self.optimize_two_sites(max_bond_dim, "left", num_krylov_vecs, tol, delta, ndiag)
      e = float(np.real(energy))
      if abs(final_energy - e) < precision:
        final_energy = e
        break
      final_energy = e
      iteration += 1
      if iteration > num_sweeps:
        break
    return final_energy


class BackendOps:
  """adapter: the CUDA backend + drivers.ncon presented as the `ops` surface above"""

  def __init__(self, backend):
    from . import drivers  # pylint: disable=import-outside-toplevel
    self.be = backend
    self._ncon = drivers.ncon

  def ncon(self, tensors, net):
    return self._ncon(tensors, net, backend=self.be)

  def __getattr__(self, name):
    return getattr(self.be, name)
