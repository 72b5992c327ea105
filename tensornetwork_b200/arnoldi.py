"""Implicitly restarted Arnoldi eigensolver on device tensors — NumPyBackend.eigs
(backends/numpy/numpy_backend.py:216-298, scipy's ARPACK there) with ARPACK's method: exact shifts (Sorensen 1992;
Lehoucq & Sorensen 1996).  Krylov vectors never leave the device: each step is one matvec and one
`tnb200_arnoldi_orth` (CGS2 into the next basis row); the restart compresses the basis with one `tensordot`.  Only
the small m x m Hessenberg problem is solved on the host, with numpy.  Host reads: beta once per step, and the
Hessenberg columns in one batched copy per restart cycle."""
import ctypes
import numpy as np
from . import _lib as L
from . import tensor as T
from .tensor import B200Tensor

_WHICH = ("LM", "SM", "LR", "SR")
_MAX_KRYLOV = 1024          # tnb200_arnoldi_orth takes at most 1024 basis rows


def _gemm(be, a, b, out):
  """out = a @ b for matrices, in the input precision (f32 bases never go through TF32)"""
  ax_a, ax_b = (ctypes.c_int32 * 1)(1), (ctypes.c_int32 * 1)(0)
  L.check(be.lib.tnb200_tensordot(a.ref(), b.ref(), out.ref(), 1, ax_a, ax_b, 0, ax_a, ax_b, L.MATH_STRICT,
                                  be._stream()))


def _order(theta, which):
  """indices of theta, best first under `which`; within a conjugate pair, Im > 0 first"""
  key = {"LM": -np.abs(theta), "SM": np.abs(theta), "LR": -theta.real, "SR": theta.real}[which]
  return np.lexsort((-theta.imag, key))


def _matvec_result(be, w, shape, n, code, who):
  """A matvec's result w as a contiguous length-n vector in the basis dtype.  w must be a `B200Tensor` of the
  operand's shape; a real problem's matvec must not return a complex tensor (other dtypes are converted)."""
  if not isinstance(w, B200Tensor):
    raise TypeError("{}: the matvec returned {}, expected a `B200Tensor`".format(who, type(w)))
  if tuple(w.shape) != shape:
    raise ValueError("{}: the matvec returned shape {}, expected {}".format(who, tuple(w.shape), shape))
  if w.code != code:
    if not T.is_complex_code(code) and T.is_complex_code(w.code):
      raise TypeError("{}: the matvec of a real problem returned a complex tensor".format(who))
    w = be.astype(w, code)
  return be.reshape(be.contiguous(w), (n,))


class _Krylov:
  """The (m + 1) x n basis in `nbufs` device buffers (rows padded to 16 bytes) and the device Hessenberg columns.
  eigs keeps two buffers, so that a restart can compress one basis into the other; gmres needs one."""

  def __init__(self, be, m, n, code, nbufs):
    self.be, self.m, self.n, self.code = be, m, n, code
    torch = be.torch
    tdt = T.code_to_torch(code)
    pad = 16 // np.dtype(T.code_to_np(code)).itemsize
    ldv = -(-n // pad) * pad
    self.bufs = [torch.empty((m + 1, ldv), dtype=tdt, device=be.device) for _ in range(nbufs)]
    self.V = [B200Tensor(b[:, :n], code) for b in self.bufs]
    self.cur = 0
    self.acc_torch = torch.complex128 if T.is_complex_code(code) else torch.float64
    self.hd = torch.zeros((m + 1, m + 1), dtype=self.acc_torch, device=be.device)    # row j: column j of H
    self.matvecs = 0
    self.host_reads = 0

  @property
  def basis(self):
    return self.V[self.cur]

  def row(self, j):
    return B200Tensor(self.bufs[self.cur][j, :self.n], self.code)

  def orth(self, j, w, hrow):
    be = self.be
    L.check(be.lib.tnb200_arnoldi_orth(self.basis.ref(), int(j), w.ref(), self.hd[hrow].data_ptr(), be._stream()))
    self.host_reads += 1
    return float(self.hd[hrow, j + 1].real.item())

  def extend(self, j, w, hrow, shape, need):
    """row j + 1 from w.  On breakdown (w in the span of rows 0..j: an invariant subspace of dimension j + 1) that
    subspace is used when it holds `need` vectors; otherwise row j + 1 is a random vector orthogonalised against the
    basis, as ARPACK's dgetv0 does, with beta = 0 kept in H.  Returns beta."""
    beta = self.orth(j, w, hrow)
    if beta == 0.0 and j + 1 < need:
      for _ in range(5):
        r = self.be.randn(shape, T.code_to_np(self.code))
        if self.orth(j, self.be.reshape(r, (self.n,)), self.m) != 0.0:
          break
      else:
        raise RuntimeError("eigs: could not extend the Krylov basis after an invariant subspace was found")
    return beta


def eigs(be, A, args=None, initial_state=None, shape=None, dtype=None, num_krylov_vecs=50, numeig=6, tol=1e-8,
         which="LR", maxiter=None, return_info=False):
  """See CudaB200Backend.eigs.  With return_info, also returns {"restarts", "matvecs", "nconv", "host_reads"}."""
  if args is None:
    args = []
  if which in ("SI", "LI"):
    raise ValueError(f"which = {which} is currently not supported.")
  if which not in _WHICH:
    raise ValueError(f"which must be one of {_WHICH}, got {which!r}")
  if numeig + 1 >= num_krylov_vecs:
    raise ValueError("`num_krylov_vecs` > `numeig + 1` required!")
  if initial_state is None:
    if shape is None or dtype is None:
      raise ValueError("if no `initial_state` is passed, then `shape` and"
                       "`dtype` have to be provided")
    initial_state = be.randn(shape, dtype)
  if not isinstance(initial_state, B200Tensor):
    raise TypeError("Expected a `B200Tensor`. Got {}".format(type(initial_state)))
  code = initial_state.code
  if code not in (L.F64, L.F32, L.C64, L.C128):
    raise TypeError("eigs needs a float32/float64/complex64/complex128 initial_state, got {}".format(initial_state.dtype))
  shape = tuple(initial_state.shape)
  n = int(initial_state.size)
  m = int(num_krylov_vecs)
  if numeig <= 0:
    raise ValueError("k={} must be greater than 0.".format(numeig))
  if numeig >= n - 1:
    raise TypeError("Cannot use scipy.linalg.eig for LinearOperator A with k >= N - 1.")
  if m > n:
    raise ValueError("ncv must be k+1<ncv<=n, ncv={}".format(m))
  if m > _MAX_KRYLOV:
    raise NotImplementedError("eigs: num_krylov_vecs <= {} on cuda_b200, got {}".format(_MAX_KRYLOV, m))
  if maxiter is None:
    maxiter = n * 10
  real = not T.is_complex_code(code)
  single = code in (L.F32, L.C64)
  eps = float(np.finfo(np.float32 if single else np.float64).eps)
  tol = max(float(tol), eps)
  eps23 = eps ** (2.0 / 3.0)
  acc_np = np.float64 if real else np.complex128

  K = _Krylov(be, m, n, code, 2)
  row0 = K.row(0)
  L.check(be.lib.tnb200_copy(be.reshape(initial_state, (n,)).ref(), row0.ref(), 0, be._stream()))
  nrm = float(be.norm(row0).item())
  K.host_reads += 1
  if not nrm > 0.0:
    raise ValueError("eigs: initial_state must be nonzero and finite, its norm is {}".format(nrm))
  L.check(be.lib.tnb200_affine_inplace(row0.ref(), 1.0 / nrm, 0.0, 0.0, 0.0, be._stream()))

  def matvec(j):
    w = A(be.reshape(K.row(j), shape), *args)
    K.matvecs += 1
    return _matvec_result(be, w, shape, n, code, "eigs")

  H = np.zeros((m + 1, m), dtype=acc_np)
  p = 0
  hi = m                                       # < m once an invariant subspace of dimension hi is found
  cycles = 0
  while True:
    for j in range(p, hi):
      if K.extend(j, matvec(j), j, shape, numeig) == 0.0 and j + 1 >= numeig:
        hi = j + 1
        break
    if hi > p:
      hcols = K.hd[p:hi].cpu().numpy()         # the columns this cycle added, one copy
      K.host_reads += 1
      for j in range(p, hi):
        H[:j + 2, j] = hcols[j - p, :j + 2]
    cycles += 1
    Hm = H[:hi, :hi]
    beta_m = abs(H[hi, hi - 1]) if hi == m else 0.0
    theta, Y = np.linalg.eig(Hm)
    theta = theta.astype(np.complex128)
    Y = Y.astype(np.complex128)
    order = _order(theta, which)
    est = beta_m * np.abs(Y[hi - 1, :])
    ok = est <= tol * np.maximum(eps23, np.abs(theta))
    nconv = int(np.sum(ok[order[:numeig]]))
    if nconv >= numeig:
      break
    if cycles >= maxiter:
      raise RuntimeError("eigs: {} of {} eigenpairs converged in {} restart cycles (maxiter)".format(
          nconv, numeig, cycles))
    # ---- restart (dnaup2 / dngets / dnapps): keep nev Ritz values, apply the other m - nev as exact shifts
    nev = numeig + min(nconv, (m - numeig) // 2)
    if nev == 1 and m >= 6:
      nev = m // 2
    elif nev == 1 and m > 2:
      nev = 2
    if real and theta[order[nev - 1]].imag > 0:       # do not split a conjugate pair
      nev += 1
    if nev >= m:
      nev = m - 1
      if real and theta[order[nev - 1]].imag > 0:
        nev -= 1
    Hs, Q = _apply_shifts(Hm.copy(), theta[order[nev:]], real)
    k = nev
    # new basis rows V Q[:, :k] and the residual f = V Q[:, k] H+[k, k-1] + beta_m Q[m-1, k-1] V[m], no matvec
    coef = np.zeros((k + 1, m + 1), dtype=acc_np)
    coef[:k, :m] = Q[:, :k].T
    coef[k, :m] = Q[:, k] * Hs[k, k - 1]
    coef[k, m] = H[m, m - 1] * Q[m - 1, k - 1]
    cdev = be.convert_to_tensor(coef.astype(T.code_to_np(code)))
    nxt = 1 - K.cur
    out = B200Tensor(K.bufs[nxt][:k + 1, :n], code)
    _gemm(be, cdev, K.basis, out)
    K.cur = nxt
    f = be.copy(K.row(k))
    # re-orthogonalise the residual into row k; the corrections join column k - 1 of H
    if K.extend(k - 1, f, k - 1, shape, numeig) == 0.0 and k >= numeig:
      hi = k
    hk = K.hd[k - 1, :k + 1].cpu().numpy()
    H = np.zeros((m + 1, m), dtype=acc_np)
    H[:k, :k] = Hs[:k, :k]
    H[:k, k - 1] += hk[:k]
    H[k, k - 1] = hk[k]
    p = k

  # ---- Ritz vectors on the device: X = Y^T V, real and imaginary parts by two real tensordots for a real basis
  sel = order[:numeig]
  lam = theta[sel]
  Ys = Y[:, sel]
  torch = be.torch
  ccode = L.C64 if single else L.C128
  cnp = T.code_to_np(ccode)
  Xt = torch.empty((numeig, n), dtype=T.code_to_torch(ccode), device=be.device)
  Vm = B200Tensor(K.bufs[K.cur][:hi, :n], code)
  if real:
    xr = torch.view_as_real(Xt)
    rnp = T.code_to_np(code)
    _gemm(be, be.convert_to_tensor(np.ascontiguousarray(Ys.real.T).astype(rnp)), Vm, B200Tensor(xr[..., 0], code))
    _gemm(be, be.convert_to_tensor(np.ascontiguousarray(Ys.imag.T).astype(rnp)), Vm, B200Tensor(xr[..., 1], code))
  else:
    _gemm(be, be.convert_to_tensor(np.ascontiguousarray(Ys.T).astype(cnp)), Vm, B200Tensor(Xt, ccode))
  vecs = []
  for i in range(numeig):
    x = B200Tensor(Xt[i], ccode)
    x /= be.norm(x)
    vecs.append(be.reshape(x, shape))
  eta = be.convert_to_tensor(lam.astype(cnp))
  if return_info:
    return eta, vecs, {"restarts": cycles - 1, "matvecs": K.matvecs, "nconv": nconv, "host_reads": K.host_reads}
  return eta, vecs


def _apply_shifts(H, shifts, real):
  """Shifted QR steps on the m x m upper Hessenberg H with the given shifts: returns (Q^H H Q, Q).  As in ARPACK's
  dnapps, a negligible subdiagonal is set to zero and each shift is applied to every unreduced diagonal block on its
  own (after a breakdown H is block triangular, and a shift that is exact for one block must not mix them).  For a
  real H a complex-conjugate pair is applied as one double-shift step in real arithmetic."""
  m = H.shape[0]
  ulp = np.finfo(np.float64).eps
  Q = np.eye(m, dtype=H.dtype)
  for mu in shifts:
    if real and mu.imag < 0:
      continue                                     # applied with its partner
    d = np.abs(np.diagonal(H))
    sub = np.abs(np.diagonal(H, -1))
    cut = [i + 1 for i in range(m - 1) if sub[i] <= ulp * (d[i] + d[i + 1])]
    for i in cut:
      H[i, i - 1] = 0.0
    q = np.eye(m, dtype=H.dtype)
    for s, e in zip([0] + cut, cut + [m]):
      if e - s < 2:
        continue
      B = H[s:e, s:e]
      eye = np.eye(e - s, dtype=H.dtype)
      if real and mu.imag > 0:
        M = B @ B - 2.0 * mu.real * B + (abs(mu) ** 2) * eye
      else:
        M = B - (mu.real if real else mu) * eye
      q[s:e, s:e] = np.linalg.qr(M)[0]
    H = np.triu(q.conj().T @ H @ q, -1)
    Q = Q @ q
  return H, Q
