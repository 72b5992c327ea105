"""Restarted GMRES on device tensors — AbstractBackend.gmres (backends/abstract_backend.py:478-615), with the control
flow of scipy.sparse.linalg.gmres and M = identity (Saad & Schultz 1986).  The Krylov basis is arnoldi._Krylov: each
inner step is one matvec, one `tnb200_arnoldi_orth` (CGS2 into the next basis row) and one copy of the new Hessenberg
column to the host.  The Givens rotations and the triangular solve work on the host, in double, with numpy.  Each
cycle ends with x += y^T V (one tensordot) and the true residual b - A x (one matvec, one subtraction), whose norm is
one host read."""
import numpy as np
from . import _lib as L
from . import tensor as T
from .tensor import B200Tensor
from .arnoldi import _MAX_KRYLOV, _Krylov, _gemm, _matvec_result


def _lartg(f, g):
  """LAPACK's lartg: (c, s, r) with c real, c f + s g = r and -conj(s) f + c g = 0"""
  if g == 0:
    return 1.0, 0.0 * g, f
  if f == 0:
    return 0.0, np.conj(g) / abs(g), abs(g)
  d = np.hypot(abs(f), abs(g))
  ph = f / abs(f)
  return abs(f) / d, ph * np.conj(g) / d, ph * d


def gmres(be, A_mv, b, A_args=None, A_kwargs=None, x0=None, tol=1e-5, atol=None, num_krylov_vectors=20, maxiter=1,
          M=None, return_info=False):
  """See CudaB200Backend.gmres.  With return_info, also returns {"cycles", "matvecs", "host_reads"}."""
  if not isinstance(b, B200Tensor):
    raise TypeError("Expected a `B200Tensor` for b. Got {}".format(type(b)))
  code = b.code
  if code not in (L.F64, L.F32, L.C64, L.C128):
    raise TypeError("gmres needs a float32/float64/complex64/complex128 b, got {}".format(b.dtype))
  shape = tuple(b.shape)
  n = int(b.size)
  if x0 is not None:
    if not isinstance(x0, B200Tensor):
      raise TypeError("Expected a `B200Tensor` for x0. Got {}".format(type(x0)))
    if tuple(x0.shape) != shape:
      raise ValueError("If x0 is supplied, its shape, {}, must match b's, {}.".format(tuple(x0.shape), shape))
    if x0.code != code:
      raise TypeError("If x0 is supplied, its dtype, {}, must match b's, {}.".format(x0.dtype, b.dtype))
  m = n if num_krylov_vectors is None else min(int(num_krylov_vectors), n)
  if tol < 0:
    raise ValueError("tol = {} must be positive.".format(tol))
  if atol is None:
    atol = tol
  elif atol < 0:
    raise ValueError("atol = {} must be positive.".format(atol))
  if m <= 0:
    raise ValueError("num_krylov_vectors must be positive, not {}.".format(m))
  if m > _MAX_KRYLOV:
    raise NotImplementedError("gmres: num_krylov_vectors <= {} on cuda_b200, got {}".format(_MAX_KRYLOV, m))
  if M is not None:
    raise NotImplementedError("gmres: a preconditioner M is only supported by the numpy backend")
  if maxiter is None:
    maxiter = 10 * n
  if maxiter < 1:
    raise ValueError("maxiter = {} must be at least 1.".format(maxiter))
  A_args = [] if A_args is None else A_args
  A_kwargs = {} if A_kwargs is None else A_kwargs
  cplx = T.is_complex_code(code)
  acc_np = np.complex128 if cplx else np.float64
  eps = float(np.finfo(T.code_to_np(code)).eps)
  st = be._stream()

  K = _Krylov(be, m, n, code, 1)
  bv = be.reshape(be.contiguous(b), (n,))
  x = be._new((n,), code)
  row0 = K.row(0)

  def matvec(v):
    w = A_mv(be.reshape(v, shape), *A_args, **A_kwargs)
    K.matvecs += 1
    return _matvec_result(be, w, shape, n, code, "gmres")

  def residual():
    """row 0 = b - A x; returns its norm"""
    w = matvec(x)
    L.check(be.lib.tnb200_binary(L.SUB, bv.ref(), w.ref(), row0.ref(), st))
    K.host_reads += 1
    return float(be.norm(row0).item())

  def result(info, cycles):
    out = (be.reshape(x, shape), int(info))
    return out + ({"cycles": cycles, "matvecs": K.matvecs, "host_reads": K.host_reads},) if return_info else out

  bnrm2 = float(be.norm(bv).item())
  K.host_reads += 1
  atol = max(float(atol), float(tol) * bnrm2)
  if bnrm2 == 0.0:
    L.check(be.lib.tnb200_fill(x.ref(), 0.0, 0.0, st))
    return result(0, 0)
  x0_zero = True
  if x0 is not None:
    L.check(be.lib.tnb200_copy(x0.ref(), be.reshape(x, shape).ref(), 0, st))
    x0_zero = float(be.norm(x).item()) == 0.0
    K.host_reads += 1
  else:
    L.check(be.lib.tnb200_fill(x.ref(), 0.0, 0.0, st))
  if x0_zero:
    L.check(be.lib.tnb200_copy(bv.ref(), row0.ref(), 0, st))
    rnorm = bnrm2
  else:
    rnorm = residual()
  if rnorm < atol or rnorm == 0.0:
    return result(0, 0)

  ptol_max_factor = 1.0
  ptol = bnrm2 * min(ptol_max_factor, atol / bnrm2)
  R = np.zeros((m, m), dtype=acc_np)               # column j: the rotated Hessenberg column j
  givens = np.zeros((m, 2), dtype=acc_np)
  cycles = 0
  for _ in range(maxiter):
    cycles += 1
    L.check(be.lib.tnb200_affine_inplace(row0.ref(), 1.0 / rnorm, 0.0, 0.0, 0.0, st))
    S = np.zeros(m + 1, dtype=acc_np)
    S[0] = rnorm
    breakdown = False
    for col in range(m):
      w = matvec(K.row(col))
      L.check(be.lib.tnb200_arnoldi_orth(K.basis.ref(), col, w.ref(), K.hd[col].data_ptr(), st))
      h = K.hd[col, :col + 2].cpu().numpy()
      K.host_reads += 1
      breakdown = h[col + 1] == 0.0
      for k in range(col):
        c, s = givens[k]
        h[k], h[k + 1] = c * h[k] + s * h[k + 1], -np.conj(s) * h[k] + c * h[k + 1]
      c, s, mag = _lartg(h[col], h[col + 1])
      givens[col] = c, s
      R[:col, col] = h[:col]
      R[col, col] = mag
      S[col], S[col + 1] = c * S[col], -np.conj(s) * S[col]
      presid = abs(S[col + 1])
      if presid <= ptol or breakdown:
        break
    # R[:col+1, :col+1] y = S[:col+1], with scipy's pseudo-solve of a singular R
    if R[col, col] == 0:
      S[col] = 0
    y = S[:col + 1].copy()
    for k in range(col, -1, -1):
      if y[k] != 0:
        y[k] /= R[k, k]
        y[:k] -= y[k] * R[:k, k]
    yd = be.convert_to_tensor(y[None, :].astype(T.code_to_np(code)))
    dx = be._new((1, n), code)
    _gemm(be, yd, B200Tensor(K.bufs[0][:col + 1, :n], code), dx)
    L.check(be.lib.tnb200_axpy(be.reshape(dx, (n,)).ref(), x.ref(), 1.0, 0.0, None, 1.0, st))
    rnorm = residual()
    if rnorm <= atol or breakdown:
      break
    if presid <= ptol:
      ptol_max_factor = max(eps, 0.25 * ptol_max_factor)
    else:
      ptol_max_factor = min(1.0, 1.5 * ptol_max_factor)
    ptol = presid * min(ptol_max_factor, atol / rnorm)
  return result(0 if rnorm <= atol else maxiter, cycles)
