"""TEST DOUBLE for libtnb200.so — lets the *host logic* of the adapters (registration in the reference's backend factory,
axes bookkeeping, views, dtype promotion, error translation, the Lanczos / Arnoldi / GMRES drivers, split control flow,
block-sparse sector maps) run in the GPU-less build container against the REAL reference callers (`tn.Node`, `tn.ncon`,
`contractors.greedy`, `split_node*`, `FiniteDMRG`, `InfiniteMPS`, block-sparse `FiniteMPS`).

`FakeLib` implements every C-ABI entry point of include/tnb200.h except tnb200_device_info, once, on HOST memory with
numpy / scipy and with the contract the header states.  Every entry point is recorded: `calls` and `raised` count, by
name, the calls made and the calls that raised a Python exception (a bug in the double, never a status code).  A test
that needs a failing entry point assigns a replacement to that one name on its instance.  Install it with
hostrun.install(); it lives under tests/ and is never importable from the product package; the product has no CPU
path."""
import collections
import ctypes
import functools
import numpy as np
import scipy.linalg
import expm_rule
from oracle import np_backend as nb
from tensornetwork_b200 import _lib

_NP = {0: np.float64, 1: np.float32, 2: np.float16, 4: np.complex64, 5: np.complex128, 6: np.int32, 7: np.int64, 8: np.bool_}
_WIDE = {0: np.float64, 1: np.float64, 4: np.complex128, 5: np.complex128}
_host_qr = np.linalg.qr       # bound here: a block-sparse test replaces np.linalg.qr to prove the host QR never runs


def _desc(arg):
  return arg._obj if hasattr(arg, "_obj") else arg


def _view(arg):
  d = _desc(arg)
  dt = np.dtype(_NP[d.dtype])
  nd = d.ndim
  shape = tuple(d.shape[i] for i in range(nd))
  strides = tuple(d.stride[i] * dt.itemsize for i in range(nd))
  if any(s == 0 for s in shape):
    return np.zeros(shape, dtype=dt)
  span = sum((s - 1) * abs(st) for s, st in zip(shape, strides)) + dt.itemsize
  buf = (ctypes.c_char * span).from_address(d.data)
  return np.ndarray(shape, dtype=dt, buffer=buf, strides=strides)


def _vec(ptr, n, dt):
  """the n elements of dtype dt at the raw address ptr"""
  dt = np.dtype(dt)
  if n == 0:
    return np.zeros(0, dtype=dt)
  return np.ndarray((n,), dtype=dt, buffer=(ctypes.c_char * (n * dt.itemsize)).from_address(int(ptr)))


def _lu(A):
  """scipy's getrf in double precision, and LAPACK's info: 1 + the first exactly zero pivot, else 0"""
  lu, piv = scipy.linalg.lu_factor(A.astype(np.complex128 if np.iscomplexobj(A) else np.float64), check_finite=False)
  zero = np.flatnonzero(np.diagonal(lu) == 0)
  return lu, piv, (int(zero[0]) + 1 if zero.size else 0)


class FakeLib:
  """same callables as the ctypes library object"""

  def __init__(self):
    self._err = b""
    self._launches = 0
    self.calls = collections.Counter()
    self.raised = collections.Counter()

  def _fail(self, code, msg):
    self._err = msg.encode()
    return code

  def tnb200_last_error(self):
    return self._err

  def tnb200_last_kernel(self):
    return b"fake"

  def tnb200_abi_version(self):
    return 1

  def tnb200_launch_count(self):
    return self._launches

  def tnb200_tensordot(self, a, b, c, naxes, axes_a, axes_b, nbatch, batch_a, batch_b, flags, stream):
    A, B, C = _view(a), _view(b), _view(c)
    ax_a = [axes_a[i] for i in range(naxes)]
    ax_b = [axes_b[i] for i in range(naxes)]
    ba = [batch_a[i] for i in range(nbatch)]
    bb = [batch_b[i] for i in range(nbatch)]
    for x, y in zip(ax_a, ax_b):
      if A.shape[x] != B.shape[y]:
        return self._fail(-1, "shape-mismatch for sum")
    if flags & 1:
      A = np.conj(A)
    if flags & 2:
      B = np.conj(B)
    self._launches += 1
    if nbatch == 0:
      C[...] = np.tensordot(A, B, (ax_a, ax_b))
      return 0
    fa = [i for i in range(A.ndim) if i not in ax_a and i not in ba]
    fb = [i for i in range(B.ndim) if i not in ax_b and i not in bb]
    L = "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOP"
    sa, sb = [None] * A.ndim, [None] * B.ndim
    n = 0
    for x, y in zip(ba, bb):
      sa[x] = sb[y] = L[n]; n += 1
    for x, y in zip(ax_a, ax_b):
      sa[x] = sb[y] = L[n]; n += 1
    for x in fa:
      sa[x] = L[n]; n += 1
    for y in fb:
      sb[y] = L[n]; n += 1
    out = "".join(sa[x] for x in ba) + "".join(sa[x] for x in fa) + "".join(sb[y] for y in fb)
    C[...] = np.einsum("".join(sa) + "," + "".join(sb) + "->" + out, A, B)
    return 0

  def tnb200_chain_create(self, nsteps, steps, first_unsupported, handle):
    self._err = b"chained launches need the CUDA library"
    return -4

  def tnb200_chain_launch(self, handle, stream):
    return -1

  def tnb200_chain_destroy(self, handle):
    return 0

  def tnb200_thin_run_create(self, nsteps, steps, first_unsupported, handle):
    self._err = b"fused thin runs need the CUDA library"
    return -4

  def tnb200_thin_run_launch(self, handle, stream):
    return -1

  def tnb200_thin_run_destroy(self, handle):
    return 0

  def tnb200_copy(self, src, dst, conj, stream):
    s, d = _view(src), _view(dst)
    self._launches += 1
    if np.iscomplexobj(s) and not np.iscomplexobj(d):
      s = s.real
    d[...] = np.conj(s) if conj else s
    return 0

  def tnb200_binary(self, op, a, b, c, stream):
    A, B, C = _view(a), _view(b), _view(c)
    self._launches += 1
    with np.errstate(all="ignore"):
      C[...] = [np.add, np.subtract, np.multiply, np.divide, np.power][op](A, B)
    return 0

  def tnb200_unary(self, op, a, c, stream):
    A, C = _view(a), _view(c)
    self._launches += 1
    f = [np.conj, np.sqrt, np.abs, np.negative, np.exp, np.log, np.sin, np.cos, np.sign, np.real, np.imag][op]
    with np.errstate(all="ignore"):
      C[...] = f(A)
    return 0

  def tnb200_affine_inplace(self, x, ar, ai, br, bi, stream):
    X = _view(x)
    self._launches += 1
    if np.iscomplexobj(X):
      X[...] = X * complex(ar, ai) + complex(br, bi)
    else:
      X[...] = X * ar + br
    return 0

  def tnb200_scale_by_device_scalar(self, x, alpha_ptr, alpha_dtype, power, stream):
    X = _view(x)
    s = _vec(alpha_ptr, 1, _NP[alpha_dtype])[0]
    self._launches += 1
    if not np.iscomplexobj(X):
      s = np.real(s)
    X[...] = X / s if power < 0 else X * s
    return 0

  def tnb200_axpy(self, x, y, ar, ai, alpha_ptr, sign, stream):
    X, Y = _view(x), _view(y)
    self._launches += 1
    if alpha_ptr:
      alpha = sign * _vec(alpha_ptr, 1, X.dtype)[0]
    else:
      alpha = complex(ar, ai) if np.iscomplexobj(X) else ar
    Y[...] = Y + alpha * X
    return 0

  def tnb200_fill(self, c, re, im, stream):
    C = _view(c)
    self._launches += 1
    C[...] = complex(re, im) if np.iscomplexobj(C) else re
    return 0

  def tnb200_compare(self, op, a, b, c, stream):
    A, B = _view(a), _view(b)
    if _desc(c).dtype != _lib.BOOL:
      return self._fail(_lib.ERR_INVALID, "compare: the output must be a bool mask")
    if np.iscomplexobj(A) or np.iscomplexobj(B):
      return self._fail(_lib.ERR_DTYPE, "compare: complex values are not ordered")
    _view(c)[...] = (np.less, np.less_equal, np.greater, np.greater_equal)[op](A, B)
    self._launches += 1
    return 0

  def tnb200_index_update(self, a, mask, re, im, value_ptr, value_dtype, out, stream):
    A, O = _view(a), _view(out)
    if value_ptr:
      value = _vec(value_ptr, 1, _NP[value_dtype])[0]
    else:
      value = complex(re, im) if im != 0.0 else re
    if np.iscomplexobj(value) and not np.iscomplexobj(A):
      return self._fail(_lib.ERR_DTYPE, "index_update: cannot assign a complex value to a real tensor")
    if A.dtype.kind == "i" and np.asarray(value).dtype.kind in "fc":
      value = np.trunc(np.real(value))
    M = np.ones(A.shape, bool) if not mask else _view(mask)
    O[...] = np.where(M, np.asarray(value).astype(A.dtype), A)
    self._launches += 1
    return 0

  def tnb200_eye(self, c, k, stream):
    C = _view(c)
    C[...] = np.eye(C.shape[0], C.shape[1], k=k, dtype=C.dtype)
    return 0

  def tnb200_randn(self, c, seed, stream):
    C = _view(c)
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(C.shape)
    if np.iscomplexobj(C):
      v = v + 1j * rng.standard_normal(C.shape)
    C[...] = v
    return 0

  def tnb200_uniform(self, c, lo, hi, seed, stream):
    C = _view(c)
    rng = np.random.default_rng(seed)
    v = rng.uniform(lo, hi, C.shape)
    if np.iscomplexobj(C):
      v = v + 1j * rng.uniform(lo, hi, C.shape)
    C[...] = v
    return 0

  def tnb200_norm(self, a, out, stream):
    A = _view(a)
    _vec(out, 1, A.real.dtype)[0] = np.linalg.norm(A)
    return 0

  def tnb200_dot(self, x, y, conj_x, out, stream):
    X, Y = _view(x), _view(y)
    _vec(out, 1, X.dtype)[0] = np.sum((np.conj(X) if conj_x else X) * Y)
    return 0

  def tnb200_sum(self, a, c, naxes, axes, stream):
    A, C = _view(a), _view(c)
    C[...] = np.sum(A, axis=tuple(axes[i] for i in range(naxes)))
    return 0

  def tnb200_trace(self, a, c, offset, axis1, axis2, stream):
    A, C = _view(a), _view(c)
    C[...] = np.trace(A, offset=offset, axis1=axis1, axis2=axis2)
    return 0

  def tnb200_diagflat(self, a, c, k, stream):
    A, C = _view(a), _view(c)
    C[...] = np.diagflat(A, k=k)
    return 0

  def tnb200_svd(self, a, u, s, vh, info, stream):
    A = _view(a)
    U, S, Vh = np.linalg.svd(A, full_matrices=False)
    _view(u)[...] = U
    _view(s)[...] = S
    _view(vh)[...] = Vh
    return 0

  def tnb200_svd_truncation_count(self, s, max_sv, use_err, max_err, relative, keep_ptr, stream):
    S = _view(s)
    keep = nb.truncation_count(S, None if max_sv < 0 else max_sv, max_err if use_err else None, bool(relative))
    _vec(keep_ptr, 1, np.int64)[0] = keep
    return 0

  def tnb200_eigh(self, a, w, v, info, stream):
    ww, vv = np.linalg.eigh(_view(a))
    _view(w)[...] = ww
    _view(v)[...] = vv
    return 0

  def tnb200_arnoldi_orth(self, v, j, w, h_ptr, stream):
    V, W = _view(v), _view(w).reshape(-1)
    k = j + 1
    acc = np.complex128 if np.iscomplexobj(V) else np.float64
    eps = np.finfo(V.real.dtype).eps
    Vk, x = V[:k].astype(acc), W.astype(acc)
    h1 = Vk.conj() @ x
    V[k] = x - Vk.T @ h1                      # stored in the basis dtype between the passes, as on the device
    u = V[k].astype(acc)
    h2 = Vk.conj() @ u
    r = u - Vk.T @ h2
    beta = np.linalg.norm(r)
    if beta <= 16.0 * np.sqrt(k + 1.0) * eps * np.linalg.norm(x):
      V[k] = 0
      beta = 0.0
    else:
      V[k] = r / beta
    h = _vec(h_ptr, k + 1, acc)
    h[:k] = h1 + h2
    h[k] = beta
    self._launches += 4
    return 0

  def tnb200_qr(self, a, q, r, nonneg, stream):
    A = _view(a)
    Q, R = _host_qr(A)
    if nonneg:
      ph = np.sign(np.diagonal(R))
      Q = Q * ph
      R = ph.conj()[:, None] * R
    _view(q)[...] = Q
    _view(r)[...] = R
    return 0

  def tnb200_lu_factor(self, a, lu, piv_ptr, info_ptr, stream):
    A = _view(a)
    if A.shape[0] != A.shape[1]:
      return self._fail(_lib.ERR_INVALID, "lu_factor: the matrix must be square")
    f, p, info = _lu(A)
    _view(lu)[...] = f
    _vec(piv_ptr, A.shape[0], np.int32)[...] = p
    _vec(info_ptr, 1, np.int32)[0] = info
    return 0

  def tnb200_inv(self, a, x, info_ptr, stream):
    A = _view(a)
    if A.shape[0] != A.shape[1]:
      return self._fail(_lib.ERR_INVALID, "inv: the matrix must be square")
    _, _, info = _lu(A)
    _vec(info_ptr, 1, np.int32)[0] = info
    if info == 0:
      _view(x)[...] = np.linalg.inv(A)
    self._launches += 1
    return 0

  def tnb200_lu_solve(self, lu, piv_ptr, b, x, stream):
    LU = _view(lu)
    _view(x)[...] = scipy.linalg.lu_solve((LU, _vec(piv_ptr, LU.shape[0], np.int32)), _view(b))
    return 0

  def tnb200_expm(self, a, x, info_ptr, stream):
    A, X = _view(a), _view(x)
    if A.ndim != 2 or A.shape[0] != A.shape[1]:
      return self._fail(_lib.ERR_INVALID, "expm: the matrix must be square")
    if _desc(a).dtype not in _WIDE:
      return self._fail(_lib.ERR_DTYPE, "expm: dtype not supported")
    n = A.shape[0]
    if n == 0:
      return 0
    wide = A.astype(_WIDE[_desc(a).dtype])
    finite = np.isfinite(wide).all()
    X[...] = scipy.linalg.expm(wide) if finite else np.nan
    if info_ptr:
      m, s = expm_rule.select(wide) if finite and n > 1 else (0, 0)
      _vec(info_ptr, 4, np.int32)[...] = (m, s, 0 if n <= _lib.EXPM_FUSED_MAX_N else 1, 0)
    self._launches += 1
    return 0

  # ---- block-sparse entry points (device memory): raw pointers + element counts
  def tnb200_gather(self, src, idx, dst, n, dtype, scatter, stream):
    n = int(n)
    if n == 0:
      return 0
    ix = _vec(idx, n, np.int64)
    hi = int(ix.max()) + 1
    if scatter:
      _vec(dst, hi, _NP[dtype])[ix] = _vec(src, n, _NP[dtype])
    else:
      _vec(dst, n, _NP[dtype])[...] = _vec(src, hi, _NP[dtype])[ix]
    self._launches += 1
    return 0

  def tnb200_blocksparse_tensordot(self, a, b, c, dtype, nsect, dims, am, ao, bm, bo, cm, co, max_m, max_n, conj_b, stream):
    """sector q reads its maps at [off[q], off[q] + size), the sizes m_q k_q, k_q n_q and m_q n_q coming from dims: the
    offsets address whole-tensor maps, so they need not increase, and only the first nsect are read"""
    nsect = int(nsect)
    if nsect == 0 or max_m == 0 or max_n == 0:
      return 0
    d = _vec(dims, 3 * nsect, np.int64).reshape(nsect, 3)
    aoff, boff, coff = (_vec(p, nsect, np.int64) for p in (ao, bo, co))
    sizes = [(d[:, 0] * d[:, 1]), (d[:, 1] * d[:, 2]), (d[:, 0] * d[:, 2])]
    maps = [_vec(mp, int((off + sz).max()), np.int64) for mp, off, sz in zip((am, bm, cm), (aoff, boff, coff), sizes)]
    A, B, C = (_vec(p, int(mp.max()) + 1, _NP[dtype]) for p, mp in zip((a, b, c), maps))
    for q in range(nsect):
      m, k, n = (int(x) for x in d[q])
      x = A[maps[0][aoff[q]:aoff[q] + m * k]].reshape(m, k)
      y = B[maps[1][boff[q]:boff[q] + k * n]].reshape(k, n)
      C[maps[2][coff[q]:coff[q] + m * n]] = (x @ (np.conj(y) if conj_b else y)).ravel()
    self._launches += 1
    return 0

  def tnb200_svd_batched(self, a, dtype, nprob, dims, aoff, u, uoff, s, soff, vh, voff, max_m, max_n, status, stream):
    nprob = int(nprob)
    d = _vec(dims, 2 * nprob, np.int64).reshape(nprob, 2)
    ao, uo, so, vo = (_vec(p, nprob + 1, np.int64) for p in (aoff, uoff, soff, voff))
    rdt = np.zeros(0, dtype=_NP[dtype]).real.dtype
    A, U = _vec(a, int(ao[-1]), _NP[dtype]), _vec(u, int(uo[-1]), _NP[dtype])
    S, V = _vec(s, int(so[-1]), rdt), _vec(vh, int(vo[-1]), _NP[dtype])
    for q in range(nprob):
      m, n = int(d[q, 0]), int(d[q, 1])
      uu, ss, vv = np.linalg.svd(A[ao[q]:ao[q + 1]].reshape(m, n), full_matrices=False)
      U[uo[q]:uo[q + 1]] = uu.ravel()
      S[so[q]:so[q + 1]] = ss
      V[vo[q]:vo[q + 1]] = vv.ravel()
    if status:
      _vec(status, 1, np.int32)[0] = 0
    self._launches += 1
    return 0

  def tnb200_qr_batched(self, a, dtype, nprob, dims, aoff, q, qoff, r, roff, max_elems, adjoint, stream):
    """f32 / c64 are factored in double, as the kernel does"""
    nprob, max_elems = int(nprob), int(max_elems)
    if nprob < 0 or max_elems < 0 or adjoint not in (0, 1):
      return self._fail(_lib.ERR_INVALID, "qr_batched: bad sizes or flag")
    if nprob == 0 or max_elems == 0:
      return 0
    if dtype not in _WIDE:
      return self._fail(_lib.ERR_DTYPE, "qr_batched: dtype")
    if max_elems * np.dtype(_WIDE[dtype]).itemsize > _lib.QR_BATCHED_MAX_BYTES:
      return self._fail(_lib.ERR_UNSUPPORTED, "qr_batched: over the limit")
    d = _vec(dims, 2 * nprob, np.int64).reshape(nprob, 2)
    ao, qo, ro = (_vec(p, nprob, np.int64) for p in (aoff, qoff, roff))
    size = np.dtype(_NP[dtype]).itemsize
    for p in range(nprob):
      m, n = int(d[p, 0]), int(d[p, 1])
      assert m * n <= max_elems
      k = min(m, n)
      A = _vec(int(a) + int(ao[p]) * size, m * n, _NP[dtype]).reshape(m, n).astype(_WIDE[dtype])
      if adjoint:
        qq, rr = _host_qr(A.conj().T)
        qout, rout = qq.conj().T, rr.conj().T     # Q = Q'^H (k x n), R = R'^H (m x k)
      else:
        qout, rout = _host_qr(A)
      assert qout.shape == ((k, n) if adjoint else (m, k)) and rout.shape == ((m, k) if adjoint else (k, n))
      _vec(int(q) + int(qo[p]) * size, qout.size, _NP[dtype])[...] = qout.ravel()
      _vec(int(r) + int(ro[p]) * size, rout.size, _NP[dtype])[...] = rout.ravel()
    self._launches += 1
    return 0

  def tnb200_blocksparse_maps(self, nlegs, dims, charges, leg_off, order, partition, split, modulus, shift, nbins, tables, nnz, map_out, stream):
    """numpy transcription of csrc/blocksparse_maps.cu (same five stages: fuse, rank, first, bucket, element)"""
    nlegs, partition, split, modulus, shift, nbins, nnz = int(nlegs), int(partition), int(split), int(modulus), int(shift), int(nbins), int(nnz)
    dims = [int(dims[i]) for i in range(nlegs)]
    leg_off = [int(leg_off[i]) for i in range(nlegs)]
    order = [int(order[i]) for i in range(nlegs)]
    ch = _vec(charges, sum(dims), np.int64)
    tab = _vec(tables, 3 * nbins, np.int64)
    start_right, sect_off, ncols = tab[:nbins], tab[nbins:2 * nbins], tab[2 * nbins:]
    if nnz == 0:
      return 0
    out = _vec(map_out, nnz, np.int64)

    def digits(legs):
      shape = [dims[t] for t in legs] or [1]
      idx = np.indices(shape).reshape(len(shape), -1) if legs else np.zeros((0, 1), dtype=np.int64)
      return idx

    def fuse(legs):
      idx = digits(legs)
      q = np.zeros(idx.shape[1] if legs else 1, dtype=np.int64)
      for k, t in enumerate(legs):
        q += ch[leg_off[t] + idx[k]]
      return (np.mod(q, modulus) if modulus else q + shift).astype(np.int64)

    def rank(b):
      r = np.zeros(b.shape[0], dtype=np.int64)
      cnt = np.zeros(nbins, dtype=np.int64)
      for v in range(nbins):
        m = b == v
        r[m] = np.arange(int(m.sum()))
        cnt[v] = m.sum()
      return r, cnt
    stored = list(range(nlegs))
    L_, R_ = stored[:split], stored[split:]
    bl, br = fuse(L_), fuse(R_)
    bro, bco = fuse(order[:partition]), fuse(order[partition:])
    rr, cr = rank(br)
    rro, _ = rank(bro)
    rco, _ = rank(bco)
    pb = (modulus - bl) % modulus if modulus else 2 * shift - bl
    first = np.zeros(bl.shape[0] + 1, dtype=np.int64)
    first[1:] = np.cumsum(cr[pb])
    assert first[-1] == nnz
    bucket = np.zeros(br.shape[0], dtype=np.int64)
    bucket[start_right[br] + rr] = np.arange(br.shape[0])
    e = np.arange(nnz)
    l = np.searchsorted(first, e, side="right") - 1
    j = e - first[l]
    r = bucket[start_right[pb[l]] + j]
    row_mul, col_mul, is_row = [0] * nlegs, [0] * nlegs, [0] * nlegs
    m = 1
    for i in range(partition - 1, -1, -1):
      row_mul[order[i]] = m; is_row[order[i]] = 1; m *= dims[order[i]]
    m = 1
    for i in range(nlegs - 1, partition - 1, -1):
      col_mul[order[i]] = m; m *= dims[order[i]]
    Rr = np.zeros(nnz, dtype=np.int64); Cc = np.zeros(nnz, dtype=np.int64); rq = np.zeros(nnz, dtype=np.int64)
    for legs, state in ((L_, l), (R_, r)):
      rem = state.copy()
      for t in reversed(legs):
        d = rem % dims[t]; rem //= dims[t]
        Rr += d * row_mul[t]; Cc += d * col_mul[t]
        if is_row[t]:
          rq += ch[leg_off[t] + d]
    qb = np.mod(rq, modulus) if modulus else rq + shift
    out[sect_off[qb] + rro[Rr] * ncols[qb] + rco[Cc]] = e
    self._launches += 10
    return 0


def _recorded(name, entry):
  @functools.wraps(entry)
  def call(self, *args):
    self.calls[name] += 1
    try:
      return entry(self, *args)
    except Exception:
      self.raised[name] += 1
      raise
  return call


for _name in [n for n in vars(FakeLib) if n.startswith("tnb200_")]:
  setattr(FakeLib, _name, _recorded(_name, vars(FakeLib)[_name]))
