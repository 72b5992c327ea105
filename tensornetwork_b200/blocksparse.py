"""Abelian-symmetric (U(1) / Z_N, and products of them) block-sparse tensors on the `cuda_b200` backend.

Covers SURVEY.md 8(a) row a11: `block_sparse.tensordot`
(tensornetwork/block_sparse/blocksparsetensor.py:925-1108) with its index maps
(blocksparse_utils.py:330-634) and charge fusion (charge.py:21-673).

Storage convention = the reference's: `data` is a flat vector holding, in row-major order of
the *stored* leg order, exactly those elements of the dense tensor whose fused charge
sum_i s_i * q_i is the identity (s_i = -1 for an outflowing leg (flow True), +1 otherwise,
charge.py:622 `fuse_charges`); transposition only permutes the logical `order`
(blocksparsetensor.py:803-860 makes it contiguous on demand).

The reference executes tensordot as a Python loop over charge sectors of
gather -> np.matmul -> scatter (:1094-1101).  Here the int64 gather/scatter maps are built once
per (charges, flows, order, partition) signature on the host (pure integer work, cached, and
checked bit-exactly against the reference's maps in tests/) and ALL sectors run in ONE launch
of the grouped kernel `tnb200_blocksparse_tensordot`.
"""
import math

import numpy as np
from . import _lib as L
from . import tensor as T
from .tensor import B200Tensor

_MAP_CACHE = {}


class Index:
  """One tensor leg: a charge per basis state and a flow (True = outflowing), the information content of
  `block_sparse.Index` (index.py).  One Abelian symmetry: charges of shape (dim,), modulus None (U(1)) or N (Z_N).  A
  product of nsym symmetries (the reference's BaseCharge with nsym charge_types): charges of shape (dim, nsym) and
  modulus a tuple with one such entry per component (a single value applies to every component).  A (dim, 1) array or a
  1-tuple is the single-symmetry leg."""

  def __init__(self, charges, flow, modulus=None):
    charges = np.asarray(charges, dtype=np.int64)
    mods = tuple(modulus) if isinstance(modulus, (tuple, list)) else None
    self.flow = bool(flow)
    if charges.ndim == 2 and charges.shape[1] > 1:
      nsym = charges.shape[1]
      mods = mods if mods is not None else (modulus,) * nsym
      if len(mods) != nsym:
        raise ValueError("{} moduli for {} charge components".format(len(mods), nsym))
      self.charges = charges
      self.modulus = tuple(None if m is None else int(m) for m in mods)
    else:
      if mods is not None and len(mods) != 1:
        raise ValueError("{} moduli for 1 charge component".format(len(mods)))
      self.charges = charges.ravel()
      self.modulus = mods[0] if mods is not None else modulus  # None: U(1); N: Z_N

  @property
  def dim(self):
    return int(self.charges.shape[0])

  @property
  def nsym(self):
    return 1 if self.charges.ndim == 1 else int(self.charges.shape[1])

  def flip_flow(self):
    return Index(self.charges, not self.flow, self.modulus)

  def key(self):
    if self.nsym == 1:
      return (self.charges.tobytes(), self.flow, self.modulus)
    return (self.charges.tobytes(), self.nsym, self.flow, self.modulus)


def _signed(ix):
  return -ix.charges if ix.flow else ix.charges


def _q2(ix):
  """signed charges as (dim, nsym)"""
  q = _signed(ix)
  return q.reshape(q.shape[0], ix.nsym)


def _mods(ix):
  return ix.modulus if ix.nsym > 1 else (ix.modulus,)


def _sym(indices):
  """(nsym, per-component moduli) of a tensor's legs, from its first leg; legs with another number of components, or a
  product leg with other moduli, raise ValueError"""
  if not indices:
    return 1, (None,)
  nsym, mods = indices[0].nsym, _mods(indices[0])
  for ix in indices[1:]:
    if ix.nsym != nsym or (nsym > 1 and _mods(ix) != mods):
      raise ValueError("legs with different symmetries: {} and {} components, moduli {} and {}".format(
          nsym, ix.nsym, mods, _mods(ix)))
  return nsym, mods


def _wrap(q, mods):
  """(n, nsym) charges with every Z_N column reduced mod N"""
  q = np.array(q, dtype=np.int64, copy=True)
  for k, m in enumerate(mods):
    if m:
      q[:, k] = np.mod(q[:, k], m)
  return q


def _shifts(indices, mods):
  """per component: sum over the legs of max |charge| (U(1)), 0 (Z_N)"""
  qs = [_q2(ix) for ix in indices]
  return tuple(0 if m else int(sum(int(np.abs(q[:, k]).max()) if q.size else 0 for q in qs)) for k, m in enumerate(mods))


def _unique_charges(q):
  """Distinct charges in the reference's sector order, and the label of every input charge (an index into them).

  q is (n,) for one symmetry or (n, nsym).  The reference orders sectors, and with them the bond charges of svd / qr / rq,
  by block_sparse.utils.unique / intersect, whose `collapse` views each int16 charge row as one wider integer before
  np.unique: one component sorts ascending; two sort by component 1 signed, then component 0 read as unsigned 16-bit;
  three get a zero fourth column and sort as an int64 (every component unsigned); four sort as an int64 (component 3
  signed, the rest unsigned); five or more are not collapsed and sort row-lexicographically (np.unique(axis=0)).
  Product charges must fit in int16, the reference's storage type (ValueError otherwise)."""
  q = np.asarray(q)
  if q.ndim == 1:
    return np.unique(q, return_inverse=True)
  n, w = q.shape
  if w == 1:
    u, inv = np.unique(q[:, 0], return_inverse=True)
    return u[:, None], inv.ravel()
  if q.size and (q.min() < np.iinfo(np.int16).min or q.max() > np.iinfo(np.int16).max):
    raise ValueError("product charges must fit in int16, got values in [{}, {}]".format(int(q.min()), int(q.max())))
  a = np.ascontiguousarray(q, dtype=np.int16)
  if w > 4:
    u, inv = np.unique(a, axis=0, return_inverse=True)
    return u.astype(np.int64), inv.ravel()
  if w == 3:
    a = np.concatenate([a, np.zeros((n, 1), dtype=np.int16)], axis=1)
  key = a.view(np.int32 if w == 2 else np.int64).ravel()
  _, first, inv = np.unique(key, return_index=True, return_inverse=True)
  return q[first].astype(np.int64), inv.ravel()


def _qkey(q):
  """a sector charge as a dict key: an int (one symmetry) or a tuple"""
  return int(q) if np.ndim(q) == 0 else tuple(int(x) for x in q)


def _fused_dense(indices, mod):
  """fused (signed) charge of every state of the product space of `indices`, row-major; `mod` a tuple of per-component
  moduli gives (states, nsym)"""
  if isinstance(mod, tuple):
    fused = np.zeros((1, len(mod)), dtype=np.int64)
    for ix in indices:
      fused = (fused[:, None, :] + _q2(ix)[None, :, :]).reshape(-1, len(mod))
    return _wrap(fused, mod)
  fused = np.zeros(1, dtype=np.int64)
  for ix in indices:
    fused = np.add.outer(fused, _signed(ix)).ravel()
  return np.mod(fused, mod) if mod else fused


def _fused_allowed(indices):
  """flat row-major positions (stored order) whose fused charge is the identity, ascending.

  The dense index space (prod of all leg dimensions: 10^8 for the reference tutorial's (100,101,102,103) legs) is never
  enumerated: the legs are cut into a left and a right group of balanced size, each group's fused charges are enumerated
  (sqrt of the dense size), the right states are bucketed by charge (stable), and every left state l pairs with the bucket
  of charge -q_l: position = l * |right| + r.  O(|left| + |right| + nnz)."""
  if not indices:
    return np.zeros(1, dtype=np.int64)
  nsym, mods = _sym(indices)
  mod = indices[0].modulus
  dims = [ix.dim for ix in indices]
  total = 1
  for d in dims:
    total *= d
  best, k, left = None, 1, 1
  for i in range(1, len(dims) + 1):
    left *= dims[i - 1]
    cost = max(left, total // max(left, 1))
    if best is None or cost < best:
      best, k = cost, i
  ql = _fused_dense(indices[:k], mod)
  qr = _fused_dense(indices[k:], mod)
  nr = qr.shape[0]
  if nsym > 1:                               # label the charge rows, then match labels
    want = _wrap(-ql, mods)
    _, lab = np.unique(np.concatenate([qr, want]), axis=0, return_inverse=True)
    qr, want = lab.ravel()[:nr], lab.ravel()[nr:]
  else:
    want = np.mod(-ql, mod) if mod else -ql
  order = np.argsort(qr, kind="stable")
  uniq, start, cnt = np.unique(qr[order], return_index=True, return_counts=True)
  idx = np.searchsorted(uniq, want)
  idx_c = np.minimum(idx, uniq.shape[0] - 1)
  valid = (idx < uniq.shape[0]) & (uniq[idx_c] == want)
  cnt_l = np.where(valid, cnt[idx_c], 0).astype(np.int64)
  nnz = int(cnt_l.sum())
  if nnz == 0:
    return np.zeros(0, dtype=np.int64)
  l_rep = np.repeat(np.arange(ql.shape[0], dtype=np.int64), cnt_l)
  first = np.cumsum(cnt_l) - cnt_l
  within = np.arange(nnz, dtype=np.int64) - np.repeat(first, cnt_l)
  return l_rep * nr + order[np.repeat(start[idx_c], cnt_l) + within].astype(np.int64)


def _sector_maps(indices, order, partition):
  """Gather maps of the matrix view (legs order[:partition] | legs order[partition:]).

  Returns (qnums, dims (nsect x 2), maps list) where maps[q] lists, row-major over the sector's
  (rows x cols), the positions inside the flat data vector.  qnums are the signed row charges, (nsect,) for one
  symmetry, (nsect, nsym) for a product; sectors are in the reference's `intersect` / `unique` order
  (blocksparse_utils.py:375-380, `_unique_charges`), ascending for one symmetry."""
  key = ("sect", tuple(ix.key() for ix in indices), tuple(order), partition)
  hit = _MAP_CACHE.get(key)
  if hit is not None:
    return hit
  pos = _fused_allowed(indices)                       # sorted => data index = rank
  dims = [ix.dim for ix in indices]
  multi = np.unravel_index(pos, dims) if dims else ()
  nsym, mods = _sym(indices)
  rows = [order[i] for i in range(partition)]
  cols = [order[i] for i in range(partition, len(order))]
  R = np.zeros(pos.shape[0], dtype=np.int64)
  rq = np.zeros((pos.shape[0], nsym), dtype=np.int64)
  for leg in rows:
    R = R * dims[leg] + multi[leg]
    rq = rq + _q2(indices[leg])[multi[leg]]
  C = np.zeros(pos.shape[0], dtype=np.int64)
  for leg in cols:
    C = C * dims[leg] + multi[leg]
  rq = _wrap(rq, mods)
  qnums, lab = _unique_charges(rq if nsym > 1 else rq[:, 0])
  perm = np.lexsort((C, R, lab))
  counts = np.bincount(lab, minlength=qnums.shape[0])
  starts = np.cumsum(counts) - counts
  maps, sdims = [], []
  for s, c in zip(starts, counts):
    idx = perm[s:s + c]
    nrows = np.unique(R[idx]).shape[0]
    maps.append(idx.astype(np.int64))
    sdims.append((nrows, c // nrows))
  out = (qnums, np.asarray(sdims, dtype=np.int64).reshape(-1, 2), maps)
  _MAP_CACHE[key] = out
  return out


def _group_hist(indices, legs, shift, mod, nbins):
  """Number of states of the product space of `legs` per fused signed charge, in the global charge bins
  (U(1): bin = q + shift; Z_N: bin = q mod N): charge-degeneracy arithmetic — a convolution of the legs' charge
  histograms; the product space itself is never enumerated.  For product charges `shift` and `mod` are per-component
  tuples, and the bins are mixed-radix numbers over the component bins (component 0 most significant, as
  tnb200_blocksparse_maps_nsym numbers them): an nsym-dimensional convolution, wrapping around on Z_N axes."""
  if isinstance(mod, tuple):
    return _group_hist_nd(indices, legs, shift, mod)
  if mod:
    h = np.zeros(mod, dtype=np.int64)
    h[0] = 1
    for t in legs:
      ht = np.bincount(np.mod(_signed(indices[t]), mod), minlength=mod).astype(np.int64)
      full = np.convolve(h, ht)
      h = np.zeros(mod, dtype=np.int64)
      np.add.at(h, np.arange(full.shape[0]) % mod, full)
    return h
  h = np.ones(1, dtype=np.int64)
  lo = 0                                     # charge of h[0]
  for t in legs:
    q = _signed(indices[t])
    qmin = int(q.min()) if q.size else 0
    ht = np.bincount(q - qmin).astype(np.int64) if q.size else np.zeros(1, dtype=np.int64)
    h = np.convolve(h, ht)
    lo += qmin
  out = np.zeros(nbins, dtype=np.int64)
  out[lo + shift:lo + shift + h.shape[0]] = h
  return out


def _group_hist_nd(indices, legs, shifts, mods):
  radix = [m if m else 2 * s + 1 for m, s in zip(mods, shifts)]
  nsym = len(mods)
  h = np.zeros([m if m else 1 for m in mods], dtype=np.int64)
  h[(0,) * nsym] = 1
  lo = [0] * nsym                            # charge of index 0 on each U(1) axis
  for t in legs:
    q = _wrap(_q2(indices[t]), mods)
    if q.shape[0] == 0:
      return np.zeros(int(np.prod(radix)), dtype=np.int64)
    qmin = np.array([0 if m else int(q[:, k].min()) for k, m in enumerate(mods)], dtype=np.int64)
    rel = q - qmin
    u, cnt = np.unique(rel, axis=0, return_counts=True)
    out = np.zeros([h.shape[k] + (0 if m else int(rel[:, k].max())) for k, m in enumerate(mods)], dtype=np.int64)
    for row, c in zip(u, cnt):
      src = h
      for k, m in enumerate(mods):
        if m and row[k]:
          src = np.roll(src, int(row[k]), axis=k)
      out[tuple(slice(None) if m else slice(int(row[k]), int(row[k]) + h.shape[k]) for k, m in enumerate(mods))] += c * src
    h = out
    lo = [lo[k] + int(qmin[k]) for k in range(nsym)]
  full = np.zeros(radix, dtype=np.int64)
  full[tuple(slice(None) if m else slice(lo[k] + shifts[k], lo[k] + shifts[k] + h.shape[k])
             for k, m in enumerate(mods))] = h
  return full.ravel()


def _count_allowed(indices):
  """number of stored elements (total signed charge zero) from the legs' charge histograms alone"""
  if not indices:
    return 1
  nsym, mods = _sym(indices)
  if nsym > 1:
    shifts = _shifts(indices, mods)
    h = _group_hist(indices, list(range(len(indices))), shifts, mods, None)
    zero = np.ravel_multi_index([0 if m else s for m, s in zip(mods, shifts)], [m if m else 2 * s + 1 for m, s in zip(mods, shifts)])
    return int(h[zero])
  mod = indices[0].modulus
  shift = 0 if mod else int(sum(int(np.abs(_signed(ix)).max()) if ix.dim else 0 for ix in indices))
  nbins = int(mod) if mod else 2 * shift + 1
  h = _group_hist(indices, list(range(len(indices))), shift, mod, nbins)
  return int(h[0] if mod else h[shift])


def _device_sector_maps(be, indices, order, partition):
  """`_sector_maps` with the element map built ON THE DEVICE (tnb200_blocksparse_maps, or tnb200_blocksparse_maps_nsym for
  product charges; SURVEY 8f rank 3).

  Returns (qnums, dims (nsect x 2), dev_map (1-D int64 device tensor, all sectors in `_sector_maps`' order), offs (nsect + 1)).
  The host computes only the per-charge tables (histogram convolutions of the legs)."""
  key = ("dsect", tuple(ix.key() for ix in indices), tuple(order), partition)
  hit = _MAP_CACHE.get(key)
  if hit is not None:
    return hit
  import ctypes  # pylint: disable=import-outside-toplevel
  torch = be.torch
  n = len(indices)
  if n == 0:                                  # a scalar: one 1 x 1 sector holding data[0]
    out = (np.zeros(1, dtype=np.int64), np.ones((1, 2), dtype=np.int64), torch.zeros(1, dtype=torch.int64, device=be.device),
           np.array([0, 1], dtype=np.int64))
    _MAP_CACHE[key] = out
    return out
  nsym, mods = _sym(indices)
  dims = [ix.dim for ix in indices]
  signed = [_q2(ix) for ix in indices]
  shifts = _shifts(indices, mods)
  radix = [m if m else 2 * s_ + 1 for m, s_ in zip(mods, shifts)]
  nbins = math.prod(radix)
  if nbins > L.BLOCKSPARSE_MAX_BINS:
    raise NotImplementedError("block-sparse maps: the charges span {} bins, more than the {} the device map builder "
                              "takes".format(nbins, L.BLOCKSPARSE_MAX_BINS))
  comp = [np.arange(nbins)] if nsym == 1 else np.unravel_index(np.arange(nbins), radix)   # per-component bin of every bin
  pcomp = [(m - c) % m if m else 2 * s_ - c for c, m, s_ in zip(comp, mods, shifts)]
  pb = pcomp[0] if nsym == 1 else np.ravel_multi_index(pcomp, radix)
  hist = ((lambda legs: _group_hist(indices, legs, shifts[0], mods[0], nbins)) if nsym == 1 else
          (lambda legs: _group_hist(indices, legs, shifts, mods, nbins)))
  # split of the STORED legs into two balanced groups (as _fused_allowed does)
  total, best, split, left = int(np.prod(dims)) if dims else 1, None, 1, 1
  for i in range(1, n + 1):
    left *= dims[i - 1]
    cost = max(left, total // max(left, 1))
    if best is None or cost < best:
      best, split = cost, i
  stored = list(range(n))
  rows, cols = list(order[:partition]), list(order[partition:])
  h_left = hist(stored[:split])
  h_right = hist(stored[split:])
  h_row = hist(rows)
  h_col = hist(cols)
  nnz = int((h_left * h_right[pb]).sum())
  start_right = np.zeros(nbins, dtype=np.int64)
  start_right[1:] = np.cumsum(h_right)[:-1]
  ncols = h_col[pb]
  sizes = h_row * ncols
  live = np.nonzero(sizes > 0)[0]
  # the sectors' charges, laid out in the reference's order (ascending bins for one symmetry)
  if nsym == 1:
    qnums = (live - shifts[0]).astype(np.int64)
  else:
    qnums, lab = _unique_charges(np.stack([comp[k][live] - shifts[k] for k in range(nsym)], axis=1).astype(np.int64))
    live = live[np.argsort(lab)]
  sect_off = np.zeros(nbins, dtype=np.int64)
  sect_off[live] = np.cumsum(sizes[live]) - sizes[live]
  sdims = np.stack([h_row[live], ncols[live]], axis=1).astype(np.int64).reshape(-1, 2)
  offs = np.append(sect_off[live], nnz).astype(np.int64)
  assert int(sizes.sum()) == nnz
  leg_off = np.zeros(n, dtype=np.int64)
  leg_off[1:] = np.cumsum(dims)[:-1]
  charges_dev = torch.from_numpy(np.ascontiguousarray(np.concatenate(signed)).ravel()).to(be.device)
  tables_dev = torch.from_numpy(np.concatenate([start_right, sect_off, ncols])).to(be.device)
  dev_map = torch.empty(max(nnz, 1), dtype=torch.int64, device=be.device)
  i64 = lambda xs: (ctypes.c_int64 * max(len(xs), 1))(*[int(x) for x in xs])
  i32 = lambda xs: (ctypes.c_int32 * max(len(xs), 1))(*[int(x) for x in xs])
  st = be._stream()  # pylint: disable=protected-access
  if nsym == 1:
    rc = be.lib.tnb200_blocksparse_maps(n, i64(dims), charges_dev.data_ptr(), i64(leg_off), i32(order), int(partition), int(split),
                                        int(mods[0] or 0), int(shifts[0]), nbins, tables_dev.data_ptr(), nnz, dev_map.data_ptr(), st)
  else:
    rc = be.lib.tnb200_blocksparse_maps_nsym(n, nsym, i64(dims), charges_dev.data_ptr(), i64(leg_off), i32(order), int(partition),
                                             int(split), i64([m or 0 for m in mods]), i64(shifts), nbins, tables_dev.data_ptr(), nnz,
                                             dev_map.data_ptr(), st)
  L.check(rc)
  out = (qnums, sdims, dev_map, offs)
  _MAP_CACHE[key] = out
  return out


class BlockSparseTensor:
  """Block-sparse tensor whose `data` vector lives in HBM (a 1-D B200Tensor)."""

  def __init__(self, data, indices, order=None, backend=None):
    from .backend import get_instance  # pylint: disable=import-outside-toplevel
    self.backend = backend or get_instance()
    self.indices = list(indices)
    self.order = list(range(len(indices))) if order is None else list(order)
    self.data = data

  # ------------------------------------------------------------------ constructors
  @classmethod
  def _nnz(cls, indices):
    key = ("nnz", tuple(ix.key() for ix in indices))
    hit = _MAP_CACHE.get(key)
    if hit is None:
      hit = _count_allowed(indices)
      _MAP_CACHE[key] = hit
    return hit

  @classmethod
  def zeros(cls, indices, dtype=np.float64, backend=None):
    from .backend import get_instance  # pylint: disable=import-outside-toplevel
    be = backend or get_instance()
    return cls(be.zeros((cls._nnz(indices),), dtype), indices, backend=be)

  @classmethod
  def randn(cls, indices, dtype=np.float64, seed=None, backend=None):
    from .backend import get_instance  # pylint: disable=import-outside-toplevel
    be = backend or get_instance()
    return cls(be.randn((cls._nnz(indices),), dtype, seed=seed), indices, backend=be)

  @classmethod
  def random(cls, indices, boundaries=(0.0, 1.0), dtype=np.float64, seed=None, backend=None):
    from .backend import get_instance  # pylint: disable=import-outside-toplevel
    be = backend or get_instance()
    return cls(be.random_uniform((cls._nnz(indices),), boundaries, dtype, seed=seed), indices, backend=be)

  @classmethod
  def from_data(cls, data, indices, order=None, backend=None):
    """wrap a host data vector laid out like the reference's `BlockSparseTensor.data`."""
    from .backend import get_instance  # pylint: disable=import-outside-toplevel
    be = backend or get_instance()
    data = np.ascontiguousarray(data).ravel()
    if data.shape[0] != cls._nnz(indices):
      raise ValueError("data has {} elements, the charges allow {}".format(data.shape[0], cls._nnz(indices)))
    return cls(be.convert_to_tensor(data), indices, order, backend=be)

  @classmethod
  def fromdense(cls, indices, array, backend=None):
    """blocksparsetensor.py:534-573: keep the symmetry-allowed elements of a dense array."""
    array = np.asarray(array)
    if tuple(array.shape) != tuple(ix.dim for ix in indices):
      raise ValueError("Cannot initialize an BlockSparseTensor of shape {} from an array of shape {}".format(
          tuple(ix.dim for ix in indices), array.shape))
    return cls.from_data(array.ravel()[_fused_allowed(indices)], indices, backend=backend)

  # ------------------------------------------------------------------ metadata
  @property
  def ndim(self):
    return len(self.indices)

  @property
  def shape(self):
    return tuple(self.indices[i].dim for i in self.order)

  @property
  def dtype(self):
    return self.data.dtype

  @property
  def flows(self):
    return [self.indices[i].flow for i in self.order]

  def todense(self):
    """blocksparsetensor.py:575-589 (host side: used by tests / user inspection)."""
    dims = [ix.dim for ix in self.indices]
    host = self.data.to_host()
    out = np.zeros(int(np.prod(dims)) if dims else 1, dtype=host.dtype)
    out[_fused_allowed(self.indices)] = host
    return out.reshape(dims).transpose(self.order) if dims else out.reshape(())

  def transpose(self, order=None):
    """lazy: only the logical order changes (blocksparsetensor.py:738-760)."""
    if order is None:
      order = list(reversed(range(self.ndim)))
    if sorted(order) != list(range(self.ndim)):
      raise ValueError("order = {} is not a permutation".format(order))
    return BlockSparseTensor(self.data, self.indices, [self.order[i] for i in order], self.backend)

  def conj(self):
    """blocksparsetensor.py:723-736: conjugate the data, flip every flow."""
    return BlockSparseTensor(self.backend.conj(self.data), [ix.flip_flow() for ix in self.indices],
                             self.order, self.backend)

  def __mul__(self, number):
    return BlockSparseTensor(self.data * number, self.indices, self.order, self.backend)

  __rmul__ = __mul__

  def __add__(self, other):
    self._same_structure(other)
    return BlockSparseTensor(self.data + other.data, self.indices, self.order, self.backend)

  def __sub__(self, other):
    self._same_structure(other)
    return BlockSparseTensor(self.data - other.data, self.indices, self.order, self.backend)

  def _same_structure(self, other):
    if self.order != other.order or [i.key() for i in self.indices] != [i.key() for i in other.indices]:
      raise ValueError("cannot combine tensors with non-matching charges / flows / orders")


def tensordot(a, b, axes):
  """block_sparse.tensordot (blocksparsetensor.py:925-1108) — all charge sectors in one launch.

  Result legs: free legs of `a` (logical order) then free legs of `b`; same data layout as the
  reference (fresh tensor, identity order)."""
  be = a.backend
  if isinstance(axes, (int, np.integer)):
    n = int(axes)
    axes_a = list(range(a.ndim - n, a.ndim))
    axes_b = list(range(n))
  else:
    axes_a = [int(x) for x in (axes[0] if not isinstance(axes[0], (int, np.integer)) else [axes[0]])]
    axes_b = [int(x) for x in (axes[1] if not isinstance(axes[1], (int, np.integer)) else [axes[1]])]
  if len(axes_a) != len(axes_b):
    raise ValueError("`axes1 = {}` and `axes2 = {}` have to be of same length.".format(axes_a, axes_b))
  if len(axes_a) > a.ndim or len(axes_b) > b.ndim:
    raise ValueError("too many axes for the given tensors")
  if len(set(axes_a)) != len(axes_a) or len(set(axes_b)) != len(axes_b):
    raise ValueError("Some values in axes appear more than once")
  if a.data.code != b.data.code:
    raise ValueError("tensor1 and tensor2 have different dtypes")
  # contracted legs need equal charges and opposite flows (blocksparsetensor.py:985-1015)
  for x, y in zip(axes_a, axes_b):
    ia, ib = a.indices[a.order[x]], b.indices[b.order[y]]
    if ia.dim != ib.dim:
      raise ValueError("axes1 and axes2 have incompatible elementary shapes")
    if ia.flow == ib.flow:
      raise ValueError("axes1 and axes2 have incompatible elementary flows")
    if not np.array_equal(ia.charges, ib.charges):
      raise ValueError("axes1 and axes2 have incompatible elementary charges")
  free_a = [i for i in range(a.ndim) if i not in axes_a]
  free_b = [i for i in range(b.ndim) if i not in axes_b]
  out_indices = [a.indices[a.order[i]] for i in free_a] + [b.indices[b.order[i]] for i in free_b]
  # everything below up to the launch depends only on the charge structure: one cached plan per
  # (legs, orders, axes), so a repeated contraction costs one kernel launch and no host index work
  pkey = ("plan", tuple(ix.key() for ix in a.indices), tuple(a.order), tuple(ix.key() for ix in b.indices),
          tuple(b.order), tuple(axes_a), tuple(axes_b), a.data.code)
  plan = _MAP_CACHE.get(pkey)
  if plan is not None:
    nnz_c, dev = plan
    c_data = be.zeros((nnz_c,), a.data.dtype)
    if dev is None:
      return BlockSparseTensor(c_data, out_indices, backend=be)
    rc = be.lib.tnb200_blocksparse_tensordot(
        a.data.t.data_ptr(), b.data.t.data_ptr(), c_data.t.data_ptr(), a.data.code, dev["nsect"],
        dev["dims"].data_ptr(), dev["am"].data_ptr(), dev["ao"].data_ptr(), dev["bm"].data_ptr(),
        dev["bo"].data_ptr(), dev["cm"].data_ptr(), dev["co"].data_ptr(), dev["max_m"], dev["max_n"], 0,
        be._stream())  # pylint: disable=protected-access
    L.check(rc)
    out = BlockSparseTensor(c_data, out_indices, backend=be)
    out.last_flops = dev["flops"]
    return out
  # matrix views: A = (free_a | axes_a), B = (axes_b | free_b), C = (free_a | free_b)
  order_a = [a.order[i] for i in free_a] + [a.order[i] for i in axes_a]
  order_b = [b.order[i] for i in axes_b] + [b.order[i] for i in free_b]
  qa, da, ma, oa = _device_sector_maps(be, a.indices, order_a, len(free_a))
  qb, db, mb, ob = _device_sector_maps(be, b.indices, order_b, len(axes_b))
  qc, dc, mc, oc = _device_sector_maps(be, out_indices, list(range(len(out_indices))), len(free_a))
  nnz_c = BlockSparseTensor._nnz(out_indices)  # pylint: disable=protected-access
  c_data = be.zeros((nnz_c,), a.data.dtype)      # blocksparsetensor.py:1088: zero-initialised
  mod = a.indices[0].modulus if a.indices else None
  # B's row charge equals A's row charge within a sector (opposite flows on contracted legs);
  sect = []
  posb = {_qkey(q): i for i, q in enumerate(qb)}
  posc = {_qkey(q): i for i, q in enumerate(qc)}
  for i, q in enumerate(qa):
    q = _qkey(q)
    if q in posb and q in posc:
      j, k = posb[q], posc[q]
      m_, k_ = int(da[i, 0]), int(da[i, 1])
      kb_, n_ = int(db[j, 0]), int(db[j, 1])
      if k_ != kb_ or int(dc[k, 0]) != m_ or int(dc[k, 1]) != n_:
        raise RuntimeError("block-sparse sector bookkeeping mismatch (internal error)")
      sect.append((i, j, k, m_, k_, n_))
  if not sect or nnz_c == 0:
    _MAP_CACHE[pkey] = (nnz_c, None)
    return BlockSparseTensor(c_data, out_indices, backend=be)
  key = ("td", id(ma), id(mb), id(mc), tuple(s[:3] for s in sect))
  dev = _MAP_CACHE.get(key)
  if dev is None:
    torch = be.torch
    dims = np.array([[m_, k_, n_] for (_, _, _, m_, k_, n_) in sect], dtype=np.int64)
    up = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(be.device)
    # the device maps hold every sector of their tensor; a contraction sector starts at that sector's offset
    ao = np.array([oa[sc[0]] for sc in sect] + [0], dtype=np.int64)
    bo = np.array([ob[sc[1]] for sc in sect] + [0], dtype=np.int64)
    co = np.array([oc[sc[2]] for sc in sect] + [0], dtype=np.int64)
    dev = dict(dims=up(dims), am=ma, ao=up(ao), bm=mb, bo=up(bo), cm=mc, co=up(co),
               max_m=int(dims[:, 0].max()), max_n=int(dims[:, 2].max()), nsect=len(sect),
               keep=(ma, mb, mc), flops=float(2 * (dims[:, 0] * dims[:, 1] * dims[:, 2]).sum()))
    _MAP_CACHE[key] = dev
  _MAP_CACHE[pkey] = (nnz_c, dev)
  rc = be.lib.tnb200_blocksparse_tensordot(
      a.data.t.data_ptr(), b.data.t.data_ptr(), c_data.t.data_ptr(), a.data.code, dev["nsect"],
      dev["dims"].data_ptr(), dev["am"].data_ptr(), dev["ao"].data_ptr(), dev["bm"].data_ptr(),
      dev["bo"].data_ptr(), dev["cm"].data_ptr(), dev["co"].data_ptr(), dev["max_m"], dev["max_n"], 0,
      be._stream())  # pylint: disable=protected-access
  L.check(rc)
  out = BlockSparseTensor(c_data, out_indices, backend=be)
  out.last_flops = dev["flops"]
  return out


def _balanced_split(dims):
  """the k in [1, len(dims)] for which the dense sizes of dims[:k] and dims[k:] are closest"""
  total, best, split, left = math.prod(dims), None, 1, 1
  for i in range(1, len(dims) + 1):
    left *= dims[i - 1]
    cost = max(left, total // max(left, 1))
    if best is None or cost < best:
      best, split = cost, i
  return split


def permutation_map(be, indices, permutation):
  """Device int64 map of block-sparse transposition (blocksparsetensor.py:803-860 `contiguous`): for a data vector stored
  over the legs `indices`, data[map] is the data vector stored over the legs [indices[p] for p in permutation], element
  for element what the reference's `contiguous(permutation)` computes.

  Built once per (legs, permutation) and cached.  Two `_device_sector_maps` with the same row legs list the same elements
  in the same order (sector after sector, row-major): the source legs viewed in the target order (map_s: positions in the
  source vector) and the permuted legs in identity order (map_t: positions in the target vector).  So the map is one
  int64 scatter, map[map_t] = map_s."""
  permutation = [int(p) for p in permutation]
  key = ("perm", tuple(ix.key() for ix in indices), tuple(permutation))
  hit = _MAP_CACHE.get(key)
  if hit is not None:
    return hit
  target = [indices[p] for p in permutation]
  part = _balanced_split([ix.dim for ix in target])
  qs, ds, map_s, _ = _device_sector_maps(be, indices, permutation, part)
  qt, dt, map_t, _ = _device_sector_maps(be, target, list(range(len(target))), part)
  if not (np.array_equal(qs, qt) and np.array_equal(ds, dt)):
    raise RuntimeError("block-sparse transposition: sector bookkeeping mismatch (internal error)")
  nnz = BlockSparseTensor._nnz(indices)  # pylint: disable=protected-access
  out = be.torch.empty(max(nnz, 1), dtype=be.torch.int64, device=be.device)
  L.check(be.lib.tnb200_gather(map_s.data_ptr(), map_t.data_ptr(), out.data_ptr(), nnz, L.I64, 1,
                               be._stream()))  # pylint: disable=protected-access
  _MAP_CACHE[key] = out
  return out


def gather(be, data, dev_map, n):
  """data[dev_map[:n]] as a new 1-D device vector (one `tnb200_gather`)."""
  out = be._new((n,), data.code)  # pylint: disable=protected-access
  if n:
    L.check(be.lib.tnb200_gather(data.t.data_ptr(), dev_map.data_ptr(), out.t.data_ptr(), n, data.code, 0,
                                 be._stream()))  # pylint: disable=protected-access
  return out


# ===================================================================================== svd
def _truncate_sectors(singvals, max_singular_values=None, max_truncation_error=None, relative=False):
  """The cross-sector truncation of backends/symmetric/decompositions.py:63-136, restated on host
  (integer outputs: how many singular values each sector keeps).  `singvals` = list of descending
  per-sector arrays.  Returns (kept counts, list of discarded-value arrays)."""
  orig = [len(s) for s in singvals]
  total = int(np.sum(orig)) if orig else 0
  if max_singular_values is not None and max_singular_values >= total:
    max_singular_values = None
  if max_truncation_error is None and max_singular_values is None:
    return orig, [np.zeros(0, dtype=s.dtype) for s in singvals]
  max_d = max(orig) if orig else 0
  ext = np.stack([np.append(s, np.zeros(max_d - len(s), dtype=s.dtype)) for s in singvals], axis=1) \
      if singvals else np.empty((0, 0))
  flat = np.ravel(ext)
  inds = np.argsort(flat, kind="stable")
  disc = np.zeros(0, dtype=np.int64)
  if max_truncation_error is not None:
    if relative and singvals:
      max_truncation_error = max_truncation_error * np.max([s[0] for s in singvals])
    kept_mask = np.sqrt(np.cumsum(np.square(flat[inds]))) > max_truncation_error
    disc = inds[np.logical_not(kept_mask)]
    inds = inds[kept_mask]
  if max_singular_values is not None:
    if max_singular_values > total:
      max_singular_values = total
    if max_singular_values < len(inds):
      disc = np.append(disc, inds[:(-1) * max_singular_values])
      inds = inds[(-1) * max_singular_values:]
  ncol = ext.shape[1]
  keep = np.divmod(inds, ncol) if ncol else (np.zeros(0, dtype=np.int64),) * 2
  dsc = np.divmod(disc, ncol) if ncol else (np.zeros(0, dtype=np.int64),) * 2
  kept = [int(np.sum(keep[1] == n)) for n in range(ncol)]
  discarded = []
  for n in range(ncol):
    d = ext[dsc[0][dsc[1] == n], dsc[1][dsc[1] == n]][::-1]
    discarded.append(d[:orig[n] - kept[n]])
  return kept, discarded


def _pack_sectors(tensor, nl):
  """The charge sectors of the matrix view (legs order[:nl] | order[nl:]) packed row-major, sector after sector, into one
  device buffer by one `tnb200_gather`.  Returns (qnums, ms, ns, a_off (nsect + 1 element offsets), buffer)."""
  be = tensor.backend
  qn, dims, maps = _sector_maps(tensor.indices, tensor.order, nl)
  ms, ns = dims[:, 0], dims[:, 1]
  a_off = np.zeros(len(maps) + 1, dtype=np.int64); a_off[1:] = np.cumsum(ms * ns)
  a_buf = be._new((int(a_off[-1]),), tensor.data.code)  # pylint: disable=protected-access
  gmap = _up(be, np.concatenate(maps) if maps else np.zeros(0, dtype=np.int64))
  L.check(be.lib.tnb200_gather(tensor.data.t.data_ptr(), gmap.data_ptr(), a_buf.t.data_ptr(), int(a_off[-1]), tensor.data.code, 0,
                               be._stream()))  # pylint: disable=protected-access
  return qn, ms, ns, a_off, a_buf


def _up(be, x):
  return be.torch.from_numpy(np.ascontiguousarray(x, dtype=np.int64)).to(be.device)


def _take(be, buf, idx, code):
  """buf[idx] as a new device vector (one `tnb200_gather`)."""
  out = be._new((len(idx),), code)  # pylint: disable=protected-access
  if len(idx):
    L.check(be.lib.tnb200_gather(buf.t.data_ptr(), _up(be, idx).data_ptr(), out.t.data_ptr(), len(idx), code, 0,
                                 be._stream()))  # pylint: disable=protected-access
  return out


def _cat(xs):
  return np.concatenate(xs) if xs else np.zeros(0, dtype=np.int64)


def _factor_tensors(tensor, nl, qn, ms, ns, kept, l_buf, l_off, r_buf, r_off):
  """The block-sparse factors of a per-sector decomposition A_q = L_q R_q with L_q (m x r) and R_q (r x n), r = min(m, n),
  row-major at l_off[q] / r_off[q] of the packed buffers, keeping the first kept[q] columns of L_q and rows of R_q.

  Returns (L, R): L legs = left legs + [bond], bond flow True; R legs = [bond] + right legs, bond flow False
  (block_sparse/linalg.py:343-392).  The bond carries the sector charge kept[q] times, sector-major: (k,) charges for one
  symmetry, (k, nsym) with the tensor's per-component moduli for a product."""
  be, code = tensor.backend, tensor.data.code
  l_idx, r_idx, bond_q = [], [], []
  for q, k in enumerate(kept):
    if k == 0:
      continue
    m_, n_, r_ = int(ms[q]), int(ns[q]), int(min(ms[q], ns[q]))
    b = np.arange(k)
    l_idx.append((l_off[q] + np.arange(m_)[None, :] * r_ + b[:, None]).ravel())      # (k x m): l_q[:, :k].T
    r_idx.append((r_off[q] + b[:, None] * n_ + np.arange(n_)[None, :]).ravel())      # (k x n): r_q[:k, :]
    bond_q.append(np.repeat(qn[q:q + 1], k, axis=0).astype(np.int64))
  l_data = _take(be, l_buf, _cat(l_idx), code)
  r_data = _take(be, r_buf, _cat(r_idx), code)
  mod = tensor.indices[0].modulus if tensor.indices else None
  bond_charges = np.concatenate(bond_q) if bond_q else np.zeros((0,) + qn.shape[1:], dtype=np.int64)
  left = [tensor.indices[tensor.order[i]] for i in range(nl)]
  right = [tensor.indices[tensor.order[i]] for i in range(nl, tensor.ndim)]
  bond_l = Index(bond_charges, True, mod)
  bond_r = Index(bond_charges, False, mod)
  Lt = BlockSparseTensor(l_data, [bond_l] + left, list(range(1, nl + 1)) + [0], be)
  Rt = BlockSparseTensor(r_data, [bond_r] + right, None, be)
  assert l_data.size == BlockSparseTensor._nnz([bond_l] + left) and r_data.size == BlockSparseTensor._nnz([bond_r] + right)  # pylint: disable=protected-access
  return Lt, Rt


def svd(tensor, pivot_axis, max_singular_values=None, max_truncation_error=None, relative=False):
  """Block-sparse SVD (backends/symmetric/decompositions.py:27-216): one small SVD per charge sector —
  all sectors in ONE `tnb200_svd_batched` launch — then the reference's global truncation.

  Returns (U, S, V, Sdisc): U legs = left legs + [bond], V legs = [bond] + right legs (block-sparse);
  S = dict(values=1-D device tensor of kept singular values, sector-major, index=bond Index);
  Sdisc = host array of the discarded singular values (sector-major)."""
  be = tensor.backend
  torch = be.torch
  nl = pivot_axis if pivot_axis >= 0 else tensor.ndim + pivot_axis
  code = tensor.data.code
  if code not in (L.F64, L.F32, L.C64, L.C128):
    raise TypeError("block-sparse svd needs a float32/float64/complex tensor")
  qn, ms, ns, a_off, a_buf = _pack_sectors(tensor, nl)
  nsect = len(qn)
  rs = np.minimum(ms, ns)
  u_off = np.zeros(nsect + 1, dtype=np.int64); u_off[1:] = np.cumsum(ms * rs)
  s_off = np.zeros(nsect + 1, dtype=np.int64); s_off[1:] = np.cumsum(rs)
  v_off = np.zeros(nsect + 1, dtype=np.int64); v_off[1:] = np.cumsum(rs * ns)
  up = lambda x: _up(be, x)
  st = be._stream()  # pylint: disable=protected-access
  u_buf = be._new((int(u_off[-1]),), code)  # pylint: disable=protected-access
  s_buf = be._new((int(s_off[-1]),), T.real_code(code))  # pylint: disable=protected-access
  v_buf = be._new((int(v_off[-1]),), code)  # pylint: disable=protected-access
  d_dims, d_ao, d_uo, d_so, d_vo = up(np.stack([ms, ns], axis=1).reshape(-1)), up(a_off), up(u_off), up(s_off), up(v_off)
  status = torch.zeros(1, dtype=torch.int32, device=be.device)
  rc = be.lib.tnb200_svd_batched(a_buf.t.data_ptr(), code, nsect, d_dims.data_ptr(), d_ao.data_ptr(), u_buf.t.data_ptr(),
                                 d_uo.data_ptr(), s_buf.t.data_ptr(), d_so.data_ptr(), v_buf.t.data_ptr(), d_vo.data_ptr(),
                                 int(ms.max()) if nsect else 0, int(ns.max()) if nsect else 0, status.data_ptr(), st)
  if rc == L.ERR_UNSUPPORTED:
    # a sector too large for the shared-memory kernel: one blocked-Jacobi SVD per sector
    for q in range(nsect):
      m_, n_, r_ = int(ms[q]), int(ns[q]), int(rs[q])
      a_q = B200Tensor(a_buf.t[a_off[q]:a_off[q + 1]].view(m_, n_), code)
      u_q = B200Tensor(u_buf.t[u_off[q]:u_off[q + 1]].view(m_, r_), code)
      s_q = B200Tensor(s_buf.t[s_off[q]:s_off[q + 1]], T.real_code(code))
      v_q = B200Tensor(v_buf.t[v_off[q]:v_off[q + 1]].view(r_, n_), code)
      L.check(be.lib.tnb200_svd(a_q.ref(), u_q.ref(), s_q.ref(), v_q.ref(), None, st))
  else:
    L.check(rc)
  s_host = s_buf.to_host()            # the one D2H of this path: data-dependent output sizes
  if int(status.item()) != 0:
    raise RuntimeError("block-sparse svd: a sector failed to converge")
  singvals = [s_host[s_off[q]:s_off[q + 1]] for q in range(nsect)]
  kept, discarded = _truncate_sectors(singvals, max_singular_values, max_truncation_error, relative)
  U, V = _factor_tensors(tensor, nl, qn, ms, ns, kept, u_buf, u_off, v_buf, v_off)
  s_vals = _take(be, s_buf, _cat([s_off[q] + np.arange(k) for q, k in enumerate(kept) if k]), T.real_code(code))
  ktot = int(np.sum(kept)) if kept else 0
  s_disc = np.concatenate(discarded) if discarded else np.zeros(0)
  disc_q = [np.repeat(qn[q:q + 1], len(d), axis=0).astype(np.int64) for q, d in enumerate(discarded)]
  disc_q = np.concatenate(disc_q) if disc_q else np.zeros((0,) + qn.shape[1:], dtype=np.int64)
  return U, dict(values=s_vals, index=U.indices[0], kept=kept, ktot=ktot, discarded=s_disc, discarded_charges=disc_q), V, s_disc


# ===================================================================================== qr / rq
def _wide_bytes(code):
  """bytes of the f64 / c128 element tnb200_qr_batched computes in"""
  return 16 if T.is_complex_code(code) else 8


def _qr_sectors(tensor, pivot_axis, adjoint):
  """A_q = L_q R_q for every charge sector of the matrix view (legs order[:nl] | order[nl:]): the QR of A_q (adjoint = 0:
  L = Q, R = R) or the RQ composed from the QR of A_q^H (adjoint = 1: L = R, R = Q).  Sectors with
  8 or 16 bytes * m n <= `_lib.QR_BATCHED_MAX_BYTES` run in ONE `tnb200_qr_batched` launch, each larger one through
  `tnb200_qr` on its slice of the packed buffer.  No host synchronisation: the factor sizes follow from the charges."""
  be = tensor.backend
  nl = pivot_axis if pivot_axis >= 0 else tensor.ndim + pivot_axis
  code = tensor.data.code
  if code not in (L.F64, L.F32, L.C64, L.C128):
    raise TypeError("block-sparse qr needs a float32/float64/complex tensor")
  qn, ms, ns, a_off, a_buf = _pack_sectors(tensor, nl)
  rs = np.minimum(ms, ns)
  l_off = np.zeros(len(qn) + 1, dtype=np.int64); l_off[1:] = np.cumsum(ms * rs)
  r_off = np.zeros(len(qn) + 1, dtype=np.int64); r_off[1:] = np.cumsum(rs * ns)
  l_buf = be._new((int(l_off[-1]),), code)  # pylint: disable=protected-access
  r_buf = be._new((int(r_off[-1]),), code)  # pylint: disable=protected-access
  st = be._stream()  # pylint: disable=protected-access
  elems = ms * ns
  small = (elems > 0) & (elems * _wide_bytes(code) <= L.QR_BATCHED_MAX_BYTES)
  batch = np.nonzero(small)[0]
  # the kernel writes Q at q_off and R at r_off; with adjoint, R_q = R'^H is the left factor and Q_q = Q'^H the right one
  q_buf, q_off, rr_buf, rr_off = (l_buf, l_off, r_buf, r_off) if not adjoint else (r_buf, r_off, l_buf, l_off)
  if batch.size:
    d_dims, d_ao = _up(be, np.stack([ms[batch], ns[batch]], axis=1).reshape(-1)), _up(be, a_off[batch])
    d_qo, d_ro = _up(be, q_off[batch]), _up(be, rr_off[batch])
    L.check(be.lib.tnb200_qr_batched(a_buf.t.data_ptr(), code, int(batch.size), d_dims.data_ptr(), d_ao.data_ptr(),
                                      q_buf.t.data_ptr(), d_qo.data_ptr(), rr_buf.t.data_ptr(), d_ro.data_ptr(),
                                      int(elems[batch].max()), int(adjoint), st))
  for q in np.nonzero(~small & (elems > 0))[0]:
    m_, n_, r_ = int(ms[q]), int(ns[q]), int(rs[q])
    a_q = B200Tensor(a_buf.t[a_off[q]:a_off[q + 1]].view(m_, n_), code)
    l_q = B200Tensor(l_buf.t[l_off[q]:l_off[q + 1]].view(m_, r_), code)
    r_q = B200Tensor(r_buf.t[r_off[q]:r_off[q + 1]].view(r_, n_), code)
    if not adjoint:
      L.check(be.lib.tnb200_qr(a_q.ref(), l_q.ref(), r_q.ref(), 0, st))
    else:
      rr, qq = be.rq(a_q, 1)
      L.check(be.lib.tnb200_copy(rr.ref(), l_q.ref(), 0, st))
      L.check(be.lib.tnb200_copy(qq.ref(), r_q.ref(), 0, st))
  return _factor_tensors(tensor, nl, qn, ms, ns, [int(r) for r in rs], l_buf, l_off, r_buf, r_off)


def qr(tensor, pivot_axis):
  """Block-sparse QR (block_sparse/linalg.py:300-393 behind backends/symmetric/decompositions.py:219-231): np.linalg.qr's
  reduced factors of every charge sector.  Returns (Q, R): Q legs = left legs + [bond] (bond flow True), R legs =
  [bond] + right legs (bond flow False); the bond carries each sector's charge min(m_q, n_q) times, ascending."""
  return _qr_sectors(tensor, pivot_axis, 0)


def rq(tensor, pivot_axis):
  """Block-sparse RQ (backends/symmetric/decompositions.py:234-248): per sector, the QR of A_q^H conjugate-transposed
  back, A_q = R_q Q_q with R_q = R'^H (m x r) and Q_q = Q'^H (r x n).  Returns (R, Q) with the leg layout of `qr`:
  R legs = left legs + [bond] (flow True), Q legs = [bond] + right legs (flow False)."""
  return _qr_sectors(tensor, pivot_axis, 1)
