"""`symmetric_b200`: the reference's `SymmetricBackend` with its hot operations on the B200.

Reference: `tensornetwork/backends/symmetric/symmetric_backend.py:30` (class), `:38-40` (tensordot ->
`block_sparse.tensordot`, blocksparsetensor.py:925-1108), `:50-59` (svd -> backends/symmetric/
decompositions.py:27-216), `:61-81` (qr / rq -> decompositions.py:219-248 -> block_sparse/linalg.py:300-393).
Registered under the name "symmetric_b200" in `backend_factory._BACKENDS` when the reference package is importable,
so `tn.Node(BlockSparseTensor, backend="symmetric_b200")`, `tn.split_node*`, `FiniteMPS` canonicalisation and
`FiniteDMRG` on block-sparse MPS run the grouped sector kernels (`tnb200_blocksparse_tensordot`, `tnb200_svd_batched`,
`tnb200_qr_batched`) of `tensornetwork_b200.blocksparse`.

Scope (stated, not hidden): tensors stay the reference's own `BlockSparseTensor` objects — charges, flows,
leg fusion (`reshape`), lazy transposition and every elementwise helper on the nnz vector are the reference's
host code, inherited unchanged; `tensordot`, `svd`, `qr` and `rq` — where the reference spends its time (SURVEY 8a
rows a11, a12; `qr` / `rq` at every site of MPS canonicalisation and one-site DMRG) — upload the nnz vectors, run on
the device and download the result.  `qr` / `rq` build their own sector maps, so they also factor the dimension-1
boundary legs of a finite MPS, on which the reference's host path fails under numpy 2.  Supported symmetries: U(1) and
Z_N charges, and the reference's product charges built from them (a `BaseCharge` with several `charge_types`, e.g.
U(1) x U(1) for particle number and S_z, or U(1) x Z_2); sectors and bond charges come out in the reference's order.
Other charge types raise NotImplementedError.  The two degenerate forms of tensordot that are not sector contractions
(outer product and full inner product) go to the reference implementation, which is a numpy dot / outer of the data
vectors.
"""
import numpy as np

from . import blocksparse as bsp

NAME = "symmetric_b200"
_CLASS = None


def _modulus(charge):
  """One entry per charge component: None for U(1), N for Z_N; raises for anything this adapter does not cover.  The
  reference builds Z_N classes in a factory (`charge.py:549-600`, class name `ModularCharge`) without recording N; the dual
  of charge 1 reveals it: -1 for U(1), N-1 for Z_N (Z2: 1)."""
  mods = []
  for t in charge.charge_types:
    d = int(np.asarray(t.dual_charges(np.array([1], dtype=np.int16))).ravel()[0])
    if d == -1:
      mods.append(None)
    elif d >= 1:
      mods.append(d + 1)
    else:
      raise NotImplementedError("symmetric_b200: unsupported charge type {}".format(t))
  return tuple(mods)


def _bond_charge(tensor, q):
  """the reference charge object of a bond with charges q ((k,) or (k, nsym)), of the type and charge_types of the
  tensor's first leg"""
  c0 = tensor._charges[0]  # pylint: disable=protected-access
  return type(c0)(np.asarray(q, dtype=np.int16), charge_types=c0.charge_types)


def _to_device(tensor, be):
  """reference BlockSparseTensor -> (ours over the ELEMENTARY legs, leg groups): groups[n] = positions (in our logical
  order = the reference's flat order) of the elementary legs of logical leg n."""
  charges, flows = tensor._charges, tensor._flows  # pylint: disable=protected-access
  indices = [bsp.Index(np.asarray(c.charges).astype(np.int64), bool(f), _modulus(c)) for c, f in zip(charges, flows)]
  flat, groups, s = [], [], 0
  for leg in tensor._order:  # pylint: disable=protected-access
    flat.extend(int(o) for o in leg)
    groups.append(list(range(s, s + len(leg))))
    s += len(leg)
  data = be.convert_to_tensor(np.ascontiguousarray(tensor.data))
  return bsp.BlockSparseTensor(data, indices, flat, be), groups


def _make_class():
  global _CLASS
  if _CLASS is not None:
    return _CLASS
  from tensornetwork.backends.symmetric import symmetric_backend as sb  # pylint: disable=import-outside-toplevel
  from tensornetwork.block_sparse.blocksparsetensor import BlockSparseTensor, ChargeArray  # pylint: disable=import-outside-toplevel

  class SymmetricB200Backend(sb.SymmetricBackend):
    """See the module docstring."""

    def __init__(self):
      super().__init__()
      self.name = NAME
      from .backend import get_instance  # pylint: disable=import-outside-toplevel
      self.device_backend = get_instance()
      self.lib = self.device_backend.lib

    # ------------------------------------------------------------------ a11
    def tensordot(self, a, b, axes):
      if not isinstance(a, BlockSparseTensor) or not isinstance(b, BlockSparseTensor):
        return super().tensordot(a, b, axes)
      if isinstance(axes, (int, np.integer)):
        n = int(axes)
        axes1, axes2 = list(range(a.ndim - n, a.ndim)), list(range(n))
      elif isinstance(axes[0], (int, np.integer)):
        return super().tensordot(a, b, axes)            # the reference's own argument check / error
      else:
        axes1, axes2 = [int(x) for x in axes[0]], [int(x) for x in axes[1]]
      degenerate = len(axes1) == 0 or (len(axes1) == a.ndim and len(axes2) == b.ndim)
      if degenerate or len(axes1) != len(axes2) or a.dtype != b.dtype:
        return super().tensordot(a, b, axes)            # outer / inner product, or the reference's ValueError
      be = self.device_backend
      da, ga = _to_device(a, be)
      db, gb = _to_device(b, be)
      ea = [p for x in axes1 for p in ga[x]]
      eb = [p for x in axes2 for p in gb[x]]
      try:
        dc = bsp.tensordot(da, db, (ea, eb))
      except ValueError:
        super().tensordot(a, b, axes)                   # mismatching charges / flows: raise exactly what the reference raises
        raise                                           # anything else, a device error included, is not the reference's
      free1 = [n for n in range(a.ndim) if n not in axes1]
      free2 = [n for n in range(b.ndim) if n not in axes2]
      charges, flows, order, s = [], [], [], 0
      for t, free in ((a, free1), (b, free2)):
        for n in free:
          leg = t._order[n]  # pylint: disable=protected-access
          charges.extend(t._charges[o] for o in leg)  # pylint: disable=protected-access
          flows.extend(t._flows[o] for o in leg)  # pylint: disable=protected-access
          order.append(list(range(s, s + len(leg))))
          s += len(leg)
      return BlockSparseTensor(data=dc.data.to_host(), charges=charges, flows=flows, order=order, check_consistency=False)

    # ------------------------------------------------------------------ a12
    def svd(self, tensor, pivot_axis=-1, max_singular_values=None, max_truncation_error=None, relative=False):
      if not isinstance(tensor, BlockSparseTensor):
        return super().svd(tensor, pivot_axis, max_singular_values, max_truncation_error, relative)
      be = self.device_backend
      left_dims, right_dims = tensor.shape[:pivot_axis], tensor.shape[pivot_axis:]
      dt, groups = _to_device(tensor, be)
      nl_logical = len(left_dims)
      nl = sum(len(g) for g in groups[:nl_logical])
      U, S, V, _ = bsp.svd(dt, nl, max_singular_values, max_truncation_error, relative)
      bond = _bond_charge(tensor, S["index"].charges)
      flat = dt.order
      left_c = [tensor._charges[o] for o in flat[:nl]]  # pylint: disable=protected-access
      left_f = [tensor._flows[o] for o in flat[:nl]]  # pylint: disable=protected-access
      right_c = [tensor._charges[o] for o in flat[nl:]]  # pylint: disable=protected-access
      right_f = [tensor._flows[o] for o in flat[nl:]]  # pylint: disable=protected-access
      u = BlockSparseTensor(U.data.to_host(), charges=[bond] + left_c, flows=[True] + left_f,
                            order=[[0], list(range(1, nl + 1))], check_consistency=False).transpose((1, 0))
      v = BlockSparseTensor(V.data.to_host(), charges=[bond] + right_c, flows=[False] + right_f,
                            order=[[0], list(range(1, len(right_c) + 1))], check_consistency=False)
      s = ChargeArray(S["values"].to_host(), [bond], [False])
      sdisc = ChargeArray(S["discarded"], [_bond_charge(tensor, S["discarded_charges"])], [False])
      k = s.shape[0]
      return u.reshape(tuple(left_dims) + (k,)), s, v.reshape((k,) + tuple(right_dims)), sdisc

    # ------------------------------------------------------------------ qr / rq
    def _split(self, tensor, pivot_axis, factor):
      """(left, right) block-sparse factors of `bsp.qr` / `bsp.rq` as the reference's decompositions.qr / rq shape them:
      left = left legs + [bond] (bond flow True), right = [bond] + right legs (bond flow False)."""
      left_dims, right_dims = tensor.shape[:pivot_axis], tensor.shape[pivot_axis:]
      dt, groups = _to_device(tensor, self.device_backend)
      nl = sum(len(g) for g in groups[:len(left_dims)])
      lf, rf = factor(dt, nl)
      bond = _bond_charge(tensor, lf.indices[0].charges)
      flat = dt.order
      cf = lambda legs: ([tensor._charges[o] for o in legs], [tensor._flows[o] for o in legs])  # pylint: disable=protected-access
      (left_c, left_f), (right_c, right_f) = cf(flat[:nl]), cf(flat[nl:])
      left = BlockSparseTensor(lf.data.to_host(), charges=[bond] + left_c, flows=[True] + left_f,
                               order=[[0], list(range(1, nl + 1))], check_consistency=False).transpose((1, 0))
      right = BlockSparseTensor(rf.data.to_host(), charges=[bond] + right_c, flows=[False] + right_f,
                                order=[[0], list(range(1, len(right_c) + 1))], check_consistency=False)
      k = lf.indices[0].dim
      return left.reshape(tuple(left_dims) + (k,)), right.reshape((k,) + tuple(right_dims))

    def qr(self, tensor, pivot_axis=-1, non_negative_diagonal=False):
      if non_negative_diagonal or not isinstance(tensor, BlockSparseTensor):
        return super().qr(tensor, pivot_axis, non_negative_diagonal)   # the reference's NotImplementedError / host path
      return self._split(tensor, pivot_axis, bsp.qr)

    def rq(self, tensor, pivot_axis=-1, non_negative_diagonal=False):
      if non_negative_diagonal or not isinstance(tensor, BlockSparseTensor):
        return super().rq(tensor, pivot_axis, non_negative_diagonal)
      return self._split(tensor, pivot_axis, bsp.rq)

  _CLASS = SymmetricB200Backend
  return _CLASS


def register():
  """Adds "symmetric_b200" to the reference's backend registry (backend_factory.py:22-28).  Returns the class, or None
  when the reference package is not importable."""
  try:
    from tensornetwork.backends import backend_factory  # pylint: disable=import-outside-toplevel
  except Exception:  # pylint: disable=broad-except
    return None
  cls = _make_class()
  backend_factory._BACKENDS[NAME] = cls  # pylint: disable=protected-access
  return cls
