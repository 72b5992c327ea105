"""`symmetric_b200`: the reference's `SymmetricBackend` with its hot operations on the B200.

Reference: `tensornetwork/backends/symmetric/symmetric_backend.py:30` (class), `:38-40` (tensordot ->
`block_sparse.tensordot`, blocksparsetensor.py:925-1108), `:50-59` (svd -> backends/symmetric/
decompositions.py:27-216), `:61-81` (qr / rq -> decompositions.py:219-248 -> block_sparse/linalg.py:300-393).
Registered under the name "symmetric_b200" in `backend_factory._BACKENDS` when the reference package is importable,
so `tn.Node(BlockSparseTensor, backend="symmetric_b200")`, `tn.split_node*`, `FiniteMPS` canonicalisation and
`FiniteDMRG` on block-sparse MPS run the grouped sector kernels (`tnb200_blocksparse_tensordot`, `tnb200_svd_batched`,
`tnb200_qr_batched`) of `tensornetwork_b200.blocksparse`.

Residency rule: an operation on `symmetric_b200` with a device-resident input returns device-resident outputs; host
inputs give host outputs, exactly as the reference does.  A device-resident tensor is a `DeviceBlockSparseTensor`
(`resident_class()`): a subclass of the reference's `BlockSparseTensor` whose nnz vector is a 1-D `B200Tensor` in HBM, so
`tn.Node`, `ncon`, `FiniteMPS` and `FiniteDMRG` accept it unchanged.  Charges, flows and the lazy leg order stay on the
host.  `transpose`, `reshape`, `conj`, scalar `*` and `/`, unary `-`, `+`, `-`, `copy` and `contiguous` (one
`tnb200_gather` through a cached permutation map, bit for bit the reference's layout) keep the data on the device.
Reading `.data` downloads it once, as a read-only array; assigning a numpy array to `.data` makes the tensor host-backed.
`item` and `todense` download.

`eigsh_lanczos` uploads the initial state and every block-sparse argument once, runs the device Lanczos of
`tensornetwork_b200.lanczos` on the nnz vectors (one norm read per step) and returns resident eigenvectors.  `FiniteDMRG`
sends them on to `norm`, `/`, `svd` / `qr` / `rq` and `ncon`, so the MPS tensors and environments it touches stay in HBM
for the rest of the sweep.

Host inputs: tensors are the reference's own `BlockSparseTensor` objects; `tensordot`, `svd`, `qr` and `rq` — where the
reference spends its time (SURVEY 8a rows a11, a12; `qr` / `rq` at every site of MPS canonicalisation and one-site DMRG)
— upload the nnz vectors, run on the device and download the result.  `qr` / `rq` build their own sector maps, so they
also factor the dimension-1 boundary legs of a finite MPS, on which the reference's host path fails under numpy 2.
Supported symmetries: U(1) and Z_N charges, and the reference's product charges built from them (a `BaseCharge` with
several `charge_types`, e.g. U(1) x U(1) for particle number and S_z, or U(1) x Z_2); sectors and bond charges come out in
the reference's order.  Other charge types raise NotImplementedError.  The two degenerate forms of tensordot that are not
sector contractions (outer product and full inner product) go to the reference implementation, which is a numpy dot /
outer of the data vectors: their result is on the host whatever the inputs.
"""
import numpy as np

from . import blocksparse as bsp

NAME = "symmetric_b200"
_CLASS = None
_RESIDENT = None


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


def _indices(charges, flows):
  """our Index per elementary leg"""
  return [bsp.Index(np.asarray(c.charges).astype(np.int64), bool(f), _modulus(c)) for c, f in zip(charges, flows)]


def _is_resident(tensor):
  return _RESIDENT is not None and isinstance(tensor, _RESIDENT) and tensor.device_data is not None


def _device_vector(tensor, be):
  """the nnz vector on the device: a resident tensor's own vector (no copy), else one upload"""
  if _is_resident(tensor):
    return tensor.device_data
  return be.convert_to_tensor(np.ascontiguousarray(tensor.data))


def _to_device(tensor, be):
  """reference BlockSparseTensor -> (ours over the ELEMENTARY legs, leg groups): groups[n] = positions (in our logical
  order = the reference's flat order) of the elementary legs of logical leg n."""
  indices = _indices(tensor._charges, tensor._flows)  # pylint: disable=protected-access
  flat, groups, s = [], [], 0
  for leg in tensor._order:  # pylint: disable=protected-access
    flat.extend(int(o) for o in leg)
    groups.append(list(range(s, s + len(leg))))
    s += len(leg)
  return bsp.BlockSparseTensor(_device_vector(tensor, be), indices, flat, be), groups


def resident_class():
  """The device-resident BlockSparseTensor class, or None when the reference package is not importable."""
  try:
    _make_class()
  except ImportError:
    return None
  return _RESIDENT


def _make_class():
  global _CLASS, _RESIDENT
  if _CLASS is not None:
    return _CLASS
  import copy  # pylint: disable=import-outside-toplevel
  from tensornetwork.backends.symmetric import symmetric_backend as sb  # pylint: disable=import-outside-toplevel
  from tensornetwork.block_sparse.blocksparsetensor import BlockSparseTensor, ChargeArray, compare_shapes  # pylint: disable=import-outside-toplevel
  from .backend import get_instance  # pylint: disable=import-outside-toplevel
  from .tensor import B200Tensor  # pylint: disable=import-outside-toplevel

  class DeviceBlockSparseTensor(BlockSparseTensor):
    """The reference's BlockSparseTensor with its nnz vector in HBM (a 1-D B200Tensor, `device_data`); charges, flows and
    the leg order stay on the host.  See the module docstring for what stays on the device and what downloads."""

    def __init__(self, data, charges, flows, order=None, check_consistency=False):  # pylint: disable=super-init-not-called,unused-argument
      self._charges = charges
      self._flows = np.asarray(flows)
      self._order = [[n] for n in range(len(charges))] if order is None else order
      self.data = data

    # ---------------------------------------------------------------- storage
    @property
    def data(self):
      """the nnz vector on the host: downloaded once and read-only while the tensor is resident"""
      if self._host is None:
        self._host = self._download()
      return self._host

    @data.setter
    def data(self, value):
      if isinstance(value, B200Tensor):
        if value.ndim != 1:
          raise ValueError("the nnz vector of a block-sparse tensor is 1-D, got shape {}".format(value.shape))
        self.device_data, self._host = value, None
      else:                                              # a host array: the tensor becomes host-backed
        self.device_data, self._host = None, np.asarray(value).reshape(-1)

    def _download(self):
      host = self.device_data.to_host()
      host.flags.writeable = False
      return host

    @property
    def dtype(self):
      return np.dtype(self.device_data.dtype) if self.device_data is not None else self.data.dtype

    def _like(self, dev, charges=None, flows=None, order=None):
      return DeviceBlockSparseTensor(dev, self._charges if charges is None else charges,
                                     self._flows if flows is None else flows, self._order if order is None else order)

    def _shell(self):
      """a data-less reference tensor of the same legs: runs the reference's metadata logic and argument checks"""
      return BlockSparseTensor(np.empty(0, dtype=self.dtype), self._charges, self._flows, self._order, False)

    # ---------------------------------------------------------------- metadata-only views
    def transpose(self, order=np.asarray([1, 0]), shuffle=False):
      if self.device_data is None:
        return super().transpose(order, shuffle)
      out = self._like(self.device_data, order=self._shell().transpose(order)._order)  # pylint: disable=protected-access
      return out.contiguous() if shuffle else out

    def reshape(self, shape):
      if self.device_data is None:
        return super().reshape(shape)
      return self._like(self.device_data, order=self._shell().reshape(shape)._order)  # pylint: disable=protected-access

    def contiguous(self, permutation=None, inplace=False):
      """the device form of the reference's `contiguous`: one gather through `blocksparse.permutation_map`"""
      if self.device_data is None:
        return super().contiguous(permutation, inplace)
      perm = [int(p) for p in (self.flat_order if permutation is None else permutation)]
      if perm == list(range(len(perm))):
        return self
      be = get_instance()
      pmap = bsp.permutation_map(be, _indices(self._charges, self._flows), perm)
      data = bsp.gather(be, self.device_data, pmap, self.device_data.size)
      new_pos = np.empty(len(perm), dtype=np.int64)
      new_pos[perm] = np.arange(len(perm))               # elementary leg o moves to position new_pos[o]
      order = [[int(new_pos[o]) for o in leg] for leg in self._order]
      charges = [self._charges[o] for o in perm]
      flows = np.asarray([self._flows[o] for o in perm])
      if not inplace:
        return DeviceBlockSparseTensor(data, charges, flows, order)
      self.data = data
      self._order, self._charges, self._flows = order, charges, flows
      return self

    def copy(self):
      if self.device_data is None:
        return super().copy()
      return DeviceBlockSparseTensor(get_instance().copy(self.device_data), [c.copy() for c in self._charges],
                                     self._flows.copy(), copy.deepcopy(self._order))

    # ---------------------------------------------------------------- arithmetic
    def conj(self):
      if self.device_data is None:
        return super().conj()
      return self._like(get_instance().conj(self.device_data), flows=list(np.logical_not(self._flows)))

    def _scaled(self, op, number, message):
      if not np.isscalar(number):
        raise TypeError(message.format(type(number)))
      return self._like(op(self.device_data, number))

    def __mul__(self, number):
      if self.device_data is None:
        return super().__mul__(number)
      return self._scaled(get_instance().multiply, number,
                          "Can only multiply BlockSparseTensor by a number. Found type {}")

    def __rmul__(self, number):
      if self.device_data is None:
        return super().__rmul__(number)
      return self._scaled(get_instance().multiply, number,
                          "Can only right-multiply BlockSparseTensor by a number. Found type {}")

    def __truediv__(self, number):
      if self.device_data is None:
        return super().__truediv__(number)
      return self._scaled(get_instance().divide, number,
                          "Can only divide BlockSparseTensor by a number. Found type {}")

    def __neg__(self):
      if self.device_data is None:
        return super().__neg__()
      return self._like(get_instance().negative(self.device_data))

    def _combine(self, other, op):
      """self (op) other with the reference's checks and storage alignment; the result is resident"""
      BlockSparseTensor._sub_add_protection(self._shell(), other)  # pylint: disable=protected-access
      self._align_storage_layout(other)
      be = get_instance()
      return self._like(op(_device_vector(self, be), _device_vector(other, be)))

    def __add__(self, other):
      if self.device_data is None and not _is_resident(other):
        return super().__add__(other)
      return self._combine(other, get_instance().addition)

    def __sub__(self, other):
      if self.device_data is None and not _is_resident(other):
        return super().__sub__(other)
      return self._combine(other, get_instance().subtraction)

  _RESIDENT = DeviceBlockSparseTensor

  def resident(tensor, be):
    """`tensor` as a resident tensor: itself when it is one, else one upload of its nnz vector"""
    if _is_resident(tensor):
      return tensor
    return DeviceBlockSparseTensor(be.convert_to_tensor(np.ascontiguousarray(tensor.data)), tensor._charges,  # pylint: disable=protected-access
                                   tensor._flows, tensor._order)  # pylint: disable=protected-access

  def _wrap(dev, keep, charges, flows, order):
    """a result's nnz vector as a resident tensor (keep) or downloaded into the reference's own class"""
    if keep:
      return DeviceBlockSparseTensor(dev, charges, flows, order)
    return BlockSparseTensor(dev.to_host(), charges=charges, flows=flows, order=order, check_consistency=False)

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
        return super().tensordot(a, b, axes)            # outer / inner product (on the host), or the reference's ValueError
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
      return _wrap(dc.data, _is_resident(a) or _is_resident(b), charges, flows, order)

    # ------------------------------------------------------------------ a12
    def svd(self, tensor, pivot_axis=-1, max_singular_values=None, max_truncation_error=None, relative=False):
      if not isinstance(tensor, BlockSparseTensor):
        return super().svd(tensor, pivot_axis, max_singular_values, max_truncation_error, relative)
      be = self.device_backend
      left_dims, right_dims = tensor.shape[:pivot_axis], tensor.shape[pivot_axis:]
      dt, groups = _to_device(tensor, be)
      res = _is_resident(tensor)
      nl_logical = len(left_dims)
      nl = sum(len(g) for g in groups[:nl_logical])
      U, S, V, _ = bsp.svd(dt, nl, max_singular_values, max_truncation_error, relative)
      bond = _bond_charge(tensor, S["index"].charges)
      flat = dt.order
      left_c = [tensor._charges[o] for o in flat[:nl]]  # pylint: disable=protected-access
      left_f = [tensor._flows[o] for o in flat[:nl]]  # pylint: disable=protected-access
      right_c = [tensor._charges[o] for o in flat[nl:]]  # pylint: disable=protected-access
      right_f = [tensor._flows[o] for o in flat[nl:]]  # pylint: disable=protected-access
      u = _wrap(U.data, res, [bond] + left_c, [True] + left_f, [[0], list(range(1, nl + 1))]).transpose((1, 0))
      v = _wrap(V.data, res, [bond] + right_c, [False] + right_f, [[0], list(range(1, len(right_c) + 1))])
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
      res = _is_resident(tensor)
      left = _wrap(lf.data, res, [bond] + left_c, [True] + left_f, [[0], list(range(1, nl + 1))]).transpose((1, 0))
      right = _wrap(rf.data, res, [bond] + right_c, [False] + right_f, [[0], list(range(1, len(right_c) + 1))])
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

    # ------------------------------------------------------------------ Lanczos
    def norm(self, tensor):
      if not _is_resident(tensor):
        return super().norm(tensor)
      # np.linalg.norm's result type: a numpy scalar of the real dtype; one scalar read
      return np.finfo(tensor.dtype).dtype.type(self.device_backend.norm(tensor.device_data).item())

    def eigsh_lanczos(self, A, args=None, initial_state=None, shape=None, dtype=None, num_krylov_vecs=20,  # pylint: disable=arguments-differ
                      numeig=1, tol=1E-8, delta=1E-8, ndiag=20, reorthogonalize=False, enable_caching=True):
      """The reference's block-sparse Lanczos (symmetric_backend.py:291-448) with the Krylov vectors in HBM: the initial
      state and every block-sparse argument are uploaded once, `lanczos.eigsh_lanczos` runs on the nnz vectors, and `A`
      gets resident tensors.  Eigenvalues as the reference returns them; eigenvectors resident.  `enable_caching` is
      accepted for the reference's signature and ignored: the sector and permutation maps are always cached."""
      del enable_caching
      if args is None:
        args = []
      if num_krylov_vecs < numeig:
        raise ValueError('`num_krylov_vecs` >= `numeig` required!')
      if numeig > 1 and not reorthogonalize:
        raise ValueError("Got numeig = {} > 1 and `reorthogonalize = False`. "
                         "Use `reorthogonalize=True` for `numeig > 1`".format(numeig))
      if initial_state is None:
        if (shape is None) or (dtype is None):
          raise ValueError("if no `initial_state` is passed, then `shape` and"
                           "`dtype` have to be provided")
        initial_state = self.randn(shape, dtype)
      if not isinstance(initial_state, BlockSparseTensor):
        raise TypeError("Expected a `BlockSparseTensor`. Got {}".format(type(initial_state)))
      from . import lanczos  # pylint: disable=import-outside-toplevel
      be = self.device_backend
      x0 = resident(initial_state, be).contiguous()       # a new tensor: the caller's keeps its layout
      args = [resident(a, be) if isinstance(a, BlockSparseTensor) else a for a in args]
      vec = lambda v: DeviceBlockSparseTensor(v, x0._charges, x0._flows, x0._order)  # pylint: disable=protected-access

      def matvec(v, *a):
        out = A(vec(v), *a)
        if not isinstance(out, BlockSparseTensor):
          raise TypeError("the matvec returned a {}, expected a `BlockSparseTensor`".format(type(out)))
        out = resident(out, be).contiguous()
        if not compare_shapes(out, x0):
          raise ValueError("the matvec result's charges or flows differ from those of `initial_state`")
        return out.device_data

      eta, states = lanczos.eigsh_lanczos(be, matvec, args, x0.device_data, num_krylov_vecs=num_krylov_vecs, numeig=numeig,
                                          tol=tol, delta=delta, ndiag=ndiag, reorthogonalize=reorthogonalize)
      return eta, [vec(s) for s in states]

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
