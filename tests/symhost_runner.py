"""Runs in a subprocess: the symmetric_b200 adapter (tensornetwork_b200/symmetric.py) driven by the REAL reference's callers
(the tests of tests/test_gpu_symmetric_adapter.py: block-sparse tn.Node @, split_node, ncon, backend.svd) with the device
layer replaced by tests/fake_lib.FakeLib (host memory): checks the conversion between the reference's BlockSparseTensor
and the elementary-leg form the kernels take, and that errors surface as the reference raises them."""
import numpy as np
import hostrun
tn, lib = hostrun.install(reference=True)
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import _lib  # noqa: E402
assert tb.registered_symmetric
hostrun.run_gpu_tests("test_gpu_symmetric_adapter.py", tn, lib)
# the contractions ran through the stand-in's kernel contract, not around it
assert lib.calls["tnb200_blocksparse_tensordot"] and not lib.raised["tnb200_blocksparse_tensordot"], (lib.calls, lib.raised)

# ---- device-side map construction (csrc/blocksparse_maps.cu; FakeLib carries a numpy transcription of the same five
# stages): the host tables (charge-degeneracy arithmetic) + the algorithm reproduce the lexsort-built maps exactly
from tensornetwork_b200 import blocksparse as bs
dbe = tb.get_backend()
rng = np.random.default_rng(1)
for trial in range(120):
  n = int(rng.integers(1, 6)); mod = [None, None, None, 2, 3, 4][rng.integers(0, 6)]
  idx = [bs.Index(rng.integers(-3, 4, rng.integers(1, 6)) if mod is None else rng.integers(0, mod, rng.integers(1, 6)),
                  bool(rng.integers(0, 2)), mod) for _ in range(n)]
  order = [int(x) for x in rng.permutation(n)]; part = int(rng.integers(0, n + 1))
  bs._MAP_CACHE.clear()
  q1, d1, m1 = bs._sector_maps(idx, order, part)
  q2, d2, dm, off = bs._device_sector_maps(dbe, idx, order, part)
  flat = np.concatenate(m1) if m1 else np.zeros(0, dtype=np.int64)
  assert np.array_equal(q1, q2) and np.array_equal(d1, d2) and np.array_equal(flat, dm.numpy()[:flat.shape[0]]), trial
print("device maps ok")

# ---- Z_N charges (the reference builds the class in a factory, charge.py:549): Z3 tensordot and svd through the adapter
from tensornetwork.backends import backend_factory as _bf
_be, _ref = _bf.get_backend("symmetric_b200"), _bf.get_backend("symmetric")
np.random.seed(7)
Z3 = tn.ZNCharge(3)
zl = [tn.Index(Z3.random(d, 0, 2), f) for d, f in zip((5, 6, 4, 7), (False, True, False, True))]
za = tn.BlockSparseTensor.random(zl, dtype=np.float64)
zb = tn.BlockSparseTensor.random([zl[3].copy().flip_flow(), zl[2].copy().flip_flow(), zl[0].copy()], dtype=np.float64)
g, w = _be.tensordot(za, zb, ([2, 3], [1, 0])), _ref.tensordot(za, zb, ([2, 3], [1, 0]))
assert g.shape == w.shape and np.allclose(g.data, w.data, atol=1e-12), "Z3 tensordot"
gu, gs, gv, _ = _be.svd(za, 2)
wu, ws, wv, _ = _ref.svd(za, 2)
assert np.allclose(gs.data, ws.data, atol=1e-10), "Z3 svd"
print("Z_N ok")

# errors: a device error surfaces instead of becoming the reference's host result; mismatched legs raise the reference's
# own message
lib.tnb200_blocksparse_tensordot = lambda *args: lib._fail(_lib.ERR_INVALID, "blocksparse: rejected by the stand-in")
hostrun.raises(ValueError, _be.tensordot, za, zb, ([2, 3], [1, 0]), match="rejected by the stand-in")
del lib.tnb200_blocksparse_tensordot
zs = tn.BlockSparseTensor.random([zl[3].copy(), zl[2].copy().flip_flow(), zl[0].copy()], dtype=np.float64)
assert (str(hostrun.raises(ValueError, _be.tensordot, za, zs, ([2, 3], [1, 0])))
        == str(hostrun.raises(ValueError, _ref.tensordot, za, zs, ([2, 3], [1, 0]))))
print("errors ok")
hostrun.done(lib)
