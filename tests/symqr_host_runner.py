"""Runs in a subprocess: tests/test_gpu_symmetric_qr.py against the symmetric_b200 adapter with the device layer replaced by
tests/fake_lib.FakeLib (host memory) plus a numpy `tnb200_qr_batched` that honours `adjoint` and, like the kernel, computes
f32 / c64 in double precision.  Checks the adapter's charge, flow and order bookkeeping and the split of sectors between
the batched launch and the per-sector tnb200_qr without a GPU."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from baseline import refenv
tn = refenv.load()
from tensornetwork_b200 import _lib, backend as tb_backend
import fake_lib

_HOST_QR = np.linalg.qr          # bound here: the MPS test replaces np.linalg.qr to prove the host QR never runs
_WIDE = {0: np.float64, 1: np.float64, 4: np.complex128, 5: np.complex128}


class QrFakeLib(fake_lib.FakeLib):
  def __init__(self):
    super().__init__()
    self.qr_batched_calls = []

  def tnb200_qr_batched(self, a, dtype, nprob, dims, aoff, q, qoff, r, roff, max_elems, adjoint, stream):
    nprob, max_elems = int(nprob), int(max_elems)
    if nprob < 0 or max_elems < 0 or adjoint not in (0, 1):
      return self._fail(-1, "qr_batched: bad sizes or flag")
    if nprob == 0 or max_elems == 0:
      return 0
    if dtype not in _WIDE:
      return self._fail(-2, "qr_batched: dtype")
    if max_elems * np.dtype(_WIDE[dtype]).itemsize > _lib.QR_BATCHED_MAX_BYTES:
      return self._fail(-4, "qr_batched: over the limit")
    d = self._vec(dims, 2 * nprob, np.int64).reshape(nprob, 2)
    ao, qo, ro = (self._vec(p, nprob, np.int64) for p in (aoff, qoff, roff))
    dt = fake_lib._NP[dtype]
    for p in range(nprob):
      m, n = int(d[p, 0]), int(d[p, 1])
      assert m * n <= max_elems
      k = min(m, n)
      A = self._vec(int(a) + int(ao[p]) * np.dtype(dt).itemsize, m * n, dt).reshape(m, n).astype(_WIDE[dtype])
      if adjoint:
        qq, rr = _HOST_QR(A.conj().T)
        lf, rf = rr.conj().T, qq.conj().T          # R = R'^H (m x k), Q = Q'^H (k x n)
      else:
        qq, rr = _HOST_QR(A)
        lf, rf = qq, rr
      qout, rout = (rf, lf) if adjoint else (lf, rf)
      self._vec(int(q) + int(qo[p]) * np.dtype(dt).itemsize, qout.size, dt)[...] = qout.ravel()
      self._vec(int(r) + int(ro[p]) * np.dtype(dt).itemsize, rout.size, dt)[...] = rout.ravel()
      assert qout.shape == ((k, n) if adjoint else (m, k)) and rout.shape == ((m, k) if adjoint else (k, n))
    self.qr_batched_calls.append(nprob)
    self._launches += 1
    return 0

  def tnb200_blocksparse_tensordot(self, a, b, c, dtype, nsect, dims, am, ao, bm, bo, cm, co, max_m, max_n, conj_b, stream):
    """sector q reads its maps at [off[q], off[q] + size): the offsets address whole-tensor maps (and end with a 0), so
    the map lengths come from the sector sizes"""
    nsect = int(nsect)
    d = self._vec(dims, 3 * nsect, np.int64).reshape(nsect, 3)
    aoff, boff, coff = (self._vec(p, nsect, np.int64) for p in (ao, bo, co))
    sizes = [(d[:, 0] * d[:, 1]), (d[:, 1] * d[:, 2]), (d[:, 0] * d[:, 2])]
    maps = [self._vec(mp, int((off + sz).max()), np.int64) for mp, off, sz in zip((am, bm, cm), (aoff, boff, coff), sizes)]
    vecs = [self._vec(p, int(mp.max()) + 1, fake_lib._NP[dtype]) for p, mp in zip((a, b, c), maps)]
    for q in range(nsect):
      m_, k_, n_ = (int(x) for x in d[q])
      x = vecs[0][maps[0][aoff[q]:aoff[q] + m_ * k_]].reshape(m_, k_)
      y = vecs[1][maps[1][boff[q]:boff[q] + k_ * n_]].reshape(k_, n_)
      vecs[2][maps[2][coff[q]:coff[q] + m_ * n_]] = (x @ (np.conj(y) if conj_b else y)).ravel()
    self._launches += 1
    return 0


FAKE = QrFakeLib()
_lib.set_lib(FAKE)
tb_backend._CONFIG["device"] = "cpu"
import tensornetwork_b200 as tb
assert tb.registered_symmetric
import importlib.util
spec = importlib.util.spec_from_file_location("tsymqr", os.path.join(ROOT, "tests", "test_gpu_symmetric_qr.py"))
m = importlib.util.module_from_spec(spec); spec.loader.exec_module(m)

for ndim in (3, 4):
  for charge in ("U1", "Z3"):
    for dtype in (np.float64, np.complex128, np.float32, np.complex64):
      m.test_qr_rq_match_reference(tn, charge, ndim, dtype)
print("parity ok")
m.test_tall_and_wide_sectors_in_one_tensor(tn); print("tall/wide ok")
m.test_fused_and_transposed_inputs(tn); print("fused ok")
for dtype in (np.float64, np.complex128):
  FAKE.qr_batched_calls.clear()
  m.test_sectors_over_the_batched_limit_fall_back(tn, dtype)
  assert FAKE.qr_batched_calls, "the batched launch did not run"
print("fallback ok")
for dtype in (np.float64, np.complex128):
  m.test_dimension_one_legs_against_numpy(tn, dtype)
print("dimension-1 legs ok")
m.test_rank_deficient_sector(tn); print("rank-deficient ok")
m.test_finite_mps_canonicalises_on_device(tn); print("FiniteMPS ok")
m.test_split_node_qr_and_rq(tn); print("split_node ok")
print("SYMQR HOST OK")
