"""Product charges on backend="symmetric_b200": map build, tensordot, svd and qr for U(1) x U(1) (particle number x 2 S_z)
MPS tensors, against the reference's backend="symmetric" on the host, and the scaling of the device map build in
states and bins.  One run on one GPU; prints the card, its power limit and one JSON line per measurement.

  python tools/blocksparse_product_bench.py"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baseline import refenv  # noqa: E402

tn = refenv.load()
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import blocksparse as bs  # noqa: E402
from tensornetwork.backends import backend_factory  # noqa: E402
from tensornetwork.block_sparse.charge import BaseCharge  # noqa: E402


def card():
  try:
    pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                        text=True, timeout=30).stdout.strip()
  except Exception:  # pylint: disable=broad-except
    pl = "not measured"
  return torch.cuda.get_device_name(0), pl


def wall(f, reps=3):
  f()
  best = None
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    f()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    best = dt if best is None else min(best, dt)
  return best * 1e3


def charge(q):
  return BaseCharge(np.asarray(q, dtype=np.int16), charge_types=[tn.U1Charge, tn.U1Charge])


def bond(rng, D, n):
  """D states of (particle number, 2 S_z) around half filling after n sites"""
  num = rng.integers(n - 4, n + 5, D)
  down = rng.binomial(num, 0.5)
  return charge(np.stack([num, num - 2 * down], axis=1))


def main():
  name, pl = card()
  print("card: %s, power limit: %s" % (name, pl))
  be, ref = backend_factory.get_backend("symmetric_b200"), backend_factory.get_backend("symmetric")
  lib = tb.get_backend().lib
  phys = charge(np.array([[0, 0], [1, 1], [1, -1], [2, 0]]))
  I = tn.Index
  for D in (256, 512, 1024):
    rng = np.random.default_rng(D)
    np.random.seed(D)
    cl, cr, cr2 = bond(rng, D, 20), bond(rng, D, 22), bond(rng, D, 24)
    site = tn.BlockSparseTensor.random([I(cl, False), I(phys, False), I(cr, True)], dtype=np.float64)
    two = tn.BlockSparseTensor.random([I(cl, False), I(phys, False), I(phys, False), I(cr2, True)], dtype=np.float64)
    for label, t in (("site (D, 4, D)", site), ("two-site (D, 4, 4, D)", two)):
      n = t.ndim
      tc = ref.conj(t)
      axes = (list(range(1, n)), list(range(1, n)))
      bs._MAP_CACHE.clear()
      l0 = lib.tnb200_launch_count()
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      be.tensordot(t, tc, axes)
      torch.cuda.synchronize()
      first = (time.perf_counter() - t0) * 1e3
      launches_first = lib.tnb200_launch_count() - l0
      dt, _ = tb.symmetric._to_device(t, tb.get_backend())
      shifts = bs._shifts(dt.indices, (None, None))
      rec = {"tensor": label, "D": D, "nnz": int(t.data.size), "bins": (2 * shifts[0] + 1) * (2 * shifts[1] + 1),
             "launches_first_tensordot": int(launches_first), "first_tensordot_ms": first,
             "tensordot_ms": wall(lambda: be.tensordot(t, tc, axes)), "svd_ms": wall(lambda: be.svd(t, 2)),
             "qr_ms": wall(lambda: be.qr(t, 2)),
             "host_tensordot_ms": wall(lambda: ref.tensordot(t, tc, axes), 1), "host_svd_ms": wall(lambda: ref.svd(t, 2), 1)}
      try:
        rec["host_qr_ms"] = wall(lambda: ref.qr(t, 2), 1)
      except Exception as e:  # pylint: disable=broad-except
        rec["host_qr_ms"] = "fails: %s" % type(e).__name__
      print(json.dumps(rec), flush=True)
  # the device map build alone: fixed bins with growing states, fixed states with growing bins
  dbe = tb.get_backend()
  def maps_ms(idx, order, part):
    def run():
      bs._MAP_CACHE.clear()
      bs._device_sector_maps(dbe, idx, order, part)
    return wall(run)
  for d in (100, 200, 400, 800):
    rng = np.random.default_rng(d)
    idx = [bs.Index(np.stack([rng.integers(-q, q + 1, d), rng.integers(-q, q + 1, d)], axis=1), f, (None, None))
           for q, f in ((30, False), (30, True), (2, False))]
    shifts = bs._shifts(idx, (None, None))
    print(json.dumps({"map_build": "fixed bins", "bins": (2 * shifts[0] + 1) * (2 * shifts[1] + 1), "row_states": d * d,
                      "ms_incl_host_tables": maps_ms(idx, [0, 1, 2], 2)}), flush=True)
  for q in (2, 8, 30, 120):
    rng = np.random.default_rng(q)
    idx = [bs.Index(np.stack([rng.integers(-q, q + 1, 400), rng.integers(-q, q + 1, 400)], axis=1), f, (None, None))
           for f in (False, True)] + [bs.Index(np.zeros((4, 2), dtype=np.int64), False, (None, None))]
    shifts = bs._shifts(idx, (None, None))
    print(json.dumps({"map_build": "fixed states", "bins": (2 * shifts[0] + 1) * (2 * shifts[1] + 1), "row_states": 160000,
                      "ms_incl_host_tables": maps_ms(idx, [0, 1, 2], 2)}), flush=True)
  # one symmetry either side of the 256-bin switch between the per-bin rank kernel and the counting sort
  for q in (30, 32, 33, 40):
    rng = np.random.default_rng(q)
    idx = [bs.Index(rng.integers(-q, q + 1, 64), f) for f in (False, False, True, True)]
    nb = 2 * int(bs._shifts(idx, (None,))[0]) + 1
    print(json.dumps({"map_build": "one U(1), 4 legs of 64", "bins": nb, "rank": "per-bin" if nb <= 256 else "counting sort",
                      "ms_incl_host_tables": maps_ms(idx, [0, 1, 2, 3], 2)}), flush=True)


if __name__ == "__main__":
  main()
