"""InfiniteMPS canonicalisation timing probe (needs a GPU): the reference's own InfiniteMPS.canonicalize (d = 2, two-site
unit cell, float64, precision 1e-10) on backend="cuda_b200" against the same call on backend="numpy".
python tools/canonicalize_bench.py [--sizes 64,256,1024] [--numpy-max 256]

One JSON line naming the card, its power limit and max SM clock, then one line per (D, backend): the wall time of one
call (host clock; the device is synchronised before and after every timed backend call) and its split into the two
`eigs` calls (transfer_matrix_eigs), the two `eigh` calls, `svd` and `inv`; "other" is the rest (QR sweeps, ncon,
elementwise work).  The numpy arm runs only up to --numpy-max (scipy's ARPACK on the host cores takes minutes beyond).
For D where both ran: |lam_norm - lam_norm_numpy| / lam_norm_numpy and the largest Schmidt-value difference."""
import json
import os
import sys
import time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from baseline import refenv  # noqa: E402
tn = refenv.load()
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402,F401  pylint: disable=unused-import
from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS  # noqa: E402
from inv_bench import card  # noqa: E402

TIMED = ("eigs", "eigh", "svd", "inv")


def sync():
  torch.cuda.synchronize()


def timed_canonicalize(mps):
  """one canonicalize call with the backend's eigs / eigh / svd / inv wrapped by synchronised host timers"""
  be = mps.backend
  spent = {k: 0.0 for k in TIMED}
  calls = {k: 0 for k in TIMED}
  for name in TIMED:
    fn = getattr(be, name)

    def wrapped(*a, _fn=fn, _name=name, **kw):
      sync()
      t0 = time.perf_counter()
      r = _fn(*a, **kw)
      sync()
      spent[_name] += time.perf_counter() - t0
      calls[_name] += 1
      return r
    setattr(be, name, wrapped)
  try:
    sync()
    t0 = time.perf_counter()
    lam = mps.canonicalize(precision=1e-10)
    sync()
    total = time.perf_counter() - t0
  finally:
    for name in TIMED:
      delattr(be, name)
  out = {"total_s": total}
  out.update({k + "_s": v for k, v in spent.items()})
  out["other_s"] = total - sum(spent.values())
  out["calls"] = calls
  return lam, out


def schmidt(c):
  return np.sort(np.abs(np.diag(np.linalg.inv(np.asarray(c)))))


def main():
  sizes, numpy_max = [64, 256, 1024], 256
  args = sys.argv[1:]
  if "--sizes" in args:
    sizes = [int(s) for s in args[args.index("--sizes") + 1].split(",")]
  if "--numpy-max" in args:
    numpy_max = int(args[args.index("--numpy-max") + 1])
  print(json.dumps({"card": card()}), flush=True)
  np.random.seed(0)
  warm = InfiniteMPS.random(d=[2, 2], D=[16] * 3, dtype=np.float64, backend="numpy")
  InfiniteMPS(tensors=[np.asarray(t) for t in warm.tensors], center_position=0, backend="cuda_b200").canonicalize()
  for D in sizes:
    np.random.seed(D)
    ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=np.float64, backend="numpy")
    host = [np.asarray(t).copy() for t in ref.tensors]
    mps = InfiniteMPS(tensors=host, center_position=0, backend="cuda_b200")
    lam, rec = timed_canonicalize(mps)
    rec = dict({"D": D, "backend": "cuda_b200"}, **rec)
    print(json.dumps(rec), flush=True)
    if D <= numpy_max:
      ref_lam, nrec = timed_canonicalize(ref)
      nrec = dict({"D": D, "backend": "numpy"}, **nrec)
      nrec["lam_norm_rel_diff"] = abs(float(lam.item()) - float(ref_lam)) / abs(float(ref_lam))
      nrec["schmidt_max_diff"] = float(np.max(np.abs(schmidt(mps.connector_matrix) - schmidt(ref.connector_matrix))))
      print(json.dumps(nrec), flush=True)


if __name__ == "__main__":
  main()
