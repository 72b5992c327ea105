"""Arnoldi eigensolver timing probe (needs a GPU): the dominant left eigenpair of an InfiniteMPS transfer matrix through
the reference's own `transfer_matrix_eigs` (d = 2, two-site unit cell, precision 1e-10, 30 Krylov vectors) on
backend="cuda_b200", against the same call on backend="numpy" (scipy's ARPACK on the host cores).
python tools/eigs_bench.py [--sizes 64,256,512,1024] [--c128 512] [--numpy-max 256]

One JSON line naming the card, its power limit and max SM clock, then one line per case: wall time (host clock around
a synchronised call, best of 3 after one warm-up), matvecs, restarts, launches, host reads, the time spent in
tnb200_arnoldi_orth (CUDA events) with the bytes it must move over that time against 3.35 TB/s, the numpy time, and
|eta - eta_numpy| / |eta_numpy|, ||T(l) - eta l|| / ||l|| and that over |eta|."""
import json
import os
import subprocess
import sys
import time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from baseline import refenv  # noqa: E402
tn = refenv.load()
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import arnoldi  # noqa: E402
from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS  # noqa: E402

HBM = 3.35e12


def card():
  out = {"name": torch.cuda.get_device_name(), "host_cores": len(os.sched_getaffinity(0))}
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.stdout.strip().split(",")]
  except Exception as e:  # pylint: disable=broad-except
    out["power_limit"] = "unknown (%s)" % e
  return out


class OrthTimer:
  """wraps the library's tnb200_arnoldi_orth with CUDA events; bytes from shapes: 3 reads of rows 0..j, w read twice,
  row j+1 written twice, read once and read + written by the scaling pass"""

  def __init__(self, lib):
    self.lib, self.fn = lib, lib.tnb200_arnoldi_orth
    self.events, self.bytes = [], 0

  def __call__(self, v, j, w, h, st):
    d = v._obj
    esz = {0: 8, 1: 4, 4: 8, 5: 16}[d.dtype]
    n = d.shape[1]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    rc = self.fn(v, j, w, h, st)
    e1.record()
    self.events.append((e0, e1))
    self.bytes += esz * n * (3 * (j + 1) + 2 + 5)
    return rc

  def ms(self):
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in self.events)


def case(D, dtype, numpy_max):
  np.random.seed(D)
  ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=dtype, backend="numpy")
  mps = InfiniteMPS(tensors=[np.asarray(t) for t in ref.tensors], center_position=0, backend="cuda_b200")
  be = mps.backend
  info = {}

  def eigs_info(*a, **k):                      # the backend method, keeping the driver's statistics
    be._no_capture("eigs")
    eta, vecs, i = arnoldi.eigs(be, *a, return_info=True, **k)
    info.update(i)
    return eta, vecs
  be.eigs = eigs_info
  times = []
  try:
    for it in range(4):
      torch.cuda.synchronize()
      n0 = be.lib.tnb200_launch_count()
      t0 = time.perf_counter()
      eta, l = mps.transfer_matrix_eigs("l", precision=1e-10, num_krylov_vecs=30)
      torch.cuda.synchronize()
      if it:
        times.append(time.perf_counter() - t0)
      launches = be.lib.tnb200_launch_count() - n0
    timer = OrthTimer(be.lib)
    lib = be.lib
    try:
      lib.tnb200_arnoldi_orth = timer
    except AttributeError:
      timer = None
    if timer is not None:
      mps.transfer_matrix_eigs("l", precision=1e-10, num_krylov_vecs=30)
      orth_ms = timer.ms()
      lib.tnb200_arnoldi_orth = timer.fn
  finally:
    del be.eigs
  e = complex(eta.item())
  lh = l.to_host()
  l2 = mps.unit_cell_transfer_operator("l", l).to_host()
  out = {"D": D, "dtype": np.dtype(dtype).name, "n": D * D, "wall_ms": min(times) * 1e3, "matvecs": info["matvecs"],
         "restarts": info["restarts"], "launches": launches, "host_reads": info["host_reads"],
         "residual": float(np.linalg.norm(l2 - e * lh) / np.linalg.norm(lh)),
         "residual_over_eta": float(np.linalg.norm(l2 - e * lh) / (abs(e) * np.linalg.norm(lh)))}
  if timer is not None:
    out.update({"orth_ms": orth_ms, "orth_GB": timer.bytes / 1e9,
                "orth_TBps": timer.bytes / (orth_ms * 1e-3) / 1e12, "orth_share_of_3.35TBps": timer.bytes / (orth_ms * 1e-3) / HBM})
  if D <= numpy_max:
    t0 = time.perf_counter()
    reta, _ = ref.transfer_matrix_eigs("l", precision=1e-10, num_krylov_vecs=30)
    out["numpy_ms"] = (time.perf_counter() - t0) * 1e3
    out["eta_rel_err"] = float(abs(e - complex(reta)) / abs(complex(reta)))
  else:
    out["numpy_ms"] = "not measured"
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  args = sys.argv[1:]

  def opt(name, default):
    return args[args.index(name) + 1] if name in args else default
  sizes = [int(s) for s in opt("--sizes", "64,256,512,1024").split(",")]
  c128 = [int(s) for s in opt("--c128", "512").split(",") if s]
  numpy_max = int(opt("--numpy-max", "256"))
  tb.get_backend()
  print(json.dumps(card()), flush=True)
  for D in sizes:
    case(D, np.float64, numpy_max)
  for D in c128:
    case(D, np.complex128, numpy_max)
