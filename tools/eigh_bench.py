"""Hermitian eigensolver timing probe (needs a GPU): tnb200_eigh on random n x n Hermitian matrices, CUDA events,
sweeps from the info words, against np.linalg.eigh on the host cores of the same machine.
python tools/eigh_bench.py 256 1024 2048 4096 [--c128 1024] [--reps 2]

One JSON line per size, after one line naming the card, its power limit and the host cores numpy ran on."""
import json
import os
import subprocess
import sys
import time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import tensornetwork_b200 as tb
from tensornetwork_b200 import _lib as L


def card():
  out = {"name": torch.cuda.get_device_name(), "host_cores": len(os.sched_getaffinity(0))}
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.stdout.strip().split(",")]
  except Exception as e:  # pylint: disable=broad-except
    out["power_limit"] = "unknown (%s)" % e
  return out


def run(be, n, dtype, reps):
  rng = np.random.default_rng(n)
  x = rng.standard_normal((n, n))
  if np.dtype(dtype).kind == "c":
    x = x + 1j * rng.standard_normal((n, n))
  a_h = ((x + x.conj().T) / 2).astype(dtype)
  a = be.convert_to_tensor(a_h)
  w = be._new((n,), tb.tensor.real_code(a.code))
  v = be._new((n, n), a.code)
  info = torch.zeros(4, dtype=torch.int32, device=be.device)
  times = []
  for it in range(reps + 1):        # call 0 warms the module and the workspace pool
    n0 = be.lib.tnb200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    L.check(be.lib.tnb200_eigh(a.ref(), w.ref(), v.ref(), info.data_ptr(), be._stream()))
    e1.record()
    torch.cuda.synchronize()
    if it:
      times.append(e0.elapsed_time(e1))
    launches = be.lib.tnb200_launch_count() - n0
  t0 = time.perf_counter()
  ref_w = np.linalg.eigh(a_h)[0]
  numpy_ms = (time.perf_counter() - t0) * 1e3
  wh, vh = w.to_host(), v.to_host()
  out = {"n": n, "dtype": np.dtype(dtype).name, "ms": min(times), "numpy_ms": numpy_ms, "sweeps": int(info[0]),
         "converged": int(info[1]), "launches": launches,
         "w_err": float(np.abs(wh - ref_w).max() / np.abs(ref_w).max()),
         "residual": float(np.linalg.norm(a_h @ vh - vh * wh[None, :]) / np.linalg.norm(a_h)),
         "orth": float(np.abs(vh.conj().T @ vh - np.eye(n)).max())}
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  args = sys.argv[1:]
  reps = int(args[args.index("--reps") + 1]) if "--reps" in args else 2
  c128 = [int(args[args.index("--c128") + 1])] if "--c128" in args else [1024]
  sizes = [int(s) for i, s in enumerate(args) if s.isdigit() and (i == 0 or args[i - 1] not in ("--reps", "--c128"))]
  be = tb.get_backend()
  print(json.dumps(card()), flush=True)
  for n in sizes:
    run(be, n, np.float64, reps)
  for n in c128:
    run(be, n, np.complex128, reps)
