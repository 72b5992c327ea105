"""SVD timing probe (needs a GPU): tnb200_svd on n x n fp64 matrices, CUDA events, sweeps from the info words.
python tools/svd_bench.py 1024 2048 4096 [--f32]"""
import json
import os
import sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import tensornetwork_b200 as tb
from tensornetwork_b200 import _lib as L


def run(be, n, dtype=np.float64, reps=2, check=True):
  rng = np.random.default_rng(4)
  a_h = (rng.standard_normal((n, n)) / np.sqrt(n)).astype(dtype)
  a = be.convert_to_tensor(a_h)
  u = be._new((n, n), a.code)
  s = be._new((n,), tb.tensor.real_code(a.code))
  vh = be._new((n, n), a.code)
  info = torch.zeros(4, dtype=torch.int32, device=be.device)
  times = []
  for it in range(reps + 1):
    n0 = be.lib.tnb200_launch_count()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    L.check(be.lib.tnb200_svd(a.ref(), u.ref(), s.ref(), vh.ref(), info.data_ptr(), be._stream()))
    e1.record()
    torch.cuda.synchronize()
    if it:
      times.append(e0.elapsed_time(e1))
    launches = be.lib.tnb200_launch_count() - n0
  out = {"n": n, "dtype": np.dtype(dtype).name, "ms": min(times), "launches": launches, "sweeps": int(info[0]), "converged": int(info[1]),
         "kernel": be.lib.tnb200_last_kernel().decode(), "tflops_equiv_21n3": 21.0 * n**3 / (min(times) * 1e-3) / 1e12}
  if check:
    ref = np.linalg.svd(a_h.astype(np.float64), compute_uv=False)
    sh = s.to_host().astype(np.float64)
    out["s_err_rel_s0"] = float(np.abs(sh - ref).max() / ref[0])
    uh, vhh = u.to_host().astype(np.float64), vh.to_host().astype(np.float64)
    out["recon_err"] = float(np.linalg.norm((uh * sh[None, :]) @ vhh - a_h) / np.linalg.norm(a_h))
    out["orth_u"] = float(np.abs(uh.T @ uh - np.eye(n)).max())
    out["orth_v"] = float(np.abs(vhh @ vhh.T - np.eye(n)).max())
  print(json.dumps(out), flush=True)


if __name__ == "__main__":
  be = tb.get_backend()
  dt = np.float32 if "--f32" in sys.argv else np.float64
  for a in sys.argv[1:]:
    if a.isdigit():
      run(be, int(a), dt, check="--nocheck" not in sys.argv)
