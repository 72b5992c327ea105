"""QR timing probe (needs a GPU): tnb200_qr on m x n fp64, CUDA events.  python tools/qr_bench.py 2048x1024 4096x4096"""
import json
import os
import sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import tensornetwork_b200 as tb

if __name__ == "__main__":
  be = tb.get_backend()
  for arg in sys.argv[1:]:
    m, n = (int(x) for x in arg.split("x"))
    rng = np.random.default_rng(1)
    a_h = rng.standard_normal((m, n))
    a = be.convert_to_tensor(a_h)
    ts = []
    for it in range(3):
      n0 = be.lib.tnb200_launch_count()
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      q, r = be.qr(a, 1)
      e1.record()
      torch.cuda.synchronize()
      ts.append(e0.elapsed_time(e1))
      launches = be.lib.tnb200_launch_count() - n0
    qh, rh = q.to_host(), r.to_host()
    rq, rr = np.linalg.qr(a_h)
    print(json.dumps({"m": m, "n": n, "ms": min(ts), "launches": int(launches), "kernel": be.lib.tnb200_last_kernel().decode(),
                      "q_err_vs_numpy": float(np.abs(qh - rq).max()), "r_err_vs_numpy": float(np.abs(rh - rr).max() / np.abs(rr).max()),
                      "recon": float(np.abs(qh @ rh - a_h).max()), "orth": float(np.abs(qh.T @ qh - np.eye(min(m, n))).max())}), flush=True)
