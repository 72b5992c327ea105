"""Matrix inverse timing probe (needs a GPU): CudaB200Backend.inv (tnb200_inv: blocked LU with partial pivoting, then
a blocked solve against the permuted identity) and tnb200_lu_factor alone, against np.linalg.inv on the host cores.
python tools/inv_bench.py [--sizes 256,1024,2048,4096] [--c128 1024]

One JSON line naming the card, its power limit and max SM clock, then one line per case: wall time of inv and of
lu_factor (host clock around a synchronised call, best of 3 after one warm-up), launches per inv, max|AX - I| in
float64 on the host, and the np.linalg.inv time (best of 3)."""
import json
import os
import subprocess
import sys
import time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import _lib as L  # noqa: E402


def card():
  out = {"name": torch.cuda.get_device_name(), "host_cores": len(os.sched_getaffinity(0))}
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.stdout.strip().split(",")]
  except Exception as e:  # pylint: disable=broad-except
    out["power_limit"] = "unknown (%s)" % e
  return out


def best(f, reps=3):
  f()
  ts = []
  for _ in range(reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    f()
    torch.cuda.synchronize()
    ts.append(time.perf_counter() - t0)
  return min(ts)


def case(be, n, dtype):
  rng = np.random.default_rng(n)
  a = rng.standard_normal((n, n))
  if np.dtype(dtype).kind == "c":
    a = a + 1j * rng.standard_normal((n, n))
  a = a.astype(dtype)
  ad = be.convert_to_tensor(a)
  lu = be._new((n, n), ad.code)
  piv = torch.empty(n, dtype=torch.int32, device=be.device)
  info = torch.empty(1, dtype=torch.int32, device=be.device)
  t_lu = best(lambda: L.check(be.lib.tnb200_lu_factor(ad.ref(), lu.ref(), piv.data_ptr(), info.data_ptr(), be._stream())))
  c0 = be.lib.tnb200_launch_count()
  x = be.inv(ad)
  launches = be.lib.tnb200_launch_count() - c0
  t_inv = best(lambda: be.inv(ad))
  xh = x.to_host()
  err = float(np.abs(a @ xh - np.eye(n)).max())
  ts = []
  for _ in range(3):
    t0 = time.perf_counter()
    np.linalg.inv(a)
    ts.append(time.perf_counter() - t0)
  return {"n": n, "dtype": np.dtype(dtype).name, "inv_ms": 1e3 * t_inv, "lu_factor_ms": 1e3 * t_lu,
          "solve_ms": 1e3 * (t_inv - t_lu), "launches": launches, "max_abs_AX_minus_I": err,
          "numpy_inv_ms": 1e3 * min(ts)}


def main():
  sizes, c128 = [256, 1024, 2048, 4096], [1024]
  args = sys.argv[1:]
  if "--sizes" in args:
    sizes = [int(s) for s in args[args.index("--sizes") + 1].split(",")]
  if "--c128" in args:
    c128 = [int(s) for s in args[args.index("--c128") + 1].split(",")]
  be = tb.get_backend()
  print(json.dumps({"card": card()}), flush=True)
  for n in sizes:
    print(json.dumps(case(be, n, np.float64)), flush=True)
  for n in c128:
    print(json.dumps(case(be, n, np.complex128)), flush=True)


if __name__ == "__main__":
  main()
