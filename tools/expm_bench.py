"""Matrix exponential timing probe (needs a GPU): CudaB200Backend.expm (tnb200_expm) against scipy.linalg.expm on the
host cores.  python tools/expm_bench.py [--sizes 4,16,32,64,128,256,1024,4096] [--no-trotter]

One JSON line naming the card, its power limit and max SM clock, then one line per case: n, dtype, the matrix ("rand":
random with ||A||_1 = 1; "herm": -i tau H with H Hermitian, ||tau H||_1 = 2), best-of-3 wall time (host clock around a
synchronised call, after one warm-up), launches, m, s, path (0 fused, 1 blocked), host reads of the selection,
||X - X_scipy||_F / ||X_scipy||_F, and the scipy.linalg.expm time (best of 3).  Then the Trotter case: the 63 two-site
gates exp(-i tau h) of a 64-site chain (d = 2 and 4) built through tn.linalg.expm, eagerly, under backend.jit, and on
backend="numpy"."""
import json
import os
import subprocess
import sys
import time
import numpy as np
import scipy.linalg
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from baseline import refenv  # noqa: E402
tn = refenv.try_load()
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import _lib as L  # noqa: E402


def card():
  out = {"name": torch.cuda.get_device_name(), "host_cores": len(os.sched_getaffinity(0)),
         "expm_fused_max_n": L.EXPM_FUSED_MAX_N}
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


def matrix(n, dtype, kind):
  rng = np.random.default_rng(n)
  if kind == "rand":
    a = rng.standard_normal((n, n))
    if np.dtype(dtype).kind == "c":
      a = a + 1j * rng.standard_normal((n, n))
    return (a / np.abs(a).sum(axis=0).max()).astype(dtype)
  h = rng.standard_normal((n, n)) + 1j * rng.standard_normal((n, n))
  h = h + h.conj().T
  h = 2.0 * h / np.abs(h).sum(axis=0).max()
  return (-1j * h).astype(dtype) if np.dtype(dtype).kind == "c" else None


def case(be, n, dtype, kind):
  a = matrix(n, dtype, kind)
  if a is None:
    return None
  ad = be.convert_to_tensor(a)
  x = be._new((n, n), ad.code)
  info = torch.empty(4, dtype=torch.int32, device=be.device)
  run = lambda: L.check(be.lib.tnb200_expm(ad.ref(), x.ref(), info.data_ptr(), be._stream()))  # noqa: E731
  t = best(run)
  c0 = be.lib.tnb200_launch_count()
  run()
  launches = be.lib.tnb200_launch_count() - c0
  m, s, path, _ = (int(v) for v in info.cpu().numpy())
  ts = []
  for _ in range(3):
    t0 = time.perf_counter()
    ref = scipy.linalg.expm(a)
    ts.append(time.perf_counter() - t0)
  xh = x.to_host()
  return {"n": n, "dtype": np.dtype(dtype).name, "matrix": kind, "expm_ms": 1e3 * t, "launches": launches, "m": m,
          "s": s, "path": path, "host_reads": 0 if path == 0 else {3: 1, 5: 1, 7: 2, 9: 2}.get(m, 3),
          "rel_err_vs_scipy": float(np.linalg.norm(xh - ref) / np.linalg.norm(ref)), "scipy_ms": 1e3 * min(ts)}


def trotter(be, d):
  """63 two-site gates exp(-i tau h_j) for a 64-site chain through tn.linalg.expm"""
  rng = np.random.default_rng(d)
  hs = []
  for _ in range(63):
    h = rng.standard_normal((d * d, d * d)) + 1j * rng.standard_normal((d * d, d * d))
    hs.append((h + h.conj().T) / 2)
  tau = 0.05

  def gates(ts):
    return [tn.linalg.linalg.expm(t) for t in ts]
  dev = [tn.Tensor(be.convert_to_tensor(-1j * tau * h), backend="cuda_b200") for h in hs]
  host = [tn.Tensor(-1j * tau * h, backend="numpy") for h in hs]
  t_eager = best(lambda: gates(dev))
  c0 = be.lib.tnb200_launch_count()
  out = gates(dev)
  launches = be.lib.tnb200_launch_count() - c0
  jf = be.jit(lambda *arrs: [be.expm(x) for x in arrs], static_argnums=())
  arrs = [t.array for t in dev]
  jf(*arrs)
  t_jit = best(lambda: jf(*arrs))
  ref = gates(host)
  t0 = time.perf_counter()
  for _ in range(3):
    gates(host)
  t_np = (time.perf_counter() - t0) / 3
  err = max(float(np.linalg.norm(o.array.to_host() - r.array) / np.linalg.norm(r.array)) for o, r in zip(out, ref))
  jerr = max(float(np.linalg.norm(o.to_host() - r.array) / np.linalg.norm(r.array)) for o, r in zip(jf(*arrs), ref))
  return {"trotter_d": d, "gates": 63, "n": d * d, "eager_ms": 1e3 * t_eager, "launches_eager": launches,
          "jit_ms": 1e3 * t_jit, "jit_stats": dict(be.jit_stats), "numpy_ms": 1e3 * t_np, "max_rel_err": err,
          "max_rel_err_jit": jerr}


def main():
  sizes = [4, 16, 32, 64, 128, 256, 1024, 4096]
  args = sys.argv[1:]
  if "--sizes" in args:
    sizes = [int(s) for s in args[args.index("--sizes") + 1].split(",")]
  be = tb.get_backend()
  print(json.dumps({"card": card()}), flush=True)
  for n in sizes:
    for dtype in (np.float64, np.complex128):
      for kind in ("rand", "herm"):
        r = case(be, n, dtype, kind)
        if r is not None:
          print(json.dumps(r), flush=True)
  if "--no-trotter" not in args and tn is not None:
    for d in (2, 4):
      print(json.dumps(trotter(be, d)), flush=True)


if __name__ == "__main__":
  main()
