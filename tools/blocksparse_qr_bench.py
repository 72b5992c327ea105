"""Block-sparse qr / rq timing probe (needs a GPU): backend="symmetric_b200" (tnb200_qr_batched + tnb200_qr fallback)
against the reference's backend="symmetric" on the host cores.  python tools/blocksparse_qr_bench.py [--sizes 256,512,1024,2048]

One JSON line naming the card, its power limit and the host core count, then:
  - one line per (D, dtype) for a U(1) MPS site tensor (D, 2, D) whose bond charges spread over 20 values (about 20
    sectors): qr (pivot 2) and rq (pivot 1) best-of-3 wall time (host clock around a synchronised call, host conversion
    included, after one warm-up), launches per call, sectors in the batch and sectors falling back to tnb200_qr, the
    reference's time (best of 3) and max |Q - Q_ref|;
  - the crossover of one problem: tnb200_qr_batched against tnb200_qr on a square n x n matrix (CUDA events, mean of 20);
  - FiniteMPS canonicalisation of an N = 32 U(1) block-sparse MPS (D = 128) on symmetric_b200, split into qr / rq,
    tensordot and the host conversion inside them, and the dense backend="numpy" canonicalisation of the same state
    (the reference's block-sparse path cannot canonicalise it: its host qr fails on the dimension-1 boundary legs)."""
import argparse
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
from tensornetwork_b200 import _lib as L, blocksparse as bsp, symmetric as sym, tensor as T  # noqa: E402
from tensornetwork.backends import backend_factory  # noqa: E402


def card():
  out = {"name": torch.cuda.get_device_name(), "host_cores": len(os.sched_getaffinity(0)),
         "qr_batched_max_bytes": L.QR_BATCHED_MAX_BYTES}
  try:
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    out["power_limit"], out["max_sm_clock"] = [s.strip() for s in q.stdout.strip().split(",")]
  except Exception as e:  # pylint: disable=broad-except
    out["power_limit"] = "unknown (%s)" % e
  return out


def best(f, reps=3, sync=True):
  f()
  ts = []
  for _ in range(reps):
    if sync:
      torch.cuda.synchronize()
    t0 = time.perf_counter()
    f()
    if sync:
      torch.cuda.synchronize()
    ts.append(time.perf_counter() - t0)
  return min(ts)


def site_tensor(D, dtype, seed):
  rng = np.random.default_rng(seed)
  I = tn.Index
  cl = tn.U1Charge(np.sort(rng.integers(0, 20, D)).astype(np.int16))
  cr = tn.U1Charge(np.sort(rng.integers(0, 21, D)).astype(np.int16))
  t = tn.BlockSparseTensor.random([I(cl, False), I(tn.U1Charge(np.array([0, 1], dtype=np.int16)), False), I(cr, True)],
                                  dtype=np.float64)
  data = rng.uniform(-1, 1, t.data.shape)
  if np.dtype(dtype).kind == "c":
    data = data + 1j * rng.uniform(-1, 1, t.data.shape)
  t.data = data.astype(dtype)
  return t


def split_counts(be, t, pivot):
  dt, groups = sym._to_device(t, be.device_backend)  # pylint: disable=protected-access
  nl = sum(len(g) for g in groups[:pivot])
  d = bsp._sector_maps(dt.indices, dt.order, nl)[1]  # pylint: disable=protected-access
  e = d[:, 0] * d[:, 1]
  small = (e > 0) & (e * (16 if T.is_complex_code(dt.data.code) else 8) <= L.QR_BATCHED_MAX_BYTES)
  return int(small.sum()), int(((e > 0) & ~small).sum())


def site_rows(sizes):
  be, ref = backend_factory.get_backend("symmetric_b200"), backend_factory.get_backend("symmetric")
  lib = be.lib
  for D in sizes:
    for dtype in (np.float64, np.complex128):
      t = site_tensor(D, dtype, D)
      for op, pivot in (("qr", 2), ("rq", 1)):
        f = getattr(be, op)
        g = getattr(ref, op)
        t_dev = best(lambda: f(t, pivot))
        n0 = lib.tnb200_launch_count()
        got = f(t, pivot)
        torch.cuda.synchronize()
        launches = lib.tnb200_launch_count() - n0
        t_ref = best(lambda: g(t, pivot), sync=False)
        want = g(t, pivot)
        qi = 0 if op == "qr" else 1
        err = float(np.abs(np.asarray(got[qi].todense()) - np.asarray(want[qi].todense())).max())
        nb, nf = split_counts(be, t, pivot)
        print(json.dumps({"case": "site", "D": D, "dtype": np.dtype(dtype).name, "op": op, "nnz": int(t.data.size),
                          "device_ms": round(t_dev * 1e3, 3), "launches": int(launches), "batched_sectors": nb,
                          "fallback_sectors": nf, "reference_ms": round(t_ref * 1e3, 3), "max_abs_q_diff": err}), flush=True)


def crossover():
  """one n x n problem: tnb200_qr_batched against tnb200_qr (CUDA events around 20 calls, after a warm-up)"""
  be = tb.get_backend()
  lib, st = be.lib, be._stream()  # pylint: disable=protected-access
  for dtype, sizes in ((np.float64, (8, 16, 32, 64, 96, 128, 160)), (np.complex128, (8, 16, 32, 64, 96, 112))):
    code = T.dtype_code(dtype)
    for n in sizes:
      a = be.randn((n, n), dtype, seed=n)
      q, r = be._new((n, n), code), be._new((n, n), code)  # pylint: disable=protected-access
      up = lambda x: torch.tensor(x, dtype=torch.int64, device=be.device)
      dims, z = up([n, n]), up([0])
      runs = {"batched": lambda: L.check(lib.tnb200_qr_batched(a.t.data_ptr(), code, 1, dims.data_ptr(), z.data_ptr(), q.t.data_ptr(),
                                                               z.data_ptr(), r.t.data_ptr(), z.data_ptr(), n * n, 0, st)),
              "tnb200_qr": lambda: L.check(lib.tnb200_qr(a.ref(), q.ref(), r.ref(), 0, st))}
      row = {"case": "crossover", "n": n, "dtype": np.dtype(dtype).name}
      for name, f in runs.items():
        f()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
          f()
        e1.record()
        torch.cuda.synchronize()
        row[name + "_us"] = round(e0.elapsed_time(e1) * 1e3 / 20, 2)
      print(json.dumps(row), flush=True)


def mps_tensors(N, D, seed):
  rng = np.random.default_rng(seed)
  I = tn.Index
  cp = tn.U1Charge(np.array([0, 1], dtype=np.int16))

  def bond(n):
    lo, hi = max(0, N // 2 - (N - n)), min(n, N // 2)
    return tn.U1Charge(np.sort(rng.integers(lo, hi + 1, D)).astype(np.int16))
  bonds = [tn.U1Charge(np.array([0], dtype=np.int16))] + [bond(n) for n in range(1, N)] + \
      [tn.U1Charge(np.array([N // 2], dtype=np.int16))]
  np.random.seed(seed)
  return [tn.BlockSparseTensor.random([I(bonds[n], False), I(cp, False), I(bonds[n + 1], True)], dtype=np.float64)
          for n in range(N)]


def canonicalise(N=32, D=128):
  be = backend_factory.get_backend("symmetric_b200")
  ts = mps_tensors(N, D, 7)
  dense = [np.asarray(t.todense()) for t in ts]
  spent = {"qr_rq": 0.0, "tensordot": 0.0, "conversion": 0.0}

  def timed(key, f):
    def g(*a, **k):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      out = f(*a, **k)
      torch.cuda.synchronize()
      spent[key] += time.perf_counter() - t0
      return out
    return g
  to_dev, to_host = sym._to_device, T.B200Tensor.to_host  # pylint: disable=protected-access
  tn.FiniteMPS([t.copy() for t in ts], canonicalize=True, backend="symmetric_b200")      # warm-up (caches, modules)
  be.qr, be.rq = timed("qr_rq", be.qr), timed("qr_rq", be.rq)
  be.tensordot = timed("tensordot", be.tensordot)
  sym._to_device = timed("conversion", to_dev)  # pylint: disable=protected-access
  T.B200Tensor.to_host = timed("conversion", to_host)
  try:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tn.FiniteMPS([t.copy() for t in ts], canonicalize=True, backend="symmetric_b200")
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
  finally:
    sym._to_device, T.B200Tensor.to_host = to_dev, to_host  # pylint: disable=protected-access
    del be.qr, be.rq, be.tensordot
  t_np = best(lambda: tn.FiniteMPS([d.copy() for d in dense], canonicalize=True, backend="numpy"), sync=False)
  print(json.dumps({"case": "FiniteMPS canonicalize", "N": N, "D": D, "nnz_total": int(sum(t.data.size for t in ts)),
                    "symmetric_b200_ms": round(total * 1e3, 2), "qr_rq_ms": round(spent["qr_rq"] * 1e3, 2),
                    "tensordot_ms": round(spent["tensordot"] * 1e3, 2),
                    "host_conversion_ms (inside qr_rq and tensordot)": round(spent["conversion"] * 1e3, 2),
                    "dense_numpy_backend_ms": round(t_np * 1e3, 2)}), flush=True)


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--sizes", default="256,512,1024,2048")
  args = p.parse_args()
  print(json.dumps(card()), flush=True)
  site_rows([int(s) for s in args.sizes.split(",")])
  crossover()
  canonicalise()


if __name__ == "__main__":
  main()
