"""Saturated interior two-site DMRG update (FiniteDMRG._optimize_2s_local, set up as bench.py's cfg5) on a U(1) XXZ chain
(2 S_z, total 0), f64, block-sparse MPS of bond dimension D.  Arms:
  (a) backend="symmetric_b200": resident tensors and the device eigsh_lanczos;
  (b) backend="symmetric_b200" with the reference's host eigsh_lanczos patched back in (every tensordot uploads its
      operands and downloads its result, and the Lanczos vectors live in numpy);
  (c) the reference's backend="symmetric" on the host cores.
Reports ms per update, libtnb200 launches per update, host<->device bytes per update (a separate torch.profiler run),
the first update's energy against the other arms, and the device bytes held by blocksparse._MAP_CACHE after each of 4
full two-site sweeps of arm (a).  Prints the card, its power limit and one JSON line per D, then a markdown table.

  python tools/blocksparse_dmrg_bench.py [--d 128 256 512 1024] [--cpu-max-d 512] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from baseline import refenv  # noqa: E402

tn = refenv.load()
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import blocksparse as bs  # noqa: E402
from tensornetwork.backends import backend_factory  # noqa: E402
from tensornetwork.backends.symmetric.symmetric_backend import SymmetricBackend  # noqa: E402

UPDATE = dict(num_krylov_vecs=10, tol=1e-5, delta=1e-6, ndiag=10)       # bench.py cfg5


def card():
  try:
    pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                        text=True, timeout=30).stdout.strip()
  except Exception:  # pylint: disable=broad-except
    pl = "not measured"
  return torch.cuda.get_device_name(0), pl


def host_eigsh(self, *args, **kwargs):
  """the reference's eigsh_lanczos, as symmetric_b200 inherited it before it had its own.  Its block cache is off: with
  it on, the reference's block-map hashing calls ndarray.tostring, which numpy 2 removed."""
  kwargs["enable_caching"] = False
  return SymmetricBackend.eigsh_lanczos(self, *args, **kwargs)


def bond_charges(N, n, D):
  """2 S_z of the D bond states after n of N sites: each charge q with multiplicity min(left states, right states that
  complete it to 0), scaled down to D states in all"""
  qs = np.arange(-n, n + 1, 2)
  mult = np.array([min(_binom(n, (n + q) // 2), _binom(N - n, (N - n - q) // 2)) for q in qs], dtype=np.float64)
  keep = qs[mult > 0], mult[mult > 0]
  qs, mult = keep
  if mult.sum() > D:
    m = np.floor(mult * D / mult.sum()).astype(np.int64)
    for i in np.argsort(-mult)[:D - int(m.sum())]:
      m[i] += 1
    mult = m
  return np.repeat(qs, mult.astype(np.int64))


def _binom(n, k):
  from math import comb  # pylint: disable=import-outside-toplevel
  return comb(n, k) if 0 <= k <= n else 0


def chain(D, nup=3):
  """(host MPS tensors centred at lo, host MPO tensors, lo) as cfg5 lays them out"""
  lo = int(np.ceil(np.log2(D)))
  N = 2 * lo + 2 + nup + 1
  N += N % 2
  I = tn.Index
  cp = tn.U1Charge(np.array([-1, 1]))
  bonds = [tn.U1Charge(bond_charges(N, n, D)) for n in range(N + 1)]
  np.random.seed(6)
  ts = [tn.BlockSparseTensor.random([I(bonds[n], False), I(cp, False), I(bonds[n + 1], True)], boundaries=(-1.0, 1.0))
        for n in range(N)]
  mps = tn.FiniteMPS(ts, canonicalize=True, backend="symmetric_b200")   # device QR / RQ; host tensors in, host tensors out
  mps.position(lo)
  dense = tn.FiniteXXZ(np.ones(N - 1), np.ones(N - 1), np.zeros(N), dtype=np.float64, backend="numpy").tensors
  qs = [np.zeros(1, dtype=np.int64)]
  for w in dense:                                  # MPO bond charges from each tensor's nonzero pattern (flows T, F, F, T)
    qr = np.zeros(w.shape[1], dtype=np.int64)
    for a, b, o, i in zip(*np.nonzero(w)):
      qr[b] = qs[-1][a] - (2 * o - 1) + (2 * i - 1)
    qs.append(qr)
  mpo = [tn.BlockSparseTensor.fromdense([I(tn.U1Charge(qs[n]), True), I(tn.U1Charge(qs[n + 1]), False), I(cp, False),
                                         I(cp, True)], np.asarray(w)) for n, w in enumerate(dense)]
  return [t.copy() for t in mps.tensors], mpo, lo


def dmrg(tensors, mpo, lo, backend):
  """a FiniteDMRG on `backend` centred at lo, its environments computed on the host tensors.  They are computed through
  symmetric_b200, host in and host out: the reference's own block maps fail on the dimension-1 boundary legs under
  numpy 2, and the interior update never touches those legs."""
  def make(name):
    mps = tn.FiniteMPS([t.copy() for t in tensors], canonicalize=False, backend=name)
    mps.center_position = lo
    return tn.FiniteDMRG(mps, tn.FiniteMPO(mpo, backend=name))
  envs = make("symmetric_b200")
  envs.compute_left_envs()
  envs.compute_right_envs()
  dm = make(backend)
  dm.left_envs, dm.right_envs = dict(envs.left_envs), dict(envs.right_envs)
  return dm


def updates(dm, D, count, sync):
  times, energies = [], []
  for _ in range(count):
    sync()
    t0 = time.perf_counter()
    e = dm._optimize_2s_local(max_bond_dim=D, sweep_dir="right", **UPDATE)  # pylint: disable=protected-access
    sync()
    times.append(time.perf_counter() - t0)
    energies.append(float(np.real(e)))
  return times, energies


def copy_bytes(dm, D):
  """host->device and device->host bytes of one update, from a torch.profiler trace"""
  from torch.profiler import profile, ProfilerActivity  # pylint: disable=import-outside-toplevel
  with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    updates(dm, D, 1, torch.cuda.synchronize)
  with tempfile.TemporaryDirectory() as d:
    path = os.path.join(d, "trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
      events = json.load(f)["traceEvents"]
  out = {"HtoD": 0, "DtoH": 0}
  for ev in events:
    if ev.get("cat") == "gpu_memcpy":
      for k in out:
        if k in ev.get("name", ""):
          out[k] += int(ev.get("args", {}).get("bytes", 0))
  return out


def cache_device_bytes():
  seen, total = set(), 0
  stack = list(bs._MAP_CACHE.values())  # pylint: disable=protected-access
  while stack:
    x = stack.pop()
    if isinstance(x, dict):
      stack.extend(x.values())
    elif isinstance(x, (tuple, list)):
      stack.extend(x)
    elif hasattr(x, "t") and isinstance(getattr(x, "t"), torch.Tensor):
      stack.append(x.t)
    elif isinstance(x, torch.Tensor) and x.is_cuda and x.data_ptr() not in seen:
      seen.add(x.data_ptr())
      total += x.numel() * x.element_size()
  return total


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--d", type=int, nargs="+", default=[128, 256, 512, 1024])
  ap.add_argument("--cpu-max-d", type=int, default=512, help="largest D for arm (c); larger ones are 'not measured'")
  ap.add_argument("--sweeps", type=int, default=4)
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("needs a CUDA device")
  name, pl = card()
  print("card: %s, power limit: %s, host cores: %d" % (name, pl, os.cpu_count()))
  cls = type(backend_factory.get_backend("symmetric_b200"))
  ref = backend_factory.get_backend("symmetric")
  ref.eigsh_lanczos = types.MethodType(host_eigsh, ref)       # arm (c): the reference's Lanczos, its block cache off
  device_eigsh = cls.eigsh_lanczos
  lib = tb.get_backend().lib
  rows = []
  for D in args.d:
    bs._MAP_CACHE.clear()  # pylint: disable=protected-access
    tensors, mpo, lo = chain(D)
    r = {"D": D}
    # (a)
    dm = dmrg(tensors, mpo, lo, "symmetric_b200")
    updates(dm, D, 1, torch.cuda.synchronize)
    n0 = lib.tnb200_launch_count()
    ta, ea = updates(dm, D, 3, torch.cuda.synchronize)
    r["a_ms"] = 1e3 * float(np.median(ta))
    r["a_launches"] = (lib.tnb200_launch_count() - n0) / len(ta)
    r["a_bytes"] = copy_bytes(dm, D)
    e_a = updates(dmrg(tensors, mpo, lo, "symmetric_b200"), D, 1, torch.cuda.synchronize)[1][0]
    # (b)
    cls.eigsh_lanczos = host_eigsh
    try:
      dm = dmrg(tensors, mpo, lo, "symmetric_b200")
      _, eb = updates(dm, D, 2, torch.cuda.synchronize)
      n0 = lib.tnb200_launch_count()
      tb2, _ = updates(dm, D, 1, torch.cuda.synchronize)
      r["b_ms"] = 1e3 * tb2[0]
      r["b_launches"] = lib.tnb200_launch_count() - n0
      r["b_bytes"] = copy_bytes(dm, D)
    finally:
      cls.eigsh_lanczos = device_eigsh
    r["energy_rel_a_b"] = abs(e_a - eb[0]) / abs(eb[0])
    # (c)
    if D <= args.cpu_max_d:
      tc, ec = updates(dmrg(tensors, mpo, lo, "symmetric"), D, 1, lambda: None)
      r["c_ms"] = 1e3 * tc[0]
      r["energy_rel_a_c"] = abs(e_a - ec[0]) / abs(ec[0])
    # _MAP_CACHE after full sweeps of arm (a)
    bs._MAP_CACHE.clear()  # pylint: disable=protected-access
    dm = dmrg(tensors, mpo, lo, "symmetric_b200")
    r["cache_mb"] = []
    for _ in range(args.sweeps):
      dm.run_two_site(max_bond_dim=D, num_sweeps=1, num_krylov_vecs=4, verbose=0)
      torch.cuda.synchronize()
      r["cache_mb"].append(cache_device_bytes() / 2**20)
    print()
    print(json.dumps(r))
    sys.stdout.flush()
    rows.append(r)
  nm = "not measured"
  f = lambda r, k, fmt: fmt % r[k] if k in r else nm
  lines = ["card: %s, power limit: %s, host cores: %d" % (name, pl, os.cpu_count()), "",
           "| D | (a) ms / update | (b) ms / update | (c) ms / update | (a) launches | (a) H2D / D2H bytes | "
           "(b) H2D / D2H bytes | rel. energy (a) vs (b) | (a) vs (c) | `_MAP_CACHE` MB after sweeps 1-%d |" % args.sweeps,
           "|---|---|---|---|---|---|---|---|---|---|"]
  for r in rows:
    lines.append("| %d | %s | %s | %s | %s | %d / %d | %d / %d | %s | %s | %s |" % (
        r["D"], f(r, "a_ms", "%.1f"), f(r, "b_ms", "%.1f"), f(r, "c_ms", "%.1f"), f(r, "a_launches", "%.0f"),
        r["a_bytes"]["HtoD"], r["a_bytes"]["DtoH"], r["b_bytes"]["HtoD"], r["b_bytes"]["DtoH"],
        f(r, "energy_rel_a_b", "%.1e"), f(r, "energy_rel_a_c", "%.1e"), ", ".join("%.1f" % x for x in r["cache_mb"])))
  print("\n".join(lines))
  if args.out:
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "blocksparse_dmrg_bench.md"), "w") as fh:
      fh.write("\n".join(lines) + "\n")
    with open(os.path.join(args.out, "blocksparse_dmrg_bench.json"), "w") as fh:
      json.dump(rows, fh)


if __name__ == "__main__":
  main()
