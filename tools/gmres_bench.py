"""GMRES timing probe (needs a GPU): the infinite-MPS environment equation x - T(x) / eta + tr(x r) l = b, with T the
unit-cell transfer operator of a random InfiniteMPS (d = 2, two-site unit cell) and l, r its dominant left and right
eigenvectors, solved through the reference's `tensornetwork.linalg.krylov.gmres` on backend="cuda_b200"
(num_krylov_vectors=30, tol=1e-10, atol=0), against scipy.sparse.linalg.gmres on the host with the same operator on
backend="numpy" (the reference's NumPyBackend.gmres passes `tol=`, which SciPy 1.14 removed, so scipy is called
directly).
python tools/gmres_bench.py [--sizes 64,256,512,1024] [--c128 512] [--numpy-max 256]

One JSON line naming the card, its power limit and max SM clock, then one line per case: wall time (host clock around
a synchronised call, best of 3 after one warm-up), cycles, matvecs, launches, host reads, the time spent in
tnb200_arnoldi_orth (CUDA events) with the bytes it must move over that time, scipy's time and info, ||b - A x|| / ||b||
and ||x - x_scipy|| / ||x_scipy||."""
import json
import os
import sys
import time
import numpy as np
import scipy.sparse.linalg as spla
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from eigs_bench import HBM, OrthTimer, card, tn  # noqa: E402
import torch  # noqa: E402
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import gmres  # noqa: E402
from tensornetwork.linalg import krylov  # noqa: E402
from tensornetwork.matrixproductstates.infinite_mps import InfiniteMPS  # noqa: E402

TOL, NKV, MAXITER = 1e-10, 30, 1000


def environment_operator(mps, l, r, eta):
  """x -> x - T(x) / eta + tr(x r) l on mps's backend"""
  be = mps.backend

  def op(x):
    tx = mps.unit_cell_transfer_operator("l", x)
    return x - tx * (1.0 / eta) + be.tensordot(x, r, ([0, 1], [1, 0])) * l
  return op


def problem(D, dtype):
  """the state on cuda_b200, its eta and l, r (tr(l r) = 1), and the same state on numpy.  The state is not
  canonicalised: for a real state canonicalize returns complex tensors (its eigh gauge carries phases), and dividing T
  by eta poses the same equation."""
  np.random.seed(D)
  ref = InfiniteMPS.random(d=[2, 2], D=[D] * 3, dtype=dtype, backend="numpy")
  mps = InfiniteMPS(tensors=[np.asarray(t) for t in ref.tensors], center_position=0, backend="cuda_b200")
  eta, l = mps.transfer_matrix_eigs("l")
  _, r = mps.transfer_matrix_eigs("r")
  eta, lh, rh = complex(eta.item()), l.to_host(), r.to_host()
  if np.dtype(dtype).kind != "c":                       # a real operator's dominant eigenpair, rotated to be real
    lh, rh = [v * (abs(v.flat[np.argmax(np.abs(v))]) / v.flat[np.argmax(np.abs(v))]) for v in (lh, rh)]
    eta, lh, rh = eta.real, lh.real, rh.real
  lh = lh / np.linalg.norm(lh)
  rh = rh / np.trace(lh @ rh)
  return mps, ref, lh.astype(dtype), rh.astype(dtype), eta


def case(D, dtype, numpy_max):
  mps, host, lh, rh, eta = problem(D, dtype)
  be = mps.backend
  op = environment_operator(mps, be.convert_to_tensor(lh), be.convert_to_tensor(rh), eta)
  b = np.random.default_rng(D).standard_normal((D, D))
  if np.dtype(dtype).kind == "c":
    b = b + 1j * np.random.default_rng(D + 1).standard_normal((D, D))
  b = b.astype(dtype)
  bT = tn.Tensor(be.convert_to_tensor(b), backend="cuda_b200")

  def A_mv(X):
    return tn.Tensor(op(X.array), backend="cuda_b200")
  info = {}

  def gmres_info(*a, **k):                    # the backend method, keeping the driver's statistics
    be._no_capture("gmres")
    x, i, st = gmres.gmres(be, *a, return_info=True, **k)
    info.update(st, info=i)
    return x, i
  be.gmres = gmres_info
  times = []
  try:
    for it in range(4):
      torch.cuda.synchronize()
      n0 = be.lib.tnb200_launch_count()
      t0 = time.perf_counter()
      x, _ = krylov.gmres(A_mv, bT, tol=TOL, atol=0.0, num_krylov_vectors=NKV, maxiter=MAXITER)
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
      krylov.gmres(A_mv, bT, tol=TOL, atol=0.0, num_krylov_vectors=NKV, maxiter=MAXITER)
      orth_ms = timer.ms()
      lib.tnb200_arnoldi_orth = timer.fn
  finally:
    del be.gmres
  xd = x.array
  res = float((be.norm(bT.array - op(xd)) / be.norm(bT.array)).item())
  out = {"D": D, "dtype": np.dtype(dtype).name, "n": D * D, "wall_ms": min(times) * 1e3, "info": info["info"],
         "cycles": info["cycles"], "matvecs": info["matvecs"], "launches": launches, "host_reads": info["host_reads"],
         "residual": res}
  if timer is not None:
    out.update({"orth_ms": orth_ms, "orth_GB": timer.bytes / 1e9, "orth_TBps": timer.bytes / (orth_ms * 1e-3) / 1e12,
                "orth_share_of_3.35TBps": timer.bytes / (orth_ms * 1e-3) / HBM})
  if D <= numpy_max:
    hop = environment_operator(host, lh, rh, eta)
    A = spla.LinearOperator((D * D, D * D), matvec=lambda v: np.asarray(hop(v.reshape(D, D))).ravel(), dtype=b.dtype)
    t0 = time.perf_counter()
    xs, sinfo = spla.gmres(A, b.ravel(), rtol=TOL, atol=0.0, restart=NKV, maxiter=MAXITER)
    out["scipy_ms"] = (time.perf_counter() - t0) * 1e3
    out["scipy_info"] = int(sinfo)
    out["x_rel_diff"] = float(np.linalg.norm(xd.to_host().ravel() - xs) / np.linalg.norm(xs))
  else:
    out["scipy_ms"] = "not measured"
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
