"""Kernel-level throughput probe (needs a GPU): times N back-to-back launches of one tensordot
shape with CUDA events, so that the host round trip is amortised.  Prints one JSON line per case."""
import json
import sys
import os
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import tensornetwork_b200 as tb


def run(be, dtype, shape_a, shape_b, axes, reps=50, batch=None):
  rng = np.random.default_rng(0)
  tdt = {"bf16": torch.bfloat16, "f32": torch.float32, "f64": torch.float64, "f16": torch.float16}[dtype]
  a = tb.B200Tensor(torch.randn(shape_a, device=be.device, dtype=torch.float32).to(tdt))
  b = tb.B200Tensor(torch.randn(shape_b, device=be.device, dtype=torch.float32).to(tdt))
  if batch:
    f = lambda: be.matmul(a, b)
  else:
    f = lambda: be.tensordot(a, b, axes)
  for _ in range(3):
    out = f()
  torch.cuda.synchronize()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    for _ in range(reps):
      out = f()
  kern = be.lib.tnb200_last_kernel().decode()
  g.replay()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  g.replay()
  e1.record()
  torch.cuda.synchronize()
  ms = e0.elapsed_time(e1) / reps
  sa, sb = a.shape, b.shape
  if batch:
    flops = 2.0 * np.prod(sa) * sb[-1]
  else:
    ka = [sa[i] for i in axes[0]]
    flops = 2.0 * np.prod(sa) * np.prod(sb) / np.prod(ka)
  es = {"bf16": 2, "f16": 2, "f32": 4, "f64": 8}[dtype]
  byts = (np.prod(sa) + np.prod(sb) + out.size) * es
  print(json.dumps({"dtype": dtype, "a": list(sa), "b": list(sb), "axes": axes if not batch else "matmul", "kernel": kern,
                    "us": ms * 1e3, "tflops": flops / ms / 1e9, "gbs": byts / ms / 1e6}))


if __name__ == "__main__":
  be = tb.get_backend()
  if len(sys.argv) > 1 and sys.argv[1] == "--flagship":
    # one batched flagship launch family only (used under ncu): 64 x [(1024 x 512) . (512 x 1024)]
    dt = sys.argv[2] if len(sys.argv) > 2 else "bf16"
    run(be, dt, (64, 1024, 512), (64, 512, 1024), None, reps=3, batch=True)
    run(be, dt, (512, 2, 512), (512, 2, 512), [[2], [0]], reps=3)
    sys.exit(0)
  if len(sys.argv) > 1 and sys.argv[1] == "--ramp":
    # the thin ramp-up steps of cfg 2 (small matrix x long tensor, 74 samples): GB/s of each layout / width
    nb = int(sys.argv[2]) if len(sys.argv) > 2 else 74
    for k in (2, 4, 8, 16, 32, 64, 128):
      L = 524288 // k
      for mode in ("A", "D"):
        if mode == "A":
          S = tb.B200Tensor(torch.randn((nb, k, k), device=be.device).to(torch.bfloat16))
          X = tb.B200Tensor(torch.randn((nb, k, L), device=be.device).to(torch.bfloat16))
          f = lambda: be._contract(S, X, [2], [1], [0], [0])
        else:
          X = tb.B200Tensor(torch.randn((nb, L, k), device=be.device).to(torch.bfloat16))
          S = tb.B200Tensor(torch.randn((nb, k, k), device=be.device).to(torch.bfloat16))
          f = lambda: be._contract(X, S, [2], [1], [0], [0])
        for _ in range(3):
          f()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 20
        e0.record()
        for _ in range(reps):
          f()
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / reps
        byts = nb * 2.0 * (2 * k * L + k * k)
        print(json.dumps({"ramp_k": k, "mode": mode, "kernel": be.lib.tnb200_last_kernel().decode(), "us": round(us, 1),
                          "gbs": round(byts / us / 1e3, 1)}))
    sys.exit(0)
  if len(sys.argv) > 1 and sys.argv[1] == "--stepab":
    # eager launches of the two bulk cfg-2 steps at NB samples (for ncu --set full captures)
    nb = int(sys.argv[2]) if len(sys.argv) > 2 else 32
    A = tb.B200Tensor(torch.randn((nb, 512, 2, 512), device=be.device, dtype=torch.float32).to(torch.bfloat16))
    E = tb.B200Tensor(torch.randn((nb, 512, 512), device=be.device, dtype=torch.float32).to(torch.bfloat16))
    Tt = tb.B200Tensor(torch.randn((nb, 2, 512, 512), device=be.device, dtype=torch.float32).to(torch.bfloat16))
    for _ in range(4):
      be._contract(A, E, [1], [2], [0], [0])
      be._contract(A, Tt, [1, 2], [3, 1], [0], [0])
    torch.cuda.synchronize()
    print("done", be.lib.tnb200_last_kernel().decode())
    sys.exit(0)
  if len(sys.argv) > 1 and sys.argv[1] == "--svd":
    import time
    sizes = [int(x) for x in sys.argv[2:]] or [1024, 2048]
    for n in sizes:
      rng = np.random.default_rng(4)
      m = rng.standard_normal((n, n)) / np.sqrt(n)
      M = be.convert_to_tensor(m)
      info = torch.zeros(4, dtype=torch.int32, device=be.device)
      u = be._new((n, n), M.code); sv = be._new((n,), M.code); vh = be._new((n, n), M.code)
      from tensornetwork_b200 import _lib as L
      for rep in range(2):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        L.check(be.lib.tnb200_svd(M.ref(), u.ref(), sv.ref(), vh.ref(), info.data_ptr(), be._stream()))
        torch.cuda.synchronize(); dt = time.perf_counter() - t0
      t0 = time.perf_counter(); ref = np.linalg.svd(m, compute_uv=True, full_matrices=False); tc = time.perf_counter() - t0
      err = float(np.abs(sv.to_host() - ref[1]).max() / ref[1][0])
      rec = float(np.linalg.norm((u.to_host() * sv.to_host()) @ vh.to_host() - m) / np.linalg.norm(m))
      print(json.dumps({"svd_n": n, "gpu_s": dt, "cpu_numpy_s": tc, "sweeps": int(info[0]), "converged": int(info[1]),
                        "s_err_rel": err, "recon_rel": rec, "gflops_21n3": 21.0 * n**3 / dt / 1e9}))
    sys.exit(0)
  if len(sys.argv) > 1 and sys.argv[1] == "--cfg2steps":
    # the two bulk steps of the cfg-2 zipper, batched over NB samples, timed individually
    dt = sys.argv[2] if len(sys.argv) > 2 else "bf16"
    tdt = {"bf16": torch.bfloat16, "f32": torch.float32, "f64": torch.float64}[dt]
    for nb in (1, 8, 32):
      A = tb.B200Tensor(torch.randn((nb, 512, 2, 512), device=be.device, dtype=torch.float32).to(tdt))
      E = tb.B200Tensor(torch.randn((nb, 512, 512), device=be.device, dtype=torch.float32).to(tdt))
      Tt = tb.B200Tensor(torch.randn((nb, 2, 512, 512), device=be.device, dtype=torch.float32).to(tdt))
      for name, f, fl in (("a: A(512,2,512)[0] x E(512,512)[1]", lambda: be._contract(A, E, [1], [2], [0], [0]), 2.0 * 1024 * 512 * 512),
                          ("b: A(512,2,512)[0,1] x T(2,512,512)[2,0]", lambda: be._contract(A, Tt, [1, 2], [3, 1], [0], [0]), 2.0 * 512 * 1024 * 512)):
        for _ in range(3):
          f()
        torch.cuda.synchronize()
        l0 = be.lib.tnb200_launch_count()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
          for _ in range(20):
            f()
        nl = (be.lib.tnb200_launch_count() - l0) / 20
        g.replay(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) / 20 * 1e3
        print(json.dumps({"step": name, "nb": nb, "dtype": dt, "kernel": be.lib.tnb200_last_kernel().decode(),
                          "launches": nl, "us": us, "tflops": nb * fl / us / 1e6}))
    sys.exit(0)
  for dt in ("bf16", "f32", "f64"):
    run(be, dt, (512, 2, 512), (512, 2, 512), [[2], [0]])
    run(be, dt, (512, 2, 512), (512, 2, 512), [[0], [2]])
    run(be, dt, (1024, 512), (512, 512), [[1], [0]])
    run(be, dt, (4096, 4096), (4096, 4096), [[1], [0]], reps=10)
    run(be, dt, (4096, 4096), (4096, 4096), [[0], [1]], reps=10)
    run(be, dt, (8192, 1024), (1024, 8192), [[1], [0]], reps=10)
    run(be, dt, (64, 1024, 512), (64, 512, 1024), None, reps=10, batch=True)
    run(be, dt, (256, 1024, 512), (256, 512, 1024), None, reps=5, batch=True)
