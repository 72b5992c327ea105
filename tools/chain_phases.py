"""Where the chained GEMM kernel spends its time: a per-phase breakdown of one of the bench's cfg2 chains.

Builds a diagnostic copy of the library with -DTNB200_CHAIN_PHASES into a temporary directory (the default
library is untouched and carries no timers), builds the cfg2 network (L=64, D=512, bf16, 74 samples, the bench's
workload), and replays only one chained launch: `--chain main` (the default) the zipper, `--chain head` the heads of
the four MPS ramps (plan steps 0-11, four independent branches of three steps).  Per launch it prints the chain's
device time (CUDA events) and, averaged over CTAs, the %globaltimer time spent in:
  chain_wait   the producer warp spinning on the dependency counters of a tile's operands
  full_wait    the consumers waiting for a ring stage (starved of operands; measured on one consumer thread)
  k_loop       the whole k loop, full_wait included
  epilogue     from the end of the k loop to the point the tile needs nothing more from the consumers
and, for --G values, the same for other round sizes (TNB200_CHAIN_G).  It also prints the chain's L2 -> SM operand
feed per launch and its rate over the launch time: the operand bytes the kernel's tiles read, computed from the shapes
(per pair of M tiles: its A rows and the B rows of one shared B tile, each K elements deep; rows past the edge of an
operand are not read), not a counter.

  python tools/chain_phases.py [--chain main|head] [--G 9 17 19 38] [--reps 20] [--networks 74]
"""
import argparse
import ctypes
import glob
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
PHASES = ["chain_wait", "full_wait", "k_loop", "epilogue", "cta_life", "tiles"]
BM, BN_16, BN_32 = 128, 256, 128        # the chained kernel's tile (16-bit operands / tf32)


def feed_bytes(m, k, n, esize):
  """L2 -> SM operand bytes of one sample of one chain step (M x K times K x N, `esize`-byte operands): every N tile
  reads all M rows of A, every pair of M tiles all N rows of B (each CTA of the pair loads half of a B tile for both)"""
  bn = BN_32 if esize == 4 else BN_16
  tm, tn = -(-m // BM), -(-n // bn)
  return (tn * m + -(-tm // 2) * n) * k * esize


def build_phase_lib(out_dir):
  from tensornetwork_b200 import build as B
  objs = []
  procs = []
  for s in sorted(glob.glob(os.path.join(B.CSRC, "*.cu"))):
    o = os.path.join(out_dir, os.path.basename(s)[:-3] + ".o")
    procs.append(subprocess.Popen([B.NVCC] + B.FLAGS + ["-DTNB200_CHAIN_PHASES", "-c", s, "-o", o],
                                  stdout=subprocess.DEVNULL, stderr=subprocess.PIPE, text=True))
    objs.append(o)
  for p in procs:
    err = p.communicate()[1]
    if p.returncode:
      sys.stderr.write(err)
      raise RuntimeError("nvcc failed")
  lib = os.path.join(out_dir, "libtnb200.so")
  subprocess.run([B.NVCC, "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
                                                         "-Xlinker", "--exclude-libs,ALL"], check=True)
  return lib


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--G", type=int, nargs="*", default=[], help="round sizes to sweep besides the default")
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--networks", type=int, default=74)
  ap.add_argument("--chain", choices=["main", "head"], default="main",
                  help="main: the zipper (the longest chain); head: the ramp heads (the chain that starts the plan)")
  args = ap.parse_args()
  tmp = tempfile.mkdtemp(prefix="tnb200_phases_")
  lib_path = build_phase_lib(tmp)
  os.environ["TNB200_LIB"] = lib_path
  import torch
  import tensornetwork_b200 as tb
  from tensornetwork_b200 import drivers
  import bench
  raw = ctypes.CDLL(lib_path)
  raw.tnb200_chain_phases.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int32]
  buf = (ctypes.c_ulonglong * (1024 * len(PHASES)))()

  def read(reset):
    if raw.tnb200_chain_phases(buf, 1 if reset else 0) != 0:
      raise RuntimeError("tnb200_chain_phases failed")
    return np.frombuffer(buf, dtype=np.uint64).reshape(1024, len(PHASES)).astype(np.float64)

  be = tb.get_backend()
  L, D, d, NB = bench.L_SITES, bench.BOND, bench.PHYS, args.networks
  dims = bench.mps_dims(L, D, d)
  labels = bench.norm_labels(L)
  core = [(dims[i], d, dims[i + 1]) for i in range(L)] * 2
  shapes = [(NB,) + c for c in core]
  path, work = bench.path_and_work(core, labels)
  kets = []
  for i in range(L):
    t = be.randn(shapes[i], np.float32, seed=1 + i)
    t *= 1.0 / np.sqrt(dims[i] * d)
    kets.append(be.astype(t, "bfloat16"))
  esize = kets[0].t.element_size()
  props = torch.cuda.get_device_properties(0)
  print("device %s, %d SMs, L2 %.0f MB" % (props.name, props.multi_processor_count, props.L2_cache_size / 2**20))
  for G in [None] + list(args.G):
    if G is None:
      os.environ.pop("TNB200_CHAIN_G", None)
    else:
      os.environ["TNB200_CHAIN_G"] = str(G)
    net = drivers.CompiledNetwork(be, shapes, "bfloat16", labels, [], path=path, nbatch=1,
                                  conj_aliases={L + i: i for i in range(L)})
    net.load(kets + list(kets))
    net()
    chains = [c for c in net.chains if c.api == "chain"]
    ch = max(chains, key=lambda c: len(c.steps)) if args.chain == "main" else min(chains, key=lambda c: c.steps[0])
    pairwise = [i for i, st in enumerate(net.steps) if st[0] != "transpose"]     # `work` skips transposes
    flops = NB * sum(2.0 * np.prod(work[pairwise.index(s)]) for s in ch.steps)
    feed = NB * sum(feed_bytes(*work[pairwise.index(s)], esize) for s in ch.steps)
    for _ in range(3):
      ch.launch()
    torch.cuda.synchronize()
    read(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
      ch.launch()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / args.reps
    ph = read(True)
    ctas = int(np.count_nonzero(ph[:, 5]))
    per = ph[:ctas].mean(axis=0) / args.reps
    print("G=%-8s chain %d steps: %8.1f us/launch  %6.1f TFLOP/s  feed %.2f GB %.2f TB/s  | per CTA, us/launch: %s  "
          "tiles %.1f  (%d CTAs)" % (
              "default" if G is None else G, len(ch.steps), us, flops / us / 1e6, feed / 1e9, feed / us / 1e6,
              "  ".join("%s %.1f" % (n, per[i] / 1e3) for i, n in enumerate(PHASES[:5])), per[5], ctas), flush=True)
    del net, ch, chains


if __name__ == "__main__":
  main()
