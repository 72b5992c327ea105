"""Build libtnb200.so (sm_90a) in-tree with nvcc.  `python -m tensornetwork_b200.build`.

The .so is git-ignored.  Objects are
rebuilt only when a source or header is newer (cheap `make`-style check).
"""
import concurrent.futures
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "lib", "libtnb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
         "-Xptxas", "-v", "-DTNB200_BUILD"]


def _newer(target, deps):
  if not os.path.exists(target):
    return True
  t = os.path.getmtime(target)
  return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, force=False):
  os.makedirs(OBJ, exist_ok=True)
  os.makedirs(os.path.dirname(LIB), exist_ok=True)
  srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
  hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
  jobs = []
  for s in srcs:
    o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
    if force or _newer(o, [s] + hdrs):
      jobs.append((s, o))

  def cc(job):
    s, o = job
    r = subprocess.run([NVCC] + FLAGS + ["-c", s, "-o", o], capture_output=True, text=True)
    return s, r
  logs = []
  with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
    for s, r in ex.map(cc, jobs):
      logs.append((s, r.stderr))
      if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed on " + s)
      if verbose:
        sys.stderr.write(r.stderr)
  objs = [os.path.join(OBJ, os.path.basename(s)[:-3] + ".o") for s in srcs]
  if force or jobs or _newer(LIB, objs):
    r = subprocess.run([NVCC, "-shared", "-o", LIB] + objs +
                       ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
                        "-Xlinker", "--exclude-libs,ALL"],
                       capture_output=True, text=True)
    if r.returncode != 0:
      sys.stderr.write(r.stdout + r.stderr)
      raise RuntimeError("link failed")
  with open(os.path.join(OBJ, "ptxas.log"), "a") as f:
    for s, l in logs:
      f.write("==== " + s + "\n" + l)
  return LIB


if __name__ == "__main__":
  print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
