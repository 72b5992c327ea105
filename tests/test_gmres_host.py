"""CPU: the restarted GMRES driver behind CudaB200Backend.gmres against scipy.sparse.linalg.gmres, on a numpy stand-in
for tnb200_arnoldi_orth (tests/gmres_host_runner.py, in a subprocess because it installs a stand-in library)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gmres_driver_on_host_stand_in():
  r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "gmres_host_runner.py")],
                     capture_output=True, text=True, cwd=ROOT, timeout=900)
  assert r.returncode == 0 and "GMRES HOST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]
