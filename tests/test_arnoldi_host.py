"""CPU: the implicitly restarted Arnoldi driver behind CudaB200Backend.eigs, on a numpy stand-in for
tnb200_arnoldi_orth (tests/arnoldi_host_runner.py, in a subprocess because it installs a stand-in library)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_arnoldi_driver_on_host_stand_in():
  r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "arnoldi_host_runner.py")],
                     capture_output=True, text=True, cwd=ROOT, timeout=900)
  assert r.returncode == 0 and "ARNOLDI HOST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]
