"""CPU: the reference's InfiniteMPS.canonicalize on backend="cuda_b200", with numpy stand-ins for the device entry points
it reaches (tests/imps_host_runner.py, in a subprocess because it installs a stand-in library): results against
backend="numpy", the comparison and index_update semantics of the adapter, and inv's error conventions."""
import os
import subprocess
import sys
import pytest
from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.refhost,
              pytest.mark.skipif(not ref_shim.available(), reason="upstream TensorNetwork checkout not present")]


def test_canonicalize_on_host_stand_in():
  r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "imps_host_runner.py")],
                     capture_output=True, text=True, cwd=ROOT, timeout=900)
  assert r.returncode == 0 and "IMPS HOST OK" in r.stdout, r.stdout[-3000:] + r.stderr[-4000:]
