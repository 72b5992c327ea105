"""Build-container only (needs the reference checkout): tests/symqr_host_runner.py runs the block-sparse qr / rq tests of
tests/test_gpu_symmetric_qr.py on the symmetric_b200 adapter with a host double of the library."""
import os
import subprocess
import sys
import pytest
from oracle import ref_shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.refhost,
              pytest.mark.skipif(not ref_shim.available(), reason="upstream TensorNetwork checkout not present")]


def test_blocksparse_qr_rq_on_symmetric_b200_adapter():
  r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "symqr_host_runner.py")],
                     capture_output=True, text=True, cwd=ROOT, timeout=600)
  assert r.returncode == 0 and "SYMQR HOST OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
