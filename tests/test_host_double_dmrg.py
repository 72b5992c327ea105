"""CPU: tests/test_gpu_symmetric_dmrg.py (device-resident block-sparse tensors, eigsh_lanczos and FiniteDMRG on
backend="symmetric_b200") on the host stand-in tests/fake_lib.FakeLib, in a process of its own (tests/hostrun.py says
why)."""
import os
import subprocess
import sys
import pytest
import hostrun
from oracle import ref_shim


@pytest.mark.refhost
@pytest.mark.skipif(not ref_shim.available(), reason="upstream TensorNetwork checkout not present")
def test_blocksparse_dmrg_on_host_stand_in():
  r = subprocess.run([sys.executable, os.path.join(hostrun.ROOT, "tests", "symdmrg_host_runner.py")],
                     capture_output=True, text=True, cwd=hostrun.ROOT, timeout=1800)
  assert r.returncode == 0 and r.stdout.splitlines()[-1:] == [hostrun.OK], r.stdout[-3000:] + r.stderr[-4000:]
