"""CPU: the adapters' host logic on tests/fake_lib.FakeLib, the numpy stand-in for libtnb200.so.  Each runner installs the
stand-in in a process of its own (tests/hostrun.py says why) and ends with hostrun.OK; the kernels are checked by the
-m gpu tests."""
import os
import subprocess
import sys
import pytest
import fake_lib
import hostrun
from oracle import ref_shim

_REFERENCE = [pytest.mark.refhost,
              pytest.mark.skipif(not ref_shim.available(), reason="upstream TensorNetwork checkout not present")]


@pytest.mark.parametrize("script,args", [
    # the implicitly restarted Arnoldi driver behind CudaB200Backend.eigs against np.linalg.eig
    pytest.param("arnoldi_host_runner.py", [], id="arnoldi"),
    # the restarted GMRES driver behind CudaB200Backend.gmres against scipy.sparse.linalg.gmres
    pytest.param("gmres_host_runner.py", [], id="gmres"),
    # CudaB200Backend.expm: errors, result dtypes, sizes 0 and 1, strided views (and tn.linalg.expm, with the reference)
    pytest.param("expm_host_runner.py", [], id="expm"),
    # the reference's InfiniteMPS.canonicalize, comparison masks, index_update and inv on backend="cuda_b200"
    pytest.param("imps_host_runner.py", [], marks=_REFERENCE, id="imps"),
    # the reference's callers (tn.Node, tn.ncon, contractors, split_node*, FiniteDMRG) on backend="cuda_b200"
    pytest.param("refhost_runner.py", [], marks=_REFERENCE, id="refhost"),
    pytest.param("refhost_runner.py", ["--dmrg"], marks=_REFERENCE, id="refhost-dmrg"),
    # tests/test_gpu_symmetric_adapter.py and the block-sparse maps and errors on backend="symmetric_b200"
    pytest.param("symhost_runner.py", [], marks=_REFERENCE, id="symhost"),
    # tests/test_gpu_symmetric_qr.py on backend="symmetric_b200"
    pytest.param("symqr_host_runner.py", [], marks=_REFERENCE, id="symqr"),
])
def test_runner_on_host_stand_in(script, args):
  r = subprocess.run([sys.executable, os.path.join(hostrun.ROOT, "tests", script)] + args,
                     capture_output=True, text=True, cwd=hostrun.ROOT, timeout=900)
  assert r.returncode == 0 and r.stdout.splitlines()[-1:] == [hostrun.OK], r.stdout[-3000:] + r.stderr[-4000:]


def test_stand_in_covers_the_abi():
  """every entry point of include/tnb200.h but the device query has one host implementation"""
  from tensornetwork_b200 import _lib
  missing = [name for name in _lib.SIGNATURES if name != "tnb200_device_info" and not hasattr(fake_lib.FakeLib, name)]
  assert not missing, missing
