"""CPU: tests/test_gpu_symmetric_product.py (product charges on backend="symmetric_b200") on the host stand-in
tests/fake_lib.FakeLib, in a process of its own (tests/hostrun.py says why)."""
import os
import subprocess
import sys
import pytest
import hostrun
from oracle import ref_shim


@pytest.mark.refhost
@pytest.mark.skipif(not ref_shim.available(), reason="upstream TensorNetwork checkout not present")
def test_product_charges_on_host_stand_in():
  r = subprocess.run([sys.executable, os.path.join(hostrun.ROOT, "tests", "symprod_host_runner.py")],
                     capture_output=True, text=True, cwd=hostrun.ROOT, timeout=1800)
  assert r.returncode == 0 and r.stdout.splitlines()[-1:] == [hostrun.OK], r.stdout[-3000:] + r.stderr[-4000:]


def test_symmetry_header_is_exported_bound_and_stood_in():
  """every entry point of include/tnb200_symmetry.h is exported by the library, has a ctypes prototype, and has a host
  implementation in tests/fake_symmetry_lib"""
  import ctypes
  import re
  import fake_symmetry_lib
  from tensornetwork_b200 import _lib
  src = open(os.path.join(hostrun.ROOT, "include", "tnb200_symmetry.h")).read()
  names = sorted(set(re.findall(r"TNB200_API[^;]*?\b(tnb200_\w+)\s*\(", src)))
  assert names and sorted(_lib.SYMMETRY_SIGNATURES) == names
  assert not set(names) & set(_lib.SIGNATURES)
  lib = ctypes.CDLL(_lib.LIB_PATH)
  for n in names:
    assert hasattr(lib, n), "missing export " + n
    assert hasattr(fake_symmetry_lib.FakeSymmetryLib, n), "no host stand-in for " + n
  assert "#define TNB200_BLOCKSPARSE_MAX_NSYM %d\n" % _lib.BLOCKSPARSE_MAX_NSYM in src
  assert _lib.BLOCKSPARSE_MAX_BINS == 1 << 22 and "#define TNB200_BLOCKSPARSE_MAX_BINS (1 << 22)\n" in src
