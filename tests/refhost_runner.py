"""Runs in a subprocess (build container only): the REAL reference's callers on backend="cuda_b200",
with the device layer replaced by tests/fake_lib.FakeLib (host memory).  Checks the adapter's host
logic and the registration path against the reference's own numpy backend."""
import sys
import numpy as np
import hostrun
from hostrun import raises
tn, lib = hostrun.install(reference=True)
import tensornetwork_b200 as tb  # noqa: E402
from tensornetwork_b200 import backend as tb_backend  # noqa: E402
assert tb.registered and tb_backend.HAVE_TENSORNETWORK
from tensornetwork.backends import backend_factory, abstract_backend
be = backend_factory.get_backend("cuda_b200")
assert isinstance(be, abstract_backend.AbstractBackend) and be.name == "cuda_b200"
assert backend_factory.get_backend("cuda_b200") is be   # singleton per name (backend_factory.py:42-46)


import ref_cases  # noqa: E402
dmrg = "--dmrg" in sys.argv
cases = [c for c in ref_cases.CASES if (c[0] == "dmrg") == dmrg]
assert cases
for name, fn, tol in cases:
  ref_cases.compare(name, fn(tn, "cuda_b200"), fn(tn, "numpy"), tol)
  print("case", name, "ok")

# ---- error conventions (numpy_backend.py:92-97, :41) and default-backend machinery
raises(TypeError, be.convert_to_tensor, [1, 2])
raises(ValueError, be.tensordot, be.convert_to_tensor(np.ones((2, 3))), be.convert_to_tensor(np.ones((4, 5))), [[1], [0]])
tn.set_default_backend("cuda_b200")
assert tn.Node(np.ones(3)).backend.name == "cuda_b200"
tn.set_default_backend("numpy")

hostrun.done(lib)
