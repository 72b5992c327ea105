"""tensornetwork_b200 — H100-native (sm_90a) contraction + split engine behind
google/TensorNetwork's `AbstractBackend` surface, selected with backend="cuda_b200".

Importing this package is cheap: it neither imports torch nor touches CUDA (the reference
requires lazy backend dependencies).  If the `tensornetwork` package is installed, the
backend is registered in its factory on import.
"""
from . import backend as _backend
from .backend import CudaB200Backend, get_instance
from .tensor import B200Tensor, bfloat16

__version__ = "0.1.0"
registered = _backend.register()
registered_symmetric = False
if registered:
  try:
    from . import symmetric as _symmetric
    registered_symmetric = _symmetric.register() is not None   # "symmetric_b200": the reference's SymmetricBackend, hot ops on the device
  except Exception:  # pylint: disable=broad-except
    registered_symmetric = False


def get_backend():
  """The singleton backend instance (constructs it: needs a CUDA device)."""
  return get_instance()
