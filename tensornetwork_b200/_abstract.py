"""Mirror of the reference plug-in base class for environments where the `tensornetwork`
package is not installed (e.g. on a GPU machine without it).  Same method names as
tensornetwork/backends/abstract_backend.py:22-1046; every operator raises
NotImplementedError("Backend '<name>' has not implemented <op>.") until a subclass
provides it (the behaviour tensornetwork/backends/backend_test.py:160ff asserts)."""

_METHODS = ("tensordot reshape transpose slice svd qr rq shape_concat shape_tensor shape_tuple "
            "sparse_shape shape_prod sqrt convert_to_tensor outer_product einsum norm eye ones "
            "zeros randn random_uniform conj eigh eigs eigsh eigsh_lanczos gmres addition "
            "subtraction multiply divide index_update inv broadcast_right_multiplication "
            "broadcast_left_multiplication sin cos exp log expm jit sum matmul diagflat diagonal "
            "trace abs sign serialize_tensor deserialize_tensor power item cholesky eps").split()


class AbstractBackend:

  def __init__(self):
    self.name = "abstract backend"

  def pivot(self, tensor, pivot_axis=-1):
    """abstract_backend.py:938-962: reshape a tensor into a matrix about `pivot_axis`."""
    ndim = len(self.shape_tuple(tensor))
    if pivot_axis > ndim:
      raise ValueError("pivot_axis = {} was invalid given ndim = {} array.".format(
          pivot_axis, ndim))
    shape = self.shape_tuple(tensor)
    left, right = 1, 1
    for s in shape[:pivot_axis]:
      left *= s
    for s in shape[pivot_axis:]:
      right *= s
    return self.reshape(tensor, (left, right))


def _stub(name):
  def method(self, *args, **kwargs):
    raise NotImplementedError("Backend '{}' has not implemented {}.".format(self.name, name))
  method.__name__ = name
  return method


for _m in _METHODS:
  setattr(AbstractBackend, _m, _stub(_m))
