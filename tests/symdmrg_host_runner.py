"""Runs in a subprocess: tests/test_gpu_symmetric_dmrg.py (device-resident block-sparse tensors, `eigsh_lanczos` and
FiniteDMRG on backend="symmetric_b200") with the device layer replaced by tests/fake_symmetry_lib.FakeSymmetryLib (host
memory).  Checks the residency bookkeeping, the permutation maps and the Lanczos plumbing without a GPU."""
import hostrun
tn, _ = hostrun.install(reference=True)
import fake_symmetry_lib  # noqa: E402
lib = fake_symmetry_lib.install()
import tensornetwork_b200 as tb  # noqa: E402
assert tb.registered_symmetric
hostrun.run_gpu_tests("test_gpu_symmetric_dmrg.py", tn, lib)
# the device paths ran: permutation maps (scatter), contiguous (gather), the grouped contraction, norms and dots
for name in ("tnb200_gather", "tnb200_blocksparse_tensordot", "tnb200_blocksparse_maps", "tnb200_blocksparse_maps_nsym",
             "tnb200_norm", "tnb200_dot", "tnb200_axpy"):
  assert lib.calls[name], (name, lib.calls)
hostrun.done(lib)
