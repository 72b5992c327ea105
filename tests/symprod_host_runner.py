"""Runs in a subprocess: tests/test_gpu_symmetric_product.py against the symmetric_b200 adapter with the device layer
replaced by tests/fake_symmetry_lib.FakeSymmetryLib (host memory), whose tnb200_blocksparse_maps_nsym transcribes the
kernel's stages.  Checks the product-charge bookkeeping (sector order, bond charges and their types, per-component
moduli) without a GPU."""
import hostrun
tn, _ = hostrun.install(reference=True)
import fake_symmetry_lib  # noqa: E402
lib = fake_symmetry_lib.install()
import tensornetwork_b200 as tb  # noqa: E402
assert tb.registered_symmetric
hostrun.run_gpu_tests("test_gpu_symmetric_product.py", tn, lib)
# product charges reached the nsym map builder, and it never raised
assert lib.calls["tnb200_blocksparse_maps_nsym"] and not lib.raised["tnb200_blocksparse_maps_nsym"], (lib.calls, lib.raised)
hostrun.done(lib)
