"""Runs in a subprocess: tests/test_gpu_symmetric_qr.py against the symmetric_b200 adapter with the device layer replaced by
tests/fake_lib.FakeLib (host memory), whose `tnb200_qr_batched` honours `adjoint` and, like the kernel, computes f32 / c64
in double precision.  Checks the adapter's charge, flow and order bookkeeping and the split of sectors between the batched
launch and the per-sector tnb200_qr without a GPU."""
import hostrun
tn, lib = hostrun.install(reference=True)
import tensornetwork_b200 as tb  # noqa: E402
assert tb.registered_symmetric
for name, params, calls in hostrun.run_gpu_tests("test_gpu_symmetric_qr.py", tn, lib):
  if name == "test_sectors_over_the_batched_limit_fall_back":
    assert calls["tnb200_qr_batched"] and calls["tnb200_qr"], ("the batched launch or the fallback did not run", params)
hostrun.done(lib)
