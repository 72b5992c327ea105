"""The fused thin run (tnb200_thin_run_*): a ramp of thin contractions in one launch, bit-identical to the per-step
kernels, and its use in CompiledNetwork."""
import ctypes

import numpy as np
import pytest

from tensornetwork_b200 import get_backend, drivers, _lib as L

pytestmark = pytest.mark.gpu


def _ramp(be, dtype, mode, nb, lc, ks, seed):
  """A ramp of len(ks) steps like an MPS boundary: step j contracts K = ks[j] with a site (K/2, 2, K) (mode A) or
  (K, 2, K/2) (mode D); the long operand starts as (nb, ks[0], lc) (mode A) or (nb, lc, ks[0]) (mode D)."""
  rng = np.random.default_rng(seed)
  def dev(shape):
    t = rng.standard_normal(shape).astype(np.float32) / np.sqrt(shape[-1] if mode == 0 else shape[1])
    return be.astype(be.convert_to_tensor(t), dtype)
  x = dev((nb, ks[0], lc) if mode == 0 else (nb, lc, ks[0]))
  sites, specs, shape = [], [], list(x.shape)
  for j, k in enumerate(ks):
    s = dev((nb, k // 2, 2, k) if mode == 0 else (nb, k, 2, k // 2))
    sites.append(s)
    if mode == 0:   # a = site (contract its last axis), b = long operand (contract axis 1)
      specs.append((3, 1))
      shape = [nb, k // 2, 2] + shape[2:]
    else:           # a = long operand (contract its last axis), b = site (axis 1)
      specs.append((len(shape) - 1, 1))
      shape = shape[:-1] + [2, k // 2]
  return x, sites, specs, tuple(shape)


def _stepwise(be, x, sites, specs, mode):
  cur = x
  kernels, outs = [], []
  for s, (ax0, ax1) in zip(sites, specs):
    a, b = (s, cur) if mode == 0 else (cur, s)
    cur = be._contract(a, b, [ax0], [ax1], [0], [0])  # pylint: disable=protected-access
    kernels.append(be.lib.tnb200_last_kernel().decode())
    outs.append(cur)
  return outs, kernels


def _create(be, x, sites, specs, mode, out, inter_shapes):
  n = len(sites)
  arr = (L.ChainStep * n)()
  keep = []
  cur = x
  for j, (s, (ax0, ax1)) in enumerate(zip(sites, specs)):
    if j == n - 1:
      c = out
    else:     # an intermediate: the run never writes it, only its layout is read
      c = be._new(inter_shapes[j], x.code)  # pylint: disable=protected-access
      keep.append(c)
    a, b = (s, cur) if mode == 0 else (cur, s)
    cs = arr[j]
    cs.a, cs.b, cs.c = a.desc(), b.desc(), c.desc()
    cs.naxes, cs.nbatch = 1, 1
    cs.axes_a[0], cs.axes_b[0] = ax0, ax1
    cs.batch_a[0] = cs.batch_b[0] = 0
    dep = j - 1 if j else -1
    cs.dep_a, cs.dep_b = (-1, dep) if mode == 0 else (dep, -1)
    cur = c
  handle, bad = ctypes.c_void_p(), ctypes.c_int32(-7)
  rc = be.lib.tnb200_thin_run_create(n, arr, ctypes.byref(bad), ctypes.byref(handle))
  return rc, bad.value, handle, keep


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("nb,lc,ks", [(74, 8192, (64, 32, 16, 8, 4)), (9, 8192, (64, 32, 16)), (1, 65536, (64, 32, 16, 8, 4)),
                                      (140, 2048, (32, 16, 8)), (5, 16384, (16, 8, 4)), (5, 16384, (8, 4))])
def test_thin_run_bit_identical_to_steps(dtype, mode, nb, lc, ks):
  import torch
  be = get_backend()
  x, sites, specs, shape = _ramp(be, dtype, mode, nb, lc, ks, seed=nb + len(ks) + 7 * mode)
  outs, kernels = _stepwise(be, x, sites, specs, mode)
  ref = outs[-1]
  assert all(k.startswith("thin_") for k in kernels), kernels
  n = int(np.prod(shape[1:]))
  tdt = torch.bfloat16 if dtype == "bfloat16" else torch.float16
  buf = torch.full((nb, n + 64), float("nan"), dtype=tdt, device=be.device)
  buf[:, n:] = 12345.0                                     # sentinel in the padding of every sample
  from tensornetwork_b200.tensor import B200Tensor
  out = B200Tensor(buf[:, :n].view((nb,) + shape[1:]), x.code)
  rc, bad, handle, _ = _create(be, x, sites, specs, mode, out, [o.shape for o in outs[:-1]])
  try:
    assert rc == 0 and bad == -1, (rc, bad)
    L.check(be.lib.tnb200_thin_run_launch(handle, be._stream()))  # pylint: disable=protected-access
    assert be.lib.tnb200_last_kernel().decode() == "thin_run"
    first = out.t.clone()
    np.testing.assert_array_equal(first.float().cpu().numpy(), ref.t.float().cpu().numpy())
    assert bool((buf[:, n:] == 12345.0).all())
    buf[:, :n] = float("nan")
    L.check(be.lib.tnb200_thin_run_launch(handle, be._stream()))  # pylint: disable=protected-access
    assert torch.equal(out.t, first)
  finally:
    be.lib.tnb200_thin_run_destroy(handle)


def test_thin_run_rejects_non_local_step():
  """Mode A whose second step contracts the physical leg instead of the bond: not local, step 1 is named."""
  be = get_backend()
  x, sites, specs, shape = _ramp(be, "bfloat16", 0, 9, 8192, (64, 32), seed=3)
  rng = np.random.default_rng(4)
  s1 = be.astype(be.convert_to_tensor(rng.standard_normal((9, 4, 2)).astype(np.float32)), "bfloat16")
  sites = [sites[0], s1]
  specs = [specs[0], (2, 2)]                # contract the (32, [2], 8192) physical axis of step 0's result
  out = be._new((9, 4, 32, 8192), x.code)  # pylint: disable=protected-access
  rc, bad, handle, _ = _create(be, x, sites, specs, 0, out, [(9, 32, 2, 8192)])
  assert rc == L.ERR_UNSUPPORTED and bad == 1 and not handle.value


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_compiled_norm_network_forms_four_thin_runs(dtype):
  be = get_backend()
  Ls, D, NB = 64, 512, 8
  dims = [1] + [min(D, 2 ** min(i, Ls - i)) for i in range(1, Ls)] + [1]
  labels = []
  for side in "kb":
    for i in range(Ls):
      labels.append(["e0" if i == 0 else "%s%d" % (side, i), "p%d" % i, "eL" if i == Ls - 1 else "%s%d" % (side, i + 1)])
  core = [(dims[i], 2, dims[i + 1]) for i in range(Ls)] * 2
  shapes = [(NB,) + s for s in core]
  sizes = {l: s[ax] for s, labs in zip(core, labels) for ax, l in enumerate(labs)}
  path = drivers.greedy_path(labels, [], sizes)
  rng = np.random.default_rng(5)
  kets = [be.astype(be.convert_to_tensor((rng.standard_normal((NB,) + core[i]) / np.sqrt(core[i][0] * 2)).astype(np.float32)),
                    dtype) for i in range(Ls)]
  al = {Ls + i: i for i in range(Ls)}
  net_c = drivers.CompiledNetwork(be, shapes, dtype, labels, [], path=path, nbatch=1, conj_aliases=al, use_chains=True)
  net_s = drivers.CompiledNetwork(be, shapes, dtype, labels, [], path=path, nbatch=1, conj_aliases=al, use_chains=False)
  runs = [c for c in net_c.chains if c.api == "thin_run"]
  assert len(runs) == 4 and all(len(r.steps) >= 5 for r in runs), [r.steps for r in runs]
  assert net_s.launches_per_replay - net_c.launches_per_replay >= 16
  net_c.load(kets + [None] * Ls)
  net_s.load(kets + [None] * Ls)
  ref = net_s().to_host()
  for _ in range(2):
    np.testing.assert_array_equal(net_c().to_host(), ref)
  assert "thin_run" in net_c.profile([(1, 1, 1)] * len(path), NB, 2)
