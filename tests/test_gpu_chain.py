"""Every step of the chained GEMM launch (tnb200_chain_create / launch / destroy: the wgmma_chain_16 and
wgmma_chain_tf32 kernels) checked element by element against float64.

The cases drive the C ABI directly with L.ChainStep arrays.  Every output is filled with NaN before each launch, so
a box the kernel fails to store stays NaN instead of keeping an earlier run's correct value.  Each element of each
step must satisfy the a-priori bound

    |c - r| <= u_out |r| + (u_in + K 2^-23) s,    r = a . b,  s = |a| . |b|   (float64, K = contracted extent)

where a, b are the operands the step actually read (for a dependent operand: the producing step's device output).
u_out bounds the rounding of the fp32 result to the output type: 2^-8 for bf16 (its unit roundoff: an 8-bit
significand, so round-to-nearest errors come within a hair of the bound), 2^-10 for f16 and 2^-23 for f32 (twice
theirs).  u_in is 0 for 16-bit inputs (their products are exact in fp32) and 2^-9 for tf32 (10 explicit mantissa bits
per operand), and K 2^-23 covers the fp32 accumulation.  The constants are derived, not fitted: a ratio above 1 is a
bug.  Each step's output must also be bit-identical to the single-GEMM launch (be._contract) on the same device
operands, tf32 included, and a second launch of the same handle must reproduce the first bit for bit (the dependency
counters are reset by every launch)."""
import ctypes
import numpy as np
import pytest
from util import get_backend, rel_err

pytestmark = pytest.mark.gpu

DTYPES = ["bfloat16", "float16", "float32"]
# (samples, TNB200_CHAIN_G): one unbatched sample with the default round size, then rounds of 1, 2 and all samples
BATCH_G = [(1, None), (5, 1), (5, 2), (7, 7)]
U_OUT = {"bfloat16": 2.0**-8, "float16": 2.0**-10, "float32": 2.0**-23}
U_IN = {"bfloat16": 0.0, "float16": 0.0, "float32": 2.0**-9}
CHAIN_KERNELS = ("wgmma_chain_16", "wgmma_chain_tf32")
# bond dimensions of the MPS environment updates: none is a multiple of the 128-row or 256-column tile
ZIP_BONDS = (136, 200, 264, 200)
# bonds under which steps s and s + 2 have the same output shape, so that they can share one buffer
RING_BONDS = (136, 200, 200, 200)
SENTINEL = -7.5


def _L():
  from tensornetwork_b200 import _lib as L  # pylint: disable=import-outside-toplevel
  return L


def _torch():
  import torch  # pylint: disable=import-outside-toplevel
  return torch


class _Step:
  """One chain step: c = einsum(spec, a, b) with tnb200's output order (batch, free modes of a, free modes of b)."""

  def __init__(self, spec, a, b, c, dep_a=-1, dep_b=-1):
    ins, out = spec.split("->")
    la, lb = ins.split(",")
    bat = [x for x in out if x in la and x in lb]
    con = [x for x in la if x in lb and x not in out]
    assert out == "".join(bat + [x for x in la if x not in lb] + [x for x in lb if x not in la]), spec
    self.spec, self.a, self.b, self.c, self.dep_a, self.dep_b = spec, a, b, c, dep_a, dep_b
    self.ax_a, self.ax_b = [la.index(x) for x in con], [lb.index(x) for x in con]
    self.ba, self.bb = [la.index(x) for x in bat], [lb.index(x) for x in bat]
    self.K = int(np.prod([a.shape[la.index(x)] for x in con]))


def _spec(spec, batched):
  return spec if batched else spec.replace("b", "")


def _dev(be, rng, shape, dtype, scale=1.0):
  x = (rng.standard_normal(shape) * scale).astype(np.float32)
  t = be.convert_to_tensor(x)
  return t if dtype == "float32" else be.astype(t, dtype)


def _host64(t):
  return t.to_host().astype(np.float64)


def _bits(t):
  torch = _torch()
  t = t.contiguous()
  return t.view(torch.int32 if t.element_size() == 4 else torch.int16).cpu().numpy()


def _chain_array(steps):
  L = _L()
  arr = (L.ChainStep * len(steps))()
  for cs, s in zip(arr, steps):
    cs.a, cs.b, cs.c = s.a.desc(), s.b.desc(), s.c.desc()
    cs.naxes, cs.nbatch = len(s.ax_a), len(s.ba)
    for j, (x, y) in enumerate(zip(s.ax_a, s.ax_b)):
      cs.axes_a[j], cs.axes_b[j] = x, y
    for j, (x, y) in enumerate(zip(s.ba, s.bb)):
      cs.batch_a[j], cs.batch_b[j] = x, y
    cs.dep_a, cs.dep_b = s.dep_a, s.dep_b
  return arr


def _create(be, steps):
  bad, handle = ctypes.c_int32(-1), ctypes.c_void_p()
  rc = be.lib.tnb200_chain_create(len(steps), _chain_array(steps), ctypes.byref(bad), ctypes.byref(handle))
  return rc, bad.value, handle


def _launch(be, handle, steps):
  """NaN into every output, one launch, synchronize; returns a device copy of every step's output."""
  torch = _torch()
  for s in steps:
    s.c.t.fill_(float("nan"))
  l0 = be.lib.tnb200_launch_count()
  assert be.lib.tnb200_chain_launch(handle, be._stream()) == 0, be.lib.tnb200_last_error()  # pylint: disable=protected-access
  torch.cuda.synchronize()
  assert be.lib.tnb200_last_kernel().decode() in CHAIN_KERNELS, be.lib.tnb200_last_kernel()
  assert be.lib.tnb200_launch_count() - l0 == 1
  return [s.c.t.clone() for s in steps]


def _launch_twice(be, steps):
  """create, launch twice (outputs NaN-filled before each), destroy; the two launches must agree bit for bit"""
  rc, bad, handle = _create(be, steps)
  assert (rc, bad) == (0, -1), (rc, bad, be.lib.tnb200_last_error())
  try:
    first = _launch(be, handle, steps)
    second = _launch(be, handle, steps)
  finally:
    be.lib.tnb200_chain_destroy(handle)
  for i, (x, y) in enumerate(zip(first, second)):
    assert _torch().isfinite(x.float()).all(), "step %d: unwritten (NaN) output elements after the launch" % i
    np.testing.assert_array_equal(_bits(x), _bits(y), err_msg="step %d: second launch differs" % i)
  return first


def _check_steps(be, steps, dtype, outs):
  """the float64 bound and bit identity with one single-GEMM launch, for every step; returns the largest error/bound"""
  worst = 0.0
  for i, (s, c) in enumerate(zip(steps, outs)):
    a, b = _host64(s.a), _host64(s.b)
    got = c.float().cpu().numpy().astype(np.float64)
    r = np.einsum(s.spec, a, b, optimize=True)
    sabs = np.einsum(s.spec, np.abs(a), np.abs(b), optimize=True)
    bound = U_OUT[dtype] * np.abs(r) + (U_IN[dtype] + s.K * 2.0**-23) * sabs
    ratio = np.abs(got - r) / bound
    worst = max(worst, float(ratio.max()))
    l0 = be.lib.tnb200_launch_count()
    single = be._contract(s.a, s.b, s.ax_a, s.ax_b, s.ba, s.bb)  # pylint: disable=protected-access
    kern = be.lib.tnb200_last_kernel().decode()
    assert kern.startswith("wgmma") and be.lib.tnb200_launch_count() - l0 == 1, (i, kern)
    differ = int((_bits(single.t) != _bits(c)).sum())
    # both checks are reported together: a rounding fault can break either or both
    assert ratio.max() <= 1.0 and differ == 0, (
        "step %d (%s): error/bound %.3g at %s; %d elements differ from the single-GEMM launch (%s)" %
        (i, s.spec, ratio.max(), np.unravel_index(ratio.argmax(), ratio.shape), differ, kern))
  print("%s: largest error/bound %.3f" % (dtype, worst))
  return worst


def _env(monkeypatch, G):
  monkeypatch.setenv("TNB200_CHAIN_FORCE", "1")     # these batches are below the size at which chaining pays off
  if G is None:
    monkeypatch.delenv("TNB200_CHAIN_G", raising=False)
  else:
    monkeypatch.setenv("TNB200_CHAIN_G", str(G))


# ------------------------------------------------------------------------------------------------ the cases
def _zipper_inputs(be, rng, dtype, nb, bonds):
  """E_0 and the ket / bra site tensors A_i, A'_i (m_i, 2, m_i+1); each scaled by 1/sqrt(K) of the step that reads it"""
  pre = (nb,) if nb > 1 else ()
  e0 = _dev(be, rng, pre + (bonds[0], bonds[0]), dtype)
  sites = []
  for m, n in zip(bonds[:-1], bonds[1:]):
    sites.append((_dev(be, rng, pre + (m, 2, n), dtype, m ** -0.5), _dev(be, rng, pre + (m, 2, n), dtype, (2 * m) ** -0.5)))
  return e0, sites


def _zipper_steps(be, inputs, nb, out=None):
  """the MPS environment update over every site: T_i[x,p,n] = E_i[x,m] A_i[m,p,n] (ragged K = m, fused (p, n) group),
  E_i+1[n,k] = T_i[x,p,n] A'_i[x,p,k] (both operands MN-major).  out(step, shape, code) allocates a step's C."""
  e, sites = inputs
  code = e.code
  pre = (nb,) if nb > 1 else ()
  out = out or (lambda i, shape, code: be._new(shape, code))  # pylint: disable=protected-access
  steps, dep = [], -1
  for a, a_bra in sites:
    x, n = e.shape[-2], a.shape[-1]
    t = out(len(steps), pre + (x, 2, n), code)
    steps.append(_Step(_spec("bxm,bmpn->bxpn", nb > 1), e, a, t, dep_a=dep))
    e = out(len(steps), pre + (n, n), code)
    steps.append(_Step(_spec("bxpn,bxpk->bnk", nb > 1), t, a_bra, e, dep_a=len(steps) - 1))
    dep = len(steps) - 1
  return steps


def _dag_steps(be, rng, dtype, nb):
  """six steps: a root, dep_a only, dep_b only (fan-out of the root), both operands from two steps, the Gram C0^T C0
  (dep_a = dep_b = 0) and an independent step placed last; K-major and MN-major operands vary across the steps."""
  pre = (nb,) if nb > 1 else ()
  bt = (lambda t: be.transpose(t, (0, 2, 1))) if nb > 1 else be.transpose
  from tensornetwork_b200 import tensor as T  # pylint: disable=import-outside-toplevel
  code = T.dtype_code(dtype)
  M0, K0, N0, N1, M5, K5, N5 = 200, 136, 264, 136, 144, 72, 328
  p0 = _dev(be, rng, pre + (M0, K0), dtype)                          # K-major
  q0 = _dev(be, rng, pre + (K0, N0), dtype, K0 ** -0.5)              # MN-major
  q1 = bt(_dev(be, rng, pre + (N1, N0), dtype, N0 ** -0.5))          # view (N0, N1), K-major
  p2 = bt(_dev(be, rng, pre + (M0, M0), dtype, M0 ** -0.5))          # view (M2, K = M0), MN-major
  x5 = _dev(be, rng, pre + (M5, K5), dtype)
  y5 = _dev(be, rng, pre + (N5, K5), dtype, K5 ** -0.5)              # read as (N, K): K-major
  new = lambda *shape: be._new(pre + shape, code)  # pylint: disable=protected-access,unnecessary-lambda-assignment
  c0, c1, c2, c3, g, c5 = new(M0, N0), new(M0, N1), new(M0, N0), new(N0, N1), new(N0, N0), new(M5, N5)
  b = nb > 1
  return [
      _Step(_spec("bmk,bkn->bmn", b), p0, q0, c0),
      _Step(_spec("bmk,bkn->bmn", b), c0, q1, c1, dep_a=0),          # both K-major (a 32 KB stage in tf32)
      _Step(_spec("bmk,bkn->bmn", b), p2, c0, c2, dep_b=0),          # both MN-major
      _Step(_spec("bkm,bkn->bmn", b), c2, c1, c3, dep_a=2, dep_b=1),
      _Step(_spec("bkm,bkn->bmn", b), c0, c0, g, dep_a=0, dep_b=0),
      _Step(_spec("bmk,bnk->bmn", b), x5, y5, c5),                   # both K-major, no dependency
  ]


@pytest.mark.parametrize("nb,G", BATCH_G)
@pytest.mark.parametrize("dtype", DTYPES)
def test_chain_zipper_ragged(dtype, nb, G, monkeypatch):
  """ragged M, N and K: partial and fully out-of-range store boxes, zero-filled K blocks, the fused (p, n) group"""
  _env(monkeypatch, G)
  be = get_backend()
  steps = _zipper_steps(be, _zipper_inputs(be, np.random.default_rng(41), dtype, nb, ZIP_BONDS), nb)
  _check_steps(be, steps, dtype, _launch_twice(be, steps))


@pytest.mark.parametrize("nb,G", BATCH_G)
@pytest.mark.parametrize("dtype", DTYPES)
def test_chain_dependency_shapes(dtype, nb, G, monkeypatch):
  """dependencies on a non-adjacent step, fan-out, both operands from one step, and a step with none"""
  _env(monkeypatch, G)
  be = get_backend()
  steps = _dag_steps(be, np.random.default_rng(42), dtype, nb)
  _check_steps(be, steps, dtype, _launch_twice(be, steps))


@pytest.mark.parametrize("nb,G", BATCH_G)
@pytest.mark.parametrize("dtype", DTYPES)
def test_chain_padded_outputs(dtype, nb, G, monkeypatch):
  """each C whose N group is one mode is a view big[:nb, :M, :N] of a buffer padded in rows (pitch N + 8) and in
  batch: the TMA store must clip to the view and leave every pad element as it was"""
  _env(monkeypatch, G)
  be = get_backend()
  torch = _torch()
  bigs = []

  def out(i, shape, code):
    if i % 2 == 0:                                 # T_i: its N group (p, n) is fused, it cannot be padded
      return be._new(shape, code)  # pylint: disable=protected-access
    rows, cols = shape[-2], shape[-1]
    pad = (shape[0] + 1, rows + 3, cols + 8) if nb > 1 else (rows + 3, cols + 8)
    big = be._new(pad, code)  # pylint: disable=protected-access
    big.t.fill_(SENTINEL)
    view = big.t[:nb, :rows, :cols] if nb > 1 else big.t[:rows, :cols]
    inside = np.zeros(pad, dtype=bool)
    if nb > 1:
      inside[:nb, :rows, :cols] = True
    else:
      inside[:rows, :cols] = True
    bigs.append((big, inside))
    return type(big)(view, code)

  steps = _zipper_steps(be, _zipper_inputs(be, np.random.default_rng(43), dtype, nb, ZIP_BONDS), nb, out)
  outs = _launch_twice(be, steps)
  sentinel = _bits(torch.full((1,), SENTINEL, dtype=bigs[0][0].t.dtype))[0]
  for k, (big, inside) in enumerate(bigs):
    pad_bits = _bits(big.t)[~inside]
    assert (pad_bits == sentinel).all(), "padded output %d: %d pad elements overwritten" % (k, (pad_bits != sentinel).sum())
  _check_steps(be, steps, dtype, outs)


@pytest.mark.parametrize("nb,G", BATCH_G)
@pytest.mark.parametrize("dtype", DTYPES)
def test_chain_aliased_ring(dtype, nb, G, monkeypatch):
  """Step s + 2 writes the buffer step s wrote (same shape), which only step s + 1 reads: the ring aliasing of
  CompiledNetwork at its tightest.  The write is safe only if the kernel orders it after that read; every output that
  survives must equal the same chain launched with distinct buffers, bit for bit."""
  _env(monkeypatch, G)
  be = get_backend()
  inputs = _zipper_inputs(be, np.random.default_rng(44), dtype, nb, RING_BONDS)
  distinct = _zipper_steps(be, inputs, nb)
  ref = _launch_twice(be, distinct)
  _check_steps(be, distinct, dtype, ref)
  last, ring = len(distinct) - 1, {}

  def out(i, shape, code):
    buf, j = ring.get(shape, (None, None))
    if i == last or j != i - 2:
      buf = be._new(shape, code)  # pylint: disable=protected-access
    ring[shape] = (buf, i)
    return buf

  aliased = _zipper_steps(be, inputs, nb, out)
  ptrs = [s.c.t.data_ptr() for s in aliased]
  assert len(set(ptrs)) < len(ptrs), "no buffer is shared"
  outs = _launch_twice(be, aliased)
  for i, p in enumerate(ptrs):
    if p not in ptrs[i + 1:]:                       # not overwritten by a later step
      np.testing.assert_array_equal(_bits(outs[i]), _bits(ref[i]), err_msg="step %d" % i)


# ------------------------------------------------------------------------------------------------ rejections
def _reject_case(be, case):
  """three dependent 256 x 256 bf16 steps, one of them made unacceptable"""
  L = _L()
  rng = np.random.default_rng(45)
  a0, b0, b1, b2 = (_dev(be, rng, (256, 256), "bfloat16") for _ in range(4))
  c0, c1, c2 = (be._new((256, 256), L.BF16) for _ in range(3))  # pylint: disable=protected-access
  a2, dep2 = c1, (1, -1)
  dep1 = (0, -1)
  if case == "c_transposed":
    c2 = be.transpose(be._new((256, 256), L.BF16))  # pylint: disable=protected-access
  elif case == "c_misaligned":
    flat = be._new((256 * 256 + 8,), L.BF16)  # pylint: disable=protected-access
    c2 = type(flat)(flat.t[1:1 + 256 * 256].view(256, 256), L.BF16)
  elif case == "dtype_mismatch":
    a2, b2, dep2 = _dev(be, rng, (256, 256), "float16"), _dev(be, rng, (256, 256), "float16"), (-1, -1)
    c2 = be._new((256, 256), L.F16)  # pylint: disable=protected-access
  elif case == "dep_b_not_operand":
    dep2 = (1, 0)
  elif case == "dep_on_later_step":
    dep1 = (2, -1)
  steps = [_Step("mk,kn->mn", a0, b0, c0), _Step("mk,kn->mn", c0, b1, c1, *dep1), _Step("mk,kn->mn", a2, b2, c2, *dep2)]
  if case == "batch_mismatch":
    a, b = (_dev(be, rng, (3, 256, 256), "bfloat16") for _ in range(2))
    steps[2] = _Step("bmk,bkn->bmn", a, b, be._new((3, 256, 256), L.BF16))  # pylint: disable=protected-access
  return steps


REJECTIONS = {
    "dep_b_not_operand": ("ERR_INVALID", -1),
    "dep_on_later_step": ("ERR_INVALID", -1),
    "c_transposed": ("ERR_UNSUPPORTED", 2),        # c_sn != 1
    "c_misaligned": ("ERR_UNSUPPORTED", 2),        # C not 16-byte aligned: no TMA store map
    "dtype_mismatch": ("ERR_UNSUPPORTED", 2),
    "batch_mismatch": ("ERR_UNSUPPORTED", 2),
}


@pytest.mark.parametrize("case", sorted(REJECTIONS))
def test_chain_create_rejects_and_names_the_step(case):
  """an invalid chain is refused; a step the kernel cannot take is named, so that the caller splits the run there"""
  L = _L()
  be = get_backend()
  rc, bad, handle = _create(be, _reject_case(be, case))
  if handle.value:
    be.lib.tnb200_chain_destroy(handle)
  err, idx = REJECTIONS[case]
  assert (rc, bad, handle.value) == (getattr(L, err), idx, None)


# ------------------------------------------------------------------------------------------------ network level
def _zipper_path(L):
  """contract left to right: E = ket_0 bra_0, then T = E ket_i, E = T bra_i (opt_einsum path convention)"""
  ids, path = list(range(2 * L)), []
  def take(x, y, new):
    i, j = ids.index(x), ids.index(y)
    path.append((i, j))
    for k in sorted((i, j), reverse=True):
      del ids[k]
    ids.append(new)
  take(0, L, "E")
  for i in range(1, L):
    take("E", i, "T")
    take("T", L + i, "E")
  return path


@pytest.mark.parametrize("ring", ["0", "2"])
@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
def test_compiled_network_ragged_bonds_open_ends(dtype, ring, monkeypatch):
  """A norm-like network whose bonds ramp up through 2 .. 64 and continue at 136, 200, 264, 200, 136, with both end
  legs open (a 136 x 136 result per sample).  The ramp steps are below the chained kernel's tile, so the driver splits
  the run at them and chains the rest; the result must equal the step-by-step network bit for bit."""
  from oracle import np_network as nn  # pylint: disable=import-outside-toplevel
  from tensornetwork_b200 import drivers  # pylint: disable=import-outside-toplevel
  monkeypatch.setenv("TNB200_CHAIN_FORCE", "1")
  monkeypatch.setenv("TNB200_CHAIN_RING", ring)
  monkeypatch.delenv("TNB200_CHAIN_G", raising=False)
  be = get_backend()
  rng = np.random.default_rng(46)
  dims = [1, 2, 4, 8, 16, 32, 64, 136, 200, 264, 200, 136]
  L, NB = len(dims) - 1, 3
  labels = []
  for side in "kb":
    for i in range(L):
      labels.append(["e0" if i == 0 else "%s%d" % (side, i), "p%d" % i, side + "R" if i == L - 1 else "%s%d" % (side, i + 1)])
  core = [(dims[i], 2, dims[i + 1]) for i in range(L)] * 2
  shapes = [(NB,) + s for s in core]
  path, out_labels = _zipper_path(L), ["kR", "bR"]
  dev = [_dev(be, rng, shapes[i], dtype, (2 * dims[i]) ** -0.5) for i in range(L)]
  al = {L + i: i for i in range(L)}
  net_c = drivers.CompiledNetwork(be, shapes, dtype, labels, out_labels, path=path, nbatch=1, conj_aliases=al, use_chains=True)
  net_s = drivers.CompiledNetwork(be, shapes, dtype, labels, out_labels, path=path, nbatch=1, conj_aliases=al, use_chains=False)
  assert net_c.chains and max(len(c.steps) for c in net_c.chains) >= 4, "no chain was formed"
  net_c.load(dev + [None] * L)
  net_s.load(dev + [None] * L)
  out = net_c().to_host().astype(np.float64)
  assert out.shape == (NB, 136, 136) and np.isfinite(out).all()
  np.testing.assert_array_equal(out, net_s().to_host().astype(np.float64))
  for b in range(NB):
    ts = [_host64(d)[b] for d in dev]
    exact = nn.contract_path(ts + ts, labels, path, out_labels)
    assert rel_err(out[b], exact) < 3e-2, (b, rel_err(out[b], exact))
