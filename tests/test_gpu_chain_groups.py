"""A chained launch of independent branches: the heads of the four MPS ramps (ket / bra x left / right) of the
L=64, D=512 norm network, three steps each, run as ONE tnb200_chain launch whose steps interleave in plan order, and
CompiledNetwork's use of it.

Each output is a view of a sentinel-filled buffer one sample longer and is filled with NaN before each launch; every
step must match its single-GEMM launch (be._contract) bit for bit and float64 within the a-priori bound of
test_gpu_chain.py, and a second launch must reproduce the first."""
import numpy as np
import pytest
from util import get_backend
import test_gpu_chain as tc

pytestmark = pytest.mark.gpu

# (samples, TNB200_CHAIN_G): odd batches, rounds of one and of two samples
BATCH_G = [(3, 1), (5, 2)]


def _head_steps(be, rng, dtype, nb):
  """bonds 512 -> 256 -> 128 -> 64 from the middle of each ramp outwards, as greedy orders them: the left ramps contract
  the next site's right bond (the result is operand b), the right ramps the result's last bond (operand a)"""
  from tensornetwork_b200 import tensor as T  # pylint: disable=import-outside-toplevel
  code = T.dtype_code(dtype)
  pads = []

  def out(shape):
    big = be._new((nb + 1,) + shape, code)  # pylint: disable=protected-access
    big.t.fill_(tc.SENTINEL)
    pads.append(big)
    return type(big)(big.t[:nb], code)

  site = lambda *s: tc._dev(be, rng, (nb,) + s, dtype, (s[0] * 2) ** -0.5)  # pylint: disable=protected-access,unnecessary-lambda-assignment
  branches = []
  for right in (False, True, False, True):
    if not right:
      c0 = out((256, 2, 2, 512))
      c1 = out((128, 2, 2, 2, 512))
      c2 = out((64, 2, 2, 2, 2, 512))
      branches.append([("bxpm,bmqn->bxpqn", site(256, 2, 512), site(512, 2, 512), c0),
                       ("bypx,bxqrn->bypqrn", site(128, 2, 256), c0, c1),
                       ("bzpy,byqrsn->bzpqrsn", site(64, 2, 128), c1, c2)])
    else:
      c0 = out((512, 2, 2, 256))
      c1 = out((512, 2, 2, 2, 128))
      c2 = out((512, 2, 2, 2, 2, 64))
      branches.append([("bmpx,bxqn->bmpqn", site(512, 2, 512), site(512, 2, 256), c0),
                       ("bmpqx,bxry->bmpqry", c0, site(256, 2, 128), c1),
                       ("bmpqry,bysz->bmpqrsz", c1, site(128, 2, 64), c2)])
  steps = []
  for depth in range(3):
    for k, br in enumerate(branches):
      spec, a, b, c = br[depth]
      dep = len(steps) - 4 if depth else -1
      right = k % 2 == 1
      steps.append(tc._Step(spec, a, b, c, dep_a=dep if right else -1, dep_b=-1 if right else dep))  # pylint: disable=protected-access
  return steps, pads


def _check(be, steps, dtype, outs):
  """per sample, float64 tensordot of the operands the step read, and bit identity with one single-GEMM launch"""
  for i, (s, c) in enumerate(zip(steps, outs)):
    a, b = tc._host64(s.a), tc._host64(s.b)  # pylint: disable=protected-access
    got = c.float().cpu().numpy().astype(np.float64)
    axes = ([x - 1 for x in s.ax_a], [x - 1 for x in s.ax_b])
    worst = 0.0
    for j in range(a.shape[0]):
      r = np.tensordot(a[j], b[j], axes)
      sabs = np.tensordot(np.abs(a[j]), np.abs(b[j]), axes)
      bound = tc.U_OUT[dtype] * np.abs(r) + (tc.U_IN[dtype] + s.K * 2.0**-23) * sabs
      worst = max(worst, float((np.abs(got[j] - r) / bound).max()))
    single = be._contract(s.a, s.b, s.ax_a, s.ax_b, s.ba, s.bb)  # pylint: disable=protected-access
    differ = int((tc._bits(single.t) != tc._bits(c)).sum())  # pylint: disable=protected-access
    assert worst <= 1.0 and differ == 0, "step %d (%s): error/bound %.3g; %d elements differ from the single launch" % (
        i, s.spec, worst, differ)


@pytest.mark.parametrize("nb,G", BATCH_G)
@pytest.mark.parametrize("dtype", tc.DTYPES)
def test_chain_of_four_independent_branches(dtype, nb, G, monkeypatch):
  tc._env(monkeypatch, G)  # pylint: disable=protected-access
  be = get_backend()
  steps, pads = _head_steps(be, np.random.default_rng(47), dtype, nb)
  outs = tc._launch_twice(be, steps)  # pylint: disable=protected-access
  sentinel = tc._bits(tc._torch().full((1,), tc.SENTINEL, dtype=pads[0].t.dtype))[0]  # pylint: disable=protected-access
  for k, big in enumerate(pads):
    tail = tc._bits(big.t[nb])  # pylint: disable=protected-access
    assert (tail == sentinel).all(), "output %d: %d elements of the pad sample overwritten" % (k, (tail != sentinel).sum())
  _check(be, steps, dtype, outs)


def _norm_network(L=64, D=512):
  dims = [1] + [min(D, 2 ** min(i, L - i)) for i in range(1, L)] + [1]
  labels = []
  for side in "kb":
    for i in range(L):
      labels.append(["e0" if i == 0 else "%s%d" % (side, i), "p%d" % i, "eL" if i == L - 1 else "%s%d" % (side, i + 1)])
  core = [(dims[i], 2, dims[i + 1]) for i in range(L)] * 2
  return dims, labels, core


def test_compiled_cfg2_runs_the_ramp_heads_as_one_chain(monkeypatch):
  """cfg2 at 20 samples, enough pairs per step for both chains: the ramp heads (steps 0-11) and the zipper are one
  launch each beside the four thin runs, 11 launches per replay; the result equals the step-by-step graph bit for bit,
  and no two head steps share a result buffer.  One unbatched network falls back to per-step launches."""
  from tensornetwork_b200 import drivers  # pylint: disable=import-outside-toplevel
  for var in ("TNB200_CHAIN_FORCE", "TNB200_CHAIN_G", "TNB200_CHAIN_RING"):
    monkeypatch.delenv(var, raising=False)
  be = get_backend()
  L, NB = 64, 20
  dims, labels, core = _norm_network(L)
  sizes = {l: s[ax] for s, labs in zip(core, labels) for ax, l in enumerate(labs)}
  path = drivers.greedy_path(labels, [], sizes)
  rng = np.random.default_rng(7)
  al = {L + i: i for i in range(L)}
  kets = [be.astype(be.convert_to_tensor((rng.standard_normal((NB,) + core[i]) / np.sqrt(core[i][0] * 2)).astype(np.float32)),
                    "bfloat16") for i in range(L)]
  shapes = [(NB,) + s for s in core]
  net_c = drivers.CompiledNetwork(be, shapes, "bfloat16", labels, [], path=path, nbatch=1, conj_aliases=al)
  chains = [c.steps for c in net_c.chains if c.api == "chain"]
  assert chains == [list(range(12)), list(range(35, 125))], chains
  assert len([c for c in net_c.chains if c.api == "thin_run"]) == 4
  assert net_c.launches_per_replay == 11
  n_in = len(shapes)
  ptrs = [net_c._vals[n_in + s].t.data_ptr() for s in range(12)]  # pylint: disable=protected-access
  assert len(set(ptrs)) == 12
  net_s = drivers.CompiledNetwork(be, shapes, "bfloat16", labels, [], path=path, nbatch=1, conj_aliases=al, use_chains=False)
  net_c.load(kets + [None] * L)
  net_s.load(kets + [None] * L)
  ref = net_s().to_host()
  for _ in range(2):
    np.testing.assert_array_equal(net_c().to_host(), ref)
  del net_c, net_s
  one = [type(k)(k.t[0], k.code) for k in kets]
  net1 = drivers.CompiledNetwork(be, core, "bfloat16", labels, [], path=path, nbatch=0, conj_aliases=al)
  net1s = drivers.CompiledNetwork(be, core, "bfloat16", labels, [], path=path, nbatch=0, conj_aliases=al, use_chains=False)
  assert not [c for c in net1.chains if c.api == "chain"]
  net1.load(one + [None] * L)
  net1s.load(one + [None] * L)
  np.testing.assert_array_equal(net1().to_host(), net1s().to_host())
