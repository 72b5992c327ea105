"""Chain groups (drivers.find_chain_groups): what CompiledNetwork offers to tnb200_chain_create, host only."""
from tensornetwork_b200 import drivers


def _norm_plan(Ls=64, D=512, nb=74):
  dims = [1] + [min(D, 2 ** min(i, Ls - i)) for i in range(1, Ls)] + [1]
  labels = []
  for side in "kb":
    for i in range(Ls):
      labels.append(["e0" if i == 0 else "%s%d" % (side, i), "p%d" % i, "eL" if i == Ls - 1 else "%s%d" % (side, i + 1)])
  core = [(dims[i], 2, dims[i + 1]) for i in range(Ls)] * 2
  shapes = [(nb,) + c for c in core]
  sizes = {l: s[ax] for s, labs in zip(core, labels) for ax, l in enumerate(labs)}
  path = drivers.greedy_path(labels, [], sizes)
  steps, res = drivers.plan_path(shapes, labels, path, [], 1)
  return steps, res, drivers.plan_shapes(shapes, steps), len(shapes)


def _deps(steps, n, group):
  """per member: the positions inside the group of the members that produce its operands"""
  pos = {sid: k for k, sid in enumerate(group)}
  return [sorted(pos[p - n] for p in (steps[sid][1], steps[sid][2]) if p - n in pos) for sid in group]


def test_bench_plan_groups_the_four_ramp_heads():
  steps, res, shp, n = _norm_plan()
  groups = drivers.find_chain_groups(steps, n, res, shp)
  assert groups == [list(range(12)), list(range(34, 127))]
  assert drivers.find_chains(steps, n) == [list(range(34, 127))]
  # ket / bra x left / right: steps 0-3 start the four ramps, step s + 4 consumes step s
  assert _deps(steps, n, groups[0]) == [[]] * 4 + [[k] for k in range(8)]
  assert _deps(steps, n, groups[1])[1:] == [[k] for k in range(92)]


def _gemm_plan(ops, n_in=8, nb=3, d=256):
  """batched (nb, d, d) x (nb, d, d) products: ops are (a, b) slot pairs"""
  shapes = [(nb, d, d)] * n_in
  steps = [("batched", a, b, (2,), (1,), (0,), (0,), n_in + i) for i, (a, b) in enumerate(ops)]
  return steps, drivers.plan_shapes(shapes, steps)


def test_operand_produced_between_members_forms_no_group():
  n = 8
  # step 3 continues step 0, and its other operand is an input: steps 0 and 3 form a group
  steps, shp = _gemm_plan([(0, 1), (2, 3), (4, 5), (n + 0, 6)])
  assert drivers.find_chain_groups(steps, n, n + 3, shp) == [[0, 3]]
  # the same operand produced by step 1, between the members: launched at step 0, the group would read it too early
  steps, shp = _gemm_plan([(0, 1), (2, 3), (4, 5), (n + 0, n + 1)])
  assert drivers.find_chain_groups(steps, n, n + 3, shp) == []


def test_only_independent_runs_merge():
  n = 8
  # runs 0 -> 3 and 1 -> 4 do not depend on each other: one group
  steps, shp = _gemm_plan([(0, 1), (2, 3), (4, 5), (n + 0, 6), (n + 1, 7)])
  assert drivers.find_chain_groups(steps, n, n + 4, shp) == [[0, 1, 3, 4]]
  # run 1 -> 6 also reads step 4, the end of run 0 -> 2 -> 4: the two are not merged, and run 1 -> 6 alone would be
  # launched before step 4
  steps, shp = _gemm_plan([(0, 1), (2, 3), (n + 0, 4), (5, 6), (n + 2, 7), (5, 6), (n + 1, n + 4)])
  assert drivers.find_chain_groups(steps, n, n + 6, shp) == [[0, 2, 4]]
