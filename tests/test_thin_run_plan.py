"""Thin-run detection (drivers.find_thin_runs) on the plan of the L=64, D=512 MPS norm network: host only."""
import numpy as np

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


def test_bench_plan_has_four_ramp_runs():
  steps, res, shp, n = _norm_plan()
  chained = {s for run in drivers.find_chains(steps, n) for s in run}
  runs = drivers.find_thin_runs(steps, n, res, shp, exclude=chained)
  assert sorted(runs) == [[12, 16, 20, 24, 28], [13, 17, 21, 25, 29], [14, 18, 22, 26, 30], [15, 19, 23, 27, 31]]
  # without the chain, the left ket run also absorbs the K = 2 join that consumes it
  assert [12, 16, 20, 24, 28, 34] in drivers.find_thin_runs(steps, n, res, shp)


def test_second_consumer_ends_a_run():
  steps, res, shp, n = _norm_plan()
  # give step 20's result a second consumer: the run from step 12 must stop at step 20
  steps = list(steps) + [("batched", n + 20, n + 20, (1,), (1,), (0,), (0,), n + len(steps))]
  shp = drivers.plan_shapes([s for s in shp[:n]], steps)
  runs = drivers.find_thin_runs(steps, n, res, shp, exclude={34})
  assert [12, 16, 20] in runs and not any(24 in r and 20 in r for r in runs)
  assert not any(len(r) < 2 or len(r) > 8 for r in runs)
  assert np.all([len(set(r)) == len(r) for r in runs])
