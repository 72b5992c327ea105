"""gloo worker (CPU, world_size 2 or 4): `parallel.ShardedNetwork.run` — the executor behind bench.py's strong_scaling
record — on a scaled-down copy of the benchmark's 32-tensor tree network.

The device layer is tests/fake_lib.FakeLib (host memory), torch.distributed runs on gloo, and `drivers.CompiledNetwork`
(CUDA graphs) is replaced by a stub that contracts its subtree pair by pair through the same backend.  What is checked:
  * the result on the root rank equals the numpy oracle (two runs: persistent receive buffers are reused);
  * the point-to-point operations `run` hands to the process group, in order, are exactly `parallel.p2p_issue_order` — the
    model `parallel.schedule_completes` simulates to refuse plans that would deadlock with serialised NCCL p2p;
  * every rank computes something and something crosses ranks;
  * (SHARDED_EXPECT_REFUSAL=1) a plan the model rejects is refused on every rank before anything is posted.
"""
import os
import numpy as np
import torch.distributed as dist
import hostrun
hostrun.install()
from tensornetwork_b200 import backend as tb_backend, drivers, parallel  # noqa: E402
from oracle import np_network as nn  # noqa: E402
import bench  # noqa: E402


class EagerNet:
  """stand-in for drivers.CompiledNetwork (same constructor / load / call surface as ShardedNetwork uses)"""

  def __init__(self, backend, shapes, dtype, labels, out_labels, path=None, **_):
    self.be, self.labels, self.out, self.path = backend, [list(l) for l in labels], list(out_labels), list(path)
    self.t = None

  def load(self, tensors):
    self.t = list(tensors)

  def __call__(self):
    ts, ls = list(self.t), [list(l) for l in self.labels]
    for i, j in self.path:
      a, b, la, lb = ts[i], ts[j], ls[i], ls[j]
      shared = [l for l in la if l in lb]
      o = self.be.tensordot(a, b, ([la.index(l) for l in shared], [lb.index(l) for l in shared]))
      lo = [l for l in la if l not in shared] + [l for l in lb if l not in shared]
      for k in sorted((i, j), reverse=True):
        del ts[k]
        del ls[k]
      ts.append(o)
      ls.append(lo)
    assert len(ts) == 1
    if ls[0] != self.out:
      return self.be.transpose(ts[0], [ls[0].index(l) for l in self.out])
    return ts[0]


def main():
  dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % os.environ["MASTER_PORT"],
                          rank=int(os.environ["RANK"]), world_size=int(os.environ["WORLD_SIZE"]))
  rank, world = dist.get_rank(), dist.get_world_size()
  drivers.CompiledNetwork = EagerNet
  be = tb_backend.CudaB200Backend()
  if os.environ.get("SHARDED_EXPECT_REFUSAL"):
    # the benchmark network at full size on a rank count whose plan would make serialised NCCL p2p wait in a cycle (3 ranks):
    # refused from the shapes alone, identically on every rank, before any buffer or operation exists
    labels, sizes, shapes, _ = bench.ttn_network(None)
    path = drivers.greedy_path(labels, [], sizes)
    try:
      parallel.ShardedNetwork(be, shapes, np.float64, labels, path, rank, world, join_graphs=False)
    except NotImplementedError as exc:
      assert "wait on each other" in str(exc)
    else:
      raise AssertionError("plan accepted")
    dist.barrier()
    if rank == 0:
      print("SHARDED REFUSED world=%d" % world)
    dist.destroy_process_group()
    return
  labels, sizes, shapes, _ = bench.ttn_network({"b3": 24, "b2": 8, "b1": 4, "p": 3})
  path = drivers.greedy_path(labels, [], sizes)
  rng = np.random.default_rng(5)          # same inputs on every rank
  n_ket = len(labels) // 2
  kets = [rng.standard_normal(shapes[i]) / np.sqrt(np.prod(shapes[i][1:])) for i in range(n_ket)]
  host = kets + [np.conj(k) for k in kets]
  want = float(nn.contract_path(host, labels, path, []))
  dev = [be.convert_to_tensor(h) for h in host]

  issued = []
  real_isend, real_irecv = dist.isend, dist.irecv

  def isend(tensor, dst, group=None):
    issued.append(("send", dst, tuple(tensor.shape)))
    return real_isend(tensor, dst, group=group)

  def irecv(tensor, src, group=None):
    issued.append(("recv", src, tuple(tensor.shape)))
    return real_irecv(tensor, src, group=group)
  dist.isend, dist.irecv = isend, irecv

  sh = parallel.ShardedNetwork(be, shapes, np.float64, labels, path, rank, world, join_graphs=False)
  sh.load(dev)
  assert set(sh.owner) == set(range(world)), sh.owner
  assert len(sh.transfers) >= world - 1
  model = parallel.p2p_issue_order(len(labels), sh.ssa, sh.owner, sh.transfers, rank)
  shape_of = lambda t: tuple(sizes[l] for l in sh.lab[t])
  for run in range(2):
    del issued[:]
    out, root_rank = sh.run()
    assert [(k, peer, shape_of(t)) for k, t, peer in model] == issued, (rank, model, issued)
    if rank == root_rank:
      got = float(out.to_host().reshape(-1)[0])
      assert abs(got - want) <= 1e-12 * abs(want), (run, got, want)
    else:
      assert out is None
  assert sh.p2p_bytes == sum(8 * int(np.prod(s)) for _, _, s in issued)
  dist.barrier()
  if rank == 0:
    print("SHARDED OK world=%d transfers=%d per_rank=%s" % (world, len(sh.transfers), ["%.3g" % x for x in sh.info["per_rank"]]))
  dist.destroy_process_group()


if __name__ == "__main__":
  main()
