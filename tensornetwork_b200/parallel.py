"""Multi-GPU execution of the contraction path (SURVEY.md 8e): one process per GPU,
`torch.distributed` (NCCL over NVLink 5 / NVSwitch) as the plumbing.

The reference has no parallelism of any kind; what shards naturally is
  (i)  independent networks / MPS batch samples  -> `shard_range`, `contract_independent`:
       every rank contracts its own units, no data-path collective, one final all-gather of the
       (tiny) results;
  (ii) one network whose contraction *tree* fans out -> `partition_tree`, `contract_tree_parallel`:
       the pairwise path (contractors/opt_einsum_paths/path_contractors.py:87-90 executes it as a
       sequential list) is a binary tree; disjoint subtrees are independent.  The tree is cut into
       subtrees weighted by 2MNK, packed onto ranks longest-processing-time first, and each subtree
       result that is consumed on another rank is moved once, point-to-point (`dist.send/recv`, i.e.
       NCCL p2p over NVLink), at the join.  Steps above the cut run on the rank that already holds
       the larger operand.
A single pairwise contraction is never split across GPUs (1 GFLOP problems do not amortise a
collective), and the DMRG sweep is serial in the site index (dmrg.py:524-547): "replicas only".
"""
import numpy as np


def shard_range(n_units, rank, world):
  """contiguous, balanced shard of `n_units` independent units for `rank`."""
  base, rem = divmod(n_units, world)
  start = rank * base + min(rank, rem)
  return range(start, start + base + (1 if rank < rem else 0))


def contract_independent(units, contract_fn, rank, world, gather=None):
  """Each rank runs `contract_fn(unit)` on its shard; `gather(list_of_local_results)` (e.g.
  dist.all_gather_object) returns the per-rank lists.  Results come back in unit order."""
  mine = [contract_fn(units[i]) for i in shard_range(len(units), rank, world)]
  if gather is None or world == 1:
    return mine
  parts = gather(mine)
  return [r for part in parts for r in part]


# ----------------------------------------------------------------------- contraction tree
def path_to_ssa(n_inputs, path):
  """opt_einsum 'linear' path -> SSA triples (id_a, id_b, id_out)."""
  ids = list(range(n_inputs))
  nxt = n_inputs
  out = []
  for a, b in path:
    ia, ib = ids[a], ids[b]
    for i in sorted([a, b], reverse=True):
      del ids[i]
    ids.append(nxt)
    out.append((ia, ib, nxt))
    nxt += 1
  return out


def partition_tree(n_inputs, path, step_flops, world, oversub=4, slack=0.03):
  """Assign every pairwise step of `path` to a rank.

  Returns (owner, transfers, info): owner[s] = rank executing SSA step s (in path order);
  transfers = list of (tensor_id, src_rank, dst_rank, before_step) point-to-point moves;
  info = dict(total, per_rank, critical) flop accounting (speed-up bound = total / critical)."""
  ssa = path_to_ssa(n_inputs, path)
  producer = {o: i for i, (_, _, o) in enumerate(ssa)}       # tensor id -> step index
  cost = {}                                                  # subtree flops per tensor id

  def subtree_cost(t):
    if t < n_inputs:
      return 0.0
    if t not in cost:
      a, b, _ = ssa[producer[t]]
      cost[t] = step_flops[producer[t]] + subtree_cost(a) + subtree_cost(b)
    return cost[t]
  root = ssa[-1][2] if ssa else 0
  total = subtree_cost(root)
  # Grow a frontier of independent subtrees by repeatedly splitting the most expensive one — but only as far as balance
  # needs it: the coarsest frontier whose longest-processing-time-first packing is within `slack` of total / world keeps
  # subtrees that are contracted with each other (a ket half and its bra half) on ONE rank, so what crosses NVLink at the
  # joins are the small results above them rather than the large halves.  Fall back to world * oversub subtrees.
  def lpt(front):
    load = [0.0] * world
    where = {}
    for t in sorted(front, key=subtree_cost, reverse=True):
      r = int(np.argmin(load))
      load[r] += subtree_cost(t)
      where[t] = r
    return load, where
  frontier = [root]
  target = max(1, world * oversub)
  def splittable(t):
    a, b, _ = ssa[producer[t]]
    return a >= n_inputs or b >= n_inputs       # a step on two inputs is a leaf of the cut
  ideal = total / world if world else total
  while True:
    load, tensor_rank = lpt(frontier)
    if len(frontier) >= world and max(load) <= (1.0 + slack) * ideal:
      break
    if len(frontier) >= target:
      break
    cand = [t for t in frontier if t >= n_inputs and splittable(t)]
    if not cand:
      break
    t = max(cand, key=subtree_cost)
    if subtree_cost(t) < total / (8.0 * target):
      break
    a, b, _ = ssa[producer[t]]
    frontier.remove(t)
    frontier.extend([x for x in (a, b) if x >= n_inputs])   # inputs live on every rank
  load, tensor_rank = lpt(frontier)

  owner = [None] * len(ssa)

  def assign_subtree(t, r):
    if t < n_inputs:
      return
    s = producer[t]
    owner[s] = r
    a, b, _ = ssa[s]
    assign_subtree(a, r)
    assign_subtree(b, r)
  for t, r in tensor_rank.items():
    assign_subtree(t, r)
  # steps above the cut: run where the larger-cost operand already lives
  transfers = []
  where = dict(tensor_rank)

  def locate(t):
    if t in where:
      return where[t]
    if t < n_inputs:
      return None                                            # inputs are available on every rank
    s = producer[t]
    if owner[s] is not None:
      where[t] = owner[s]
      return owner[s]
    a, b, _ = ssa[s]
    ra, rb = locate(a), locate(b)
    if ra is None and rb is None:
      r = int(np.argmin(load))
    elif ra is None:
      r = rb
    elif rb is None:
      r = ra
    else:
      r = ra if subtree_cost(a) >= subtree_cost(b) else rb
    owner[s] = r
    load[r] += step_flops[s]
    for x, rx in ((a, ra), (b, rb)):
      if rx is not None and rx != r:
        transfers.append((x, rx, r, s))
    where[t] = r
    return r
  locate(root)
  for s in range(len(ssa)):
    if owner[s] is None:
      owner[s] = 0
  # critical path (flops) through the tree = lower bound on any schedule
  crit = {}

  def critical(t):
    if t < n_inputs:
      return 0.0
    if t not in crit:
      a, b, _ = ssa[producer[t]]
      crit[t] = step_flops[producer[t]] + max(critical(a), critical(b))
    return crit[t]
  info = dict(total=total, per_rank=load, critical=critical(root), root_rank=where.get(root, 0))
  return owner, sorted(transfers, key=lambda x: x[3]), info


def contract_tree_parallel(tensors, labels, out_labels, path, rank, world, contract_pair, send, recv,
                           step_flops=None, irecv=None, plan=None):
  """Execute `path` with the steps spread over `world` ranks.

  contract_pair(t1, labels1, t2, labels2) -> (tensor, labels)   (contract_between semantics)
  send(tensor, dst)                                              (point-to-point, may be asynchronous)
  recv(tensor_id, src) -> tensor                                 (blocking receive), or
  irecv(tensor_id, src) -> callable returning the tensor         (receive POSTED up front, waited on at the join)
  A subtree result consumed on another rank is sent the moment it exists (right after the step that produces it), not
  at the join; with `irecv` every rank posts all its receives before its first contraction, per source in the order
  the source produces them (point-to-point messages between two ranks match in order).
  Every rank holds all inputs.  Returns (result or None, root_rank, info)."""
  n = len(tensors)
  ssa = path_to_ssa(n, path)
  if step_flops is None:
    step_flops = [1.0] * len(ssa)
  owner, transfers, info = plan if plan is not None else partition_tree(n, path, step_flops, world)
  producer = {o: i for i, (_, _, o) in enumerate(ssa)}
  vals = {i: (tensors[i], list(labels[i])) for i in range(n)}
  outgoing = {}
  incoming = []
  for t, src, dst, _before in transfers:
    if rank == src:
      outgoing.setdefault(t, []).append(dst)
    if rank == dst:
      incoming.append((producer.get(t, -1), t, src))
  # labels of every intermediate are needed on the receiving side: replay them symbolically
  lab = {i: list(labels[i]) for i in range(n)}
  for a, b, o in ssa:
    shared = [l for l in lab[a] if l in lab[b]]
    lab[o] = [l for l in lab[a] if l not in shared] + [l for l in lab[b] if l not in shared]
  handles = {}
  incoming.sort()
  if irecv is not None:
    for _, t, src in incoming:
      handles[t] = irecv(t, src)
  arriving = {t: src for _, t, src in incoming}
  for s, (a, b, o) in enumerate(ssa):
    if owner[s] != rank:
      continue
    for x in (a, b):
      if x not in vals and x in arriving:
        vals[x] = ((handles.pop(x)() if x in handles else recv(x, arriving[x])), lab[x])
    ta, la = vals[a]
    tb, lb = vals[b]
    vals[o] = contract_pair(ta, la, tb, lb)
    for dst in outgoing.get(o, ()):
      send(vals[o][0], dst)
    # free operands that are intermediates
    for x in (a, b):
      if x >= n:
        vals.pop(x, None)
  root = ssa[-1][2] if ssa else 0
  root_rank = owner[-1] if ssa else 0
  res = vals.get(root, (None, None))[0] if rank == root_rank else None
  info = dict(info)
  info["transfers"] = [(t, src, dst) for t, src, dst, _ in transfers]
  return res, root_rank, info


# ------------------------------------------------------------------------ NCCL execution
def contract_network_parallel(backend, tensors, labels, out_labels=(), path=None, step_flops=None, group=None, plan=None):
  """`contract_tree_parallel` on the CUDA backend with torch.distributed (NCCL over NVLink) as transport.
  Every rank passes the same inputs (B200Tensors or host arrays); returns (result B200Tensor on the root
  rank / None elsewhere, root_rank, info)."""
  import torch.distributed as dist  # pylint: disable=import-outside-toplevel
  from . import drivers  # pylint: disable=import-outside-toplevel
  from .tensor import B200Tensor  # pylint: disable=import-outside-toplevel
  rank, world = dist.get_rank(group), dist.get_world_size(group)
  ts = [backend.convert_to_tensor(t) for t in tensors]
  sizes = {l: t.shape[ax] for t, labs in zip(ts, labels) for ax, l in enumerate(labs)}
  if path is None:
    path = drivers.greedy_path(labels, out_labels, sizes)
  n = len(ts)
  ssa = path_to_ssa(n, path)
  lab = {i: list(l) for i, l in enumerate(labels)}
  flops = []
  for a, b, o in ssa:
    shared = [l for l in lab[a] if l in lab[b]]
    lab[o] = [l for l in lab[a] if l not in shared] + [l for l in lab[b] if l not in shared]
    k = float(np.prod([sizes[l] for l in shared])) if shared else 1.0
    flops.append(2.0 * k * float(np.prod([sizes[l] for l in lab[o]] or [1.0])))
  if step_flops is None:
    step_flops = flops
  code = ts[0].code

  def pair(t1, l1, t2, l2):
    shared = [l for l in l1 if l in l2]
    a1 = [l1.index(l) for l in shared]
    a2 = [l2.index(l) for l in shared]
    srt = sorted(range(len(a1)), key=lambda i: a1[i])
    out = backend.tensordot(t1, t2, ([a1[i] for i in srt], [a2[i] for i in srt]))
    return out, [l for l in l1 if l not in shared] + [l for l in l2 if l not in shared]

  keep = []                                   # isend works / buffers stay alive until the caller synchronises
  moved = [0]

  def send(t, dst):
    buf = backend.contiguous(t)
    moved[0] += buf.t.numel() * buf.t.element_size()
    keep.append((buf, dist.isend(buf.t, dst, group=group)))

  def recv(tid, src):
    buf = backend._new([sizes[l] for l in lab[tid]], code)  # pylint: disable=protected-access
    dist.recv(buf.t, src, group=group)
    return buf

  def irecv(tid, src):
    buf = backend._new([sizes[l] for l in lab[tid]], code)  # pylint: disable=protected-access
    work = dist.irecv(buf.t, src, group=group)
    moved[0] += buf.t.numel() * buf.t.element_size()

    def ready():
      work.wait()                             # the compute stream waits for the transfer; the host does not
      return buf
    return ready
  res, root_rank, info = contract_tree_parallel(ts, labels, out_labels, path, rank, world, pair, send, recv, step_flops,
                                                irecv=irecv, plan=plan)
  for _, w in keep:
    w.wait()
  info["p2p_bytes_this_rank"] = moved[0]
  if res is not None and len(lab[ssa[-1][2]]) > 1 and list(out_labels):
    final = lab[ssa[-1][2]]
    res = backend.transpose(res, tuple(final.index(l) for l in out_labels))
  return res, root_rank, info


# ------------------------------------------------------------------------ graph-replayed shards
def local_subtrees(n_inputs, ssa, owner, rank):
  """The maximal subtrees of the contraction tree that `rank` can contract without hearing from anyone: every step
  is owned by `rank` and every operand is an input or the result of such a step.
  Returns (roots, pure): roots = {root_tensor_id: (leaf_input_ids, steps_in_order)}, pure = set of step indices."""
  pure, of = set(), {}
  for s, (a, b, o) in enumerate(ssa):
    if owner[s] != rank:
      continue
    if all(x < n_inputs or x in of for x in (a, b)):
      pure.add(s)
      of[o] = s
  consumed = {}
  for s, (a, b, o) in enumerate(ssa):
    for x in (a, b):
      consumed[x] = s
  roots = {}
  for o, s in of.items():
    c = consumed.get(o)
    if c is None or c not in pure:                       # consumed above the cut (or the network's result)
      leaves, steps = [], []

      def walk(t):
        if t < n_inputs:
          if t not in leaves:
            leaves.append(t)
          return
        a, b, _ = ssa[of[t]]
        walk(a)
        walk(b)
        steps.append(of[t])
      walk(o)
      roots[o] = (leaves, sorted(steps))
  return roots, pure


def ssa_to_linear(leaves, steps, ssa):
  """SSA steps over the tensor ids `leaves` -> opt_einsum 'linear' path of the sub-network whose inputs are `leaves`."""
  ids = list(leaves)
  path = []
  for s in steps:
    a, b, o = ssa[s]
    i, j = ids.index(a), ids.index(b)
    path.append((i, j))
    for k in sorted((i, j), reverse=True):
      del ids[k]
    ids.append(o)
  return path


class ShardedNetwork:
  """ONE network on `world` GPUs (SURVEY 8e (ii)): the pairwise path (path_contractors.py:87-90 runs it as a sequential
  loop) is a binary tree; `partition_tree` cuts it into subtrees packed onto the ranks.  Each rank holds its local
  subtrees as `CompiledNetwork`s (one CUDA-graph replay each) and runs the few steps above the cut eagerly; a subtree
  result consumed on another rank is sent once, point to point (NCCL isend over NVLink) the moment it exists, into a
  receive the consumer posted once its own subtrees were enqueued.  No collective on the data path."""

  def __init__(self, backend, shapes, dtype, labels, path, rank, world, group=None, join_graphs=True):
    from . import drivers  # pylint: disable=import-outside-toplevel
    from . import tensor as T  # pylint: disable=import-outside-toplevel
    self.backend, self.rank, self.world, self.group = backend, rank, world, group
    n = self.n = len(shapes)
    self.ssa = ssa = path_to_ssa(n, path)
    sizes = {l: s[ax] for s, labs in zip(shapes, labels) for ax, l in enumerate(labs)}
    self.sizes = sizes
    lab = self.lab = {i: list(l) for i, l in enumerate(labels)}
    flops = []
    for a, b, o in ssa:
      shared = [l for l in lab[a] if l in lab[b]]
      lab[o] = [l for l in lab[a] if l not in shared] + [l for l in lab[b] if l not in shared]
      k = float(np.prod([sizes[l] for l in shared])) if shared else 1.0
      flops.append(2.0 * k * float(np.prod([sizes[l] for l in lab[o]] or [1.0])))
    self.step_flops = flops
    # join_graphs: runs of steps above the cut replayed as CUDA graphs
    self.join_graphs = join_graphs
    self.owner, self.transfers, self.info = partition_tree(n, path, flops, world)
    if world > 1 and not schedule_completes(n, ssa, self.owner, self.transfers, world):
      # e.g. 3, 5 or 6 ranks on the benchmark tree: three ranks each start with a large send to the next one.  Every rank
      # reaches the same verdict from the same integers, so all of them raise instead of some of them hanging in NCCL.
      raise NotImplementedError("this partition makes ranks wait on each other when point-to-point operations complete in issue "
                                "order (serialised NCCL p2p); supported on this network: 2, 4, 7, 8 ranks")
    self.producer = {o: i for i, (_, _, o) in enumerate(ssa)}
    self.roots, self.pure = local_subtrees(n, ssa, self.owner, rank)
    self.code = T.dtype_code(dtype)
    self.nets = {}
    for root, (leaves, steps) in self.roots.items():
      sub_path = ssa_to_linear(leaves, steps, ssa)
      self.nets[root] = (leaves, drivers.CompiledNetwork(backend, [tuple(shapes[i]) for i in leaves], dtype,
                                                         [labels[i] for i in leaves], list(lab[root]), path=sub_path))
    self.outgoing, self.incoming = {}, []
    for t, src, dst, _ in self.transfers:
      if rank == src:
        self.outgoing.setdefault(t, []).append(dst)
      if rank == dst:
        self.incoming.append((self.producer.get(t, -1), t, src))
    self.incoming.sort()
    # persistent receive buffers (static addresses: the steps above the cut are replayed as CUDA graphs)
    self._recv = {t: backend._new([sizes[l] for l in lab[t]], self.code) for _, t, _ in self.incoming}  # pylint: disable=protected-access
    # this rank's program above the cut: maximal runs of steps between two receives ("segments")
    arriving = {t for _, t, _ in self.incoming}
    self._segments, cur, have = [], [], set()
    for s_i, (a_, b_, o_) in enumerate(ssa):
      if self.owner[s_i] != rank or s_i in self.pure:
        continue
      need = [x for x in (a_, b_) if x in arriving and x not in have]
      if need and cur:
        self._segments.append(("steps", cur))
        cur = []
      for x in need:
        self._segments.append(("recv", x))
        have.add(x)
      cur.append(s_i)
    if cur:
      self._segments.append(("steps", cur))
    self._seg_graphs = {}
    self._runs = 0
    self.inputs = None
    self.p2p_bytes = 0

  def load(self, tensors):
    """static inputs (every rank holds all of them; only the ones its steps touch are copied into graph arenas)"""
    self.inputs = list(tensors)
    for root, (leaves, net) in self.nets.items():
      net.load([tensors[i] for i in leaves])

  def _pair(self, t1, l1, t2, l2):
    shared = [l for l in l1 if l in l2]
    a1 = [l1.index(l) for l in shared]
    a2 = [l2.index(l) for l in shared]
    srt = sorted(range(len(a1)), key=lambda i: a1[i])
    return self.backend.tensordot(t1, t2, ([a1[i] for i in srt], [a2[i] for i in srt]))

  def run(self):
    """-> (result B200Tensor on the root rank / None elsewhere, root_rank).  Stream-ordered; nothing blocks the host
    except NCCL's own enqueue.  From the second call on, every run of steps above the cut is ONE CUDA-graph replay
    (captured on static buffers: subtree outputs, persistent receive buffers, the inputs)."""
    import torch.distributed as dist  # pylint: disable=import-outside-toplevel
    be, rank, lab = self.backend, self.rank, self.lab
    torch = be.torch
    handles, keep = {}, []
    moved = 0
    vals = {}

    def emit(o, tensor):
      nonlocal moved
      vals[o] = tensor
      for dst in self.outgoing.get(o, ()):
        buf = be.contiguous(tensor)
        moved += buf.t.numel() * buf.t.element_size()
        keep.append((buf, dist.isend(buf.t, dst, group=self.group)))
    for root, (_, net) in self.nets.items():
      emit(root, net())
    # receives are posted after the local subtrees are enqueued: NCCL orders its stream behind them, so the receive
    # kernels do not occupy the GPU while it computes
    for _, t, src in self.incoming:
      buf = self._recv[t]
      handles[t] = dist.irecv(buf.t, src, group=self.group)
      moved += buf.t.numel() * buf.t.element_size()

    def get(x):
      return self.inputs[x] if x < self.n else vals[x]

    def run_steps(steps):
      out = {}
      for s_i in steps:
        a_, b_, o_ = self.ssa[s_i]
        vals[o_] = out[o_] = self._pair(get(a_), lab[a_], get(b_), lab[b_])
      return out
    for k, (kind, what) in enumerate(self._segments):
      if kind == "recv":
        handles.pop(what).wait()           # the compute stream waits for the transfer; the host does not
        vals[what] = self._recv[what]
        continue
      if k in self._seg_graphs:
        graph, outs = self._seg_graphs[k]
        graph.replay()
        vals.update(outs)
      elif self._runs >= 1 and self.join_graphs:
        graph = torch.cuda.CUDAGraph()
        torch.cuda.current_stream().synchronize()
        with torch.cuda.graph(graph):
          outs = run_steps(what)
        self._seg_graphs[k] = (graph, outs)
        graph.replay()
      else:
        outs = run_steps(what)
      for o_ in outs:
        emit(o_, vals[o_])
    for _, w in keep:
      w.wait()
    self._keep = keep
    self._runs += 1
    self.p2p_bytes = moved
    root_rank = self.owner[-1] if self.ssa else 0
    res = vals.get(self.ssa[-1][2]) if (self.ssa and rank == root_rank) else None
    return res, root_rank


def p2p_issue_order(n_inputs, ssa, owner, transfers, rank):
  """The order in which `ShardedNetwork.run` (late receives) hands point-to-point operations of `rank` to NCCL:
  sends of local subtree results, then every receive (by producer step), then the sends of results computed above the cut, in
  step order.  torch's eagerly initialised NCCL group completes a rank's operations in this order (one stream), which is what
  `tests/test_host_logic_r2.py` simulates to show that no two ranks can wait on each other.  -> [("send"|"recv", tensor, peer)]"""
  producer = {o: i for i, (_, _, o) in enumerate(ssa)}
  roots, pure = local_subtrees(n_inputs, ssa, owner, rank)
  outgoing, incoming = {}, []
  for t, src, dst, _ in transfers:
    if rank == src:
      outgoing.setdefault(t, []).append(dst)
    if rank == dst:
      incoming.append((producer.get(t, -1), t, src))
  incoming.sort()
  ops = []
  for root in roots:                                  # (dict order = the order ShardedNetwork builds and runs its local graphs)
    for dst in outgoing.get(root, ()):
      ops.append(("send", root, dst))
  for _, t, src in incoming:
    ops.append(("recv", t, src))
  for s, (_, _, o) in enumerate(ssa):
    if owner[s] != rank or s in pure:
      continue
    for dst in outgoing.get(o, ()):
      ops.append(("send", o, dst))
  return ops


def schedule_completes(n_inputs, ssa, owner, transfers, world):
  """True iff every point-to-point operation of the plan completes when each rank's operations complete strictly in issue
  order and a send needs its matching receive (the conservative model of torch's eagerly initialised NCCL group with large
  messages).  Pure integer simulation: every rank evaluates it identically before anything is posted."""
  queues = [p2p_issue_order(n_inputs, ssa, owner, transfers, r) for r in range(world)]
  progress = True
  while progress and any(queues):
    progress = False
    for r in range(world):
      if not queues[r]:
        continue
      kind, t, peer = queues[r][0]
      want = ("recv" if kind == "send" else "send", t, r)
      if queues[peer] and queues[peer][0] == want:
        queues[r].pop(0)
        queues[peer].pop(0)
        progress = True
  return not any(queues)
