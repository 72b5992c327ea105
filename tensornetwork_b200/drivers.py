"""Host-side contraction / split drivers for the `cuda_b200` backend.

These mirror the reference's *callers* of the backend (SURVEY.md 8a rows a7-a10) so the hot
path can be driven — and benchmarked — on a box where the `tensornetwork` package is not
installed.  With the package installed the reference's own `tn.ncon`, `contractors.greedy`,
`split_node*` call the same backend methods and produce the same results.

  ncon(...)             <-> tensornetwork/ncon_interface.py:523-663 (`_jittable_ncon` :364-520)
  contract_network(...) <-> contractors/opt_einsum_paths/path_contractors.py:36-97 (`base`),
                            `contract_between` network_components.py:1984-2095
  split_svd / split_full_svd / split_qr / split_rq
                        <-> network_operations.py:130-255, 446-588, 258-348, 351-443

Design difference from the reference: the label bookkeeping (pure integer work) is compiled
once into a *plan* (a flat list of backend calls) keyed by (shapes, labels, orders); executing
a cached plan is a straight loop of kernel launches with no Python list surgery, which is
what makes CUDA-graph capture of a whole network possible (graph.py).
"""
import ctypes
import os

import numpy as np
from .tensor import B200Tensor

_PLAN_CACHE = {}


# =============================================================================== ncon
def _canonicalize(network_structure):
  """ncon_interface.py:69-115."""
  flat = [l for sub in network_structure for l in sub]
  neg_int = sorted({l for l in flat if not isinstance(l, str) and l < 0})
  pos_int = sorted({l for l in flat if not isinstance(l, str) and l > 0})
  neg_str = sorted({l for l in flat if isinstance(l, str) and l[0] == '-'}, reverse=True)
  pos_str = sorted({l for l in flat if isinstance(l, str) and l[0] != '-'})
  mapping = dict(zip(neg_str + neg_int, range(-len(neg_int + neg_str), 0)))
  mapping.update(dict(zip(pos_int + pos_str, range(1, 1 + len(pos_int + pos_str)))))
  return [[mapping[l] for l in labels] for labels in network_structure], mapping


def _check_network(net, shapes, con_order, out_order):
  """The argument checks of ncon_interface.py:118-238 that guard the hot loop."""
  if len(net) != len(shapes):
    raise ValueError("len(tensors) != len(network_structure)")
  for n, (labels, shape) in enumerate(zip(net, shapes)):
    if len(labels) != len(shape):
      raise ValueError("number of indices does not match number of labels on tensor {}. "
                       "len(labels) = {}, len(shape) = {}".format(n, len(labels), len(shape)))
  sizes = {}
  for labels, shape in zip(net, shapes):
    for l, s in zip(labels, shape):
      if l in sizes and sizes[l] != s:
        raise ValueError("tensor dimensions for label {} are mismatching: {} != {}".format(
            l, sizes[l], s))
      sizes[l] = s


def plan_ncon(shapes, network_structure, con_order=None, out_order=None):
  """Symbolic replay of `_jittable_ncon`: returns (steps, result_slot).

  Each step is a tuple whose first entry names a backend call; operands are slot indices
  into a growing list of tensors (inputs occupy slots 0..n-1)."""
  net, mapping = _canonicalize(network_structure)
  _check_network(net, shapes, con_order, out_order)
  flat = [l for sub in net for l in sub]
  uniq = list(set(flat))
  if not out_order:
    out_order = sorted([l for l in uniq if l < 0], reverse=True)
  else:
    out_order = [mapping[o] for o in out_order]
  if not con_order:
    con_order = sorted([l for l in uniq if l > 0])
  else:
    con_order = [mapping[o] for o in con_order]
  init_con_order = list(con_order)

  steps = []
  nslots = len(shapes)
  slots = list(range(len(shapes)))       # live tensors (slot ids), parallel to `net`
  shp = {i: tuple(s) for i, s in enumerate(shapes)}

  def emit(step, shape):
    nonlocal nslots
    steps.append(step + (nslots,))
    shp[nslots] = tuple(shape)
    nslots += 1
    return nslots - 1

  # partial traces (ncon_interface.py:241-277)
  for n in range(len(slots)):
    labels = net[n]
    tl = [l for l in labels if labels.count(l) == 2]
    if tl:
      num = len(tl) // 2
      uq = sorted(tl)[0:-1:2]
      pos = [[i for i, l in enumerate(labels) if l == t] for t in uq]
      contracted = [p[0] for p in pos] + [p[1] for p in pos]
      free = [i for i in range(len(labels)) if i not in contracted]
      s = shp[slots[n]]
      cdim = int(np.prod([s[d] for d in contracted[:num]]))
      tmp = tuple([s[p] for p in free] + [cdim, cdim])
      slots[n] = emit(("ptrace", slots[n], tuple(free + contracted), tmp),
                      [s[p] for p in free])
      net[n] = [l for l in labels if l not in uq]
      con_order = [c for c in con_order if c not in uq]

  flat = [l for sub in net for l in sub]
  single = [l for l in flat if flat.count(l) == 1 and l > 0]
  if single:
    con_order = [o for o in con_order if o not in single]
  for n, labels in enumerate(net):
    if set(labels).intersection(single):
      inds = tuple(labels.index(l) for l in single if l in labels)
      s = shp[slots[n]]
      slots[n] = emit(("sum", slots[n], inds), [x for i, x in enumerate(s) if i not in inds])
      net[n] = [l for l in labels if l not in single]

  batch_labels, batch_cnts = [], []
  for l in set(flat):
    cnt = flat.count(l)
    if cnt > 2 or (cnt == 2 and l < 0):
      batch_labels.append(l)
      batch_cnts.append(cnt)

  def batch_cont(s1, s2, l1, l2, cb):
    """ncon_interface.py:280-354 as ONE batched tensordot (no transposes/reshapes)."""
    nonlocal con_order
    cb = list(cb)
    b1 = [l1.index(l) for l in cb]
    b2 = [l2.index(l) for l in cb]
    nb1 = {l for l in l1 if l not in cb}
    nb2 = {l for l in l2 if l not in cb}
    cc = list(nb1.intersection(nb2))
    c1 = [l1.index(l) for l in cc]
    c2 = [l2.index(l) for l in cc]
    fp1 = [n for n, l in enumerate(l1) if l not in cc and l not in cb]
    fp2 = [n for n, l in enumerate(l2) if l not in cc and l not in cb]
    sh1, sh2 = shp[s1], shp[s2]
    out_shape = [sh1[i] for i in b1] + [sh1[i] for i in fp1] + [sh2[i] for i in fp2]
    new = emit(("batched", s1, s2, tuple(c1), tuple(c2), tuple(b1), tuple(b2)), out_shape)
    slots.append(new)
    net.append([l1[i] for i in b1] + [l1[i] for i in fp1] + [l2[i] for i in fp2])
    con_order = [c for c in con_order if c not in cc]

  skip = 0
  while con_order:
    ci = con_order[0]
    if ci in batch_labels:
      con_order.append(con_order.pop(0))
      skip += 1
      if skip > len(con_order):
        raise ValueError("ncon seems stuck in an infinite loop. \n"
                         "Please check if `con_order` = {} is a valid contraction order for \n"
                         "`network_structure` = {}".format(init_con_order, network_structure))
      continue
    locs = [n for n, labels in enumerate(net) if ci in labels]
    s2 = slots.pop(locs[1])
    s1 = slots.pop(locs[0])
    l2 = net.pop(locs[1])
    l1 = net.pop(locs[0])
    common = list(set(l1).intersection(l2))
    c1 = [l1.index(l) for l in common]
    c2 = [l2.index(l) for l in common]
    cb = set(batch_labels).intersection(common)
    if cb:
      delete = []
      for i, bl in enumerate(batch_labels):
        if bl in cb:
          batch_cnts[i] -= 1
          if (bl > 0 and batch_cnts[i] <= 2) or (bl < 0 and batch_cnts[i] < 2):
            delete.append(i)
      for i in sorted(delete, reverse=True):
        del batch_cnts[i]
        del batch_labels[i]
      batch_cont(s1, s2, l1, l2, cb)
    else:
      srt = sorted(range(len(c1)), key=lambda i: c1[i])
      a1 = tuple(c1[i] for i in srt)
      a2 = tuple(c2[i] for i in srt)
      sh1, sh2 = shp[s1], shp[s2]
      out_shape = [x for i, x in enumerate(sh1) if i not in a1] + \
          [x for i, x in enumerate(sh2) if i not in a2]
      slots.append(emit(("tensordot", s1, s2, a1, a2), out_shape))
      net.append([l for l in l1 if l not in common] + [l for l in l2 if l not in common])
      con_order = [c for c in con_order if c not in common]

  while len(slots) > 1:
    s2 = slots.pop()
    s1 = slots.pop()
    l2 = net.pop()
    l1 = net.pop()
    common = list(set(l1).intersection(l2))
    cb = set(batch_labels).intersection(common)
    if cb:
      batch_cont(s1, s2, l1, l2, cb)
    else:
      slots.append(emit(("tensordot", s1, s2, (), ()), list(shp[s1]) + list(shp[s2])))
      net.append(l1 + l2)

  res = slots[0]
  if len(net[0]) > 1:
    perm = tuple(net[0].index(l) for l in out_order)
    if perm != tuple(range(len(perm))):
      s = shp[res]
      res = emit(("transpose", res, perm), [s[p] for p in perm])
  return steps, res


def execute_plan(backend, tensors, steps, result_slot):
  vals = list(tensors)
  for st in steps:
    op = st[0]
    if op in ("tensordot", "batched"):
      ba, bb = _batch_axes(st)
      vals.append(backend._contract(vals[st[1]], vals[st[2]], list(st[3]), list(st[4]), list(ba), list(bb)))  # pylint: disable=protected-access
    elif op == "ptrace":
      vals.append(backend.trace(backend.reshape(backend.transpose(vals[st[1]], st[2]), st[3])))
    elif op == "sum":
      vals.append(backend.sum(vals[st[1]], st[2]))
    elif op == "transpose":
      vals.append(backend.transpose(vals[st[1]], st[2]))
    else:
      raise RuntimeError("unknown plan step " + str(op))
  return vals[result_slot]


def ncon(tensors, network_structure, con_order=None, out_order=None, backend=None):
  """Same call signature / semantics as `tn.ncon` (ncon_interface.py:523) for backend tensors
  or numpy arrays (converted with `convert_to_tensor`, i.e. copied host->device)."""
  backend = backend or _default()
  ts = [backend.convert_to_tensor(t) for t in tensors]
  shapes = tuple(t.shape for t in ts)
  key = ("ncon", shapes, _freeze(network_structure), _freeze(con_order), _freeze(out_order))
  plan = _PLAN_CACHE.get(key)
  if plan is None:
    plan = plan_ncon(shapes, [list(n) for n in network_structure], con_order, out_order)
    _PLAN_CACHE[key] = plan
  return execute_plan(backend, ts, *plan)


def _freeze(x):
  if x is None:
    return None
  if isinstance(x, (list, tuple)):
    return tuple(_freeze(y) for y in x)
  return x


# =================================================================== path contraction
def greedy_path(labels, out_labels, size_dict, memory_limit=None):
  """Pairwise order in opt_einsum's convention.  Uses `opt_einsum.paths.greedy` when that
  package is installed (what `contractors.greedy` calls, path_contractors.py:192), otherwise
  numpy's own greedy einsum path search, which reproduces the reference's greedy path
  known-answers (path_calculation_test.py:83-93)."""
  input_sets = [set(l) for l in labels]
  try:
    import opt_einsum  # type: ignore  # pylint: disable=import-outside-toplevel
    return [tuple(p) for p in opt_einsum.paths.greedy(input_sets, set(out_labels),
                                                     dict(size_dict), memory_limit)]
  except ImportError:
    from numpy._core.einsumfunc import _greedy_path  # pylint: disable=import-outside-toplevel
    return [tuple(p) for p in _greedy_path(input_sets, set(out_labels), dict(size_dict),
                                           2**62 if memory_limit is None else memory_limit)]


def _prefer_swapped(l1, l2, shared, sizes=None):
  """True when tensordot(t2, t1) addresses memory better than tensordot(t1, t2): count operands whose
  contracted axes are exactly the trailing axes (first operand, K-major rows) resp. the leading axes
  (second operand, K x N row-major)."""
  n = len(shared)
  if n == 0:
    return False
  cs = set(shared)

  def trailing(l):
    return set(l[len(l) - n:]) == cs

  def leading(l):
    return set(l[:n]) == cs
  keep = int(trailing(l1)) + int(leading(l2))
  swap = int(trailing(l2)) + int(leading(l1))
  if keep != swap or sizes is None:
    return swap > keep
  f1 = int(np.prod([sizes[0][i] for i, l in enumerate(l1) if l not in cs] or [1]))
  f2 = int(np.prod([sizes[1][i] for i, l in enumerate(l2) if l not in cs] or [1]))
  if leading(l1) and leading(l2):      # [k, m] . [k, n]: stream the long operand's free axes last
    return f1 > f2
  if trailing(l1) and trailing(l2):    # [m, k] . [n, k]: the long operand's rows first
    return f1 < f2
  return False


def plan_path(shapes, labels, path, out_labels, nbatch=0):
  """contract_between (network_components.py:2048-2085) replayed symbolically along `path`.

  nbatch > 0: every tensor carries `nbatch` leading sample axes that are never contracted
  (independent networks of identical structure, e.g. MPS batch samples, advanced in lock-step by
  one batched kernel per pairwise step); `labels` describe the remaining axes."""
  labels = [list(l) for l in labels]
  slots = list(range(len(shapes)))
  shp = {i: tuple(s) for i, s in enumerate(shapes)}
  steps = []
  nslots = len(shapes)
  for a, b in path:
    l1, l2 = labels[a], labels[b]
    s1, s2 = slots[a], slots[b]
    shared = [l for l in l1 if l in l2]
    if _prefer_swapped(l1, l2, shared, (shp[s1][nbatch:], shp[s2][nbatch:])):
      # the order of an INTERMEDIATE's axes is ours to choose (only the final result's order is
      # observable, and the closing transpose restores it): put first the operand whose contracted
      # axes trail, so that both operands and the output are plain row-major GEMM views
      l1, l2, s1, s2 = l2, l1, s2, s1
      shared = [l for l in l1 if l in l2]
    a1 = [l1.index(l) for l in shared]
    a2 = [l2.index(l) for l in shared]
    srt = sorted(range(len(a1)), key=lambda i: a1[i])
    a1 = tuple(a1[i] + nbatch for i in srt)
    a2 = tuple(a2[i] + nbatch for i in srt)
    if nbatch:
      bax = tuple(range(nbatch))
      steps.append(("batched", s1, s2, a1, a2, bax, bax, nslots))
      shp[nslots] = tuple(list(shp[s1][:nbatch]) + [x for i, x in enumerate(shp[s1]) if i not in a1 and i >= nbatch] +
                          [x for i, x in enumerate(shp[s2]) if i not in a2 and i >= nbatch])
    else:
      steps.append(("tensordot", s1, s2, a1, a2, nslots))
      shp[nslots] = tuple([x for i, x in enumerate(shp[s1]) if i not in a1] +
                          [x for i, x in enumerate(shp[s2]) if i not in a2])
    new_labels = [l for l in l1 if l not in shared] + [l for l in l2 if l not in shared]
    for i in sorted([a, b], reverse=True):
      del labels[i]
      del slots[i]
    labels.append(new_labels)
    slots.append(nslots)
    nslots += 1
  res = slots[0]
  lab = labels[0]
  if len(lab) > 1:
    perm = tuple(range(nbatch)) + tuple(lab.index(l) + nbatch for l in out_labels)
    if perm != tuple(range(len(perm))):
      steps.append(("transpose", res, perm, nslots))
      res = nslots
  return steps, res


def plan_shapes(shapes, steps):
  """output shape of every slot of a path plan (inputs first, then one slot per step)"""
  shp = [tuple(s) for s in shapes]
  for st in steps:
    op = st[0]
    if op in ("tensordot", "batched"):
      a, b = shp[st[1]], shp[st[2]]
      ba, bb = _batch_axes(st)
      ua, ub = set(st[3]) | set(ba), set(st[4]) | set(bb)
      out = [a[i] for i in ba] + [x for i, x in enumerate(a) if i not in ua] + [x for i, x in enumerate(b) if i not in ub]
    elif op == "transpose":
      out = [shp[st[1]][p] for p in st[2]]
    else:
      raise NotImplementedError("plan_shapes: step kind " + str(op))
    shp.append(tuple(out))
  return shp


def find_chains(steps, n_inputs, min_len=2):
  """Maximal runs of CONSECUTIVE contraction steps in which every step consumes the previous step's result:
  candidates for one chained launch (tnb200_chain_create).  Returns lists of step indices."""
  runs, cur = [], []
  for idx, st in enumerate(steps):
    ok = st[0] in ("tensordot", "batched")
    if ok and cur and (n_inputs + cur[-1]) in (st[1], st[2]):
      cur.append(idx)
      continue
    if len(cur) >= min_len:
      runs.append(cur)
    cur = [idx] if ok else []
  if len(cur) >= min_len:
    runs.append(cur)
  return runs


def _source(steps, n_inputs, slot):
  """the slot `slot` is a view of, looking through transposes"""
  while slot >= n_inputs and steps[slot - n_inputs][0] == "transpose":
    slot = steps[slot - n_inputs][1]
  return slot


def _inputs(st):
  """the operand slots of a plan step"""
  return (st[1], st[2]) if st[0] in ("tensordot", "batched") else (st[1],)


def _batch_axes(st):
  """the batch axes of a contraction step: a tensordot is a batched contraction without any"""
  return st[5:7] if st[0] == "batched" else ((), ())


def _contracted(st, shapes):
  """the number of elements a contraction step sums over; `shapes` are the slot shapes of plan_shapes"""
  return int(np.prod([shapes[st[1]][a] for a in st[3]] or [1]))


def _users(steps):
  """{slot: the steps that read it}, once per operand: a step that reads a slot twice is listed twice"""
  users = {}
  for i, st in enumerate(steps):
    for x in _inputs(st):
      users.setdefault(x, []).append(i)
  return users


def _linked_paths(nxt):
  """the maximal paths s -> nxt[s] -> nxt[nxt[s]] ... of a successor map, in order of their first step"""
  paths = []
  for s in sorted(set(nxt) - set(nxt.values())):
    paths.append([s])
    while paths[-1][-1] in nxt:
      paths[-1].append(nxt[paths[-1][-1]])
  return paths


def find_chain_groups(steps, n_inputs, res_slot, shapes):
  """Candidates for one chained launch each (tnb200_chain_create): lists of step indices in plan order.

  The runs of find_chains go through unchanged.  Among the other contraction steps that are not thin (they contract
  more than 64 elements), step s continues into step u when u is the only consumer of s's result, that result is not
  the network's result and no earlier step continues into u.  Runs linked this way (at least two steps long) that do
  not depend on each other, even transitively, merge into one group: the heads of the four ramps of an MPS
  contraction interleave in plan order, and one launch runs all four.  A group is launched at its first step, so every
  operand a member takes from outside the group must be an input (or a view of one) or come from a step before the
  group's first step; a run that would break this joins no group, and is dropped if it breaks it on its own.
  `shapes` are the slot shapes of plan_shapes."""
  runs = find_chains(steps, n_inputs)
  taken = {i for r in runs for i in r}

  def wide(i):
    return i not in taken and steps[i][0] in ("tensordot", "batched") and _contracted(steps[i], shapes) > 64
  users = {}                                # consumers of each slot, looking through transposes
  for i, st in enumerate(steps):
    for x in _inputs(st):
      users.setdefault(_source(steps, n_inputs, x), set()).add(i)
  anc = []                                  # steps each step depends on, transitively
  for st in steps:
    a = set()
    for x in _inputs(st):
      p = _source(steps, n_inputs, x) - n_inputs
      if p >= 0:
        a |= anc[p] | {p}
    anc.append(a)
  nxt, has_prev = {}, set()
  for s in range(len(steps)):
    u = sorted(users.get(n_inputs + s, ()))
    if wide(s) and n_inputs + s != res_slot and len(u) == 1 and wide(u[0]) and u[0] not in has_prev:
      nxt[s] = u[0]
      has_prev.add(u[0])

  def placeable(group):
    first, members = group[0], set(group)
    for i in group:
      for x in _inputs(steps[i]):
        p = _source(steps, n_inputs, x) - n_inputs
        if p >= 0 and p not in members and p >= first:
          return False
    return True
  groups = []
  for run in _linked_paths(nxt):
    for k, g in enumerate(groups):
      if all(not (anc[i] & set(run)) for i in g) and all(not (anc[i] & set(g)) for i in run) \
          and placeable(sorted(g + run)):
        groups[k] = sorted(g + run)
        break
    else:
      if placeable(run):
        groups.append(run)
  return sorted(runs + groups)


def find_thin_runs(steps, n_inputs, res_slot, shapes, exclude=(), max_len=8):
  """Runs of thin contraction steps linked by dependency (not by index: the ramps of an MPS contraction interleave):
  candidates for one fused launch (tnb200_thin_run_create).  A step is thin when it contracts at most 64 elements;
  step s continues into step u when u is the only consumer of s's result, that result is not the network's result and
  it is u's long operand (larger than u's other operand).  `shapes` are the slot shapes of plan_shapes; steps in
  `exclude` take no part.  Returns lists of at most `max_len` step indices, each at least two long."""
  def thin(i):
    return i not in exclude and steps[i][0] in ("tensordot", "batched") and _contracted(steps[i], shapes) <= 64
  users = _users(steps)
  nxt = {}
  for s in range(len(steps)):
    out = n_inputs + s
    u = users.get(out, [])
    if not thin(s) or out == res_slot or len(u) != 1 or not thin(u[0]):
      continue
    other = steps[u[0]][2] if steps[u[0]][1] == out else steps[u[0]][1]
    if other != out and np.prod(shapes[out]) > np.prod(shapes[other]):
      nxt[s] = u[0]
  runs = []
  for path in _linked_paths(nxt):
    runs += [path[i:i + max_len] for i in range(0, len(path), max_len) if len(path[i:i + max_len]) >= 2]
  return runs


class _Chain:
  """A created chained launch (api "chain") or fused thin run (api "thin_run"): owns the library handle; `steps` are
  the plan step indices it covers."""

  def __init__(self, backend, handle, step_ids, api="chain"):
    self.backend, self.handle, self.steps, self.api = backend, handle, list(step_ids), api

  def launch(self):
    from . import _lib as L  # pylint: disable=import-outside-toplevel
    L.check(getattr(self.backend.lib, "tnb200_%s_launch" % self.api)(self.handle, self.backend._stream()))  # pylint: disable=protected-access

  def __del__(self):
    try:
      if self.handle:
        getattr(self.backend.lib, "tnb200_%s_destroy" % self.api)(self.handle)
        self.handle = None
    except Exception:  # pylint: disable=broad-except
      pass


class CompiledNetwork:
  """A network contraction frozen into a CUDA graph (the `jit` of this backend).

  The plan's kernel launches — with their TMA descriptors — are captured once on static
  buffers; each call copies the inputs into those buffers (device->device, or host->device
  for host inputs) and replays the graph: one driver call instead of one Python round trip
  per pairwise contraction.  The returned tensor is the graph's static output buffer: it is
  overwritten by the next call (clone it to keep it)."""

  def __init__(self, backend, shapes, dtype, labels, out_labels=(), path=None, nbatch=0,
               algorithm=None, num_streams=4, conj_aliases=None, use_chains=True):
    from . import tensor as T  # pylint: disable=import-outside-toplevel
    self.backend = backend
    self.nbatch = nbatch
    torch = backend.torch
    code = T.dtype_code(dtype)
    core_shapes = [tuple(s[nbatch:]) for s in shapes]
    if path is None:
      sizes = {l: s[ax] for s, labs in zip(core_shapes, labels) for ax, l in enumerate(labs)}
      path = (algorithm or greedy_path)(labels, out_labels, sizes)
    self.path = path
    self.steps, self.res_slot = plan_path([tuple(s) for s in shapes], labels, path,
                                          list(out_labels), nbatch)
    # all static inputs live in ONE device arena (256-byte aligned slots) mirrored by ONE pinned host
    # staging arena, so a step's host->device transfer is a single cudaMemcpyAsync
    tdt = T.code_to_torch(code)
    esz = torch.empty((), dtype=tdt).element_size()
    # conj_aliases {i: j}: input i is conj(input j) — e.g. the bra layer of <psi|psi>, which the reference
    # builds on the backend with `tn.conj(node)`.  For real dtypes conj is the identity, so input i is a
    # VIEW of input j's static buffer (as torch's lazy conj is): nothing is staged or copied for it.
    self._alias = dict(conj_aliases or {})
    if self._alias and T.is_complex_code(code):
      raise NotImplementedError("conj_aliases are views and therefore limited to real dtypes")
    for i, j in self._alias.items():
      if j in self._alias or tuple(shapes[i]) != tuple(shapes[j]):
        raise ValueError("conj_aliases must map to a non-aliased input of the same shape")
    offs, tot = [], 0
    for i, shp in enumerate(shapes):
      if i in self._alias:
        offs.append(None)
        continue
      n = int(np.prod(shp)) if len(shp) else 1
      offs.append(tot)
      tot += (n * esz + 255) // 256 * 256
    offs = [offs[self._alias[i]] if i in self._alias else o for i, o in enumerate(offs)]
    self._arena = torch.zeros(max(tot, 256), dtype=torch.uint8, device=backend.device)
    self._host_arena = None
    self._offs, self._esz, self._tdt, self._shapes = offs, esz, tdt, [tuple(s) for s in shapes]
    self.inputs = []
    for shp, off in zip(shapes, offs):
      n = int(np.prod(shp)) if len(shp) else 1
      view = self._arena[off:off + n * esz].view(tdt).view(tuple(shp))
      self.inputs.append(B200Tensor(view, code))
    self.num_pairwise = len(path)
    self.streams = [torch.cuda.Stream() for _ in range(max(1, num_streams))]
    self._build_static(code, use_chains)
    # warm-up on a side stream (loads kernels, sets function attributes), then capture
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      self._run_nodes([side])
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    self.graph = torch.cuda.CUDAGraph()
    l0 = backend.lib.tnb200_launch_count()
    with torch.cuda.graph(self.graph):
      self.output = self._run_nodes(self.streams)
    self.launches_per_replay = int(backend.lib.tnb200_launch_count() - l0)

  # ------------------------------------------------------------------ static plan with chained launches
  def _build_static(self, code, use_chains):
    """Preallocate every step's result (addresses must be known before capture: chained launches freeze their
    operand pointers at creation) and group the plan into nodes: single steps and chains.  Without `use_chains`
    every contraction is a node of its own, writing its own buffer."""
    from . import _lib as L  # pylint: disable=import-outside-toplevel
    be = self.backend
    n_in = len(self.inputs)
    shp = plan_shapes(self._shapes, self.steps)
    # A result whose ONLY consumer is the next step of its run needs no buffer of its own: such results
    # alternate between two ring buffers (step s+2 starts, per sample, after step s+1 has consumed step s),
    # so a run's intermediates are overwritten while still dirty in L2 instead of being written back to HBM.
    torch = be.torch
    ring_of = {}
    nring = int(os.environ.get("TNB200_CHAIN_RING", "2"))
    groups = find_chain_groups(self.steps, n_in, self.res_slot, shp) if use_chains else []
    if nring >= 2:
      users = _users(self.steps)
      # Ring slots are shared ONLY between results of identical shape (so sample b occupies the same region in
      # every step that uses the slot) and are handed out round-robin per shape: a slot written by step s is
      # next written by a step s' >= s + 2, which (per sample, through the run's read-after-write counters)
      # cannot start before step s + 1 — the only reader of step s — has finished that sample.  Results of
      # different per-sample extents never alias (the cfg 2 ramp boundary [256,2,512] -> [512,2,512]).  In a
      # group with branches a member need not wait for the one before it, so nothing there is aliased.
      for run in groups:
        if any(n_in + a not in self.steps[b][1:3] for a, b in zip(run, run[1:])):
          continue
        rings, count = {}, {}
        for k, sid in enumerate(run[:-1]):
          if users.get(n_in + sid, []) == [run[k + 1]] and n_in + sid != self.res_slot:
            key = tuple(shp[n_in + sid])
            if key not in rings:
              need = int(np.prod(key))
              rings[key] = [torch.empty(need, dtype=self._tdt, device=be.device) for _ in range(nring)]
              count[key] = 0
            ring_of[sid] = rings[key][count[key] % nring]
            count[key] += 1
    vals = list(self.inputs)
    for i, st in enumerate(self.steps):
      if st[0] == "transpose":
        vals.append(be.transpose(vals[st[1]], st[2]))
      elif i in ring_of:
        n = int(np.prod(shp[n_in + i]))
        vals.append(B200Tensor(ring_of[i][:n].view(tuple(shp[n_in + i])), code))
      else:
        vals.append(be._new(shp[n_in + i], code))  # pylint: disable=protected-access
    self._vals = vals
    chain_of = {}
    self.chains = []
    def step_array(run):
      pos = {sid: k for k, sid in enumerate(run)}
      arr = (L.ChainStep * len(run))()
      for k, sid in enumerate(run):
        st = self.steps[sid]
        a, b, c = vals[st[1]], vals[st[2]], vals[n_in + sid]
        cs = arr[k]
        cs.a, cs.b, cs.c = a.desc(), b.desc(), c.desc()
        ax_a, ax_b = st[3], st[4]
        ba, bb = _batch_axes(st)
        cs.naxes, cs.nbatch = len(ax_a), len(ba)
        for j, x in enumerate(ax_a):
          cs.axes_a[j] = x
        for j, x in enumerate(ax_b):
          cs.axes_b[j] = x
        for j, x in enumerate(ba):
          cs.batch_a[j] = x
        for j, x in enumerate(bb):
          cs.batch_b[j] = x
        # operands that are (views of) results of earlier steps of this run: their position in it, else -1
        cs.dep_a, cs.dep_b = (pos.get(_source(self.steps, n_in, x) - n_in, -1) for x in _inputs(st))
      return arr

    def create(api, pending):
      while pending:
        run = pending.pop(0)
        if len(run) < 2:
          continue
        handle = ctypes.c_void_p()
        bad = ctypes.c_int32(-1)
        rc = getattr(be.lib, "tnb200_%s_create" % api)(len(run), step_array(run), ctypes.byref(bad), ctypes.byref(handle))
        if rc == 0:
          ch = _Chain(be, handle, run, api)
          self.chains.append(ch)
          for sid in run:
            chain_of[sid] = ch
        elif rc == L.ERR_UNSUPPORTED and bad.value >= 0:
          k = bad.value                               # split the run around the step the kernel cannot take
          pending[:0] = [run[:k], run[k + 1:]]
        elif rc == L.ERR_UNSUPPORTED:
          continue                                    # refused as a whole (too few tiles per step): step by step
        else:
          L.check(rc)
    if use_chains:
      # the chained kernel computes fp32 as TF32: strict fp32 stays on per-step launches
      if not (be.math_mode == L.MATH_SIMT or (code == L.F32 and be.math_mode == L.MATH_STRICT)):
        create("chain", [list(g) for g in groups])
      # fused thin runs (16-bit only) among the steps no chain took; their intermediates stay on chip, so their
      # buffers are released
      if be.math_mode != L.MATH_SIMT:
        create("thin_run", find_thin_runs(self.steps, n_in, self.res_slot, shp, exclude=set(chain_of)))
    for ch in self.chains:
      if ch.api == "thin_run":
        for sid in ch.steps[:-1]:
          vals[n_in + sid] = None
    nodes, seen = [], set()
    for i, st in enumerate(self.steps):
      ch = chain_of.get(i)
      if ch is None:
        nodes.append(("step", i))
      elif ch.api == "thin_run":
        # at its last step: the small operands of its steps may come from steps between its first and last
        if i == ch.steps[-1]:
          nodes.append((ch.api, ch))
      elif id(ch) not in seen:
        seen.add(id(ch))
        nodes.append((ch.api, ch))
    self._nodes = nodes

  def _node_io(self, node):
    n_in = len(self.inputs)
    if node[0] == "step":
      return list(_inputs(self.steps[node[1]])), [n_in + node[1]]
    outs = [n_in + sid for sid in node[1].steps]
    ins = []
    for sid in node[1].steps:
      ins += [x for x in _inputs(self.steps[sid]) if x not in outs]
    if node[0] == "thin_run":
      outs = outs[-1:]                  # the run's intermediates never leave the chip
    return ins, outs

  def _launch_node(self, node):
    be, n_in, vals = self.backend, len(self.inputs), self._vals
    if node[0] in ("chain", "thin_run"):
      node[1].launch()
      return
    st = self.steps[node[1]]
    ba, bb = _batch_axes(st)
    be._contract(vals[st[1]], vals[st[2]], list(st[3]), list(st[4]), list(ba), list(bb), out=vals[n_in + node[1]])  # pylint: disable=protected-access

  def _run_nodes(self, streams):
    """Dependency-aware execution of the node list on `streams`: a node runs on the stream of its most recently
    produced operand and waits (event) only for operands produced on other streams, so independent branches of the
    contraction tree overlap; under CUDA-graph capture this stream/event structure becomes the graph's dependency
    edges.  A transpose is a view and inherits its operand's stream.  All chained launches share streams[0]: two
    persistent chain kernels must never wait for each other's SMs.  A node fed only by graph inputs or chained
    launches takes the next stream in turn: the branches a chain leaves (the ramps after their heads) then go on side
    by side instead of queueing behind one another on streams[0]."""
    torch = self.backend.torch
    main = torch.cuda.current_stream()
    multi = len(streams) > 1 or streams[0] is not main
    home, events, from_chain = {}, {}, set()
    if multi:
      for s in streams:
        s.wait_stream(main)
    rr = 0
    for node in self._nodes:
      ins, outs = self._node_io(node)
      if node[0] == "step" and self.steps[node[1]][0] == "transpose":      # a view: inherits its operand's stream
        src = ins[0]
        if src in home:
          home[outs[0]] = home[src]
          events[outs[0]] = events[src]
          if src in from_chain:
            from_chain.add(outs[0])
        continue
      produced = [i for i in ins if i in home]
      if node[0] == "chain":
        si = 0
      elif all(i in from_chain for i in produced):
        si = rr % len(streams)
        rr += 1
      else:
        si = home[max(produced)]
      stream = streams[si]
      for i in produced:
        if home[i] != si:
          stream.wait_event(events[i])
      with torch.cuda.stream(stream):
        self._launch_node(node)
        e = torch.cuda.Event()
        e.record(stream)
      for o in outs:
        home[o] = si
        events[o] = e
        if node[0] == "chain":
          from_chain.add(o)
    if multi:
      for s in streams:
        main.wait_stream(s)
    return self._vals[self.res_slot]

  def profile(self, work, nb, esize, reps=3):
    """Per-kernel-family device time of one replay, measured live with CUDA events around every node of the
    static plan (a chained launch is one node).  `work` = (M, K, N) of every pairwise step in plan order.
    Bytes are algorithmic: operands + result of a step once; for a chain, only what enters and leaves the launch."""
    torch = self.backend.torch
    cidx, k = {}, 0
    for i, st in enumerate(self.steps):
      if st[0] != "transpose":
        cidx[i] = k
        k += 1
    numel = lambda slot: float(np.prod(self._vals[slot].shape[self.nbatch:]) if self._vals[slot].shape[self.nbatch:] else 1.0)
    stats = {}
    for rep in range(reps + 1):
      evs = []
      for node in self._nodes:
        if node[0] == "step" and self.steps[node[1]][0] == "transpose":
          continue
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        self._launch_node(node)
        e1.record()
        name = self.backend.lib.tnb200_last_kernel().decode()
        ins, outs = self._node_io(node)
        sids = [node[1]] if node[0] == "step" else node[1].steps
        flops = sum(2.0 * work[cidx[s]][0] * work[cidx[s]][1] * work[cidx[s]][2] for s in sids)
        if node[0] == "step":
          m, kk, n = work[cidx[node[1]]]
          byts = float(m * kk + kk * n + m * n)
        else:
          ext_out = [o for o in outs if o == self.res_slot or any(o in self._node_io(nd)[0] for nd in self._nodes if nd is not node)]
          byts = sum(numel(i) for i in set(ins)) + sum(numel(o) for o in ext_out)
        evs.append((name, e0, e1, flops * nb, byts * nb * esize, len(sids)))
      torch.cuda.synchronize()
      if rep == 0:
        continue
      for name, e0, e1, fl, by, nst in evs:
        d = stats.setdefault(name, {"launches": 0.0, "us": 0.0, "flops": 0.0, "bytes": 0.0, "pairwise_steps": 0.0})
        d["launches"] += 1.0 / reps
        d["us"] += e0.elapsed_time(e1) * 1e3 / reps
        d["flops"] += fl / reps
        d["bytes"] += by / reps
        d["pairwise_steps"] += nst / reps
    return stats

  def host_staging(self):
    """Pinned host views (one torch tensor per input) carved from a single staging arena.  Fill them
    in place, then call `run_staged()`: the whole step's input moves with ONE host->device copy."""
    torch = self.backend.torch
    if self._host_arena is None:
      self._host_arena = torch.zeros(self._arena.numel(), dtype=torch.uint8).pin_memory()
      self._host_views = []
      for i, (shp, off) in enumerate(zip(self._shapes, self._offs)):
        if i in self._alias:
          self._host_views.append(None)           # a view of another input: nothing to stage
          continue
        n = int(np.prod(shp)) if len(shp) else 1
        self._host_views.append(self._host_arena[off:off + n * self._esz].view(self._tdt).view(shp))
    return self._host_views

  def stage(self):
    """ONE asynchronous host->device copy of the pinned staging arena on the current stream (pair it with
    `__call__()` on another stream + events to overlap the transfer of the next step with this step's compute)"""
    self._arena.copy_(self._host_arena, non_blocking=True)

  def run_staged(self):
    """one H2D of the staging arena + graph replay"""
    self._arena.copy_(self._host_arena, non_blocking=True)
    self.graph.replay()
    return self.output

  def load(self, tensors):
    """copy inputs (B200Tensor, torch tensors or pinned host tensors) into the static buffers"""
    for i, (dst, src) in enumerate(zip(self.inputs, tensors)):
      if i in self._alias or src is None:
        continue
      t = src.t if isinstance(src, B200Tensor) else src
      dst.t.copy_(t, non_blocking=True)

  def __call__(self, tensors=None):
    if tensors is not None:
      self.load(tensors)
    self.graph.replay()
    return self.output


def contract_network(tensors, labels, out_labels=(), path=None, backend=None,
                     algorithm=greedy_path, nbatch=0):
  """`contractors.greedy(nodes, output_edge_order)` on (tensor, labels) pairs: every label
  that appears on two tensors is a connected edge, labels in `out_labels` dangle."""
  backend = backend or _default()
  ts = [backend.convert_to_tensor(t) for t in tensors]
  shapes = tuple(t.shape for t in ts)
  key = ("path", shapes, _freeze(labels), _freeze(out_labels), _freeze(path), nbatch)
  plan = _PLAN_CACHE.get(key)
  if plan is None:
    if path is None:
      sizes = {l: s[nbatch + ax] for s, labs in zip(shapes, labels) for ax, l in enumerate(labs)}
      path = algorithm(labels, out_labels, sizes)
    plan = plan_path(shapes, labels, path, list(out_labels), nbatch)
    _PLAN_CACHE[key] = plan
  return execute_plan(backend, ts, *plan)


# ============================================================================== split
def _edge_order(backend, tensor, left_axes, right_axes):
  order = tuple(left_axes) + tuple(right_axes)
  if sorted(order) != list(range(tensor.ndim)):
    raise ValueError("left_axes + right_axes must be a permutation of the tensor's axes")
  return backend.transpose(tensor, order)


def split_svd(tensor, left_axes, right_axes, max_singular_values=None, max_truncation_err=None,
              relative=False, backend=None):
  """`tn.split_node` (network_operations.py:130-255): U*sqrt(S), sqrt(S)*Vh, discarded s."""
  backend = backend or _default()
  t = _edge_order(backend, backend.convert_to_tensor(tensor), left_axes, right_axes)
  u, s, vh, trun = backend.svd(t, len(left_axes), max_singular_values, max_truncation_err,
                               relative=relative)
  sq = backend.sqrt(s)
  return (backend.broadcast_right_multiplication(u, sq),
          backend.broadcast_left_multiplication(sq, vh), trun)


def split_full_svd(tensor, left_axes, right_axes, max_singular_values=None,
                   max_truncation_err=None, relative=False, backend=None):
  """`tn.split_node_full_svd` (network_operations.py:446-588): U, diagflat(S), Vh, discarded s."""
  backend = backend or _default()
  t = _edge_order(backend, backend.convert_to_tensor(tensor), left_axes, right_axes)
  u, s, vh, trun = backend.svd(t, len(left_axes), max_singular_values, max_truncation_err,
                               relative=relative)
  return u, backend.diagflat(s), vh, trun


def split_qr(tensor, left_axes, right_axes, backend=None):
  """`tn.split_node_qr` (network_operations.py:258-348)."""
  backend = backend or _default()
  t = _edge_order(backend, backend.convert_to_tensor(tensor), left_axes, right_axes)
  return backend.qr(t, len(left_axes))


def split_rq(tensor, left_axes, right_axes, backend=None):
  """`tn.split_node_rq` (network_operations.py:351-443)."""
  backend = backend or _default()
  t = _edge_order(backend, backend.convert_to_tensor(tensor), left_axes, right_axes)
  return backend.rq(t, len(left_axes))


def _default():
  from .backend import get_instance  # pylint: disable=import-outside-toplevel
  return get_instance()
