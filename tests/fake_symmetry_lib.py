"""TEST DOUBLE for the entry points of include/tnb200_symmetry.h (product charges on block-sparse legs), on top of
tests/fake_lib.FakeLib, which covers include/tnb200.h.  `FakeSymmetryLib` adds a numpy transcription of
tnb200_blocksparse_maps_nsym with the kernel's stages, and routes tnb200_blocksparse_maps through it as the library does
(the nsym = 1 case of one map builder).  Its calls are recorded like FakeLib's.  Import this module after
hostrun.install(), which loads the reference before tensornetwork_b200, then call `install()`."""
import numpy as np
import fake_lib
from fake_lib import _vec
from tensornetwork_b200 import _lib


class FakeSymmetryLib(fake_lib.FakeLib):
  """FakeLib and the product-charge map builder"""

  def tnb200_blocksparse_maps(self, nlegs, dims, charges, leg_off, order, partition, split, modulus, shift, nbins, tables, nnz, map_out, stream):
    """the nsym = 1 case of tnb200_blocksparse_maps_nsym, as in csrc/blocksparse_maps.cu"""
    return self._maps(int(nlegs), 1, dims, charges, leg_off, order, partition, split, [int(modulus)], [int(shift)], nbins, tables, nnz,
                      map_out)

  def tnb200_blocksparse_maps_nsym(self, nlegs, nsym, dims, charges, leg_off, order, partition, split, moduli, shifts, nbins, tables,
                                   nnz, map_out, stream):
    nsym = int(nsym)
    if nsym < 1 or nsym > _lib.BLOCKSPARSE_MAX_NSYM:
      return self._fail(_lib.ERR_INVALID, "blocksparse_maps: nsym = %d outside [1, %d]" % (nsym, _lib.BLOCKSPARSE_MAX_NSYM))
    return self._maps(int(nlegs), nsym, dims, charges, leg_off, order, partition, split, [int(moduli[k]) for k in range(nsym)],
                      [int(shifts[k]) for k in range(nsym)], nbins, tables, nnz, map_out)

  def _maps(self, nlegs, nsym, dims, charges, leg_off, order, partition, split, mods, shifts, nbins, tables, nnz, map_out):
    """numpy transcription of csrc/blocksparse_maps.cu: fuse (mixed-radix bins), rank (one pass per bin up to 256 bins, the
    tiled counting sort above), first, bucket, element"""
    partition, split, nbins, nnz = int(partition), int(split), int(nbins), int(nnz)
    if any(m < 0 for m in mods) or any(s < 0 for s in shifts):
      return self._fail(_lib.ERR_INVALID, "blocksparse_maps: negative modulus or shift")
    radix = [m if m > 0 else 2 * s + 1 for m, s in zip(mods, shifts)]
    shifts = [0 if m > 0 else s for m, s in zip(mods, shifts)]
    bins = int(np.prod(np.array(radix, dtype=object)))
    if bins > _lib.BLOCKSPARSE_MAX_BINS or nbins > _lib.BLOCKSPARSE_MAX_BINS:
      return self._fail(_lib.ERR_UNSUPPORTED, "blocksparse_maps: the charges span more than TNB200_BLOCKSPARSE_MAX_BINS bins")
    if bins != nbins:
      return self._fail(_lib.ERR_INVALID, "blocksparse_maps: nbins does not match the moduli and shifts")
    dims = [int(dims[i]) for i in range(nlegs)]
    leg_off = [int(leg_off[i]) for i in range(nlegs)]
    order = [int(order[i]) for i in range(nlegs)]
    ch = _vec(charges, sum(dims) * nsym, np.int64).reshape(-1, nsym)
    tab = _vec(tables, 3 * nbins, np.int64)
    start_right, sect_off, ncols = tab[:nbins], tab[nbins:2 * nbins], tab[2 * nbins:]
    if nnz == 0:
      return 0
    out = _vec(map_out, nnz, np.int64)

    def to_bin(q):
      b = np.zeros(q.shape[0], dtype=np.int64)
      for k in range(nsym):
        c = np.mod(q[:, k], mods[k]) if mods[k] > 0 else q[:, k] + shifts[k]
        b = b * radix[k] + c
      return b

    def partner(b):
      p, mul, rem = np.zeros_like(b), 1, b.copy()
      for k in reversed(range(nsym)):
        c = rem % radix[k]; rem //= radix[k]
        p += ((mods[k] - c) % mods[k] if mods[k] > 0 else 2 * shifts[k] - c) * mul
        mul *= radix[k]
      return p

    def fuse(legs):
      shape = [dims[t] for t in legs] or [1]
      idx = np.indices(shape).reshape(len(shape), -1) if legs else np.zeros((0, 1), dtype=np.int64)
      q = np.zeros((idx.shape[1] if legs else 1, nsym), dtype=np.int64)
      for k, t in enumerate(legs):
        q += ch[leg_off[t] + idx[k]]
      return to_bin(q)

    def rank(b):
      n = b.shape[0]
      self._launches += 1 if nbins <= 256 else 5
      if nbins <= 256:                       # one CTA per bin
        r = np.zeros(n, dtype=np.int64)
        cnt = np.zeros(nbins, dtype=np.int64)
        for v in np.unique(b):
          m = b == v
          r[m] = np.arange(int(m.sum()))
          cnt[v] = m.sum()
        return r, cnt
      # counting sort: tiles of T states, rank in the tile, exclusive scan over (bin, tile), offset + rank in the tile
      ntiles = max(1, min(-(-n // 256), (1 << 22) // nbins))
      T = -(-n // ntiles)
      ntiles = -(-n // T)
      tile = np.arange(n) // T
      key = b * ntiles + tile
      srt = np.argsort(key, kind="stable")
      tcnt = np.bincount(key, minlength=nbins * ntiles)
      off = np.concatenate([[0], np.cumsum(tcnt)])
      trank = np.empty(n, dtype=np.int64)
      trank[srt] = np.arange(n) - off[key[srt]]
      r = off[key] + trank - off[b * ntiles]
      cnt = off[(np.arange(nbins) + 1) * ntiles] - off[np.arange(nbins) * ntiles]
      return r, cnt
    stored = list(range(nlegs))
    L_, R_ = stored[:split], stored[split:]
    bl, br = fuse(L_), fuse(R_)
    bro, bco = fuse(order[:partition]), fuse(order[partition:])
    rr, cr = rank(br)
    rro, _ = rank(bro)
    rco, _ = rank(bco)
    pb = partner(bl)
    first = np.zeros(bl.shape[0] + 1, dtype=np.int64)
    first[1:] = np.cumsum(cr[pb])
    assert first[-1] == nnz
    bucket = np.zeros(br.shape[0], dtype=np.int64)
    bucket[start_right[br] + rr] = np.arange(br.shape[0])
    e = np.arange(nnz)
    l = np.searchsorted(first, e, side="right") - 1
    j = e - first[l]
    r = bucket[start_right[pb[l]] + j]
    row_mul, col_mul, is_row = [0] * nlegs, [0] * nlegs, [0] * nlegs
    m = 1
    for i in range(partition - 1, -1, -1):
      row_mul[order[i]] = m; is_row[order[i]] = 1; m *= dims[order[i]]
    m = 1
    for i in range(nlegs - 1, partition - 1, -1):
      col_mul[order[i]] = m; m *= dims[order[i]]
    Rr = np.zeros(nnz, dtype=np.int64); Cc = np.zeros(nnz, dtype=np.int64); rq = np.zeros((nnz, nsym), dtype=np.int64)
    for legs, state in ((L_, l), (R_, r)):
      rem = state.copy()
      for t in reversed(legs):
        d = rem % dims[t]; rem //= dims[t]
        Rr += d * row_mul[t]; Cc += d * col_mul[t]
        if is_row[t]:
          rq += ch[leg_off[t] + d]
    qb = to_bin(rq)
    out[sect_off[qb] + rro[Rr] * ncols[qb] + rco[Cc]] = e
    self._launches += 7
    return 0


for _name in [n for n in vars(FakeSymmetryLib) if n.startswith("tnb200_")]:
  setattr(FakeSymmetryLib, _name, fake_lib._recorded(_name, vars(FakeSymmetryLib)[_name]))  # pylint: disable=protected-access


def install():
  """puts a fresh FakeSymmetryLib in place of the FakeLib hostrun.install() installed, and returns it"""
  lib = FakeSymmetryLib()
  _lib.set_lib(lib)
  return lib
