"""CPU: block-sparse legs that carry a product of Abelian charges (U(1) x U(1), U(1) x Z_2, Z_2 x Z_3, three to five
components).  The host sector maps, their charges and their order equal the reference's
`_find_transposed_diagonal_sparse_blocks`; the charge-degeneracy arithmetic equals brute-force counting; the sector
order helper equals the reference's `block_sparse.utils.unique`."""
import itertools
import numpy as np
import pytest
from tensornetwork_b200 import blocksparse as bs

U1 = None
# (name, per-component modulus: None = U(1), N = Z_N)
SYMMETRIES = [("U1xU1", (U1, U1)), ("U1xZ2", (U1, 2)), ("Z2xZ3", (2, 3)), ("U1x3", (U1, U1, U1)), ("U1xZ2xU1xZ3", (U1, 2, U1, 3)),
              ("5comp", (U1, 2, U1, U1, 3))]


def _ref_types(tn, mods):
  return [tn.U1Charge if m is None else tn.Z2Charge if m == 2 else tn.ZNCharge(m) for m in mods]


def _random_legs(rng, mods, dims):
  out = []
  for d in dims:
    cols = [rng.integers(-2, 3, d) if m is None else rng.integers(0, m, d) for m in mods]
    out.append((np.stack(cols, axis=1).astype(np.int64), bool(rng.integers(0, 2))))
  return out


def _ours(legs, mods):
  return [bs.Index(q, f, mods) for q, f in legs]


def _ref(tn, legs, mods):
  from tensornetwork.block_sparse.charge import BaseCharge
  types = _ref_types(tn, mods)
  return [BaseCharge(q.astype(np.int16), charge_types=types) for q, _ in legs], [f for _, f in legs]


@pytest.mark.parametrize("name,mods", SYMMETRIES)
def test_sector_maps_equal_the_reference(tn, name, mods):
  from tensornetwork.block_sparse.blocksparse_utils import _find_transposed_diagonal_sparse_blocks
  rng = np.random.default_rng(sum(map(ord, name)))
  checked = 0
  for trial in range(12):
    n = int(rng.integers(2, 5))
    legs = _random_legs(rng, mods, rng.integers(2, 6, n))          # the reference fails on dimension-1 legs under numpy 2
    idx = _ours(legs, mods)
    if bs._count_allowed(idx) == 0:
      continue
    charges, flows = _ref(tn, legs, mods)
    for order in itertools.permutations(range(n)):
      for part in range(n + 1):
        bs._MAP_CACHE.clear()
        qn, dims, maps = bs._sector_maps(idx, list(order), part)
        rmaps, rq, rdims = _find_transposed_diagonal_sparse_blocks(charges, flows, part, list(order))
        assert qn.shape == (len(rmaps), len(mods)), (trial, order, part)
        np.testing.assert_array_equal(qn, np.asarray(rq.charges, dtype=np.int64))
        np.testing.assert_array_equal(dims, np.asarray(rdims).T.reshape(-1, 2))
        for m, r in zip(maps, rmaps):
          np.testing.assert_array_equal(m, np.asarray(r).ravel())
        checked += 1
  assert checked > 100


@pytest.mark.parametrize("name,mods", SYMMETRIES)
def test_count_allowed_and_group_hist(name, mods):
  rng = np.random.default_rng(7 + sum(map(ord, name)))
  for trial in range(20):
    n = int(rng.integers(1, 5))
    idx = _ours(_random_legs(rng, mods, rng.integers(0 if trial == 3 else 1, 6, n)), mods)
    assert bs._count_allowed(idx) == bs._fused_allowed(idx).shape[0], trial
    shifts = bs._shifts(idx, mods)
    radix = [m if m else 2 * s + 1 for m, s in zip(mods, shifts)]
    legs = sorted(rng.choice(n, int(rng.integers(0, n + 1)), replace=False).tolist())
    h = bs._group_hist(idx, legs, shifts, tuple(mods), int(np.prod(radix)))
    fused = bs._fused_dense([idx[t] for t in legs], tuple(mods))            # brute force: every state of the group
    comps = [fused[:, k] if m else fused[:, k] + s for k, (m, s) in enumerate(zip(mods, shifts))]
    want = np.bincount(np.ravel_multi_index(comps, radix), minlength=int(np.prod(radix)))
    np.testing.assert_array_equal(h, want)


def test_single_symmetry_legs_are_unchanged():
  q = np.array([0, 1, -1, 2])
  for charges, mod in ((q, None), (q[:, None], None), (q[:, None], (None,)), (np.mod(q, 3), 3)):
    ix = bs.Index(charges, True, mod)
    assert ix.nsym == 1 and ix.charges.shape == (4,) and ix.modulus == (mod[0] if isinstance(mod, tuple) else mod)
    assert ix.key() == (ix.charges.tobytes(), True, ix.modulus)
  qn, _, _ = bs._sector_maps([bs.Index(q, False), bs.Index(q, True)], [0, 1], 1)
  assert qn.ndim == 1 and np.array_equal(qn, np.unique(q))


@pytest.mark.parametrize("width", [1, 2, 3, 4, 5, 6])
def test_sector_order_equals_reference_unique(tn, width):
  from tensornetwork.block_sparse.utils import unique
  rng = np.random.default_rng(width)
  for trial in range(10):
    cols = []
    for k in range(width):
      kind = rng.integers(0, 3)
      cols.append(rng.integers(-300, 300, 200) if kind == 0 else rng.integers(0, 3, 200) if kind == 1 else
                  rng.integers(-32768, 32768, 200))
    rows = np.stack(cols, axis=1).astype(np.int16)
    rows = rows[rng.integers(0, 200, 400)]                                    # repeated rows
    got, lab = bs._unique_charges(rows.astype(np.int64))
    want = unique(rows)
    np.testing.assert_array_equal(got, np.asarray(want, dtype=np.int64).reshape(-1, width))
    np.testing.assert_array_equal(got[lab], rows)


def test_product_charges_outside_int16_raise():
  with pytest.raises(ValueError, match="int16"):
    bs._unique_charges(np.array([[40000, 0], [0, 1]]))


def test_legs_with_different_symmetries_raise():
  a = bs.Index(np.zeros((3, 2), dtype=np.int64), False, (None, 2))
  b = bs.Index(np.zeros((3, 2), dtype=np.int64), True, (None, None))
  with pytest.raises(ValueError, match="different symmetries"):
    bs._count_allowed([a, b])


def test_tutorial_sized_product_legs_run_without_dense_enumeration():
  """four legs of dim 100 (10^8 dense states): the counts come from histograms, the stored positions from two groups"""
  rng = np.random.default_rng(3)
  mods = (None, 2)
  idx = _ours([(np.stack([rng.integers(-3, 4, 100), rng.integers(0, 2, 100)], axis=1), f)
               for f in (False, False, True, True)], mods)
  nnz = bs._count_allowed(idx)
  pos = bs._fused_allowed(idx)
  assert pos.shape[0] == nnz and 0 < nnz < 10 ** 8 and np.all(np.diff(pos) > 0)
