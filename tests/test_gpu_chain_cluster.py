"""The chained GEMM launch runs its tiles as pairs of M tiles (2j, 2j + 1) in 2-CTA clusters that share one B tile:
each CTA loads its own A tile and half of B, multicast into both.  These cases aim at the pairing:

  * odd tiles_m, where the partner of the last M tile has no tile but still loads and multicasts its half of B, and
    tiles_m == 1, where every pair is such a pair;
  * K-major B, split into two half-height boxes, also with two free modes (inner extent 64: several inner rows per
    box; inner extent 256: one box inside one inner row), and MN-major B, split by 128-byte chunks, also with two
    free modes; an MN-major A on a ragged pair;
  * fewer pairs than co-resident clusters (one sample: at most 14 pairs per step) and several waves of them;
  * padded and aliased outputs, through the cases of test_gpu_chain with bonds that give tiles_m 1 and 3.

Every output is checked element by element against float64 with the bound of test_gpu_chain, bit for bit against the
single-GEMM launch, and a second launch of the same handle must reproduce the first bit for bit."""
import numpy as np
import pytest
import test_gpu_chain as C
from util import get_backend

pytestmark = pytest.mark.gpu

# (samples, TNB200_CHAIN_G)
PAIR_BATCH_G = [(1, None), (6, 2), (24, None)]
# M of the zipper steps 128, 304, 304, 128, 128, 136: tiles_m 1, 3, 3, 1, 1, 2
PAIR_ZIP_BONDS = (128, 304, 128, 136)
# steps s and s + 2 have the same output shape; M of every step 128 or 304
PAIR_RING_BONDS = (128, 304, 304, 304)


def _pair_steps(be, rng, dtype, nb):
  """six steps; 304 rows give tiles_m = 3, 128 rows tiles_m = 1"""
  from tensornetwork_b200 import tensor as T  # pylint: disable=import-outside-toplevel
  code = T.dtype_code(dtype)
  pre = (nb,) if nb > 1 else ()
  b = nb > 1
  sl = (slice(None),) if b else ()
  new = lambda *shape: be._new(pre + shape, code)  # pylint: disable=protected-access,unnecessary-lambda-assignment
  dev = lambda shape, k: C._dev(be, rng, pre + shape, dtype, k ** -0.5)  # pylint: disable=protected-access,unnecessary-lambda-assignment

  def cut(x, idx):   # a strided view of x: its free modes cannot be merged into one
    return type(x)(x.t[sl + idx], code)

  p0 = C._dev(be, rng, pre + (304, 136), dtype)               # pylint: disable=protected-access
  q0 = dev((136, 264), 136)                                   # MN-major B
  r1 = dev((128, 264), 264)
  b2 = cut(dev((3, 72, 304), 304), (slice(None), slice(0, 64), slice(None)))     # K-major, free (3, 64 of 72)
  a3 = C._dev(be, rng, pre + (260, 96), dtype)                # pylint: disable=protected-access
  b3 = cut(dev((2, 260, 96), 96), (slice(None), slice(0, 256), slice(None)))     # K-major, free (2, 256 of 260)
  b4 = cut(dev((136, 3, 72), 136), (slice(None), slice(None), slice(0, 64)))     # MN-major, free (3, 64 of 72)
  q5 = dev((128, 200), 128)                                   # MN-major B
  c0, c1, c2, c3, c4, c5 = new(304, 264), new(128, 304), new(128, 3, 64), new(260, 2, 256), new(304, 3, 64), new(304, 200)
  sp = lambda s: C._spec(s, b)  # pylint: disable=protected-access,unnecessary-lambda-assignment
  return [
      C._Step(sp("bmk,bkn->bmn"), p0, q0, c0),                         # tiles_m 3, MN-major B
      C._Step(sp("bmk,bnk->bmn"), r1, c0, c1, dep_b=0),                # tiles_m 1, K-major B (ragged N)
      C._Step(sp("bmk,bpnk->bmpn"), c1, b2, c2, dep_a=1),              # tiles_m 1, K-major B, inner free extent 64
      C._Step(sp("bmk,bpnk->bmpn"), a3, b3, c3),                       # tiles_m 3, K-major B, inner free extent 256
      C._Step(sp("bmk,bkpn->bmpn"), p0, b4, c4),                       # tiles_m 3, MN-major B with two free modes
      C._Step(sp("bkm,bkn->bmn"), c1, q5, c5, dep_a=1),                # tiles_m 3, MN-major A and B
  ]


@pytest.mark.parametrize("nb,G", PAIR_BATCH_G)
@pytest.mark.parametrize("dtype", C.DTYPES)
def test_pair_tiles_and_b_splits(dtype, nb, G, monkeypatch):
  """ragged pairs, tiles_m == 1, every way of splitting B between the two CTAs of a pair"""
  C._env(monkeypatch, G)  # pylint: disable=protected-access
  be = get_backend()
  steps = _pair_steps(be, np.random.default_rng(51), dtype, nb)
  C._check_steps(be, steps, dtype, C._launch_twice(be, steps))  # pylint: disable=protected-access


@pytest.mark.parametrize("nb,G", C.BATCH_G[:2])
@pytest.mark.parametrize("dtype", C.DTYPES)
def test_pair_zipper_ragged(dtype, nb, G, monkeypatch):
  monkeypatch.setattr(C, "ZIP_BONDS", PAIR_ZIP_BONDS)
  C.test_chain_zipper_ragged(dtype, nb, G, monkeypatch)


@pytest.mark.parametrize("nb,G", C.BATCH_G[:2])
@pytest.mark.parametrize("dtype", C.DTYPES)
def test_pair_padded_outputs(dtype, nb, G, monkeypatch):
  monkeypatch.setattr(C, "ZIP_BONDS", PAIR_ZIP_BONDS)
  C.test_chain_padded_outputs(dtype, nb, G, monkeypatch)


@pytest.mark.parametrize("nb,G", C.BATCH_G[:2])
@pytest.mark.parametrize("dtype", C.DTYPES)
def test_pair_aliased_ring(dtype, nb, G, monkeypatch):
  monkeypatch.setattr(C, "RING_BONDS", PAIR_RING_BONDS)
  C.test_chain_aliased_ring(dtype, nb, G, monkeypatch)
