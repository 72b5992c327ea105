"""Every single-launch contraction kernel of tnb200_tensordot checked element by element against float64, at the tile,
mask and template edges where a kernel goes wrong: wgmma (bf16 / f16 / tf32), DMMA (f64, split-K), the thin streaming
kernels (thin_simt_{a,d}, thin_mma_{a,d}, thin_mma_tf32_{a,d}), skinny_outer, skinny_dot and the generic SIMT kernel.

Every case goes through be._contract(..., out=view), the path CompiledNetwork takes for its non-chained steps:

  * C is a view into a larger buffer: extra elements on every row and a trailing slab (batch or outermost mode).  The
    pad holds a sentinel and the view NaN, so a box the kernel fails to store stays NaN, and a store outside the view
    overwrites a sentinel.
  * A and B are views into buffers whose out-of-view elements are NaN (a large sentinel for integers).  Their row pads
    keep the 16-byte alignment that selects the kernel under test, so a kernel that folds an element outside its view
    into the arithmetic produces NaN; one that over-reads but masks by selection stays correct.
  * One launch must name the expected kernel (tnb200_last_kernel) with the expected launch count (no repack, no
    fallback), leave every pad element as it was bit for bit, and write finite values within the bound below.
  * A second launch into the NaN-refilled view must reproduce the first bit for bit.  skinny_dot and simt_splitk are
    exempt: they add K-slice partial sums into a workspace with atomics, so the order of their fp32 / fp64 additions
    changes from run to run; for them the second launch is held to the bound only.  Integer results are exact.

The bound, elementwise, with r = a . b and s = |a| . |b| in float64 from the operands as stored:

    |c - r| <= u_out |r| + (u_in + K u_acc) s + eta_out

  u_out  rounding of the accumulator to the output type: 2^-8 for bf16 (its unit roundoff, an 8-bit significand) and
         2^-10 for f16 (twice its unit roundoff); 2^-23 for f32 and 2^-52 for f64 (twice theirs; nothing is rounded
         there, the accumulator is the output type).  The same constants as the chained-launch test.
  eta_out  the absolute error of that rounding below the output type's normal range, where a relative bound does not
         hold: f16's subnormals are spaced 2^-24 apart, so round-to-nearest is off by up to 2^-25 for |c| < 2^-14.
         A K = 2 contraction of O(1) operands produces such results (r = 3e-6 with s = 1.4e-3, rounded correctly, is
         5x over the relative bound alone).  bf16 and f32 share fp32's exponent range, where the term (<= 2^-134) is
         far below every other one here, and f64's is below 2^-1074: it is 0 for them.
  u_in   rounding of the inputs before they are multiplied: 0 for 16-bit inputs (a product of two 11- or 8-bit
         significands is exact in fp32) and for f64.  The TF32 paths (wgmma_tf32, thin_mma_tf32_{a,d}) hand the fp32
         bit patterns to the tensor cores, which use the top 10 explicit mantissa bits: truncation, |x - t(x)| <
         2^-10 |x| and |t(x)| <= |x|, so |ab - t(a)t(b)| < 2^-10 |a||b| + 2^-10 |a||b| = 2^-9 |a||b|.  Round-to-nearest
         conversion would halve that; 2^-9 holds for either.
  u_acc  one accumulation step: 2^-23 for fp32 accumulators, 2^-52 for f64.  A sum of K terms in any order (sequential,
         tree, atomics in any order) is within (K - 1) u sum |x_i| of the exact sum for a round-to-nearest unit
         roundoff u, so K u_acc = 2 K u leaves a factor of two, which also covers an accumulator that truncates.

Complex (c64 / c128, simt only): the accumulator is the output type, so u_out = 0.  Each of Re c and Im c is a sum of
2K real products ar br - ai bi (or ar bi + ai br), each added by one fma: an error of at most 2K u sum(|ar br| + |ai bi|)
<= 2K u sum |a||b| = K u_acc s with s built from the moduli |a|, |b|.  The bound is applied to the real and the imaginary
part separately.  Conjugation (TNB200_CONJ_A / _B) is exact, and the reference applies np.conj before the product.

The constants are derived, not fitted: a ratio above 1 is a bug.  Each parametrised test prints its largest
error/bound ratio."""
import ctypes
import math
import numpy as np
import pytest
from util import get_backend

pytestmark = pytest.mark.gpu

SENTINEL = -7.5                    # C pad (float types)
INT_SENTINEL = -7                  # C pad (integer types)
INT_FILL = -(1 << 30) + 7          # integers have no NaN: unwritten / out-of-view integer elements hold this
U_OUT = {"bfloat16": 2.0**-8, "float16": 2.0**-10, "float32": 2.0**-23, "float64": 2.0**-52,
         "complex64": 0.0, "complex128": 0.0}
U_ACC = {"float64": 2.0**-52, "complex128": 2.0**-52}      # 2^-23 for every other (fp32-accumulating) type
ETA_OUT = {"float16": 2.0**-25}                            # 0 for every other type
U_IN_TF32 = 2.0**-9
TF32_KERNELS = ("wgmma_tf32", "thin_mma_tf32_a", "thin_mma_tf32_d")
ATOMIC_KERNELS = ("skinny_dot", "simt_splitk")             # nondeterministic summation order: bound only
LAUNCHES = {"skinny_dot": 2, "simt_splitk": 2, "dmma_f64_splitk": 2}   # kernel + finalize / reduce; 1 for the others
INT_DTYPES = ("int32", "int64")
COMPLEX_DTYPES = ("complex64", "complex128")
ITEMSIZE = {"bfloat16": 2, "float16": 2, "float32": 4, "float64": 8, "complex64": 8, "complex128": 16, "int32": 4,
            "int64": 8}


def _torch():
  import torch  # pylint: disable=import-outside-toplevel
  return torch


def _tdtype(dtype):
  torch = _torch()
  return getattr(torch, dtype)


def _host_dtype(dtype):
  return np.complex128 if dtype in COMPLEX_DTYPES else (np.int64 if dtype in INT_DTYPES else np.float64)


def _align(dtype):
  """elements per 16 bytes (at least 1)"""
  return max(1, 16 // ITEMSIZE[dtype])


def _fill_value(dtype):
  return INT_FILL if dtype in INT_DTYPES else float("nan")


# ---------------------------------------------------------------------------------------------- host-side helpers
def parse_spec(spec):
  """'bmk,bkn->bmn' -> (la, lb, out, batch, free a, free b, contracted); the output must be in tnb200's order"""
  ins, out = spec.split("->")
  la, lb = ins.split(",")
  bat = [x for x in out if x in la and x in lb]
  fa = [x for x in la if x not in lb]
  fb = [x for x in lb if x not in la]
  con = [x for x in la if x in lb and x not in out]
  assert out == "".join(bat + fa + fb), spec
  return la, lb, out, bat, fa, fb, con


def default_pad(shape, dtype):
  """a trailing slab of the outermost mode, and each innermost row padded to the next 16-byte multiple plus 16 bytes"""
  pad = [0] * len(shape)
  if not shape:
    return pad
  al = _align(dtype)
  pad[0] += 1
  pad[-1] += -shape[-1] % al + al
  return pad


def padded_view(shape, dtype, pad, fill, off=0, device="cuda"):
  """A view of `shape` into a flat buffer of shape + pad elements per mode (starting `off` elements in), the whole
  buffer filled with `fill`.  Returns (flat, view, inside): inside marks the flat buffer's elements under the view."""
  torch = _torch()
  big = tuple(int(s) + int(p) for s, p in zip(shape, pad))
  n = math.prod(big) + off
  flat = torch.empty(n, dtype=_tdtype(dtype), device=device)
  flat.fill_(fill)
  box = tuple(slice(0, int(s)) for s in shape)
  view = flat[off:].view(big)[box]
  idx = torch.arange(n)[off:].view(big)[box]
  inside = np.zeros(n, dtype=bool)
  inside[idx.reshape(-1).numpy()] = True
  return flat, view, inside


def sample(rng, shape, dtype, scale=1.0):
  if dtype in INT_DTYPES:
    return rng.integers(-3, 4, size=shape).astype(np.int64)
  x = rng.standard_normal(shape) * scale
  if dtype in COMPLEX_DTYPES:
    x = x + 1j * rng.standard_normal(shape) * scale
  return x


def to_host(t):
  """a device view as float64 / complex128 / int64 numpy"""
  torch = _torch()
  t = t.detach()
  if t.is_complex():
    return t.to(torch.complex128).cpu().numpy()
  if t.dtype in (torch.int32, torch.int64):
    return t.to(torch.int64).cpu().numpy()
  return t.to(torch.float64).cpu().numpy()


def raw_bits(t):
  """the bit patterns of a tensor as unsigned integers of its element size (NaN-safe comparison)"""
  torch = _torch()
  t = t.detach().contiguous().cpu()
  if t.is_complex():
    t = torch.view_as_real(t).contiguous()
  if t.dtype == torch.bfloat16:
    t = t.view(torch.int16)
  a = t.numpy()
  return a.view("u%d" % a.itemsize)


def make_operand(rng, shape, dtype, pad=None, scale=1.0, device="cuda"):
  """(device view, the values it holds as float64 / complex128 / int64); out-of-view elements are NaN (INT_FILL)"""
  torch = _torch()
  pad = default_pad(shape, dtype) if pad is None else pad
  _, view, _ = padded_view(shape, dtype, pad, _fill_value(dtype), device=device)
  view.copy_(torch.from_numpy(sample(rng, shape, dtype, scale)).to(device=view.device, dtype=view.dtype))
  return view, to_host(view)


def reference(spec, a, b, conj=(False, False)):
  """(r, s, K): r = a . b and s = |a| . |b| in float64 / complex128 (int64 for integers), in the output's order"""
  la, lb, out, bat, fa, fb, con = parse_spec(spec)
  dims = dict(zip(la, a.shape))
  dims.update(zip(lb, b.shape))
  size = lambda labels: math.prod(dims[x] for x in labels)  # pylint: disable=unnecessary-lambda-assignment

  def mat(x, labels, rows, cols):
    order = bat + rows + cols
    return np.ascontiguousarray(np.einsum(labels + "->" + "".join(order), x)).reshape(size(bat), size(rows), size(cols))

  am, bm = mat(a, la, fa, con), mat(b, lb, con, fb)
  if conj[0]:
    am = np.conj(am)
  if conj[1]:
    bm = np.conj(bm)
  shape = [dims[x] for x in out]
  r = np.matmul(am, bm).reshape(shape)
  s = np.matmul(np.abs(am), np.abs(bm)).reshape(shape)
  return r, s, size(con)


def error_ratio(got, r, s, K, dtype, tf32=False):
  """(largest |c - r| / bound over the elements, per component for complex; a description of that element).
  Integers must be exact (ratio 0)."""
  if dtype in INT_DTYPES:
    np.testing.assert_array_equal(got, r)
    return 0.0, ""
  u_in = U_IN_TF32 if tf32 else 0.0
  bound = U_OUT[dtype] * np.abs(r) + (u_in + K * U_ACC.get(dtype, 2.0**-23)) * s + ETA_OUT.get(dtype, 0.0)
  if dtype in COMPLEX_DTYPES:
    diff = np.maximum(np.abs(got.real - r.real), np.abs(got.imag - r.imag))
  else:
    diff = np.abs(got - r)
  with np.errstate(divide="ignore", invalid="ignore"):
    ratio = np.where(bound > 0, diff / bound, np.where(diff == 0, 0.0, np.inf))
  if not ratio.size:
    return 0.0, ""
  i = np.unravel_index(ratio.argmax(), ratio.shape)
  return float(ratio[i]), "at %s: c = %r, r = %r, s = %.3g" % (tuple(int(x) for x in i), got[i], r[i], s[i])


# --------------------------------------------------------------------------------------------- the check
def run_case(be, spec, a, b, dtype, kernel, c_store=None, c_pad=None, c_off=0, conj=(False, False), simt_math=False):
  """One _contract call into a padded, NaN-filled view of C, checked as the module docstring says; then a second
  launch.  a, b: (device view, stored values).  c_store: C's storage order (default: the output order).  Returns the
  largest error/bound ratio."""
  from tensornetwork_b200 import _lib as L  # pylint: disable=import-outside-toplevel
  from tensornetwork_b200 import tensor as T  # pylint: disable=import-outside-toplevel
  torch = _torch()
  la, lb, out, bat, _, _, con = parse_spec(spec)
  (av, a64), (bv, b64) = a, b
  code = T.dtype_code(_tdtype(dtype))
  dims = dict(zip(la, av.shape))
  dims.update(zip(lb, bv.shape))
  cst = c_store or out
  cshape = [dims[x] for x in cst]
  flat, cview, inside = padded_view(cshape, dtype, default_pad(cshape, dtype) if c_pad is None else c_pad,
                                    INT_SENTINEL if dtype in INT_DTYPES else SENTINEL, off=c_off)
  cview = cview.permute([cst.index(x) for x in out])
  A, B, C = T.B200Tensor(av, code), T.B200Tensor(bv, code), T.B200Tensor(cview, code)
  ax_a, ax_b = [la.index(x) for x in con], [lb.index(x) for x in con]
  ba, bb = [la.index(x) for x in bat], [lb.index(x) for x in bat]
  r, s, K = reference(spec, a64, b64, conj)
  tf32 = kernel in TF32_KERNELS
  pad_bits = raw_bits(flat)[~inside]
  results, worst = [], 0.0
  for launch in range(2):
    cview.fill_(_fill_value(dtype))
    saved = be.math_mode
    be.math_mode = L.MATH_SIMT if simt_math else L.MATH_DEFAULT
    try:
      l0 = be.lib.tnb200_launch_count()
      be._contract(A, B, ax_a, ax_b, ba, bb, conj[0], conj[1], out=C)  # pylint: disable=protected-access
      torch.cuda.synchronize()
      got_kernel, launches = be.lib.tnb200_last_kernel().decode(), be.lib.tnb200_launch_count() - l0
    finally:
      be.math_mode = saved
    assert (got_kernel, launches) == (kernel, LAUNCHES.get(kernel, 1)), (spec, dtype, got_kernel, launches)
    after = raw_bits(flat)[~inside]
    assert (after == pad_bits).all(), "launch %d: %d pad elements of C overwritten" % (launch, (after != pad_bits).sum())
    got = to_host(cview)
    if dtype not in INT_DTYPES:
      assert np.isfinite(got).all(), "launch %d: %d elements of C unwritten (NaN) or not finite" % (
          launch, (~np.isfinite(got)).sum())
    results.append(raw_bits(cview))
    if launch == 0 or kernel in ATOMIC_KERNELS:
      ratio, where = error_ratio(got, r, s, K, dtype, tf32)
      worst = max(worst, ratio)
      assert ratio <= 1.0, "launch %d (%s, %s, %s): error/bound %.3g %s" % (launch, spec, dtype, kernel, ratio, where)
  if kernel not in ATOMIC_KERNELS:
    differ = int((results[0] != results[1]).sum())
    assert differ == 0, "%d elements differ between two launches (%s)" % (differ, kernel)
  return worst


def _report(family, worst):
  print("%s: largest error/bound %.3f" % (family, worst))


def _spec(spec, batched):
  return spec if batched else spec.replace("b", "")


def _pre(nb):
  return (nb,) if nb > 1 else ()


def _operands(spec, dims, dtype, seed, a_pad=None, b_pad=None, scale_b=None):
  """operands of `spec` with extents `dims` (label -> extent); B is scaled by 1/sqrt(K) unless told otherwise"""
  la, lb, _, _, _, _, con = parse_spec(spec)
  rng = np.random.default_rng(seed)
  K = math.prod(dims[x] for x in con)
  sa = [dims[x] for x in la]
  sb = [dims[x] for x in lb]
  scale = K ** -0.5 if scale_b is None else scale_b
  return make_operand(rng, sa, dtype, a_pad), make_operand(rng, sb, dtype, b_pad, scale)


def sm_count(be):
  sms, major, minor, mem = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int64()
  assert be.lib.tnb200_device_info(ctypes.byref(sms), ctypes.byref(major), ctypes.byref(minor), ctypes.byref(mem)) == 0
  return sms.value


# ------------------------------------------------------------------------------------------------- wgmma
WG_DTYPES = ["bfloat16", "float16", "float32"]
WG_KERNEL = {"bfloat16": "wgmma_bf16", "float16": "wgmma_f16", "float32": "wgmma_tf32"}
# A: K-major (k innermost) or MN-major (m innermost); B likewise
MAJORS = {"A_K,B_K": "bmk,bnk->bmn", "A_K,B_MN": "bmk,bkn->bmn", "A_MN,B_K": "bkm,bnk->bmn", "A_MN,B_MN": "bkm,bkn->bmn"}


def wgmma_bn(M, N, batch, sms):
  """The single-launch kernel's tile width, as tc_prepare (gemm_wgmma.cu) picks it for a problem that is not swapped:
  the first of 256, 128, 64 whose tile count tiles_m * ceil(N / BN) * batch reaches one tile per SM, skipping 256 and
  128 when half the tile already covers N; 64 otherwise."""
  tiles_m = -(-M // 128)
  for bn in (256, 128, 64):
    if bn > 64 and bn // 2 >= N:
      continue
    if tiles_m * -(-N // bn) * batch >= sms or bn == 64:
      return bn
  raise AssertionError("unreachable")


def batch_for_bn(M, N, bn, sms):
  """the smallest batch under which the rule above picks `bn`"""
  for nb in range(1, 4 * sms + 1):
    if wgmma_bn(M, N, nb, sms) == bn:
      return nb
  raise AssertionError("no batch selects BN = %d for %d x %d" % (bn, M, N))


@pytest.mark.parametrize("majors", ["A_K,B_MN", "A_MN,B_K"])
@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("dtype", WG_DTYPES)
def test_wgmma_every_tile_width(dtype, bn, majors):
  """M = 200, N = 264, K = 72: ragged against the 128-row tile, every BN and the 64- or 32-element k-block; the batch
  is chosen from the device's SM count so that the tile-width rule picks `bn`"""
  be = get_backend()
  M, N, K = 200, 264, 72
  nb = batch_for_bn(M, N, bn, sm_count(be))
  spec = _spec(MAJORS[majors], nb > 1)
  a, b = _operands(spec, {"b": nb, "m": M, "n": N, "k": K}, dtype, 101)
  _report("wgmma BN=%d %s" % (bn, dtype), run_case(be, spec, a, b, dtype, WG_KERNEL[dtype]))


@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("K", ["below_one_kblock_8", "below_one_kblock_40", "ring_wraps_2056"])
@pytest.mark.parametrize("majors", sorted(MAJORS))
@pytest.mark.parametrize("dtype", WG_DTYPES)
def test_wgmma_majors_and_k(dtype, majors, K, nb):
  """M = 136, N = 200 (BN = 64): every K-major / MN-major combination; K below one k-block (the ring is clamped to
  num_kb + 1 stages) and long enough for the ring to wrap many times"""
  be = get_backend()
  k = int(K.rsplit("_", 1)[1])
  assert wgmma_bn(136, 200, nb, sm_count(be)) == 64
  spec = _spec(MAJORS[majors], nb > 1)
  a, b = _operands(spec, {"b": nb, "m": 136, "n": 200, "k": k}, dtype, 102)
  _report("wgmma %s" % dtype, run_case(be, spec, a, b, dtype, WG_KERNEL[dtype]))


@pytest.mark.parametrize("mnk", [(1, 300, 136, 1), (64, 264, 72, 3), (40, 130, 2056, 1)])
@pytest.mark.parametrize("dtype", WG_DTYPES)
def test_wgmma_swap_ab(dtype, mnk):
  """M <= 64 under N >= 128 runs as C^T = B^T A^T, stored transposed through the scalar epilogue"""
  be = get_backend()
  M, N, K, nb = mnk
  spec = _spec("bmk,bkn->bmn", nb > 1)
  a, b = _operands(spec, {"b": nb, "m": M, "n": N, "k": K}, dtype, 103)
  _report("wgmma swap-AB %s" % dtype, run_case(be, spec, a, b, dtype, WG_KERNEL[dtype]))


@pytest.mark.parametrize("nb", [1, 3])
@pytest.mark.parametrize("pitch", ["odd", "aligned"])
@pytest.mark.parametrize("dtype", WG_DTYPES)
def test_wgmma_c_pitch(dtype, pitch, nb):
  """C rows padded to N + 1 elements (not 16-byte aligned: the scalar epilogue, vec_ok false) or to the next 16-byte
  multiple plus 16 bytes (the paired stores, vec_ok true)"""
  be = get_backend()
  M, N, K = 136, 200, 72
  spec = _spec("bmk,bkn->bmn", nb > 1)
  a, b = _operands(spec, {"b": nb, "m": M, "n": N, "k": K}, dtype, 104)
  cshape = list(_pre(nb)) + [M, N]
  c_pad = default_pad(cshape, dtype) if pitch == "aligned" else [1] + [0] * (len(cshape) - 2) + [1]
  _report("wgmma C pitch %s %s" % (pitch, dtype), run_case(be, spec, a, b, dtype, WG_KERNEL[dtype], c_pad=c_pad))


# -------------------------------------------------------------------------------------------------- DMMA
def dmma_bn(M, N, batch, sms):
  """gemm_dmma_f64's tile width: 128 once tiles_m * ceil(N / 128) * batch fills the SMs and N > 64, else 64"""
  return 64 if -(-M // 128) * -(-N // 128) * batch < sms or N <= 64 else 128


@pytest.mark.parametrize("pitch", ["odd", "even"])
@pytest.mark.parametrize("majors", sorted(MAJORS))
@pytest.mark.parametrize("bn", [64, 128])
def test_dmma_f64(bn, majors, pitch):
  """M = 200, N = 264, K = 40: ragged against 128, BN and the 16-deep k-block; every A_K / B_K instance; C rows of an
  odd pitch (scalar stores, vec_ok false) or an even one (double2 stores)"""
  be = get_backend()
  M, N, K = 200, 264, 40
  sms = sm_count(be)
  nb = 1 if bn == 64 else next(x for x in range(1, 4 * sms) if dmma_bn(M, N, x, sms) == 128)
  assert dmma_bn(M, N, nb, sms) == bn
  spec = _spec(MAJORS[majors], nb > 1)
  a, b = _operands(spec, {"b": nb, "m": M, "n": N, "k": K}, "float64", 105, a_pad=None)
  cshape = list(_pre(nb)) + [M, N]
  c_pad = [1] + [0] * (len(cshape) - 2) + [1 if pitch == "odd" else 2]
  _report("dmma_f64", run_case(be, spec, a, b, "float64", "dmma_f64", c_pad=c_pad))


@pytest.mark.parametrize("majors", sorted(MAJORS))
def test_dmma_f64_splitk(majors):
  """100 x 72 per sample, batch 3, K = 4100: cut into slices of 528 with a ragged last one (404), reduced in order"""
  be = get_backend()
  spec = MAJORS[majors]
  a, b = _operands(spec, {"b": 3, "m": 100, "n": 72, "k": 4100}, "float64", 106)
  _report("dmma_f64_splitk", run_case(be, spec, a, b, "float64", "dmma_f64_splitk", c_pad=[1, 0, 1]))


# ------------------------------------------------------------------------------------------- thin kernels
THIN_DTYPES = ["float64", "float32", "float16", "bfloat16"]
L_ONE, L_BATCHED = 65552, 21856   # L x batch >= 65536 (a thin problem); multiples of 16, not of 64


@pytest.mark.parametrize("P", [1, 3, 6, 8])
@pytest.mark.parametrize("K", [2, 3, 5, 7, 8])
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_thin_simt_a(dtype, K, P):
  """C[p][l] = S[p][k] X[k][l] on CUDA cores: K and P are rounded up to 2, 4 or 8 in the template and the rest masked"""
  be = get_backend()
  nb = 3 if P in (3, 8) else 1
  spec = _spec("bpk,bkl->bpl", nb > 1)
  a, b = _operands(spec, {"b": nb, "p": P, "k": K, "l": L_BATCHED if nb > 1 else L_ONE}, dtype, 107)
  _report("thin_simt_a %s" % dtype, run_case(be, spec, a, b, dtype, "thin_simt_a"))


@pytest.mark.parametrize("kp", [(5, (2, 3)), (8, (2, 4))])
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_thin_simt_a_multimode_p(dtype, kp):
  """a P group of two modes that do not merge in C (its middle mode has a trailing slab), batched"""
  be = get_backend()
  K, (P0, P1) = kp
  spec = "bpqk,bkl->bpql"
  a, b = _operands(spec, {"b": 3, "p": P0, "q": P1, "k": K, "l": L_BATCHED}, dtype, 108)
  c_pad = [1, 0, 1, _align(dtype)]
  _report("thin_simt_a %s" % dtype, run_case(be, spec, a, b, dtype, "thin_simt_a", c_pad=c_pad))


@pytest.mark.parametrize("P", [2, 4, 8])
@pytest.mark.parametrize("K", [2, 4, 8])
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_thin_simt_d(dtype, K, P):
  """C[l][p] = X[l][k] S[k][p] on CUDA cores, X rows and C rows packed (the kernel requires it)"""
  be = get_backend()
  nb = 3 if K == P else 1
  spec = _spec("blk,bkp->blp", nb > 1)
  L = L_BATCHED if nb > 1 else L_ONE
  x_pad = [1] + [0] * (1 + (nb > 1))
  a, b = _operands(spec, {"b": nb, "l": L, "k": K, "p": P}, dtype, 109, a_pad=x_pad)
  _report("thin_simt_d %s" % dtype, run_case(be, spec, a, b, dtype, "thin_simt_d", c_pad=list(x_pad)))


@pytest.mark.parametrize("kp", [(3, 4), (4, 3), (6, 8)])
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_thin_d_shape_outside_the_grid(dtype, kp):
  """thin_simt_d has instances for K, P in {2, 4, 8} only; the planner sends other mode-D shapes to skinny_outer"""
  be = get_backend()
  K, P = kp
  spec = "lk,kp->lp"
  a, b = _operands(spec, {"l": L_ONE, "k": K, "p": P}, dtype, 110, a_pad=[1, 0])
  _report("skinny_outer (mode D shapes) %s" % dtype, run_case(be, spec, a, b, dtype, "skinny_outer", c_pad=[1, 0]))


MMA_KERNEL = {"bfloat16": ("thin_mma_a", "thin_mma_d"), "float16": ("thin_mma_a", "thin_mma_d"),
              "float32": ("thin_mma_tf32_a", "thin_mma_tf32_d")}


@pytest.mark.parametrize("K", [16, 32, 64])
@pytest.mark.parametrize("P", [9, 17, 40, 63, 64])
@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32"])
def test_thin_mma_a(dtype, P, K):
  """mode A on the tensor cores: P rounded up to a 16-, 32- or 64-row tile and masked.  L is a multiple of 64 for the
  16-bit kernel; for TF32 a multiple of 32 but not of 64"""
  be = get_backend()
  nb = 3 if P in (17, 63) else 1
  if dtype == "float32":
    L = L_BATCHED if nb > 1 else L_ONE + 16
  else:
    L = L_BATCHED + 32 if nb > 1 else L_ONE + 48
  assert L % (32 if dtype == "float32" else 64) == 0 and (dtype != "float32" or L % 64)
  spec = _spec("bpk,bkl->bpl", nb > 1)
  a, b = _operands(spec, {"b": nb, "p": P, "k": K, "l": L}, dtype, 111)
  _report("%s %s" % (MMA_KERNEL[dtype][0], dtype), run_case(be, spec, a, b, dtype, MMA_KERNEL[dtype][0]))


@pytest.mark.parametrize("K", [16, 32, 64])
@pytest.mark.parametrize("P", [16, 32, 64])
@pytest.mark.parametrize("dtype", ["bfloat16", "float16", "float32"])
def test_thin_mma_d(dtype, P, K):
  """mode D on the tensor cores, X rows padded to K + 8 and C rows to P + 8 elements"""
  be = get_backend()
  nb = 3 if P == K else 1
  L = L_BATCHED + 32 if nb > 1 else L_ONE + 48
  spec = _spec("blk,bkp->blp", nb > 1)
  row_pad = [1] + [0] * (nb > 1) + [8]
  a, b = _operands(spec, {"b": nb, "l": L, "k": K, "p": P}, dtype, 112, a_pad=row_pad)
  _report("%s %s" % (MMA_KERNEL[dtype][1], dtype), run_case(be, spec, a, b, dtype, MMA_KERNEL[dtype][1], c_pad=row_pad))


# ------------------------------------------------------------------------------------------------ skinny
@pytest.mark.parametrize("path", ["vector_L1024", "scalar_L1027", "scalar_C_offset"])
@pytest.mark.parametrize("K", [5, 32])
@pytest.mark.parametrize("S", [1, 3, 16])
@pytest.mark.parametrize("orient", ["a_short", "a_long"])
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_skinny_outer(dtype, orient, S, K, path):
  """one side S <= 16, K <= 32, the other side L long: 16-byte vectors when the long mode is unit-stride in the
  operand and in C and everything is aligned (L = 1024), one element per thread otherwise (L = 1027, or C one
  element off its 16-byte alignment).  a_long stores C as [p][l] so that its long mode is unit-stride too."""
  be = get_backend()
  nb = 3 if K == 5 else 1
  L = 1027 if path == "scalar_L1027" else 1024
  if orient == "a_short":
    spec, c_store = _spec("bpk,bkl->bpl", nb > 1), None
  else:
    spec, c_store = _spec("bkl,bkp->blp", nb > 1), _spec("bpl", nb > 1)
  a, b = _operands(spec, {"b": nb, "p": S, "k": K, "l": L}, dtype, 113)
  c_off = 1 if path == "scalar_C_offset" else 0
  _report("skinny_outer %s" % dtype, run_case(be, spec, a, b, dtype, "skinny_outer", c_store=c_store, c_off=c_off))


@pytest.mark.parametrize("MN", [1, 2, 4])
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_skinny_dot_packed(dtype, MN):
  """A = [K][M], B = [K][N] packed with M == N: the vectorised reduction; batch 3, K = 12288.  (In f64 a 16-byte
  vector holds two elements, so M = N = 4 takes the general kernel.)"""
  be = get_backend()
  spec, K = "bkm,bkn->bmn", 12288
  op_pad = [1, _align(dtype), 0]        # keeps the rows packed and the batch stride a 16-byte multiple
  a, b = _operands(spec, {"b": 3, "k": K, "m": MN, "n": MN}, dtype, 114, a_pad=op_pad, b_pad=op_pad)
  _report("skinny_dot %s" % dtype, run_case(be, spec, a, b, dtype, "skinny_dot"))


DOT_GENERAL = {
    "divisor_carve_12288": ("bmk,bnk->bmn", {"k": 12288}),        # one K mode > DOT_IB: split as (6, 2048)
    "prime_4099": ("bkm,bkn->bmn", {"k": 4099}),                  # no divisor <= DOT_IB: one k per outer step
    "two_modes_3x2000": ("bmij,bnji->bmn", {"i": 3, "j": 2000}),  # K modes that do not merge; inner block 2000
}


@pytest.mark.parametrize("case", sorted(DOT_GENERAL))
@pytest.mark.parametrize("dtype", THIN_DTYPES)
def test_skinny_dot_general(dtype, case):
  """M x N = 3 x 2 (not the packed square), batch 3: the strided reduction over an offset table of the inner K block"""
  be = get_backend()
  spec, kdims = DOT_GENERAL[case]
  dims = dict({"b": 3, "m": 3, "n": 2}, **kdims)
  a, b = _operands(spec, dims, dtype, 115)
  _report("skinny_dot %s" % dtype, run_case(be, spec, a, b, dtype, "skinny_dot"))


# -------------------------------------------------------------------------------------------------- SIMT
# (spec, extents, kernel): 37 x 45 is below one 64 x 64 tile; a K of 3000 over 3 tiles is cut into atomic K-slices
SIMT_SHAPES = {
    "simt": ("bkm,bkn->bmn", {"b": 2, "m": 37, "n": 45, "k": 100}, "simt"),
    "simt_splitk": ("bmk,bnk->bmn", {"b": 3, "m": 37, "n": 45, "k": 3000}, "simt_splitk"),
}


@pytest.mark.parametrize("conj", [(False, False), (True, False), (False, True), (True, True)], ids=str)
@pytest.mark.parametrize("kernel", sorted(SIMT_SHAPES))
@pytest.mark.parametrize("dtype", COMPLEX_DTYPES)
def test_simt_complex_conj(dtype, kernel, conj):
  """c64 / c128 under every TNB200_CONJ_A / TNB200_CONJ_B combination, against np.conj in complex128"""
  be = get_backend()
  spec, dims, kern = SIMT_SHAPES[kernel]
  a, b = _operands(spec, dims, dtype, 116)
  _report("%s %s" % (kern, dtype), run_case(be, spec, a, b, dtype, kern, conj=conj))


@pytest.mark.parametrize("kernel", sorted(SIMT_SHAPES))
@pytest.mark.parametrize("dtype", INT_DTYPES)
def test_simt_integer_exact(dtype, kernel):
  be = get_backend()
  spec, dims, kern = SIMT_SHAPES[kernel]
  a, b = _operands(spec, dims, dtype, 117, scale_b=1.0)
  run_case(be, spec, a, b, dtype, kern)


@pytest.mark.parametrize("shape", [("bmk,bkn->bmn", {"b": 1, "m": 130, "n": 70, "k": 300}, "simt"),
                                   SIMT_SHAPES["simt_splitk"]], ids=["simt", "simt_splitk"])
@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_simt_16bit_math_simt(dtype, shape):
  """16-bit operands under TNB200_MATH_SIMT: the generic kernel instead of the tensor cores"""
  be = get_backend()
  spec, dims, kern = shape
  spec = _spec(spec, dims["b"] > 1)
  a, b = _operands(spec, dims, dtype, 118)
  _report("%s %s" % (kern, dtype), run_case(be, spec, a, b, dtype, kern, simt_math=True))


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_simt_splitk_long_k(dtype):
  """a tile below 64 x 64 over K = 9001 skips the GEMM (the skinny long-K rule) and runs split-K on CUDA cores"""
  be = get_backend()
  spec = "bmk,bkn->bmn"
  a, b = _operands(spec, {"b": 3, "m": 37, "n": 45, "k": 9001}, dtype, 119)
  _report("simt_splitk %s" % dtype, run_case(be, spec, a, b, dtype, "simt_splitk", c_pad=[1, 0, 1]))
