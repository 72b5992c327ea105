"""The Padé degree m and squaring count s that scipy.sparse.linalg._matfuncs._expm(A, use_exact_onenorm=True) chooses
(Al-Mohy & Higham 2009, Algorithm 5.1), restated in numpy so the tests do not import a private function.  tnb200_expm
reports its own (m, s) in info; the tests compare the two."""
import numpy as np

THETA = {3: 1.495585217958292e-002, 5: 2.539398330063230e-001, 7: 9.504178996162932e-001, 9: 2.097847961257068e+000}
THETA_13 = 4.25
# 1 / |c_{2m+1}| of the backward-error bound
ELL_C = {3: 100800., 5: 10059033600., 7: 4487938430976000., 9: 5914384781877411840000.,
         13: 113250775606021113483283660800000000.}


def onenorm(a):
  return float(np.abs(a).sum(axis=0).max())


def ell(a, m):
  """_ell(A, m): the extra squarings the backward-error bound asks for, from ||(|A|)^(2m+1)||_1"""
  v = np.ones(a.shape[0])
  b = np.abs(a)
  for _ in range(2 * m + 1):
    v = b.T.dot(v)
  nrm = float(v.max())
  if not nrm:
    return 0
  alpha = nrm / (onenorm(a) * ELL_C[m])
  return max(int(np.ceil(np.log2(alpha / 2.0**-53) / (2 * m))), 0)


def select(a):
  """(m, s) for the square matrix a (n >= 2), computed in double / complex double"""
  a = np.asarray(a, dtype=np.complex128 if np.iscomplexobj(a) else np.float64)
  a2 = a @ a
  a4 = a2 @ a2
  a6 = a4 @ a2
  d4, d6 = onenorm(a4)**(1 / 4.), onenorm(a6)**(1 / 6.)
  eta1 = max(d4, d6)
  if eta1 < THETA[3] and ell(a, 3) == 0:
    return 3, 0
  if eta1 < THETA[5] and ell(a, 5) == 0:
    return 5, 0
  a8 = a6 @ a2
  d8 = onenorm(a8)**(1 / 8.)
  eta3 = max(d6, d8)
  if eta3 < THETA[7] and ell(a, 7) == 0:
    return 7, 0
  if eta3 < THETA[9] and ell(a, 9) == 0:
    return 9, 0
  d10 = onenorm(a4 @ a6)**(1 / 10.)
  eta5 = min(eta3, max(d8, d10))
  s = 0 if eta5 == 0 else max(int(np.ceil(np.log2(eta5 / THETA_13))), 0)
  return 13, s + ell(2.0**-s * a, 13)
