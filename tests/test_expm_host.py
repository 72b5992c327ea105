"""CPU: the restatement of scipy's degree rule in expm_rule.py on hand-built matrices, and the fused-path limit against
the header.  The adapter itself runs on the host stand-in in tests/expm_host_runner.py."""
import os
import numpy as np
import pytest
import expm_rule

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_fused_limit_mirrors_header():
  from tensornetwork_b200 import _lib
  src = open(os.path.join(ROOT, "include", "tnb200.h")).read()
  assert "#define TNB200_EXPM_FUSED_MAX_N {}\n".format(_lib.EXPM_FUSED_MAX_N) in src
  assert _lib.EXPM_FUSED_MAX_N >= 32


# t I: every ||A^p||_1^(1/p) is t, and _ell(tI, m) = max(0, ceil((2m log2 t - log2 c_m + 53) / 2m))
@pytest.mark.parametrize("t,expect", [(0.0, (3, 0)), (0.9 * expm_rule.THETA[3], (3, 0)),
                                      (1.1 * expm_rule.THETA[3], (5, 0)), (0.9 * expm_rule.THETA[5], (5, 0)),
                                      (1.1 * expm_rule.THETA[5], (7, 0)), (0.9 * expm_rule.THETA[7], (7, 0)),
                                      (1.1 * expm_rule.THETA[7], (9, 0)), (0.9 * expm_rule.THETA[9], (9, 0)),
                                      (1.1 * expm_rule.THETA[9], (13, 0)), (0.9 * 4.25, (13, 0)),
                                      (1.1 * 4.25, (13, 1)), (4.25 * 2**7 * 1.1, (13, 8)), (-5.0, (13, 1))])
def test_rule_on_scaled_identity(t, expect):
  a = t * np.eye(3)
  assert expm_rule.select(a) == expect
  for m in (3, 5, 7, 9, 13):
    if t:
      assert expm_rule.ell(a, m) == max(0, int(np.ceil((2 * m * np.log2(abs(t)) - np.log2(expm_rule.ELL_C[m]) + 53)
                                                       / (2 * m))))


def test_rule_nilpotent_and_ell_terms():
  # strictly upper triangular: |A|^p = 0 for p >= n, so every _ell is 0, and A^4 = 0 for n = 4 gives degree 3
  n = np.triu(np.full((4, 4), 100.0), 1)
  assert all(expm_rule.ell(n, m) == 0 for m in (3, 5, 7, 9, 13))
  assert expm_rule.select(n) == (3, 0)
  # A^2 = 0 but |A| = ones: every theta test passes (eta = 0), and the _ell terms alone push the degree to 9
  # (_ell(A, 3) = ceil((6 + 53 - log2 c_3) / 6) = 8, _ell(A, 5) = 3, _ell(A, 7) = 2, _ell(A, 9) = 0)
  a = np.array([[1.0, 1.0], [-1.0, -1.0]])
  assert [expm_rule.ell(a, m) for m in (3, 5, 7, 9)] == [8, 3, 2, 0]
  assert expm_rule.select(a) == (9, 0)
