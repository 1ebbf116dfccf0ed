"""CPU: oracle/trf_exact_model.py `exact_first_step`, the float64 model of the exact trust-region step that
tests/test_gpu_exact_paths.py holds the device to, against scipy's own `solve_lsq_trust_region` fed the eigendecomposition of
A = D H D (s = sqrt(lambda), s * uf = V^T g_h): the same number of alpha iterations, alpha within 1e-12 relative, the step within 1e-12.
On seeded nonsingular A (the Gauss-Newton step inside and outside Delta, a warm-started alpha), with dead columns (the model equals scipy
on the live submatrix), and on a singular A, where both take scipy's rank-deficient path."""
import numpy as np
import pytest
from numpy.linalg import norm
from scipy.optimize._lsq.common import solve_lsq_trust_region

from oracle.trf_exact_model import exact_first_step, exact_subproblem, probe_rank

BAR = 1e-12


def normal_equations(seed, n, rank=None):
  """H = J^T J of a seeded J (columns of very different norms), g = J^T f, x."""
  rng = np.random.default_rng(seed)
  m = 3 * n
  J = rng.standard_normal((m, rank or n)) @ rng.standard_normal((rank or n, n)) if rank else rng.standard_normal((m, n))
  J *= 10.0 ** rng.uniform(-2, 3, n)
  f = rng.standard_normal(m)
  return J.T @ J, J.T @ f, rng.standard_normal(n)


def scipy_step(A, g_h, Delta, alpha):
  lam, V = np.linalg.eigh(A)
  lam, V = lam[::-1], V[:, ::-1]                          # scipy's SVD order: s[0] the largest
  s = np.sqrt(np.maximum(lam, 0.0))
  null = s <= 1e-10 * s[0]                                # a singular A: singular values of J_h at rounding level, as an SVD gives them
  s[null] = 1e-15 * s[0]
  uf = np.where(null, 0.0, V.T @ g_h / s)
  return solve_lsq_trust_region(A.shape[0], A.shape[0], uf, s, V, Delta, initial_alpha=alpha)


def scaled(H, g, x):
  scale_inv = np.sqrt(np.diag(H))
  d = 1.0 / scale_inv
  return d[:, None] * H * d[None, :], d * g, norm(x * scale_inv), d


def check_against_scipy(A, g_h, Delta, alpha, full_rank):
  p, a, it, _, _ = exact_subproblem(A, g_h, Delta, full_rank, alpha)
  p_s, a_s, it_s = scipy_step(A, g_h, Delta, alpha)
  assert it == it_s, (it, it_s)
  assert abs(a - a_s) <= BAR * abs(a_s), (a, a_s)
  assert norm(p - p_s) <= BAR * norm(p_s), norm(p - p_s) / norm(p_s)
  return it, a


@pytest.mark.parametrize("seed", range(6))
def test_exact_step_is_scipys_on_a_nonsingular_system(seed):
  """The radius at 1e3, 0.9, 0.3 and 0.05 times the Gauss-Newton step's norm, and again from a warm-started alpha."""
  H, g, x = normal_equations(seed, 24)
  A, g_h, _, _ = scaled(H, g, x)
  full_rank, ratio = probe_rank(A, np.ones(24, bool), np.arange(24))
  assert full_rank and ratio.min() > 10
  gn = norm(np.linalg.solve(A, g_h))
  iters = []
  for f in (1e3, 0.9, 0.3, 0.05):
    it, a = check_against_scipy(A, g_h, f * gn, 0.0, True)
    iters.append(it)
    if it: assert a > 0
    if it: check_against_scipy(A, g_h, f * gn, 3.0 * a, True)
  assert iters[0] == 0 and min(iters[1:]) > 0


def test_first_step_is_the_subproblem_in_the_scaled_variables():
  H, g, x = normal_equations(11, 30)
  A, g_h, Delta, d = scaled(H, g, x)
  x = x * 1e-3                                            # a radius small enough for the search
  Delta = norm(x / d)
  r = exact_first_step(H, g, x, frame_cols=np.arange(18, 30))
  p_s, a_s, it_s = scipy_step(A, g_h, Delta, 0.0)
  assert r.full_rank and r.iterations == it_s > 0 and r.trials == 1
  assert abs(r.alpha - a_s) <= BAR * a_s
  assert norm(r.step / d - p_s) <= BAR * norm(p_s)
  assert all(abs(q - 0.01) > 1e-6 for q in r.phi_ratios)


@pytest.mark.parametrize("seed", range(3))
def test_dead_columns_are_left_out(seed):
  """Zero rows and columns of H (skew, a held intrinsic) are absent from the step: the model on the whole system equals scipy on the
  live submatrix, and the step is zero in the dead columns."""
  H0, g0, x0 = normal_equations(20 + seed, 20)
  n = 26
  dead = np.sort(np.random.default_rng(seed).choice(n, n - 20, replace=False))
  live = np.setdiff1d(np.arange(n), dead)
  H = np.zeros((n, n)); H[np.ix_(live, live)] = H0
  g = np.zeros(n); g[live] = g0
  x = np.zeros(n); x[live] = x0 * 1e-2; x[dead] = 7.0       # a dead column's x adds to Delta through scale_inv = 1
  r = exact_first_step(H, g, x, frame_cols=[])
  A, g_h, _, d = scaled(H0, g0, x0)
  Delta = norm(np.r_[x0 * 1e-2 / d, x[dead]])
  p_s, a_s, it_s = scipy_step(A, g_h, Delta, 0.0)
  assert r.full_rank and r.iterations == it_s
  assert np.all(r.step[dead] == 0)
  assert norm(r.step[live] / d - p_s) <= BAR * norm(p_s)
  assert abs(r.alpha - a_s) <= BAR * abs(a_s)


@pytest.mark.parametrize("seed", range(3))
def test_a_singular_system_takes_scipys_rank_deficient_path(seed):
  """rank(A) = n - 4: the probe finds it, alpha_lower = 0, scipy's reset, every alpha far above the 1e-12 floor, so the step is
  scipy's from the SVD."""
  H, g, x = normal_equations(40 + seed, 24, rank=20)
  x = x * 1e-4                                            # the minimum-norm solution lies outside Delta: phi has a root
  r = exact_first_step(H, g, x, frame_cols=np.arange(12, 24))
  A, g_h, Delta, d = scaled(H, g, x)
  assert not r.full_rank
  p_s, a_s, it_s = scipy_step(A, g_h, Delta, 0.0)
  assert r.iterations == it_s > 0
  assert abs(r.alpha - a_s) <= BAR * a_s
  assert norm(r.step / d - p_s) <= BAR * norm(p_s)


def test_the_probe_eliminates_the_frame_columns_first():
  """The rank is that of the Schur complement of the shared columns: a shared block that is nonsingular on its own is singular once a
  frame column that duplicates one of its columns is eliminated; the same frame column made independent leaves it full rank."""
  J = np.array([[1.0, 0.0, 1.0], [1.0, 0.0, 1.0], [0.0, 1.0, 0.0], [0.0, 0.0, 0.0]])
  live = np.ones(3, bool)
  assert np.linalg.matrix_rank(J[:, :2]) == 2
  full, ratio = probe_rank(J.T @ J, live, [0, 1])
  assert not full and ratio[0] < 0.1
  J[3, 2] = 1.0
  full, ratio = probe_rank(J.T @ J, live, [0, 1])
  assert full and ratio.min() > 10
