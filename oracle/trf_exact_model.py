"""ORACLE — TEST INFRASTRUCTURE ONLY.

scipy's `trf_no_bounds` (scipy/optimize/_lsq/trf.py, the solver behind calibration.py:209-210) restated with ONE change: the
regularised Gauss-Newton direction is solved exactly (dense normal equations) instead of by LSMR.  Everything else is
scipy's own code, imported, not re-typed: `minimize_quadratic_1d`, `solve_trust_region_2d`, `update_tr_radius`,
`check_termination`.  The GPU solver claims exactly these semantics; tests compare its per-iteration table with this model
driven by the oracle residual and a 3-point finite-difference Jacobian, and its first step with `first_step` on its own normal
equations.  `exact_first_step` is the same for tr_solver='exact' (scipy's `solve_lsq_trust_region` on factorisations of A + alpha I,
with the engine's rank rule)."""
from collections import namedtuple

import numpy as np
from numpy.linalg import norm
from scipy.linalg import cho_factor, cho_solve
from scipy.optimize._lsq.common import (check_termination, minimize_quadratic_1d, solve_trust_region_2d,
                                        update_tr_radius)


def subspace(H, g, d, Delta, reg_floor=1e-12):
  """The 2-D subspace of one trf iteration from the normal equations H = JᵀJ, g = Jᵀf in the scaled variables (d = 1/scale_inv):
  the regularisation of the Gauss-Newton system (trf.py's `reg_term`, floored), its exact solve, the orthonormal basis S of
  [g_h, gn_h], and the 2x2 model B_S, g_S.  Returns (S, B_S, g_S, g_h, A) with A = D H D."""
  g_h = d * g
  A = d[:, None] * H * d[None, :]
  a, b = g_h @ A @ g_h, -(g_h @ g_h)
  ag_value = minimize_quadratic_1d(a, b, 0, Delta / norm(g_h))[1]
  reg = max(-ag_value / Delta ** 2, reg_floor)
  gn_h = np.linalg.solve(A + reg * np.eye(A.shape[0]), g_h)
  S, _ = np.linalg.qr(np.vstack((g_h, gn_h)).T)
  return S, S.T @ A @ S, S.T @ g_h, g_h, A


def first_step(H, g, x, reg_floor=1e-12, cost=None, trial_cost=None, max_trials=20):
  """The first step of the model from the normal equations at x0: scale_inv = sqrt(diag H) (zeros -> 1),
  Delta = |x * scale_inv| (or 1), the subspace of `subspace`, then scipy's 2-D trust-region solve.  Without `trial_cost` that is the
  first trial; with it (and the cost at x0) trials that do not lower the cost shrink Delta as trf does, and the first accepted step
  is returned together with the number of trials it took."""
  scale_inv = np.sqrt(np.diag(H)).copy(); scale_inv[scale_inv == 0] = 1
  d = 1.0 / scale_inv
  Delta = norm(x * scale_inv) or 1.0
  S, B_S, g_S, g_h, A = subspace(H, g, d, Delta, reg_floor)
  for trials in range(1, max_trials + 1):
    p_S, _ = solve_trust_region_2d(B_S, g_S, Delta)
    step_h = S @ p_S
    step = d * step_h
    if trial_cost is None: return step
    reduction = cost - trial_cost(x + step)
    if reduction > 0: return step, trials
    predicted = -(0.5 * step_h @ A @ step_h + g_h @ step_h)
    shn = norm(step_h)
    Delta, _ = update_tr_radius(Delta, reduction, predicted, shn, shn > 0.95 * Delta)
  raise RuntimeError(f"no accepted step in {max_trials} trials")


EPS = np.finfo(float).eps
ExactStep = namedtuple("ExactStep", "step alpha iterations full_rank pivot_min pivot_bad_min pivot_before_bad phi_ratios trials Delta cond")
ExactStep.__doc__ = """The first step of `exact_first_step`: step (x1 - x0), the final alpha (unclamped: trf.py's warm start), the alpha
iterations summed over the trials, the rank decision of the probe, the smallest live L_kk^2 / tol, the smallest L_kk^2 / tol among the
pivots that fail (the most clearly failing one: a single failing pivot decides) and the smallest one before the first failure (None
both when none fails), |phi| / Delta of every Newton iteration (the search ends below 0.01), the number of trials, the radius of the last one, and cond, the 2-norm condition number of A + reg I at the damping reg the step was solved
at (live columns): a solve in float64 is determined to about eps * cond of its norm, so two correct implementations differ by that much."""


def probe_rank(A, live, shared):
  """The probe of the exact step at alpha = 0 (DESIGN.md §2): the Schur complement of the shared columns `shared` (in the order the
  engine factors them) after eliminating every other live column, its unpivoted Cholesky pivots against tol = n_s eps max_j A_jj over
  the live shared columns.  A pivot that is not positive is clamped as the device does (rsqrt of max(a_kk, 1e-30)) and the factorisation
  goes on.  Dead columns are left out.  Returns (full rank, L_kk^2 / tol of the live shared pivots in order)."""
  shared = np.asarray(shared, int)
  s = shared[live[shared]]
  other = np.setdiff1d(np.flatnonzero(live), s)
  S = A[np.ix_(s, s)]
  if other.size: S = S - A[np.ix_(s, other)] @ np.linalg.solve(A[np.ix_(other, other)], A[np.ix_(other, s)])
  if s.size == 0: return True, np.zeros(0)
  tol = shared.size * EPS * np.diag(A)[s].max()
  S = S.copy()
  piv = np.zeros(s.size)
  for k in range(s.size):
    rs = 1.0 / np.sqrt(min(max(S[k, k], 1e-30), 1e30))
    col = S[k:, k] * rs
    piv[k] = col[0]
    S[k + 1:, k + 1:] -= np.outer(col[1:], col[1:])
  ratio = np.sign(piv) * piv ** 2 / tol
  return bool(np.all(ratio > 1.0)), ratio


def exact_subproblem(A, g_h, Delta, full_rank, alpha, reg_floor=1e-12, rtol=0.01, max_iter=10):
  """common.py solve_lsq_trust_region on factorisations of A + alpha I with the engine's rank decision `full_rank`: the Gauss-Newton
  step if full rank and inside Delta, else Newton on phi(alpha) = ||p(alpha)|| - Delta in scipy's bracket with its reset, every alpha
  factored as max(alpha, 0 if full rank else reg_floor), p at the last alpha scaled onto the boundary.  Returns
  (step_h, alpha, iterations, |phi| / Delta of each iteration, the damping p was solved at)."""
  eye = np.eye(A.shape[0])

  def p_phi(reg):
    c = cho_factor(A + reg * eye)
    p = -cho_solve(c, g_h)
    pn = norm(p)
    return p, pn - Delta, -(p @ cho_solve(c, p)) / pn

  if full_rank:
    p, phi0, dphi0 = p_phi(0.0)
    if norm(p) <= Delta: return p, 0.0, 0, [], 0.0
  upper = norm(g_h) / Delta
  lower = -phi0 / dphi0 if full_rank else 0.0
  if not full_rank and alpha == 0: alpha = max(1e-3 * upper, np.sqrt(lower * upper))
  floor = 0.0 if full_rank else reg_floor
  ratios = []
  for it in range(max_iter):
    if alpha < lower or alpha > upper: alpha = max(1e-3 * upper, np.sqrt(lower * upper))
    _, phi, dphi = p_phi(max(alpha, floor))
    ratios.append(abs(phi) / Delta)
    if phi < 0: upper = alpha
    ratio = phi / dphi
    lower = max(lower, alpha - ratio)
    alpha -= (phi + Delta) * ratio / Delta
    if abs(phi) < rtol * Delta: break
  p, _, _ = p_phi(max(alpha, floor))
  return p * (Delta / norm(p)), alpha, it + 1, ratios, max(alpha, floor)


def exact_first_step(H, g, x, frame_cols, reg_floor=1e-12, cost=None, trial_cost=None, max_trials=20, shared_cols=None):
  """The first step of tr_solver='exact' from the normal equations at x0 (DESIGN.md §2), the exact-mode counterpart of `first_step`:
  scale_inv = sqrt(diag H) (zeros -> 1), Delta = |x * scale_inv| (or 1), A = D H D, g_h = d * g, dead columns (zero row and column)
  dropped; the rank from `probe_rank` over the shared columns (every column not in `frame_cols`, the frame blocks the engine eliminates;
  `shared_cols` gives their order where the engine's differs from the vector's), then `exact_subproblem`.  With `trial_cost` (and the
  cost at x0) a trial that does not lower the cost shrinks Delta by update_tr_radius and multiplies alpha by Delta / Delta_new, as
  trf.py does, and the first accepted step is returned.  Returns an ExactStep."""
  n = H.shape[0]
  hd = np.diag(H).copy()
  live = hd > 0
  scale_inv = np.sqrt(hd); scale_inv[~live] = 1
  d = 1.0 / scale_inv
  Delta = norm(x * scale_inv) or 1.0
  A = d[:, None] * H * d[None, :]
  g_h = d * g
  if shared_cols is None: shared_cols = np.setdiff1d(np.arange(n), np.asarray(frame_cols, int))
  full_rank, ratio = probe_rank(A, live, shared_cols)
  pivot_min = ratio.min() if ratio.size else np.inf
  bad = np.flatnonzero(ratio <= 1.0)
  pivot_bad_min, pivot_before_bad = (ratio[bad].min(), ratio[:bad[0]].min(initial=np.inf)) if bad.size else (None, None)
  A_l, g_l = A[np.ix_(live, live)], g_h[live]
  alpha, total, phis = 0.0, 0, []
  for trials in range(1, max_trials + 1):
    p, alpha, iters, ph, reg = exact_subproblem(A_l, g_l, Delta, full_rank, alpha, reg_floor)
    total += iters; phis += ph
    step_h = np.zeros(n); step_h[live] = p
    step = d * step_h
    lam = np.linalg.eigvalsh(A_l)[[0, -1]] if A_l.size else np.ones(2)
    out = ExactStep(step, alpha, total, full_rank, pivot_min, pivot_bad_min, pivot_before_bad, phis, trials, Delta,
                    (lam[1] + reg) / (max(lam[0], 0.0) + reg))
    if trial_cost is None: return out
    reduction = cost - trial_cost(x + step)
    if reduction > 0: return out
    predicted = -(0.5 * step_h @ A @ step_h + g_h @ step_h)
    shn = norm(step_h)
    Delta_new, _ = update_tr_radius(Delta, reduction, predicted, shn, shn > 0.95 * Delta)
    alpha *= Delta / Delta_new
    Delta = Delta_new
  raise RuntimeError(f"no accepted step in {max_trials} trials")


def trf_exact(fun, jac, x0, ftol=1e-8, xtol=1e-8, gtol=1e-8, max_nfev=100, reg_floor=1e-12):
  x = np.array(x0, float)
  f = fun(x); nfev = 1
  J = jac(x); njev = 1
  cost = 0.5 * f @ f
  H, g = J.T @ J, J.T @ f
  scale_inv = np.sqrt((J ** 2).sum(0)); scale_inv[scale_inv == 0] = 1
  Delta = norm(x * scale_inv) or 1.0
  rows, it, status, step_norm, reduction = [], 0, None, None, None
  while True:
    g_norm = norm(g, np.inf)
    if g_norm < gtol: status = 1
    rows.append((it, nfev, cost, reduction, step_norm, g_norm))
    if status is not None or nfev >= max_nfev: break
    d = 1.0 / scale_inv
    S, B_S, g_S, g_h, A = subspace(H, g, d, Delta, reg_floor)
    reduction = -1
    while reduction <= 0 and nfev < max_nfev:
      p_S, _ = solve_trust_region_2d(B_S, g_S, Delta)
      step_h = S @ p_S
      predicted = -(0.5 * step_h @ A @ step_h + g_h @ step_h)
      step = d * step_h
      f_new = fun(x + step); nfev += 1
      cost_new = 0.5 * f_new @ f_new
      reduction = cost - cost_new
      shn = norm(step_h)
      Delta_new, ratio = update_tr_radius(Delta, reduction, predicted, shn, shn > 0.95 * Delta)
      step_norm = norm(step)
      status = check_termination(reduction, cost, step_norm, norm(x), ratio, ftol, xtol)
      if status is not None: break
      Delta = Delta_new
    if reduction > 0:
      x = x + step; f = f_new; cost = cost_new
      J = jac(x); njev += 1
      H, g = J.T @ J, J.T @ f
      scale_inv = np.maximum(scale_inv, np.sqrt((J ** 2).sum(0)))
    else:
      step_norm, reduction = 0, 0
    it += 1
  return x, cost, nfev, njev, (status or 0), rows
