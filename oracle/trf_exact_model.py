"""ORACLE — TEST INFRASTRUCTURE ONLY.

scipy's `trf_no_bounds` (scipy/optimize/_lsq/trf.py, the solver behind calibration.py:209-210) restated with ONE change: the
regularised Gauss-Newton direction is solved exactly (dense normal equations) instead of by LSMR.  Everything else is
scipy's own code, imported, not re-typed: `minimize_quadratic_1d`, `solve_trust_region_2d`, `update_tr_radius`,
`check_termination`.  The GPU solver claims exactly these semantics; tests compare its per-iteration table with this model
driven by the oracle residual and a 3-point finite-difference Jacobian, and its first step with `first_step` on its own normal
equations."""
import numpy as np
from numpy.linalg import norm
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
