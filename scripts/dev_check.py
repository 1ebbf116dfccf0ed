"""Developer diagnostics on a GPU box: prints parity numbers without asserting."""
import sys, time, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from scipy.optimize._numdiff import approx_derivative, group_columns
from multical_b200 import synthetic
from multical_b200.calibration import from_scene
from oracle.ba_oracle import Problem

def check(name, **kw):
  print(f"==== {name} {kw}", flush=True)
  scene = synthetic.make_workload("cfg1", **kw)
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  eng = calib._upload(calib.inliers)
  x0 = prob.param_vec
  print(" N", eng.N, "n", eng.num_params, "x0 diff", np.abs(eng.param_vec - x0).max())
  r = eng.residuals(); r0 = prob.residuals()
  print(" resid diff", np.abs(r - r0).max())
  x1 = x0 + np.random.default_rng(1).normal(0, 1e-3, x0.size)
  r1, c1 = eng.residuals(x1, with_cost=True)
  ro = prob.residuals(x1)
  print(" resid diff @x1", np.abs(r1 - ro).max(), "cost rel", abs(c1 - 0.5 * ro @ ro) / (0.5 * ro @ ro))
  S = prob.sparsity_matrix(); groups = group_columns(S)
  J = approx_derivative(prob.residuals, x1, method="3-point", sparsity=(S, groups)).toarray()
  JtJ, Jtr, cost = eng.linearize(x1)
  H = J.T @ J; g = J.T @ ro
  dH = np.abs(JtJ - H); scale = np.sqrt(np.outer(np.diag(H), np.diag(H))) + 1e-300
  print(" JtJ max rel (diag-normalised)", (dH / scale).max(), " Jtr rel", np.abs(Jtr - g).max() / np.abs(g).max(), "cost rel", abs(cost - 0.5 * ro @ ro) / cost)
  bad = np.argwhere(dH / scale > 1e-5)
  if len(bad): print("  bad entries (first 10)", bad[:10].tolist())
  t = time.time(); out = calib.bundle_adjust(); res = out.last_solve; t1 = time.time() - t
  for row in res.log: print("  ", row)
  print(" gpu solve", res.status, res.message, "cost %.10f" % res.cost, "nfev", res.nfev, "njev", res.njev, "dev_ms %.3f" % res.device_ms, "wall %.3f" % t1, "launches", res.kernel_launches, "chol_fail", res.chol_retries)
  t = time.time(); _, ref = prob.bundle_adjust(); t2 = time.time() - t
  print(" scipy ref cost %.10f nfev %d njev %d wall %.2f" % (ref.cost, ref.nfev, ref.njev, t2))
  out2 = out.bundle_adjust(tolerance=1e-12, xtol=1e-12, gtol=1e-12)
  print(" gpu tight cost %.12f nfev %d status %d" % (out2.last_solve.cost, out2.last_solve.nfev, out2.last_solve.status))

if __name__ == "__main__":
  check("standard")
  check("fisheye", model="fisheye")
  check("rational", model="rational")
  check("thin_prism", model="thin_prism")
  check("cube3", boards=("cube", 10, 10, 0.04, 3), rig="dome", C=3, F=7)
  for wl in ["cfg2", "cfg3"]:
    scene = synthetic.make_workload(wl)
    calib = from_scene(scene).enable(cameras=True)
    t = time.time(); out = calib.bundle_adjust(); res = out.last_solve
    print(wl, "N", int(scene["valid"].sum()), "cost %.6f" % res.cost, "nfev", res.nfev, "njev", res.njev, "status", res.status, "dev_ms %.3f" % res.device_ms, "wall %.3f" % (time.time() - t), "launches", res.kernel_launches, flush=True)
    for row in res.log: print("  ", row)
