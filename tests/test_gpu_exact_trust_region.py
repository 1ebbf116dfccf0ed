"""GPU (-m gpu): the exact trust-region step, `bundle_adjust(tr_solver="exact")` -- scipy's trf with tr_solver='exact' (the full
subproblem by a search on the Levenberg-Marquardt parameter, common.py solve_lsq_trust_region) on the factorisations of k_lm.

  step parity     against least_squares(method='trf', x_scale='jac', tr_solver='exact') on the dense oracle with a fourth-order
                  finite-difference Jacobian: the first step <= 1e-9 relative, then the cost after every accepted evaluation <= 1e-9
                  relative with the same nfev / njev / status, where the problem has no gauge freedom (camera and board poses fixed);
                  with gauge freedom, the converged cost <= 1e-9 relative and the gauge-normalised parameters.  Dead columns (skew,
                  invalid poses) are left out of scipy's problem: its SVD counts them as rank deficiency, the engine does not (DESIGN.md §2).
  the valley      a 50-view rational camera: the RMS of cv2.calibrateCamera(CALIB_RATIONAL_MODEL, (COUNT+EPS, 3000, 1e-15)) <= 1e-12
                  relative, fx fy cx cy <= 1e-7, where the default subspace step stops higher; the same for thin-prism and tilted
                  cameras with k4..k6 (and s1..s4) held as OpenCV holds them.
  isolation       two identical exact solves agree bit for bit; a default solve after an exact one is the default solve, bit for bit;
                  a bad tr_solver raises ValueError.
The bodies take no device-specific argument so that tests/test_simt_exact_trust_region.py runs the small ones on the interpreter."""
import numpy as np
import pytest
from scipy import optimize

import test_gpu_intrinsics as gi
import test_gpu_motion as gm
import test_gpu_parity as gp
from conftest import load_golden, optimize_of
from multical_b200 import intrinsics
from multical_b200.board import Board
from multical_b200.calibration import from_scene
from multical_b200.structs import struct
from oracle.ba_oracle import Problem
from test_gpu_step_parity import fd5_jacobian

pytestmark = pytest.mark.gpu

BAR = 1e-9
# fisheye k3, k4 (theta^7, theta^9) are so weakly determined that the finite-difference noise of their Jacobian columns (~1e-11) moves
# the reference's first step along them by ~1e-6 of its norm (test_gpu_parity.py allows the fisheye normal equations 3e-9 for the same
# reason); the cost after that step moves by ~3e-9 (bar 1e-8), the converged cost keeps the 1e-9 bar
STEP_BAR, ROW_BAR = {"fisheye_3x5": 1e-6}, {"fisheye_3x5": 1e-8}


# ---------------------------------------------------------------------------------------------------------------- step parity
def fixed_gauge(name):
  """(Calibration, oracle Problem) of a golden scene with camera and board poses held fixed: no gauge freedom."""
  if name in gm.CASES:
    _, calib, prob = gm.make(name)
  else:
    scene, z = load_golden(name)
    calib = from_scene(scene)
    if bool(z["cameras_enabled"]): calib = calib.enable(cameras=True)
    prob = Problem.from_scene(scene, optimize=optimize_of(z))
  prob.optimize.update(camera_poses=False, board_poses=False)
  return calib.enable(camera_poses=False, board_poses=False), prob


def scipy_exact(prob, max_nfev, **kw):
  """least_squares(tr_solver='exact') over the live columns of the oracle's problem: (result, its x over all columns)."""
  x0 = prob.param_vec
  live = np.asarray(np.sqrt(fd5_jacobian(prob, x0).power(2).sum(0))).ravel() > 0

  def full(xl):
    x = x0.copy(); x[live] = xl
    return x

  res = optimize.least_squares(lambda xl: prob.residuals(full(xl)), x0[live], x_scale="jac", method="trf", tr_solver="exact",
                               jac=lambda xl: fd5_jacobian(prob, full(xl)).toarray()[:, live], max_nfev=max_nfev, **kw)
  return res, full(res.x)


def run_step_parity(name, loss="linear", f_scale=1.0):
  calib, prob = fixed_gauge(name)
  x0 = prob.param_vec
  assert np.abs(calib.param_vec - x0).max() < 1e-12
  kw = dict(loss=loss, f_scale=f_scale)
  # the first accepted step (a trial that raises the cost leaves x where it was)
  for nfev in range(2, 12):
    _, x1 = scipy_exact(prob, nfev, **kw)
    if np.any(x1 != x0): break
  first = calib.bundle_adjust(max_iterations=nfev, loss=loss, f_scale=f_scale, tr_solver="exact")
  step_g, step_s = first.param_vec - x0, x1 - x0
  assert np.linalg.norm(step_s) > 0
  bar = STEP_BAR.get(name, BAR)
  assert np.linalg.norm(step_g - step_s) <= bar * np.linalg.norm(step_s), (np.linalg.norm(step_g - step_s) / np.linalg.norm(step_s))
  # the whole solve: the cost after each accepted evaluation
  out = calib.bundle_adjust(max_iterations=60, loss=loss, f_scale=f_scale, tr_solver="exact", tolerance=1e-8)
  ref, _ = scipy_exact(prob, 60, ftol=1e-8, xtol=1e-8, gtol=1e-8, **kw)
  res = out.last_solve
  assert (res.nfev, res.njev, res.status) == (ref.nfev, ref.njev, ref.status), ((res.nfev, res.njev, res.status), (ref.nfev, ref.njev, ref.status))
  assert abs(res.cost - ref.cost) <= BAR * ref.cost, (res.cost, ref.cost)
  # every logged iteration against scipy run to that many evaluations (same path: its cost after the same accepted evaluation)
  for it, nfev, cost, *_ in res.log[1:-1]:
    part, _ = scipy_exact(prob, nfev, ftol=1e-8, xtol=1e-8, gtol=1e-8, **kw)
    assert abs(cost - part.cost) <= ROW_BAR.get(name, BAR) * part.cost, (it, nfev, cost, part.cost)
  return res


@pytest.mark.parametrize("name", ["standard_2x6", "fisheye_3x5", "rolling_2x6"])
def test_step_parity_with_scipy_exact(name):
  run_step_parity(name)


def test_step_parity_with_a_robust_loss():
  run_step_parity("standard_2x6", loss="soft_l1", f_scale=1000.0)


def run_gauge_parity(name):
  scene, z, calib, prob = gp.make(name)
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=lambda x: fd5_jacobian(prob, x).toarray(), x_scale="jac",
                               ftol=1e-14, xtol=1e-14, gtol=1e-14, max_nfev=300, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=1e-13, xtol=1e-13, gtol=1e-13, max_iterations=200, tr_solver="exact")
  res = out.last_solve
  assert abs(res.cost - ref.cost) <= BAR * ref.cost, (res.cost, ref.cost)
  assert res.alpha_iterations > 0
  o = prob.with_param_vec(ref.x)
  a = gp.gauge_normalised(out.camera_poses.poses, out.motion.poses, out.board_poses.poses)
  b = gp.gauge_normalised(o.cam_poses, o.frame_poses, o.board_poses)
  ok_c, ok_f, ok_b = scene["cam_valid"], scene["frame_valid"], scene["board_valid"]
  assert np.abs(a[0][ok_c] - b[0][ok_c]).max() < 1e-6
  assert np.abs(a[1][ok_f] - b[1][ok_f]).max() < 1e-6
  assert np.abs(a[2][ok_b] - b[2][ok_b]).max() < 1e-6
  uv_o, _ = o.reprojected()
  assert np.abs(out.projected.points - uv_o)[calib.valid].max() < 1e-4


@pytest.mark.parametrize("name", ["standard_2x6", "cube3_3x6"])
def test_converged_solution_with_gauge_freedom_matches_scipy_exact(name):
  run_gauge_parity(name)


# ---------------------------------------------------------------------------------------------------------------- the valley
W, H, FOCAL = 1920, 1080, 1200.0
VALLEY = {   # distortion of the generating camera in OpenCV's order, the calibrateCamera flag, the parameters OpenCV holds at zero
  "rational": ([0.12, -0.08, 1e-3, -5e-4, 0.02, 0.35, -0.06, 0.04], "CALIB_RATIONAL_MODEL", []),
  "thin_prism": ([0.12, -0.08, 1e-3, -5e-4, 0.02, 0, 0, 0, 1e-3, -4e-4, 8e-4, 2e-4], "CALIB_THIN_PRISM_MODEL", [5, 6, 7]),
  "tilted": ([0.12, -0.08, 1e-3, -5e-4, 0.02, 0, 0, 0, 0, 0, 0, 0, 0.01, -0.006], "CALIB_TILTED_MODEL", [5, 6, 7, 8, 9, 10, 11]),
}


def valley_views(model, seed=5, F=50, noise=0.3):
  """F views of a 15 x 10 board (5 cm squares) by a 1920 x 1080 camera with f = 1200 px, sigma = 0.3 px noise: (board, views)."""
  import cv2
  rng = np.random.default_rng(seed)
  gx, gy = np.meshgrid(np.arange(15) * 0.05, np.arange(10) * 0.05)
  obj = np.stack([gx.ravel(), gy.ravel(), np.zeros(gx.size)], 1)
  K = np.array([[FOCAL, 0, (W - 1) / 2], [0, FOCAL, (H - 1) / 2], [0, 0, 1]])
  dist = np.array(VALLEY[model][0])
  board = Board(obj, size=(15, 10), min_points=20)
  det = []
  while len(det) < F:
    rvec = rng.uniform(-0.6, 0.6, 3)
    z = rng.uniform(0.9, 2.2)
    R = cv2.Rodrigues(rvec)[0]
    centre = R @ np.array([0.35, 0.225, 0.0])
    t = np.array([rng.uniform(-0.45, 0.45) * z, rng.uniform(-0.25, 0.25) * z, z]) - centre
    uv = cv2.projectPoints(obj, rvec, t, K, dist)[0].reshape(-1, 2) + rng.normal(0, noise, (obj.shape[0], 2))
    cam = (R @ obj.T).T + t
    ok = (uv[:, 0] >= 0) & (uv[:, 0] < W) & (uv[:, 1] >= 0) & (uv[:, 1] < H) & (cam[:, 2] > 0.1)
    if ok.sum() < 40: continue
    det.append([struct(corners=uv[ok].astype(np.float32), ids=np.flatnonzero(ok))])
  views = intrinsics.calibration_points([board], det)
  assert len(views) == F
  return board, views


def run_valley(model, report=print):
  import cv2
  board, views = valley_views(model)
  _, flag, held = VALLEY[model]
  rms, K, d, _, _ = gi.cv_calibrate(views, (W, H), getattr(cv2, flag), (3, 3000, 1e-15))
  nd = len(VALLEY[model][0])
  fixed = None
  if held:
    fixed = np.zeros(5 + nd, bool); fixed[[5 + i for i in held]] = True
  tight = dict(ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=500)
  r = intrinsics.calibrate_views([board], [views], [(W, H)], model=model, fixed=fixed, tr_solver="exact", **tight)[0]
  default = intrinsics.calibrate_views([board], [views], [(W, H)], model=model, fixed=fixed, **tight)[0]
  x = r.intrinsics
  k_err = np.abs(x[:4] / K[[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max()
  report(f"\n{model}: OpenCV RMS {rms!r}, exact {r.rms!r} ({r.solve.nfev} nfev, {r.solve.alpha_iterations} alpha iterations), "
         f"default {default.rms!r} ({default.solve.nfev} nfev, status {default.solve.status}); fx..cy {k_err:.2e}")
  assert abs(r.rms / rms - 1) <= 1e-12, (r.rms, rms)
  assert k_err <= 1e-7, k_err
  if held: assert (x[[5 + i for i in held]] == 0).all()


@pytest.mark.parametrize("model", list(VALLEY))
def test_exact_step_reaches_opencvs_minimum_in_the_valley(model):
  run_valley(model)


# ---------------------------------------------------------------------------------------------------------------- isolation
def solve_arrays(out):
  res = out.last_solve
  return res.cost, np.array(res.log, float), np.asarray(out.param_vec)


def same_bits(a, b):
  assert a[0] == b[0]
  assert np.array_equal(a[1], b[1], equal_nan=True)
  assert np.array_equal(a[2], b[2])


def run_isolation(name, max_iterations=100):
  scene, z, calib, prob = gp.make(name)
  base = solve_arrays(calib.bundle_adjust(max_iterations=max_iterations))
  e1 = solve_arrays(calib.bundle_adjust(max_iterations=max_iterations, tr_solver="exact"))
  e2 = solve_arrays(calib.bundle_adjust(max_iterations=max_iterations, tr_solver="exact"))
  same_bits(e1, e2)
  after = solve_arrays(calib.bundle_adjust(max_iterations=max_iterations))
  same_bits(base, after)
  assert calib.bundle_adjust(max_iterations=max_iterations).last_solve.alpha_iterations == 0
  with pytest.raises(ValueError):
    calib.bundle_adjust(tr_solver="svd")


@pytest.mark.parametrize("name", ["standard_2x6", "rational_2x5"])
def test_exact_solves_are_bit_reproducible_and_leave_the_default_alone(name):
  run_isolation(name)
