"""GPU (-m gpu): the exact trust-region step (`tr_solver="exact"`, the alpha search in k_lm) at every path of the kernel, against
`oracle.trf_exact_model.exact_first_step` on the device's own normal equations at x0.  A trust-region method converges even when its
step is slightly wrong, so a wrong second solve (`solve_again`: phi' of the Newton iteration) or a wrong rank decision would still leave
every converged-cost test passing; these tests compare the first step itself:
  first step   <= max(1e-9, eps cond(A + reg I)) relative in norm, <= max(1e-8, eps cond) per component over max|step|, cond at the
               damping the step was solved at (a float64 solve is determined to about eps cond: ~1e-5 where a gauge-singular search ends
               at alpha ~ 1e-12, 1e-9 everywhere else); the same number of alpha iterations; the same rank decision, seen as a
               Gauss-Newton step inside Delta or a step on the boundary (|step_h| = Delta to 1e-12); no Cholesky retry.  The model's
               decisions must not be ties on rounding: on a full-rank probe every pivot L_kk^2 >= 10 tol; on a rank-deficient one some
               failing pivot <= 0.1 tol and every pivot before the first failure >= 10 tol (a case that misses this checks everything else
               and then reports itself as xfail with the pivots); |phi| / Delta of every Newton iteration at least 1e-6 from rtol 0.01.
The paths: the one-CTA reduced Cholesky at its limit (n_s = 127) and the blocked one from 128 (last panels of 1, 18, 32 and 30 rows at
n_s = 129, 146, 160, 286), at frames of 6 (static) and 12 (rolling) parameters, on an 8-CTA grid with one SYRK frame chunk (6 frames)
and on the whole machine with several (40 frames), all rank-deficient (free camera or board poses); a gauge-fixed full-rank blocked
probe with dead skew columns, its Gauss-Newton step, and its full-rank alpha search after rejected trials with one and several chunks;
hand-eye frames folded by k_fold_hand_eye beyond one batch; no frame block (F = 0), no shared block (n_s = 0) and nothing free; a
rejected first trial on a gauge-singular system, after which exact mode relinearises at x.  Whole solves: the converged cost on a
gauge-singular blocked problem against scipy's tr_solver='exact', and two exact solves at cfg4's n_s bit for bit.
The bodies take the device's SM count as an argument so that tests/test_simt_exact_paths.py runs the cheap ones on the interpreter."""
import numpy as np
import pytest
from numpy.linalg import norm
from scipy import optimize
from scipy.optimize._numdiff import approx_derivative, group_columns

import test_gpu_blocked_cholesky as bc
import test_gpu_exact_trust_region as et
import test_gpu_parity as gp
import test_gpu_step_parity as sp
from multical_b200 import synthetic
from multical_b200.calibration import from_scene
from oracle.ba_oracle import Problem
from oracle.trf_exact_model import EPS, exact_first_step

pytestmark = pytest.mark.gpu

PIVOT_MARGIN, PHI_MARGIN, RTOL = 10.0, 1e-6, 0.01
DEFAULT_OPT = dict(camera_poses=True, board_poses=True, motion=True)


def num_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------- the check
def motion_cols(opt, C, B, fb, F):
  """The frame blocks k_lm eliminates, as indices of the parameter vector [camera_poses 6C | board_poses 6B | motion fb F | ...]
  (`opt`: the enabled blocks, Calibration's defaults where it says nothing)."""
  on = lambda k: opt.get(k, DEFAULT_OPT[k])
  off = (6 * C if on("camera_poses") else 0) + (6 * B if on("board_poses") else 0)
  return np.arange(off, off + fb * F) if on("motion") else np.arange(0)


def check_exact_step(eng, prob, label, frame_cols, shared_cols=None):
  """The first accepted step of an exact solve against the model on the device's normal equations at x0, trials that raise the
  oracle's cost rejected.  Returns the model's step."""
  x0 = eng.param_vec.copy()
  JtJ, Jtr, _ = eng.linearize()
  cost = lambda x: 0.5 * np.sum(prob.residuals(x) ** 2)
  m = exact_first_step(JtJ, Jtr, x0, frame_cols, shared_cols=shared_cols, cost=cost(x0), trial_cost=cost)
  pivots = f"min pivot/tol {m.pivot_min:.3g}" if m.full_rank else \
    f"smallest failing pivot/tol {m.pivot_bad_min:.3g}, smallest passing one before it {m.pivot_before_bad:.3g}"
  phi = min((abs(r - RTOL) for r in m.phi_ratios), default=np.inf)
  # a float64 solve is determined to ~eps cond(A + reg I) of its norm: where the search ends at reg ~ 1e-12 on a gauge-singular A
  # (cond ~ 1e12) two correct solves differ by ~1e-5 of the step, everywhere else the bars are 1e-9 / 1e-8
  bar, component_bar = max(sp.STEP_BAR, EPS * m.cond), max(sp.STEP_COMPONENT_BAR, EPS * m.cond)
  print(f"[exact step] {label}: {'full rank' if m.full_rank else 'rank-deficient'}, {pivots}, {m.iterations} alpha iterations over "
        f"{m.trials} trial(s), min | |phi|/Delta - 0.01 | {phi:.3g}, cond(A + reg I) {m.cond:.3g} (step bar {bar:.3g})")
  if m.full_rank: assert m.pivot_min >= PIVOT_MARGIN, (label, m.pivot_min)
  assert phi >= PHI_MARGIN, (label, m.phi_ratios)
  step, res = sp.device_first_step(eng, trials=m.trials, tr_solver="exact")
  sp.check_step(step, m.step, label, bar, component_bar)
  assert res.alpha_iterations == m.iterations, (label, res.alpha_iterations, m.iterations)
  assert res.chol_retries == 0, (label, res.chol_retries)
  # the rank decision as the step shows it: the Gauss-Newton step lies inside Delta, any other step on the boundary
  scale_inv = np.sqrt(np.diag(JtJ)).copy(); scale_inv[scale_inv == 0] = 1
  shn = norm(step * scale_inv)
  gauss_newton = m.iterations == 0
  if gauss_newton: assert shn <= m.Delta * (1 + 1e-12), (label, shn, m.Delta)
  else: assert abs(shn - m.Delta) <= 1e-12 * m.Delta, (label, shn, m.Delta)
  if not m.full_rank and not (m.pivot_bad_min <= 1.0 / PIVOT_MARGIN and m.pivot_before_bad >= PIVOT_MARGIN):
    # everything above holds, but the rank decision sits within a factor 10 of a tie: reported, not counted as a pass
    pytest.xfail(f"{label}: rank decision within a factor 10 of the tolerance (smallest failing pivot {m.pivot_bad_min:.3g} tol, "
                 f"smallest passing one before it {m.pivot_before_bad:.3g} tol)")
  return m


# ---------------------------------------------------------------------------------------------------------------- (a) reduced paths
def reduced_scene(n_s, F):
  """The scenes of tests/test_gpu_step_parity.py (n_s = 127, 128, 129, 160) and tests/test_gpu_blocked_cholesky.py (146, 286)."""
  if n_s in bc.SHAPES: return bc.scene_of(n_s, F)
  model, C, B, opt = sp.REDUCED[n_s]
  return synthetic.make_scene(C=C, F=F, vis=0.5, seed=29, model=model, rig="dome", boards=("cube", 4, 4, 0.06, B)), opt


def run_reduced_path(n_s, motion, F, sms):
  """(lm_grid, SYRK chunks, the model's step) of the first exact step at a reduced size."""
  fb = 12 if motion == "rolling" else 6
  scene, opt = reduced_scene(n_s, F)
  calib, prob = sp.static_or_rolling(scene, opt, motion=motion)
  eng, _ = sp.upload(calib, prob)
  assert eng.num_params - fb * F == n_s
  lm_grid, chunks = sp.lm_shape(F, n_s, fb, sms)
  m = check_exact_step(eng, prob, f"n_s={n_s} FB={fb} F={F} (lm_grid {lm_grid}, SYRK chunks {chunks})",
                       motion_cols(opt, scene["C"], scene["B"], fb, F))
  return lm_grid, chunks, m


REDUCED_SIZES = [127, 128, 129, 146, 160, 286]


@pytest.mark.parametrize("F", [6, 40])
@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("n_s", REDUCED_SIZES)
def test_exact_step_at_the_reduced_solve_paths(n_s, motion, F):
  """6 frames: an 8-CTA grid and one SYRK chunk; 40 frames: the whole machine and several chunks.  Free camera or board poses make
  every one of these probes rank-deficient (the gauge), read from the one-CTA factor at 127 and from the blocked factor above."""
  sms = num_sms()
  lm_grid, chunks = sp.lm_shape(F, n_s, 12 if motion == "rolling" else 6, sms)
  if F == 6: assert (lm_grid, chunks) == (8, 1)
  else: assert lm_grid == sms and chunks > 1
  *shape, m = run_reduced_path(n_s, motion, F, sms)
  assert tuple(shape) == (lm_grid, chunks) and not m.full_rank


# ---------------------------------------------------------------------------------------------------------------- (b) full rank, blocked
def full_rank_problem(F):
  """13 standard cameras' intrinsics (n_s = 13 x 10 = 130, a blocked probe; the 13 skew columns are dead), camera and board poses
  held: no gauge freedom."""
  scene = synthetic.make_scene(C=13, F=F, vis=0.6, seed=37, rig="dome", boards=("cube", 4, 4, 0.06, 2))
  opt = dict(cameras=True, camera_poses=False, board_poses=False)
  calib, prob = sp.static_or_rolling(scene, opt)
  return scene, opt, calib, prob


def run_full_rank_blocked(F, sms):
  scene, opt, calib, prob = full_rank_problem(F)
  eng, _ = sp.upload(calib, prob)
  n_s = eng.num_params - 6 * F
  assert n_s == 130
  JtJ, _, _ = eng.linearize()
  assert (np.diag(JtJ) == 0).sum() == 13
  lm_grid, chunks = sp.lm_shape(F, n_s, 6, sms)
  m = check_exact_step(eng, prob, f"full rank n_s={n_s} F={F} (lm_grid {lm_grid}, SYRK chunks {chunks})", motion_cols(opt, 13, 2, 6, F))
  assert m.full_rank and m.iterations == 0          # the Gauss-Newton step, inside Delta
  return m


def test_full_rank_blocked_probe_takes_the_gauss_newton_step():
  run_full_rank_blocked(6, num_sms())


def run_full_rank_search(F, sms):
  """The same problem from focal lengths a quarter of the true ones: the Gauss-Newton trial raises the cost, and the trials at the
  smaller radii run the full-rank alpha search on the blocked factor -- alpha_lower = -phi / phi' of the probe, phi' from `solve_again`
  at every iteration (its rhs summed per SYRK frame chunk), alpha warm-started across trials.  Returns (lm_grid, SYRK chunks)."""
  scene, opt, calib, prob = full_rank_problem(F)
  eng, x = sp.upload(calib, prob)
  k0 = x.size - 10 * 13                                  # standard model: [fx fy cx cy skew k1..k5] per camera, last in the vector
  for c in range(13): x[k0 + 10 * c:k0 + 10 * c + 2] *= 0.25
  eng.set_param_vec(x)
  lm_grid, chunks = sp.lm_shape(F, 130, 6, sms)
  m = check_exact_step(eng, prob, f"full-rank search n_s=130 F={F} (lm_grid {lm_grid}, SYRK chunks {chunks})",
                       motion_cols(opt, 13, 2, 6, F))
  assert m.full_rank and m.trials >= 2 and m.iterations > 0
  return lm_grid, chunks


@pytest.mark.parametrize("F", [6, 40])
def test_full_rank_blocked_alpha_search(F):
  """6 frames: an 8-CTA grid, one SYRK chunk; 40 frames: the whole machine, several chunks."""
  sms = num_sms()
  lm_grid, chunks = run_full_rank_search(F, sms)
  assert (lm_grid, chunks) == (8, 1) if F == 6 else (lm_grid == sms and chunks > 1)


# ---------------------------------------------------------------------------------------------------------------- (c) hand-eye
def run_hand_eye(F):
  """Hand-eye frames with free world_wrt_base / gripper_wrt_camera: k_lm sees no frame block (F = 0), the 12 hand-eye rows come from
  k_fold_hand_eye in batches of 64 frames.  The engine factors its shared columns as [board poses | intrinsics | hand-eye]."""
  assert F > sp.FOLD_FRAMES and F % sp.FOLD_FRAMES != 0
  scene = synthetic.make_scene(C=2, F=F, vis=0.8, seed=19, boards=("charuco", 6, 5, 0.08, 1))
  calib, prob = sp.hand_eye(scene, dict(camera_poses=False, cameras=True, boards=False))
  eng, _ = sp.upload(calib, prob)
  nb, n = 6 * scene["B"], eng.num_params
  shared = np.r_[np.arange(nb), np.arange(nb + 12, n), np.arange(nb, nb + 12)]
  return check_exact_step(eng, prob, f"hand-eye F={F} ({-(-F // sp.FOLD_FRAMES)} fold batches)", [], shared_cols=shared)


def test_exact_step_with_hand_eye_frames_beyond_one_fold_batch():
  run_hand_eye(150)


# ---------------------------------------------------------------------------------------------------------------- (d) degenerate
DEGENERATE = gp.test_degenerate_block_selections.pytestmark[0].args[1]


def run_degenerate(opt):
  """F = 0 (the rhs of the second solve is zero), n_s = 0 (a rank test over nothing), nothing free (one evaluation, no step)."""
  scene = synthetic.make_scene(C=2, F=6, vis=0.5, seed=91)
  calib = from_scene(scene).enable(**opt)
  prob = Problem.from_scene(scene, optimize=opt)
  if prob.param_vec.size == 0:
    res = calib._upload(calib.inliers).solve(tr_solver="exact")
    assert res.nfev == 1 and res.alpha_iterations == 0 and res.chol_retries == 0
    return None
  eng, _ = sp.upload(calib, prob)
  return check_exact_step(eng, prob, f"degenerate {opt}", motion_cols(calib.optimize, 2, scene["B"], 6, 6))


@pytest.mark.parametrize("opt", DEGENERATE)
def test_exact_step_at_degenerate_block_selections(opt):
  run_degenerate(opt)


# ---------------------------------------------------------------------------------------------------------------- (e) rejection
def run_rejected_first_trial(n_s=146, F=6, scale=0.3):
  """From intrinsics 30 % off (focal lengths, principal points) the first trial raises the cost; exact mode relinearises at x and
  solves again at the smaller radius with alpha scaled by Delta / Delta_new.  The accepted second trial against the model with the
  oracle's cost."""
  scene, opt = reduced_scene(n_s, F)
  calib, prob = sp.static_or_rolling(scene, opt)
  eng = upload_perturbed(calib, prob, scale)
  m = check_exact_step(eng, prob, f"rejected first trial n_s={n_s} F={F}", motion_cols(opt, scene["C"], scene["B"], 6, F))
  assert m.trials >= 2
  return m


def upload_perturbed(calib, prob, scale):
  eng, x0 = sp.upload(calib, prob)
  C = len(calib.cameras)
  x = x0.copy()
  k0 = x0.size - 10 * C                                  # standard model: [fx fy cx cy skew k1..k5] per camera, last in the vector
  for c in range(C):
    x[k0 + 10 * c:k0 + 10 * c + 4] *= 1 + scale * (-1) ** c
  eng.set_param_vec(x)
  return eng


def test_rejected_first_trial_relinearises():
  run_rejected_first_trial()


# ---------------------------------------------------------------------------------------------------------------- (f) whole solves
def run_gauge_singular_converged(tolerance=1e-13):
  """n_s = 150 (nine cameras with intrinsics, free camera and board poses: the scene of test_many_cameras_use_the_cooperative_blocked_
  reduced_solve): the converged cost of the exact solve within 1e-8 relative of scipy's exact trust region."""
  scene = synthetic.make_scene(C=9, F=4, vis=0.12, seed=11, rig="dome")
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-14, xtol=1e-14, gtol=1e-14,
                               max_nfev=300, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=tolerance, xtol=tolerance, gtol=tolerance, max_iterations=200, tr_solver="exact")
  res = out.last_solve
  print(f"[gauge-singular n_s=150] exact {res.cost!r} ({res.nfev} nfev, {res.alpha_iterations} alpha iterations), scipy {ref.cost!r}")
  assert abs(res.cost - ref.cost) <= 1e-8 * ref.cost, (res.cost, ref.cost)
  assert res.chol_retries == 0


def test_gauge_singular_blocked_solve_converges_to_scipys_cost():
  run_gauge_singular_converged()


def run_exact_bit_reproducible(n_s, F, max_iterations=6):
  scene, opt = reduced_scene(n_s, F)
  calib, _ = sp.static_or_rolling(scene, opt)
  a, b = (et.solve_arrays(calib.bundle_adjust(tolerance=1e-9, max_iterations=max_iterations, tr_solver="exact")) for _ in range(2))
  et.same_bits(a, b)


def test_exact_solves_at_cfg4s_size_are_bit_reproducible():
  run_exact_bit_reproducible(286, 40)
