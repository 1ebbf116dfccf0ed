"""GPU (-m gpu): the first trust-region step and the normal equations against float64 references, at the shapes where the kernels
switch paths.

A trust-region method converges even when its Gauss-Newton direction is slightly wrong (the 2-D subspace also holds the gradient),
so a wrong reduced solve shows up as extra iterations, not as a wrong converged cost.  These tests therefore compare the pieces
directly:
  normal equations  J^T J, J^T r, cost of `linearize` against fourth-order central differences of the oracle's residuals
                    (`fd5_jacobian`, noise ~1e-11): H <= 1e-9 (entries over sqrt(H_ii H_jj)), g <= 1e-10 max|g|, cost <= 1e-12
  first step        x1 - x0 of a solve that stops after its first (accepted) trial, against `oracle.trf_exact_model.first_step`
                    on the device's own normal equations at x0: <= 1e-9 relative in norm, <= 1e-8 per component over max|step|
                    (robust losses: the model's normal equations come from `fd5_jacobian`, bar 1e-8)
The paths: views whose corner count ends a 32-corner chunk while several warps share a view (`split` > 1), CTAs of k_linearize that
own several frames, k_fold_hand_eye over more than one batch of frames, the one-CTA and the blocked Cholesky of the reduced system
at their boundaries (n_s = 127 / 128 / 129 / 160) with one and several SYRK frame chunks, and the robust losses.

The test bodies take the device's SM count as an argument so that tests/test_simt_kernels.py runs the cheap shapes on the
interpreter with the same code.
"""
import numpy as np
import pytest
from scipy.optimize._lsq.least_squares import construct_loss_function
from scipy.optimize._numdiff import group_columns

from multical_b200 import synthetic
from multical_b200.calibration import from_scene
from multical_b200.motion import HandEye, RollingFrames
from multical_b200.pose_set import pose_table
from oracle.ba_oracle import Problem
from oracle.trf_exact_model import first_step

pytestmark = pytest.mark.gpu

H_BAR, G_BAR, COST_BAR = 1e-9, 1e-10, 1e-12
STEP_BAR, STEP_COMPONENT_BAR = 1e-9, 1e-8
LIN_WARPS = 8                 # warps of a k_linearize CTA when several warps share a view (csrc/linearize.cuh)


# ---------------------------------------------------------------------------------------------------------------- references
def fd5_jacobian(prob, x, rel_step=1e-3):
  """Fourth-order central differences of `prob.residuals` at x on the oracle's sparsity pattern, one column group of
  `group_columns` at a time (four evaluations per group): f'(x) = (8 (f(x+h) - f(x-h)) - (f(x+2h) - f(x-2h))) / 12h with
  h = rel_step * max(1, |x_i|).  Returns a scipy.sparse CSC matrix (rows x columns of the sparsity matrix)."""
  x = np.asarray(x, np.float64)
  S = prob.sparsity_matrix().tocoo()
  groups = group_columns(S.tocsc())
  h = rel_step * np.maximum(1.0, np.abs(x))
  rows, cols = S.row, S.col
  vals = np.zeros(rows.size)
  entry_group = groups[cols]
  order = np.argsort(entry_group, kind="stable")
  bounds = np.searchsorted(entry_group[order], np.arange(groups.max() + 2))
  for k in range(groups.max() + 1):
    sel = order[bounds[k]:bounds[k + 1]]
    if sel.size == 0: continue
    e = np.zeros_like(x); e[groups == k] = h[groups == k]
    df = 8.0 * (prob.residuals(x + e) - prob.residuals(x - e)) - (prob.residuals(x + 2 * e) - prob.residuals(x - 2 * e))
    vals[sel] = df[rows[sel]] / (12.0 * h[cols[sel]])
  from scipy.sparse import csc_matrix
  return csc_matrix((vals, (rows, cols)), shape=S.shape)


def normalised_h_error(A, B, rows=2048):
  """max |A - B| / sqrt(B_ii B_jj) over the entries with a non-zero normaliser, in row blocks (dense n x n temporaries of the
  large scenes would not fit twice)."""
  d = np.sqrt(np.diag(B))
  worst = 0.0
  for i0 in range(0, A.shape[0], rows):
    nrm = d[i0:i0 + rows, None] * d[None, :]
    live = nrm > 0
    if live.any(): worst = max(worst, float((np.abs(A[i0:i0 + rows] - B[i0:i0 + rows])[live] / nrm[live]).max()))
  return worst


def check_normal_equations(JtJ, Jtr, cost, J, r, label):
  """Device normal equations against J^T J, J^T r, r^T r / 2 of a finite-difference Jacobian J.  Returns the errors."""
  H = (J.T @ J).toarray()
  g = J.T @ r
  ref_cost = 0.5 * r @ r
  eH = normalised_h_error(JtJ, H)
  eg = float(np.abs(Jtr - g).max() / np.abs(g).max())
  ec = abs(cost - ref_cost) / ref_cost
  print(f"[normal equations] {label}: H {eH:.2e}  g {eg:.2e}  cost {ec:.2e}")
  assert eH <= H_BAR, (label, eH)
  assert eg <= G_BAR, (label, eg)
  assert ec <= COST_BAR, (label, ec)
  dead = np.sqrt(np.diag(H)) == 0
  assert np.abs(JtJ[dead]).max(initial=0.0) == 0.0                    # dead columns (skew, invalid poses) stay exactly zero
  return eH, eg, ec


def device_first_step(eng, trials=1, **solve_kw):
  """x1 - x0 of a solve stopped after `trials` trials, of which the log must show the last one accepted (trf shrinks the trust region
  and tries again after a trial that does not lower the cost).  The engine is put back at x0."""
  x0 = eng.param_vec.copy()
  res = eng.solve(max_nfev=trials + 1, ftol=1e-12, xtol=1e-12, gtol=1e-12, **solve_kw)
  assert res.nfev == trials + 1 and len(res.log) == 2 and res.log[1][3] > 0, res.log      # the last trial accepted
  step = eng.param_vec - x0
  eng.set_param_vec(x0)
  assert abs(np.linalg.norm(step) - res.log[1][4]) <= 1e-9 * res.log[1][4]
  return step, res


def check_step(step, ref, label, bar=STEP_BAR, component_bar=STEP_COMPONENT_BAR):
  en = float(np.linalg.norm(step - ref) / np.linalg.norm(ref))
  ec = float(np.abs(step - ref).max() / np.abs(ref).max())
  print(f"[first step] {label}: norm {en:.2e}  component {ec:.2e}  (|step| {np.linalg.norm(ref):.3e})")
  assert en <= bar, (label, en)
  assert ec <= component_bar, (label, ec)
  return en, ec


def check_device_step(eng, label):
  """First step of the device against the model on the device's own normal equations at x0."""
  x0 = eng.param_vec.copy()
  JtJ, Jtr, _ = eng.linearize()
  ref = first_step(JtJ, Jtr, x0)
  step, _ = device_first_step(eng)
  return check_step(step, ref, label)


def lm_shape(F_free, n_s, fb, num_sms):
  """(lm_grid, syrk_chunks) of the persistent trust-region kernel as the host driver picks them (csrc/solver.cu): the whole machine
  once F * n_s >= 4096, else 8 CTAs; frame chunks of the Schur SYRK in whole steps of 48 / fb frames, at most one per CTA per tile
  pair of the 32-row tiles."""
  lm_grid = num_sms if max(F_free, 1) * max(n_s, 1) >= 4096 else max(1, min(num_sms, 8))
  fr = 48 // fb
  tiles = -(-max(n_s, 1) // 32)
  npair = tiles * (tiles + 1) // 2
  chunks = max(1, min(-(-F_free // fr), lm_grid // max(1, npair)))
  cf = max(fr, -(-(-(-max(F_free, 1) // chunks)) // fr) * fr)
  return lm_grid, max(1, -(-F_free // cf))


# ---------------------------------------------------------------------------------------------------------------- problems
def static_or_rolling(scene, opt, motion="static", seed=7):
  """(Calibration, oracle Problem) of a synthetic scene; rolling frames end 1e-3 away from where they start."""
  if motion == "static":
    return from_scene(scene).enable(**opt), Problem.from_scene(scene, optimize=opt)
  start = scene["init"]["frame_poses"]
  end = synthetic.to_matrix(synthetic.from_matrix(start) + 1e-3 * np.random.default_rng(seed).standard_normal((scene["F"], 6)))
  prob = Problem.from_scene(scene, optimize=opt, motion="rolling", frame_poses_end=end, image_size=scene["image_size"])
  frames = RollingFrames(start, end, scene["frame_valid"], [str(i) for i in range(scene["F"])])
  return from_scene(scene).copy(motion=frames).enable(**opt), prob


def hand_eye(scene, opt):
  """Hand-eye frames with non-identity world_wrt_base W and gripper_wrt_camera G; the arm poses G^-1 T_f W^-1 make the derived
  frames G A_f W the scene's frames T_f."""
  W = synthetic.to_matrix([0.1, -0.2, 0.3, 0.05, -0.02, 0.4])[0]
  G = synthetic.to_matrix([-0.2, 0.1, 0.05, 0.03, 0.06, -0.1])[0]
  T = scene["init"]["frame_poses"]
  arm = np.linalg.inv(G)[None] @ T @ np.linalg.inv(W)[None]
  prob = Problem.from_scene(scene, optimize=opt, motion="hand_eye", base_wrt_gripper=arm, world_wrt_base=W, gripper_wrt_camera=G)
  assert np.abs(prob.frame_poses - T).max() < 1e-12
  calib = from_scene(scene).copy(motion=HandEye(pose_table(arm, scene["frame_valid"]), W, G)).enable(**opt)
  return calib, prob


def upload(calib, prob):
  eng = calib._upload(calib.inliers)
  x0 = prob.param_vec
  assert eng.num_params == x0.size and np.abs(eng.param_vec - x0).max() <= 1e-12 * max(1.0, np.abs(x0).max())
  return eng, x0


def check_linearisation_and_step(calib, prob, label):
  eng, x0 = upload(calib, prob)
  JtJ, Jtr, cost = eng.linearize()
  check_normal_equations(JtJ, Jtr, cost, fd5_jacobian(prob, x0), prob.residuals(x0), label)
  ref = first_step(JtJ, Jtr, eng.param_vec)
  step, _ = device_first_step(eng)
  check_step(step, ref, label)
  return eng


# ---------------------------------------------------------------------------------------------------------------- (a) chunk tails
CHUNK_TAIL_COUNTS = (1, 31, 32, 33, 64, 65)


def chunk_tail_scene(C):
  """Two 10 x 9 charuco boards (72 corners each); every camera sees board 0 in each frame with exactly 1, 31, 32, 33, 64 or 65
  corners (each count once per camera), board 1 whole, which keeps every frame pose determined."""
  scene = synthetic.make_scene(C=C, F=len(CHUNK_TAIL_COUNTS), vis=1.0, seed=13, boards=("charuco", 10, 9, 0.05, 2))
  valid = scene["valid"]
  assert scene["P"] >= 65
  for c in range(C):
    for f in range(scene["F"]):
      n = CHUNK_TAIL_COUNTS[(f + c) % len(CHUNK_TAIL_COUNTS)]
      on = np.flatnonzero(valid[c, f, 0])
      assert on.size >= n, (c, f, on.size, n)
      valid[c, f, 0, on[n:]] = False
  counts = valid[:, :, 0].sum(axis=-1)
  assert all(sorted(counts[c]) == sorted(CHUNK_TAIL_COUNTS) for c in range(C))
  return scene


def lin_split(C):
  """Warps that share a view in k_linearize (csrc/solver.cu): doubled while C * split * 2 <= 8."""
  split = 1
  while split < LIN_WARPS and C * split * 2 <= LIN_WARPS: split *= 2
  return split


def run_chunk_tails(C):
  """Views of 1, 31, 32, 33, 64 and 65 corners: a view's corners run in 32-corner chunks, chunk `sub` of `split` warps starting at
  beg + 32 * sub with stride 32 * split, so these counts end a chunk just before, at and after a chunk boundary, on a warp that is
  not the view's first."""
  scene = chunk_tail_scene(C)
  calib, prob = static_or_rolling(scene, dict(cameras=True))
  check_linearisation_and_step(calib, prob, f"chunk tails C={C} split={lin_split(C)}")


@pytest.mark.parametrize("C, split", [(1, 8), (2, 4), (3, 2), (5, 1)])
def test_views_that_end_a_corner_chunk_under_a_split_view(C, split):
  """Split views (one camera: 8 warps share a view, 2: 4, 3: 2) and the unsplit path (5 cameras), views of 1, 31, 32, 33, 64, 65
  corners: normal equations against fd5_jacobian, first step against the model."""
  assert lin_split(C) == split
  run_chunk_tails(C)


# ---------------------------------------------------------------------------------------------------------------- (b) frames per CTA
def run_frames_per_cta(motion, F, num_sms):
  """k_linearize maps frames to CTAs statically: at most 2 CTAs of 8 warps are resident per SM, so the grid is the smallest one that
  keeps every CTA at ceil(F / (2 * num_SMs)) frames (csrc/solver.cu), and CTA b owns frames b, b + grid, b + 2 grid, ...  The next
  frame's pose table is fetched by a bulk copy into the other of two buffers while the CTA works on the current one (mbarrier phase
  parity per buffer), and the CTA's shared records sum over its frames.  Returns (grid, frames of the fullest CTA)."""
  scene = synthetic.make_scene(C=2, F=F, vis=0.9, seed=17, boards=("charuco", 6, 5, 0.08, 1))
  calib, prob = static_or_rolling(scene, dict(cameras=True), motion=motion)
  per = -(-F // (2 * num_sms))
  grid = -(-F // per)
  assert lin_split(2) > 1 and per >= 3                            # every CTA owns several frames
  check_linearisation_and_step(calib, prob, f"frames per CTA {motion} F={F} (grid {grid}, {F // grid}-{per} frames per CTA)")
  return grid, per


@pytest.mark.parametrize("motion", ["static", "rolling"])
def test_ctas_that_own_several_frames(motion):
  """F = 3 * 2 * num_SMs + 5 (797 on 132 SMs): 2 resident CTAs of 8 warps per SM allow 264, ceil(797 / 264) = 4 frames per CTA give a
  grid of ceil(797 / 4) = 200 CTAs: 197 own 4 frames, the last 3 own 3.  Static and rolling frames, 2 cameras (4 warps share a view)."""
  import torch
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  F = 3 * 2 * num_sms + 5
  grid, per = run_frames_per_cta(motion, F, num_sms)
  assert F % grid != 0                                            # CTAs that own fewer frames than the others


# ---------------------------------------------------------------------------------------------------------------- (c) hand-eye folds
FOLD_FRAMES = 64              # frames per batch of k_fold_hand_eye (csrc/linearize.cuh)


def run_hand_eye_folds(F, boards):
  """k_fold_hand_eye folds the per-frame blocks into the 12 hand-eye rows in batches of 64 frames."""
  assert F > FOLD_FRAMES and F % FOLD_FRAMES != 0
  scene = synthetic.make_scene(C=2, F=F, vis=0.8, seed=19, boards=("charuco", 6, 5, 0.08, 1))
  opt = dict(camera_poses=False, cameras=True, boards=boards)
  calib, prob = hand_eye(scene, opt)
  eng = calib._upload(calib.inliers)
  x0 = prob.param_vec
  keep = np.ones(eng.num_params, bool)
  if boards: keep[-calib._board_block_slices().size:] = calib._board_block_slices()    # padded board slots have no oracle column
  assert keep.sum() == x0.size and np.abs(eng.param_vec[keep] - x0).max() <= 1e-12 * np.abs(x0).max()
  JtJ, Jtr, cost = eng.linearize()
  label = f"hand-eye F={F} ({-(-F // FOLD_FRAMES)} fold batches) boards={boards}"
  check_normal_equations(JtJ[np.ix_(keep, keep)], Jtr[keep], cost, fd5_jacobian(prob, x0), prob.residuals(x0), label)
  check_step(device_first_step(eng)[0], first_step(JtJ, Jtr, eng.param_vec), label)


@pytest.mark.parametrize("boards", [False, True])
def test_hand_eye_beyond_one_fold_batch(boards):
  """150 frames = fold batches of 64 + 64 + 22, non-identity hand-eye transforms, board points fixed and free."""
  run_hand_eye_folds(150, boards)


# ---------------------------------------------------------------------------------------------------------------- (d) reduced solve
REDUCED = {   # n_s: (model, cameras, boards, enabled blocks) -- n_s = shared parameters of the Schur complement
  127: ("rational", 7, 6, dict(cameras=True, camera_poses=False)),      # 13 * 7 + 6 * 6: the largest one-CTA register Cholesky
  128: ("standard", 8, 2, dict(cameras=True, board_poses=False)),       # 16 * 8: the first blocked size, 4 whole panels
  129: ("fisheye", 7, 4, dict(cameras=True)),                           # 15 * 7 + 6 * 4: blocked, a last panel of one row
  160: ("standard", 10, 2, dict(cameras=True, board_poses=False)),      # 16 * 10: blocked, 5 whole panels
}


def run_reduced_solve(n_s, motion, F, num_sms, converge=False):
  model, C, B, opt = REDUCED[n_s]
  fb = 12 if motion == "rolling" else 6
  scene = synthetic.make_scene(C=C, F=F, vis=0.5, seed=29, model=model, rig="dome", boards=("cube", 4, 4, 0.06, B))
  calib, prob = static_or_rolling(scene, opt, motion=motion)
  eng, x0 = upload(calib, prob)
  assert eng.num_params - fb * F == n_s
  lm_grid, chunks = lm_shape(F, n_s, fb, num_sms)
  label = f"n_s={n_s} FB={fb} F={F} (lm_grid {lm_grid}, SYRK chunks {chunks})"
  check_device_step(eng, label)
  if converge:
    from scipy import optimize
    from scipy.optimize._numdiff import approx_derivative
    S = prob.sparsity_matrix(); groups = group_columns(S)
    jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
    ref = optimize.least_squares(prob.residuals, x0, jac=jac, x_scale="jac", ftol=1e-13, xtol=1e-13, gtol=1e-13,
                                 max_nfev=200, method="trf", tr_solver="exact")
    out = calib.bundle_adjust(tolerance=1e-13, xtol=1e-13, gtol=1e-13, max_iterations=200)
    assert abs(out.last_solve.cost - ref.cost) <= 1e-8 * ref.cost, (out.last_solve.cost, ref.cost)
  return lm_grid, chunks


@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("n_s", sorted(REDUCED))
def test_reduced_solve_at_the_cholesky_boundaries(n_s, motion):
  """The one-CTA register Cholesky up to n_s = 127, the blocked cooperative one (32-wide panels, look-ahead tile, inverted
  diagonal blocks) from 128, with a ragged last panel at 129 and whole tiles at 160; frames of 6 (static) and 12 (rolling) parameters.
  6 frames: F * n_s < 4096, an 8-CTA grid and one SYRK chunk (plus the converged cost against scipy's dense exact trust region at
  129; the 128 scene, intrinsics of 8 cameras from 9-corner boards, is too ill-conditioned for two trust-region runs to end at the same
  cost); 40 frames: the whole machine and several SYRK chunks."""
  import torch
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  assert run_reduced_solve(n_s, motion, 6, num_sms, converge=n_s == 129) == (8, 1)
  lm_grid, chunks = run_reduced_solve(n_s, motion, 40, num_sms)
  assert lm_grid == num_sms and chunks > 1


# ---------------------------------------------------------------------------------------------------------------- (e) robust losses
def run_robust_loss(loss, f_scale=2.0):
  """Under a robust loss the solver works on Triggs-scaled normal equations: J_scale = max(rho' + 2 rho'' z, 0.1 rho', eps) per
  residual (DESIGN.md §2), g = J^T (rho' r).  The model builds them from fd5_jacobian and scipy's own rho.  From x0 the full
  Gauss-Newton trial overshoots on these scenes, so the compared step is the first accepted one, after the trust region shrank."""
  scene = synthetic.make_scene(C=2, F=6, vis=0.5, seed=31, outlier_fraction=0.03)
  calib, prob = static_or_rolling(scene, dict(cameras=True))
  eng, x0 = upload(calib, prob)
  r = prob.residuals(x0)
  loss_function = construct_loss_function(r.size, loss, f_scale)
  rho = loss_function(r)
  J_scale = np.maximum(np.maximum(rho[1] + 2 * rho[2] * r ** 2, 0.1 * rho[1]), np.finfo(float).eps)
  J = fd5_jacobian(prob, x0)
  H = (J.multiply(J_scale[:, None]).tocsc().T @ J).toarray()
  g = J.T @ (rho[1] * r)
  cost0 = 0.5 * rho[0].sum()
  ref, trials = first_step(H, g, x0, cost=cost0, trial_cost=lambda x: loss_function(prob.residuals(x), cost_only=True))
  step, res = device_first_step(eng, trials=trials, loss=loss, f_scale=f_scale)
  ec = abs(res.log[0][2] - cost0) / cost0
  print(f"[robust initial cost] {loss}: {ec:.2e}")
  assert ec <= 1e-12, (res.log[0][2], cost0)
  check_step(step, ref, f"robust {loss} ({trials} trials)", bar=1e-8, component_bar=1e-8)


@pytest.mark.parametrize("loss", ["soft_l1", "huber", "cauchy", "arctan"])
def test_first_step_under_a_robust_loss(loss):
  """soft_l1, huber, cauchy, arctan at f_scale = 2 on a scene with 3 % gross outliers."""
  run_robust_loss(loss)
