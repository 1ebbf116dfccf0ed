"""GPU (-m gpu): the CUDA path through the C-ABI against the oracle and the golden vectors.

Tolerances (all fp64 on the device):
  indexing / parameter layout ........ bit exact
  residuals at identical x ........... <= 1e-9 px       (observed ~5e-13)
  J^T J, J^T r vs oracle 5-point FD .. J^T J <= 1e-9 over sqrt(H_ii H_jj), J^T r <= 1e-10 max|J^T r| (FD noise ~1e-11)
  converged cost vs dense exact-TR oracle (scipy tr_solver='exact', tight tolerances) <= 1e-8 relative
  gauge-normalised converged parameters vs the same oracle: intrinsics rel 1e-6, poses 1e-6
  final cost at the reference's default tolerance: never worse than the reference's own result (+1e-6 rel)
"""
import numpy as np
import pytest
from scipy import optimize
from scipy.optimize._numdiff import approx_derivative, group_columns

from conftest import GOLDEN_CASES, load_golden, optimize_of
from multical_b200 import synthetic
from multical_b200.calibration import from_scene, select_threshold
from oracle.ba_oracle import Problem, matrix_to_rtvec
from test_gpu_step_parity import fd5_jacobian

pytestmark = pytest.mark.gpu


def make(name):
  scene, z = load_golden(name)
  calib = from_scene(scene)
  if bool(z["cameras_enabled"]): calib = calib.enable(cameras=True)
  return scene, z, calib, Problem.from_scene(scene, optimize=optimize_of(z))


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_residuals_match_reference_golden_and_oracle(name):
  scene, z, calib, prob = make(name)
  eng = calib._upload(calib.inliers)
  assert eng.N == z["r0"].size // 2
  assert np.abs(eng.param_vec - z["x0"]).max() < 1e-13                # layout exact; values converted on the device
  eng.set_params(*calib._state_arrays())                               # the rtvec entry point takes the host's own conversion
  assert np.array_equal(eng.param_vec, z["x0"])                       # -> bit exact
  r0 = eng.residuals()
  assert np.abs(r0 - z["r0"]).max() < 1e-9                            # vs the running reference
  r1, cost = eng.residuals(z["x1"], with_cost=True)
  assert np.abs(r1 - z["r1"]).max() < 1e-9
  assert np.abs(r1 - prob.residuals(z["x1"])).max() < 1e-9           # vs the oracle
  assert abs(cost - 0.5 * z["r1"] @ z["r1"]) <= 1e-12 * cost
  assert np.array_equal(eng.param_vec, z["x0"])                       # evaluating at x1 must not move the state
  err = eng.reprojection_error()
  assert np.abs(err - np.linalg.norm(z["r0"].reshape(-1, 2), axis=1)).max() < 1e-9


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_reprojection_error_over_valid(name):
  scene, z, calib, prob = make(name)
  assert np.abs(calib.reprojection_error - z["err_valid"]).max() < 1e-9


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_normal_equations_match_finite_differences(name):
  scene, z, calib, prob = make(name)
  eng = calib._upload(calib.inliers)
  x1 = z["x1"]
  J = fd5_jacobian(prob, x1)
  r = prob.residuals(x1)
  H, g = (J.T @ J).toarray(), J.T @ r
  JtJ, Jtr, cost = eng.linearize(x1)
  nrm = np.sqrt(np.outer(np.diag(H), np.diag(H)))
  live = nrm > 0
  # fisheye k4 (theta^9) is so weakly excited (H_ii ~ 1e-2) that the rounding of the pixel values (~1e-13 px) over the difference step
  # already moves its finite-difference entries by ~1e-9 of sqrt(H_ii H_jj)
  assert (np.abs(JtJ - H)[live] / nrm[live]).max() < (3e-9 if name == "fisheye_3x5" else 1e-9)
  assert np.abs(JtJ[~live]).max(initial=0.0) == 0.0                   # dead columns (skew, invalid poses) stay exactly zero
  assert np.abs(Jtr - g).max() < 1e-10 * np.abs(g).max()
  assert abs(cost - 0.5 * r @ r) < 1e-12 * cost
  assert np.abs(JtJ - JtJ.T).max() <= 1e-12 * np.abs(JtJ).max()


def gauge_normalised(cam_poses, frame_poses, board_poses):
  """camera 0 and board 0 as the two free gauges (calibration.py:99-112 `with_master`)."""
  G = cam_poses[0]; Hb = board_poses[0]
  cams = cam_poses @ np.linalg.inv(G)
  frames = G @ frame_poses @ Hb
  boards = np.linalg.inv(Hb) @ board_poses
  return matrix_to_rtvec(cams), matrix_to_rtvec(frames), matrix_to_rtvec(boards)


@pytest.mark.parametrize("name", ["standard_2x6", "fisheye_3x5", "cube3_3x6", "poses_only_2x6", "invalid_poses_3x6"])
def test_converged_solution_matches_dense_exact_oracle(name):
  scene, z, calib, prob = make(name)
  # tight-tolerance oracle: scipy dense exact trust region on the oracle residual with a 3-point Jacobian
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-14, xtol=1e-14, gtol=1e-14,
                               max_nfev=300, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=1e-13, xtol=1e-13, gtol=1e-13, max_iterations=200)
  res = out.last_solve
  assert abs(res.cost - ref.cost) <= 1e-8 * ref.cost, (res.cost, ref.cost)
  # at default tolerance the GPU solve must not be worse than what the reference reached
  quick = calib.bundle_adjust()
  assert quick.last_solve.cost <= float(z["ba_cost"]) * (1 + 1e-6)
  assert quick.last_solve.status in (1, 2, 3, 4)
  # gauge-normalised parameters
  o = prob.with_param_vec(ref.x)
  a = gauge_normalised(out.camera_poses.poses, out.motion.poses, out.board_poses.poses)
  b = gauge_normalised(o.cam_poses, o.frame_poses, o.board_poses)
  ok_c, ok_f, ok_b = scene["cam_valid"], scene["frame_valid"], scene["board_valid"]
  if ok_c[0] and ok_b[0]:
    assert np.abs(a[0][ok_c] - b[0][ok_c]).max() < 1e-6
    assert np.abs(a[1][ok_f] - b[1][ok_f]).max() < 1e-6
    assert np.abs(a[2][ok_b] - b[2][ok_b]).max() < 1e-6
  if bool(z["cameras_enabled"]):
    Kg = np.stack([c.intrinsic for c in out.cameras]); dg = np.stack([np.ravel(c.dist) for c in out.cameras])
    # K[0,1] (skew) is a dead parameter (cv2 ignores it): it must come back exactly as it went in; scipy's dense
    # SVD step lets it drift by numerical noise, so it is excluded from the comparison with that oracle
    assert all(c.intrinsic[0, 1] == 0.0 for c in out.cameras)
    Kg[:, 0, 1] = o.K[:, 0, 1]
    assert np.abs(Kg - o.K)[ok_c].max() < 1e-6 * 1000.0
    if scene["model"] != "fisheye":      # fisheye k3,k4 (theta^7, theta^9) are too weakly determined to compare directly
      assert np.abs(dg - o.dist.reshape(dg.shape))[ok_c].max() < 1e-5
  # gauge-free check that covers every parameter: both solutions project every valid corner to the same pixel
  uv_o, _ = o.reprojected()
  assert np.abs(out.projected.points - uv_o)[calib.valid].max() < 1e-4
  # invalid poses must come back untouched (empty Jacobian columns, parameters.py:145-147)
  assert np.allclose(out.camera_poses.poses[~ok_c], calib.camera_poses.poses[~ok_c], atol=1e-12)
  assert np.allclose(out.motion.poses[~ok_f], calib.motion.poses[~ok_f], atol=1e-12)


def test_many_cameras_use_the_cooperative_blocked_reduced_solve():
  """n_s > 128 (BASELINE configs[3], configs[4]: 16 and 64 cameras): the reduced system is factored by the grid (32-wide panels, diagonal
  blocks by one warp, csrc/lm_kernel.cuh) instead of by one CTA.  Nine cameras with their intrinsics give n_s = 54 + 6 + 90 = 150:
  normal equations against finite differences of the oracle, converged cost against scipy's dense exact trust region, and two
  identical solves must agree bit for bit (no atomics on data anywhere on this path)."""
  from multical_b200 import synthetic
  scene = synthetic.make_scene(C=9, F=4, vis=0.12, seed=11, rig="dome")
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  eng = calib._upload(calib.inliers)
  assert eng.num_params == prob.param_vec.size and 6 * 9 + 6 + 10 * 9 == 150
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-14, xtol=1e-14, gtol=1e-14,
                               max_nfev=300, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=1e-13, xtol=1e-13, gtol=1e-13, max_iterations=200)
  assert abs(out.last_solve.cost - ref.cost) <= 1e-8 * ref.cost, (out.last_solve.cost, ref.cost)
  a, b = calib.bundle_adjust().last_solve, calib.bundle_adjust().last_solve
  assert a.cost == b.cost and np.array_equal(np.array(a.log, float), np.array(b.log, float), equal_nan=True) and a.chol_retries == 0


def test_frame_count_that_ends_a_syrk_chunk_in_a_partial_step():
  """The Schur SYRK stages 8 frames per step in a 4-stage ring: a chunk whose frame count is not a multiple of 8 ends in a partial step,
  and after more than 4 steps that step lands in a stage that still holds an earlier step's frames behind its own (75 frames, 2 chunks:
  40 + 35 -> the second chunk's 5th step holds 3 frames).  Converged cost against scipy's dense exact trust region."""
  from multical_b200 import synthetic
  scene = synthetic.make_scene(C=2, F=75, vis=0.2, seed=23)
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-13, xtol=1e-13, gtol=1e-13,
                               max_nfev=200, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=1e-13, xtol=1e-13, gtol=1e-13, max_iterations=200)
  assert abs(out.last_solve.cost - ref.cost) <= 1e-8 * ref.cost, (out.last_solve.cost, ref.cost)


def test_sixty_four_cameras_configs4_shape():
  """BASELINE configs[4]'s shape (64-camera dome, one board, cameras + intrinsics optimised: n_s = 6*64 + 6 + 10*64 = 1030, 33 panels of
  the cooperative factorisation, eight cameras per warp of the linearisation) at a frame count the dense oracle can hold: converged cost
  against scipy's exact trust region on the oracle's residuals, bit-identical repeat."""
  from multical_b200 import synthetic
  scene = synthetic.make_scene(C=64, F=4, vis=0.10, seed=5, rig="dome")
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  eng = calib._upload(calib.inliers)
  assert eng.num_params == prob.param_vec.size and eng.num_params - 6 * 4 == 1030
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-12, xtol=1e-12, gtol=1e-12,
                               max_nfev=60, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=1e-12, xtol=1e-12, gtol=1e-12, max_iterations=60)
  assert abs(out.last_solve.cost - ref.cost) <= 1e-8 * ref.cost, (out.last_solve.cost, ref.cost)
  a, b = calib.bundle_adjust().last_solve, calib.bundle_adjust().last_solve
  assert a.cost == b.cost and np.array_equal(np.array(a.log, float), np.array(b.log, float), equal_nan=True)


def test_two_identical_solves_agree_bit_for_bit():
  """The reference is bit-reproducible run to run (single-threaded numpy / scipy, calibration.py:204-212).  So is this engine on the
  standard path: fixed-order sums everywhere (per-CTA records, frame-chunk partials, rank-ordered exchanges), no atomics on data."""
  scene, z, calib, prob = make("cube3_3x6")
  runs = [calib.bundle_adjust(tolerance=1e-9, max_iterations=30) for _ in range(3)]
  for r in runs[1:]:
    assert r.last_solve.cost == runs[0].last_solve.cost
    assert np.array_equal(np.array(r.last_solve.log, float), np.array(runs[0].last_solve.log, float), equal_nan=True)
    assert np.array_equal(r.param_vec, runs[0].param_vec)
  eng = calib._upload(calib.inliers)
  H0, g0, c0 = eng.linearize(z["x1"])
  H1, g1, c1 = eng.linearize(z["x1"])
  assert np.array_equal(H0, H1) and np.array_equal(g0, g1) and c0 == c1


@pytest.mark.parametrize("loss", ["soft_l1", "huber", "cauchy", "arctan"])
def test_robust_losses_follow_scipy(loss):
  scene = synthetic.make_scene(C=2, F=6, vis=0.5, seed=31, outlier_fraction=0.03)
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  out = calib.bundle_adjust(loss=loss, f_scale=2.0, tolerance=1e-10, max_iterations=200)
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-12, xtol=1e-12, gtol=1e-12,
                               max_nfev=400, method="trf", tr_solver="exact", loss=loss, f_scale=2.0)
  # never worse than scipy's dense exact trust region; equal where that converges (it does not for arctan in 400 nfev)
  assert out.last_solve.cost <= ref.cost * (1 + 1e-6), (out.last_solve.cost, ref.cost)
  if ref.status > 0:
    assert abs(out.last_solve.cost - ref.cost) <= 1e-6 * ref.cost, (out.last_solve.cost, ref.cost)


def test_outlier_loop_matches_reference_semantics():
  scene = synthetic.make_scene(C=3, F=8, vis=0.5, seed=41, outlier_fraction=0.02)
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  err, mask = prob.reprojection_error()
  thr = select_threshold(quantile=0.75, factor=5.0)(err[mask])
  rejected = calib.reject_outliers(select_threshold(quantile=0.75, factor=5.0)(calib.reprojection_error))
  assert np.array_equal(rejected.inliers, (err < thr) & mask)          # same inlier set as the reference rule
  final = calib.adjust_outliers(num_adjustments=2, select_outliers=select_threshold(quantile=0.75, factor=5.0))
  rms = np.sqrt(np.mean(final.reprojection_inliers ** 2))
  assert 0.35 < rms < 0.5                                              # 0.3 px noise -> 0.3*sqrt(2) expected


def test_fixed_blocks_and_fix_aspect():
  scene = synthetic.make_scene(C=2, F=6, vis=0.5, seed=51)
  calib = from_scene(scene).enable(cameras=True, board_poses=False, camera_poses=False)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True, board_poses=False, camera_poses=False))
  eng = calib._upload(calib.inliers)
  assert np.abs(eng.param_vec - prob.param_vec).max() < 1e-13
  x1 = prob.param_vec + np.random.default_rng(3).normal(0, 1e-3, prob.param_vec.size)
  assert np.abs(eng.residuals(x1) - prob.residuals(x1)).max() < 1e-9
  out = calib.bundle_adjust(tolerance=1e-12, max_iterations=100)
  assert np.allclose(out.camera_poses.poses, calib.camera_poses.poses) and np.allclose(out.board_poses.poses, calib.board_poses.poses)
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-14, xtol=1e-14, gtol=1e-14,
                               max_nfev=300, method="trf", tr_solver="exact")
  assert abs(out.last_solve.cost - ref.cost) <= 1e-8 * ref.cost, (out.last_solve.cost, ref.cost)
  # fix_aspect: one focal parameter drives fx and fy (camera.py:147-148,159-160)
  for c in calib.cameras.param_objects: c.fix_aspect = True
  calib2 = from_scene(scene).enable(cameras=True)
  for c in calib2.cameras.param_objects: c.fix_aspect = True
  prob2 = Problem.from_scene(scene, optimize=dict(cameras=True), fix_aspect=True)
  eng2 = calib2._upload(calib2.inliers)
  x0 = prob2.param_vec
  assert np.abs(eng2.param_vec - x0).max() < 1e-13
  x1 = x0 + np.random.default_rng(4).normal(0, 1e-3, x0.size)
  assert np.abs(eng2.residuals(x1) - prob2.residuals(x1)).max() < 1e-9
  J = fd5_jacobian(prob2, x1)
  JtJ, Jtr, _ = eng2.linearize(x1)
  H = (J.T @ J).toarray()
  nrm = np.sqrt(np.outer(np.diag(H), np.diag(H))); live = nrm > 0
  assert (np.abs(JtJ - H)[live] / nrm[live]).max() < 1e-9
  out2 = calib2.bundle_adjust(tolerance=1e-10)
  for c in out2.cameras: assert c.intrinsic[0, 0] == c.intrinsic[1, 1]


def test_bad_inputs_raise_like_the_reference():
  scene = synthetic.make_scene(C=2, F=4, vis=0.5, seed=61)
  calib = from_scene(scene).enable(cameras=True)
  eng = calib._upload(calib.inliers)
  with pytest.raises(AssertionError):
    eng.set_param_vec(np.zeros(3))                                    # parameters.py:93-95
  with pytest.raises(ValueError):
    eng.solve(loss="bogus")
  bad = from_scene(scene).enable(cameras=True)
  bad.cameras.param_objects[0].intrinsic[0, 0] = np.nan
  with pytest.raises(ValueError):                                      # scipy: residuals not finite at x0
    bad.bundle_adjust()


@pytest.mark.parametrize("workload", ["cfg2", "cfg3", "cfg4", "cfg5"])
def test_large_scene_properties(workload):
  """BASELINE cfg2 .. cfg5 at their full sizes (cfg3: fisheye, 1 M corners; cfg4: 5.5 M corners, n_s = 286, the cooperative Cholesky;
  cfg5: 64 cameras, 50.8 M corners, n_s = 1030): size-independent properties (no oracle run): cost decreases monotonically, RMS lands
  at sigma*sqrt(2), re-solving from the solution is a fixed point, gradient ~0 at the optimum (dense normal equations: not at cfg5,
  whose 13 030 x 13 030 matrix is 1.4 GB on the host)."""
  scene = synthetic.make_workload(workload)
  calib = from_scene(scene).enable(cameras=True)
  out = calib.bundle_adjust()
  costs = [row[2] for row in out.last_solve.log]
  assert all(b <= a for a, b in zip(costs, costs[1:]))
  rms = np.sqrt(np.mean(out.reprojection_error ** 2))
  assert abs(rms - 0.3 * np.sqrt(2)) < 5e-3
  again = out.bundle_adjust()
  assert again.last_solve.nfev <= 3 and abs(again.last_solve.cost - out.last_solve.cost) <= 1e-6 * out.last_solve.cost
  if workload == "cfg5": return
  eng = out._upload(out.inliers)
  JtJ, Jtr, cost = eng.linearize()
  d = np.sqrt(np.diag(JtJ)); d[d == 0] = 1
  assert np.abs(Jtr / d).max() < 1e-3 * np.sqrt(2 * cost)


@pytest.mark.parametrize("name", ["standard_2x6", "cube3_3x6", "invalid_poses_3x6"])
def test_device_packing_equals_host_packing(name):
  """mcba_upload_dense (mask + dense table, packed on the GPU) and mcba_upload (np.argwhere rows packed on the host)
  must give the same corner order, residuals and normal equations."""
  from multical_b200.calibration import get_engine
  from multical_b200.engine import pack_corners
  scene, z, calib, prob = make(name)
  eng = calib._upload(calib.inliers)                 # dense path
  r_dense = eng.residuals(z["x1"]).copy()
  H_dense, g_dense, _ = eng.linearize(z["x1"])
  idx, obs = pack_corners(calib.inliers, np.asarray(calib.point_table.points))
  s = calib.size
  eng.upload(calib.engine_model, calib._optimize_bits(), (s.cameras, s.rig_poses, s.boards, s.points), idx, obs, calib.board_points.points)
  eng.set_params(*calib._state_arrays())
  assert eng.N == idx.shape[0]
  assert np.array_equal(eng.residuals(z["x1"]), r_dense)
  H, g, _ = eng.linearize(z["x1"])
  assert np.allclose(H, H_dense, rtol=1e-12, atol=0) and np.allclose(g, g_dense, rtol=1e-10, atol=1e-9)
  # the two-part mask (detections as they are + pose validity per view, conjunction on the device: what bundle_adjust uploads)
  fresh = from_scene(scene).enable(cameras=True)
  assert "valid" not in fresh.__dict__
  eng = fresh._upload_inliers()
  assert "valid" not in fresh.__dict__ and eng.N == idx.shape[0]
  assert np.array_equal(eng.residuals(z["x1"]), r_dense)
  # a float32 table (the dtype make_point_table keeps for cv2's corners) goes over as float32 and must be the float64 table of the same values
  pts32 = np.asarray(calib.point_table.points).astype(np.float32)
  eng = calib._upload(calib.inliers, points=pts32.astype(np.float64))
  r_64 = eng.residuals(z["x1"]).copy()
  eng = calib._upload(calib.inliers, points=pts32)
  assert eng.N == idx.shape[0] and np.array_equal(eng.residuals(z["x1"]), r_64)
  eng = calib._upload(np.asarray(calib.point_table.valid), points=pts32, view_valid=calib.pose_valid)
  assert eng.N == idx.shape[0] and np.array_equal(eng.residuals(z["x1"]), r_64)


def test_empty_and_ragged_inputs():
  scene = synthetic.make_scene(C=2, F=4, vis=0.5, seed=71)
  # a camera that sees nothing, a frame that nobody sees, single-corner views
  scene["valid"][1] = False
  scene["valid"][:, 2] = False
  scene["valid"][0, 0, 0, 1:] = False
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  eng = calib._upload(calib.inliers)
  assert eng.N == int(scene["valid"].sum())
  assert np.abs(eng.residuals() - prob.residuals()).max() < 1e-9
  out = calib.bundle_adjust(max_iterations=30)
  assert np.isfinite(out.last_solve.cost)
  assert np.allclose(out.motion.poses[2], calib.motion.poses[2]) and np.allclose(out.camera_poses.poses[1], calib.camera_poses.poses[1])
  # nothing selected at all
  empty = from_scene(scene).copy(inlier_mask=np.zeros_like(scene["valid"]))
  eng = empty._upload(empty.inliers)
  assert eng.N == 0 and eng.residuals().size == 0
  res = eng.solve(max_nfev=5)
  assert res.cost == 0.0 and res.status == 1        # gradient is exactly zero -> gtol


def test_board_points_as_parameters():
  """boards=True (adjust_board): 3 parameters per board point, axis-3 columns of the reference's Jacobian
  (calibration.py:188-190, board/charuco.py:112-117)."""
  scene = synthetic.make_scene(C=3, F=8, vis=0.6, seed=81, boards=("cube", 6, 5, 0.05, 2), rig="dome")
  opt = dict(cameras=True, boards=True)
  calib = from_scene(scene).enable(**opt)
  prob = Problem.from_scene(scene, optimize=opt)
  x0 = prob.param_vec
  assert np.array_equal(calib.param_vec, x0)
  eng = calib._upload(calib.inliers)
  assert np.abs(calib._from_engine_vec(eng.param_vec) - x0).max() < 1e-13
  x1 = x0 + np.random.default_rng(8).normal(0, 1e-3, x0.size)
  r1 = eng.residuals(calib._to_engine_vec(x1))
  assert np.abs(r1 - prob.residuals(x1)).max() < 1e-9
  J = fd5_jacobian(prob, x1)
  H, g = (J.T @ J).toarray(), J.T @ prob.residuals(x1)
  JtJ, Jtr, cost = eng.linearize(calib._to_engine_vec(x1))
  keep = calib._board_block_slices()
  head = JtJ.shape[0] - keep.size
  sel = np.concatenate([np.ones(head, bool), keep])
  JtJ, Jtr = JtJ[np.ix_(sel, sel)], Jtr[sel]
  nrm = np.sqrt(np.outer(np.diag(H), np.diag(H))); live = nrm > 0
  # k3 (r^6) of these small cube boards has H_ii ~ 1e-3: the rounding of the pixel values alone moves its finite-difference entries by
  # ~4e-9 of sqrt(H_ii H_jj)
  assert (np.abs(JtJ - H)[live] / nrm[live]).max() < 1e-8
  assert np.abs(Jtr - g).max() < 1e-10 * np.abs(g).max()
  # the solve: never worse than the reference algorithm, and board points actually move
  out = calib.bundle_adjust(tolerance=1e-8, max_iterations=60)
  _, ref = prob.bundle_adjust(tolerance=1e-8, max_iterations=60)
  assert out.last_solve.cost <= ref.cost * (1 + 1e-6), (out.last_solve.cost, ref.cost)
  moved = max(np.abs(np.asarray(b1.adjusted_points) - np.asarray(b0.adjusted_points)).max() for b0, b1 in zip(calib.boards, out.boards))
  assert 0 < moved < 0.05
  # without boards=True the same scene must reach a higher (or equal) cost
  base = from_scene(scene).enable(cameras=True).bundle_adjust(tolerance=1e-8, max_iterations=60)
  assert out.last_solve.cost <= base.last_solve.cost * (1 + 1e-9)


@pytest.mark.parametrize("name", ["standard_2x6", "cube3_3x6"])
def test_iteration_table_matches_the_trf_model(name):
  """The device solver claims scipy's trf_no_bounds semantics with an exact inner solve.  oracle/trf_exact_model.py is
  that statement in numpy (scipy's own helper functions); the per-iteration table (nfev, cost, cost reduction, step norm)
  must agree until the two Jacobians (analytic vs finite differences) differ by more than their noise."""
  from oracle.trf_exact_model import trf_exact
  scene, z, calib, prob = make(name)
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  _, cost, nfev, njev, status, rows = trf_exact(prob.residuals, jac, prob.param_vec, ftol=1e-4)
  out = calib.bundle_adjust(tolerance=1e-4)
  log = out.last_solve.log
  compared = 0
  for (it, nf, c, red, sn, gn), (it2, nf2, c2, red2, sn2, gn2) in zip(log, rows):
    if red2 is not None and not red2 > 1e-6 * c2:
      break            # from here on the step is inside the finite-difference noise of the model's Jacobian
    assert (it, nf) == (it2, nf2)
    assert abs(c - c2) <= 1e-7 * c2
    if gn2 > 1e-4 * rows[0][5]:                       # later gradients are dominated by the finite-difference noise
      assert abs(gn - gn2) <= 1e-3 * gn2
    if red2 is not None:
      # both costs agree to 1e-7 relative, so their difference can only agree to ~1e-7 * cost in absolute terms
      assert abs(red - red2) <= 1e-5 * red2 + 2e-7 * c2 and abs(sn - sn2) <= 1e-3 * sn2
    compared += 1
  assert compared >= 3
  assert out.last_solve.cost <= cost * (1 + 1e-7)


@pytest.mark.parametrize("opt", [dict(cameras=True, motion=False), dict(camera_poses=False, board_poses=False, motion=True),
                                 dict(cameras=False, camera_poses=False, board_poses=False, motion=False)])
def test_degenerate_block_selections(opt):
  """No frame block to eliminate (motion fixed), no shared block at all (only the rig poses free), nothing free."""
  scene = synthetic.make_scene(C=2, F=6, vis=0.5, seed=91)
  calib = from_scene(scene).enable(**opt)
  prob = Problem.from_scene(scene, optimize=opt)
  x0 = prob.param_vec
  eng = calib._upload(calib.inliers)
  assert eng.num_params == x0.size
  if x0.size:
    x1 = x0 + np.random.default_rng(9).normal(0, 1e-3, x0.size)
    assert np.abs(eng.residuals(x1) - prob.residuals(x1)).max() < 1e-9
    S = prob.sparsity_matrix()
    J = fd5_jacobian(prob, x1)
    JtJ, Jtr, _ = eng.linearize(x1)
    H = (J.T @ J).toarray()
    nrm = np.sqrt(np.outer(np.diag(H), np.diag(H))); live = nrm > 0
    assert (np.abs(JtJ - H)[live] / nrm[live]).max() < 1e-9
  out = calib.bundle_adjust(tolerance=1e-10, max_iterations=60)
  r0 = prob.residuals()
  assert out.last_solve.cost <= 0.5 * r0 @ r0 * (1 + 1e-12)
  if x0.size:
    jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, group_columns(S))).toarray()
    ref = optimize.least_squares(prob.residuals, x0, jac=jac, x_scale="jac", ftol=1e-14, xtol=1e-14, gtol=1e-14,
                                 max_nfev=300, method="trf", tr_solver="exact")
    assert abs(out.last_solve.cost - ref.cost) <= 1e-7 * ref.cost, (out.last_solve.cost, ref.cost)
  else:
    assert out.last_solve.nfev == 1 and np.allclose(out.motion.poses, calib.motion.poses)
