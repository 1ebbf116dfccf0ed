"""GPU (-m gpu): the two non-static motion models through the C-ABI -- RollingFrames (motion/rolling_frames.py:66-150) and
HandEye (motion/hand_eye.py:14-90), SURVEY.md §8f rank 2 -- against the golden vectors of the running reference
(tests/golden/rolling_2x6.npz, handeye_2x6.npz) and the oracle.  Same bars as tests/test_gpu_parity.py:
  parameter layout bit exact; residuals at identical x <= 1e-9 px; J^T J, J^T r vs 5-point FD of the oracle <= 1e-9 / 1e-10 relative;
  converged cost vs scipy's dense exact trust region on the oracle <= 1e-8 relative; never worse than the reference's own run.
"""
import numpy as np
import pytest
from scipy import optimize
from scipy.optimize._numdiff import approx_derivative, group_columns

from conftest import load_golden
from multical_b200 import _native
from multical_b200.calibration import from_scene
from multical_b200.motion import HandEye, RollingFrames
from multical_b200.pose_set import pose_table
from oracle.ba_oracle import Problem
from test_gpu_step_parity import fd5_jacobian

pytestmark = pytest.mark.gpu
CASES = ["rolling_2x6", "handeye_2x6"]


def make(name):
  """(golden dict, Calibration on this package's mirrors, oracle Problem) of one motion-model fixture."""
  scene, z = load_golden(name)
  enabled = dict(zip((str(k) for k in z["enabled_keys"]), (bool(v) for v in z["enabled_values"])))
  kw = dict(optimize=enabled, motion=str(z["motion"]), image_size=z["image_size"])
  for key in ("frame_poses_end", "base_wrt_gripper", "world_wrt_base", "gripper_wrt_camera"):
    if key in z: kw[key] = z[key]
  prob = Problem.from_scene(scene, **kw)
  calib = from_scene(scene)
  if str(z["motion"]) == "rolling":
    motion = RollingFrames(z["frame_poses"], z["frame_poses_end"], z["frame_valid"], [str(i) for i in range(scene["F"])])
  else:
    motion = HandEye(pose_table(z["base_wrt_gripper"], z["frame_valid"]), z["world_wrt_base"], z["gripper_wrt_camera"])
  return z, calib.copy(motion=motion).enable(**enabled), prob


@pytest.mark.parametrize("name", CASES)
def test_layout_residuals_and_errors_match_reference_golden(name):
  z, calib, prob = make(name)
  assert np.abs(calib.param_vec - z["x0"]).max() < 1e-12              # host mirror: block order and the motion block's own layout
  eng = calib._upload(calib.inliers)
  assert eng.N == z["r0"].size // 2 and eng.num_params == z["x0"].size
  assert np.abs(eng.param_vec - z["x0"]).max() < 1e-12                # device: matrices -> rtvecs, internal -> reference order
  eng.set_param_vec(z["x1"])
  assert np.array_equal(eng.param_vec, z["x1"])                       # the permutation round-trips bit exactly
  eng.set_param_vec(z["x0"])
  assert np.abs(eng.residuals() - z["r0"]).max() < 1e-9               # vs the running reference
  r1, cost = eng.residuals(z["x1"], with_cost=True)
  assert np.abs(r1 - z["r1"]).max() < 1e-9
  assert np.abs(r1 - prob.residuals(z["x1"])).max() < 1e-9           # vs the oracle
  assert abs(cost - 0.5 * z["r1"] @ z["r1"]) <= 1e-12 * cost
  assert np.array_equal(eng.param_vec, z["x0"])                       # evaluating at x1 must not move the state
  assert np.abs(calib.reprojection_error - z["err_valid"]).max() < 1e-9
  S = calib.sparsity_matrix.tocsr(); S.sort_indices()
  assert tuple(S.shape) == tuple(z["sp_shape"]) and np.array_equal(S.indptr, z["sp_indptr"]) and np.array_equal(S.indices, z["sp_indices"])


@pytest.mark.parametrize("name", CASES)
def test_normal_equations_match_finite_differences(name):
  z, calib, prob = make(name)
  eng = calib._upload(calib.inliers)
  x1 = z["x1"]
  J = fd5_jacobian(prob, x1)
  r = prob.residuals(x1)
  H, g = (J.T @ J).toarray(), J.T @ r
  JtJ, Jtr, cost = eng.linearize(x1)
  nrm = np.sqrt(np.outer(np.diag(H), np.diag(H)))
  live = nrm > 0
  assert (np.abs(JtJ - H)[live] / nrm[live]).max() < 1e-9
  assert np.abs(JtJ[~live]).max(initial=0.0) == 0.0
  assert np.abs(Jtr - g).max() < 1e-10 * np.abs(g).max()
  assert abs(cost - 0.5 * r @ r) < 1e-12 * cost
  assert np.abs(JtJ - JtJ.T).max() <= 1e-12 * np.abs(JtJ).max()


@pytest.mark.parametrize("name", CASES)
def test_converged_solution_matches_dense_exact_oracle(name):
  z, calib, prob = make(name)
  out = calib.bundle_adjust()                                          # the reference's defaults (tolerance 1e-4)
  assert out.last_solve.cost <= float(z["ba_cost"]) * (1 + 1e-6)      # never worse than the reference's own run
  assert np.abs(prob.residuals(out.param_vec) @ prob.residuals(out.param_vec) * 0.5 - out.last_solve.cost) <= 1e-9 * out.last_solve.cost
  tight = calib.bundle_adjust(tolerance=1e-14, xtol=1e-14, gtol=1e-12, max_iterations=200)
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac_sparsity=None, x_scale="jac", method="trf", tr_solver="exact",
                               ftol=1e-14, xtol=1e-14, gtol=1e-12, max_nfev=300)
  assert abs(tight.last_solve.cost - ref.cost) <= 1e-8 * ref.cost
  assert np.abs(tight.reprojection_error - Problem.reprojection_error(prob.with_param_vec(ref.x))[0][calib.valid]).max() < 1e-4


@pytest.mark.parametrize("name", CASES)
def test_iteration_table_matches_the_trf_model(name):
  """The solver's trust-region semantics under the motion models: per-iteration table against scipy's trf_no_bounds logic with an exact
  inner solve (oracle/trf_exact_model.py) driven by the oracle's residual and a finite-difference Jacobian -- same comparison, same
  tolerances as tests/test_gpu_parity.py for static frames."""
  from oracle.trf_exact_model import trf_exact
  z, calib, prob = make(name)
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  _, cost, nfev, njev, status, rows = trf_exact(prob.residuals, jac, prob.param_vec, ftol=1e-4)
  log = calib.bundle_adjust(tolerance=1e-4).last_solve.log
  compared = 0
  for (it, nf, c, red, sn, gn), (it2, nf2, c2, red2, sn2, gn2) in zip(log, rows):
    if red2 is not None and not red2 > 1e-6 * c2: break       # inside the finite-difference noise of the model's Jacobian from here on
    assert (it, nf) == (it2, nf2) and abs(c - c2) <= 1e-7 * c2
    # step norms: 1e-3 while the step is large; the last steps before convergence (|step| ~ 1e-4 in the 18-parameter hand-eye problem)
    # move along weakly determined directions, where the model's finite-difference Jacobian is only good for a few per cent
    if red2 is not None: assert abs(red - red2) <= 1e-5 * red2 + 2e-7 * c2 and abs(sn - sn2) <= (1e-3 if sn2 > 1e-2 else 5e-2) * sn2
    compared += 1
  assert compared >= 3


def test_rolling_projection_without_measurements_iterates_like_the_reference():
  """`Calibration.projected` (calibration.py:115-121): rows from mid-exposure, then max_iterations re-projections with the rows
  of the previous projection (rolling_frames.py:115-133); `reprojected` takes the rows of the measurements."""
  z, calib, prob = make("rolling_2x6")
  H = float(z["image_size"][1])
  est = np.zeros_like(prob.points); est[..., 1] = 0.5 * H
  uv, ok = prob.copy(points=est).reprojected()
  for _ in range(4): uv, ok = prob.copy(points=uv).reprojected()
  got = calib.projected
  assert np.array_equal(np.asarray(got.valid), ok)
  assert np.abs(np.asarray(got.points)[ok] - uv[ok]).max() < 1e-9
  uv2, _ = prob.reprojected()
  assert np.abs(np.asarray(calib.reprojected.points)[ok] - uv2[ok]).max() < 1e-9


@pytest.mark.parametrize("name", CASES)
def test_outlier_loop_on_the_resident_table_equals_the_host_loop(name, monkeypatch):
  """adjust_outliers (calibration.py:254-268) with the table resident on the device must reproduce the host loop for the two motion
  models too: the motion state has to survive every re-selection of the table (mcba_table_select keeps the parameter state)."""
  from multical_b200.calibration import select_threshold
  z, calib, prob = make(name)
  pts = np.asarray(calib.point_table.points).copy()
  idx = np.argwhere(calib.valid)
  rng = np.random.default_rng(7)
  for c, f, b, p in idx[rng.choice(len(idx), 25, replace=False)]: pts[c, f, b, p] += rng.normal(0, 30.0, 2)     # gross outliers
  calib = calib.copy(point_table=calib.point_table._extend(points=pts))
  res = calib.adjust_outliers(num_adjustments=2, select_outliers=select_threshold(quantile=0.75, factor=4), max_iterations=6)
  monkeypatch.setenv("MCBA_HOST_OUTLIERS", "1")
  host = calib.adjust_outliers(num_adjustments=2, select_outliers=select_threshold(quantile=0.75, factor=4), max_iterations=6)
  assert np.array_equal(res.inliers, host.inliers) and res.inliers.sum() < calib.valid.sum()
  assert abs(res.last_solve.cost - host.last_solve.cost) <= 1e-6 * host.last_solve.cost
  assert np.abs(res.reprojection_error - host.reprojection_error).max() < 1e-2


@pytest.mark.parametrize("name", CASES)
def test_board_points_as_parameters_under_a_motion_model(name):
  """boards=True (board/charuco.py:112-117; sparsity axis 3, calibration.py:188-190) together with rolling / hand-eye frames: the
  point blocks and their couplings with the 12-wide frame block resp. the hand-eye pair, against finite differences of the oracle."""
  z, calib, prob = make(name)
  calib = calib.enable(boards=True)
  prob = prob.copy(optimize=dict(prob.optimize, boards=True))
  x0 = prob.param_vec
  assert np.abs(calib.param_vec - x0).max() < 1e-12 and np.abs(x0 - z["boards_x0"]).max() < 1e-12       # layout of the running reference
  eng = calib._upload(calib.inliers)
  assert np.abs(eng.residuals(calib._to_engine_vec(z["boards_x1"])) - z["boards_r1"]).max() < 1e-9        # evaluate() of the running reference
  x1 = x0 + np.random.default_rng(3).normal(0, 1e-4, x0.size)
  assert np.abs(eng.residuals(calib._to_engine_vec(x1)) - prob.residuals(x1)).max() < 1e-9
  J = fd5_jacobian(prob, x1)
  r = prob.residuals(x1)
  H, g = (J.T @ J).toarray(), J.T @ r
  JtJ_e, Jtr_e, cost = eng.linearize(calib._to_engine_vec(x1))
  keep = np.ones(JtJ_e.shape[0], bool)
  keep[-calib._board_block_slices().size:] = calib._board_block_slices()          # padded board slots have no counterpart in the reference vector
  JtJ, Jtr = JtJ_e[np.ix_(keep, keep)], Jtr_e[keep]
  nrm = np.sqrt(np.outer(np.diag(H), np.diag(H)))
  live = nrm > 0
  assert (np.abs(JtJ - H)[live] / nrm[live]).max() < 1e-9
  assert np.abs(Jtr - g).max() < 1e-10 * np.abs(g).max()
  assert abs(cost - 0.5 * r @ r) < 1e-12 * cost
  out = calib.bundle_adjust(max_iterations=5)                       # a few iterations of the ~1000-parameter system are enough here
  assert out.last_solve.cost < 0.5 * z["r0"] @ z["r0"]
  rr = prob.residuals(out.param_vec)
  assert abs(0.5 * rr @ rr - out.last_solve.cost) <= 1e-9 * out.last_solve.cost      # the returned objects hold the solved state


@pytest.mark.parametrize("name", CASES)
def test_mirror_classes_keep_the_reference_semantics(name):
  """What callers of the reference rely on (calibration.py:99-112,164-171,222-232; rolling_frames.py:95-103; hand_eye.py:54-58): a change
  of master camera leaves every projection where it was, the parameter vector round-trips, objects pickle with their state keys."""
  import pickle
  z, calib, prob = make(name)
  base = np.asarray(calib.reprojected.points)
  ok = np.asarray(calib.reprojected.valid)
  moved = calib.with_master(1)
  assert np.abs(np.asarray(moved.camera_poses.poses)[1] - np.eye(4)).max() < 1e-12
  assert np.abs(np.asarray(moved.reprojected.points)[ok] - base[ok]).max() < 1e-8
  again = calib.with_param_vec(calib.param_vec)
  assert np.abs(again.param_vec - calib.param_vec).max() < 1e-12
  assert np.abs(np.asarray(again.reprojected.points)[ok] - base[ok]).max() < 1e-8
  clone = pickle.loads(pickle.dumps(calib))
  assert type(clone.motion) is type(calib.motion) and np.array_equal(clone.param_vec, calib.param_vec)
  assert sorted(clone.motion.__getstate__()) == sorted(calib.motion.__getstate__())



def test_two_identical_hand_eye_solves_agree_bit_for_bit():
  """Hand-eye frames go through the same linearisation as static frames (the hand-eye blocks are fixed-order folds of the per-frame
  blocks, k_fold_hand_eye): two identical solves, and two linearisations at the same point, agree bit for bit."""
  z, calib, prob = make("handeye_2x6")
  runs = [calib.bundle_adjust(tolerance=1e-9, max_iterations=30) for _ in range(2)]
  assert runs[1].last_solve.cost == runs[0].last_solve.cost
  assert np.array_equal(np.array(runs[1].last_solve.log, float), np.array(runs[0].last_solve.log, float), equal_nan=True)
  assert np.array_equal(runs[1].param_vec, runs[0].param_vec)
  eng = calib._upload(calib.inliers)
  H0, g0, c0 = eng.linearize(z["x1"])
  H1, g1, c1 = eng.linearize(z["x1"])
  assert np.array_equal(H0, H1) and np.array_equal(g0, g1) and c0 == c1


def test_hand_eye_calibration_wrapper_from_arm_poses():
  """HandEyeCalibration (optimization/hand_eye.py:13-97): robot-world initialisation from the arm's poses, then the GPU bundle adjustment
  over the 12 hand-eye parameters (+ board poses); the known transforms of the fixture are recovered."""
  from multical_b200.hand_eye import HandEyeCalibration
  z, calib, prob = make("handeye_2x6")
  static = from_scene(load_golden("handeye_2x6")[0])                                      # StaticFrames over the same frame poses
  gripper_wrt_base = np.linalg.inv(z["base_wrt_gripper"])
  he = HandEyeCalibration.initialise(static, gripper_wrt_base)
  assert he.calib.optimize["cameras"] is False and he.calib.optimize["camera_poses"] is False and he.calib.optimize["motion"] is True
  # the fixture's arm poses reproduce its frame poses exactly under the TRUE transforms (make_golden.py): the initialisation, which sees
  # the perturbed start values' frames, must land within the perturbation (5 mm / 0.3 deg) of them
  frames_true = np.asarray(static.motion.poses)
  assert np.abs(np.asarray(he.calib.motion.poses) - frames_true).max() < 5e-2
  before = 0.5 * float(np.sum((np.asarray(he.calib.reprojected.points) - np.asarray(he.calib.point_table.points))[he.calib.inliers] ** 2))
  out = he.bundle_adjust()
  assert isinstance(out, HandEyeCalibration) and out.calib.last_solve.cost < before
  assert out.calib.last_solve.cost <= float(z["ba_cost"]) * (1 + 1e-3)                    # as good as the reference's run from its own start
  assert set(out.cameras_wrt_gripper) == set(out.calib.cameras.names)


def test_motion_state_entry_points_refuse_the_wrong_problem():
  z, calib, prob = make("rolling_2x6")
  eng = calib._upload(calib.inliers)
  with pytest.raises(_native.NativeError): eng.set_hand_eye(np.tile(np.eye(4), (eng.desc.F, 1, 1)), np.eye(4), np.eye(4))
  assert np.abs(eng.get_rolling() - z["frame_poses_end"]).max() < 1e-12
  z, calib, prob = make("handeye_2x6")
  eng = calib._upload(calib.inliers)
  with pytest.raises(_native.NativeError): eng.set_rolling(np.tile(np.eye(4), (eng.desc.F, 1, 1)), np.ones(eng.desc.C))
  w, g = eng.get_hand_eye()
  assert np.abs(w - z["world_wrt_base"]).max() < 1e-12 and np.abs(g - z["gripper_wrt_camera"]).max() < 1e-12
  frames = eng.get_state_matrices()[2]                                                     # derived: G A_f W
  assert np.abs(frames - z["gripper_wrt_camera"] @ z["base_wrt_gripper"] @ z["world_wrt_base"]).max() < 1e-12
