"""CPU (-m "not gpu"): the REAL CUDA kernels and the REAL host driver of multical_b200/csrc, executed by the SIMT interpreter of
tests/simt (every CUDA thread a fiber, blocks one after the other) behind the same C-ABI, against the same oracle / golden
assertions as the GPU suite.  The test functions are the ones of tests/test_gpu_parity.py and tests/test_gpu_table.py -- imported,
not copied -- with the ctypes binding pointed at tests/simt/build/libmcba_simt.so for the duration of each test.

What this proves without a GPU: indexing, math, shared-memory layouts, warp-collective usage (full-mask discipline, barrier
placement -- a divergent barrier aborts the interpreter) and the host-side plumbing of every kernel launched by these tests.
What it cannot prove: anything about concurrency (blocks and fibers run deterministically) or speed; that is the GPU suite's job.
The library is test infrastructure: the product (multical_b200/_native.py) never loads it.
"""

import os
import pytest

import test_gpu_parity as gp
import test_gpu_table as gt
import test_gpu_motion as gm
import test_gpu_pnp as gn
import test_gpu_step_parity as sp
import test_gpu_linearize_shapes as lin_shapes
from multical_b200 import _native, calibration


@pytest.fixture(scope="session")
def simt_library():
  import simt                     # tests/simt/__init__.py (tests/ is on sys.path: pytest rootdir/conftest import mode)
  return simt.build()


@pytest.fixture(autouse=True)
def on_the_interpreter(simt_library, monkeypatch):
  """Point the ctypes binding at the interpreter build for one test; engines are per-library, so the cache is swapped as well."""
  monkeypatch.setattr(_native, "LIB_PATH", simt_library)
  monkeypatch.setattr(_native, "_lib", None)
  monkeypatch.setattr(_native, "_allow_interpreter", True)
  monkeypatch.setattr(calibration, "_engines", {})
  monkeypatch.delenv("SIMT_SMS", raising=False)
  yield
  for eng in calibration._engines.values(): eng.close()


# ---- tests/test_gpu_parity.py on the interpreter (the two large-scene property tests stay GPU-only: minutes of fiber switching)
test_residuals_match_reference_golden_and_oracle = gp.test_residuals_match_reference_golden_and_oracle
test_reprojection_error_over_valid = gp.test_reprojection_error_over_valid
test_normal_equations_match_finite_differences = gp.test_normal_equations_match_finite_differences
test_converged_solution_matches_dense_exact_oracle = gp.test_converged_solution_matches_dense_exact_oracle


@pytest.mark.parametrize("loss", ["soft_l1", "huber", "cauchy"])          # arctan (slow to converge: 45 s of fiber switching) stays GPU-only
def test_robust_losses_follow_scipy(loss):
  gp.test_robust_losses_follow_scipy(loss)


test_outlier_loop_matches_reference_semantics = gp.test_outlier_loop_matches_reference_semantics
test_fixed_blocks_and_fix_aspect = gp.test_fixed_blocks_and_fix_aspect
test_bad_inputs_raise_like_the_reference = gp.test_bad_inputs_raise_like_the_reference
test_device_packing_equals_host_packing = gp.test_device_packing_equals_host_packing
test_empty_and_ragged_inputs = gp.test_empty_and_ragged_inputs
test_board_points_as_parameters = gp.test_board_points_as_parameters
test_iteration_table_matches_the_trf_model = gp.test_iteration_table_matches_the_trf_model
test_degenerate_block_selections = gp.test_degenerate_block_selections
test_many_cameras_use_the_cooperative_blocked_reduced_solve = gp.test_many_cameras_use_the_cooperative_blocked_reduced_solve
test_frame_count_that_ends_a_syrk_chunk_in_a_partial_step = gp.test_frame_count_that_ends_a_syrk_chunk_in_a_partial_step
if os.environ.get("MCBA_SIMT_FULL") == "1":      # three minutes on the interpreter (n_s = 1030): opt-in, the GPU suite always runs it
  test_sixty_four_cameras_configs4_shape = gp.test_sixty_four_cameras_configs4_shape
test_two_identical_solves_agree_bit_for_bit = gp.test_two_identical_solves_agree_bit_for_bit

def test_more_views_per_frame_and_more_boards_than_the_staged_tables_hold():
  """k_linearize stages a frame's view records (up to 96) and the board pose tables (up to 8) in shared memory and reads them from
  global memory beyond that (csrc/linearize.cuh LIN_MAXV, LIN_MAXB).  12 cameras x 9 boards, frames of 96, 97 and 108 views: the step
  from staged to global view lists inside one launch, with global board tables.  Residuals against the oracle, normal equations
  against fourth-order differences of the oracle and the first step against the model (tests/test_gpu_linearize_shapes.py)."""
  lin_shapes.run_shape("both unstaged, 96 / 97 / 108", 132)


def test_rolling_frames_with_a_frame_count_that_ends_in_a_partial_syrk_step():
  """Rolling frames eliminate a 12 x 12 block per frame and the Schur SYRK stages 4 of them per step: 19 frames = 5 steps, the last one
  partial, in a stage that held an earlier step (the frame-count pattern of test_frame_count_that_ends_a_syrk_chunk_in_a_partial_step for
  FB = 12).  Residuals against the oracle, converged cost against scipy's dense exact trust region on the oracle's residuals."""
  import numpy as np
  from scipy import optimize
  from scipy.optimize._numdiff import approx_derivative, group_columns
  from multical_b200 import synthetic
  from multical_b200.calibration import from_scene
  from multical_b200.motion import RollingFrames
  from oracle.ba_oracle import Problem
  scene = synthetic.make_scene(C=2, F=19, vis=0.3, seed=5)
  rng = np.random.default_rng(7)
  start = scene["init"]["frame_poses"]
  end = synthetic.to_matrix(synthetic.from_matrix(start) + 1e-3 * rng.standard_normal((scene["F"], 6)))
  enabled = dict(cameras=True, camera_poses=True, board_poses=True, motion=True)
  prob = Problem.from_scene(scene, optimize=enabled, motion="rolling", frame_poses_end=end, image_size=scene["image_size"])
  calib = from_scene(scene).copy(motion=RollingFrames(start, end, scene["frame_valid"], [str(i) for i in range(scene["F"])])).enable(**enabled)
  eng = calib._upload(calib.inliers)
  assert eng.num_params == prob.param_vec.size
  assert np.abs(eng.residuals(prob.param_vec) - prob.residuals(prob.param_vec)).max() < 1e-9
  S = prob.sparsity_matrix(); groups = group_columns(S)
  jac = lambda x: approx_derivative(prob.residuals, x, method="3-point", sparsity=(S, groups)).toarray()
  ref = optimize.least_squares(prob.residuals, prob.param_vec, jac=jac, x_scale="jac", ftol=1e-13, xtol=1e-13, gtol=1e-13,
                               max_nfev=200, method="trf", tr_solver="exact")
  out = calib.bundle_adjust(tolerance=1e-13, xtol=1e-13, gtol=1e-13, max_iterations=200)
  assert abs(out.last_solve.cost - ref.cost) <= 1e-8 * ref.cost, (out.last_solve.cost, ref.cost)


# ---- tests/test_gpu_step_parity.py on the interpreter (the cheap shapes; the interpreter has 132 SMs unless SIMT_SMS says otherwise)
@pytest.mark.parametrize("C", [1, 2, 3, 5])
def test_step_parity_views_that_end_a_corner_chunk(C):
  sp.run_chunk_tails(C)


@pytest.mark.parametrize("motion", ["static", "rolling"])
def test_step_parity_ctas_that_own_several_frames(motion, monkeypatch):
  """One SM: 2 resident CTAs, 24 frames -> 12 frames per CTA (set before the first engine of the test is created)."""
  monkeypatch.setenv("SIMT_SMS", "1")
  sp.run_frames_per_cta(motion, 24, 1)


def test_step_parity_hand_eye_beyond_one_fold_batch():
  """70 frames: fold batches of 64 + 6."""
  sp.run_hand_eye_folds(70, False)


@pytest.mark.parametrize("n_s", [127, 128])
def test_step_parity_reduced_solve_at_the_cholesky_boundary(n_s):
  assert sp.run_reduced_solve(n_s, "static", 6, 132) == (8, 1)


def test_step_parity_robust_loss():
  sp.run_robust_loss("cauchy")


# ---- tests/test_gpu_table.py on the interpreter
test_table_errors_ranks_and_reject_are_numpy_on_the_same_errors = gt.test_table_errors_ranks_and_reject_are_numpy_on_the_same_errors
test_resident_adjust_outliers_equals_host_loop = gt.test_resident_adjust_outliers_equals_host_loop
test_table_from_detections_is_make_point_table = gt.test_table_from_detections_is_make_point_table
test_table_state_machine_refuses_stale_errors = gt.test_table_state_machine_refuses_stale_errors
test_outlier_steps_match_reference_golden = gt.test_outlier_steps_match_reference_golden
test_workspace_calibrate_is_enable_plus_the_outlier_loop = gt.test_workspace_calibrate_is_enable_plus_the_outlier_loop

# ---- tests/test_gpu_motion.py on the interpreter (RollingFrames, HandEye)
test_motion_layout_residuals_and_errors_match_reference_golden = gm.test_layout_residuals_and_errors_match_reference_golden
test_motion_normal_equations_match_finite_differences = gm.test_normal_equations_match_finite_differences
test_motion_converged_solution_matches_dense_exact_oracle = gm.test_converged_solution_matches_dense_exact_oracle
test_motion_iteration_table_matches_the_trf_model = gm.test_iteration_table_matches_the_trf_model
test_rolling_projection_without_measurements_iterates_like_the_reference = gm.test_rolling_projection_without_measurements_iterates_like_the_reference
test_motion_state_entry_points_refuse_the_wrong_problem = gm.test_motion_state_entry_points_refuse_the_wrong_problem
test_motion_mirror_classes_keep_the_reference_semantics = gm.test_mirror_classes_keep_the_reference_semantics
test_hand_eye_calibration_wrapper_from_arm_poses = gm.test_hand_eye_calibration_wrapper_from_arm_poses
test_two_identical_hand_eye_solves_agree_bit_for_bit = gm.test_two_identical_hand_eye_solves_agree_bit_for_bit
test_motion_board_points_as_parameters_under_a_motion_model = gm.test_board_points_as_parameters_under_a_motion_model
test_motion_outlier_loop_on_the_resident_table_equals_the_host_loop = gm.test_outlier_loop_on_the_resident_table_equals_the_host_loop

# ---- tests/test_gpu_pnp.py on the interpreter (batched board-pose initialisation)
test_pnp_pose_table_matches_reference_golden = gn.test_pose_table_matches_reference_golden
test_pnp_every_camera_model_against_opencv = gn.test_every_camera_model_against_opencv
test_pnp_minimum_detections_rule_and_bad_inputs = gn.test_minimum_detections_rule_and_bad_inputs
test_pnp_april_grid_style_ids_use_the_tag_grid = gn.test_april_grid_style_ids_use_the_tag_grid


def test_the_product_refuses_the_interpreter_build(simt_library, monkeypatch):
  """Pointing the product at the interpreter library (e.g. through MCBA_LIB) must fail loudly: there is no CPU path."""
  monkeypatch.setattr(_native, "_allow_interpreter", False)
  monkeypatch.setattr(_native, "_lib", None)
  with pytest.raises(_native.NativeError, match="no CPU path"):
    _native.load()


def test_every_kernel_launch_and_shared_declaration_is_translated(simt_library):
  """The interpreter build is a textual translation of csrc/: no `<<<`, `__shared__` or inline PTX may survive it, and every launch of
  the sources must have become exactly one simt::launch."""
  import os, re
  import simt
  n_src = n_out = 0
  for f in simt.sources():
    src = open(os.path.join(simt.CSRC, f)).read()
    out = open(os.path.join(simt.OUT, f[:-3] + ".cpp" if f.endswith(".cu") else f)).read()
    n_src += src.count("<<<"); n_out += out.count("simt::launch(")
    assert "<<<" not in out and "asm volatile" not in out and not re.search(r"\b__shared__\b", out), f
  assert n_src == n_out and n_src > 30


# ---- this package's Calibration against what the reference's own Calibration computed over its own objects ------------------------
@pytest.mark.parametrize("motion", ["static", "rolling", "hand_eye"])
def test_calibration_over_the_reference_objects(motion):
  """INTEGRATION.md A: this package's Calibration, built from its mirror classes over the scene the reference's ParamList / Camera /
  PoseSet / Table / motion-model objects were built from (tests/golden/reference_objects_2x5.npz), has the reference's parameter
  vector, projections and errors; bundle_adjust returns the same classes again, with a cost that matches its own residuals."""
  import numpy as np
  from conftest import load_golden
  from multical_b200.calibration import from_scene
  from multical_b200.motion import HandEye, RollingFrames
  from multical_b200.pose_set import pose_table
  scene, z = load_golden("reference_objects_2x5")
  mine = from_scene(scene)
  if motion == "rolling":
    mine = mine.copy(motion=RollingFrames(scene["init"]["frame_poses"], z["rolling_frame_poses_end"], scene["frame_valid"],
                                          [str(i) for i in range(scene["F"])]))
  elif motion == "hand_eye":
    mine = mine.copy(motion=HandEye(pose_table(scene["init"]["frame_poses"], scene["frame_valid"]), np.eye(4), np.eye(4)))
  mine = mine.enable(camera_poses=False, cameras=False) if motion == "hand_eye" else mine.enable(cameras=True)
  assert np.abs(np.asarray(mine.param_vec) - z[f"{motion}_x0"]).max() < 1e-12
  ok = z[f"{motion}_ok"]
  assert np.array_equal(np.asarray(mine.reprojected.valid) & np.asarray(mine.point_table.valid), ok)
  assert np.abs(np.asarray(mine.reprojected.points)[ok] - z[f"{motion}_proj"][ok]).max() < 1e-9
  assert np.abs(np.asarray(mine.reprojection_error) - z[f"{motion}_err"]).max() < 1e-9
  out = mine.bundle_adjust(max_iterations=10)
  assert type(out.motion) is type(mine.motion) and type(out.cameras[0]) is type(mine.cameras[0])
  r = (np.asarray(out.reprojected.points) - np.asarray(out.point_table.points))[np.asarray(out.inliers)]
  assert abs(0.5 * float(np.sum(r ** 2)) - out.last_solve.cost) <= 1e-9 * out.last_solve.cost
  assert out.last_solve.cost < float(z[f"{motion}_cost0"])


def test_cfg1_the_reference_cpu_case_end_to_end():
  """BASELINE.json configs[0] (2 cameras x 20 frames of charuco_16x22, ~5k corners: the case the reference itself runs on the CPU):
  Calibration.bundle_adjust through the C-ABI against the reference algorithm (oracle: dense numpy evaluate + the identical scipy call)."""
  import numpy as np
  from multical_b200 import synthetic
  from multical_b200.calibration import from_scene
  from oracle.ba_oracle import Problem
  scene = synthetic.make_workload("cfg1")
  calib = from_scene(scene).enable(cameras=True)
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  assert np.array_equal(calib.param_vec, prob.param_vec)                                   # indexing / layout: bit exact
  eng = calib._upload(calib.inliers)
  assert 4000 < eng.N < 8000 and np.abs(eng.residuals() - prob.residuals()).max() < 1e-9
  out = calib.bundle_adjust()
  _, ref = prob.bundle_adjust()
  assert out.last_solve.cost <= ref.cost * (1 + 1e-6) and out.last_solve.nfev <= ref.nfev
  rms = np.sqrt(np.mean(out.reprojection_error ** 2))
  assert abs(rms - np.sqrt(2 * ref.cost / eng.N)) < 1e-3 and 0.3 < rms < 0.5              # 0.3 px noise per coordinate
