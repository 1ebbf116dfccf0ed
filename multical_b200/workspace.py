"""The `Workspace` methods around the hot path, as functions over a `Calibration` or the detections (the rest of the reference's
`Workspace` -- image loading, detection, export -- is out of scope and stays the reference's own):
  calibrate_single(boards, detected_points, ...)   = Workspace.calibrate_single   multical/workspace.py:165-194 (the pinhole and,
                                    with isFisheye, the fisheye branch: every camera's intrinsics, multical_b200/intrinsics.py)

  calibrate(calib, ...)          = Workspace.calibrate          multical/workspace.py:228-247  (enable the chosen blocks, then the outlier
                                    loop around bundle_adjust with the quantile selectors the command line builds, config/workspace.py:47-58)
  pose_table(point_table, ...)   = the first statement of Workspace.initialise_poses   multical/workspace.py:196-198  (tables.make_pose_table:
                                    one board pose per view, here in one launch -- multical_b200/tables.py)
  initialise_poses(point_table, ...) = Workspace.initialise_poses  multical/workspace.py:196-226 (pose table, pose graph, initial Calibration;
                                    is_non_overlapping: the camera poses of nonoverlap.HandEye, workspace.py:203-207)

A `Workspace` keeps working unchanged when its module imports `Calibration`, `select_threshold` and `tables.make_pose_table` from this
package (INTEGRATION.md A, D); these functions are the same steps for callers that do not carry a `Workspace` around (bench.py, tests)."""
import numpy as np

from .calibration import Calibration, select_threshold
from .intrinsics import calibrate_cameras, calibrate_cameras_fisheye
from .log import info
from .nonoverlap import HandEye
from .parameters import ParamList
from .pose_set import PoseSet, StaticFrames
from .tables import initialise_poses as _initialise_poses, make_pose_table


def calibrate_single(boards, detected_points, image_sizes, camera_model, intrinsic_error_limit, fix_aspect=False, has_skew=False,
                     max_images=None, isFisheye=False):
  """workspace.py:165-189: every camera's intrinsics from its detections[frame][board] -> (cameras, errs).  isFisheye routes to
  calibrate_cameras_fisheye, which takes no error limit (CameraOpts.isFisheye, config/arguments.py:36)."""
  if isFisheye:
    return calibrate_cameras_fisheye(boards, detected_points, image_sizes, model=camera_model, fix_aspect=fix_aspect, has_skew=has_skew,
                                     max_images=max_images)
  return calibrate_cameras(boards, detected_points, image_sizes, intrinsic_error_limit, model=camera_model, fix_aspect=fix_aspect,
                           has_skew=has_skew, max_images=max_images)


def calibrate(calib: Calibration, camera_poses=True, motion=True, board_poses=True, cameras=False, boards=False,
              loss="linear", tolerance=1e-4, num_adjustments=3, quantile=0.75, auto_scale=None, outlier_threshold=5.0,
              tr_solver="lsmr") -> Calibration:
  """workspace.py:228-247: same arguments, defaults and order of operations; tr_solver as Calibration.bundle_adjust."""
  calib = calib.enable(cameras=cameras, boards=boards, camera_poses=camera_poses, motion=motion, board_poses=board_poses)
  return calib.adjust_outliers(
    loss=loss, tolerance=tolerance, num_adjustments=num_adjustments, tr_solver=tr_solver,
    select_outliers=select_threshold(quantile=quantile, factor=outlier_threshold),
    select_scale=select_threshold(quantile=quantile, factor=auto_scale) if auto_scale is not None else None)


def optimize(calib: Calibration, iter=3, loss="linear", outlier_quantile=0.75, outlier_threshold=5.0, auto_scale=None,
             fix_intrinsic=False, fix_camera_poses=False, fix_board_poses=False, fix_motion=False, adjust_board=False,
             tr_solver="lsmr") -> Calibration:
  """config/workspace.py:47-58 with the fields of OptimizerOpts (config/arguments.py:53-69) as keyword arguments.  Like the reference's
  `optimize`, the `iter` option is NOT forwarded: Workspace.calibrate runs its own default of 3 adjustments."""
  del iter
  return calibrate(calib, loss=loss, boards=adjust_board, cameras=not fix_intrinsic, camera_poses=not fix_camera_poses,
                   board_poses=not fix_board_poses, motion=not fix_motion, auto_scale=auto_scale,
                   outlier_threshold=outlier_threshold, quantile=outlier_quantile, tr_solver=tr_solver)


def pose_table(point_table, boards, cameras, exclude_bad_poses=True, pose_error_limit=1.0):
  """workspace.py:196-198 (the defaults are initialise_poses' own: bad poses excluded, limit 1 px)."""
  return make_pose_table(point_table, boards, cameras, exclude_bad_poses, pose_error_limit)


def table_info(valid, camera_names, board_names):
  """tables.table_info (tables.py:190-204): view counts per camera and board."""
  valid = np.asarray(valid)
  info(f"Total: {int(valid.sum())}, cameras: {dict(zip(camera_names, valid.sum(axis=(1, 2)).tolist()))}, "
       f"Boards: {dict(zip(board_names, valid.sum(axis=(0, 1)).tolist()))}")
  if len(camera_names) > 1 and len(board_names) > 1:
    info("Camera-board matrix")
    info(valid.sum(axis=1))


def initialise_poses(point_table, boards, cameras, motion_model=StaticFrames, camera_poses=None, exclude_bad_poses=True,
                     pose_error_limit=1.0, camera_names=None, board_names=None, image_names=None, is_non_overlapping=False,
                     image_path=None):
  """workspace.py:196-226: make_pose_table, initialise_poses, then the initial Calibration (reported as "Initialisation").
  camera_poses: {camera name: 4x4} or a [C,4,4] array in camera order.  is_non_overlapping (used only without camera_poses): the
  camera poses come from nonoverlap.HandEye, which writes camera_groups.pkl and initial_guess.json into image_path when it is given."""
  camera_names = camera_names or [str(i) for i in range(len(cameras))]
  board_names = board_names or [str(i) for i in range(len(boards))]
  table = make_pose_table(point_table, boards, cameras, exclude_bad_poses, pose_error_limit)
  info("Pose counts:")
  table_info(table.valid, camera_names, board_names)
  if is_non_overlapping and camera_poses is None:
    handeye = HandEye(table, camera_names, image_path)
    handeye.initialise_camera_poses()
    camera_poses = handeye.cam_init
  if isinstance(camera_poses, dict):
    camera_poses = np.array([camera_poses[k] for k in camera_names])
  init = _initialise_poses(table, camera_poses=camera_poses)
  calib = Calibration(ParamList(cameras, camera_names), ParamList(boards, board_names), point_table, PoseSet(init.camera, camera_names), PoseSet(init.board, board_names),
                      motion_model.init(init.times, image_names))
  calib.report("Initialisation")
  return calib
