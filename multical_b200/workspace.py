"""The `Workspace` methods around the hot path, as functions over a `Calibration` or the detections (the rest of the reference's
`Workspace` -- image loading, detection, export -- is out of scope and stays the reference's own):
  calibrate_single(boards, detected_points, ...)   = Workspace.calibrate_single   multical/workspace.py:165-194 (the pinhole branch:
                                    every camera's intrinsics, multical_b200/intrinsics.py)

  calibrate(calib, ...)          = Workspace.calibrate          multical/workspace.py:228-247  (enable the chosen blocks, then the outlier
                                    loop around bundle_adjust with the quantile selectors the command line builds, config/workspace.py:47-58)
  pose_table(point_table, ...)   = the first statement of Workspace.initialise_poses   multical/workspace.py:196-198  (tables.make_pose_table:
                                    one board pose per view, here in one launch -- multical_b200/tables.py)

A `Workspace` keeps working unchanged when its module imports `Calibration`, `select_threshold` and `tables.make_pose_table` from this
package (INTEGRATION.md A, D); these functions are the same steps for callers that do not carry a `Workspace` around (bench.py, tests)."""
from .calibration import Calibration, select_threshold
from .intrinsics import calibrate_cameras
from .tables import make_pose_table


def calibrate_single(boards, detected_points, image_sizes, camera_model, intrinsic_error_limit, fix_aspect=False, has_skew=False,
                     max_images=None):
  """workspace.py:165-180 (the pinhole branch): every camera's intrinsics from its detections[frame][board] -> (cameras, errs)."""
  return calibrate_cameras(boards, detected_points, image_sizes, intrinsic_error_limit, model=camera_model, fix_aspect=fix_aspect,
                           has_skew=has_skew, max_images=max_images)


def calibrate(calib: Calibration, camera_poses=True, motion=True, board_poses=True, cameras=False, boards=False,
              loss="linear", tolerance=1e-4, num_adjustments=3, quantile=0.75, auto_scale=None, outlier_threshold=5.0) -> Calibration:
  """workspace.py:228-247: same arguments, defaults and order of operations."""
  calib = calib.enable(cameras=cameras, boards=boards, camera_poses=camera_poses, motion=motion, board_poses=board_poses)
  return calib.adjust_outliers(
    loss=loss, tolerance=tolerance, num_adjustments=num_adjustments,
    select_outliers=select_threshold(quantile=quantile, factor=outlier_threshold),
    select_scale=select_threshold(quantile=quantile, factor=auto_scale) if auto_scale is not None else None)


def optimize(calib: Calibration, iter=3, loss="linear", outlier_quantile=0.75, outlier_threshold=5.0, auto_scale=None,
             fix_intrinsic=False, fix_camera_poses=False, fix_board_poses=False, fix_motion=False, adjust_board=False) -> Calibration:
  """config/workspace.py:47-58 with the fields of OptimizerOpts (config/arguments.py:53-69) as keyword arguments.  Like the reference's
  `optimize`, the `iter` option is NOT forwarded: Workspace.calibrate runs its own default of 3 adjustments."""
  del iter
  return calibrate(calib, loss=loss, boards=adjust_board, cameras=not fix_intrinsic, camera_poses=not fix_camera_poses,
                   board_poses=not fix_board_poses, motion=not fix_motion, auto_scale=auto_scale,
                   outlier_threshold=outlier_threshold, quantile=outlier_quantile)


def pose_table(point_table, boards, cameras, exclude_bad_poses=True, pose_error_limit=1.0):
  """workspace.py:196-198 (the defaults are initialise_poses' own: bad poses excluded, limit 1 px)."""
  return make_pose_table(point_table, boards, cameras, exclude_bad_poses, pose_error_limit)
