"""Triangulating points of a calibrated rig on the GPU (DESIGN.md §3j).

`triangulate_points` is a drop-in for cv2.triangulatePoints: two 3x4 projection matrices, the linear (DLT) solution, no distortion.
`triangulate` takes pixels seen by any number of cameras of a calibrated rig through their full camera model: the linear solution of
the undistorted views, refined by Levenberg-Marquardt on the reprojection error in pixels.  `Calibration.triangulate()` applies it to a
calibration's own detections.  The kernels are in csrc/triangulate_kernels.cuh; everything runs on the undistortion engine, so the
bundle adjustment engine's uploaded problem survives it."""
import numpy as np

from .structs import struct
from .undistort import camera_vector, undistort_engine


def triangulate_points(projMatr1, projMatr2, projPoints1, projPoints2):
  """cv2.triangulatePoints(projMatr1, projMatr2, projPoints1, projPoints2): 3x4 projection matrices and points [2, N] -> homogeneous
  points [4, N] of unit norm (their sign is unspecified, as OpenCV's).  Computed in fp64; float32 points give float32 out, as OpenCV
  does."""
  P1, P2 = np.asarray(projMatr1, np.float64), np.asarray(projMatr2, np.float64)
  x1, x2 = np.asarray(projPoints1), np.asarray(projPoints2)
  if P1.shape != (3, 4) or P2.shape != (3, 4):
    raise ValueError(f"projection matrices must be 3x4, got {P1.shape} and {P2.shape}")
  if x1.ndim != 2 or x1.shape[0] != 2 or x1.shape != x2.shape:
    raise ValueError(f"points must be two arrays [2, N] of one shape, got {x1.shape} and {x2.shape}")
  out = undistort_engine().triangulate_linear(P1, P2, x1, x2)
  return out.astype(np.float32) if x1.dtype == np.float32 else out


def triangulate(cameras, camera_poses, pixels, valid):
  """N-view triangulation through the full camera model.  cameras: C (reference or mirror) cameras of one model; camera_poses
  [C, 4, 4] rig -> camera (x_cam = T_c x_rig); pixels [C, N, 2]; valid [C, N] bool.  Returns struct(points [N, 3] f64 in the rig frame,
  valid [N] bool, rms [N] px over the point's views).  A point needs at least two views; where it is invalid, points and rms are NaN."""
  vectors = [camera_vector(c) for c in cameras]
  models = [m for m, _ in vectors]
  if len(set(models)) > 1:
    groups = {m: [i for i, mi in enumerate(models) if mi == m] for m in dict.fromkeys(models)}
    raise NotImplementedError("triangulation needs one camera model for all cameras, got "
                              + "; ".join(f"{m} for cameras {idx}" for m, idx in groups.items()))
  C = len(vectors)
  poses, pixels, valid = np.asarray(camera_poses), np.asarray(pixels), np.asarray(valid)
  if C == 0:
    raise ValueError("no cameras")
  if poses.shape != (C, 4, 4):
    raise ValueError(f"camera_poses must be [{C}, 4, 4] for {C} cameras, got {poses.shape}")
  if pixels.ndim != 3 or pixels.shape[0] != C or pixels.shape[2] != 2:
    raise ValueError(f"pixels must be [{C}, N, 2] for {C} cameras, got {pixels.shape}")
  if valid.shape != pixels.shape[:2]:
    raise ValueError(f"valid must be {pixels.shape[:2]} like pixels [C, N], got {valid.shape}")
  points, ok, rms = undistort_engine().triangulate(models[0], np.stack([v for _, v in vectors]), poses, pixels, valid.astype(bool))
  return struct(points=points, valid=ok, rms=rms)
