"""numpy restatement of the start of stereo calibration (csrc/stereo_kernels.cuh k_stereo_start; cv2.stereoCalibrate's initial pose):
per view the relative pose of the right camera to the left one, then the median of each of its six rtvec components."""
import numpy as np
from scipy.spatial.transform import Rotation


def relative_poses(left, right):
  """left, right [F, 4, 4] board wrt camera -> rtvecs [F, 6] of R = R2 R1^T, T = T2 - R T1 (x_right = R x_left + T)."""
  left, right = np.asarray(left, np.float64), np.asarray(right, np.float64)
  R = right[:, :3, :3] @ np.transpose(left[:, :3, :3], (0, 2, 1))
  T = right[:, :3, 3] - np.einsum("fij,fj->fi", R, left[:, :3, 3])
  return np.hstack([Rotation.from_matrix(R).as_rotvec(), T])


def median_start(left, right, ok):
  """The start over the views where ok: each component's median, the two middle values averaged for an even count."""
  rt = relative_poses(left, right)[np.asarray(ok, bool)]
  return np.median(rt, axis=0)
