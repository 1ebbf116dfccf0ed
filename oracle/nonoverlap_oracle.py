"""numpy / scipy / cv2 restatement of the reference's non-overlapping camera initialisation (multical/hand_eye/hand_eye.py,
hand_eye/helper.py): test infrastructure for tests/test_gpu_nonoverlap.py and tests/test_simt_nonoverlap.py, never imported by the
package.  The solves call cv2.calibrateRobotWorldHandEye live, as the reference does; the vote calls scipy.stats.gaussian_kde live.

Edge cases where the reference fails without a clean message follow multical_b200/nonoverlap.py (DESIGN.md §3f): a (master, slave)
set of 3 transforms or fewer raises ValueError (the reference raises IndexError at 0, scipy raises at 1 and 2, and at 3 the covariance
is singular), 4 transforms (d + 1 points: equal densities in exact arithmetic) pick the lowest index within 1e-12 relative of the
maximum, and no camera qualifying as the reference raises ValueError."""
import cv2
import numpy as np
from scipy import stats

LIMIT_BOARD_IMAGE = 6
TIE_REL = 1e-12


def viewed_boards(valid):
  """check_viewed_boards: per camera, the boards valid in more than 6 images."""
  counts = np.asarray(valid, bool).sum(axis=1)
  return [[b for b in range(counts.shape[1]) if counts[c, b] > LIMIT_BOARD_IMAGE] for c in range(counts.shape[0])]


def quadruples(valid):
  """(master, slave, boardM, boardS) in the reference's loop order."""
  vb = viewed_boards(valid)
  C = len(vb)
  return [(m, s, bm, bs) for m in range(C) for s in range(C) if s != m for bm in vb[m] for bs in vb[s]]


def hand_eye_robot_world(A, B):
  """cv2.calibrateRobotWorldHandEye(SHAH) with cam_world = A, base_gripper = B ([n,4,4]) -> (X, Z) 4x4, or None where OpenCV raises."""
  try:
    xr, xt, zr, zt = cv2.calibrateRobotWorldHandEye(list(A[:, :3, :3]), list(A[:, :3, 3]), list(B[:, :3, :3]), list(B[:, :3, 3]),
                                                    method=cv2.CALIB_ROBOT_WORLD_HAND_EYE_SHAH)
  except cv2.error:
    return None
  X, Z = np.eye(4), np.eye(4)
  X[:3, :3], X[:3, 3], Z[:3, :3], Z[:3, 3] = xr, xt.reshape(-1), zr, zt.reshape(-1)
  return X, Z


def master_slave_pair(poses, valid, m, s, bm, bs):
  """-> (X, Z, image_ids), or None for fewer than 3 common images or where OpenCV raises."""
  ids = np.flatnonzero(valid[m, :, bm] & valid[s, :, bs])
  if len(ids) < 3:
    return None
  out = hand_eye_robot_world(np.linalg.inv(poses[m, ids, bm]), np.linalg.inv(poses[s, ids, bs]))
  return None if out is None else (*out, ids)


def kde_vote(points):
  """probabilistic_guess on translations [n,3] -> (densities [n], index of the densest)."""
  points = np.asarray(points, np.float64)
  if len(points) <= 3:
    raise ValueError(f"{len(points)} points: a 3-D kernel density estimate needs at least 4")
  density = stats.gaussian_kde(points.T)(points.T)
  best = int(np.flatnonzero(density >= density.max() * (1 - TIE_REL))[0])
  return density, best


def initialise_camera_poses(poses, valid, cam_names):
  """HandEye(...).initialise_camera_poses() -> dict(handeye_df, sets {(m, s): (X list, densities, best)}, reference_camera,
  camera_poses, cam_init)."""
  poses, valid = np.asarray(poses, np.float64), np.asarray(valid, bool)
  vb = viewed_boards(valid)
  df, sets, camera_poses = [], {}, {}
  max_density, max_group, reference = 0, 0, None
  for m, master in enumerate(cam_names):
    temp_density, temp_group = 0, 0
    camera_poses[master] = {master: np.eye(4).tolist()}
    for s, slave in enumerate(cam_names):
      if slave == master:
        continue
      xs = []
      for bm in vb[m]:
        for bs in vb[s]:
          r = master_slave_pair(poses, valid, m, s, bm, bs)
          if r is not None:
            df.append(dict(master_cam=master, slave_cam=slave, boardM=bm, boardS=bs, image_ids=r[2], slaveCam_wrt_masterCam=r[0]))
            xs.append(r[0])
      if len(xs) <= 3:
        raise ValueError(f"master camera {master}, slave camera {slave}: {len(xs)} hand-eye solutions, the vote needs at least 4")
      density, best = kde_vote(np.array([x[:3, 3] for x in xs]))
      sets[(m, s)] = (xs, density, best)
      camera_poses[master][slave] = xs[best].tolist()
      temp_density += density[best]
      temp_group += len(xs)
    if temp_density > max_density and temp_group > max_group:
      max_density, max_group, reference = temp_density, temp_group, master
  if reference is None:
    raise ValueError("no camera qualifies as the reference camera")
  camera_poses["Reference_camera"] = reference
  rel = {k: np.array(v) for k, v in camera_poses[reference].items()}
  new_pose = np.linalg.inv(rel[cam_names[0]])
  cam_init = {k: np.linalg.inv(new_pose @ v) for k, v in rel.items()}
  return dict(handeye_df=df, sets=sets, reference_camera=reference, camera_poses=camera_poses, cam_init=cam_init)
