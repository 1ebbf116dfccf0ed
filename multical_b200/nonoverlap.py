"""`HandEye` with the reference's surface (multical/hand_eye/hand_eye.py, hand_eye/helper.py): the camera poses of a rig whose
cameras rarely see the same board in the same frame, from robot-world hand-eye solves between every pair of (camera, board) view
sequences.  Workspace.initialise_poses (workspace.py:203-207) runs it when is_non_overlapping is set and passes its `cam_init` to
tables.initialise_poses as the camera poses.

Every cv2.calibrateRobotWorldHandEye(SHAH) of master_slave_pair runs on the GPU in one launch (include/mcba.h mcba_hand_eye_quads), and
so does every probabilistic_guess (gaussian_kde vote, mcba_hand_eye_vote).  The host keeps check_viewed_boards, the quadruple list in
the reference's loop order, the image ids, the reference-camera choice, relative_to_cam and the final inversions.  The module is not
named hand_eye because multical_b200.hand_eye and multical_b200.motion.HandEye (the motion model) already exist.

Where the reference fails without a clean message, this raises ValueError (DESIGN.md §3f): a (master, slave) pair with 3 accepted
solves or fewer (the reference raises IndexError at 0 and scipy raises at 1 to 3) and a rig where no camera qualifies as the
reference (the reference raises KeyError after writing its files)."""
import json
import os
import pickle

import numpy as np

from .calibration import get_engine
from .log import info

LIMIT_BOARD_IMAGE = 6          # check_viewed_boards: a board counts when a camera sees it in more than this many images


class HandEye:
  def __init__(self, pose_table, cam_name, image_path=None):
    self.cam_names = list(cam_name)
    self.pose_table = pose_table
    self.image_path = image_path
    self.num_cameras, self.num_images, self.num_boards = np.asarray(pose_table.valid).shape
    assert len(self.cam_names) == self.num_cameras, f"{len(self.cam_names)} camera names for {self.num_cameras} cameras"
    self.viewed_boards = self.check_viewed_boards()
    self.camera_poses = {}
    self.camera_groups = {}
    self.reference_camera = None
    self.cam_init = {}
    self.handeye_df = []

  def check_viewed_boards(self):
    counts = np.asarray(self.pose_table.valid, bool).sum(axis=1)
    return {cam: [b for b in range(self.num_boards) if counts[idx, b] > LIMIT_BOARD_IMAGE] for idx, cam in enumerate(self.cam_names)}

  def quadruples(self):
    """(master, slave, boardM, boardS) indices in the reference's loop order (master, slave, boardM, boardS)."""
    return [(m, s, bm, bs) for m, master in enumerate(self.cam_names) for s, slave in enumerate(self.cam_names) if slave != master
            for bm in self.viewed_boards[master] for bs in self.viewed_boards[slave]]

  def initialise_camera_poses(self):
    valid = np.asarray(self.pose_table.valid, bool)
    quads = self.quadruples()
    X, _, _, ok = get_engine().hand_eye_quads(self.pose_table.poses, valid, np.array(quads, np.int32).reshape(-1, 4))
    groups = {}                                      # (master, slave) -> accepted X, in the reference's order
    for (m, s, bm, bs), x, good in zip(quads, X, ok):
      g = groups.setdefault((m, s), [])
      if good:
        master, slave = self.cam_names[m], self.cam_names[s]
        self.handeye_df.append({"master_cam": master, "slave_cam": slave, "boardM": bm, "boardS": bs,
                                "image_ids": np.flatnonzero(valid[m, :, bm] & valid[s, :, bs]), "slaveCam_wrt_masterCam": x})
        g.append(x)
    pairs = [(m, s) for m, master in enumerate(self.cam_names) for s, slave in enumerate(self.cam_names) if slave != master]
    for m, s in pairs:
      n = len(groups.get((m, s), []))
      if n <= 3:
        raise ValueError(f"master camera {self.cam_names[m]}, slave camera {self.cam_names[s]}: {n} hand-eye solutions, "
                         "the vote needs at least 4")
    density, best = get_engine().hand_eye_vote([np.array([x[:3, 3] for x in groups[p]]) for p in pairs]) if pairs else ([], [])
    pick = {p: (float(d[b]), groups[p][b]) for p, d, b in zip(pairs, density, best)}

    max_density, max_group = 0, 0
    for m, master in enumerate(self.cam_names):
      temp_density, temp_group = 0, 0
      self.camera_poses[master] = {}
      self.camera_groups[master] = {}
      self.camera_poses[master][master] = np.eye(4).tolist()
      for s, slave in enumerate(self.cam_names):
        if slave != master:
          self.camera_groups[master][slave] = [g.tolist() for g in groups[(m, s)]]
          d, x = pick[(m, s)]
          self.camera_poses[master][slave] = x.tolist()
          temp_density += d
          temp_group += len(groups[(m, s)])
      if temp_density > max_density and temp_group > max_group:
        max_density, max_group, self.reference_camera = temp_density, temp_group, master
    if self.reference_camera is None:
      raise ValueError("no camera qualifies as the reference camera: none has a positive density sum and group count")

    self.camera_poses["Reference_camera"] = self.reference_camera
    if self.image_path is not None:
      with open(os.path.join(self.image_path, "camera_groups.pkl"), "wb") as f:
        pickle.dump(self.camera_groups, f)
      with open(os.path.join(self.image_path, "initial_guess.json"), "w") as fp:
        json.dump(self.camera_poses, fp)
    del self.camera_groups

    info(f"Reference camera {self.reference_camera} with density {max_density} and number of groups {max_group}")
    init0 = relative_to_cam(self.cam_names[0], self.camera_poses[self.reference_camera])
    for k in self.cam_names:                         # Multical's camera poses are masterCam_wrt_slaveCam
      init0[k] = np.linalg.inv(init0[k])
    self.cam_init = init0


def relative_to_cam(new_ref, camera_poses):
  """hand_eye/helper.py:20-24 (in place, as the reference does)."""
  new_pose = np.linalg.inv(camera_poses[new_ref])
  for k, v in camera_poses.items():
    camera_poses[k] = new_pose @ camera_poses[k]
  return camera_poses
