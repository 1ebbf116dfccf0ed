"""`make_pose_table` and `initialise_poses` with the reference's signatures and results (multical/tables.py:44-66, 354-377): the
per-view board poses that initialise the bundle adjustment (workspace.py:196-226), computed in one launch on the GPU (include/mcba.h
mcba_pnp_views) instead of C*F*B calls of `board.estimate_pose_points` (board/common.py:36-47), and the camera, board and rig poses
built from them.  Every align_transforms_robust of the pose graph runs on the GPU (mcba_pose_pairs, mcba_pose_times: Ward clustering
without a distance matrix, DESIGN.md §3e); only pattern_overlaps and the spanning tree of graph.select_pairs stay on the host."""
import numpy as np
from scipy.spatial.transform import Rotation

from .board import stack_boards
from .calibration import get_engine
from .camera import engine_model_of
from .log import info
from .structs import Table, struct


def board_grid_of(board):
  """{id-grid width, height, id divisor, min_points, min_rows} of `board.has_min_detections` (charuco.py:104-106: corner ids on
  the (w, h) = board.size grid; aprilgrid.py:197-199: tag ids = corner ids // 4)."""
  w, h = (int(v) for v in board.size)
  return [w, h, int(getattr(board, "id_divisor", 1)), int(board.min_points), int(board.min_rows)]


def detection_lists(point_table):
  """Dense [C,F,B,P] table -> CSR detection lists in (c, f, b) order: what tables.sparse_points (tables.py:34-36) extracts view by view."""
  valid = np.asarray(point_table.valid)
  pts = np.asarray(point_table.points)
  counts = valid.reshape(-1, valid.shape[-1]).sum(axis=1)
  det_start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
  idx = np.argwhere(valid)
  return det_start, idx[:, 3].astype(np.int32), np.ascontiguousarray(pts[valid])


def make_pose_table(point_table, boards, cameras, exclude_bad_poses=False, pose_error_limit=1.0):
  """tables.py:44-66.  Returns Table(poses [C,F,B,4,4], valid, num_points, reprojection_error, view_angles [C,F,B,3]); a view without
  the minimum detections, or (exclude_bad_poses) with error above pose_error_limit, is the reference's invalid_pose."""
  valid = np.asarray(point_table.valid)
  Cn, F, B, P = valid.shape
  models = {engine_model_of(c) for c in cameras}
  assert len(models) == 1, f"all cameras must share one model, got {models}"
  det_start, det_ids, det_xy = detection_lists(point_table)
  bp, _ = stack_boards(boards)
  intr = np.stack([np.asarray(c.param_vec, np.float64) for c in cameras])
  grid = np.array([board_grid_of(b) for b in boards], np.int32)
  poses, err, npts, ok = get_engine().pnp_views(models.pop(), (Cn, F, B, P), det_start, det_ids, det_xy, bp, intr, grid)
  if exclude_bad_poses:
    ok = ok & ~(err > pose_error_limit)
  poses = np.where(ok[..., None, None], poses, np.eye(4))
  angles = np.zeros((Cn, F, B, 3))
  if ok.any():                                       # rtvec.rtvec_to_euler (transform/rtvec.py:55-58)
    angles[ok] = Rotation.from_matrix(poses[ok][:, :3, :3]).as_euler("xyz", degrees=True)
  return Table.create(poses=poses, valid=ok, num_points=np.where(ok, npts, 0), reprojection_error=np.where(ok, err, 0.0), view_angles=angles)


def pattern_overlaps(valid, num_points, axis=0):
  """tables.py:131-144, vectorised: overlaps[i, j] = sum of valid_i valid_j min(num_points_i, num_points_j) (integer sums: exact)."""
  n = valid.shape[axis]
  v = np.moveaxis(np.asarray(valid, bool), axis, 0).reshape(n, -1).astype(np.int64)
  p = np.moveaxis(np.asarray(num_points), axis, 0).reshape(n, -1).astype(np.int64)
  out = np.zeros((n, n))
  for i in range(n):
    out[i] = (v[i] * v * np.minimum(p[i], p)).sum(axis=1)
  out[np.arange(n), np.arange(n)] = 0
  return out


def select_pairs(overlaps, hop_penalty=0.9):
  """graph.py:7-30: the master (most overlap) and a greedy spanning tree with a hop penalty; ties go to the first argmax."""
  overlaps = np.array(overlaps, dtype=np.float64)
  n = overlaps.shape[0]
  master = int(np.argmax(overlaps.sum(1)))
  weight = (np.arange(n) == master).astype(np.float32).reshape(n, 1)
  overlaps[:, master] = 0
  pairs = []
  while len(pairs) + 1 < n:
    w = overlaps * weight
    parent, child = np.unravel_index(np.argmax(w), w.shape)
    if w[parent, child] <= 0: break
    overlaps[:, child] = 0
    weight[child] = weight[parent] * hop_penalty
    pairs.append((int(parent), int(child)))
  return master, pairs


def _rms(x): return np.sqrt(np.square(x).mean())


def _pose_errors(p1, p2):
  """matrix.pose_errors (transform/matrix.py:156-166): Frobenius norm, rotation angle (degrees) and translation of p1 inv(p2)."""
  d = p1 @ np.linalg.inv(p2)
  r, t = d[:, :3, :3], d[:, :3, 3]
  angle = np.linalg.norm(Rotation.from_matrix(r).as_rotvec(), axis=-1) if len(d) else np.zeros(0)
  return dict(frobius=_rms(np.linalg.norm(d - np.eye(4), axis=(1, 2))), rotation_deg=_rms(np.degrees(angle)),
              translation=_rms(np.linalg.norm(t, axis=-1)))


def relative_poses(pose_table, axis=0, hop_penalty=0.9):
  """estimate_relative_poses (axis 0) / estimate_relative_poses_inv (axis 2), tables.py:207-228 -> Table(poses [n,4,4], valid [n])."""
  poses, valid = np.asarray(pose_table.poses, np.float64), np.asarray(pose_table.valid, bool)
  name = {0: "camera", 2: "board"}[axis]
  n = valid.shape[axis]
  overlaps = pattern_overlaps(valid, pose_table.num_points, axis)
  info(f"Overlaps by {name}:")
  info(overlaps)
  master, pairs = select_pairs(overlaps, hop_penalty)
  info(f"Selected master {master} and pairs {pairs}")
  est = {master: np.eye(4)}
  if pairs:
    ts, inliers, _ = get_engine().pose_pairs(poses, valid, axis, pairs)
    flat_p = np.moveaxis(np.linalg.inv(poses) if axis == 2 else poses, axis, 0).reshape(n, -1, 4, 4)
    flat_v = np.moveaxis(valid, axis, 0).reshape(n, -1)
    for (parent, child), t, inl in zip(pairs, ts, inliers):
      pi, pj, ok = flat_p[parent], flat_p[child], flat_v[parent] & flat_v[child]
      err, err_inl = _pose_errors(t @ pi[ok], pj[ok]), _pose_errors(t @ pi[inl], pj[inl])
      info(f"Estimate transform axis={axis}, pair {(parent, child)}, inliers {inl.sum()}/{ok.sum()}")
      info(f"RMS (frobius): {err_inl['frobius']:.4f} ({err['frobius']:.4f})"
           f" (deg): {err_inl['rotation_deg']:.4f} ({err['rotation_deg']:.4f})"
           f" (trans): {err_inl['translation']:.4f} ({err['translation']:.4f})")
      info(t)
      est[child] = t @ est[parent]
  out = np.broadcast_to(np.eye(4), (n, 4, 4)).copy()
  ok = np.zeros(n, bool)
  for k, m in est.items(): out[k], ok[k] = m, True
  out = out @ np.linalg.inv(out[0])
  return Table.create(poses=np.linalg.inv(out) if axis == 2 else out, valid=ok)


def initialise_poses(pose_table, camera_poses=None):
  """tables.py:354-377: struct(times, camera, board) from a make_pose_table result; camera_poses [C,4,4] replaces the camera estimate."""
  camera = relative_poses(pose_table, axis=0)
  if camera_poses is not None:
    camera_poses = np.asarray(camera_poses, np.float64)
    info("Camera initialisation vs. supplied calibration")
    for i in range(camera_poses.shape[0]):
      e = _pose_errors(camera_poses[i:i + 1], camera.poses[i:i + 1])
      info(f"camera {i}: frobius {e['frobius']:.4f}, rotation (deg): {e['rotation_deg']:.4f}, translation: {e['translation']:.4f}")
    camera = Table.create(poses=camera_poses, valid=np.ones(camera_poses.shape[0], dtype=bool))
  board = relative_poses(pose_table, axis=2)
  times, ok = get_engine().pose_times(pose_table.poses, pose_table.valid, camera.poses, camera.valid, board.poses, board.valid)
  F = ok.shape[0]
  times = Table.create(poses=times, valid=ok, num_points=np.zeros(F, np.int64), reprojection_error=np.zeros(F),
                       view_angles=np.zeros((F, 3)))
  return struct(times=times, camera=camera, board=board)
