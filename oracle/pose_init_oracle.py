"""numpy + scipy restatement of the reference's pose-graph initialisation (tables.initialise_poses, tables.py:354-377), written from its
semantics: the CPU suite pins it to the goldens of tests/golden/make_pose_init_golden.py, the GPU suite compares the device against it
at full size.

  align_transforms_robust(m1, m2, valid)   transform/matrix.py:140-153
  mean_robust(m)                           transform/matrix.py:109-113 + transform/common.py:6-19 (whiten, Ward, maxclust, Counter)
  estimate_relative_poses(table, axis)     tables.py:207-225 (pattern_overlaps 131-144, graph.select_pairs, estimate_transform 149-174)
  initialise_poses(table, camera_poses)    tables.py:354-377
"""
from collections import Counter

import numpy as np
from scipy.cluster.hierarchy import fcluster, linkage
from scipy.spatial.transform import Rotation


def to_rtvec(m):
  return np.hstack([Rotation.from_matrix(m[:, :3, :3]).as_rotvec(), m[:, :3, 3]])


def to_matrix(rt):
  out = np.zeros((4, 4))
  out[:3, :3] = Rotation.from_rotvec(rt[:3]).as_matrix()
  out[:3, 3] = rt[3:]
  out[3, 3] = 1.0
  return out


def largest_cluster(v):
  """mask of mean_robust's cluster of the rows of v (n >= 2)."""
  sd = v.std(axis=0)
  sd[sd == 0] = 1.0
  z = linkage(v / sd, "ward")
  labels = fcluster(z, t=max(v.shape[0] / 10, 3), criterion="maxclust")
  most = Counter(labels).most_common(1)[0][0]
  return labels == most


def mean_robust(m):
  v = to_rtvec(m)
  return to_matrix(v[0] if len(v) == 1 else v[largest_cluster(v)].mean(axis=0))


def align_transforms_robust(m1, m2, valid=None, threshold=1.5):
  mask = np.ones(m1.shape[0], bool) if valid is None else np.asarray(valid, bool)
  m = mean_robust(m2[mask] @ np.linalg.inv(m1[mask]))
  errs = np.linalg.norm(m @ m1 - m2, axis=(1, 2))
  inliers = (errs < np.quantile(errs, 0.75) * threshold) & mask
  return mean_robust(m2[inliers] @ np.linalg.inv(m1[inliers])), inliers


def pattern_overlaps(valid, num_points, axis):
  n = valid.shape[axis]
  v, p = np.moveaxis(valid, axis, 0).reshape(n, -1), np.moveaxis(num_points, axis, 0).reshape(n, -1)
  out = np.zeros((n, n))
  for i in range(n):
    for j in range(i + 1, n):
      out[i, j] = out[j, i] = np.sum((v[i] & v[j]).astype(np.float32) * np.minimum(p[i], p[j]))
  return out


def select_pairs(overlaps, hop_penalty):
  overlaps = overlaps.copy()
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


def relative_poses(poses, valid, num_points, axis, hop_penalty=0.9, calls=None):
  """estimate_relative_poses on a table of [C,F,B,4,4] poses -> (poses [n,4,4], valid [n], master, pairs)."""
  n = valid.shape[axis]
  master, pairs = select_pairs(pattern_overlaps(valid, num_points, axis), hop_penalty)
  P, V = np.moveaxis(poses, axis, 0).reshape(n, -1, 4, 4), np.moveaxis(valid, axis, 0).reshape(n, -1)
  est = {master: np.eye(4)}
  for parent, child in pairs:
    t, inl = align_transforms_robust(P[parent], P[child], V[parent] & V[child])
    if calls is not None: calls.append((t, inl))
    est[child] = t @ est[parent]
  out = np.broadcast_to(np.eye(4), (n, 4, 4)).copy()
  ok = np.zeros(n, bool)
  for k, m in est.items(): out[k], ok[k] = m, True
  return out @ np.linalg.inv(out[0]), ok, master, pairs


def initialise_poses(poses, valid, num_points, camera_poses=None):
  """-> dict(camera=(poses, valid), board=(poses, valid), times=(poses, valid), camera_master/pairs, board_master/pairs)."""
  poses, valid, num_points = np.asarray(poses, np.float64), np.asarray(valid, bool), np.asarray(num_points)
  cam, cam_ok, cm, cp = relative_poses(poses, valid, num_points, 0)
  if camera_poses is not None:
    cam, cam_ok = np.asarray(camera_poses, np.float64), np.ones(len(camera_poses), bool)
  inv_poses = np.linalg.inv(poses)
  board, board_ok, bm, bpairs = relative_poses(inv_poses, valid, num_points, 2)
  board = np.linalg.inv(board)
  rel = poses @ np.linalg.inv(board)[None, None]
  rel_ok = valid & board_ok[None, None]
  C, F, B = valid.shape
  times, times_ok = np.broadcast_to(np.eye(4), (F, 4, 4)).copy(), np.zeros(F, bool)
  for f in range(F):
    c, b = np.nonzero(cam_ok[:, None] & rel_ok[:, f, :])
    if c.size == 0: continue
    t, _ = align_transforms_robust(np.linalg.inv(cam[c]), np.linalg.inv(rel[c, f, b]))
    times[f], times_ok[f] = np.linalg.inv(t), True
  return dict(camera=(cam, cam_ok), board=(board, board_ok), times=(times, times_ok), camera_master=cm, camera_pairs=cp,
              board_master=bm, board_pairs=bpairs)
