"""Synthetic multi-camera calibration scenes {N_cam, N_frame, N_board, K_corners}.

Produces plain-numpy dictionaries shaped like the reference's inputs to
`Calibration(...)` (reference: multical/optimization/calibration.py:44-61):
  points f64[C,F,B,P,2] + valid bool[C,F,B,P]      (tables.make_point_table, tables.py:68-81)
  board_points  list of f64[P_b,3]                 (board.adjusted_points, board/charuco.py:56-58)
  cam/frame/board poses f64[*,4,4] + valid flags   (PoseSet, optimization/pose_set.py:12-16)
  K f64[C,3,3], dist f64[C,nd]                     (Camera, camera.py:27-40)
Pose chain (tables.py:368-371): x_cam = T_cam[c] @ T_frame[f] @ T_board[b] @ [X;1].

This module is data tooling for tests and bench.py, not part of the solver; it carries its
own small numpy projection so that nothing in the product imports `oracle/`.
"""
import numpy as np
from scipy.spatial.transform import Rotation

WORKLOADS = {
  # name: BASELINE.json configs[i]; vis tuned so that measured N lands near the nominal count
  "cfg1": dict(C=2, F=20, boards=("charuco", 16, 22, 0.025, 1), model="standard", vis=0.50, rig="arc"),
  "cfg2": dict(C=4, F=200, boards=("charuco", 16, 22, 0.025, 1), model="standard", vis=0.65, rig="arc"),
  "cfg3": dict(C=8, F=500, boards=("charuco", 16, 22, 0.025, 1), model="fisheye", vis=0.85, rig="arc"),
  "cfg4": dict(C=16, F=1000, boards=("cube", 10, 10, 0.040, 5), model="standard", vis=0.85, rig="dome"),
  "cfg5": dict(C=64, F=2000, boards=("charuco", 20, 22, 0.020, 1), model="standard", vis=0.995, rig="dome"),
}


def grid_board_points(w, h, square):
  """(w-1)(h-1) inner corners at ((x+1)s,(y+1)s,0), x fastest, rounded through float32 like
  cv2's chessboardCorners (board/charuco.py:56-58, tables.py:389)."""
  xs, ys = np.meshgrid(np.arange(1, w, dtype=np.float32), np.arange(1, h, dtype=np.float32))
  pts = np.stack([xs.ravel() * np.float32(square), ys.ravel() * np.float32(square),
                  np.zeros(xs.size, np.float32)], axis=1)
  return pts.astype(np.float64)


def to_matrix(rtvec):
  rtvec = np.asarray(rtvec, np.float64).reshape(-1, 6)
  T = np.tile(np.eye(4), (rtvec.shape[0], 1, 1))
  T[:, :3, :3] = Rotation.from_rotvec(rtvec[:, :3]).as_matrix()
  T[:, :3, 3] = rtvec[:, 3:]
  return T


def from_matrix(T):
  T = np.asarray(T, np.float64).reshape(-1, 4, 4)
  return np.hstack([Rotation.from_matrix(T[:, :3, :3]).as_rotvec(), T[:, :3, 3]])


def look_at(eye, target, up=(0.0, -1.0, 0.0)):
  """4x4 mapping rig coordinates to a camera at `eye` whose +z axis points at `target`."""
  z = target - eye; z = z / np.linalg.norm(z)
  x = np.cross(np.asarray(up), z)
  if np.linalg.norm(x) < 1e-6: x = np.cross(np.array([1.0, 0.0, 0.0]), z)
  x = x / np.linalg.norm(x)
  y = np.cross(z, x)
  R = np.stack([x, y, z])          # rows: camera axes in rig coordinates
  T = np.eye(4); T[:3, :3] = R; T[:3, 3] = -R @ eye
  return T


def distort_project(model, X, K, dist):
  """numpy pinhole / fisheye projection used only to synthesise observations
  (same formulas as cv2.projectPoints / cv2.fisheye.projectPoints, SURVEY.md §8 a8/a9)."""
  x = X[..., 0] / X[..., 2]; y = X[..., 1] / X[..., 2]
  fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
  if model == "fisheye":
    r = np.sqrt(x * x + y * y)
    th = np.arctan(r); t2 = th * th
    thd = th * (1 + t2 * (dist[0] + t2 * (dist[1] + t2 * (dist[2] + t2 * dist[3]))))
    s = np.where(r > 1e-8, thd / np.maximum(r, 1e-300), 1.0)
    xd, yd = x * s, y * s
  else:
    d = np.zeros(14); d[:dist.size] = dist
    k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4 = d[:12]
    r2 = x * x + y * y
    rad = (1 + r2 * (k1 + r2 * (k2 + r2 * k3))) / (1 + r2 * (k4 + r2 * (k5 + r2 * k6)))
    xd = x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x) + r2 * (s1 + r2 * s2)
    yd = y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y + r2 * (s3 + r2 * s4)
    if d[12] != 0 or d[13] != 0:      # tilted sensor (14 coefficients)
      cx_, sx_, cy_, sy_ = np.cos(d[12]), np.sin(d[12]), np.cos(d[13]), np.sin(d[13])
      Rxy = np.array([[cy_, 0, -sy_], [0, 1, 0], [sy_, 0, cy_]]) @ np.array([[1, 0, 0], [0, cx_, sx_], [0, -sx_, cx_]])
      M = np.array([[Rxy[2, 2], 0, -Rxy[0, 2]], [0, Rxy[2, 2], -Rxy[1, 2]], [0, 0, 1]]) @ Rxy
      vt = np.stack([xd, yd, np.ones_like(xd)], axis=-1) @ M.T
      xd, yd = vt[..., 0] / vt[..., 2], vt[..., 1] / vt[..., 2]
  return np.stack([fx * xd + cx, fy * yd + cy], axis=-1)


DIST_GT = {
  "standard": np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01]),
  "rational": np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01, 0.02, -0.01, 0.005]),
  "thin_prism": np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01, 0.02, -0.01, 0.005, 1e-3, -5e-4, 5e-4, 1e-3]),
  "tilted": np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01, 0.02, -0.01, 0.005, 1e-3, -5e-4, 5e-4, 1e-3, 0.02, -0.015]),
  "fisheye": np.array([0.02, -0.01, 3e-3, -1e-3]),
}


def _boards(kind, w, h, square, count, rng):
  pts = grid_board_points(w, h, square)
  centre = pts.mean(axis=0)
  side = max(w, h) * square
  if kind == "charuco":
    boards, poses = [pts.copy() for _ in range(count)], []
    for i in range(count):
      T = np.eye(4); T[:3, 3] = [i * side * 1.1, 0, 0]
      poses.append(T)
    return boards, np.stack(poses), side
  if kind == "tiles":     # `count` boards on a near-square grid in one plane: many boards, all in view of an arc rig
    cols = int(np.ceil(np.sqrt(count)))
    boards, poses = [pts.copy() for _ in range(count)], []
    for i in range(count):
      T = np.eye(4); T[:3, 3] = [(i % cols) * side * 1.1, (i // cols) * side * 1.1, 0]
      poses.append(T)
    return boards, np.stack(poses), side
  # cube: faces of a cube of side `side` centred at the origin, each board face-centred
  face_rot = [np.zeros(3), [0, np.pi / 2, 0], [-np.pi / 2, 0, 0], [0, -np.pi / 2, 0],
              [np.pi / 2, 0, 0], [0, np.pi, 0]]
  boards, poses = [], []
  for i in range(count):
    R = Rotation.from_rotvec(face_rot[i % 6]).as_matrix()
    T = np.eye(4); T[:3, :3] = R
    T[:3, 3] = R @ (-centre + np.array([0, 0, -side / 2]))
    boards.append(pts.copy()); poses.append(T)
  return boards, np.stack(poses), side


def make_scene(C=2, F=20, boards=("charuco", 16, 22, 0.025, 1), model="standard", vis=0.5,
               rig="arc", noise=0.3, seed=0, pose_jitter=0.01, intrinsic_jitter=0.0,
               image_size=(1920, 1080), outlier_fraction=0.0, frame_chunk=64, focal=None):
  """Returns the scene dict described in the module docstring. Deterministic in `seed`.  focal: the nominal focal length in pixels
  (default 1200, fisheye 900)."""
  rng = np.random.default_rng(seed)
  kind, w, h, square, nb = boards
  board_points, board_poses, side = _boards(kind, w, h, square, nb, rng)
  B = len(board_points)
  P = max(p.shape[0] for p in board_points)
  W, H = image_size
  nd = DIST_GT[model].size

  # world centre of all boards
  centre = np.mean([(T[:3, :3] @ p.T).T.mean(axis=0) + T[:3, 3] for T, p in zip(board_poses, board_points)], axis=0)

  # cameras (rig frame): arc of small baselines in front of the target, or inward-looking dome
  planar = kind in ("charuco", "tiles")
  dist_target = 1.1 if planar else 1.4
  target = np.array([0.0, 0.0, dist_target])
  cam_poses = []
  for i in range(C):
    if rig == "arc":
      a = (i - (C - 1) / 2) * min(0.12, 0.5 / max(C - 1, 1))
      eye = np.array([np.sin(a) * dist_target, 0.03 * ((i % 2) * 2 - 1), dist_target - np.cos(a) * dist_target])
    else:
      # Fibonacci cap (half-angle ~50deg) centred on -z as seen from the target
      t = (i + 0.5) / C
      polar = np.arccos(1 - t * (1 - np.cos(np.deg2rad(50.0))))
      az = i * np.pi * (3 - np.sqrt(5))
      eye = target + dist_target * np.array([np.sin(polar) * np.cos(az), np.sin(polar) * np.sin(az), -np.cos(polar)])
    cam_poses.append(look_at(eye, target + rng.normal(0, 0.02, 3)))
  cam_poses = np.stack(cam_poses)

  f0 = focal if focal is not None else 1200.0 if model != "fisheye" else 900.0
  K = np.tile(np.eye(3), (C, 1, 1))
  K[:, 0, 0] = f0 * (1 + rng.normal(0, 0.01, C)); K[:, 1, 1] = K[:, 0, 0] * (1 + rng.normal(0, 0.002, C))
  K[:, 0, 2] = W / 2 + rng.normal(0, 5, C); K[:, 1, 2] = H / 2 + rng.normal(0, 5, C)
  dist = DIST_GT[model][None, :] * (1 + rng.normal(0, 0.05, (C, nd)))

  # frame poses: world -> rig; board-set centre lands near the target with a random attitude
  rot_sigma = 0.25 if planar else 0.6
  rv = rng.normal(0, rot_sigma, (F, 3))
  Rf = Rotation.from_rotvec(rv).as_matrix()
  tf = target[None, :] + rng.normal(0, [0.08, 0.05, 0.08], (F, 3)) - np.einsum("fij,j->fi", Rf, centre)
  frame_poses = np.tile(np.eye(4), (F, 1, 1)); frame_poses[:, :3, :3] = Rf; frame_poses[:, :3, 3] = tf

  # board points padded to P (tables.stack_boards, tables.py:385-394)
  Xb = np.zeros((B, P, 3)); pvalid = np.zeros((B, P), bool)
  for b, p in enumerate(board_points):
    Xb[b, :p.shape[0]] = p; pvalid[b, :p.shape[0]] = True
  Xw = np.einsum("bij,bpj->bpi", board_poses[:, :3, :3], Xb) + board_poses[:, None, :3, 3]

  points = np.zeros((C, F, B, P, 2)); valid = np.zeros((C, F, B, P), bool)
  for f0_ in range(0, F, frame_chunk):
    f1 = min(F, f0_ + frame_chunk)
    Xr = np.einsum("fij,bpj->fbpi", frame_poses[f0_:f1, :3, :3], Xw) + frame_poses[f0_:f1, None, None, :3, 3]
    for c in range(C):
      Xc = np.einsum("ij,fbpj->fbpi", cam_poses[c, :3, :3], Xr) + cam_poses[c, :3, 3]
      uv = distort_project(model, Xc, K[c], dist[c])
      ok = (Xc[..., 2] > 0.1) & (uv[..., 0] >= 0) & (uv[..., 0] < W) & (uv[..., 1] >= 0) & (uv[..., 1] < H)
      ok &= pvalid[None]
      ok &= rng.random(ok.shape) < vis
      uv = uv + rng.normal(0, noise, uv.shape)
      if outlier_fraction > 0:
        bad = rng.random(ok.shape) < outlier_fraction
        uv = uv + bad[..., None] * rng.normal(0, 30.0, uv.shape)
      points[c, f0_:f1] = np.where(ok[..., None], uv, 0.0)
      valid[c, f0_:f1] = ok

  gt = dict(K=K, dist=dist, cam_poses=cam_poses, frame_poses=frame_poses, board_poses=board_poses)

  def jitter(T):
    n = T.shape[0]
    d = to_matrix(np.hstack([rng.normal(0, pose_jitter, (n, 3)), rng.normal(0, pose_jitter, (n, 3))]))
    return T @ d
  Ki = K.copy()
  if intrinsic_jitter > 0:
    Ki[:, 0, 0] *= 1 + rng.normal(0, intrinsic_jitter, C); Ki[:, 1, 1] *= 1 + rng.normal(0, intrinsic_jitter, C)
  init = dict(K=Ki, dist=dist.copy(), cam_poses=jitter(cam_poses), frame_poses=jitter(frame_poses),
              board_poses=jitter(board_poses))

  return dict(C=C, F=F, B=B, P=P, model=model, image_size=tuple(image_size), seed=seed,
              board_points=board_points, points=points, valid=valid,
              cam_valid=np.ones(C, bool), frame_valid=np.ones(F, bool), board_valid=np.ones(B, bool),
              gt=gt, init=init, noise=noise)


def make_workload(name, seed=0, **overrides):
  cfg = dict(WORKLOADS[name]); cfg.update(overrides)
  return make_scene(seed=seed, **cfg)


def make_pose_table_scene(C, F, B, p_valid, seed, outliers=0.0, cam_spread=0.3, dead_camera=None, empty_frame=None, disjoint=False):
  """A make_pose_table result without images, for the pose-graph initialisation: view (c, f, b) = cam[c] frame[f] board[b] times a
  small perturbation; a fraction `outliers` of the views gets a large one; invalid views hold the identity.  dead_camera: a camera
  that shares no view with the others; empty_frame: a frame without views; disjoint: camera c sees only the boards b with
  b % C == c (a non-overlapping rig: no two cameras see the same board, so the camera-overlap matrix is zero; B >= 3 C gives every
  camera pair at least 9 hand-eye quadruples).  -> (poses [C,F,B,4,4], valid, num_points, cam poses)."""
  rng = np.random.default_rng(seed)
  cam = to_matrix(np.hstack([rng.normal(0, cam_spread, (C, 3)), rng.normal(0, 0.3, (C, 3))]))
  frm = to_matrix(np.hstack([rng.normal(0, 0.5, (F, 3)), rng.normal(0, 0.3, (F, 3)) + [0, 0, 1.0]]))
  brd = to_matrix(np.hstack([rng.normal(0, 0.8, (B, 3)), rng.normal(0, 0.1, (B, 3))]))
  T = cam[:, None, None] @ frm[None, :, None] @ brd[None, None, :]
  noise = np.hstack([rng.normal(0, 0.003, (C * F * B, 3)), rng.normal(0, 0.002, (C * F * B, 3))])
  bad = rng.random(C * F * B) < outliers
  noise[bad] += np.hstack([rng.normal(0, 0.5, (bad.sum(), 3)), rng.normal(0, 0.3, (bad.sum(), 3))])
  T = T @ to_matrix(noise).reshape(C, F, B, 4, 4)
  valid = rng.random((C, F, B)) < p_valid
  if dead_camera is not None:
    mine = np.arange(F) % 4 == 0
    valid[dead_camera] = mine[:, None] & valid[dead_camera]
    valid[np.ix_(np.arange(C) != dead_camera, mine)] = False
  if empty_frame is not None:
    valid[:, empty_frame] = False
  if disjoint:
    valid &= (np.arange(B)[None, :] % C == np.arange(C)[:, None])[:, None, :]
  T = np.where(valid[..., None, None], T, np.eye(4))
  npts = np.where(valid, rng.integers(20, 80, (C, F, B)), 0)
  return T, valid, npts, cam
