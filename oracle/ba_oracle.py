"""ORACLE — TEST INFRASTRUCTURE ONLY (never imported by multical_b200, the product).

CPU restatement, in plain numpy + the same scipy call, of the reference hot path
`Calibration.bundle_adjust()` (reference: multical/optimization/calibration.py:199-212).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this file.

Pinning status: the reference ships NO tests, golden vectors or fixtures for this path
(SURVEY.md §4, §8c) — "parity unpinned" by the reference's own tests.  The restatement is
instead pinned against the *running reference itself* (imported unmodified through
tests/refshim) by tests/golden/make_golden.py, whose outputs are
committed under tests/golden/ and re-checked by tests/test_oracle.py on every run.

Each function cites the reference lines it follows.  All arithmetic is float64 like the
reference.  The dense [C,F,B,P] evaluation order and masking are kept (no packing), so this
is also the honest CPU cost model of the reference for bench.py's cpu_baseline.
"""
import numpy as np
from scipy import optimize
from scipy.sparse import csr_matrix

POSE = 6
OPTIMIZE_KEYS = ("camera_poses", "board_poses", "motion", "cameras", "boards")   # calibration.py:146-153
DEFAULT_OPTIMIZE = dict(cameras=False, boards=False, camera_poses=True, board_poses=True, motion=True)  # 28-35
DIST_SIZES = {"standard": 5, "rational": 8, "thin_prism": 12, "tilted": 14, "fisheye": 4}  # camera.py:43-48


# ----------------------------------------------------------------------------- SE(3)
def rotvec_to_matrix(rvec):
  """transform/rtvec.py:24-27 (scipy Rotation.from_rotvec(...).as_matrix()), restated as Rodrigues."""
  rvec = np.asarray(rvec, np.float64).reshape(-1, 3)
  th = np.linalg.norm(rvec, axis=1)
  small = th < 1e-3
  th2 = th * th
  safe = np.where(small, 1.0, th)
  A = np.where(small, 1 - th2 / 6 + th2 * th2 / 120, np.sin(safe) / safe)
  Bc = np.where(small, 0.5 - th2 / 24 + th2 * th2 / 720, (1 - np.cos(safe)) / (safe * safe))
  x, y, z = rvec[:, 0], rvec[:, 1], rvec[:, 2]
  Kx = np.zeros((rvec.shape[0], 3, 3))
  Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 0], Kx[:, 1, 2], Kx[:, 2, 0], Kx[:, 2, 1] = -z, y, z, -x, -y, x
  return np.eye(3)[None] + A[:, None, None] * Kx + Bc[:, None, None] * (Kx @ Kx)


def matrix_to_rotvec(R):
  """transform/rtvec.py:29-32 (Rotation.from_matrix(...).as_rotvec(), angle in [0, pi])."""
  from scipy.spatial.transform import Rotation
  return Rotation.from_matrix(np.asarray(R).reshape(-1, 3, 3)).as_rotvec()


def rtvec_to_matrix(rtvec):
  """transform/rtvec.py:24-27 + transform/matrix.py:33-39 (join)."""
  rtvec = np.asarray(rtvec, np.float64).reshape(-1, POSE)
  T = np.tile(np.eye(4), (rtvec.shape[0], 1, 1))
  T[:, :3, :3] = rotvec_to_matrix(rtvec[:, :3])
  T[:, :3, 3] = rtvec[:, 3:]
  return T


def matrix_to_rtvec(T):
  """transform/rtvec.py:29-32 + transform/matrix.py:42-44 (split)."""
  T = np.asarray(T, np.float64).reshape(-1, 4, 4)
  return np.hstack([matrix_to_rotvec(T[:, :3, :3]), T[:, :3, 3]])


# ----------------------------------------------------------------------------- projection
def project_pinhole(X, K, dist):
  """camera.py:124-128 = cv2.projectPoints(pts, rvec=0, tvec=0, K, dist).  K[0,1] (skew) is
  ignored by cv2; Z is not clamped; supports 5/8/12/14 coefficients (SURVEY.md §8 a8)."""
  d = np.zeros(14); d[:np.size(dist)] = np.ravel(dist)
  k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4, tx, ty = d
  Z = X[..., 2]
  iz = np.where(Z != 0, 1.0 / np.where(Z != 0, Z, 1.0), 1.0)
  x, y = X[..., 0] * iz, X[..., 1] * iz
  r2 = x * x + y * y; r4 = r2 * r2; r6 = r4 * r2
  cdist = 1 + k1 * r2 + k2 * r4 + k3 * r6
  icdist2 = 1.0 / (1 + k4 * r2 + k5 * r4 + k6 * r6)
  a1 = 2 * x * y; a2 = r2 + 2 * x * x; a3 = r2 + 2 * y * y
  xd = x * cdist * icdist2 + p1 * a1 + p2 * a2 + s1 * r2 + s2 * r4
  yd = y * cdist * icdist2 + p1 * a3 + p2 * a1 + s3 * r2 + s4 * r4
  if tx != 0 or ty != 0:      # tilted sensor (14-coefficient model)
    cx_, sx_, cy_, sy_ = np.cos(tx), np.sin(tx), np.cos(ty), np.sin(ty)
    Rx = np.array([[1, 0, 0], [0, cx_, sx_], [0, -sx_, cx_]])
    Ry = np.array([[cy_, 0, -sy_], [0, 1, 0], [sy_, 0, cy_]])
    Rxy = Ry @ Rx
    Pz = np.array([[Rxy[2, 2], 0, -Rxy[0, 2]], [0, Rxy[2, 2], -Rxy[1, 2]], [0, 0, 1]])
    M = Pz @ Rxy
    v = np.stack([xd, yd, np.ones_like(xd)], axis=-1) @ M.T
    iw = np.where(v[..., 2] != 0, 1.0 / np.where(v[..., 2] != 0, v[..., 2], 1.0), 1.0)
    xd, yd = v[..., 0] * iw, v[..., 1] * iw
  return np.stack([xd * K[0, 0] + K[0, 2], yd * K[1, 1] + K[1, 2]], axis=-1)


def project_fisheye(X, K, dist):
  """camera_fisheye.py:113-117 = cv2.fisheye.projectPoints(pts, 0, 0, K, D) with alpha=0
  (K[0,1] ignored as called) (SURVEY.md §8 a9)."""
  k = np.ravel(dist)
  a, b = X[..., 0] / X[..., 2], X[..., 1] / X[..., 2]
  r = np.sqrt(a * a + b * b)
  th = np.arctan(r); t2 = th * th
  thd = th * (1 + k[0] * t2 + k[1] * t2 * t2 + k[2] * t2 ** 3 + k[3] * t2 ** 4)
  s = np.where(r > 1e-8, thd / np.where(r > 1e-8, r, 1.0), 1.0)     # cv2: inv_r = r > 1e-8 ? 1/r : 1
  return np.stack([K[0, 0] * a * s + K[0, 2], K[1, 1] * b * s + K[1, 2]], axis=-1)


# ----------------------------------------------------------------------------- problem
class Problem:
  """Plain-array view of what `Calibration.__init__` holds (calibration.py:44-61)."""

  def __init__(self, model, K, dist, cam_poses, frame_poses, board_poses, board_points,
               points, valid, cam_valid=None, frame_valid=None, board_valid=None,
               inlier_mask=None, optimize=None, fix_aspect=False, has_skew=False,
               motion="static", frame_poses_end=None, image_size=None,
               base_wrt_gripper=None, world_wrt_base=None, gripper_wrt_camera=None):
    """motion: "static"  -- one rig pose per frame (motion/static_frames.py:29-42; every BASELINE configuration);
               "rolling" -- RollingFrames: a start pose (frame_poses) and an end pose (frame_poses_end) per frame, blended per
                            corner by its observed image row (motion/rolling_frames.py:15-41,66-150); needs image_size (W, H);
               "hand_eye" -- HandEye: frame pose f = gripper_wrt_camera @ base_wrt_gripper[f] @ world_wrt_base with the two
                            outer transforms as the 12 motion parameters (motion/hand_eye.py:14-90); frame_poses is ignored."""
    assert motion in ("static", "rolling", "hand_eye")
    self.motion = motion
    self.image_size = None if image_size is None else tuple(int(v) for v in image_size)
    self.frame_poses_end = None if frame_poses_end is None else np.array(frame_poses_end, np.float64)
    self.base_wrt_gripper = None if base_wrt_gripper is None else np.array(base_wrt_gripper, np.float64)
    self.world_wrt_base = None if world_wrt_base is None else np.array(world_wrt_base, np.float64)
    self.gripper_wrt_camera = None if gripper_wrt_camera is None else np.array(gripper_wrt_camera, np.float64)
    if motion == "hand_eye":        # motion/hand_eye.py:43-46
      frame_poses = self.gripper_wrt_camera[None] @ self.base_wrt_gripper @ self.world_wrt_base[None]
    if motion == "rolling":
      assert self.image_size is not None and self.frame_poses_end is not None
    self.model = model
    self.K = np.array(K, np.float64); self.dist = np.array(dist, np.float64)
    self.cam_poses = np.array(cam_poses, np.float64)
    self.frame_poses = np.array(frame_poses, np.float64)
    self.board_poses = np.array(board_poses, np.float64)
    self.board_points = [np.array(p, np.float64) for p in board_points]
    self.points = np.asarray(points, np.float64); self.point_valid = np.asarray(valid, bool)
    C, F, B, P = self.point_valid.shape
    self.C, self.F, self.B, self.P = C, F, B, P
    self.cam_valid = np.ones(C, bool) if cam_valid is None else np.asarray(cam_valid, bool)
    self.frame_valid = np.ones(F, bool) if frame_valid is None else np.asarray(frame_valid, bool)
    self.board_valid = np.ones(B, bool) if board_valid is None else np.asarray(board_valid, bool)
    self.inlier_mask = inlier_mask
    self.optimize = dict(DEFAULT_OPTIMIZE); self.optimize.update(optimize or {})
    self.fix_aspect, self.has_skew = fix_aspect, has_skew

  @staticmethod
  def from_scene(scene, guess=True, **kw):
    src = scene["init"] if guess else scene["gt"]
    return Problem(scene["model"], src["K"], src["dist"], src["cam_poses"], src["frame_poses"],
                   src["board_poses"], scene["board_points"], scene["points"], scene["valid"],
                   scene["cam_valid"], scene["frame_valid"], scene["board_valid"], **kw)

  def copy(self, **k):
    d = dict(model=self.model, K=self.K, dist=self.dist, cam_poses=self.cam_poses,
             frame_poses=self.frame_poses, board_poses=self.board_poses,
             board_points=self.board_points, points=self.points, valid=self.point_valid,
             cam_valid=self.cam_valid, frame_valid=self.frame_valid, board_valid=self.board_valid,
             inlier_mask=self.inlier_mask, optimize=self.optimize, fix_aspect=self.fix_aspect,
             has_skew=self.has_skew, motion=self.motion, frame_poses_end=self.frame_poses_end,
             image_size=self.image_size, base_wrt_gripper=self.base_wrt_gripper,
             world_wrt_base=self.world_wrt_base, gripper_wrt_camera=self.gripper_wrt_camera)
    d.update(k)
    return Problem(**d)

  # calibration.py:69-81
  @property
  def valid(self):
    v = (self.cam_valid[:, None, None] & self.frame_valid[None, :, None] & self.board_valid[None, None, :])
    return self.point_valid & v[..., None]

  @property
  def inliers(self):
    return self.valid if self.inlier_mask is None else self.inlier_mask

  # tables.py:385-394
  def stacked_board_points(self):
    X = np.zeros((self.B, self.P, 3)); ok = np.zeros((self.B, self.P), bool)
    for b, p in enumerate(self.board_points):
      X[b, :p.shape[0]] = p; ok[b, :p.shape[0]] = True
    return X, ok

  # ---- parameter vector (parameters.py:44-50,88-106; calibration.py:144-171; camera.py:144-171)
  def camera_params(self):
    rows = []
    for c in range(self.C):
      f = np.array([self.K[c, 0, 0], self.K[c, 1, 1]])
      if self.fix_aspect: f = np.array([f.mean(), f.mean()])
      skew = self.K[c, 0, 1] if self.has_skew else 0.0
      rows.append(np.concatenate([f, [self.K[c, 0, 2], self.K[c, 1, 2]], [skew], np.ravel(self.dist[c])]))
    return np.stack(rows)

  def blocks(self):
    """Ordered (name, flat vector) of every parameter block; order = calibration.py:146-153."""
    return [("camera_poses", matrix_to_rtvec(self.cam_poses).ravel()),
            ("board_poses", matrix_to_rtvec(self.board_poses).ravel()),
            ("motion", self.motion_params()),
            ("cameras", self.camera_params().ravel()),
            ("boards", np.concatenate([p.ravel() for p in self.board_points]))]

  def motion_params(self):
    if self.motion == "rolling":        # rolling_frames.py:135-140: [start rtvecs | end rtvecs]
      return np.concatenate([matrix_to_rtvec(self.frame_poses).ravel(), matrix_to_rtvec(self.frame_poses_end).ravel()])
    if self.motion == "hand_eye":       # hand_eye.py:76-81: struct(world_wrt_base, gripper_wrt_camera)
      return np.concatenate([matrix_to_rtvec(self.world_wrt_base).ravel(), matrix_to_rtvec(self.gripper_wrt_camera).ravel()])
    return matrix_to_rtvec(self.frame_poses).ravel()   # pose_set.py:51-53

  @property
  def param_vec(self):
    return np.concatenate([v for k, v in self.blocks() if self.optimize[k] is True] or [np.zeros(0)])

  def with_param_vec(self, x):
    x = np.asarray(x, np.float64)
    total = sum(v.size for k, v in self.blocks() if self.optimize[k] is True)
    assert x.size == total, f"inconsistent parameter sizes, got {x.size}, expected {total}"   # parameters.py:93-95
    upd, i = {}, 0
    for k, v in self.blocks():
      if self.optimize[k] is not True: continue
      p = x[i:i + v.size]; i += v.size
      if k == "camera_poses": upd["cam_poses"] = rtvec_to_matrix(p)            # pose_set.py:55-57
      elif k == "board_poses": upd["board_poses"] = rtvec_to_matrix(p)
      elif k == "motion":
        if self.motion == "rolling":      # rolling_frames.py:142-144
          upd["frame_poses"] = rtvec_to_matrix(p[:p.size // 2]); upd["frame_poses_end"] = rtvec_to_matrix(p[p.size // 2:])
        elif self.motion == "hand_eye":   # hand_eye.py:83-87
          upd["world_wrt_base"] = rtvec_to_matrix(p[:POSE])[0]; upd["gripper_wrt_camera"] = rtvec_to_matrix(p[POSE:])[0]
        else: upd["frame_poses"] = rtvec_to_matrix(p)
      elif k == "cameras":                                                       # camera.py:157-171
        cp = p.reshape(self.C, -1)
        K = np.tile(np.eye(3), (self.C, 1, 1))
        K[:, 0, 0] = cp[:, 0]; K[:, 1, 1] = cp[:, 0] if self.fix_aspect else cp[:, 1]
        K[:, 0, 2] = cp[:, 2]; K[:, 1, 2] = cp[:, 3]; K[:, 0, 1] = cp[:, 4]
        upd["K"] = K; upd["dist"] = cp[:, 5:].reshape(self.dist.shape)
      elif k == "boards":
        out, j = [], 0
        for bp in self.board_points:
          out.append(p[j:j + bp.size].reshape(bp.shape)); j += bp.size
        upd["board_points"] = out
    return self.copy(**upd)

  # ---- projection (calibration.py:87-90,124-130; static_frames.py:10-25; tables.py:284-304,400-405)
  def reprojected(self):
    X, ok = self.stacked_board_points()
    Tb = self.board_poses
    Xw = np.einsum("bij,bpj->bpi", Tb[:, :3, :3], X) + Tb[:, None, :3, 3]           # world_points
    Tcf = self.cam_poses[:, None] @ self.frame_poses[None, :]                        # expand_views
    Xc = np.einsum("cfij,bpj->cfbpi", Tcf[..., :3, :3], Xw) + Tcf[:, :, None, None, :3, 3]
    if self.motion == "rolling":
      # rolling_frames.py:15-41,115-123 with estimates = the measured point table (calibration.py:124-130): the corner is
      # transformed by the start and by the end pose and the two camera-frame points are blended by its observed row / height
      Tce = self.cam_poses[:, None] @ self.frame_poses_end[None, :]
      Xe = np.einsum("cfij,bpj->cfbpi", Tce[..., :3, :3], Xw) + Tce[:, :, None, None, :3, 3]
      t = (self.points[..., 1] / float(self.image_size[1]))[..., None]
      Xc = Xc * (1 - t) + Xe * t
    proj = project_fisheye if self.model == "fisheye" else project_pinhole
    with np.errstate(all="ignore"):
      uv = np.stack([proj(Xc[c], self.K[c], self.dist[c]) for c in range(self.C)])  # project_cameras
    v = (self.cam_valid[:, None, None, None] & self.frame_valid[None, :, None, None]
         & (self.board_valid[:, None] & ok)[None, None])
    return uv, v

  def residuals(self, x=None):
    """`evaluate` closure, calibration.py:204-206."""
    calib = self if x is None else self.with_param_vec(x)
    uv, _ = calib.reprojected()
    return (uv - calib.points)[self.inliers].ravel()

  def reprojection_error(self):
    """calibration.py:134-136 + tables.py:239-249: per-corner L2 over valid."""
    uv, v = self.reprojected()
    mask = v & self.point_valid
    err = np.linalg.norm(uv - self.points, axis=-1)
    err[~mask] = 0
    return err, mask

  # ---- sparsity (calibration.py:173-196, parameters.py:109-150, pose_set.py:59-60)
  def sparsity_matrix(self):
    C, F, B, P = self.C, self.F, self.B, self.P
    inl = self.inliers
    idx = np.argwhere(inl)                                   # row-major == boolean-mask order
    N = idx.shape[0]
    rows2 = np.arange(2 * N).reshape(N, 2)
    cols, rws = [], []
    col0 = 0
    def add(axis_idx, block_index_of_corner, nper, enabled_mask):
      nonlocal col0
      nblocks = enabled_mask.size
      on = enabled_mask[block_index_of_corner]
      base = col0 + block_index_of_corner[on] * nper
      r = rows2[on]
      for j in range(nper):
        for comp in range(2):
          cols.append(base + j); rws.append(r[:, comp])
      col0 += nblocks * nper
    if self.optimize["camera_poses"] is True: add(0, idx[:, 0], POSE, self.cam_valid)
    if self.optimize["board_poses"] is True: add(2, idx[:, 2], POSE, self.board_valid)
    if self.optimize["motion"] is True:
      if self.motion == "hand_eye":       # hand_eye.py:89-90: every residual depends on the 12 shared parameters
        for j in range(2 * POSE):
          for comp in range(2):
            cols.append(np.full(N, col0 + j)); rws.append(rows2[:, comp])
        col0 += 2 * POSE
      else:
        add(1, idx[:, 1], POSE, self.frame_valid)
        if self.motion == "rolling": add(1, idx[:, 1], POSE, self.frame_valid)     # rolling_frames.py:146-150: start + end
    if self.optimize["cameras"] is True:
      add(0, idx[:, 0], self.camera_params().shape[1], np.ones(C, bool))
    if self.optimize["boards"] is True:
      for b, bp in enumerate(self.board_points):
        # every board's points are indexed on axis 3 regardless of board (calibration.py:188-190)
        on = idx[:, 3] < bp.shape[0]
        base = col0 + idx[on, 3] * 3
        r = rows2[on]
        for j in range(3):
          for comp in range(2):
            cols.append(base + j); rws.append(r[:, comp])
        col0 += bp.shape[0] * 3
    if not cols:
      return csr_matrix((2 * N, col0), dtype=np.int16)
    cols = np.concatenate(cols); rws = np.concatenate(rws)
    S = csr_matrix((np.ones(cols.size, np.int16), (rws, cols)), shape=(2 * N, col0))
    S.data[:] = 1
    return S

  # ---- the solve (calibration.py:199-212)
  def bundle_adjust(self, tolerance=1e-4, f_scale=1.0, max_iterations=100, loss="linear",
                    verbose=0, xtol=1e-8, gtol=1e-8, counter=None):
    def evaluate(x):
      if counter is not None: counter[0] += 1
      return self.residuals(x)
    res = optimize.least_squares(evaluate, self.param_vec, jac_sparsity=self.sparsity_matrix(),
                                 verbose=verbose, x_scale="jac", f_scale=f_scale, ftol=tolerance,
                                 xtol=xtol, gtol=gtol, max_nfev=max_iterations, method="trf", loss=loss)
    return self.with_param_vec(res.x), res


def error_stats(errors):
  """calibration.py:303-310."""
  errors = np.asarray(errors)
  if errors.size == 0: errors = np.zeros((1, 1), np.float32)
  mse = np.square(errors).mean()
  q = np.array([np.quantile(errors, n) for n in [0, 0.25, 0.5, 0.75, 1]])
  return dict(mse=mse, rms=np.sqrt(mse), quantiles=q, n=errors.size)
