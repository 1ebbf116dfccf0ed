"""`Calibration` with the reference's public surface (multical/optimization/calibration.py:43-300)
whose `bundle_adjust()` runs on an H100 through libmcba.so instead of
`scipy.optimize.least_squares` over numpy + cv2 (calibration.py:199-212).

Constructor signature, method names, argument meanings, logging and error behaviour follow the
reference so that callers (`Workspace.calibrate`, workspace.py:228-247) can swap the class in.
The objects passed in may be this package's mirrors (camera.py, pose_set.py, board.py) or the
reference's own `Camera`, `PoseSet`, `StaticFrames`, `ParamList`, `Table`: only attributes that both
expose are touched (duck typing)."""
import os
from functools import cached_property
from numbers import Integral

import numpy as np

from . import rtvec
from ._native import OPT_BITS, OPT_FIX_ASPECT
from .board import stack_boards
from .camera import engine_model_of
from .engine import Engine, format_log
from .log import info
from .motion import MOTION_HAND_EYE, MOTION_ROLLING, motion_kind
from .outliers import QuantileThreshold, select_threshold      # noqa: F401  (select_threshold: calibration.py:37-40)
from .parameters import Parameters
from .structs import Table, struct

default_optimize = struct(cameras=False, boards=False, camera_poses=True, board_poses=True, motion=True)


_engines = {}


def default_device():
  return int(os.environ.get("MCBA_DEVICE", os.environ.get("LOCAL_RANK", "0")))


def get_engine(device=None):
  """One C-ABI context per (process, GPU); the caller is single threaded like the reference (SURVEY §8b)."""
  device = default_device() if device is None else device
  if device not in _engines:
    _engines[device] = Engine(device)
  return _engines[device]


def _mk_table(like, **arrays):
  """Build a points/valid table of the same kind the caller handed us (reference Table or ours)."""
  create = getattr(type(like), "create", None)
  return create(**arrays) if create is not None else Table.create(**arrays)


class Calibration(Parameters):
  def __init__(self, cameras, boards, point_table, camera_poses, board_poses, motion,
               inlier_mask=None, optimize=default_optimize):
    self.cameras = cameras
    self.boards = boards
    self.point_table = point_table
    self.camera_poses = camera_poses
    self.board_poses = board_poses
    self.motion = motion
    self.optimize = optimize
    self.inlier_mask = inlier_mask
    assert len(self.cameras) == self.size.cameras
    assert camera_poses.size == self.size.cameras
    assert board_poses.size == self.size.boards

  # ---- shapes and masks (calibration.py:64-81) --------------------------------------------------
  @cached_property
  def size(self):
    cameras, rig_poses, boards, points = np.shape(self.point_table.valid)
    return struct(cameras=cameras, rig_poses=rig_poses, boards=boards, points=points)

  @cached_property
  def pose_valid(self):
    return (np.asarray(self.camera_poses.valid)[:, None, None] & np.asarray(self.motion.valid)[None, :, None]
            & np.asarray(self.board_poses.valid)[None, None, :])

  @cached_property
  def valid(self):
    return np.asarray(self.point_table.valid) & self.pose_valid[..., None]

  @cached_property
  def inliers(self):
    return self.valid if self.inlier_mask is None else self.inlier_mask

  @cached_property
  def board_points(self):
    pts, valid = stack_boards(self.boards)
    return Table.create(points=pts, valid=valid)

  @cached_property
  def world_points(self):
    """calibration.py:87-90 (host utility for viewers; the solver recomputes this on the GPU)."""
    T = np.asarray(self.board_poses.poses)
    bp = self.board_points
    pts = np.einsum("bij,bpj->bpi", T[:, :3, :3], bp.points) + T[:, None, :3, 3]
    return Table.create(points=pts, valid=np.asarray(self.board_poses.valid)[:, None] & bp.valid)

  @cached_property
  def pose_estimates(self):
    return struct(camera=self.camera_poses.pose_table, board=self.board_poses.pose_table, times=self.motion.frame_poses)

  def with_master(self, camera):
    if isinstance(camera, str): camera = self.camera_poses.names.index(camera)
    assert isinstance(camera, Integral)
    return self.transform_views(self.camera_poses.poses[camera])

  def transform_views(self, t):
    """calibration.py:107-112: cameras by t^-1, frame poses by t (projection unchanged)."""
    return self.copy(camera_poses=self.camera_poses.post_transform(np.linalg.inv(t)), motion=self.motion.pre_transform(t))

  # ---- GPU problem ------------------------------------------------------------------------------
  @cached_property
  def engine_model(self):
    models = {engine_model_of(c) for c in self.cameras}
    assert len(models) == 1, f"all cameras must share one model, got {models}"
    return models.pop()

  def _optimize_bits(self):
    bits = sum(bit for k, bit in OPT_BITS.items() if self.optimize[k] is True)
    fix = {bool(getattr(c, "fix_aspect", False)) for c in self.cameras}
    assert len(fix) == 1, "fix_aspect must agree across cameras"
    return bits | (OPT_FIX_ASPECT if fix.pop() else 0) | motion_kind(self.motion)

  def _state_arrays(self):
    # one rotation-vector conversion for all pose sets (the scipy call dominates the host time of a small solve)
    sets = [np.asarray(self.camera_poses.poses), np.asarray(self.board_poses.poses), np.asarray(self.motion.poses)]
    rt = rtvec.from_matrix(np.concatenate(sets, axis=0))
    n0, n1 = sets[0].shape[0], sets[0].shape[0] + sets[1].shape[0]
    intr = np.stack([np.asarray(c.param_vec, np.float64) for c in self.cameras])
    return rt[:n0], rt[n0:n1], rt[n1:], intr

  # The C-ABI keeps the `boards` block as the padded [B][P][3] stack (tables.stack_boards); the reference's vector holds
  # only each board's own points (board/charuco.py:112-117).  These two helpers translate between the two layouts.
  def _board_block_slices(self):
    P = self.size.points
    keep = np.concatenate([np.arange(3 * P) < 3 * b.num_points for b in self.boards])
    return keep

  def _to_engine_vec(self, x):
    if self.optimize["boards"] is not True: return np.asarray(x, np.float64)
    keep = self._board_block_slices()
    head = x.size - int(keep.sum())
    out = np.zeros(head + keep.size)
    out[:head] = x[:head]
    tail = np.asarray(self.board_points.points, np.float64).ravel().copy()
    tail[keep] = x[head:]
    out[head:] = tail
    return out

  def _from_engine_vec(self, xe):
    if self.optimize["boards"] is not True: return xe
    keep = self._board_block_slices()
    head = xe.size - keep.size
    return np.concatenate([xe[:head], xe[head:][keep]])

  def _upload(self, mask, points=None, device=None, view_valid=None):
    eng = get_engine(device)
    pts = np.asarray(self.point_table.points) if points is None else points
    eng.upload_dense(self.engine_model, self._optimize_bits(), mask, pts, self.board_points.points, view_valid=view_valid)
    self._push_state(eng)
    return eng

  def _upload_inliers(self, device=None):
    """`_upload(self.inliers)` without building `valid` on the host when no inlier mask is set (and `valid` has not been asked for
    yet): the detection table goes over as it is, the pose validity of the views ([C,F,B]) beside it, and the device takes the
    conjunction (calibration.py:73-81)."""
    if self.inlier_mask is None and "valid" not in self.__dict__ and "inliers" not in self.__dict__:
      return self._upload(np.asarray(self.point_table.valid), view_valid=self.pose_valid, device=device)
    return self._upload(self.inliers, device=device)

  def _push_state(self, eng):
    # poses go over as 4x4 matrices: the matrix -> rotation-vector conversion (transform/rtvec.py:29-32) runs on the device
    kind = motion_kind(self.motion)
    frames = self.motion.pose_start if kind == MOTION_ROLLING else self.motion.poses
    mats = np.concatenate([np.asarray(self.camera_poses.poses, np.float64), np.asarray(self.board_poses.poses, np.float64),
                           np.asarray(frames, np.float64)], axis=0)
    eng.set_state_matrices(mats, np.stack([np.asarray(c.param_vec, np.float64) for c in self.cameras]))
    if kind == MOTION_ROLLING:      # `motion.poses` above were the start poses
      eng.set_rolling(self.motion.pose_end, [c.image_size[1] for c in self.cameras])
    elif kind == MOTION_HAND_EYE:   # the frames above are derived poses, ignored by the engine
      eng.set_hand_eye(self.motion.base_wrt_gripper.poses, self.motion.world_wrt_base, self.motion.gripper_wrt_camera)

  def _with_engine_state(self, eng):
    """New Calibration holding the engine's solved state -- what `self.with_param_vec(res.x)` returns in the reference
    (calibration.py:212), built from the pose matrices the device hands back (rtvec -> matrix, rtvec.py:24-27, done there)."""
    if self.optimize["boards"] is True or not hasattr(self.motion, "pose_table"):
      return self.with_param_vec(self._from_engine_vec(eng.param_vec))
    cam_T, board_T, frame_T, intr = eng.get_state_matrices()
    def moved(pose_set, poses):
      return pose_set.copy(pose_table=pose_set.pose_table._update(poses=poses))
    changes = {}
    if self.optimize["camera_poses"] is True: changes["camera_poses"] = moved(self.camera_poses, cam_T)
    if self.optimize["board_poses"] is True: changes["board_poses"] = moved(self.board_poses, board_T)
    if self.optimize["motion"] is True:
      kind = motion_kind(self.motion)
      if kind == MOTION_ROLLING: changes["motion"] = self.motion.copy(pose_start=frame_T, pose_end=eng.get_rolling())
      elif kind == MOTION_HAND_EYE:
        world_wrt_base, gripper_wrt_camera = eng.get_hand_eye()
        changes["motion"] = self.motion.copy(world_wrt_base=world_wrt_base, gripper_wrt_camera=gripper_wrt_camera)
      else: changes["motion"] = moved(self.motion, frame_T)
    if self.optimize["cameras"] is True: changes["cameras"] = self.cameras.with_param_vec(intr.ravel())
    return self.copy(**changes)

  # ---- projection / errors (calibration.py:115-141, tables.py:239-249) ---------------------------
  def _project(self, mask, estimates=None):
    """Dense [C,F,B,P,2] projections of the points selected by `mask` (zeros elsewhere).  `estimates` [C,F,B,P,2]: image
    points whose rows give the rolling-shutter blend weights (rolling_frames.py:115-123); irrelevant for other motion models."""
    out = np.zeros((*mask.shape, 2))
    if mask.any():
      obs = np.zeros((*mask.shape, 2)) if estimates is None else np.ascontiguousarray(estimates, dtype=np.float64)
      eng = self._upload(mask, points=obs)
      out[mask] = eng.residuals().reshape(-1, 2) + obs[mask]      # residual = projected - "observed"
    return out

  @cached_property
  def _projectable(self):
    return self.pose_valid[..., None] & self.board_points.valid[None, None]

  @cached_property
  def projected(self):
    """calibration.py:115-121: projection without measurements.  Rolling frames start from mid-exposure (row = height / 2) and
    re-project `max_iterations` times with the rows of the previous projection (rolling_frames.py:115-133)."""
    ok = self._projectable
    if motion_kind(self.motion) != MOTION_ROLLING:
      return _mk_table(self.point_table, points=self._project(ok), valid=ok)
    heights = np.array([c.image_size[1] for c in self.cameras], dtype=np.float64)
    est = np.zeros((*ok.shape, 2)); est[..., 1] = 0.5 * heights[:, None, None, None]
    points = self._project(ok, est)
    for _ in range(getattr(self.motion, "max_iterations", 4)):
      points = self._project(ok, points)
    return _mk_table(self.point_table, points=points, valid=ok)

  @cached_property
  def reprojected(self):
    """calibration.py:124-130: projection given the measured points; they only matter to rolling frames (their rows)."""
    if motion_kind(self.motion) != MOTION_ROLLING: return self.projected
    ok = self._projectable
    return _mk_table(self.point_table, points=self._project(ok, np.asarray(self.point_table.points)), valid=ok)

  @cached_property
  def _valid_errors(self):
    """Per-corner pixel error over `valid`, in boolean-mask order (tables.py:244-249)."""
    if not self.valid.any(): return np.zeros(0)
    return self._upload(self.valid).reprojection_error()

  @cached_property
  def reprojection_error(self):
    return self._valid_errors

  @cached_property
  def reprojection_inliers(self):
    return self._valid_errors[self.inliers[self.valid]]

  def triangulate(self):
    """The calibration's inlier detections triangulated through its cameras and camera poses (multical_b200/triangulate.py): a Table of
    points [F, B, P, 3] in each frame's rig coordinates (where the projection reads camera_pose @ rig point, the rig point being
    frame_pose @ board_pose @ X), valid [F, B, P] (at least two inlier views) and rms [F, B, P] in pixels.  Independent of the solved
    frame and board poses, so it checks a calibration against them.  RollingFrames raise NotImplementedError: each image row sees the
    rig at another time, so a detection has no single rig point."""
    if motion_kind(self.motion) == MOTION_ROLLING:
      raise NotImplementedError("triangulation of RollingFrames: each image row sees the rig at a different time, so there is no single "
                                "rig point to triangulate")
    from .triangulate import triangulate
    C, F, B, P = self.size.cameras, self.size.rig_poses, self.size.boards, self.size.points
    pixels = np.asarray(self.point_table.points, np.float64).reshape(C, F * B * P, 2)
    res = triangulate(list(self.cameras), np.asarray(self.camera_poses.poses), pixels, np.asarray(self.inliers).reshape(C, F * B * P))
    return Table.create(points=res.points.reshape(F, B, P, 3), valid=res.valid.reshape(F, B, P), rms=res.rms.reshape(F, B, P))

  # ---- parameters (calibration.py:144-171) ------------------------------------------------------
  @cached_property
  def param_objects(self):
    return struct(camera_poses=self.camera_poses, board_poses=self.board_poses, motion=self.motion,
                  cameras=self.cameras, boards=self.boards)

  @cached_property
  def params(self):
    return struct(**{k: p.param_vec for k, p in self.param_objects.items() if self.optimize[k] is True})

  def with_params(self, params):
    updated = {k: self.param_objects[k].with_param_vec(v) for k, v in params.items()}
    return self.copy(**updated)

  def with_param_vec(self, param_vec):
    """parameters.py:48-50 semantics (split the vector over the enabled blocks in order) without first flattening the
    current parameters just to learn the block sizes -- that costs three rotation-vector conversions per call."""
    param_vec = np.asarray(param_vec)
    sizes = {}
    for k, obj in self.param_objects.items():
      if self.optimize[k] is True:
        n = getattr(obj, "num_params", None)
        sizes[k] = int(n) if n is not None else int(obj.param_vec.size)
    total = sum(sizes.values())
    assert param_vec.size == total, f"inconsistent parameter sizes, got {param_vec.size}, expected {total}"
    chunks, pos = {}, 0
    for k, n in sizes.items():
      chunks[k] = param_vec[pos:pos + n]; pos += n
    return self.with_params(chunks)

  @cached_property
  def sparsity_matrix(self):
    """Jacobian sparsity as the reference builds it for scipy (calibration.py:173-196).  The GPU solver
    uses analytic block Jacobians and never needs it; kept for API compatibility."""
    from scipy.sparse import csr_matrix
    idx = np.argwhere(self.inliers)
    N = idx.shape[0]
    rows2 = np.arange(2 * N).reshape(N, 2)
    rr, cc, col0 = [], [], 0
    def add(block_of_corner, nper, enabled):
      nonlocal col0
      on = enabled[block_of_corner]
      base = col0 + block_of_corner[on] * nper
      for j in range(nper):
        for comp in range(2):
          cc.append(base + j); rr.append(rows2[on][:, comp])
      col0 += enabled.size * nper
    if self.optimize["camera_poses"] is True: add(idx[:, 0], 6, np.asarray(self.camera_poses.valid))
    if self.optimize["board_poses"] is True: add(idx[:, 2], 6, np.asarray(self.board_poses.valid))
    if self.optimize["motion"] is True:
      kind = motion_kind(self.motion)
      if kind == MOTION_HAND_EYE:       # hand_eye.py:89-90: all 12 parameters touch every row
        add(np.zeros(N, dtype=np.int64), 12, np.ones(1, bool))
      else:
        add(idx[:, 1], 6, np.asarray(self.motion.valid))
        if kind == MOTION_ROLLING: add(idx[:, 1], 6, np.asarray(self.motion.valid))   # rolling_frames.py:146-150: start + end
    if self.optimize["cameras"] is True:
      add(idx[:, 0], self.cameras.param_vec.size // self.size.cameras, np.ones(self.size.cameras, bool))
    if self.optimize["boards"] is True:
      for board in self.boards:
        add(idx[:, 3].clip(max=board.num_points - 1), 3, np.ones(board.num_points, bool))
    if not cc: return csr_matrix((2 * N, col0), dtype=np.int16)
    S = csr_matrix((np.ones(sum(c.size for c in cc), np.int16), (np.concatenate(rr), np.concatenate(cc))), shape=(2 * N, col0))
    S.data[:] = 1
    return S

  # ---- the hot path -----------------------------------------------------------------------------
  def bundle_adjust(self, tolerance=1e-4, f_scale=1.0, max_iterations=100, loss="linear", xtol=1e-8, gtol=1e-8):
    """Non-linear least squares on point reprojection error (calibration.py:199-212), solved on the GPU
    with scipy-TRF semantics: ftol=tolerance, max_nfev=max_iterations, x_scale='jac', robust `loss`."""
    eng = self._upload_inliers()
    res = self._solve_logged(eng, tolerance, f_scale, max_iterations, loss, xtol, gtol)
    out = self._with_engine_state(eng)
    out.__dict__["last_solve"] = res
    return out

  @staticmethod
  def _solve_logged(eng, tolerance=1e-4, f_scale=1.0, max_iterations=100, loss="linear", xtol=1e-8, gtol=1e-8):
    res = eng.solve(ftol=tolerance, xtol=xtol, gtol=gtol, f_scale=f_scale, max_nfev=max_iterations, loss=loss)
    for line in format_log(res.log): info(line)
    info(res.message)
    info(f"Function evaluations {res.nfev}, initial cost {res.initial_cost:.4e}, final cost {res.cost:.4e}, "
         f"first-order optimality {res.optimality:.2e}.")
    return res

  def enable(self, **flags):
    for k in flags.keys():
      assert k in self.optimize, f"unknown option {k}, options are {list(self.optimize.keys())}"
    return self.copy(optimize=self.optimize._extend(**flags))

  def __getstate__(self):
    attrs = ["cameras", "boards", "point_table", "camera_poses", "board_poses", "motion", "inlier_mask", "optimize"]
    return {k: self.__dict__[k] for k in attrs}

  def __setstate__(self, d): self.__dict__.update(d)

  def copy(self, **k):
    d = self.__getstate__(); d.update(k)
    return Calibration(**d)

  # ---- outliers (same rules and log lines as calibration.py:234-268, 290-310) -------------------------
  def reject_outliers_quantile(self, quantile=0.95, factor=1.0):
    """Inliers = valid corners whose pixel error is below factor x the given error quantile."""
    return self.reject_outliers(threshold=factor * np.quantile(self.reprojection_error, quantile))

  def reject_outliers(self, threshold):
    """New Calibration whose inlier mask keeps the valid corners with error < threshold (pixels)."""
    valid = self.valid
    keep = np.zeros(valid.shape, dtype=bool)
    keep[valid] = self._valid_errors < threshold          # errors come back in boolean-mask order
    n_valid, n_keep = int(valid.sum()), int(keep.sum())
    info(f"Rejecting {n_valid - n_keep} outliers with error > {threshold:.2f} pixels, "
         f"keeping {n_keep} / {n_valid} inliers, ({100.0 * n_keep / n_valid:.2f}%)")
    return self.copy(inlier_mask=keep)

  def adjust_outliers(self, num_adjustments=3, select_scale=None, select_outliers=None, **kwargs):
    """Alternate outlier rejection and bundle adjustment `num_adjustments` times (workspace.py:228-247 drives this).
    select_outliers / select_scale map the current error vector to a pixel threshold / to the loss f_scale."""
    info(f"Beginning adjustments ({num_adjustments}) enabled: {self.optimize}, options: {kwargs}")
    on_device = all(s is None or isinstance(s, QuantileThreshold) for s in (select_scale, select_outliers))
    if on_device and self.valid.any() and not os.environ.get("MCBA_HOST_OUTLIERS"):
      return self._adjust_outliers_resident(num_adjustments, select_scale, select_outliers, **kwargs)
    calib = self
    for round_index in range(num_adjustments):
      calib.report(f"Adjust_outliers {round_index}:")
      errors = calib.reprojection_error
      f_scale = 1.0
      if select_scale is not None:
        f_scale = select_scale(errors) or 1.0
        info(f"Auto scaling for outliers influence at {f_scale:.2f} pixels")
      if select_outliers is not None:
        calib = calib.reject_outliers(select_outliers(errors))
      calib = calib.bundle_adjust(f_scale=f_scale, **kwargs)
    calib.report("Adjust_outliers end:")
    return calib

  def _adjust_outliers_resident(self, num_adjustments, select_scale, select_outliers, comm=None, **kwargs):
    """The same loop with the point table resident on the GPU (include/mcba.h "resident point table"): the dense table is
    uploaded once; each round the host sees the five-number summaries for the log, the order statistics around the selected
    quantiles and the inlier count.  The error vector, the masks and the repacking stay on the device.
    comm (multical_b200/distributed.py adjust_outliers): `self` is this rank's frame shard; counts and sums of squares are summed
    over the ranks, quantiles are taken over the union of all ranks' errors (outliers.merged_order_statistics), the solves are the
    collective solves of the engine's communicator -- thresholds, masks and log lines are those of the unsharded loop."""
    from .outliers import merged_order_statistics, quantile_from_sorted
    eng = get_engine()
    eng.table_upload(self.engine_model, self._optimize_bits(), self.valid, np.asarray(self.point_table.points),
                     self.board_points.points)
    self._push_state(eng)
    masked = self.inlier_mask is not None
    if masked: eng.table_set_inliers(np.asarray(self.inlier_mask))
    five = np.array([0.0, 0.25, 0.5, 0.75, 1.0])

    local_n = {}

    def quantile(which, n, q):
      """np.quantile over the chosen set: this rank's sorted errors, or the union over the ranks (n = global count)."""
      if comm is None: return eng.table_quantile(which, n, q)
      return quantile_from_sorted(lambda r: merged_order_statistics(comm, lambda lr: eng.table_error_ranks(which, lr),
                                                                    lambda v: eng.table_count_below(which, v), local_n[which], r), n, q)

    def summary(which, n, sumsq):
      if n == 0:                                   # the reference's guard: an empty vector counts as a single zero
        return struct(mse=0.0, rms=0.0, quantiles=np.zeros(5), n=1)
      return struct(mse=sumsq / n, rms=float(np.sqrt(sumsq / n)), quantiles=quantile(which, n, five), n=n)

    def report(stage):
      st = eng.table_errors()
      local_n["valid"], local_n["inliers"] = int(st.n_valid), int(st.n_inliers)
      if comm is not None:
        counts = comm.all_reduce_sum(np.array([st.n_valid, st.n_inliers], np.int64))
        sums = np.sum(comm.all_gather(np.array([st.sumsq_valid, st.sumsq_inliers])), axis=0)       # rank order: the same value everywhere
        st = type(st)(n_valid=int(counts[0]), n_inliers=int(counts[1]), sumsq_valid=float(sums[0]), sumsq_inliers=float(sums[1]))
      _report_line(stage, summary("valid", st.n_valid, st.sumsq_valid),
                   summary("inliers", st.n_inliers, st.sumsq_inliers) if masked else None)
      return st

    res = None
    for round_index in range(num_adjustments):
      st = report(f"Adjust_outliers {round_index}:")
      f_scale = 1.0
      if select_scale is not None:
        f_scale = quantile("valid", st.n_valid, select_scale.quantile) * select_scale.factor or 1.0
        info(f"Auto scaling for outliers influence at {f_scale:.2f} pixels")
      if select_outliers is not None:
        threshold = quantile("valid", st.n_valid, select_outliers.quantile) * select_outliers.factor
        n_valid, n_keep = eng.table_reject(threshold)
        if comm is not None: n_valid, n_keep = (int(v) for v in comm.all_reduce_sum(np.array([n_valid, n_keep], np.int64)))
        masked = True
        info(f"Rejecting {n_valid - n_keep} outliers with error > {threshold:.2f} pixels, "
             f"keeping {n_keep} / {n_valid} inliers, ({100.0 * n_keep / n_valid:.2f}%)")
      eng.table_select("inliers")
      res = self._solve_logged(eng, f_scale=f_scale, **_solve_args(**kwargs))
    report("Adjust_outliers end:")
    out = self._with_engine_state(eng)
    if masked: out = out.copy(inlier_mask=eng.table_get_inliers())
    out.__dict__["last_solve"] = res
    return out

  def report(self, stage=""):
    _report_line(stage, error_stats(self.reprojection_error),
                 None if self.inlier_mask is None else error_stats(self.reprojection_inliers))


def _solve_args(tolerance=1e-4, max_iterations=100, loss="linear", xtol=1e-8, gtol=1e-8):
  """bundle_adjust's keyword arguments (f_scale is chosen by the outlier loop), checked the way a call would check them."""
  return dict(tolerance=tolerance, max_iterations=max_iterations, loss=loss, xtol=xtol, gtol=gtol)


def _report_line(stage, everything, kept):
  if kept is None:
    info(f"{stage} reprojection RMS={everything.rms:.3f}, n={everything.n}, quantiles={everything.quantiles}")
  else:
    info(f"{stage} reprojection RMS={kept.rms:.3f} ({everything.rms:.3f}), "
         f"n={kept.n} ({everything.n}), quantiles={everything.quantiles}")


def error_stats(errors):
  """mse / rms / five-number summary of a pixel-error vector; an empty vector counts as a single zero
  (the reference's guard, calibration.py:303-310)."""
  e = np.asarray(errors, dtype=np.float64).ravel()
  if e.size == 0:
    e = np.zeros(1)
  mse = float(np.mean(e * e))
  return struct(mse=mse, rms=float(np.sqrt(mse)), quantiles=np.quantile(e, [0.0, 0.25, 0.5, 0.75, 1.0]), n=e.size)


def from_scene(scene, guess=True, **kwargs):
  """Calibration over a multical_b200.synthetic scene (plain numpy) using this package's mirror classes."""
  from .board import Board
  from .camera import Camera, CameraFisheye
  from .parameters import ParamList
  from .pose_set import PoseSet, StaticFrames, pose_table
  src = scene["init"] if guess else scene["gt"]
  fisheye = scene["model"] == "fisheye"
  cams = [(CameraFisheye(scene["image_size"], src["K"][i], src["dist"][i]) if fisheye else
           Camera(scene["image_size"], src["K"][i], src["dist"][i], model=scene["model"])) for i in range(scene["C"])]
  names = [f"cam{i}" for i in range(scene["C"])]
  bnames = [f"board{i}" for i in range(scene["B"])]
  return Calibration(ParamList(cams, names), ParamList([Board(p) for p in scene["board_points"]], bnames),
                     Table.create(points=scene["points"], valid=scene["valid"]),
                     PoseSet(pose_table(src["cam_poses"], scene["cam_valid"]), names),
                     PoseSet(pose_table(src["board_poses"], scene["board_valid"]), bnames),
                     StaticFrames(pose_table(src["frame_poses"], scene["frame_valid"])), **kwargs)
