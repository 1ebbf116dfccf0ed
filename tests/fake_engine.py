"""TEST INFRASTRUCTURE: a numpy stand-in for multical_b200.engine.Engine, built on the oracle.

It lets the CPU suite exercise the *host-side control flow* of `Calibration` (which engine calls are made, in what order,
what is logged, how masks and states are threaded through) without a GPU.  It is never importable from the product: it
lives under tests/ and depends on oracle/.  The numerical parity of the real engine is the business of tests/test_gpu_parity.py.
"""
import numpy as np

from multical_b200 import _native as nat
from multical_b200.engine import Engine, SolveInfo
from oracle.ba_oracle import Problem

OPT_KEYS = {1: "camera_poses", 2: "board_poses", 4: "motion", 8: "cameras", 16: "boards"}


class FakeEngine(Engine):
  def __init__(self, image_size=(1600, 1200)):          # no library, no device
    self.calls = []
    self.table = None

  def close(self): pass

  # ---- problem / state ----------------------------------------------------------------------------------------------
  def _set_problem(self, model, optimize_bits, mask, points, board_points):
    Cn, F, B, P = mask.shape
    self.model, self.kint = model, 5 + nat.DIST_SIZES[model]
    self.desc = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], int(optimize_bits), int(mask.sum()))
    self.N = int(mask.sum())
    self.optimize = {name: bool(optimize_bits & bit) for bit, name in OPT_KEYS.items()}
    self.fix_aspect = bool(optimize_bits & nat.OPT_FIX_ASPECT)
    self.mask, self.points = np.array(mask, bool), np.array(points, np.float64)
    self.board_points = np.array(board_points, np.float64).reshape(B, P, 3)

  def upload_dense(self, model, optimize_bits, mask, points, board_points, view_valid=None):
    self.calls.append("upload_dense")
    self.table = None
    mask = np.asarray(mask)
    if view_valid is not None: mask = mask & np.asarray(view_valid)[..., None]      # the conjunction the device takes (mcba_upload_dense with view_valid)
    self._set_problem(model, optimize_bits, mask, points, board_points)

  def set_state_matrices(self, pose_matrices, intrinsics):
    self.calls.append("set_state_matrices")
    d = self.desc
    mats = np.array(pose_matrices, np.float64)
    self.cam_T, self.board_T, self.frame_T = mats[:d.C], mats[d.C:d.C + d.B], mats[d.C + d.B:]
    self.intr = np.array(intrinsics, np.float64).reshape(d.C, self.kint)
    self.errors = None

  def get_state_matrices(self):
    return self.cam_T, self.board_T, self.frame_T, self.intr

  def _problem(self, mask):
    K = np.tile(np.eye(3), (self.desc.C, 1, 1))
    K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2], K[:, 0, 1] = (self.intr[:, i] for i in range(5))
    return Problem(self.model, K, self.intr[:, 5:], self.cam_T, self.frame_T, self.board_T, list(self.board_points),
                   self.points, mask, inlier_mask=mask, optimize=self.optimize, fix_aspect=self.fix_aspect)

  def reprojection_error(self):
    self.calls.append("reprojection_error")
    prob = self._problem(self.mask)
    uv, _ = prob.reprojected()
    return np.linalg.norm(uv - self.points, axis=-1)[self.mask]

  def solve(self, ftol=1e-8, xtol=1e-8, gtol=1e-8, f_scale=1.0, max_nfev=100, loss="linear"):
    self.calls.append(f"solve(f_scale={f_scale:.6g})")
    prob = self._problem(self.mask)
    out, res = prob.bundle_adjust(tolerance=ftol, f_scale=f_scale, max_iterations=max_nfev, loss=loss, xtol=xtol, gtol=gtol)
    self.cam_T, self.board_T, self.frame_T = out.cam_poses, out.board_poses, out.frame_poses
    self.intr = out.camera_params()
    self.errors = None
    return SolveInfo(cost=res.cost, initial_cost=0.5 * float(np.sum(prob.residuals() ** 2)), optimality=res.optimality,
                     nfev=res.nfev, njev=res.njev, status=res.status, message=res.message, device_ms=0.0,
                     kernel_launches=0, log=[], chol_retries=0)

  # ---- resident table ------------------------------------------------------------------------------------------------
  def table_upload(self, model, optimize_bits, valid, points, board_points):
    self.calls.append("table_upload")
    valid = np.array(valid, bool)
    self._set_problem(model, optimize_bits, valid, points, board_points)
    self.table = dict(valid=valid, inliers=valid.copy(), selected="valid")
    self.errors = None
    return self.N

  def table_set_inliers(self, mask=None):
    self.calls.append("table_set_inliers")
    t = self.table
    t["inliers"] = t["valid"].copy() if mask is None else (np.asarray(mask, bool) & t["valid"])
    self.errors = None

  def table_get_inliers(self):
    return self.table["inliers"].copy()

  def table_select(self, which):
    self.calls.append(f"table_select({which})")
    self.mask = self.table[which].copy()
    self.table["selected"] = which
    self.N = int(self.mask.sum())
    return self.N

  def table_errors(self):
    self.calls.append("table_errors")
    t = self.table
    self.table_select("valid"); self.calls.pop()
    err = self.reprojection_error(); self.calls.pop()
    inl = t["inliers"][t["valid"]]
    self.errors = dict(valid=np.sort(err), inliers=np.sort(err[inl]), raw=err)
    return SolveInfo(n_valid=err.size, n_inliers=int(inl.sum()), sumsq_valid=float(np.sum(err ** 2)),
                     sumsq_inliers=float(np.sum(err[inl] ** 2)))

  def table_error_ranks(self, which, ranks):
    assert self.errors is not None, "table_errors has not run since the state changed"
    return self.errors[which][np.asarray(ranks, np.int64)]

  def table_reject(self, threshold):
    self.calls.append("table_reject")
    assert self.errors is not None and self.table["selected"] == "valid"
    t = self.table
    keep = np.zeros(t["valid"].shape, bool)
    keep[t["valid"]] = self.errors["raw"] < threshold
    t["inliers"] = keep
    self.errors = None
    return int(t["valid"].sum()), int(keep.sum())
