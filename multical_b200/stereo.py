"""Stereo calibration of a camera pair on the GPU: `stereo_calibrate` (multical/camera.py:261-286, cv2.stereoCalibrate),
`stereo_calibrate_fisheye` (camera_fisheye.py:180-205, cv2.fisheye.stereoCalibrate) and `stereo_calibrate_detections`
(image/detect.py:45-59).

A pair is a two-camera problem of the bundle-adjustment engine with one board and the views as frames:
  1. the board is the unique float32 rows of all views' object points, each corner points into it;
  2. mcba_stereo_init (include/mcba.h, csrc/stereo_kernels.cuh): the per-view poses of both cameras by PnP under their intrinsics and
     OpenCV's start, the median relative pose over the views;
  3. the solve: cameras [I, start], frames at the left camera's view poses, the board at identity; camera poses and frames free, and the
     intrinsics of both cameras with fix_intrinsic=False.  The pair's pose is read as T_cam1 T_cam0^-1 (x_right = R x_left + T), which
     does not depend on the gauge the free camera poses leave; err is sqrt(sum |e|^2 / (2 N)) over the N corners of each camera, the RMS
     cv2.stereoCalibrate returns.

The solve iterates to its own tolerances (ftol = xtol = gtol = 1e-10, at most 100 evaluations, overridable by keyword): it reaches the
minimum that OpenCV's Levenberg-Marquardt approaches.  `max_iter` and `eps` are accepted for the reference's signature and unused.  The
calibration runs on the intrinsic calibration's engine, so the process-wide bundle-adjustment engine keeps its problem."""
import numpy as np

from . import _native as nat
from .camera import Camera, CameraFisheye
from .rtvec import to_matrix
from .structs import struct

FREE_INTRINSIC_MODELS = ("standard", "fisheye")
UNSUPPORTED_FREE = {
  "rational": "k1..k3 and k4..k6 are nearly degenerate, and the engine's trust region stops short of OpenCV's minimum (DESIGN.md §3d)",
  "thin_prism": "under CALIB_THIN_PRISM_MODEL OpenCV keeps k4..k6 at zero; the engine's fixed-intrinsics mask can hold them, but this "
                "model's free-intrinsics solve is not checked against OpenCV yet",
  "tilted": "under CALIB_TILTED_MODEL OpenCV keeps k4..k6 and s1..s4 at zero; the engine's fixed-intrinsics mask can hold them, but this "
            "model's free-intrinsics solve is not checked against OpenCV yet",
}


def _camera_params(cam, model):
  """[fx fy cx cy skew dist...] of a camera (skew 0: OpenCV's projection of the pair does not use K[0, 1])."""
  K = np.asarray(cam.intrinsic, np.float64)
  d = np.asarray(cam.dist, np.float64).ravel()
  assert d.size == nat.DIST_SIZES[model], f"camera model {model} expects {nat.DIST_SIZES[model]} distortion coefficients, got {d.size}"
  return np.concatenate([[K[0, 0], K[1, 1], K[0, 2], K[1, 2], 0.0], d])


def pair_problem(matches):
  """The views of `matches` (per-view lists object_points, points1, points2; float32 as OpenCV converts them) as the engine's detection
  lists: (board [P, 3], det_start over lists c*F + f, det_ids, det_xy, views F)."""
  op = [np.asarray(o, np.float32).reshape(-1, 3) for o in matches.object_points]
  p1 = [np.asarray(p, np.float32).reshape(-1, 2) for p in matches.points1]
  p2 = [np.asarray(p, np.float32).reshape(-1, 2) for p in matches.points2]
  assert len(op) == len(p1) == len(p2) and len(op) > 0, "object_points, points1 and points2 must hold the same non-zero number of views"
  for f, (o, a, b) in enumerate(zip(op, p1, p2)):
    assert len(o) == len(a) == len(b), f"view {f}: object_points, points1 and points2 differ in length"
  board, pid = np.unique(np.concatenate(op), axis=0, return_inverse=True)
  pid = pid.reshape(-1).astype(np.int32)
  counts = [len(o) for o in op]
  det_start = np.concatenate([[0], np.cumsum(counts + counts)]).astype(np.int64)
  det_ids = np.concatenate([pid, pid])
  det_xy = np.concatenate([np.concatenate(p1), np.concatenate(p2)]).astype(np.float64)
  return board.astype(np.float64), det_start, det_ids, det_xy, len(op)


def stereo_init(model, intrinsics, problem, engine=None):
  """mcba_stereo_init of a pair_problem: (rt0 [6], left poses [F, 4, 4], ok [F])."""
  from .intrinsics import intrinsics_engine
  board, det_start, det_ids, det_xy, F = problem
  eng = engine or intrinsics_engine()
  return eng.stereo_init(model, F, len(board), det_start, det_ids, det_xy, board, intrinsics)


def solve_pair(model, intrinsics, problem, fix_intrinsic=True, fix_aspect=False, engine=None, **solve_opts):
  """The stereo solve of a pair_problem from the cameras' parameters intrinsics [2, 5+nd]: a struct of R [3, 3], T [3], the intrinsics
  after the solve, err, the start and the solve summary."""
  from .intrinsics import intrinsics_engine
  eng = engine or intrinsics_engine()
  opts = dict(ftol=1e-10, xtol=1e-10, gtol=1e-10, max_nfev=100)
  opts.update(solve_opts)
  board, det_start, det_ids, det_xy, F = problem
  rt0, left, ok = stereo_init(model, intrinsics, problem, eng)
  if not ok.all():
    raise ValueError(f"view {int(np.flatnonzero(~ok)[0])}: the initial pose of the left or the right camera failed")
  bits = nat.OPT_BITS["camera_poses"] | nat.OPT_BITS["motion"]
  if not fix_intrinsic:
    bits |= nat.OPT_BITS["cameras"] | (nat.OPT_FIX_ASPECT if fix_aspect else 0)
  eng.table_from_detections(model, bits, (2, F, 1, len(board)), det_start, det_ids, det_xy, board[None])
  mats = np.concatenate([np.eye(4)[None], to_matrix(rt0)[None], np.eye(4)[None], left])
  eng.set_state_matrices(mats, intrinsics)
  info = eng.solve(**opts)
  sumsq, count = eng.view_errors()
  cams, _, _, intr = eng.get_state_matrices()
  T = cams[1] @ np.linalg.inv(cams[0])
  return struct(R=T[:3, :3], T=T[:3, 3], intrinsics=intr, err=float(np.sqrt(sumsq.sum() / count.sum())), rt0=rt0, solve=info)


def _calibrate(cameras, matches, fisheye, fix_aspect, fix_intrinsic, solve_opts):
  left, right = cameras
  assert left.image_size == right.image_size
  assert left.model == right.model
  model = "fisheye" if fisheye else left.model
  if not fix_intrinsic:
    if model in UNSUPPORTED_FREE:
      raise NotImplementedError(f"stereo calibration with free intrinsics of the {model} model: {UNSUPPORTED_FREE[model]}")
    if fix_aspect and not fisheye and any(c.intrinsic[0, 0] != c.intrinsic[1, 1] for c in cameras):
      raise NotImplementedError("fix_aspect with free intrinsics keeps each camera's fx / fy in OpenCV; the engine's aspect constraint "
                                "is fx = fy, so both cameras need fx == fy")
  intr = np.stack([_camera_params(left, model), _camera_params(right, model)])
  r = solve_pair(model, intr, pair_problem(matches), fix_intrinsic=fix_intrinsic, fix_aspect=fix_aspect and not fisheye, **solve_opts)
  Cam = CameraFisheye if fisheye else Camera
  out = []
  for c, cam in enumerate(cameras):
    if fix_intrinsic:
      K, d = cam.intrinsic, cam.dist
    else:
      x = r.intrinsics[c]
      K = np.array([[x[0], 0.0, x[2]], [0.0, x[1], x[3]], [0.0, 0.0, 1.0]])
      d = x[5:].reshape(np.shape(cam.dist))
    out.append(Cam(dist=d, intrinsic=K, image_size=left.image_size, model=left.model))
  pose = np.eye(4)
  pose[:3, :3], pose[:3, 3] = r.R, r.T
  return out[0], out[1], pose, r.err


def stereo_calibrate(cameras, matches, max_iter=60, eps=1e-6, fix_aspect=False, fix_intrinsic=True, **solve_opts):
  """camera.py:261-286 on the GPU: (left, right, 4x4 pose of the left camera in the right one's frame, err).  `matches` holds per-view
  lists object_points, points1, points2.  With fix_intrinsic the cameras' K and dist come back unchanged; free intrinsics are supported for
  the standard model.  `max_iter` / `eps` are accepted for the signature (module docstring); ftol, xtol, gtol, max_nfev go to the solve."""
  del max_iter, eps
  return _calibrate(cameras, matches, False, fix_aspect, fix_intrinsic, solve_opts)


def stereo_calibrate_fisheye(cameras, matches, max_iter=60, eps=1e-6, fix_aspect=False, fix_intrinsic=True, **solve_opts):
  """camera_fisheye.py:180-205 on the GPU, as the reference evidently meant it (it raises TypeError there: CameraFisheye.flags() takes no
  arguments): cv2.fisheye.stereoCalibrate with CameraFisheye.flags() | CALIB_USE_INTRINSIC_GUESS | CALIB_FIX_INTRINSIC * fix_intrinsic.
  fix_aspect is accepted and, as in those flags, has no effect."""
  del max_iter, eps
  return _calibrate(cameras, matches, True, fix_aspect, fix_intrinsic, solve_opts)


def intersect_detections(board, d1, d2):
  """image/detect.py:37-43: the corners both detections share, or None."""
  ids, i1, i2 = np.intersect1d(d1.ids, d2.ids, return_indices=True)
  if len(ids) == 0: return None
  return struct(points1=d1.corners[i1], points2=d2.corners[i2], object_points=np.asarray(board.points)[ids], ids=ids)


def matching_frames(detections, board, i, j):
  """The frames where cameras i and j see common corners of `board`, as per-view lists object_points, points1, points2, ids."""
  matching = [m for m in (intersect_detections(board, d1, d2) for d1, d2 in zip(detections[i], detections[j])) if m is not None]
  return struct(**{k: [m[k] for m in matching] for k in ("points1", "points2", "object_points", "ids")})


def stereo_calibrate_detections(detections, board, cameras, i, j, **kwargs):
  """image/detect.py:45-59: stereo_calibrate of cameras i and j over the corners of `board` that both detect, frame by frame;
  detections[camera][frame] = struct(corners, ids) of that board."""
  return stereo_calibrate((cameras[i], cameras[j]), matching_frames(detections, board, i, j), **kwargs)
