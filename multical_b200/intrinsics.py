"""Single-camera intrinsic calibration on the GPU: `Camera.calibrate` and `calibrate_cameras` of the reference (multical/camera.py:68-105,
237-241), which call cv2.calibrateCameraExtended once per round of a view-rejection loop, one camera at a time.

What stays on the host is the bookkeeping of the reference: the view set (calibration_points, camera.py:184-195, 229-235), the optional
`max_images` selection (top_detection_coverage, camera.py:206-227, with the same np.random.normal draws in the same order) and the loop
(camera.py:84-99).  Per round:
  1. one mcba_intrinsic_init for every camera still in the loop (include/mcba.h): homographies, OpenCV's initIntrinsicParams2D, per-view
     poses by PnP under K0 (csrc/intrinsics_kernels.cuh);
  2. per camera, the bundle-adjustment engine on a problem of one camera whose frames are its views (frame pose = board wrt camera;
     camera and board poses fixed at identity), optimising the frames and the intrinsics (fx = fy under fix_aspect; skew is a dead column
     as in OpenCV);
  3. mcba_view_errors: the per-view RMS and the total RMS of calibrateCameraExtended.

The solve iterates to its own tolerances (ftol = xtol = gtol = 1e-10, at most 100 evaluations): it reaches the minimum that OpenCV's
Levenberg-Marquardt approaches, not the point where OpenCV's criteria (`max_iter`, `eps`: accepted for the reference's signature, unused)
stop it -- with the reference's (10, 1e-3), OpenCV stops ~1e-5 relative away from it in fx.  The calibration runs on an engine of its own, so
the process-wide bundle-adjustment engine keeps its problem.

The fisheye model (CameraFisheye.calibrate / calibrate_cameras_fisheye, camera_fisheye.py:70-94, 173-177: one cv2.fisheye.calibrate per
camera, no loop) takes the same steps once: the same view set, OpenCV's fisheye start K0 with per-view poses by fisheye PnP under it
(mcba_intrinsic_init), the same one-camera problem without an aspect constraint, and the total RMS as err.

Both paths take OpenCV's fixed-parameter `flags` (CALIB_FIX_K1.., CALIB_FIX_PRINCIPAL_POINT, ...; pinhole_flags, fisheye_flags) as the
engine's fixed-intrinsics mask: the parameters they name keep K0's values, which are OpenCV's without an intrinsic guess."""
import numpy as np

from . import _native as nat
from .board import stack_boards
from .camera import Camera
from .structs import struct

SUPPORTED_MODELS = ("standard",)
UNSUPPORTED = {
  "rational": "k1..k3 and k4..k6 are nearly degenerate; in that valley the engine's trust region stops on xtol 1.7e-4 - 1.8e-4 above the "
              "RMS OpenCV's LM settles at (50-view scenes, restarts do not help), so the result would not be OpenCV's minimum",
  "thin_prism": "under CALIB_THIN_PRISM_MODEL OpenCV keeps k4..k6 at zero; the engine's fixed-intrinsics mask can hold them, but this "
                "model's free-intrinsics solve is not checked against OpenCV yet",
  "tilted": "under CALIB_TILTED_MODEL OpenCV keeps k4..k6 and s1..s4 at zero; the engine's fixed-intrinsics mask can hold them, but this "
            "model's free-intrinsics solve is not checked against OpenCV yet",
  "fisheye": "fisheye cameras calibrate with calibrate_cameras_fisheye / CameraFisheye.calibrate (the reference's camera_fisheye.py "
             "signature: no intrinsic_error_limit, no rejection loop)",
}
# CameraFisheye.model (camera_fisheye.py:43-49): stored on the camera; the reference never passes them to OpenCV's flags
FISHEYE_MODELS = ("standard", "fix_k1", "fix_k2", "fix_k3", "fix_k4")

# The `flags` the reference ORs into OpenCV's (camera.py:81, camera_fisheye.py:80), as the engine's fixed-intrinsics mask
# (mcba_set_fixed_intrinsics): flag bit -> (OpenCV's name, indices into Camera.params [fx fy cx cy skew dist...]).  Without an intrinsic
# guess OpenCV holds a fixed distortion coefficient at 0 and a fixed principal point at its start, which are K0's values; the fisheye
# focal lengths' start max(w, h) / 2 is K0's too.
PINHOLE_FIXED = {
  4: ("CALIB_FIX_PRINCIPAL_POINT", (2, 3)), 8: ("CALIB_ZERO_TANGENT_DIST", (7, 8)), 32: ("CALIB_FIX_K1", (5,)),
  64: ("CALIB_FIX_K2", (6,)), 128: ("CALIB_FIX_K3", (9,)),
  1 << 21: ("CALIB_FIX_TANGENT_DIST", (7, 8)),       # holds p1, p2 at their start, 0 without a guess: ZERO_TANGENT_DIST (OpenCV 4.13)
}
PINHOLE_FIX_ASPECT_RATIO = 2                          # the same as fix_aspect=True
PINHOLE_NO_EFFECT = {2048: "CALIB_FIX_K4", 4096: "CALIB_FIX_K5", 8192: "CALIB_FIX_K6", 65536: "CALIB_FIX_S1_S2_S3_S4",
                     524288: "CALIB_FIX_TAUX_TAUY"}     # coefficients the standard model does not have
FISHEYE_FIXED = {
  16: ("CALIB_FIX_K1", (5,)), 32: ("CALIB_FIX_K2", (6,)), 64: ("CALIB_FIX_K3", (7,)), 128: ("CALIB_FIX_K4", (8,)),
  512: ("CALIB_FIX_PRINCIPAL_POINT", (2, 3)), 2048: ("CALIB_FIX_FOCAL_LENGTH", (0, 1)),
}
FISHEYE_NO_EFFECT = {2: "CALIB_RECOMPUTE_EXTRINSIC", 8: "CALIB_FIX_SKEW"}      # the reference sets both itself
_NO_GUESS = "the reference passes no initial camera matrix (camera.py:86-88, camera_fisheye.py:91-92), so there is no guess to use"
PINHOLE_REFUSED = {
  1: ("CALIB_USE_INTRINSIC_GUESS", _NO_GUESS),
  16: ("CALIB_FIX_FOCAL_LENGTH", "OpenCV holds fx, fy at its own initCameraMatrix2D start, which K0 matches only to 1e-3 relative, so "
                                 "the held focal lengths and the whole fit would differ from OpenCV's"),
  16384: ("CALIB_RATIONAL_MODEL", "the camera model comes from `model`; this flag contradicts model='standard'"),
  32768: ("CALIB_THIN_PRISM_MODEL", "the camera model comes from `model`; this flag contradicts model='standard'"),
  262144: ("CALIB_TILTED_MODEL", "the camera model comes from `model`; this flag contradicts model='standard'"),
}
FISHEYE_REFUSED = {
  1: ("CALIB_USE_INTRINSIC_GUESS", _NO_GUESS),
  4: ("CALIB_CHECK_COND", "OpenCV's condition-number check of every view's extrinsic Jacobian is not implemented"),
}

_engines = {}


def intrinsics_engine(device=None):
  """An engine used only by the intrinsic calibration (one per GPU), so that calibration.get_engine()'s problem survives it."""
  from .calibration import default_device
  from .engine import Engine
  device = default_device() if device is None else device
  if device not in _engines:
    _engines[device] = Engine(device)
  return _engines[device]


def image_bins(image_size, approx_bins=10):
  """Bin edges over the image: square bins of side min(w, h) / approx_bins (camera.py:212-216)."""
  side = min(image_size[0] / approx_bins, image_size[1] / approx_bins)
  return [np.linspace(0, image_size[axis], int(image_size[axis] / side)) for axis in (0, 1)]


def top_detection_coverage(views, k, image_size, approx_bins=10, jitter=0.1):
  """The k views whose corners occupy the most bins of the image, ties broken by normal jitter (camera.py:219-227).  Draws one
  np.random.normal per view in view order, as the reference does."""
  bins = image_bins(image_size, approx_bins=10)
  scale = jitter * approx_bins * approx_bins
  score = []
  for v in views:
    hist, _, _ = np.histogram2d(v.corners[:, 0], v.corners[:, 1], bins)
    score.append(-np.count_nonzero(hist) + np.random.normal(0, scale))
  return [views[i] for i in np.argsort(score)][:k]


def calibration_points(boards, detections):
  """One view per (frame, board) with board.has_min_detections, board-major (camera.py:184-195, 229-235).  Corners and object points
  are rounded to float32, as the reference hands them to OpenCV."""
  views = []
  for b, board in enumerate(boards):
    for f, frame in enumerate(detections):
      d = frame[b]
      if board.has_min_detections(d):
        ids = np.asarray(d.ids).reshape(-1)
        views.append(struct(frame=f, board=b, ids=ids, corners=np.asarray(d.corners, np.float32).reshape(-1, 2),
                            object_points=np.asarray(board.points, np.float64)[ids].astype(np.float32)))
  return views


def _check_model(model):
  if model in UNSUPPORTED:
    raise NotImplementedError(f"intrinsic calibration of the {model} model: {UNSUPPORTED[model]}")
  assert model in SUPPORTED_MODELS, f"unknown camera model {model}"


def fixed_of_flags(flags, kint, fixed_bits, no_effect, refused, what):
  """OpenCV calibration flags -> the fixed-intrinsics mask bool[kint] (None when nothing is fixed).  A refused, unknown or unsupported
  bit raises NotImplementedError naming it."""
  flags = int(flags)
  for bit, (name, reason) in refused.items():
    if flags & bit: raise NotImplementedError(f"{what} flag {name} ({bit}) is not supported: {reason}")
  fixed = np.zeros(kint, bool)
  rest = flags
  for bit, (_, idx) in fixed_bits.items():
    if flags & bit: fixed[list(idx)] = True
    rest &= ~bit
  for bit in no_effect: rest &= ~bit
  if rest: raise NotImplementedError(f"{what} flag bits {rest} ({rest:#x}) are not supported flags of this calibration")
  return fixed if fixed.any() else None


def pinhole_flags(flags, model="standard"):
  """calibrateCamera flags -> (fixed-intrinsics mask or None, whether they fix the aspect ratio)."""
  fixed = fixed_of_flags(flags, 5 + nat.DIST_SIZES[model], PINHOLE_FIXED, set(PINHOLE_NO_EFFECT) | {PINHOLE_FIX_ASPECT_RATIO},
                         PINHOLE_REFUSED, "calibrateCamera")
  return fixed, bool(int(flags) & PINHOLE_FIX_ASPECT_RATIO)


def fisheye_flags(flags):
  """cv2.fisheye.calibrate flags -> fixed-intrinsics mask or None."""
  return fixed_of_flags(flags, 5 + nat.DIST_SIZES["fisheye"], FISHEYE_FIXED, FISHEYE_NO_EFFECT, FISHEYE_REFUSED, "cv2.fisheye.calibrate")


def _solve_camera(eng, model, fix_aspect, views, k0, poses, board_points, solve_opts, fixed=None):
  """One calibrateCameraExtended: the views as frames of a one-camera problem, started from K0 and the PnP poses."""
  nv = len(views)
  B, P = board_points.shape[:2]
  counts = np.zeros(nv * B, np.int64)                 # list i*B + v.board holds view i, every other list is empty
  for i, v in enumerate(views): counts[i * B + v.board] = v.ids.size
  det_start = np.concatenate([[0], np.cumsum(counts)])
  det_ids = np.concatenate([v.ids for v in views])
  det_xy = np.concatenate([v.corners.astype(np.float64) for v in views])
  bits = nat.OPT_BITS["motion"] | nat.OPT_BITS["cameras"] | (nat.OPT_FIX_ASPECT if fix_aspect else 0)
  eng.table_from_detections(model, bits, (1, nv, B, P), det_start, det_ids, det_xy, board_points)
  mats = np.concatenate([np.eye(4)[None], np.tile(np.eye(4), (B, 1, 1)), poses])
  eng.set_state_matrices(mats, k0[None])          # K0: zero distortion, and the principal point OpenCV holds fixed
  if fixed is not None: eng.set_fixed_intrinsics(fixed)
  info = eng.solve(**solve_opts)
  sumsq, count = eng.view_errors()
  per_view = np.array([sumsq[0, i, v.board] for i, v in enumerate(views)])
  n = np.array([count[0, i, v.board] for i, v in enumerate(views)])
  _, _, frame_rt, intr = eng.get_params()
  return struct(intrinsics=intr[0], rtvecs=frame_rt, per_view=np.sqrt(per_view / n), rms=float(np.sqrt(per_view.sum() / n.sum())),
                solve=info)


def init_views(boards, cam_views, image_sizes, model="standard", fix_aspect=False, engine=None):
  """mcba_intrinsic_init for each camera's list of views: (K0 [C, 5+nd], initial board-wrt-camera poses [C,F,B,4,4], ok [C,F,B]),
  indexed by the views' (frame, board)."""
  eng = engine or intrinsics_engine()
  board_points = stack_boards(boards)[0].astype(np.float32).astype(np.float64)
  F = max(max((v.frame for v in views), default=0) for views in cam_views) + 1
  B, P = board_points.shape[:2]
  Cn = len(cam_views)
  # detection lists of the views only: every other list of the [C, F, B] grid is empty
  counts = np.zeros(Cn * F * B, np.int64)
  order = sorted(((c, v.frame, v.board, v) for c, views in enumerate(cam_views) for v in views), key=lambda t: (t[0] * F + t[1]) * B + t[2])
  for c, f, b, v in order: counts[(c * F + f) * B + b] = v.ids.size
  det_start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
  det_ids = np.concatenate([t[3].ids for t in order]).astype(np.int32) if order else np.zeros(0, np.int32)
  det_xy = np.concatenate([t[3].corners.astype(np.float64) for t in order]) if order else np.zeros((0, 2))
  use = counts.reshape(Cn, F, B) > 0
  grid = np.array([[1, 1, 1, 0, 0]] * B, np.int32)              # the views are chosen already: no minimum-detections rule on the device
  return eng.intrinsic_init(model, (Cn, F, B, P), det_start, det_ids, det_xy, board_points, grid, image_sizes, use, fix_aspect)


def calibrate_views(boards, cam_views, image_sizes, model="standard", fix_aspect=False, engine=None, camera_ids=None, fixed=None,
                    **solve_opts):
  """One calibrateCameraExtended (model "fisheye": one cv2.fisheye.calibrate) for each camera's list of views (calibration_points
  entries, any order): returns per camera a struct of the intrinsics [fx fy cx cy skew dist...], the views' rtvecs (board wrt camera),
  per-view RMS, total RMS, K0 and the solve summary.  camera_ids: how errors name the cameras (default: their position in cam_views).
  fixed: bool[5+nd], the intrinsics held at K0's values (fixed_of_flags; None: all free)."""
  eng = engine or intrinsics_engine()
  opts = dict(ftol=1e-10, xtol=1e-10, gtol=1e-10, max_nfev=100)
  opts.update(solve_opts)
  board_points = stack_boards(boards)[0].astype(np.float32).astype(np.float64)
  k0, poses, ok = init_views(boards, cam_views, image_sizes, model, fix_aspect, eng)
  out = []
  names = list(range(len(cam_views))) if camera_ids is None else list(camera_ids)
  for c, views in enumerate(cam_views):
    if not np.isfinite(k0[c]).all():
      raise ValueError(f"camera {names[c]}: no initial camera matrix (degenerate homographies)")
    sel = [(v.frame, v.board) for v in views]
    failed = [(f, b) for f, b in sel if not ok[c, f, b]]
    if failed:
      raise ValueError(f"camera {names[c]}: the initial pose of the view (frame {failed[0][0]}, board {failed[0][1]}) failed")
    res = _solve_camera(eng, model, fix_aspect, views, k0[c], np.stack([poses[c, f, b] for f, b in sel]), board_points, opts,
                       fixed)
    res.k0 = k0[c]
    out.append(res)
  return out


def _camera_of(res, image_size, model, fix_aspect, has_skew, views, per_view):
  x = res.intrinsics
  K = np.array([[x[0], 0.0, x[2]], [0.0, x[1], x[3]], [0.0, 0.0, 1.0]])
  return Camera(image_size=image_size, intrinsic=K, dist=x[5:].reshape(1, -1), model=model, fix_aspect=fix_aspect, has_skew=has_skew,
                error_perview=per_view.reshape(-1, 1),
                intrinsic_dataset={"board_ids": [np.float64(v.board) for v in views], "image_ids": [v.frame for v in views]})


def calibrate_cameras(boards, points, image_sizes, intrinsic_error_limit, max_iter=10, eps=1e-3, model="standard", fix_aspect=False,
                      has_skew=False, flags=0, max_images=None, **solve_opts):
  """camera.py:237-241: (cameras, errs) for the nested detections points[camera][frame][board] = struct(corners, ids).  Every camera runs
  the loop of camera.py:84-99 on its own views; the initialisation of a round is one launch for all cameras still in the loop.
  `max_iter` / `eps` are accepted for the reference's signature: the device solves to its own tolerances (module docstring); the keyword
  arguments ftol, xtol, gtol, max_nfev go to the solve."""
  del max_iter, eps
  _check_model(model)
  fixed, flag_aspect = pinhole_flags(flags, model)
  aspect = fix_aspect or flag_aspect          # the returned Camera keeps the fix_aspect it was given, as the reference's does
  Cn = len(points)
  views, err, result, per_view = [], [None] * Cn, [None] * Cn, [None] * Cn
  for c in range(Cn):
    v = calibration_points(boards, points[c])
    if not v:
      raise ValueError(f"camera {c}: no view with the minimum detections of its board")
    if max_images is not None:
      v = top_detection_coverage(v, max_images, image_sizes[c])
    views.append(v)
  active = list(range(Cn))
  while active:
    res = calibrate_views(boards, [views[c] for c in active], [image_sizes[c] for c in active], model, aspect, camera_ids=active,
                          fixed=fixed, **solve_opts)
    still = []
    for c, r in zip(active, res):
      result[c], per_view[c] = r, r.per_view
      if len(views[c]) >= 15:
        err[c] = float("{:.2f}".format(r.rms))
        threshold = np.quantile(r.per_view, 0.95)
        views[c] = [v for v, e in zip(views[c], r.per_view) if e < threshold]
        if abs(err[c]) >= intrinsic_error_limit: still.append(c)
      else:
        # the reference raises its limit by 0.1 and calibrates the same views again until the limit passes the (unrounded) error:
        # identical input, identical result
        err[c] = r.rms
    active = still
  cams = [_camera_of(result[c], tuple(image_sizes[c]), model, fix_aspect, has_skew, views[c], per_view[c]) for c in range(Cn)]
  return cams, err


def calibrate(boards, intrinsic_error_limit, detections, image_size, max_iter=10, eps=1e-3, model="standard", fix_aspect=False,
              has_skew=False, flags=0, max_images=None, **solve_opts):
  """Camera.calibrate (camera.py:68-105) for one camera's detections[frame][board]: (Camera, err)."""
  cams, errs = calibrate_cameras(boards, [detections], [image_size], intrinsic_error_limit, max_iter=max_iter, eps=eps, model=model,
                                 fix_aspect=fix_aspect, has_skew=has_skew, flags=flags, max_images=max_images, **solve_opts)
  return cams[0], errs[0]


def calibrate_cameras_fisheye(boards, points, image_sizes, max_iter=10, eps=1e-3, model="standard", fix_aspect=False, has_skew=False,
                              flags=0, max_images=None, **solve_opts):
  """camera_fisheye.py:173-177: (cameras, errs) for the nested detections points[camera][frame][board], one cv2.fisheye.calibrate per
  camera (camera_fisheye.py:70-94) with CALIB_RECOMPUTE_EXTRINSIC | CALIB_FIX_SKEW: no rejection loop, no error limit.  The start is
  OpenCV's (mcba_intrinsic_init with the fisheye model, one launch for all cameras), the solve the same engine problem as the pinhole
  path's without an aspect constraint, err the total RMS sqrt(sum |e|^2 / corners).  `model` (fix_k1..fix_k4) and `fix_aspect` are only
  stored on the cameras, as the reference never passes them to OpenCV; `max_iter` / `eps` are accepted for the signature (the device
  solves to its own tolerances, module docstring).  With max_images, the np.random draws run camera by camera in order (the reference
  draws them from a thread pool, in whatever order its threads run)."""
  from .camera import CameraFisheye
  del max_iter, eps
  assert model in FISHEYE_MODELS, f"unknown camera model {model} options are {list(FISHEYE_MODELS)}"
  fixed = fisheye_flags(flags)
  views = []
  for c in range(len(points)):
    v = calibration_points(boards, points[c])
    if not v:
      raise ValueError(f"camera {c}: no view with the minimum detections of its board")
    if max_images is not None:
      v = top_detection_coverage(v, max_images, image_sizes[c])
    views.append(v)
  res = calibrate_views(boards, views, image_sizes, model="fisheye", fix_aspect=False, fixed=fixed, **solve_opts)
  cams = []
  for r, size in zip(res, image_sizes):
    x = r.intrinsics
    K = np.array([[x[0], 0.0, x[2]], [0.0, x[1], x[3]], [0.0, 0.0, 1.0]])
    cams.append(CameraFisheye(image_size=tuple(size), intrinsic=K, dist=x[5:9].reshape(4, 1).copy(), model=model, fix_aspect=fix_aspect,
                              has_skew=has_skew))
  return cams, [r.rms for r in res]


def calibrate_fisheye(boards, detections, image_size, max_iter=10, eps=1e-3, model="standard", fix_aspect=False, has_skew=False, flags=0,
                      max_images=None, **solve_opts):
  """CameraFisheye.calibrate (camera_fisheye.py:70-94) for one camera's detections[frame][board]: (CameraFisheye, err)."""
  cams, errs = calibrate_cameras_fisheye(boards, [detections], [image_size], max_iter=max_iter, eps=eps, model=model,
                                         fix_aspect=fix_aspect, has_skew=has_skew, flags=flags, max_images=max_images, **solve_opts)
  return cams[0], errs[0]
