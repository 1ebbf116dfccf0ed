"""GPU (-m gpu): stereo calibration of a camera pair (multical_b200/stereo.py stereo_calibrate, stereo_calibrate_fisheye,
stereo_calibrate_detections; include/mcba.h mcba_stereo_init; csrc/stereo_kernels.cuh k_stereo_start) against cv2.stereoCalibrate and
cv2.fisheye.stereoCalibrate, called live, against oracle/stereo_oracle.py and against the reference's own stereo_calibrate_detections
(tests/golden/stereo_*.npz, tests/golden/make_stereo_golden.py).

Bars:
  start              the median relative pose of mcba_stereo_init equals the oracle's on the device's own per-view poses to 1e-12
  converged solution against OpenCV with criteria (COUNT+EPS, 500, 1e-15) (free intrinsics: CV_FREE) and the reference's flags.
                     Fixed intrinsics: rotation vector and T <= 1e-6, RMS <= 1e-9 relative (fisheye: the RMS at the solution OpenCV
                     returns, see fisheye_rms).  Free intrinsics: OpenCV's LM has not converged (run_converged), so the device's RMS
                     must not be above OpenCV's, started from the cameras and from the device's solution, and the parameters meet the
                     FREE_* bars against the second run
  the reference's criteria (60, 1e-6): the device's RMS is not worse than OpenCV's (x (1 + 1e-12))
  against the reference's goldens: the same frames and the bars of GOLDEN, set from the measured gaps (OpenCV's early stop at
                     (60, 1e-6); with free intrinsics its LM is far from converged there), and err not above the reference's
"""
import time

import numpy as np
import pytest

from conftest import GOLDEN as GOLDEN_DIR
from multical_b200 import intrinsics, stereo, synthetic
from multical_b200.camera import Camera, CameraFisheye, stereo_calibrate, stereo_calibrate_fisheye
from multical_b200.rtvec import from_matrix
from multical_b200.structs import struct
from oracle import stereo_oracle

pytestmark = pytest.mark.gpu

TIGHT = dict(ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)
CV_TIGHT = (3, 500, 1e-15)                                          # cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS
CV_REF = (3, 60, 1e-6)                                              # the reference's default criteria
# free intrinsics: OpenCV's LM never meets eps 1e-15 there and runs every iteration allowed (cv2.fisheye: 64 s for 500 at 40 views on
# a 16-thread host; its RMS at 60, 100 and 500 iterations agrees to 2e-11 relative)
CV_FREE = (3, 100, 1e-15)
POSE_BAR, RMS_BAR = 1e-6, 1e-9
# OpenCV does not converge over free pinhole intrinsics (run_converged).  Measured at 40 views on an H100 80GB HBM3 (700 W): standard
# pose 6.3e-5, K 1.1e-4, dist 3.9e-4; fisheye pose 9.5e-8, K 1.4e-7, dist 3.0e-4 (k3, k4 are poorly determined, as in DESIGN.md §3d)
FREE_POSE_BAR, FREE_K_BAR, FREE_DIST_BAR = 5e-4, 1e-3, 5e-3
GOLDEN = dict(fixed=dict(err=1e-6, pose=1e-6, K=0.0), free=dict(err=5e-4, pose=1e-4, K=5e-4))
SIGMA_RMS = 0.3 * np.sqrt(2)                                        # make_scene's pixel noise, over u and v
CONVERGED = [("standard", True), ("rational", True), ("thin_prism", True), ("tilted", True), ("fisheye", True), ("standard", False),
             ("fisheye", False)]


def scene_of(F, seed, model="standard", vis=0.5, **kw):
  return synthetic.make_scene(C=2, F=F, seed=seed, model=model, vis=vis, **kw)


def matches_of(scene, equal=None):
  """What stereo_calibrate_detections hands to stereo_calibrate: per view the corners both cameras see (float32, as detected).
  equal (default: for fisheye scenes) keeps the first n of each view's corners, n the smallest count: cv2.fisheye.stereoCalibrate of
  OpenCV 4.13 fails on views of different sizes ("Can't reallocate Mat with locked size")."""
  bp = scene["board_points"][0].astype(np.float32)
  m = struct(object_points=[], points1=[], points2=[], ids=[])
  common = [np.intersect1d(np.flatnonzero(scene["valid"][0, f, 0]), np.flatnonzero(scene["valid"][1, f, 0])) for f in range(scene["F"])]
  n = min(c.size for c in common if c.size)
  for f, ids in enumerate(common):
    if ids.size == 0: continue
    if equal or (equal is None and scene["model"] == "fisheye"): ids = ids[:n]
    m.object_points.append(bp[ids]); m.ids.append(ids)
    m.points1.append(scene["points"][0, f, 0, ids].astype(np.float32)); m.points2.append(scene["points"][1, f, 0, ids].astype(np.float32))
  return m


def cameras_of(scene, jitter=0.0, square=False, seed=0):
  fisheye = scene["model"] == "fisheye"
  K, d = scene["gt"]["K"].copy(), scene["gt"]["dist"].copy()
  rng = np.random.default_rng(seed)
  if jitter:
    K[:, 0, 0] *= 1 + rng.normal(0, jitter, 2); K[:, 1, 1] *= 1 + rng.normal(0, jitter, 2)
  if square: K[:, 1, 1] = K[:, 0, 0]
  if fisheye:
    return [CameraFisheye(image_size=scene["image_size"], intrinsic=K[c], dist=d[c].reshape(4, 1)) for c in range(2)]
  return [Camera(image_size=scene["image_size"], intrinsic=K[c], dist=d[c], model=scene["model"]) for c in range(2)]


def cv_stereo(cams, m, criteria, fix_intrinsic=True, fix_aspect=False):
  """The reference's OpenCV call (copies in: OpenCV writes K and dist into the arrays it is given) -> (err, K1, d1, K2, d2, rtvec)."""
  import cv2
  l, r = cams
  args = [l.intrinsic.copy(), l.dist.copy(), r.intrinsic.copy(), r.dist.copy(), tuple(l.image_size)]
  if isinstance(l, CameraFisheye):
    flags = (cv2.fisheye.CALIB_RECOMPUTE_EXTRINSIC | cv2.fisheye.CALIB_FIX_SKEW | cv2.fisheye.CALIB_USE_INTRINSIC_GUESS
             | cv2.fisheye.CALIB_FIX_INTRINSIC * fix_intrinsic)
    err, K1, d1, K2, d2, R, T, rv, tv = cv2.fisheye.stereoCalibrate([o[None] for o in m.object_points], [p[None] for p in m.points1],
                                                                    [p[None] for p in m.points2], *args, flags=flags, criteria=criteria)
    return fisheye_rms(m, K1, d1, K2, d2, R, T, rv, tv), K1, d1, K2, d2, np.concatenate([cv2.Rodrigues(R)[0].ravel(), np.ravel(T)]), err
  else:
    model = dict(standard=0, rational=cv2.CALIB_RATIONAL_MODEL, tilted=cv2.CALIB_TILTED_MODEL, thin_prism=cv2.CALIB_THIN_PRISM_MODEL)
    flags = (model[l.model] | cv2.CALIB_FIX_ASPECT_RATIO * fix_aspect | cv2.CALIB_USE_INTRINSIC_GUESS
             | cv2.CALIB_FIX_INTRINSIC * fix_intrinsic)
    out = cv2.stereoCalibrate([o[:, None] for o in m.object_points], [p[:, None] for p in m.points1], [p[:, None] for p in m.points2],
                              *args, criteria=criteria, flags=flags)
  err, K1, d1, K2, d2, R, T = out[:7]
  return err, K1, d1, K2, d2, np.concatenate([cv2.Rodrigues(R)[0].ravel(), np.ravel(T)]), err


def fisheye_rms(m, K1, d1, K2, d2, R, T, rvecs, tvecs):
  """sqrt(sum |e|^2 / 2N) at the solution cv2.fisheye.stereoCalibrate returns.  The err it returns is not this: it is 1e-7 - 5e-7
  relative above the RMS of its own returned poses (12 and 40 views), while its poses agree with the device's to 1e-8."""
  import cv2
  s, n = 0.0, 0
  for o, a, b, rv, tv in zip(m.object_points, m.points1, m.points2, rvecs, tvecs):
    X = o[None].astype(np.float64)
    pa, _ = cv2.fisheye.projectPoints(X, rv, tv, K1, d1)
    R1 = cv2.Rodrigues(rv)[0]
    pb, _ = cv2.fisheye.projectPoints(X, cv2.Rodrigues(R @ R1)[0], R @ np.ravel(tv) + np.ravel(T), K2, d2)
    s += ((pa.reshape(-1, 2) - a) ** 2).sum() + ((pb.reshape(-1, 2) - b) ** 2).sum()
    n += len(o)
  return float(np.sqrt(s / (2 * n)))


def calibrate(cams, m, **kw):
  fn = stereo_calibrate_fisheye if isinstance(cams[0], CameraFisheye) else stereo_calibrate
  return fn(cams, m, **kw)


def run_start(F, report=print):
  """The start against the oracle on the device's own per-view poses (k_pnp_views through mcba_pnp_views: the same kernel)."""
  scene = scene_of(F, 71)
  m = matches_of(scene)
  assert len(m.object_points) == F
  cams = cameras_of(scene)
  problem = stereo.pair_problem(m)
  board, det_start, det_ids, det_xy, nv = problem
  intr = np.stack([stereo._camera_params(c, "standard") for c in cams])
  rt0, left, ok = stereo.stereo_init("standard", intr, problem)
  poses, _, _, valid = intrinsics.intrinsics_engine().pnp_views("standard", (2, nv, 1, len(board)), det_start, det_ids, det_xy, board[None],
                                                                intr, [[1, 1, 1, 0, 0]])
  assert np.array_equal(poses[0, :, 0], left) and np.array_equal(valid[0, :, 0] & valid[1, :, 0], ok) and ok.all()
  want = stereo_oracle.median_start(poses[0, :, 0], poses[1, :, 0], ok)
  gap = np.abs(rt0 - want).max()
  report(f"\nstart ({F} views): {gap:.2e} from the oracle")
  assert gap <= 1e-12, (rt0, want)
  again = stereo.stereo_init("standard", intr, problem)
  assert all(np.array_equal(a, b) for a, b in zip(again, (rt0, left, ok)))


@pytest.mark.parametrize("F", [21, 40])
def test_start_is_the_median_relative_pose(F):
  run_start(F)


def run_converged(model, fix_intrinsic, F, seed=73, report=print):
  scene = scene_of(F, seed, model)
  m = matches_of(scene)
  cams = cameras_of(scene, jitter=0.0 if fix_intrinsic else 0.01)
  left, right, pose, err = calibrate(cams, m, fix_intrinsic=fix_intrinsic, **TIGHT)
  criteria = CV_TIGHT if fix_intrinsic else CV_FREE
  err_cv, K1, d1, K2, d2, rt_cv, raw = cv_stereo(cams, m, criteria, fix_intrinsic)
  if not fix_intrinsic:
    # OpenCV's LM over free pinhole intrinsics is still descending after 500 iterations (40 views: RMS 0.42427 at 500, 0.42423 at 5000;
    # the device's minimum is 0.42417).  Started from the device's solution it restarts its own extrinsics and ends 4.5e-6 relative
    # above the device's RMS (12 views).  So: the device's RMS is not above either run, and the parameters are compared with the second
    # one at the FREE_* bars, set from those measured gaps
    assert err <= err_cv * (1 + RMS_BAR), (err, err_cv)
    err_cv, K1, d1, K2, d2, rt_cv, raw = cv_stereo((left, right), m, criteria, fix_intrinsic)
    assert err <= err_cv * (1 + RMS_BAR), (err, err_cv)
  assert type(left) is type(cams[0]) and left.image_size == cams[0].image_size and pose.shape == (4, 4)
  got = dict(rms=abs(err / err_cv - 1), pose=np.abs(from_matrix(pose) - rt_cv).max())
  if fix_intrinsic:
    for a, b in zip((left, right), cams):
      assert np.array_equal(a.intrinsic, b.intrinsic) and np.array_equal(a.dist, b.dist)
  else:
    idx = ([0, 1, 0, 1], [0, 1, 2, 2])
    got["K"] = max(np.abs(left.intrinsic[idx] / K1[idx] - 1).max(), np.abs(right.intrinsic[idx] / K2[idx] - 1).max())
    got["dist"] = max(np.abs(left.dist.ravel() - d1.ravel()).max(), np.abs(right.dist.ravel() - d2.ravel()).max())
    assert left.dist.shape == cams[0].dist.shape
  report(f"\nmargins {model} fix_intrinsic={fix_intrinsic} ({len(m.object_points)} views): "
         + ", ".join(f"{k} {v:.2e}" for k, v in got.items()) + f"; OpenCV's own err {abs(raw / err - 1):.2e} relative")
  if fix_intrinsic:
    assert got["rms"] <= RMS_BAR and got["pose"] <= POSE_BAR, got
  else:
    assert got["pose"] <= FREE_POSE_BAR and got["K"] <= FREE_K_BAR and got["dist"] <= FREE_DIST_BAR, got
    if model == "fisheye": assert got["rms"] <= RMS_BAR, got          # cv2.fisheye.stereoCalibrate does reach the minimum
  # the reference's own criteria stop OpenCV early: the device's minimum is not worse
  err60 = cv_stereo(cams, m, CV_REF, fix_intrinsic)[0]
  err_dev = calibrate(cams, m, fix_intrinsic=fix_intrinsic)[3]
  assert err_dev <= err60 * (1 + 1e-12), (err_dev, err60)


@pytest.mark.parametrize("model,fix_intrinsic", CONVERGED)
def test_converged_solution_matches_opencv(model, fix_intrinsic):
  run_converged(model, fix_intrinsic, 40)


def detections_of(z):
  return [[struct(corners=z["points"][c, f][z["valid"][c, f]], ids=np.flatnonzero(z["valid"][c, f])) for f in range(z["valid"].shape[1])]
          for c in range(2)]


def run_golden(name, report=print):
  z = dict(np.load(f"{GOLDEN_DIR}/{name}.npz", allow_pickle=False))
  dets = detections_of(z)
  board = struct(points=z["board_points"])
  size, model = tuple(int(v) for v in z["image_size"]), str(z["model"])
  cams = [Camera(image_size=size, intrinsic=z["K_in"][c], dist=z["dist_in"][c], model=model) for c in range(2)]
  m = stereo.matching_frames(dets, board, 0, 1)
  kept = [f for f in range(len(dets[0])) if np.intersect1d(dets[0][f].ids, dets[1][f].ids).size]
  assert np.array_equal(kept, z["frames"]) and np.array_equal([len(o) for o in m.object_points], z["view_sizes"])
  left, right, pose, err = stereo.stereo_calibrate_detections(dets, board, cams, 0, 1, fix_intrinsic=bool(z["fix_intrinsic"]))
  idx = ([0, 1, 0, 1], [0, 1, 2, 2])
  got = dict(err=abs(err / float(z["err"]) - 1), pose=np.abs(from_matrix(pose) - from_matrix(z["pose"])).max(),
             K=max(np.abs(left.intrinsic[idx] / z["K1"][idx] - 1).max(), np.abs(right.intrinsic[idx] / z["K2"][idx] - 1).max()))
  report(f"\ngolden {name} ({len(kept)} views): " + ", ".join(f"{k} {v:.2e}" for k, v in got.items()))
  bars = GOLDEN["fixed" if bool(z["fix_intrinsic"]) else "free"]
  assert all(got[k] <= bars[k] for k in bars), got
  assert err <= float(z["err"]) * (1 + 1e-12)


@pytest.mark.parametrize("name", ["stereo_standard_fixed", "stereo_standard_free", "stereo_rational_fixed"])
def test_matches_reference_golden(name):
  run_golden(name)


def run_refusals(F=12):
  import cv2
  scene = scene_of(F, 74)
  m = matches_of(scene)
  cams = cameras_of(scene)
  # mismatched image sizes or models: the reference's asserts
  with pytest.raises(AssertionError):
    stereo_calibrate([cams[0], cams[1].copy(image_size=(1280, 720))], m)
  with pytest.raises(AssertionError):
    stereo_calibrate([cams[0], Camera(cams[1].image_size, cams[1].intrinsic, np.zeros(8), model="rational")], m)
  # free intrinsics of a model whose OpenCV fit the engine cannot restate
  for model, nd in (("rational", 8), ("thin_prism", 12), ("tilted", 14)):
    pair = [Camera(c.image_size, c.intrinsic, np.zeros(nd), model=model) for c in cams]
    with pytest.raises(NotImplementedError, match=model):
      stereo_calibrate(pair, m, fix_intrinsic=False)
  # fix_aspect with free intrinsics: OpenCV keeps each camera's fx / fy, which the engine's fx = fy constraint restates only at 1
  skewed = cameras_of(scene, jitter=0.01)
  with pytest.raises(NotImplementedError, match="fx == fy"):
    stereo_calibrate(skewed, m, fix_aspect=True, fix_intrinsic=False)
  _, K1, _, K2, _, _, _ = cv_stereo(skewed, m, CV_REF, fix_intrinsic=False, fix_aspect=True)
  for Kin, Kout in zip((c.intrinsic for c in skewed), (K1, K2)):
    assert Kout[0, 0] != Kin[0, 0] and abs(Kout[0, 0] / Kout[1, 1] - Kin[0, 0] / Kin[1, 1]) <= 1e-12
  square = cameras_of(scene, jitter=0.01, square=True)
  left, right, _, _ = stereo_calibrate(square, m, fix_aspect=True, fix_intrinsic=False)
  assert left.intrinsic[0, 0] == left.intrinsic[1, 1] and right.intrinsic[0, 0] == right.intrinsic[1, 1]
  # non-planar object points: OpenCV runs its own (non-planar) start, the device's PnP is planar
  lifted = m._extend(object_points=[(o + np.array([0, 0, 0.01]) * (np.arange(len(o))[:, None] % 2)).astype(np.float32)
                                    for o in m.object_points])
  with pytest.raises(NotImplementedError, match="non-planar"):
    stereo_calibrate(cams, lifted)
  cv_stereo(cams, lifted, CV_REF)
  # a view of 3 points: OpenCV 4.13 asserts npoints >= 4 in solvePnPGeneric
  short = m._extend(**{k: [v[:3] if i == 2 else v for i, v in enumerate(m[k])] for k in ("object_points", "points1", "points2")})
  with pytest.raises(ValueError, match="view 2 has 3 points"):
    stereo_calibrate(cams, short)
  with pytest.raises(cv2.error, match="npoints >= 4"):
    cv_stereo(cams, short, CV_REF)


def test_refusals():
  run_refusals()


def run_reproducible_and_isolated(F=20):
  """Two identical calls agree bit for bit; a bundle-adjustment problem uploaded on calibration.get_engine() survives a stereo call."""
  from multical_b200.calibration import from_scene, get_engine
  calib = from_scene(synthetic.make_scene(C=3, F=8, vis=0.6, seed=75)).enable(cameras=True)
  eng = calib._upload(calib.inliers)
  r0 = eng.residuals()
  scene = scene_of(F, 76)
  m = matches_of(scene)
  for jit in (0.0, 0.01):
    cams = cameras_of(scene, jitter=jit)
    a = stereo_calibrate(cams, m, fix_intrinsic=jit == 0.0)
    b = stereo_calibrate(cams, m, fix_intrinsic=jit == 0.0)
    assert np.array_equal(a[2], b[2]) and a[3] == b[3]
    assert all(np.array_equal(x.intrinsic, y.intrinsic) and np.array_equal(x.dist, y.dist) for x, y in zip(a[:2], b[:2]))
  assert get_engine() is eng and np.array_equal(eng.residuals(), r0)


def test_reproducible_and_leaves_the_bundle_adjustment_problem_alone():
  run_reproducible_and_isolated()


def test_thousand_views_converge_to_the_noise():
  scene = scene_of(1000, 77, vis=0.4)
  m = matches_of(scene)
  cams = cameras_of(scene)
  stereo_calibrate(cams, m)                                         # warm-up: module load, buffers
  t0 = time.perf_counter()
  _, _, pose, err = stereo_calibrate(cams, m)
  dt = time.perf_counter() - t0
  n = sum(len(o) for o in m.object_points)
  want = SIGMA_RMS * np.sqrt(1 - (6 * len(m.object_points) + 6) / (4 * n))      # less the degrees of freedom the fit absorbs
  gt = scene["gt"]["cam_poses"]
  truth = from_matrix(gt[1] @ np.linalg.inv(gt[0]))
  print(f"\n2 x {len(m.object_points)} views, {n} corners per camera: {dt * 1e3:.1f} ms end to end, RMS {err:.4f} (expected {want:.4f}), "
        f"pose {np.abs(from_matrix(pose) - truth).max():.2e} from the truth")
  assert abs(err / want - 1) <= 0.01, (err, want)
