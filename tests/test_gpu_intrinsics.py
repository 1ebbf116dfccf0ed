"""GPU (-m gpu): single-camera intrinsic calibration (multical_b200/intrinsics.py; include/mcba.h mcba_intrinsic_init, mcba_view_errors;
csrc/intrinsics_kernels.cuh) against OpenCV, called live, and against the reference's own Camera.calibrate (tests/golden/intrinsics_*.npz,
tests/golden/make_intrinsics_golden.py).

Bars:
  K0                 <= 1e-9 relative against oracle/intrinsics_oracle.py (the same homographies, initIntrinsicParams2D restated),
                     <= 1e-3 relative against cv2.initCameraMatrix2D, principal point exactly ((w-1)/2, (h-1)/2)
  converged solution against cv2.calibrateCameraExtended with criteria (COUNT+EPS, 500, 1e-15) and the same flags:
                     fx fy cx cy <= 1e-6 relative, dist <= 1e-6, total RMS <= 1e-9 relative, per-view RMS <= 1e-6 px, rvec / tvec <= 1e-6
  the reference's criteria (10, 1e-3): the device's RMS is not worse than OpenCV's (x (1 + 1e-12))
  full loop against the reference's goldens: same rounds, identical intrinsic_dataset, identical rounded err (unrounded: 1e-6 relative),
                     error_perview <= 1e-3 px and K <= 1e-3 relative (the gap is OpenCV's early stop)
"""
import numpy as np
import pytest

from conftest import GOLDEN
from multical_b200 import intrinsics, synthetic
from multical_b200.board import Board
from multical_b200.camera import Camera, calibrate_cameras
from multical_b200.structs import struct
from oracle import intrinsics_oracle

pytestmark = pytest.mark.gpu

TIGHT = dict(ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=200)     # k3 is weakly determined: solve well past the default 1e-10
CV_TIGHT = (3, 500, 1e-15)                                          # cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS


def scene_of(C, F, seed, model="standard", cube=False):
  kw = dict(boards=("cube", 10, 10, 0.04, 5), rig="dome", vis=0.8) if cube else dict(vis=0.4)
  return synthetic.make_scene(C=C, F=F, seed=seed, model=model, **kw)


def boards_of(scene, cube=False):
  size = (9, 9) if cube else (16, 22)
  return [Board(p, size=size, min_points=12 if cube else 20) for p in scene["board_points"]]


def detections(points, valid):
  """points [F,B,P,2], valid [F,B,P] -> detections[frame][board] = struct(corners, ids) (what Workspace.detected_points holds)."""
  return [[struct(corners=points[f, b][valid[f, b]].astype(np.float32), ids=np.flatnonzero(valid[f, b])) for b in range(valid.shape[1])]
          for f in range(valid.shape[0])]


def cv_calibrate(views, image_size, flags, criteria):
  import cv2
  op = [v.object_points.reshape(-1, 1, 3) for v in views]
  ip = [v.corners.reshape(-1, 1, 2) for v in views]
  rms, K, d, rv, tv, _, _, pv = cv2.calibrateCameraExtended(op, ip, tuple(image_size), None, None, criteria=criteria, flags=flags)
  return rms, K, d.ravel(), np.hstack([np.stack(rv)[:, :, 0], np.stack(tv)[:, :, 0]]), pv.ravel()


def run_init(C, F, fix_aspect):
  import cv2
  scene = scene_of(C, F, 71)
  boards = boards_of(scene)
  views = [intrinsics.calibration_points(boards, detections(scene["points"][c], scene["valid"][c])) for c in range(C)]
  eng = intrinsics.intrinsics_engine()
  res = intrinsics.calibrate_views(boards, views, [scene["image_size"]] * C, fix_aspect=fix_aspect, engine=eng, max_nfev=1)
  w, h = scene["image_size"]
  for c in range(C):
    k0 = res[c].k0
    assert k0[2] == (w - 1) * 0.5 and k0[3] == (h - 1) * 0.5 and (k0[4:] == 0).all()
    Hs = [intrinsics_oracle.homography(v.object_points, v.corners) for v in views[c]]
    K = intrinsics_oracle.init_intrinsics(Hs, scene["image_size"], aspect_ratio=1.0 if fix_aspect else 0.0)
    assert np.abs(k0[:2] / K[[0, 1], [0, 1]] - 1).max() <= 1e-9
    Kcv = cv2.initCameraMatrix2D([v.object_points.reshape(-1, 1, 3) for v in views[c]], [v.corners.reshape(-1, 1, 2) for v in views[c]],
                                 tuple(scene["image_size"]), aspectRatio=1.0 if fix_aspect else 0.0)
    assert np.abs(k0[:4] / Kcv[[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max() <= 1e-3
    if fix_aspect: assert k0[0] == k0[1]


@pytest.mark.parametrize("fix_aspect", [False, True])
def test_initial_camera_matrix_is_initIntrinsicParams2D(fix_aspect):
  run_init(3, 30, fix_aspect)


CONVERGED = {"standard": dict(model="standard"), "fix_aspect": dict(model="standard", fix_aspect=True),
             "cube": dict(model="standard", cube=True)}


def run_converged(case, F, report=None):
  import cv2
  spec = dict(CONVERGED[case])
  cube, fix_aspect = spec.pop("cube", False), spec.pop("fix_aspect", False)
  model = spec["model"]
  scene = scene_of(1, F, 72, model=model, cube=cube)
  boards = boards_of(scene, cube)
  views = intrinsics.calibration_points(boards, detections(scene["points"][0], scene["valid"][0]))
  assert len(views) >= (3 * F if cube else F // 2)
  flags = cv2.CALIB_FIX_ASPECT_RATIO if fix_aspect else 0
  rms, K, d, rt, pv = cv_calibrate(views, scene["image_size"], flags, CV_TIGHT)
  r = intrinsics.calibrate_views(boards, [views], [scene["image_size"]], model=model, fix_aspect=fix_aspect, **TIGHT)[0]
  x = r.intrinsics
  got = dict(K=np.abs(x[:4] / K[[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max(), dist=np.abs(x[5:] - d).max(), rms=abs(r.rms / rms - 1),
             per_view=np.abs(r.per_view - pv).max(), pose=np.abs(r.rtvecs - rt).max())
  if report is not None: report(case, len(views), got)
  assert got["K"] <= 1e-6 and got["dist"] <= 1e-6 and got["rms"] <= 1e-9 and got["per_view"] <= 1e-6 and got["pose"] <= 1e-6, got
  # the reference's own criteria stop OpenCV early: the device's minimum is not worse
  rms10 = cv_calibrate(views, scene["image_size"], flags, (3, 10, 1e-3))[0]
  r10 = intrinsics.calibrate_views(boards, [views], [scene["image_size"]], model=model, fix_aspect=fix_aspect)[0]
  assert r10.rms <= rms10 * (1 + 1e-12), (r10.rms, rms10)


@pytest.mark.parametrize("case", list(CONVERGED))
def test_converged_solution_matches_opencv(case):
  run_converged(case, 12 if case == "cube" else 50, report=lambda c, n, g: print(f"\nmargins {c} ({n} views): " +
                                                                                 ", ".join(f"{k} {v:.2e}" for k, v in g.items())))


def load_golden(name):
  z = dict(np.load(f"{GOLDEN}/{name}.npz", allow_pickle=False))
  boards = [Board(p, size=(16, 22)) for p in z["board_points"]]
  return z, boards, detections(z["points"], z["valid"])


def run_golden(name, monkeypatch):
  z, boards, dets = load_golden(name)
  rounds = []
  real = intrinsics.calibrate_views
  monkeypatch.setattr(intrinsics, "calibrate_views", lambda *a, **k: rounds.append(1) or real(*a, **k))
  if int(z["np_seed"]) >= 0: np.random.seed(int(z["np_seed"]))
  kw = dict(model=str(z["model"]))
  if int(z["max_images"]) >= 0: kw["max_images"] = int(z["max_images"])
  cam, err = Camera.calibrate(boards, float(z["limit"]), dets, tuple(int(v) for v in z["image_size"]), **kw)
  ds = cam.intrinsic_dataset
  assert np.array_equal(np.asarray(ds["board_ids"], np.float64), z["board_ids"])
  assert np.array_equal(np.asarray(ds["image_ids"]), z["image_ids"])
  pv = np.asarray(cam.error_perview).ravel()
  assert pv.shape == z["error_perview"].shape and np.abs(pv - z["error_perview"]).max() <= 1e-3
  assert np.abs(cam.intrinsic[[0, 1, 0, 1], [0, 1, 2, 2]] / z["K"][[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max() <= 1e-3
  if len(pv) >= 15:
    assert err == float(z["err"]) and len(rounds) == int(z["rounds"])
  else:
    assert abs(err / float(z["err"]) - 1) <= 1e-6 and len(rounds) == 1
  return cam, err


@pytest.mark.parametrize("name", ["intrinsics_loop_40", "intrinsics_small_12", "intrinsics_max_images_36"])
def test_calibrate_loop_matches_reference_golden(name, monkeypatch):
  run_golden(name, monkeypatch)


def test_golden_errors_are_away_from_the_rounding_boundary():
  """The rounded err of the >= 15-view branch is compared for equality: the device's RMS of the last round sits more than 1e-4 px from a
  rounding boundary (and the reference's differs from it by far less: OpenCV's early stop moves the RMS by ~1e-7 relative)."""
  for name in ["intrinsics_loop_40", "intrinsics_max_images_36"]:
    z, boards, dets = load_golden(name)
    if int(z["np_seed"]) >= 0: np.random.seed(int(z["np_seed"]))
    views = intrinsics.calibration_points(boards, dets)
    if int(z["max_images"]) >= 0: views = intrinsics.top_detection_coverage(views, int(z["max_images"]), tuple(z["image_size"]))
    for _ in range(int(z["rounds"])):
      r = intrinsics.calibrate_views(boards, [views], [tuple(z["image_size"])])[0]
      views = [v for v, e in zip(views, r.per_view) if e < np.quantile(r.per_view, 0.95)]
    assert abs(r.rms * 100 - np.floor(r.rms * 100) - 0.5) * 0.01 > 1e-4, (name, r.rms)
    assert {(v.frame, v.board) for v in views} == {(int(f), int(b)) for f, b in zip(z["image_ids"], z["board_ids"])}


def test_unsupported_models_non_planar_boards_and_cameras_without_views():
  scene = scene_of(1, 6, 73)
  boards = boards_of(scene)
  dets = detections(scene["points"][0], scene["valid"][0])
  for model in ["rational", "thin_prism", "tilted", "fisheye"]:
    with pytest.raises(NotImplementedError, match=model):
      Camera.calibrate(boards, 1.0, dets, scene["image_size"], model=model)
  with pytest.raises(NotImplementedError):
    Camera.calibrate(boards, 1.0, dets, scene["image_size"], flags=1)
  lifted = [Board(np.asarray(b.points) + [0, 0, 0.01], size=(16, 22)) for b in boards]
  with pytest.raises(NotImplementedError, match="non-planar"):
    Camera.calibrate(lifted, 1.0, dets, scene["image_size"])
  empty = [[struct(corners=np.zeros((0, 2), np.float32), ids=np.zeros(0, np.int64)) for _ in boards] for _ in dets]
  with pytest.raises(ValueError, match="camera 1"):
    calibrate_cameras(boards, [dets, empty], [scene["image_size"]] * 2, 1.0)
  # an error in a later round names the camera by its place in the caller's list, not among the cameras still in the loop
  bad = intrinsics.calibration_points(boards, dets)
  bad[0] = bad[0]._extend(corners=np.full_like(bad[0].corners, 100.0))        # every corner at one pixel: no homography
  with pytest.raises(ValueError, match="camera 2"):
    intrinsics.calibrate_views(boards, [bad], [scene["image_size"]], camera_ids=[2])


def run_batched_and_reproducible(C, F):
  """Two identical calls agree bit for bit, and the batched initialisation of several cameras gives each camera exactly what it gets alone."""
  scene = scene_of(C, F, 74)
  boards = boards_of(scene)
  dets = [detections(scene["points"][c], scene["valid"][c]) for c in range(C)]
  a, ea = calibrate_cameras(boards, dets, [scene["image_size"]] * C, 0.1)
  b, eb = calibrate_cameras(boards, dets, [scene["image_size"]] * C, 0.1)
  for c in range(C):
    alone, e1 = Camera.calibrate(boards, 0.1, dets[c], scene["image_size"])
    for cam in (b[c], alone):
      assert np.array_equal(a[c].intrinsic, cam.intrinsic) and np.array_equal(a[c].dist, cam.dist)
      assert np.array_equal(a[c].error_perview, cam.error_perview) and a[c].intrinsic_dataset == cam.intrinsic_dataset
    assert ea[c] == eb[c] == e1


def test_batched_cameras_and_bit_reproducible():
  run_batched_and_reproducible(3, 20)


def run_view_errors_of_a_bundle_adjustment(motion):
  """mcba_view_errors on ordinary bundle-adjustment problems, static and rolling frames: per-(camera, frame, board) sums of the squared
  residuals of the oracle's own projection (oracle/ba_oracle.py) and corner counts."""
  from multical_b200.calibration import from_scene
  from multical_b200.motion import RollingFrames
  from oracle.ba_oracle import Problem
  scene = synthetic.make_scene(C=2, F=5, vis=0.5, seed=75)
  calib = from_scene(scene)
  if motion == "rolling":
    start = scene["init"]["frame_poses"]
    end = synthetic.to_matrix(synthetic.from_matrix(start) + 1e-3 * np.random.default_rng(7).standard_normal((scene["F"], 6)))
    calib = calib.copy(motion=RollingFrames(start, end, scene["frame_valid"], [str(i) for i in range(scene["F"])]))
    prob = Problem.from_scene(scene, optimize=dict(cameras=True), motion="rolling", frame_poses_end=end, image_size=scene["image_size"])
  else:
    prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  calib = calib.enable(cameras=True)
  eng = calib._upload(calib.inliers)
  x = prob.param_vec
  eng.set_param_vec(x)
  r = prob.residuals(x).reshape(-1, 2)
  idx = np.argwhere(np.asarray(calib.inliers))
  want, n = np.zeros((2, 5, scene["B"])), np.zeros((2, 5, scene["B"]), np.int64)
  np.add.at(want, tuple(idx[:, :3].T), (r ** 2).sum(axis=1))
  np.add.at(n, tuple(idx[:, :3].T), 1)
  sumsq, count = eng.view_errors()
  assert np.array_equal(count, n) and (n > 0).sum() > 4
  assert (np.abs(sumsq - want) <= 1e-8 * want + 1e-12).all(), np.abs(sumsq - want).max()


@pytest.mark.parametrize("motion", ["static", "rolling"])
def test_view_errors_of_a_bundle_adjustment(motion):
  run_view_errors_of_a_bundle_adjustment(motion)


def test_calibrate_single_keeps_the_bundle_adjustment_engine_problem():
  from multical_b200 import workspace
  from multical_b200.calibration import from_scene, get_engine
  scene = scene_of(2, 16, 76)
  calib = from_scene(scene).enable(cameras=True)
  eng = calib._upload(calib.inliers)
  r0 = eng.residuals()
  boards = boards_of(scene)
  cams, errs = workspace.calibrate_single(boards, [detections(scene["points"][c], scene["valid"][c]) for c in range(2)],
                                          [scene["image_size"]] * 2, "standard", 1.0)
  assert get_engine() is eng and np.array_equal(eng.residuals(), r0)
  assert len(cams) == 2 and all(abs(e) < 1.0 for e in errs)
  K = scene["gt"]["K"]
  for c in range(2): assert np.abs(cams[c].intrinsic[[0, 1], [0, 1]] / K[c][[0, 1], [0, 1]] - 1).max() < 0.01
