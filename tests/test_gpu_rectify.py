"""GPU (-m gpu): rectifying a calibrated pair (multical_b200/rectify.py; include/mcba.h mcba_rectify_*; csrc/undistort_kernels.cuh
k_rectify_map, k_rectify_points) against OpenCV, called live.

Bars:
  stereo_rectify          R1, R2 within 1e-12; P1, P2, Q within 1e-9 relative; ROIs equal to cv2.stereoRectify's: the four pinhole
                          models, horizontal and vertical pairs, alpha -1, 0, 0.5, 1, new_size equal to and unlike the image, with and
                          without CALIB_ZERO_DISPARITY
  stereo_rectify_fisheye  the same bars against cv2.fisheye.stereoRectify over balance and fov_scale
  maps                    bit-identical to cv2.initUndistortRectifyMap(K, d, R, P, size, CV_32FC2) for the five models (the fisheye twin's
                          CV_32F pair stacked), with and without skew, at odd widths and a size unlike the image's; rows longer than one
                          segment of the kernel's row walk, for the rectification and the undistortion (R = I, P = K)
  images                  bit-identical to cv2.remap(image, OpenCV's map, None, INTER_CUBIC), 1 and 3 channels
  points                  within 1e-9 px of cv2.undistortPoints(R=R, P=P) and cv2.fisheye.undistortPoints(R, P)
  end to end              a pair calibrated by stereo_calibrate, rectified: noise-free detections land on equal rows (1e-6 px) and Q
                          recovers the point in the rectified left frame (1e-9 relative); the same for two cameras of a bundle-adjusted rig
  repeated calls          bit for bit
"""
import ctypes as C

import numpy as np
import pytest

from multical_b200 import rectify, undistort
from multical_b200.camera import Camera, CameraFisheye, rectify_images, stereo_calibrate, stereo_rectify, stereo_rectify_fisheye
from test_gpu_undistort import DIST, MODELS, images, make_camera
from test_gpu_undistort import cv_map as cv_undistort_map

pytestmark = pytest.mark.gpu

PINHOLE = ["standard", "rational", "thin_prism", "tilted"]


def make_pair(model, w, h, skew=0.0, vertical=False, seed=0):
  """Two cameras of one model and size with different K and distortion, and the pose x_right = R x_left + T of the pair."""
  import cv2
  rng = np.random.default_rng(seed)
  cams = []
  for c in range(2):
    f = 0.73 * max(w, h) * (1 + 0.02 * c)
    K = np.array([[f, skew, w / 2 - 3.3 + 4 * c], [0, 1.007 * f, h / 2 + 2.1 - 3 * c], [0, 0, 1]])
    d = np.array(DIST[model]) * (1 + 0.1 * c)
    cams.append(CameraFisheye(image_size=(w, h), intrinsic=K, dist=d.reshape(4, 1)) if model == "fisheye"
                else Camera(image_size=(w, h), intrinsic=K, dist=d, model=model))
  T = np.array([0.004, -0.12, 0.003]) if vertical else np.array([-0.12, 0.005, 0.003])
  pose = np.eye(4)
  pose[:3, :3] = cv2.Rodrigues(rng.normal(0, 0.04, 3))[0]
  pose[:3, 3] = T + rng.normal(0, 0.002, 3)
  return cams, pose


def rel(a, b):
  return float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))


def cv_rectify(cams, pose, alpha, new_size, zero_disparity):
  import cv2
  l, r = cams
  return cv2.stereoRectify(l.intrinsic, l.dist, r.intrinsic, r.dist, l.image_size, pose[:3, :3], pose[:3, 3],
                           flags=cv2.CALIB_ZERO_DISPARITY if zero_disparity else 0, alpha=alpha, newImageSize=new_size or (0, 0))


def run_stereo_rectify(w, h):
  k = 0
  for model in PINHOLE:
    for vertical in (False, True):
      cams, pose = make_pair(model, w, h, skew=0.0, vertical=vertical, seed=k)
      for alpha in (-1, 0, 0.5, 1):
        for new_size, zd in (((None, True)), ((w + 40, h - 20), False), ((w * 2, h * 2), True), (None, False)):
          k += 1
          ours = stereo_rectify(*cams, pose, alpha=alpha, new_size=new_size, zero_disparity=zd)
          R1, R2, P1, P2, Q, roi1, roi2 = cv_rectify(cams, pose, alpha, new_size, zd)
          case = (model, vertical, alpha, new_size, zd)
          assert np.abs(ours.R1 - R1).max() <= 1e-12 and np.abs(ours.R2 - R2).max() <= 1e-12, case
          for a, b in ((ours.P1, P1), (ours.P2, P2), (ours.Q, Q)):
            assert rel(a, b) <= 1e-9, (case, rel(a, b))
          # alpha = 0 puts an edge of the inner rectangle on the image border, where ceil / floor of a value that is an integer up to
          # rounding decides: 1 px there, equal everywhere else
          for o, ref in ((ours.roi1, roi1), (ours.roi2, roi2)):
            d = np.abs(np.subtract(o, ref)).max()
            assert d == 0 or (alpha == 0 and d == 1), (case, ours.roi1, roi1, ours.roi2, roi2)


def run_stereo_rectify_fisheye(w, h):
  import cv2
  k = 0
  for balance in (0.0, 0.4, 1.0):
    for fov_scale in (1.0, 1.3):
      for new_size, zd in ((None, True), ((w + 40, h - 20), False)):
        k += 1
        cams, pose = make_pair("fisheye", w, h, seed=k)
        l, r = cams
        ours = stereo_rectify_fisheye(l, r, pose, zero_disparity=zd, new_size=new_size, balance=balance, fov_scale=fov_scale)
        R1, R2, P1, P2, Q = cv2.fisheye.stereoRectify(l.intrinsic, l.dist, r.intrinsic, r.dist, l.image_size, pose[:3, :3], pose[:3, 3],
                                                      cv2.CALIB_ZERO_DISPARITY if zd else 0, newImageSize=new_size or (0, 0),
                                                      balance=balance, fov_scale=fov_scale)
        case = (balance, fov_scale, new_size, zd)
        assert np.abs(ours.R1 - R1).max() <= 1e-12 and np.abs(ours.R2 - R2).max() <= 1e-12, case
        for a, b in ((ours.P1, P1), (ours.P2, P2), (ours.Q, Q)):
          assert rel(a, b) <= 1e-9, (case, rel(a, b))


def cv_rectification(cams, pose, new_size):
  """OpenCV's (R1, P1) of the left camera, so that the map checks do not lean on stereo_rectify."""
  import cv2
  l, r = cams
  if isinstance(l, CameraFisheye):
    R1, _, P1, _, _ = cv2.fisheye.stereoRectify(l.intrinsic, l.dist, r.intrinsic, r.dist, l.image_size, pose[:3, :3], pose[:3, 3],
                                                cv2.CALIB_ZERO_DISPARITY, newImageSize=new_size, balance=0.3)
    return R1, P1
  return cv_rectify(cams, pose, 0.3, new_size, True)[:3:2]


def cv_map(camera, R, P, size):
  import cv2
  K, d = camera.intrinsic, camera.dist
  if isinstance(camera, CameraFisheye):
    return np.dstack(cv2.fisheye.initUndistortRectifyMap(K, d, R, P, size, cv2.CV_32F))
  return cv2.initUndistortRectifyMap(K, d, R, P, size, cv2.CV_32FC2)[0]


def run_maps(sizes):
  for w, h in sizes:
    for model in MODELS:
      for skew in (0.0, 2.5):
        for size in ((w, h), (w + 13, h - 7)):
          cams, pose = make_pair(model, w, h, skew=skew, seed=w + h)
          R1, P1 = cv_rectification(cams, pose, size)
          m, ref = cams[0].rectify_map(R1, P1, size), cv_map(cams[0], R1, P1, size)
          assert m.shape == (size[1], size[0], 2) and m.dtype == np.float32
          bad = int((m.view(np.int32) != ref.view(np.int32)).sum())
          assert bad == 0, f"{model} {w}x{h} -> {size} skew {skew}: {bad} map values differ from OpenCV's"


def run_wide_maps():
  """k_rectify_map walks a row 512 entries (block starts, then tail pixels) at a time: a fisheye row of 9001 pixels takes 18 segments,
  a pinhole row of 4109 (513 blocks of 8 and a tail of 5) has its last block and its tail in the second segment, and one of 4087 (510
  blocks and a tail of 7) crosses into the second segment inside its tail."""
  import cv2
  rng = np.random.default_rng(9)
  for model, w in (("fisheye", 9001), ("standard", 4109), ("thin_prism", 4087)):
    h = 3
    cam = make_camera(model, w, h, skew=1.5)
    K = cam.intrinsic
    R = cv2.Rodrigues(rng.normal(0, 0.05, 3))[0]
    P = np.array([[K[0, 0] * 0.9, 0, w / 2 + 1.7, 0], [0, K[1, 1] * 0.9, h / 2 - 0.6, 0], [0, 0, 1, 0]])
    for what, m, ref in (("undistort_map", cam.undistort_map, cv_undistort_map(cam)),
                         ("rectify_map", cam.rectify_map(R, P), cv_map(cam, R, P, (w, h)))):
      assert m.shape == (h, w, 2) and m.dtype == np.float32
      bad = int((m.view(np.int32) != ref.view(np.int32)).sum())
      assert bad == 0, f"{what} {model} {w}x{h}: {bad} map values differ from OpenCV's"


def run_images(w, h):
  import cv2
  rng = np.random.default_rng(5)
  for model in ("standard", "tilted", "fisheye"):
    cams, pose = make_pair(model, w, h, seed=3)
    size = (w + 11, h - 5)
    l, r = cams
    if model == "fisheye":
      R1, R2, P1, P2, _ = cv2.fisheye.stereoRectify(l.intrinsic, l.dist, r.intrinsic, r.dist, l.image_size, pose[:3, :3], pose[:3, 3],
                                                    cv2.CALIB_ZERO_DISPARITY, newImageSize=size, balance=0.3)
    else:
      R1, R2, P1, P2 = cv_rectify(cams, pose, 0.3, size, True)[:4]
    recs = [(R1, P1), (R2, P2)]
    batch = [images(rng, 2, (h, w)), images(rng, 2, (h, w, 3))]
    out = rectify_images(batch, cams, recs, size=size)
    for k, (cam, (R, P)) in enumerate(zip(cams, recs)):
      m = cv_map(cam, R, P, size)
      for i, im in enumerate(batch[k]):
        ref = cv2.remap(im, m, None, cv2.INTER_CUBIC)
        assert out[k][i].shape == ref.shape and out[k][i].dtype == np.uint8
        assert np.array_equal(out[k][i], ref), f"{model} camera {k} image {i}: {int((out[k][i] != ref).sum())} pixels differ"


def run_points(w, h, n):
  import cv2
  rng = np.random.default_rng(7)
  for model in MODELS:
    cams, pose = make_pair(model, w, h, skew=0.8, seed=2)
    R1, P1 = cv_rectification(cams, pose, (w, h))
    K, d = cams[0].intrinsic, cams[0].dist
    pix = np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], -1)
    if model == "fisheye":
      ref = cv2.fisheye.undistortPoints(pix.reshape(-1, 1, 2), K, d, R=R1, P=P1).reshape(-1, 2)
    else:
      ref = cv2.undistortPoints(pix.reshape(-1, 1, 2), K, d, R=R1, P=P1).reshape(-1, 2)
    out = cams[0].rectify_points(pix, R1, P1)
    assert out.dtype == np.float64 and out.shape == (n, 2)
    assert np.abs(out - ref).max() <= 1e-9, (model, np.abs(out - ref).max())
    p32 = cams[0].rectify_points(pix.reshape(2, -1, 2).astype(np.float32), R1, P1)
    assert p32.dtype == np.float32 and p32.shape == (2, n // 2, 2)


def check_rectified_pair(cams, pose, depth=1.2):
  """Noise-free detections of a board grid in front of the pair, rectified: equal rows, and Q recovers the rectified left point."""
  r = stereo_rectify(*cams, pose)
  g = np.stack(np.meshgrid(np.linspace(-0.25, 0.25, 9), np.linspace(-0.15, 0.15, 7)), -1).reshape(-1, 2)
  X = np.concatenate([g, depth + 0.1 * g[:, :1]], 1)
  Xr = X @ pose[:3, :3].T + pose[:3, 3]
  ul, ur = cams[0].project(X), cams[1].project(Xr)
  ql, qr = cams[0].rectify_points(ul, r.R1, r.P1), cams[1].rectify_points(ur, r.R2, r.P2)
  assert np.abs(ql[:, 1] - qr[:, 1]).max() <= 1e-6, np.abs(ql[:, 1] - qr[:, 1]).max()
  h = np.c_[ql, ql[:, 0] - qr[:, 0], np.ones(len(ql))] @ r.Q.T
  Y = h[:, :3] / h[:, 3:]
  want = X @ r.R1.T
  assert rel(Y, want) <= 1e-9, rel(Y, want)


def run_end_to_end(F=12):
  from multical_b200 import synthetic
  scene = synthetic.make_scene(C=2, F=F, seed=21, vis=0.6, noise=0.0)
  K, d = scene["gt"]["K"], scene["gt"]["dist"]
  cams = [Camera(image_size=scene["image_size"], intrinsic=K[c], dist=d[c], model="standard") for c in range(2)]
  from test_gpu_stereo import matches_of
  _, _, pose, _ = stereo_calibrate(cams, matches_of(scene))
  check_rectified_pair(cams, pose)
  return scene, cams


def run_reproducible(w, h):
  rng = np.random.default_rng(3)
  for model in MODELS:
    cams, pose = make_pair(model, w, h, skew=0.5, seed=4)
    R1, P1 = cv_rectification(cams, pose, (w, h))
    a, b = cams[0].rectify_map(R1, P1), cams[0].rectify_map(R1, P1)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    src = [images(rng, 2, (h, w, 3))]
    x, y = rectify_images(src, cams[:1], [(R1, P1)]), rectify_images(src, cams[:1], [(R1, P1)])
    assert all(np.array_equal(p, q) for p, q in zip(x[0], y[0]))
    P = rng.uniform(0, w, (64, 2))
    assert np.array_equal(cams[0].rectify_points(P, R1, P1), cams[0].rectify_points(P, R1, P1))
    if model != "fisheye":
      s1, s2 = stereo_rectify(*cams, pose, alpha=0.5), stereo_rectify(*cams, pose, alpha=0.5)
      assert all(np.array_equal(s1[k], s2[k]) for k in ("R1", "R2", "P1", "P2", "Q"))


def run_errors(w, h):
  cams, pose = make_pair("standard", w, h)
  # mixed models, mixed sizes, fisheye through the pinhole entry and back
  fish, _ = make_pair("fisheye", w, h)
  with pytest.raises(AssertionError, match="one camera model"):
    stereo_rectify(cams[0], fish[1], pose)
  with pytest.raises(AssertionError, match="one camera model"):
    stereo_rectify(cams[0], Camera((w, h), cams[1].intrinsic, np.zeros(8), model="rational"), pose)
  with pytest.raises(AssertionError, match="one image size"):
    stereo_rectify(cams[0], cams[1].copy(image_size=(w + 2, h)), pose)
  with pytest.raises(AssertionError, match="stereo_rectify_fisheye"):
    stereo_rectify(*fish, pose)
  with pytest.raises(AssertionError, match="fisheye cameras"):
    stereo_rectify_fisheye(*cams, pose)
  flat = pose.copy(); flat[:3, 3] = 0
  with pytest.raises(ValueError, match="zero baseline"):
    stereo_rectify(*cams, flat)
  with pytest.raises(ValueError, match="zero baseline"):
    stereo_rectify_fisheye(*fish, flat)
  ok = np.zeros((h, w), np.uint8)
  R, P = np.eye(3), cams[0].intrinsic
  with pytest.raises(NotImplementedError, match="dtype uint16"):
    rectify_images([[ok.astype(np.uint16)]], cams[:1], [(R, P)])
  with pytest.raises(NotImplementedError, match="shape"):
    rectify_images([[np.zeros((h, w, 4), np.uint8)]], cams[:1], [(R, P)])
  # the C ABI: singular P R -> MCBA_ERR_ARG (1), non-finite R or P -> MCBA_ERR_NONFINITE (5), bad images -> MCBA_ERR_ARG
  eng = undistort.undistort_engine()
  model, vec = undistort.camera_vector(cams[0])
  D = C.POINTER(C.c_double)
  vp = vec.ctypes.data_as(D)
  Rf, Pf = np.eye(3).ravel().copy(), P.ravel().copy()
  sing = Pf.copy(); sing[3:6] = sing[0:3]
  nanR = Rf.copy(); nanR[4] = np.nan
  pts, out = np.zeros((1, 2)), np.zeros((1, 2))
  for r_, p_, want in ((Rf, sing, 1), (np.zeros(9), Pf, 1), (nanR, Pf, 5), (Rf, Pf, 0)):
    assert eng.lib.mcba_rectify_map(eng.h, 0, vp, r_.ctypes.data_as(D), p_.ctypes.data_as(D), w, h, None) == want, want
    assert eng.lib.mcba_rectify_points(eng.h, 0, vp, r_.ctypes.data_as(D), p_.ctypes.data_as(D), 1, pts.ctypes.data_as(D),
                                       out.ctypes.data_as(D)) == want, want
  U8 = C.POINTER(C.c_uint8)
  src, dst = ok.copy(), np.zeros_like(ok)
  sp, dp = (U8 * 1)(src.ctypes.data_as(U8)), (U8 * 1)(dst.ctypes.data_as(U8))
  for dtype, channels in [(1, 1), (0, 2), (-1, 3)]:
    assert eng.lib.mcba_rectify_images(eng.h, 0, vp, Rf.ctypes.data_as(D), Pf.ctypes.data_as(D), w, h, 1, w, h, channels, dtype, sp,
                                       dp) == 1
  assert eng.lib.mcba_rectify_images(eng.h, 0, vp, Rf.ctypes.data_as(D), Pf.ctypes.data_as(D), w, h, 1, w, h, 1, 0, sp, dp) == 0
  bad = vec.copy(); bad[5] = np.nan
  with pytest.raises(ValueError, match="non-finite"):
    eng.rectify_points(model, bad, R, P, np.zeros((1, 2)))
  with pytest.raises(AssertionError, match="singular"):
    eng.rectify_map(model, vec, np.zeros((3, 3)), P, (w, h))


def test_stereo_rectify_matches_opencv():
  run_stereo_rectify(1920, 1200)


def test_stereo_rectify_fisheye_matches_opencv():
  run_stereo_rectify_fisheye(1280, 960)


def test_maps_are_opencvs_bit_for_bit():
  run_maps([(1920, 1200), (641, 479), (97, 61)])


def test_wide_maps_are_opencvs_bit_for_bit():
  run_wide_maps()


def test_rectify_images_are_cv2_remap_bit_for_bit():
  run_images(640, 480)


def test_rectify_points_match_opencv():
  run_points(1920, 1200, 5000)


def test_calibrated_pair_rectifies_to_equal_rows():
  run_end_to_end()


def test_bundle_adjusted_rig_pair_rectifies_to_equal_rows():
  """The pose of two cameras of a rig after bundle_adjust(): camera_poses[j] @ inv(camera_poses[i])."""
  from multical_b200 import synthetic
  from multical_b200.calibration import from_scene
  scene = synthetic.make_scene(C=3, F=10, vis=0.6, seed=8, noise=0.0)
  calib = from_scene(scene).enable(cameras=True).bundle_adjust()
  poses = np.asarray(calib.camera_poses.poses)
  cams = [calib.cameras[0], calib.cameras[2]]
  check_rectified_pair(cams, poses[2] @ np.linalg.inv(poses[0]))


def test_repeated_calls_agree_bit_for_bit():
  run_reproducible(641, 479)


def test_refusals():
  run_errors(64, 48)
