"""GPU (-m gpu): applying a finished calibration (multical_b200/undistort.py; include/mcba.h mcba_rectify_* at R = I, P = K,
mcba_project_points; csrc/undistort_kernels.cuh) against OpenCV, called live.

Bars:
  maps             bit-identical to cv2.initUndistortRectifyMap(K, dist, None, K, size, CV_32FC2) for the standard, rational, thin
                   prism and tilted models, and to cv2.fisheye.initUndistortRectifyMap(..., CV_32F) stacked to [h, w, 2] (OpenCV 4.13
                   refuses CV_32FC2 there) for the fisheye, with and without skew, at odd sizes
  remap            bit-identical to cv2.remap(image, OpenCV's map, None, INTER_CUBIC): 1 and 3 channels, maps that leave the image,
                   source images larger and smaller than the map
  undistort_images bit-identical to the reference's per-image cv2.remap(image, camera.undistort_map, None, INTER_CUBIC) over a batch of
                   cameras of different sizes wherever the maps are bit-identical, and to cv2.remap on the device's own map everywhere
  points           project / undistort_points within 1e-9 px of cv2.projectPoints, cv2.undistortPoints(P=K) and the cv2.fisheye twins
  repeated calls   bit for bit
"""
import ctypes as C

import numpy as np
import pytest

from multical_b200 import undistort
from multical_b200.camera import Camera, CameraFisheye, undistort_images

pytestmark = pytest.mark.gpu

MODELS = ["standard", "rational", "thin_prism", "tilted", "fisheye"]
DIST = dict(standard=[-0.21, 0.09, 0.0012, -0.0008, -0.02],
            rational=[-0.21, 0.09, 0.0012, -0.0008, -0.02, 0.03, 0.01, -0.005],
            thin_prism=[-0.21, 0.09, 0.0012, -0.0008, -0.02, 0.03, 0.01, -0.005, 0.001, -0.0005, 0.0007, 0.0002],
            tilted=[-0.21, 0.09, 0.0012, -0.0008, -0.02, 0.03, 0.01, -0.005, 0.001, -0.0005, 0.0007, 0.0002, 0.01, -0.008],
            fisheye=[0.05, -0.01, 0.003, -0.0007])


def make_camera(model, w, h, skew=0.0, scale=1.0, strong=False):
  f = 0.73 * max(w, h) * scale
  K = np.array([[f, skew, w / 2 - 3.3 * scale], [0, 1.007 * f, h / 2 + 2.1 * scale], [0, 0, 1]])
  d = np.array(DIST[model], np.float64)
  if strong: d[0] = 1.5 if model == "fisheye" else 0.45             # pincushion: the map leaves the image towards the corners
  if model == "fisheye": return CameraFisheye(image_size=(w, h), intrinsic=K, dist=d.reshape(4, 1))
  return Camera(image_size=(w, h), intrinsic=K, dist=d, model=model)


def cv_map(camera):
  """The reference's Camera.undistort_map (camera.py:113-117, camera_fisheye.py:102-106)."""
  import cv2
  K, d, size = camera.intrinsic, camera.dist, camera.image_size
  if isinstance(camera, CameraFisheye):
    return np.dstack(cv2.fisheye.initUndistortRectifyMap(K, d, None, K, size, cv2.CV_32F))
  return cv2.initUndistortRectifyMap(K, d, None, K, size, cv2.CV_32FC2)[0]


def cv_remap(image, m):
  import cv2
  return cv2.remap(image, m, None, cv2.INTER_CUBIC)


def images(rng, n, shape):
  """Seeded synthetic images: smooth structure plus noise, so that the cubic weights matter and values clip at both ends."""
  h, w = shape[:2]
  yy, xx = np.mgrid[0:h, 0:w]
  out = []
  for _ in range(n):
    base = 128 + 140 * np.sin(xx / rng.uniform(3, 9) + rng.uniform(0, 6)) * np.cos(yy / rng.uniform(3, 9))
    if len(shape) == 3: base = base[..., None] + rng.uniform(-40, 40, shape[2])
    out.append(np.clip(base + rng.normal(0, 25, shape), 0, 255).astype(np.uint8))
  return out


def run_maps(sizes):
  for w, h in sizes:
    for model in MODELS:
      for skew in (0.0, 2.5):
        cam = make_camera(model, w, h, skew)
        m, ref = cam.undistort_map, cv_map(cam)
        assert m.shape == (h, w, 2) and m.dtype == np.float32
        bad = int((m.view(np.int32) != ref.view(np.int32)).sum())
        assert bad == 0, f"{model} {w}x{h} skew {skew}: {bad} map values differ from OpenCV's"


def run_remap(w, h):
  rng = np.random.default_rng(5)
  for model in ("standard", "fisheye"):
    cam = make_camera(model, w, h, strong=True)
    ref_map = cv_map(cam)
    assert (ref_map[..., 0] < -1).any() or (ref_map[..., 0] > w).any(), "the map should leave the image"
    for shape in [(h, w), (h, w, 3), (h + 7, w + 13), (h - 9, w - 5, 3), (h // 2 + 1, w // 3 + 2)]:
      src = images(rng, 2, shape)
      out = undistort_images([src], [cam])[0]
      for i, (a, b) in enumerate(zip(out, (cv_remap(s, ref_map) for s in src))):
        assert a.shape == b.shape and a.dtype == np.uint8, (a.shape, b.shape)
        bad = int((a != b).sum())
        assert bad == 0, f"{model} source {shape} image {i}: {bad} pixels differ from cv2.remap"


def run_undistort_images(sizes, n_per_camera):
  rng = np.random.default_rng(11)
  cams = [make_camera(MODELS[k % len(MODELS)], w, h, skew=1.5 * (k % 2)) for k, (w, h) in enumerate(sizes)]
  batch = [images(rng, n_per_camera, (h, w) if k % 3 else (h, w, 3)) for k, (w, h) in enumerate(sizes)]
  batch.append([])                                                   # a camera without images
  cams.append(make_camera("standard", 40, 30))
  out = undistort_images(batch, cams, j=3, chunksize=2)
  assert len(out) == len(batch) and [len(o) for o in out] == [len(b) for b in batch]
  for k, (cam, ims, outs) in enumerate(zip(cams, batch, out)):
    m, ours = cv_map(cam), cam.undistort_map
    same = (m == ours).all(axis=-1)                                  # pixels whose map entries are bit-identical
    for i, (im, o) in enumerate(zip(ims, outs)):
      ref = cv_remap(im, m)
      assert o.shape == ref.shape and o.dtype == ref.dtype
      assert np.array_equal(o[same], ref[same]), f"camera {k} image {i}: {int((o != ref)[same].sum())} pixels differ"
      assert np.array_equal(o, cv_remap(im, ours)), f"camera {k} image {i}: differs from cv2.remap on the device's own map"
  return out


def run_points(w, h, n):
  import cv2
  rng = np.random.default_rng(7)
  for model in MODELS:
    cam = make_camera(model, w, h, skew=0.8)
    K, d = cam.intrinsic, cam.dist
    X = np.stack([rng.uniform(-0.6, 0.6, n), rng.uniform(-0.4, 0.4, n), rng.uniform(0.8, 3.0, n)], -1)
    fish = isinstance(cam, CameraFisheye)
    proj = cv2.fisheye.projectPoints if fish else cv2.projectPoints
    ref = proj(X.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, d)[0].reshape(-1, 2)
    uv = cam.project(X)
    assert uv.dtype == np.float64 and uv.shape == (n, 2)
    assert np.abs(uv - ref).max() <= 1e-9, (model, np.abs(uv - ref).max())
    # any leading shape; float32 in -> float32 out as OpenCV
    p = cam.project(X.reshape(2, -1, 3).astype(np.float32))
    assert p.shape == (2, n // 2, 2) and p.dtype == np.float32
    pix = np.stack([rng.uniform(0, w, n), rng.uniform(0, h, n)], -1)
    und = cv2.fisheye.undistortPoints if fish else cv2.undistortPoints
    ref = und(pix.reshape(-1, 1, 2), K, d, P=K).reshape(-1, 2)
    out = cam.undistort_points(pix)
    assert out.dtype == np.float64 and out.shape == (n, 2)
    assert np.abs(out - ref).max() <= 1e-9, (model, np.abs(out - ref).max())
    p32 = pix.reshape(n // 2, 2, 2).astype(np.float32)
    o32, r32 = cam.undistort_points(p32), und(p32.reshape(-1, 1, 2), K, d, P=K).reshape(n // 2, 2, 2)
    assert o32.dtype == np.float32 and o32.shape == (n // 2, 2, 2)
    assert (np.abs(o32 - r32) <= np.spacing(np.abs(r32))).all(), model          # one float32 ulp: both round the same fp64 value


def run_reproducible(w, h):
  rng = np.random.default_rng(3)
  for model in MODELS:
    cam = make_camera(model, w, h, skew=0.5)
    a, b = undistort.undistort_map(cam), undistort.undistort_map(cam)
    assert np.array_equal(a.view(np.int32), b.view(np.int32))
    src = images(rng, 3, (h, w, 3))
    x, y = undistort_images([src], [cam])[0], undistort_images([src], [cam])[0]
    assert all(np.array_equal(p, q) for p, q in zip(x, y))
    X = rng.uniform(0.5, 2.0, (64, 3))
    assert np.array_equal(cam.project(X), cam.project(X))
    P = rng.uniform(0, w, (64, 2))
    assert np.array_equal(cam.undistort_points(P), cam.undistort_points(P))


def run_errors(w, h):
  cam = make_camera("standard", w, h)
  ok = np.zeros((h, w), np.uint8)
  with pytest.raises(NotImplementedError, match="dtype uint16"):
    undistort_images([[ok.astype(np.uint16)]], [cam])
  with pytest.raises(NotImplementedError, match="dtype float32"):
    undistort_images([[ok.astype(np.float32)]], [cam])
  with pytest.raises(NotImplementedError, match="shape"):
    undistort_images([[np.zeros((h, w, 4), np.uint8)]], [cam])
  with pytest.raises(NotImplementedError, match="shape"):
    undistort_images([[np.zeros((h, w, 2), np.uint8)]], [cam])
  with pytest.raises(AssertionError, match="share one shape"):
    undistort_images([[ok, np.zeros((h + 1, w), np.uint8)]], [cam])
  # the C ABI: unsupported dtype or channel count -> MCBA_ERR_ARG (1)
  eng = undistort.undistort_engine()
  model, vec = undistort.camera_vector(cam)
  R, P = (np.ascontiguousarray(a).ravel() for a in undistort.identity_rectification(vec))
  U8, D = C.POINTER(C.c_uint8), C.POINTER(C.c_double)
  src, dst = ok.copy(), np.zeros_like(ok)
  sp, dp = (U8 * 1)(src.ctypes.data_as(U8)), (U8 * 1)(dst.ctypes.data_as(U8))
  vp, rp, pp = vec.ctypes.data_as(D), R.ctypes.data_as(D), P.ctypes.data_as(D)
  for dtype, channels in [(1, 1), (0, 2), (0, 4), (-1, 3)]:
    rc = eng.lib.mcba_rectify_images(eng.h, 0, vp, rp, pp, w, h, 1, w, h, channels, dtype, sp, dp)
    assert rc == 1, (dtype, channels, rc)
  assert eng.lib.mcba_rectify_images(eng.h, 0, vp, rp, pp, w, h, 1, w, h, 1, 0, sp, dp) == 0
  bad = vec.copy(); bad[5] = np.nan
  with pytest.raises(ValueError, match="non-finite"):
    eng.rectify_points(model, bad, *undistort.identity_rectification(bad), np.zeros((1, 2)))


def test_maps_are_opencvs_bit_for_bit():
  run_maps([(1920, 1200), (641, 479), (97, 61)])


def test_remap_is_cv2_remap_bit_for_bit():
  run_remap(320, 240)


def test_undistort_images_match_reference_per_image_remap():
  run_undistort_images([(1920, 1200), (1280, 1024), (641, 479), (640, 480), (333, 217)], 4)


def test_project_and_undistort_points_match_opencv():
  run_points(1920, 1200, 5000)


def test_repeated_calls_agree_bit_for_bit():
  run_reproducible(641, 479)


def test_unsupported_images_raise():
  run_errors(64, 48)


def test_bundle_adjustment_problem_survives():
  """The undistortion runs on its own engine: a problem uploaded to the bundle adjustment engine is untouched."""
  from multical_b200 import synthetic
  from multical_b200.calibration import from_scene
  scene = synthetic.make_scene(C=2, F=6, vis=0.5, seed=3)
  calib = from_scene(scene).enable(cameras=True)
  eng = calib._upload(calib.inliers)
  before = eng.residuals()
  run_undistort_images([(160, 120), (97, 61)], 2)
  assert undistort.undistort_engine() is not eng
  assert np.array_equal(before, eng.residuals())
