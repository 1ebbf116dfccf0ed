"""Applying a finished calibration on the GPU: the reference's Camera.undistort_map, undistort_points and project (camera.py:113-128,
camera_fisheye.py:102-117) and undistort_images (camera.py:244-258), which run OpenCV on the host there.

The kernels are in csrc/undistort_kernels.cuh.  Maps are OpenCV's to the bit (R = I, newK = K), except rare 1-ulp fisheye values
(DESIGN.md §3g); the remap is cv2.remap's fixed-point
bicubic with the constant-zero border for uint8 images of 1 or 3 channels.  Everything runs on an engine of its own, so the bundle
adjustment engine's uploaded problem survives it."""
import numpy as np

from .camera import engine_model_of

_engines = {}


def undistort_engine(device=None):
  """An engine used only to apply calibrations (one per GPU): camera maps stay resident on it between calls."""
  from .calibration import default_device
  from .engine import Engine
  device = default_device() if device is None else device
  if device not in _engines:
    _engines[device] = Engine(device)
  return _engines[device]


def camera_vector(camera):
  """(engine model, [fx fy cx cy skew dist...]) of a (reference or mirror) camera.  K[0, 1] is passed as it is: OpenCV reads it in
  K^-1 whatever `has_skew` says."""
  model = engine_model_of(camera)
  K = np.asarray(camera.intrinsic, np.float64)
  return model, np.concatenate([[K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[0, 1]], np.asarray(camera.dist, np.float64).reshape(-1)])


def undistort_map(camera):
  """float32 [h, w, 2]: cv2.initUndistortRectifyMap(K, dist, None, K, image_size, CV_32FC2), or the fisheye variant."""
  model, cam = camera_vector(camera)
  return undistort_engine().undistort_map(model, cam, camera.image_size)


def _out_dtype(points):
  return np.float32 if np.asarray(points).dtype == np.float32 else np.float64


def undistort_points(camera, points):
  """cv2.undistortPoints(points, K, dist, P=K) (cv2.fisheye.undistortPoints) over any leading shape [..., 2]; float32 in gives float32
  out, anything else float64, as OpenCV does."""
  points = np.asarray(points)
  model, cam = camera_vector(camera)
  out = undistort_engine().undistort_points(model, cam, points.reshape(-1, 2))
  return out.astype(_out_dtype(points)).reshape(*points.shape[:-1], 2)


def project(camera, points):
  """cv2.projectPoints(points, 0, 0, K, dist) (cv2.fisheye.projectPoints) of camera-frame points [..., 3] -> pixels [..., 2]; float64
  unless the points are float32, which gives float32 as OpenCV does."""
  points = np.asarray(points)
  model, cam = camera_vector(camera)
  out = undistort_engine().project_points(model, cam, points.reshape(-1, 3))
  return out.astype(_out_dtype(points)).reshape(*points.shape[:-1], 2)


def _check_images(images, k):
  for i, im in enumerate(images):
    im = np.asarray(im)
    if im.dtype != np.uint8:
      raise NotImplementedError(f"camera {k}, image {i}: dtype {im.dtype} is not supported; the GPU remap takes uint8 images")
    if not (im.ndim == 2 or (im.ndim == 3 and im.shape[2] in (1, 3))):
      raise NotImplementedError(f"camera {k}, image {i}: shape {im.shape} is not supported; the GPU remap takes [h, w] or [h, w, 1|3]")


def undistort_images(images, cameras, j=None, chunksize=4):
  """camera.py:247-258 on the GPU: images[k] (a list of same-shape uint8 images of camera k) remapped through camera k's undistortion
  map with bicubic interpolation, returned as nested lists shaped like `images`.  `j` and `chunksize` (the reference's thread pool)
  are accepted and unused."""
  eng = undistort_engine()
  out = []
  for k, (camera, cam_images) in enumerate(zip(cameras, images)):
    cam_images = list(cam_images)
    _check_images(cam_images, k)
    shapes = {np.shape(im) for im in cam_images}
    assert len(shapes) <= 1, f"camera {k}: images of one camera must share one shape, got {sorted(shapes)}"
    model, cam = camera_vector(camera)
    out.append(eng.undistort_images(model, cam, camera.image_size, cam_images))
  return out
