"""Camera intrinsics as optimisable parameters, mirroring the reference's `Camera`
(multical/camera.py:27-181: model names 43-48, params 144-155, with_params 157-171) and
`CameraFisheye` (multical/camera_fisheye.py:28-170).  Projection itself runs on the GPU
(csrc/geometry.cuh); these classes only carry values across the API."""
from functools import cached_property

import numpy as np

from .parameters import Parameters
from .structs import struct

MODELS = ("standard", "rational", "thin_prism", "tilted")
DIST_SIZE = dict(standard=5, rational=8, thin_prism=12, tilted=14, fisheye=4)


class Camera(Parameters):
  engine_model = None      # resolved from .model

  def __init__(self, image_size, intrinsic, dist, model="standard", fix_aspect=False, has_skew=False, error_perview=None,
               intrinsic_dataset={}, **_):
    assert model in MODELS, f"unknown camera model {model} options are {list(MODELS)}"
    self.model = model
    self.image_size = tuple(image_size)
    self.intrinsic = np.asarray(intrinsic, np.float64)
    self.dist = np.zeros(5) if dist is None else np.asarray(dist, np.float64)
    self.fix_aspect = fix_aspect
    self.has_skew = has_skew
    self.error_perview = error_perview              # per-view RMS of the last intrinsic calibration (camera.py:40-41)
    self.intrinsic_dataset = intrinsic_dataset      # {'board_ids', 'image_ids'} of the views it kept

  @staticmethod
  def calibrate(boards, intrinsic_error_limit, detections, image_size, max_iter=10, eps=1e-3, model="standard", fix_aspect=False,
                has_skew=False, flags=0, max_images=None, **solve_opts):
    """camera.py:68-105 on the GPU (multical_b200/intrinsics.py): (Camera, err)."""
    from .intrinsics import calibrate
    return calibrate(boards, intrinsic_error_limit, detections, image_size, max_iter=max_iter, eps=eps, model=model, fix_aspect=fix_aspect,
                     has_skew=has_skew, flags=flags, max_images=max_images, **solve_opts)

  def __repr__(self): return f"Camera(intrinsic={self.intrinsic!r}, dist={self.dist!r}, image_size={self.image_size})"

  @property
  def focal_length(self): return np.array([self.intrinsic[0, 0], self.intrinsic[1, 1]])
  @property
  def principle_point(self): return np.array([self.intrinsic[0, 2], self.intrinsic[1, 2]])
  @property
  def skew(self): return self.intrinsic[0, 1] if self.has_skew else 0.0

  @cached_property
  def params(self):
    f = self.focal_length
    if self.fix_aspect: f = np.array([f.mean(), f.mean()])
    return struct(focal_length=f, principle_point=self.principle_point, skew=np.array([self.skew]), dist=self.dist)

  def with_params(self, params):
    f = params["focal_length"]
    fx, fy = (f[0], f[0]) if self.fix_aspect else (f[0], f[1])
    px, py = params["principle_point"]
    skew, = params["skew"]
    K = np.array([[fx, skew, px], [0, fy, py], [0, 0, 1]], np.float64)
    return self.copy(intrinsic=K, dist=params["dist"])

  @cached_property
  def undistort_map(self):
    """camera.py:113-117 on the GPU (multical_b200/undistort.py): float32 [h, w, 2] of cv2.initUndistortRectifyMap with R = I, newK = K."""
    from .undistort import undistort_map
    return undistort_map(self)

  def undistort_points(self, points):
    """camera.py:119-122 on the GPU: cv2.undistortPoints(points, K, dist, P=K) over any leading shape [..., 2]."""
    from .undistort import undistort_points
    return undistort_points(self, points)

  def project(self, points):
    """camera.py:124-128 on the GPU: cv2.projectPoints of camera-frame points [..., 3] with rvec = tvec = 0 -> pixels [..., 2]."""
    from .undistort import project
    return project(self, points)

  def rectify_map(self, R, P, size=None):
    """float32 [h, w, 2] of cv2.initUndistortRectifyMap(K, dist, R, P, size) on the GPU (multical_b200/rectify.py); size defaults to
    image_size."""
    from .rectify import rectify_map
    return rectify_map(self, R, P, size)

  def rectify_points(self, points, R, P):
    """cv2.undistortPoints(points, K, dist, R=R, P=P) on the GPU over any leading shape [..., 2]."""
    from .rectify import rectify_points
    return rectify_points(self, points, R, P)

  def approx_eq(self, other):
    return self.image_size == other.image_size and np.allclose(other.intrinsic, self.intrinsic) and np.allclose(other.dist, self.dist)

  def scale_image(self, factor):
    K = self.intrinsic.copy(); K[:2] *= factor
    return self.copy(intrinsic=K)

  def __getstate__(self):
    return dict(image_size=self.image_size, intrinsic=self.intrinsic, dist=self.dist, fix_aspect=self.fix_aspect,
                has_skew=self.has_skew, model=self.model)
  def __setstate__(self, d): self.__dict__.update(d)
  def copy(self, **k):
    d = self.__getstate__(); d.update(k)
    return self.__class__(**d)


class CameraFisheye(Camera):
  def __init__(self, image_size, intrinsic, dist, model="standard", fix_aspect=False, has_skew=False, **_):
    self.model = model
    self.image_size = tuple(image_size)
    self.intrinsic = np.asarray(intrinsic, np.float64)
    self.dist = np.zeros((4, 1)) if dist is None else np.asarray(dist, np.float64)
    self.fix_aspect = fix_aspect
    self.has_skew = has_skew

  @staticmethod
  def calibrate(boards, detections, image_size, max_iter=10, eps=1e-3, model="standard", fix_aspect=False, has_skew=False, flags=0,
                max_images=None, **solve_opts):
    """camera_fisheye.py:70-94 on the GPU (multical_b200/intrinsics.py): (CameraFisheye, err)."""
    from .intrinsics import calibrate_fisheye
    return calibrate_fisheye(boards, detections, image_size, max_iter=max_iter, eps=eps, model=model, fix_aspect=fix_aspect,
                             has_skew=has_skew, flags=flags, max_images=max_images, **solve_opts)


def calibrate_cameras(boards, points, image_sizes, intrinsic_error_limit, **kwargs):
  """camera.py:237-241 on the GPU (multical_b200/intrinsics.py): (cameras, errs)."""
  from .intrinsics import calibrate_cameras
  return calibrate_cameras(boards, points, image_sizes, intrinsic_error_limit, **kwargs)


def calibrate_cameras_fisheye(boards, points, image_sizes, **kwargs):
  """camera_fisheye.py:173-177 on the GPU (multical_b200/intrinsics.py): (cameras, errs)."""
  from .intrinsics import calibrate_cameras_fisheye
  return calibrate_cameras_fisheye(boards, points, image_sizes, **kwargs)


def stereo_calibrate(cameras, matches, max_iter=60, eps=1e-6, fix_aspect=False, fix_intrinsic=True, **solve_opts):
  """camera.py:261-286 on the GPU (multical_b200/stereo.py): (left, right, 4x4 pose of the pair, err)."""
  from .stereo import stereo_calibrate
  return stereo_calibrate(cameras, matches, max_iter=max_iter, eps=eps, fix_aspect=fix_aspect, fix_intrinsic=fix_intrinsic, **solve_opts)


def stereo_calibrate_fisheye(cameras, matches, max_iter=60, eps=1e-6, fix_aspect=False, fix_intrinsic=True, **solve_opts):
  """camera_fisheye.py:180-205 on the GPU (multical_b200/stereo.py): (left, right, 4x4 pose of the pair, err)."""
  from .stereo import stereo_calibrate_fisheye
  return stereo_calibrate_fisheye(cameras, matches, max_iter=max_iter, eps=eps, fix_aspect=fix_aspect, fix_intrinsic=fix_intrinsic,
                                  **solve_opts)


def undistort_images(images, cameras, j=None, chunksize=4):
  """camera.py:247-258 on the GPU (multical_b200/undistort.py): per camera, its images remapped through its undistortion map."""
  from .undistort import undistort_images
  return undistort_images(images, cameras, j=j, chunksize=chunksize)


def stereo_rectify(left, right, pose, alpha=-1, new_size=None, zero_disparity=True):
  """cv2.stereoRectify of a calibrated pinhole pair on the GPU (multical_b200/rectify.py): struct(R1, R2, P1, P2, Q, roi1, roi2)."""
  from .rectify import stereo_rectify
  return stereo_rectify(left, right, pose, alpha=alpha, new_size=new_size, zero_disparity=zero_disparity)


def stereo_rectify_fisheye(left, right, pose, zero_disparity=True, new_size=None, balance=0.0, fov_scale=1.0):
  """cv2.fisheye.stereoRectify of a calibrated fisheye pair on the GPU (multical_b200/rectify.py): struct(R1, R2, P1, P2, Q)."""
  from .rectify import stereo_rectify_fisheye
  return stereo_rectify_fisheye(left, right, pose, zero_disparity=zero_disparity, new_size=new_size, balance=balance, fov_scale=fov_scale)


def rectify_images(images, cameras, rectifications, size=None):
  """Per camera, its images remapped through its rectification map under rectifications[k] = (R, P) (multical_b200/rectify.py)."""
  from .rectify import rectify_images
  return rectify_images(images, cameras, rectifications, size=size)


def engine_model_of(camera):
  """Which CUDA camera model a (reference or mirror) camera object needs."""
  if type(camera).__name__ == "CameraFisheye": return "fisheye"
  model = getattr(camera, "model", "standard")
  nd = np.size(camera.dist)
  expect = DIST_SIZE[model]
  assert nd == expect, f"camera model {model} expects {expect} distortion coefficients, got {nd}"
  return model
