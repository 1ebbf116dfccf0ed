"""Rectifying a calibrated stereo pair on the GPU: `stereo_rectify` (cv2.stereoRectify), `stereo_rectify_fisheye`
(cv2.fisheye.stereoRectify), and the maps, points and images of a rectified camera (cv2.initUndistortRectifyMap, cv2.undistortPoints and
cv2.remap with R and P).

`pose` is the 4x4 of a pair as `stereo_calibrate` returns it, x_right = R x_left + T (for two cameras i, j of a bundle-adjusted rig:
camera_poses[j] @ inv(camera_poses[i])).  The 3x3 algebra of the rectification runs in fp64 numpy, once per pair; its point steps (the
image corners, OpenCV's 9 x 9 border grid, the fisheye edge points) go through the device's k_rectify_points.  The per-pixel work is
csrc/undistort_kernels.cuh: k_rectify_map, OpenCV's row walk to the bit (DESIGN.md §3i), and the same bicubic remap as undistortion.
Everything runs on the undistortion engine, so the bundle adjustment engine's uploaded problem survives it."""
import numpy as np

from .camera import engine_model_of
from .structs import struct
from .undistort import _check_images, _out_dtype, camera_vector, undistort_engine


def rodrigues_vector(R):
  """cv2.Rodrigues of a rotation matrix: the rotation vector of the nearest rotation (SVD), as OpenCV computes it."""
  U, _, Vt = np.linalg.svd(np.asarray(R, np.float64))
  R = U @ Vt
  r = np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
  s = np.sqrt((r @ r) * 0.25)
  c = min(max((R[0, 0] + R[1, 1] + R[2, 2] - 1) * 0.5, -1.0), 1.0)
  theta = np.arccos(c)
  if s >= 1e-5:
    return r * (1 / (2 * s) * theta)
  if c > 0:
    return np.zeros(3)
  t = np.sqrt(np.maximum((np.diag(R) + 1) * 0.5, 0))
  r = np.array([t[0], t[1] * (-1 if R[0, 1] < 0 else 1), t[2] * (-1 if R[0, 2] < 0 else 1)])
  if abs(r[0]) < abs(r[1]) and abs(r[0]) < abs(r[2]) and (R[1, 2] > 0) != (r[1] * r[2] > 0):
    r[2] = -r[2]
  return r * (theta / np.linalg.norm(r))


def rodrigues_matrix(r):
  """cv2.Rodrigues of a rotation vector."""
  r = np.asarray(r, np.float64).reshape(3)
  theta = np.linalg.norm(r)
  if theta < np.finfo(np.float64).eps:
    return np.eye(3)
  c, s = np.cos(theta), np.sin(theta)
  r = r * (1 / theta)
  rx = np.array([[0, -r[2], r[1]], [r[2], 0, -r[0]], [-r[1], r[0], 0]])
  return c * np.eye(3) + (1 - c) * np.outer(r, r) + s * rx


def _pair(left, right, fisheye):
  model = engine_model_of(left)
  assert model == engine_model_of(right), f"a rectified pair needs one camera model, got {model} and {engine_model_of(right)}"
  assert tuple(left.image_size) == tuple(right.image_size), \
    f"a rectified pair needs one image size, got {tuple(left.image_size)} and {tuple(right.image_size)}"
  if fisheye:
    assert model == "fisheye", f"stereo_rectify_fisheye takes fisheye cameras, got {model}"
  else:
    assert model != "fisheye", "fisheye cameras are rectified by stereo_rectify_fisheye"
  return model


def _pose(pose):
  pose = np.asarray(pose, np.float64)
  R, T = pose[:3, :3], pose[:3, 3]
  if not np.linalg.norm(T) > 0:
    raise ValueError("zero baseline: the pair's translation T is 0, so there is no direction to rectify along")
  return R, T


def _points(camera, points, R, P):
  model, cam = camera_vector(camera)
  return undistort_engine().rectify_points(model, cam, R, P, np.asarray(points, np.float64).reshape(-1, 2))


def _rectangles(camera, R, P, size):
  """OpenCV's icvGetRectangles: the inner and outer rectangles (x, y, w, h) of a 9 x 9 grid from pixel 0 to pixel size - 1, rectified
  by (R, P), all in fp64 (OpenCV 4.13; pinned against cv2.stereoRectify, whose ROIs and alpha scaling differ with a float32 grid or one
  that ends at size)."""
  w, h = size
  g = np.arange(9, dtype=np.float64)
  xs, ys = g * (w - 1) / 8, g * (h - 1) / 8
  grid = np.stack(np.broadcast_arrays(xs[None, :], ys[:, None]), -1).reshape(-1, 2)
  p = _points(camera, grid, R, P).reshape(9, 9, 2)
  o = (p[..., 0].min(), p[..., 1].min(), p[..., 0].max(), p[..., 1].max())
  i = (p[:, 0, 0].max(), p[0, :, 1].max(), p[:, 8, 0].min(), p[8, :, 1].min())
  return (i[0], i[1], i[2] - i[0], i[3] - i[1]), (o[0], o[1], o[2] - o[0], o[3] - o[1])


def _roi(inner, c0, c, s, size):
  """cv::Rect(ceil((x - c0) s + c), ..., floor(w s), floor(h s)) & the image."""
  x, y = int(np.ceil((float(inner[0]) - c0[0]) * s + c[0])), int(np.ceil((float(inner[1]) - c0[1]) * s + c[1]))
  w, h = int(np.floor(float(inner[2]) * s)), int(np.floor(float(inner[3]) * s))
  x1, y1 = max(x, 0), max(y, 0)
  w, h = min(x + w, size[0]) - x1, min(y + h, size[1]) - y1
  return (0, 0, 0, 0) if w <= 0 or h <= 0 else (x1, y1, w, h)


def stereo_rectify(left, right, pose, alpha=-1, new_size=None, zero_disparity=True):
  """cv2.stereoRectify(K1, d1, K2, d2, image_size, R, T, flags, alpha, new_size) of a pinhole pair (standard, rational, thin prism or
  tilted) with pose x_right = R x_left + T: struct(R1, R2, P1 [3, 4], P2 [3, 4], Q [4, 4], roi1, roi2) with the ROIs as (x, y, w, h).
  flags is CALIB_ZERO_DISPARITY when `zero_disparity`, else 0.  Vertical pairs (|T_y| > |T_x|) are rectified along y, as OpenCV does."""
  _pair(left, right, False)
  R, T = _pose(pose)
  nx, ny = left.image_size
  size = tuple(int(v) for v in (new_size if new_size is not None and np.prod(new_size) != 0 else left.image_size))
  r_r = rodrigues_matrix(rodrigues_vector(R) * -0.5)             # half of the rotation for each camera
  t = r_r @ T
  idx = 0 if abs(t[0]) > abs(t[1]) else 1
  c, nt = t[idx], np.linalg.norm(t)
  uu = np.zeros(3)
  uu[idx] = 1 if c > 0 else -1
  ww = np.cross(t, uu)                                             # the rotation that takes the baseline onto axis idx
  nw = np.linalg.norm(ww)
  if nw > 0:
    ww = ww * (np.arccos(abs(c) / nt) / nw)
  wR = rodrigues_matrix(ww)
  R1, R2 = wR @ r_r.T, wR @ r_r
  t = R2 @ T
  ratio = (size[0] / nx / 2) if idx == 1 else (size[1] / ny / 2)
  fc = (left.intrinsic[idx ^ 1, idx ^ 1] + right.intrinsic[idx ^ 1, idx ^ 1]) * ratio
  cc = []
  for cam, Rk in ((left, R1), (right, R2)):
    corners = np.array([[0, 0], [nx - 1, 0], [0, ny - 1], [nx - 1, ny - 1]], np.float32)
    xy = _points(cam, corners, np.eye(3), np.eye(3)).astype(np.float32).astype(np.float64)
    X = np.concatenate([xy, np.ones((4, 1))], 1) @ Rk.T
    z = 1 / X[:, 2]
    uv = (np.stack([X[:, 0] * z, X[:, 1] * z], 1) * fc).astype(np.float32).astype(np.float64)
    avg = uv.sum(0) / 4
    cc.append(np.array([(nx - 1) / 2 - avg[0], (ny - 1) / 2 - avg[1]]))
  if zero_disparity:
    cc[0] = cc[1] = (cc[0] + cc[1]) * 0.5
  else:
    k = 1 if idx == 0 else 0
    cc[0], cc[1] = cc[0].copy(), cc[1].copy()
    cc[0][k] = cc[1][k] = (cc[0][k] + cc[1][k]) * 0.5
  P1, P2 = np.zeros((3, 4)), np.zeros((3, 4))
  for P, cck in ((P1, cc[0]), (P2, cc[1])):
    P[0, 0] = P[1, 1] = fc
    P[0, 2], P[1, 2], P[2, 2] = cck[0], cck[1], 1
  P2[idx, 3] = t[idx] * fc
  alpha = min(alpha, 1.0)
  inner1, outer1 = _rectangles(left, R1, P1[:, :3], (nx, ny))
  inner2, outer2 = _rectangles(right, R2, P2[:, :3], (nx, ny))
  c0 = [cc[0], cc[1]]
  cn = [np.array([size[0] * ck[0] / nx, size[1] * ck[1] / ny]) for ck in c0]
  s = 1.0
  if alpha >= 0:
    def bounds(rect, ck0, ck):
      return (ck[0] / (ck0[0] - rect[0]), ck[1] / (ck0[1] - rect[1]),
              (size[0] - 1 - ck[0]) / (rect[0] + rect[2] - ck0[0]), (size[1] - 1 - ck[1]) / (rect[1] + rect[3] - ck0[1]))
    s0 = max(max(bounds(inner1, c0[0], cn[0])), max(bounds(inner2, c0[1], cn[1])))
    s1 = min(min(bounds(outer1, c0[0], cn[0])), min(bounds(outer2, c0[1], cn[1])))
    s = s0 * (1 - alpha) + s1 * alpha
  fc *= s
  for P, ck in ((P1, cn[0]), (P2, cn[1])):
    P[0, 0] = P[1, 1] = fc
    P[0, 2], P[1, 2] = ck
  P2[idx, 3] *= s
  roi1, roi2 = _roi(inner1, c0[0], cn[0], s, size), _roi(inner2, c0[1], cn[1], s, size)
  Q = np.array([[1, 0, 0, -cn[0][0]], [0, 1, 0, -cn[0][1]], [0, 0, 0, fc],
                [0, 0, -1 / t[idx], (cn[0][idx] - cn[1][idx]) / t[idx]]])
  return struct(R1=R1, R2=R2, P1=P1, P2=P2, Q=Q, roi1=roi1, roi2=roi2)


def _new_camera_fisheye(camera, R, balance, new_size, fov_scale):
  """cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(K, D, image_size, R, balance, new_size, fov_scale): 3x3."""
  w, h = camera.image_size
  K = np.asarray(camera.intrinsic, np.float64)
  balance = min(max(balance, 0.0), 1.0)
  pts = np.array([[w // 2, 0], [w, h // 2], [w // 2, h], [0, h // 2]], np.float64)
  p = _points(camera, pts, R, np.eye(3))
  cn = p.sum(0) / 4
  aspect = K[0, 0] / K[1, 1]
  cn[1] *= aspect
  p[:, 1] *= aspect
  minx, maxx, miny, maxy = p[:, 0].min(), p[:, 0].max(), p[:, 1].min(), p[:, 1].max()
  fs = (w * 0.5 / (cn[0] - minx), w * 0.5 / (maxx - cn[0]), h * 0.5 * aspect / (cn[1] - miny), h * 0.5 * aspect / (maxy - cn[1]))
  f = balance * min(fs) + (1.0 - balance) * max(fs)
  f *= 1.0 / fov_scale if fov_scale > 0 else 1.0
  new_f = np.array([f, f])
  new_c = -cn * f + np.array([w, h * aspect]) * 0.5
  new_f[1] /= aspect
  new_c[1] /= aspect
  if new_size is not None and np.prod(new_size) != 0:
    rx, ry = new_size[0] / w, new_size[1] / h
    new_f *= [rx, ry]
    new_c *= [rx, ry]
  return np.array([[new_f[0], 0, new_c[0]], [0, new_f[1], new_c[1]], [0, 0, 1]])


def stereo_rectify_fisheye(left, right, pose, zero_disparity=True, new_size=None, balance=0.0, fov_scale=1.0):
  """cv2.fisheye.stereoRectify(K1, D1, K2, D2, image_size, R, T, flags, new_size, balance, fov_scale) of a fisheye pair with pose
  x_right = R x_left + T: struct(R1, R2, P1 [3, 4], P2 [3, 4], Q [4, 4]).  OpenCV rectifies fisheye pairs along x only."""
  _pair(left, right, True)
  R, T = _pose(pose)
  r_r = rodrigues_matrix(rodrigues_vector(R) * -0.5)
  t = r_r @ T
  uu = np.array([1.0 if t[0] > 0 else -1.0, 0, 0])
  ww = np.cross(t, uu)
  nw = np.linalg.norm(ww)
  if nw > 0:
    ww = ww * (np.arccos(abs(t[0]) / np.linalg.norm(t)) / nw)
  wr = rodrigues_matrix(ww)
  R1, R2 = wr @ r_r.T, wr @ r_r
  tnew = R2 @ T
  K1 = _new_camera_fisheye(left, R1, balance, new_size, fov_scale)
  K2 = _new_camera_fisheye(right, R2, balance, new_size, fov_scale)
  fc = min(K1[1, 1], K2[1, 1])
  cc = [K1[:2, 2].copy(), K2[:2, 2].copy()]
  if zero_disparity:
    cc[0] = cc[1] = (cc[0] + cc[1]) * 0.5
  else:
    cc[0][1] = cc[1][1] = (cc[0][1] + cc[1][1]) * 0.5
  P1 = np.array([[fc, 0, cc[0][0], 0], [0, fc, cc[0][1], 0], [0, 0, 1, 0]])
  P2 = np.array([[fc, 0, cc[1][0], tnew[0] * fc], [0, fc, cc[1][1], 0], [0, 0, 1, 0]])
  Q = np.array([[1, 0, 0, -cc[0][0]], [0, 1, 0, -cc[0][1]], [0, 0, 0, fc], [0, 0, -1 / tnew[0], (cc[0][0] - cc[1][0]) / tnew[0]]])
  return struct(R1=R1, R2=R2, P1=P1, P2=P2, Q=Q)


def rectify_map(camera, R, P, size=None):
  """float32 [h, w, 2]: cv2.initUndistortRectifyMap(K, dist, R, P, size, CV_32FC2), or the fisheye variant's two CV_32F maps stacked.
  `size` = (w, h) of the rectified image, the camera's image size by default."""
  model, cam = camera_vector(camera)
  return undistort_engine().rectify_map(model, cam, R, P, camera.image_size if size is None else size)


def rectify_points(camera, points, R, P):
  """cv2.undistortPoints(points, K, dist, R=R, P=P) (cv2.fisheye.undistortPoints) over any leading shape [..., 2]; float32 in gives
  float32 out, anything else float64, as OpenCV does."""
  points = np.asarray(points)
  out = _points(camera, points, R, P)
  return out.astype(_out_dtype(points)).reshape(*points.shape[:-1], 2)


def rectify_images(images, cameras, rectifications, size=None):
  """images[k] (a list of same-shape uint8 images of camera k) remapped with bicubic interpolation through camera k's rectification map
  under rectifications[k] = (R, P), returned as nested lists shaped like `images`.  `size` = (w, h) of the rectified images, each
  camera's image size by default."""
  eng = undistort_engine()
  out = []
  for k, (camera, (R, P), cam_images) in enumerate(zip(cameras, rectifications, images)):
    cam_images = list(cam_images)
    _check_images(cam_images, k)
    shapes = {np.shape(im) for im in cam_images}
    assert len(shapes) <= 1, f"camera {k}: images of one camera must share one shape, got {sorted(shapes)}"
    model, cam = camera_vector(camera)
    out.append(eng.rectify_images(model, cam, R, P, camera.image_size if size is None else size, cam_images))
  return out
