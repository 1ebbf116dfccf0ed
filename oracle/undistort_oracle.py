"""numpy restatement of what the reference does with OpenCV to apply a finished calibration (camera.py:113-128, 244-258;
camera_fisheye.py:102-117): the undistortion map with R = I and newK = K (cv2.initUndistortRectifyMap,
cv2.fisheye.initUndistortRectifyMap) and cv2.remap(image, map, None, INTER_CUBIC) with the default constant-zero border, for
uint8 images.

This is the arithmetic the device kernels in multical_b200/csrc/undistort_kernels.cuh follow; the tests compare both this and the
device against live cv2.
"""
import numpy as np

TAB = 32                  # INTER_TAB_SIZE: 1/32-pixel sub-positions
COEF_BITS = 15            # INTER_REMAP_COEF_BITS
COEF_SCALE = 1 << COEF_BITS


def cubic_coeffs(x):
  """The four 1-D cubic weights at sub-position x (float32 arithmetic, A = -0.75)."""
  f = np.float32
  A, x = f(-0.75), f(x)
  one = f(1)
  c0 = ((A * (x + one) - f(5) * A) * (x + one) + f(8) * A) * (x + one) - f(4) * A
  c1 = ((A + f(2)) * x - (A + f(3))) * x * x + one
  y = one - x
  c2 = ((A + f(2)) * y - (A + f(3))) * y * y + one
  c3 = one - c0 - c1 - c2
  return np.array([c0, c1, c2, c3], np.float32)


def cubic_table():
  """int32 [32*32][16]: entry (Y&31)*32 + (X&31) holds the 4x4 fixed-point weights (row-major, rows = y taps)."""
  one_d = [cubic_coeffs(np.float32(k) * np.float32(1.0 / TAB)) for k in range(TAB)]
  tab = np.zeros((TAB * TAB, 16), np.int32)
  for i in range(TAB):
    for j in range(TAB):
      w = np.outer(one_d[i], one_d[j]).astype(np.float32)            # float32 products
      t = np.rint(w * np.float32(COEF_SCALE)).astype(np.int32).reshape(4, 4)
      diff = int(t.sum()) - COEF_SCALE
      if diff:
        mk = Mk = (2, 2)
        for k1 in (2, 3):
          for k2 in (2, 3):
            if t[k1, k2] < t[mk]: mk = (k1, k2)
            elif t[k1, k2] > t[Mk]: Mk = (k1, k2)
        if diff < 0: t[Mk] -= diff
        else: t[mk] -= diff
      tab[i * TAB + j] = t.reshape(16)
  return tab


def fixed_point_map(m):
  """float32 [h][w][2] map -> (sx, sy, table index) as remap reads it: X = rint(32 x), taps from (X >> 5) - 1."""
  m = np.asarray(m, np.float32)

  def cv_round(v):                      # ties to even; NaN and values outside int32 give INT_MIN, as OpenCV's x86 conversion does
    ok = (v >= -2.0 ** 31) & (v < 2.0 ** 31)
    return np.where(ok, np.rint(np.where(ok, v, 0)), -2.0 ** 31).astype(np.int64)

  with np.errstate(invalid="ignore", over="ignore"):
    X = cv_round(m[..., 0] * np.float32(TAB))
    Y = cv_round(m[..., 1] * np.float32(TAB))
  sx = np.clip(X >> 5, -32768, 32767) - 1
  sy = np.clip(Y >> 5, -32768, 32767) - 1
  return sx, sy, (Y & 31) * TAB + (X & 31)


def remap_cubic(src, m):
  """cv2.remap(src, m, None, INTER_CUBIC) for uint8 src [h][w] or [h][w][3] and a float32 map [H][W][2]."""
  src = np.asarray(src)
  gray = src.ndim == 2
  s = src[..., None] if gray else src
  h, w, cn = s.shape
  sx, sy, idx = fixed_point_map(m)
  tab = cubic_table()[idx]                                            # [H][W][16]
  acc = np.zeros(sx.shape + (cn,), np.int64)
  for ky in range(4):
    yy = sy + ky
    for kx in range(4):
      xx = sx + kx
      inside = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
      v = s[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
      acc += np.where(inside[..., None], v, 0) * tab[..., 4 * ky + kx, None]
  out = np.clip((acc + (1 << (COEF_BITS - 1))) >> COEF_BITS, 0, 255).astype(np.uint8)
  return out[..., 0] if gray else out


def _tilt(tx, ty):
  cx, sx, cy, sy = np.cos(tx), np.sin(tx), np.cos(ty), np.sin(ty)
  Rx = np.array([[1, 0, 0], [0, cx, sx], [0, -sx, cx]])
  Ry = np.array([[cy, 0, -sy], [0, 1, 0], [sy, 0, cy]])
  R = Ry @ Rx
  Pz = np.array([[R[2, 2], 0, -R[0, 2]], [0, R[2, 2], -R[1, 2]], [0, 0, 1]])
  return Pz @ R


def undistort_map(K, dist, size, fisheye=False):
  """float32 [h][w][2] map of initUndistortRectifyMap(K, dist, None, K, size) (or the fisheye variant), in fp64.  The normalised
  coordinates come from K^-1 (skew included); the forward projection uses fx, fy, cx, cy only, as OpenCV's does."""
  w, h = size
  K = np.asarray(K, np.float64)
  fx, fy, cx, cy, s = K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[0, 1]
  v, u = np.mgrid[0:h, 0:w].astype(np.float64)
  y = (v - cy) / fy
  x = (u - cx - s * y) / fx
  d = np.zeros(14)
  dd = np.asarray(dist, np.float64).reshape(-1)
  d[:dd.size] = dd
  if fisheye:
    r = np.sqrt(x * x + y * y)
    th = np.arctan(r)
    t2 = th * th
    t4 = t2 * t2
    thd = th * (1 + d[0] * t2 + d[1] * t4 + d[2] * (t4 * t2) + d[3] * (t4 * t4))
    with np.errstate(invalid="ignore", divide="ignore"):
      scale = np.where(r == 0, 1.0, thd / r)
    mu, mv = fx * x * scale + cx, fy * y * scale + cy
  else:
    k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4, tx, ty = d
    x2, y2 = x * x, y * y
    r2 = x2 + y2
    _2xy = 2 * x * y
    kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2)
    xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2) + s1 * r2 + s2 * r2 * r2
    yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy + s3 * r2 + s4 * r2 * r2
    M = _tilt(tx, ty)
    t0 = M[0, 0] * xd + M[0, 1] * yd + M[0, 2]
    t1 = M[1, 0] * xd + M[1, 1] * yd + M[1, 2]
    t2 = M[2, 0] * xd + M[2, 1] * yd + M[2, 2]
    ip = np.where(t2 != 0, 1.0 / np.where(t2 != 0, t2, 1.0), 1.0)
    mu, mv = fx * ip * t0 + cx, fy * ip * t1 + cy
  return np.stack([mu, mv], -1).astype(np.float32)
