"""numpy restatement of OpenCV's rectification map, cv2.initUndistortRectifyMap(K, dist, R, P, size) and
cv2.fisheye.initUndistortRectifyMap(K, D, R, P, size): the row walk whose rounding reaches the float32 map, then the distortion.  At
R = I, P = K it is the undistortion map.  This is the arithmetic k_rectify_map (multical_b200/csrc/undistort_kernels.cuh) follows.

Row i starts at (x, y, w) = i * ir[:, 1] + ir[:, 2], ir = (P[:, :3] R)^-1, and steps by ir[:, 0]:
  pinhole  blocks of 8 pixels (OpenCV's SIMD loop, 2 vectors of 4 doubles): pixel k of a block is cur + k * step, then cur += 8 * step;
           the last W mod 8 pixels take cur, then cur += step.  x = _x * (1 / _w).
  fisheye  one pixel at a time, cur += step; x = _x / _w, and _w <= 0 gives an infinite entry.
"""
import numpy as np

from .undistort_oracle import _tilt

BLOCK = 8


def walk(ir, w, h, block):
  """(x, y, w) [h][w] of the row walk with blocks of `block` pixels (1: pixel by pixel)."""
  ir = np.asarray(ir, np.float64).reshape(9)
  out = np.zeros((3, h, w))
  i = np.arange(h, dtype=np.float64)
  nb = w // block
  for r in range(3):
    step = ir[3 * r]
    cur = i * ir[3 * r + 1] + ir[3 * r + 2]
    for b in range(nb):
      for k in range(block):
        out[r, :, b * block + k] = cur + k * step
      cur = cur + block * step
    for j in range(nb * block, w):
      out[r, :, j] = cur
      cur = cur + step
  return out


def inverse(M):
  """3x3 Gauss-Jordan elimination with partial pivoting, as the host driver computes (P R)^-1."""
  A, I = np.array(M, np.float64).reshape(3, 3).copy(), np.eye(3)
  for c in range(3):
    p = c + int(np.argmax(np.abs(A[c:, c])))
    A[[c, p]], I[[c, p]] = A[[p, c]], I[[p, c]]
    for r in range(3):
      if r != c:
        f = A[r, c] / A[c, c]
        A[r], I[r] = A[r] - f * A[c], I[r] - f * I[c]
  return I / np.diag(A)[:, None]


def rectify_map(K, dist, R, P, size, fisheye=False):
  """float32 [h][w][2] map of initUndistortRectifyMap(K, dist, R, P, size) (fisheye: its two CV_32F maps stacked)."""
  w, h = size
  K = np.asarray(K, np.float64)
  fx, fy, cx, cy = K[0, 0], K[1, 1], K[0, 2], K[1, 2]
  P3 = np.asarray(P, np.float64).reshape(3, -1)[:, :3]
  R = np.asarray(R, np.float64).reshape(3, 3)
  PR = np.array([[P3[i, 0] * R[0, j] + P3[i, 1] * R[1, j] + P3[i, 2] * R[2, j] for j in range(3)] for i in range(3)])
  X, Y, W = walk(inverse(PR), w, h, 1 if fisheye else BLOCK)
  d = np.zeros(14)
  dd = np.asarray(dist, np.float64).reshape(-1)
  d[:dd.size] = dd
  with np.errstate(divide="ignore", invalid="ignore"):
    if fisheye:
      x, y = X / W, Y / W
      r = np.sqrt(x * x + y * y)
      th = np.arctan(r)
      t2 = th * th
      t4 = t2 * t2
      thd = th * (1 + d[0] * t2 + d[1] * t4 + d[2] * (t4 * t2) + d[3] * (t4 * t4))
      scale = np.where(r == 0, 1.0, thd / r)
      mu, mv = fx * x * scale + cx, fy * y * scale + cy
      mu = np.where(W <= 0, np.where(X > 0, -np.inf, np.inf), mu)
      mv = np.where(W <= 0, np.where(Y > 0, -np.inf, np.inf), mv)
    else:
      iw = 1.0 / W
      x, y = X * iw, Y * iw
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
