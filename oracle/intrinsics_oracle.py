"""numpy restatement of the initialisation of single-camera intrinsic calibration (csrc/intrinsics_kernels.cuh):

  homography(board_xy, pixels)          the homography from the board plane to pixels (float32-rounded inputs) that minimises the pixel
                                        reprojection error, as cv2.findHomography refines it: the device's normalised DLT (h33 = 1), then
                                        scipy's Levenberg-Marquardt to convergence
  init_intrinsics(Hs, image_size, ...)  OpenCV's initIntrinsicParams2D (calibration.cpp; what cv2.initCameraMatrix2D exposes), fed the
                                        homographies above instead of OpenCV's LM-refined ones
"""
import numpy as np
from scipy.optimize import least_squares


def homography(board_xy, pixels):
  X = np.asarray(board_xy, np.float32).astype(np.float64)[:, :2]
  x = np.asarray(pixels, np.float32).astype(np.float64)
  def normalise(p):
    m = p.mean(axis=0)
    d = np.sqrt(((p - m) ** 2).sum(axis=1)).mean()
    s = np.sqrt(2.0) / d if d > 0 else 1.0
    return (p - m) * s, m, s
  Xn, mX, sB = normalise(X)
  xn, mx, sP = normalise(x)
  n = X.shape[0]
  A = np.zeros((2 * n, 8)); b = np.zeros(2 * n)
  A[0::2, 0:2] = Xn; A[0::2, 2] = 1; A[0::2, 6:8] = -xn[:, :1] * Xn
  A[1::2, 3:5] = Xn; A[1::2, 5] = 1; A[1::2, 6:8] = -xn[:, 1:] * Xn
  b[0::2] = xn[:, 0]; b[1::2] = xn[:, 1]
  h = np.linalg.solve(A.T @ A, A.T @ b)
  def resid(g):
    w = g[6] * Xn[:, 0] + g[7] * Xn[:, 1] + 1.0
    return np.concatenate([(g[0] * Xn[:, 0] + g[1] * Xn[:, 1] + g[2]) / w - xn[:, 0], (g[3] * Xn[:, 0] + g[4] * Xn[:, 1] + g[5]) / w - xn[:, 1]])
  h = least_squares(resid, h, method="lm", ftol=1e-15, xtol=1e-15, gtol=1e-15).x
  Hn = np.append(h, 1.0).reshape(3, 3)
  Tb = np.array([[sB, 0, -sB * mX[0]], [0, sB, -sB * mX[1]], [0, 0, 1]])
  Tp_inv = np.array([[1 / sP, 0, mx[0]], [0, 1 / sP, mx[1]], [0, 0, 1]])
  H = Tp_inv @ Hn @ Tb
  return H / H[2, 2]


def init_intrinsics(Hs, image_size, aspect_ratio=0.0):
  """3x3 camera matrix from per-view homographies (board plane -> pixels).  aspect_ratio 0: fx, fy free; otherwise fx = aspect_ratio * tf,
  fy = tf with tf = (fx + fy) / (aspect_ratio + 1)."""
  w, h = image_size
  cx, cy = (w - 1) * 0.5, (h - 1) * 0.5
  A, b = [], []
  for H in Hs:
    H = np.array(H, np.float64)
    H[0] -= H[2] * cx
    H[1] -= H[2] * cy
    hv, vv = H[:, 0], H[:, 1]
    d1, d2 = (hv + vv) * 0.5, (hv - vv) * 0.5
    hv, vv, d1, d2 = (u / np.linalg.norm(u) for u in (hv, vv, d1, d2))
    A += [[hv[0] * vv[0], hv[1] * vv[1]], [d1[0] * d2[0], d1[1] * d2[1]]]
    b += [-hv[2] * vv[2], -d1[2] * d2[2]]
  A, b = np.array(A), np.array(b)
  f = np.linalg.solve(A.T @ A, A.T @ b)
  fx, fy = np.sqrt(np.abs(1.0 / f))
  if aspect_ratio:
    tf = (fx + fy) / (aspect_ratio + 1.0)
    fx, fy = aspect_ratio * tf, tf
  return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
