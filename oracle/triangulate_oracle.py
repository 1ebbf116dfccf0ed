"""numpy + scipy restatement of triangulation (multical_b200/triangulate.py; test infrastructure only).

  dlt / triangulate_linear   the linear solution by np.linalg.svd per point: the right singular vector of the smallest singular value of
                             the rows x P3 - P1, y P3 - P2 (what cv2.triangulatePoints computes for two views)
  triangulate                N views through the full camera model: the DLT of the undistorted normalised views (cv2.undistortPoints /
                             cv2.fisheye.undistortPoints), refined by scipy.optimize.least_squares(method="lm") at tight tolerances
                             with a central-difference Jacobian, over the oracle's distorted projection (ba_oracle.project_pinhole / project_fisheye)
"""
import numpy as np
from scipy.optimize import least_squares

from .ba_oracle import project_fisheye, project_pinhole


def dlt(Ps, xs):
  """Unit homogeneous 4-vector of views (P 3x4, (x, y))."""
  A = np.concatenate([[x * P[2] - P[0], y * P[2] - P[1]] for P, (x, y) in zip(Ps, xs)])
  return np.linalg.svd(A)[2][-1]


def triangulate_linear(P1, P2, x1, x2):
  """cv2.triangulatePoints: [4, N] of unit columns."""
  return np.stack([dlt([P1, P2], [x1[:, i], x2[:, i]]) for i in range(x1.shape[1])], axis=1).reshape(4, -1)


def project(model, K, dist, Xc):
  return project_fisheye(Xc, K, dist) if model == "fisheye" else project_pinhole(Xc, K, dist)


def normalised(model, K, dist, pixels):
  import cv2
  pts = np.ascontiguousarray(pixels, np.float64).reshape(-1, 1, 2)          # cv2 misreads some strided views
  if model == "fisheye": return cv2.fisheye.undistortPoints(pts, K, np.asarray(dist, np.float64).reshape(4, 1)).reshape(-1, 2)
  return cv2.undistortPoints(pts, K, np.asarray(dist, np.float64).reshape(-1)).reshape(-1, 2)


def cost(model, Ks, dists, poses, pixels, valid, X):
  """sum |e|^2 / 2 of each point [N, 3] over its valid views (scipy's cost)."""
  out = np.zeros(len(X))
  for c in range(len(Ks)):
    e = project(model, Ks[c], dists[c], X @ poses[c, :3, :3].T + poses[c, :3, 3]) - pixels[c]
    out += np.where(valid[c], 0.5 * (e * e).sum(1), 0.0)
  return out


def central_jacobian(f, x):
  """Central differences: MINPACK's forward differences leave a gradient of 1e-4 px^2/m at two-view minima, whose depth is flat to
  working precision within 1e-9 relative."""
  h = 1e-6 * max(np.abs(x).max(), 1.0)
  return np.stack([(f(x + h * e) - f(x - h * e)) / (2 * h) for e in np.eye(3)], axis=1)


def triangulate(model, Ks, dists, poses, pixels, valid):
  """Ks [C,3,3], dists [C,nd], poses [C,4,4] rig -> camera, pixels [C,N,2], valid [C,N] -> (points [N,3], rms [N], cost [N]) with
  cost = sum |e|^2 / 2 (scipy's); NaN where a point has fewer than 2 views."""
  C, N = valid.shape
  norm = np.stack([normalised(model, Ks[c], dists[c], pixels[c]) for c in range(C)])
  X, rms, cost = np.full((N, 3), np.nan), np.full(N, np.nan), np.full(N, np.nan)
  for i in range(N):
    cams = np.flatnonzero(valid[:, i])
    if cams.size < 2: continue
    h = dlt([poses[c, :3] for c in cams], [norm[c, i] for c in cams])

    def residuals(x):
      return np.concatenate([project(model, Ks[c], dists[c], poses[c, :3, :3] @ x + poses[c, :3, 3]) - pixels[c, i] for c in cams])
    r = least_squares(residuals, h[:3] / h[3], jac=lambda x: central_jacobian(residuals, x), method="lm", xtol=1e-15, ftol=1e-15,
                      gtol=1e-15, max_nfev=10000)
    X[i], cost[i], rms[i] = r.x, r.cost, np.sqrt(2 * r.cost / cams.size)
  return X, rms, cost
