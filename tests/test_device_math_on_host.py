"""CPU: the kernels' own math (csrc/geometry.cuh, solve_tr_2d of csrc/solver_kernels.cuh), compiled for the host by
tests/host_math/host_math.cu, against the libraries the reference delegates to:
  cv2.projectPoints / cv2.fisheye.projectPoints  (camera.py:124-128, camera_fisheye.py:113-117) -- values AND the Jacobian
  cv2 returns and the reference throws away; scipy Rotation (transform/rtvec.py:24-27); scipy's solve_trust_region_2d and
  loss functions (the pieces of least_squares behind calibration.py:209-210)."""
import ctypes as C
import os
import subprocess

import cv2
import numpy as np
import pytest
from scipy.optimize._lsq.common import solve_trust_region_2d
from scipy.optimize._lsq.least_squares import IMPLEMENTED_LOSSES
from scipy.spatial.transform import Rotation

from conftest import ROOT

HM = os.path.join(ROOT, "tests", "host_math")
D = C.POINTER(C.c_double)
dp = lambda a: a.ctypes.data_as(D)


@pytest.fixture(scope="module")
def hm():
  so, src = os.path.join(HM, "libhostmath.so"), os.path.join(HM, "host_math.cu")
  deps = [src] + [os.path.join(ROOT, "multical_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "multical_b200", "csrc"))]
  if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
    subprocess.run([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                    "-Xcompiler", "-fPIC", "-shared", "-diag-suppress", "550", "-I", os.path.join(ROOT, "multical_b200", "csrc"),
                    "-o", so, src], check=True)
  lib = C.CDLL(so)
  lib.hm_project.argtypes = [C.c_int, C.c_int, D, D, D, D, D]
  lib.hm_undistort.argtypes = [C.c_int, C.c_int, D, D, D]
  lib.hm_pose_from_homography.argtypes = [D, D, D]
  lib.hm_spd_solve8.argtypes = [D, D]
  lib.hm_rodrigues.argtypes = [D, D, D]
  lib.hm_twist_map.argtypes = [D, D, D, D]
  lib.hm_hand_eye_frame_map.argtypes = [D] * 7
  lib.hm_matrix_to_rtvec.argtypes = [D, D]
  lib.hm_tr2d.argtypes = [C.c_double] * 6 + [D]
  lib.hm_loss.argtypes = [C.c_int, C.c_double, D]
  lib.hm_lin_smem_doubles.argtypes = [C.c_int] * 4
  lib.hm_lin_smem_doubles.restype = C.c_size_t
  return lib


DIST = {
  0: np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01]),
  1: np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01, 0.02, -0.01, 0.005]),
  2: np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01, 0.02, -0.01, 0.005, 1e-3, -5e-4, 5e-4, 1e-3]),
  4: np.array([-0.1, 0.05, 1e-3, -1e-3, 0.01, 0.02, -0.01, 0.005, 1e-3, -5e-4, 5e-4, 1e-3, 0.02, -0.015]),
}


def points(n=300, seed=0):
  rng = np.random.default_rng(seed)
  return np.ascontiguousarray(np.column_stack([rng.normal(0, 0.35, n), rng.normal(0, 0.25, n), rng.uniform(0.7, 1.6, n)]))


def run_project(hm, model, X, kvec):
  n, nk = X.shape[0], kvec.size - 1          # kvec = [fx fy cx cy skew dist...]; Jk columns = [fx fy cx cy dist...]
  uv, J, Jk = np.zeros((n, 2)), np.zeros((2 * n, 3)), np.zeros((2 * n, nk))
  assert hm.hm_project(model, n, dp(X), dp(kvec), dp(uv), dp(J), dp(Jk)) == 0
  assert np.isfinite(uv).all(), "residual-only and Jacobian code paths disagree"
  return uv, J, Jk


@pytest.mark.parametrize("model", [0, 1, 2, 4])
def test_pinhole_projection_and_jacobian_match_cv2(hm, model):
  X = points()
  K = np.array([[1203.0, 0.0, 957.0], [0.0, 1198.0, 544.0], [0.0, 0.0, 1.0]])
  dist = DIST[model]
  kvec = np.concatenate([[K[0, 0], K[1, 1], K[0, 2], K[1, 2], 0.37], dist])        # a non-zero skew must be ignored
  uv, J, Jk = run_project(hm, model, X, kvec)
  uv_cv, jac = cv2.projectPoints(X.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, dist)
  assert np.abs(uv - uv_cv.reshape(-1, 2)).max() < 1e-10
  # cv2 Jacobian columns: rvec(3) tvec(3) f(2) c(2) dist(nd); with rvec = tvec = 0 the tvec block is d(u,v)/dX_cam
  scale = np.abs(jac).max(axis=0) + 1e-300
  assert (np.abs(J - jac[:, 3:6]) / scale[3:6]).max() < 1e-9
  assert (np.abs(Jk - jac[:, 6:6 + 4 + dist.size]) / scale[6:6 + 4 + dist.size]).max() < 1e-9


def test_fisheye_projection_and_jacobian_match_cv2(hm):
  X = points(seed=1)
  K = np.array([[903.0, 0.0, 957.0], [0.0, 899.0, 544.0], [0.0, 0.0, 1.0]])
  dist = np.array([0.02, -0.01, 3e-3, -1e-3])
  kvec = np.concatenate([[K[0, 0], K[1, 1], K[0, 2], K[1, 2], 0.0], dist])
  uv, J, Jk = run_project(hm, 3, X, kvec)
  uv_cv, jac = cv2.fisheye.projectPoints(X.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, dist)
  assert np.abs(uv - uv_cv.reshape(-1, 2)).max() < 1e-10
  # cv2.fisheye Jacobian columns: f(2) c(2) k(4) om(3) T(3) alpha(1)
  scale = np.abs(jac).max(axis=0) + 1e-300
  assert (np.abs(J - jac[:, 11:14]) / scale[11:14]).max() < 1e-9
  assert (np.abs(Jk - jac[:, 0:8]) / scale[0:8]).max() < 1e-9


def test_rodrigues_and_left_jacobian(hm):
  rng = np.random.default_rng(2)
  for r in list(rng.normal(0, 0.8, (20, 3))) + [np.zeros(3), np.array([1e-5, -2e-5, 1e-5]), np.array([3.0, 0.3, -0.2])]:
    r = np.ascontiguousarray(r, dtype=np.float64)
    R, JL = np.zeros(9), np.zeros(9)
    hm.hm_rodrigues(dp(r), dp(R), dp(JL))
    R, JL = R.reshape(3, 3), JL.reshape(3, 3)
    assert np.abs(R - Rotation.from_rotvec(r).as_matrix()).max() < 1e-14
    # R(r + d) = exp([JL d]x) R(r) to first order
    for d in np.eye(3) * 1e-6:
      lhs = Rotation.from_rotvec(r + d).as_matrix()
      rhs = Rotation.from_rotvec(JL @ d).as_matrix() @ R
      assert np.abs(lhs - rhs).max() < 1e-11


def test_matrix_to_rtvec_matches_scipy(hm):
  """Device-side restatement of transform/rtvec.py:29-32 (Rotation.from_matrix(...).as_rotvec()), incl. angles near 0 and pi."""
  rng = np.random.default_rng(5)
  rvs = list(rng.normal(0, 1.2, (200, 3))) + [np.zeros(3), np.array([1e-9, 0, 0]), np.array([2e-4, -1e-4, 3e-4]),
                                                 np.array([np.pi - 1e-7, 0, 0]), np.array([0, np.pi, 0]), np.array([2.2, -2.2, 0.1])]
  for r in rvs:
    T = np.eye(4); T[:3, :3] = Rotation.from_rotvec(r).as_matrix(); T[:3, 3] = rng.normal(0, 1, 3)
    rt = np.zeros(6)
    hm.hm_matrix_to_rtvec(dp(np.ascontiguousarray(T)), dp(rt))
    ref = Rotation.from_matrix(T[:3, :3]).as_rotvec()
    if np.linalg.norm(ref) > np.pi - 1e-6:          # at pi the axis sign is arbitrary: compare the rotations
      assert np.abs(Rotation.from_rotvec(rt[:3]).as_matrix() - T[:3, :3]).max() < 1e-9
    else:
      assert np.abs(rt[:3] - ref).max() < 1e-14
    assert np.array_equal(rt[3:], T[:3, 3])


def test_twist_map_is_the_derivative_of_the_pose_chain(hm):
  """x_cam = T_c T_f T_b X; the map of the FRAME pose must turn (dr, dt) of the frame rtvec into the camera-frame twist."""
  rng = np.random.default_rng(3)
  rc, rf = rng.normal(0, 0.5, 3), rng.normal(0, 0.5, 3)
  tc, tf = rng.normal(0, 0.3, 3), rng.normal(0, 0.3, 3)
  Xw = rng.normal(0, 0.3, 3)
  Rc = Rotation.from_rotvec(rc).as_matrix()
  def xcam(rf_, tf_): return Rc @ (Rotation.from_rotvec(rf_).as_matrix() @ Xw + tf_) + tc
  Rf, JLf = np.zeros(9), np.zeros(9)
  hm.hm_rodrigues(dp(np.ascontiguousarray(rf)), dp(Rf), dp(JLf))
  tcf = Rc @ tf + tc
  A = np.zeros(36)
  hm.hm_twist_map(dp(np.ascontiguousarray(Rc.ravel())), dp(JLf), dp(np.ascontiguousarray(tcf)), dp(A))
  A = A.reshape(6, 6)
  x0 = xcam(rf, tf)
  for j in range(6):
    d = np.zeros(6); d[j] = 1e-6
    num = (xcam(rf + d[:3], tf + d[3:]) - xcam(rf - d[:3], tf - d[3:])) / 2e-6
    xi = A[:, j]                                      # (omega, v)
    assert np.abs(np.cross(xi[:3], x0) + xi[3:] - num).max() < 1e-8



def test_hand_eye_frame_map_factors_the_hand_eye_twist_maps(hm):
  """Hand-eye frame T_f = G A_f W.  The maps of W (left part T_c G A_f, chain translation t_cf) and of G (left part T_c, chain translation
  R_c t_G + t_c) are the frame's own map, taken with JL = I, times M_f (csrc/kernels.cuh hand_eye_frame_map): what lets k_fold_hand_eye
  build the hand-eye blocks from the per-frame ones."""
  rng = np.random.default_rng(5)
  c = lambda a: np.ascontiguousarray(a, dtype=np.float64)
  def tmap(Rl, JL, t):
    A = np.zeros(36); hm.hm_twist_map(dp(c(Rl.ravel())), dp(c(JL.ravel())), dp(c(t)), dp(A)); return A.reshape(6, 6)
  for trial in range(20):
    Rc, RG, RA, RW = (Rotation.from_rotvec(rng.normal(0, 1.0, 3)).as_matrix() for _ in range(4))
    tc, tG, tA, tW = (rng.normal(0, 0.5, 3) for _ in range(4))
    JLW, JLG = np.zeros(9), np.zeros(9)
    hm.hm_rodrigues(dp(c(rng.normal(0, 1.0, 3))), dp(np.zeros(9)), dp(JLW))
    hm.hm_rodrigues(dp(c(rng.normal(0, 1.0, 3))), dp(np.zeros(9)), dp(JLG))
    JLW, JLG = JLW.reshape(3, 3), JLG.reshape(3, 3)
    RGA, tGA = RG @ RA, RG @ tA + tG
    tf = RGA @ tW + tGA
    tcf = Rc @ tf + tc
    M = np.zeros(72)
    hm.hm_hand_eye_frame_map(dp(c(RG.ravel())), dp(c(RA.ravel())), dp(c(JLW.ravel())), dp(c(JLG.ravel())), dp(c(tG)), dp(c(tf)), dp(M))
    Eh = np.hstack([tmap(Rc @ RGA, JLW, tcf), tmap(Rc, JLG, Rc @ tG + tc)])
    assert np.abs(tmap(Rc, np.eye(3), tcf) @ M.reshape(6, 12) - Eh).max() < 1e-14 * max(1.0, np.abs(Eh).max())


def test_trust_region_2d_matches_scipy(hm):
  rng = np.random.default_rng(4)
  for trial in range(300):
    M = rng.normal(0, 1, (2, 2))
    B = M @ M.T * 10 ** rng.uniform(-3, 3)
    if trial % 5 == 0: B = B - np.eye(2) * np.abs(np.linalg.eigvalsh(B)).max() * 0.6      # indefinite model
    if trial % 7 == 0: B[0, 1] = B[1, 0] = 0.0
    g = rng.normal(0, 1, 2) * 10 ** rng.uniform(-2, 2)
    Delta = 10 ** rng.uniform(-3, 2)
    p = np.zeros(2)
    hm.hm_tr2d(B[0, 0], B[0, 1], B[1, 1], g[0], g[1], Delta, dp(p))
    ps, _ = solve_trust_region_2d(B, g, Delta)
    q = lambda v: 0.5 * v @ B @ v + g @ v
    assert np.linalg.norm(p) <= Delta * (1 + 1e-9)
    assert q(p) <= q(ps) + 1e-9 * (abs(q(ps)) + 1e-300), (trial, p, ps)     # at least as good a minimiser as scipy's


@pytest.mark.parametrize("loss,index", [("soft_l1", 1), ("huber", 2), ("cauchy", 3), ("arctan", 4)])
def test_losses_match_scipy(hm, loss, index):
  z = np.concatenate([np.linspace(0, 3, 31), [10.0, 1e3]])
  rho = np.empty((3, z.size))
  IMPLEMENTED_LOSSES[loss](z, rho, cost_only=False)
  for i, zi in enumerate(z):
    r = np.zeros(3)
    hm.hm_loss(index, float(zi), dp(r))
    assert np.allclose(r, rho[:, i], rtol=1e-13, atol=1e-15)


# ---- batched pose initialisation (csrc/pnp_kernels.cuh): the pieces whose reference arithmetic is OpenCV's
@pytest.mark.parametrize("model", [0, 1, 2, 4, 3])
def test_undistort_pixel_is_cv2_undistort_points(hm, model):
  """camera.py:119-122 cv2.undistortPoints(pts, K, dist, P=K) (5 fixed-point iterations) and camera_fisheye.py:108-111
  cv2.fisheye.undistortPoints (Newton on theta); the distorted pixels come from cv2's own projection of points in front of the camera."""
  K = np.array([[1200.0, 0, 960], [0, 1190.0, 540], [0, 0, 1]])
  X = points(400, seed=model)
  if model == 3:
    dist = np.array([0.02, -0.01, 3e-3, -1e-3])
    uv = cv2.fisheye.projectPoints(X.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, dist)[0].reshape(-1, 2)
    want = cv2.fisheye.undistortPoints(uv.reshape(-1, 1, 2), K, dist.reshape(4, 1), P=K).reshape(-1, 2)
  else:
    dist = DIST[model]
    uv = cv2.projectPoints(X.reshape(-1, 1, 3), np.zeros(3), np.zeros(3), K, dist)[0].reshape(-1, 2)
    want = cv2.undistortPoints(uv.reshape(-1, 1, 2), K, dist, P=K).reshape(-1, 2)
  kvec = np.concatenate([[K[0, 0], K[1, 1], K[0, 2], K[1, 2], 0.0], dist])
  got = np.zeros_like(uv)
  uv = np.ascontiguousarray(uv)
  assert hm.hm_undistort(model, uv.shape[0], dp(uv), dp(kvec), dp(got)) == 0
  assert np.abs(got - want).max() < 1e-9                                     # same iteration count, same formula: round-off only


def test_pose_from_homography_recovers_a_plane_pose(hm):
  rng = np.random.default_rng(3)
  for _ in range(50):
    R = Rotation.from_rotvec(rng.normal(0, 0.6, 3)).as_matrix()
    t = np.array([rng.normal(0, 0.2), rng.normal(0, 0.2), rng.uniform(0.5, 2.0)])
    H = np.column_stack([R[:, 0], R[:, 1], t]) * rng.uniform(0.2, 5.0)      # any positive scale
    Rg, tg = np.zeros((3, 3)), np.zeros(3)
    Hc = np.ascontiguousarray(H)
    hm.hm_pose_from_homography(dp(Hc), dp(Rg), dp(tg))
    assert np.abs(Rg - R).max() < 1e-12 and np.abs(tg - t).max() < 1e-12


def test_spd_solve_matches_numpy(hm):
  rng = np.random.default_rng(4)
  for _ in range(20):
    M = rng.normal(size=(12, 8)); A = M.T @ M; b = rng.normal(size=8)
    Ac, bc = np.ascontiguousarray(A.copy()), b.copy()
    assert hm.hm_spd_solve8(dp(Ac), dp(bc)) == 1
    assert np.abs(bc - np.linalg.solve(A, b)).max() < 1e-9 * np.abs(b).max() * np.linalg.cond(A)
  Z = np.zeros((8, 8)); zb = np.ones(8)
  assert hm.hm_spd_solve8(dp(Z), dp(zb)) == 0                                 # not positive definite -> reported, never NaN-propagated silently
