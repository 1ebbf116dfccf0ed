"""GPU (-m gpu): triangulation (multical_b200/triangulate.py; include/mcba.h mcba_triangulate*; csrc/triangulate_kernels.cuh) against
live cv2.triangulatePoints and the numpy + scipy oracle (oracle/triangulate_oracle.py).

Bars:
  triangulate_points   against cv2.triangulatePoints (float64): dehomogenised points within 1e-9 relative, columns of unit norm within
                       1e-15, |cos| >= 1 - 1e-15 (the sign is OpenCV's SVD's choice); horizontal, vertical, narrow and wide baselines.
                       float32 in gives float32 out, dehomogenised within 3e-7 relative (a few float32 ulps; measured 0) of cv2's float32 result
  noise-free           synthetic.make_scene(C=4, noise=0) at ground truth, all five models: frame_pose @ board_pose @ X within 1e-9 of
                       the point's depth, rms <= 1e-9 px
  oracle parity        sigma = 0.3 px, all five models, C in {2, 3, 7, 33, 64}: points within 1e-9 relative of the oracle's LM minimum
                       (or, for a few two- and three-view points, apart by a step that changes the linearised cost by < 1e-12 of it),
                       rms within 1e-10 relative beyond 1e-13 px of rounding, the device's cost not above the oracle's (both evaluated by the oracle) by more
                       than 1e-9 relative: a residual of 0.01 px left over from pixels of 1000 px carries 1e-13 px of rounding
  validity             0 or 1 views, a point behind a camera, a non-finite pixel: invalid with NaN outputs; refusals
  Calibration          noise-free at ground truth reproduces the model points (StaticFrames and HandEye) and projects onto the chain's
                       own projections; after bundle_adjust valid == "at least 2 inlier views"; RollingFrames raise
  repeated calls       bit for bit; chunked calls; the cfg5 dome against the oracle on a 2000-point subsample
"""
import ctypes as C

import numpy as np
import pytest

from multical_b200 import synthetic, undistort
from multical_b200.camera import Camera, CameraFisheye
from multical_b200.triangulate import triangulate, triangulate_points
from oracle import triangulate_oracle as to

pytestmark = pytest.mark.gpu

MODELS = ["standard", "rational", "thin_prism", "fisheye", "tilted"]


def rel(a, b):
  return float(np.abs(np.asarray(a) - b).max() / max(np.abs(b).max(), 1e-300))


def cameras_of(scene, src="gt"):
  g = scene[src]
  if scene["model"] == "fisheye":
    return [CameraFisheye(scene["image_size"], g["K"][c], g["dist"][c].reshape(4, 1)) for c in range(scene["C"])]
  return [Camera(scene["image_size"], g["K"][c], g["dist"][c], model=scene["model"]) for c in range(scene["C"])]


def scene_views(scene):
  """pixels [C, N, 2], valid [C, N] and the rig points [N, 3] (frame_pose @ board_pose @ X) of a scene's F * B * P corners."""
  C, F, B, P = scene["C"], scene["F"], scene["B"], scene["P"]
  g = scene["gt"]
  Xb = np.zeros((B, P, 3))
  for b, p in enumerate(scene["board_points"]): Xb[b, :len(p)] = p
  Xw = np.einsum("bij,bpj->bpi", g["board_poses"][:, :3, :3], Xb) + g["board_poses"][:, None, :3, 3]
  Xr = np.einsum("fij,bpj->fbpi", g["frame_poses"][:, :3, :3], Xw) + g["frame_poses"][:, None, None, :3, 3]
  return scene["points"].reshape(C, F * B * P, 2), scene["valid"].reshape(C, F * B * P), Xr.reshape(-1, 3)


# ---- 1. the linear path against cv2.triangulatePoints -----------------------------------------------------------------------------
def linear_pair(kind, n, seed=0):
  """Two pixel projection matrices K [R | t] of a pair and the noisy pixels [2, n] of n points in front of both."""
  rng = np.random.default_rng(seed)
  K = np.array([[1100.0, 0.0, 960.0], [0.0, 1105.0, 540.0], [0.0, 0.0, 1.0]])
  base = {"horizontal": [0.12, 0.004, 0.002], "vertical": [0.003, 0.12, 0.002], "narrow": [0.02, 0.001, 0.0005],
          "wide": [1.8, 0.1, 0.4]}[kind]
  import cv2
  R2 = cv2.Rodrigues(np.array([0.01, -0.2 if kind == "wide" else -0.02, 0.005]))[0]
  P1 = K @ np.hstack([np.eye(3), np.zeros((3, 1))])
  P2 = K @ np.hstack([R2, -R2 @ np.array(base).reshape(3, 1)])
  X = np.stack([rng.uniform(-0.6, 0.6, n), rng.uniform(-0.4, 0.4, n), rng.uniform(1.0, 4.0, n), np.ones(n)])
  x = [(P @ X) for P in (P1, P2)]
  x = [v[:2] / v[2] + rng.normal(0, 0.5, (2, n)) for v in x]
  return P1, P2, x[0], x[1]


def run_linear(Ns, kinds=("horizontal", "vertical", "narrow", "wide")):
  import cv2
  worst = dict(point=0.0, norm=0.0, cos=0.0, f32=0.0)
  for kind in kinds:
    for n in Ns:
      P1, P2, x1, x2 = linear_pair(kind, n, seed=n)
      ours = triangulate_points(P1, P2, x1, x2)
      ref = cv2.triangulatePoints(P1, P2, x1, x2)
      assert ours.dtype == np.float64 and ours.shape == (4, n)
      d_ours, d_ref = ours[:3] / ours[3], ref[:3] / ref[3]
      e_point = float((np.linalg.norm(d_ours - d_ref, axis=0) / np.linalg.norm(d_ref, axis=0)).max())
      e_norm = float(np.abs(np.linalg.norm(ours, axis=0) - 1).max())
      cos = np.abs((ours * ref).sum(0)) / (np.linalg.norm(ours, axis=0) * np.linalg.norm(ref, axis=0))
      e_cos = float((1 - cos).max())
      assert e_point <= 1e-9, (kind, n, e_point)
      assert e_norm <= 1e-15, (kind, n, e_norm)
      assert e_cos <= 1e-15, (kind, n, e_cos)
      o32 = triangulate_points(P1, P2, x1.astype(np.float32), x2.astype(np.float32))
      r32 = cv2.triangulatePoints(P1, P2, x1.astype(np.float32), x2.astype(np.float32))
      assert o32.dtype == np.float32 and r32.dtype == np.float32
      d32, r32d = o32[:3].astype(np.float64) / o32[3], r32[:3].astype(np.float64) / r32[3]
      e32 = float((np.linalg.norm(d32 - r32d, axis=0) / np.linalg.norm(r32d, axis=0)).max())
      assert e32 <= 3e-7, (kind, n, e32)
      for k, v in zip(worst, (e_point, e_norm, e_cos, e32)): worst[k] = max(worst[k], v)
  print(f"linear vs cv2: {worst}")
  return worst


# ---- 2. noise-free recovery -------------------------------------------------------------------------------------------------------
def depth_of(scene, X, valid):
  T = scene["gt"]["cam_poses"]
  z = np.einsum("cj,nj->cn", T[:, 2, :3], X) + T[:, 2, 3][:, None]
  return np.where(valid, z, 0).sum(0) / np.maximum(valid.sum(0), 1)


def run_noise_free(models=MODELS, F=2):
  worst = {}
  for model in models:
    scene = synthetic.make_scene(C=4, F=F, model=model, noise=0.0, seed=11)
    pixels, valid, X = scene_views(scene)
    out = triangulate(cameras_of(scene), scene["gt"]["cam_poses"], pixels, valid)
    want = valid.sum(0) >= 2
    assert np.array_equal(out.valid, want), model
    assert np.isnan(out.points[~want]).all() and np.isnan(out.rms[~want]).all()
    err = np.linalg.norm(out.points[want] - X[want], axis=1) / depth_of(scene, X, valid)[want]
    assert err.max() <= 1e-9, (model, err.max())
    assert out.rms[want].max() <= 1e-9, (model, out.rms[want].max())
    worst[model] = (float(err.max()), float(out.rms[want].max()))
  print(f"noise-free: {worst}")
  return worst


# ---- 3. against the oracle ----------------------------------------------------------------------------------------------------------
def parity(scene, idx, cams=None, poses=None):
  """Triangulate the whole scene, compare the points `idx` with the oracle."""
  pixels, valid, _ = scene_views(scene)
  g = scene["gt"]
  out = triangulate(cams or cameras_of(scene), g["cam_poses"] if poses is None else poses, pixels, valid)
  assert np.array_equal(out.valid, valid.sum(0) >= 2)
  Xo, rms_o, cost_o = to.triangulate(scene["model"], g["K"], g["dist"], g["cam_poses"], pixels[:, idx], valid[:, idx])
  ok = out.valid[idx]
  assert np.array_equal(ok, ~np.isnan(rms_o))
  e_pt = np.linalg.norm(out.points[idx][ok] - Xo[ok], axis=1) / np.linalg.norm(Xo[ok], axis=1)
  # where the two differ by more than 1e-9, the step between them must change the oracle's linearised cost by less than 1e-12 of it:
  # along the flattest direction of a two- or three-view point the cost cannot tell such points apart in fp64
  for i in np.flatnonzero(e_pt > 1e-9):
    k = idx[np.flatnonzero(ok)[i]]
    cams = np.flatnonzero(valid[:, k])
    res = lambda x: np.concatenate([to.project(scene["model"], g["K"][c], g["dist"][c], g["cam_poses"][c, :3, :3] @ x
                                               + g["cam_poses"][c, :3, 3]) - pixels[c, k] for c in cams])
    Jd = to.central_jacobian(res, Xo[ok][i]) @ (out.points[k] - Xo[ok][i])
    assert 0.5 * Jd @ Jd <= 1e-12 * cost_o[ok][i], (k, e_pt[i], 0.5 * Jd @ Jd, cost_o[ok][i])
    e_pt[i] = 0.0
  # each side computes its rms from residuals of pixels near 1000 px, which carry about 1e-13 px of rounding
  e_rms = np.maximum(np.abs(out.rms[idx][ok] - rms_o[ok]) - 1e-13, 0.0) / rms_o[ok]
  cost_d = to.cost(scene["model"], g["K"], g["dist"], g["cam_poses"], pixels[:, idx][:, ok], valid[:, idx][:, ok], out.points[idx][ok])
  e_cost = float(((cost_d - cost_o[ok]) / cost_o[ok]).max()) if ok.any() else 0.0
  return out, float(e_pt.max(initial=0)), float(e_rms.max(initial=0)), e_cost


def run_oracle_parity(models=MODELS, Cs=(2, 3, 7, 33, 64), F=2, n=None):
  worst = {}
  for model in models:
    for Cn in Cs:
      scene = synthetic.make_scene(C=Cn, F=F, model=model, noise=0.3, rig="arc" if Cn <= 3 else "dome", seed=Cn)
      N = scene["F"] * scene["B"] * scene["P"]
      idx = np.arange(N) if n is None else np.random.default_rng(Cn).choice(N, min(n, N), replace=False)
      _, e_pt, e_rms, e_cost = parity(scene, idx)
      assert e_pt <= 1e-9, (model, Cn, e_pt)
      assert e_rms <= 1e-10, (model, Cn, e_rms)
      assert e_cost <= 1e-9, (model, Cn, e_cost)
      worst[(model, Cn)] = (e_pt, e_rms, e_cost)
  print("oracle parity (point, rms, cost excess):", {k: tuple(f"{v:.1e}" for v in vs) for k, vs in worst.items()})
  return worst


# ---- 4. validity and refusals ---------------------------------------------------------------------------------------------------------
def rig3():
  K = np.array([[1000.0, 0, 320], [0, 1000.0, 240], [0, 0, 1]])
  cams = [Camera((640, 480), K, np.array([-0.1, 0.02, 0.001, -0.001, 0.0])) for _ in range(3)]
  poses = np.tile(np.eye(4), (3, 1, 1))
  poses[1, :3, 3] = [-0.2, 0.0, 0.0]
  poses[2, :3, 3] = [0.0, 0.0, -3.0]                 # camera 2 sits 3 m in front of the rig origin, looking the same way
  return cams, poses


def run_validity():
  from oracle.ba_oracle import project_pinhole
  cams, poses = rig3()
  X = np.array([[0.05, 0.02, 1.5], [0.05, 0.02, 1.5], [0.05, 0.02, 1.5], [0.1, -0.05, 1.2], [0.0, 0.03, 2.0], [-0.02, 0.01, 4.0]])
  pixels = np.stack([project_pinhole(X @ T[:3, :3].T + T[:3, 3], c.intrinsic, c.dist) for c, T in zip(cams, poses)])
  valid = np.ones((3, len(X)), bool)
  valid[:, 0] = False                                # no view
  valid[1:, 1] = False                               # one view
  valid[2, 2] = False
  pixels[1, 2] = [np.nan, 100.0]                     # point 2: a non-finite pixel in a valid view
  # points 3 and 4 (z = 1.2, 2.0 < 3) are behind camera 2, point 5 is in front of all three
  out = triangulate(cams, poses, pixels, valid)
  assert out.valid.tolist() == [False, False, False, False, False, True], out.valid
  assert np.isnan(out.points[:5]).all() and np.isnan(out.rms[:5]).all()
  assert np.abs(out.points[5] - X[5]).max() < 1e-9 and out.rms[5] < 1e-9


def run_errors():
  cams, poses = rig3()
  pixels, valid = np.zeros((3, 4, 2)), np.ones((3, 4), bool)
  fish = CameraFisheye((640, 480), cams[0].intrinsic, np.zeros((4, 1)))
  with pytest.raises(NotImplementedError, match=r"fisheye for cameras \[1\]"):
    triangulate([cams[0], fish, cams[2]], poses, pixels, valid)
  with pytest.raises(ValueError): triangulate(cams, poses[:2], pixels, valid)
  with pytest.raises(ValueError): triangulate(cams, poses, pixels[:2], valid)
  with pytest.raises(ValueError): triangulate(cams, poses, pixels[..., :1], valid)
  with pytest.raises(ValueError): triangulate(cams, poses, pixels, valid[:, :3])
  with pytest.raises(ValueError): triangulate_points(np.eye(3), np.eye(3, 4), np.zeros((2, 3)), np.zeros((2, 3)))
  with pytest.raises(ValueError): triangulate_points(np.eye(3, 4), np.eye(3, 4), np.zeros((3, 2)), np.zeros((3, 2)))
  with pytest.raises(ValueError): triangulate_points(np.eye(3, 4), np.eye(3, 4), np.zeros((2, 3)), np.zeros((2, 4)))
  # the C-ABI's codes
  eng = undistort.undistort_engine()
  lib, D, U8 = eng.lib, C.POINTER(C.c_double), C.POINTER(C.c_uint8)
  vec = np.stack([undistort.camera_vector(c)[1] for c in cams])
  pts, ok, rms = np.zeros((4, 3)), np.zeros(4, np.uint8), np.zeros(4)
  v8 = valid.astype(np.uint8)

  def tri(model=0, n_cams=3, cameras=vec, T=poses, N=4):
    T = np.ascontiguousarray(T, np.float64); cameras = np.ascontiguousarray(cameras, np.float64)
    return lib.mcba_triangulate(eng.h, model, n_cams, cameras.ctypes.data_as(D), T.ctypes.data_as(D), N, pixels.ctypes.data_as(D),
                                v8.ctypes.data_as(U8), pts.ctypes.data_as(D), ok.ctypes.data_as(U8), rms.ctypes.data_as(D))
  assert tri() == 0
  assert tri(n_cams=0) == 1 and tri(n_cams=257) == 1 and tri(N=-1) == 1 and tri(model=9) == 1
  bad = vec.copy(); bad[1, 5] = np.inf
  assert tri(cameras=bad) == 5 and "camera 1" in lib.mcba_last_error(eng.h).decode()
  badT = poses.copy(); badT[2, 0, 3] = np.nan
  assert tri(T=badT) == 5
  P = np.eye(3, 4); Pn = P.copy(); Pn[1, 1] = np.nan
  x = np.zeros((2, 2)); out = np.zeros((4, 2))
  lin = lambda P1, N=2: lib.mcba_triangulate_linear(eng.h, P1.ctypes.data_as(D), P.ctypes.data_as(D), N, x.ctypes.data_as(D),
                                                    x.ctypes.data_as(D), out.ctypes.data_as(D))
  assert lin(P) == 0 and lin(Pn) == 5 and lin(P, N=-1) == 1
  assert lib.mcba_triangulate_linear(eng.h, None, P.ctypes.data_as(D), 2, x.ctypes.data_as(D), x.ctypes.data_as(D),
                                     out.ctypes.data_as(D)) == 1


# ---- 5. Calibration.triangulate ---------------------------------------------------------------------------------------------------------
def hand_eye_copy(calib, seed=3):
  """The calibration with HandEye motion whose frame poses G A_f W equal the static frame poses (G, W random)."""
  from multical_b200.motion import HandEye
  from multical_b200.pose_set import pose_table
  rng = np.random.default_rng(seed)
  G, W = synthetic.to_matrix(rng.normal(0, 0.3, (2, 6)))
  A = np.linalg.inv(G)[None] @ np.asarray(calib.motion.poses) @ np.linalg.inv(W)[None]
  return calib.copy(motion=HandEye(pose_table(A, calib.motion.valid), W, G))


def run_calibration(F=3, ba_F=6):
  from oracle.ba_oracle import project_fisheye, project_pinhole
  from multical_b200.calibration import from_scene
  from multical_b200.motion import RollingFrames
  scene = synthetic.make_scene(C=3, F=F, noise=0.0, seed=5)
  calib = from_scene(scene, guess=False)
  for c in (calib, hand_eye_copy(calib)):
    tab = c.triangulate()
    _, valid, X = scene_views(scene)
    assert tab.points.shape == (F, scene["B"], scene["P"], 3)
    want = (valid.sum(0) >= 2).reshape(tab.valid.shape)
    assert np.array_equal(tab.valid, want)
    Xm = np.asarray(c.motion.poses)[:, None, None, :3, :3] @ np.asarray(c.world_points.points)[None, ..., None]
    Xm = Xm[..., 0] + np.asarray(c.motion.poses)[:, None, None, :3, 3]
    assert np.abs(tab.points[want] - Xm[want]).max() <= 1e-9
    assert np.abs(Xm.reshape(-1, 3) - X).max() <= 1e-9
    # the chain's own projection (Calibration.projected) of these points is camera_pose @ rig point
    proj = c.projected
    for k, cam in enumerate(c.cameras):
      T = np.asarray(c.camera_poses.poses)[k]
      Xc = tab.points[want] @ T[:3, :3].T + T[:3, 3]
      uv = (project_fisheye if scene["model"] == "fisheye" else project_pinhole)(Xc, cam.intrinsic, cam.dist)
      assert np.abs(uv - np.asarray(proj.points)[k][want]).max() <= 1e-6
  noisy = from_scene(synthetic.make_scene(C=3, F=ba_F, noise=0.3, seed=6, outlier_fraction=0.02))
  solved = noisy.bundle_adjust().reject_outliers_quantile(0.95, 3.0).bundle_adjust()
  tab = solved.triangulate()
  inl = np.asarray(solved.inliers)
  assert np.array_equal(tab.valid, inl.sum(0) >= 2)
  assert not np.isnan(tab.points[tab.valid]).any() and np.isnan(tab.points[~tab.valid]).all()
  rolling = calib.copy(motion=RollingFrames(np.asarray(calib.motion.poses), np.asarray(calib.motion.poses), calib.motion.valid,
                                            [str(i) for i in range(F)]))
  with pytest.raises(NotImplementedError, match="RollingFrames"):
    rolling.triangulate()


# ---- 6. reproducibility and sizes ---------------------------------------------------------------------------------------------------
def run_reproducible(Cs=(3, 40), F=2):
  for Cn in Cs:
    scene = synthetic.make_scene(C=Cn, F=F, noise=0.3, rig="dome", seed=Cn, vis=0.8)
    pixels, valid, _ = scene_views(scene)
    a = triangulate(cameras_of(scene), scene["gt"]["cam_poses"], pixels, valid)
    b = triangulate(cameras_of(scene), scene["gt"]["cam_poses"], pixels, valid)
    for k in ("points", "rms", "valid"):
      assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (Cn, k)
    # an odd point count that ends inside a group and a CTA, and a prefix of the same points: the same bits
    n = pixels.shape[1] - 3
    c = triangulate(cameras_of(scene), scene["gt"]["cam_poses"], pixels[:, :n], valid[:, :n])
    assert np.array_equal(c.points.view(np.uint8), a.points[:n].view(np.uint8))


def run_chunks(N=100003, Cn=64):
  """N points of Cn cameras, more than one chunk (include/mcba.h MCBA_TRI_CHUNK_BYTES): the same bits as the points one by one."""
  scene = synthetic.make_scene(C=Cn, F=1, noise=0.3, rig="dome", seed=9, vis=0.9)
  pixels, valid, _ = scene_views(scene)
  rng = np.random.default_rng(1)
  pick = rng.integers(0, pixels.shape[1], N)
  big = triangulate(cameras_of(scene), scene["gt"]["cam_poses"], pixels[:, pick], valid[:, pick])
  small = triangulate(cameras_of(scene), scene["gt"]["cam_poses"], pixels, valid)
  assert np.array_equal(big.points.view(np.uint8), small.points[pick].view(np.uint8))
  assert np.array_equal(big.valid, small.valid[pick])


def test_linear_matches_cv2_triangulate_points():
  run_linear([1, 1000, 100003])


def test_noise_free_recovery_all_models():
  run_noise_free()


@pytest.mark.parametrize("model", MODELS)
def test_refined_points_match_the_oracle(model):
  run_oracle_parity([model], n=300)


def test_validity():
  run_validity()


def test_refusals():
  run_errors()


def test_calibration_triangulate():
  run_calibration()


def test_repeated_calls_agree_bit_for_bit():
  run_reproducible()


def test_chunked_calls():
  run_chunks()


def test_cfg5_dome_against_the_oracle():
  scene = synthetic.make_workload("cfg5")
  pixels, valid, X = scene_views(scene)
  idx = np.random.default_rng(0).choice(pixels.shape[1], 2000, replace=False)
  out, e_pt, e_rms, e_cost = parity(scene, idx)
  assert e_pt <= 1e-9 and e_rms <= 1e-10 and e_cost <= 1e-9, (e_pt, e_rms, e_cost)
  print(f"cfg5: {valid.sum()} observations, {out.valid.sum()} valid points; vs oracle on 2000: point {e_pt:.1e}, rms {e_rms:.1e}")
