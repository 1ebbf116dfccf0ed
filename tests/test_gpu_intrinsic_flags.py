"""GPU (-m gpu): OpenCV's fixed-parameter calibration flags in the intrinsic calibration (`flags` of Camera.calibrate / calibrate_cameras
and CameraFisheye.calibrate / calibrate_cameras_fisheye; multical_b200/intrinsics.py pinhole_flags, fisheye_flags) and the engine's
fixed-intrinsics mask underneath (include/mcba.h mcba_set_fixed_intrinsics).

Bars:
  pinhole, against cv2.calibrateCameraExtended with criteria (COUNT+EPS, 500, 1e-15) and the same flags, called live: the converged bars
                     of tests/test_gpu_intrinsics.py (fx fy cx cy <= 1e-6 relative, dist <= 1e-6, total RMS <= 1e-9 relative, per-view
                     RMS <= 1e-6 px, rvec / tvec <= 1e-6)
  fisheye, against cv2.fisheye.calibrate with criteria (COUNT+EPS, 1000, 1e-15) and the reference's flags | the flag: the converged bars
                     of tests/test_gpu_fisheye_intrinsics.py
  fixed values       a fixed coefficient is exactly 0, a fixed principal point (fisheye: focal lengths) exactly K0's (==)
  full loop with CALIB_FIX_K3 against the reference's goldens (tests/golden/intrinsic_flags_loop_40*.npz, make_intrinsic_flags_golden.py):
                     same rounds and views; OpenCV converged: the bars of tests/test_gpu_intrinsics.py's golden test; at the reference's
                     default criteria OpenCV stops short, and the device's error is not above the reference's
  engine             with the mask, J^T J and J^T r have zero rows and columns at the fixed indices and equal the unmasked
                     linearisation's bit for bit elsewhere; the solve leaves the fixed entries of param_vec bit for bit; identical
                     masked solves agree bit for bit; the next upload clears the mask (and the cached solve graph follows)
"""
import numpy as np
import pytest

import test_gpu_fisheye_intrinsics as gf
import test_gpu_intrinsics as gi
from conftest import GOLDEN
from multical_b200 import intrinsics, synthetic
from multical_b200.board import Board
from multical_b200.camera import Camera, CameraFisheye

pytestmark = pytest.mark.gpu

# case -> (OpenCV flag names, fix_aspect): the flags go to the device and to OpenCV, fix_aspect adds CALIB_FIX_ASPECT_RATIO on OpenCV's side
PINHOLE = {
  "FIX_K1": (["CALIB_FIX_K1"], False), "FIX_K2": (["CALIB_FIX_K2"], False), "FIX_K3": (["CALIB_FIX_K3"], False),
  "ZERO_TANGENT_DIST": (["CALIB_ZERO_TANGENT_DIST"], False), "FIX_TANGENT_DIST": (["CALIB_FIX_TANGENT_DIST"], False),
  "FIX_PRINCIPAL_POINT": (["CALIB_FIX_PRINCIPAL_POINT"], False), "FIX_ASPECT_RATIO": (["CALIB_FIX_ASPECT_RATIO"], False),
  "FIX_K4_K5_K6_S_TAU": (["CALIB_FIX_K4", "CALIB_FIX_K5", "CALIB_FIX_K6", "CALIB_FIX_S1_S2_S3_S4", "CALIB_FIX_TAUX_TAUY"], False),
  "FIX_K3|ZERO_TANGENT_DIST": (["CALIB_FIX_K3", "CALIB_ZERO_TANGENT_DIST"], False),
  "FIX_PRINCIPAL_POINT|fix_aspect": (["CALIB_FIX_PRINCIPAL_POINT"], True),
}
FISHEYE = {"FIX_K3|FIX_K4": ["CALIB_FIX_K3", "CALIB_FIX_K4"], "FIX_K1": ["CALIB_FIX_K1"],
           "FIX_PRINCIPAL_POINT": ["CALIB_FIX_PRINCIPAL_POINT"], "FIX_FOCAL_LENGTH": ["CALIB_FIX_FOCAL_LENGTH"]}


def flag_bits(names, fisheye=False):
  import cv2
  ns = cv2.fisheye if fisheye else cv2
  out = 0
  for n in names: out |= getattr(ns, n)
  return out


def run_pinhole(case, F, report=print):
  import cv2
  names, fix_aspect = PINHOLE[case]
  flags = flag_bits(names)
  scene = gi.scene_of(1, F, 72)
  boards = gi.boards_of(scene)
  views = intrinsics.calibration_points(boards, gi.detections(scene["points"][0], scene["valid"][0]))
  size = scene["image_size"]
  rms, K, d, rt, pv = gi.cv_calibrate(views, size, flags | (cv2.CALIB_FIX_ASPECT_RATIO if fix_aspect else 0), gi.CV_TIGHT)
  fixed, flag_aspect = intrinsics.pinhole_flags(flags)
  r = intrinsics.calibrate_views(boards, [views], [size], fix_aspect=fix_aspect or flag_aspect, fixed=fixed, **gi.TIGHT)[0]
  x = r.intrinsics
  got = dict(K=np.abs(x[:4] / K[[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max(), dist=np.abs(x[5:] - d).max(), rms=abs(r.rms / rms - 1),
             per_view=np.abs(r.per_view - pv).max(), pose=np.abs(r.rtvecs - rt).max())
  report(f"\nmargins {case} ({len(views)} views, RMS {rms:.6f}): " + ", ".join(f"{k} {v:.2e}" for k, v in got.items()))
  assert got["K"] <= 1e-6 and got["dist"] <= 1e-6 and got["rms"] <= 1e-9 and got["per_view"] <= 1e-6 and got["pose"] <= 1e-6, got
  w, h = size
  if fixed is not None:
    assert (x[5:][fixed[5:]] == 0).all() and (d[fixed[5:]] == 0).all()
    if fixed[2]: assert x[2] == r.k0[2] == (w - 1) * 0.5 and x[3] == r.k0[3] == (h - 1) * 0.5
  assert x[4] == 0.0
  if fix_aspect or flag_aspect: assert x[0] == x[1]


@pytest.mark.parametrize("case", list(PINHOLE))
def test_pinhole_flags_match_opencv(case):
  run_pinhole(case, 50)


def run_fisheye(case, F, report=print):
  import cv2
  flags = flag_bits(FISHEYE[case], fisheye=True)
  scene = gf.scene_of(1, F, 92)
  boards = gf.boards_of(scene)
  views = intrinsics.calibration_points(boards, gi.detections(scene["points"][0], scene["valid"][0]))
  size = scene["image_size"]
  rms, K, d, rv, tv = cv2.fisheye.calibrate([v.object_points[None] for v in views], [v.corners[None] for v in views], tuple(size), None,
                                            None, criteria=gf.CV_TIGHT, flags=gf.cv_flags() | flags)
  d = d.ravel()
  rt = np.hstack([np.stack(rv).reshape(-1, 3), np.stack(tv).reshape(-1, 3)])
  fixed = intrinsics.fisheye_flags(flags)
  r = intrinsics.calibrate_views(boards, [views], [size], model="fisheye", fixed=fixed, **gf.TIGHT)[0]
  x = r.intrinsics
  got = dict(rms=abs(r.rms / rms - 1), K=np.abs(x[:4] / K[[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max(), dist=np.abs(x[5:] - d).max(),
             pose=np.abs(r.rtvecs - rt).max(), px=np.abs(gf.project(gf.K_of(x), x[5:], r.rtvecs, views) - gf.project(K, d, rt, views)).max())
  report(f"\nmargins fisheye {case} ({len(views)} views, RMS {rms:.6f}): " + ", ".join(f"{k} {v:.2e}" for k, v in got.items()))
  assert got["rms"] <= 1e-9 and got["K"] <= 1e-6 and got["px"] <= 1e-6 and got["dist"] <= gf.DIST_BAR and got["pose"] <= gf.POSE_BAR, got
  assert (x[5:][fixed[5:]] == 0).all() and (d[fixed[5:]] == 0).all() and x[4] == 0.0
  assert (x[:4][fixed[:4]] == r.k0[:4][fixed[:4]]).all() and (K[[0, 1, 0, 1], [0, 1, 2, 2]][fixed[:4]] == r.k0[:4][fixed[:4]]).all()
  # the public entry takes the same flags to the same solve
  cam, err = CameraFisheye.calibrate(boards, gi.detections(scene["points"][0], scene["valid"][0]), size, flags=flags)
  r_def = intrinsics.calibrate_views(boards, [views], [size], model="fisheye", fixed=fixed)[0]
  assert np.array_equal(cam.intrinsic[[0, 1, 0, 1], [0, 1, 2, 2]], r_def.intrinsics[:4]) and err == r_def.rms


@pytest.mark.parametrize("case", list(FISHEYE))
def test_fisheye_flags_match_opencv(case):
  run_fisheye(case, 40)


def load_golden(name):
  z = dict(np.load(f"{GOLDEN}/{name}.npz", allow_pickle=False))
  boards = [Board(p, size=(16, 22)) for p in z["board_points"]]
  return z, boards, gi.detections(z["points"], z["valid"])


def run_golden(name, monkeypatch, report=print):
  """Camera.calibrate with the golden's arguments: the same rounds and the same views as the reference's loop.  With OpenCV converged
  (the _tight golden) the bars of test_gpu_intrinsics.py's golden test; at the reference's default criteria OpenCV stops 1.2 % in fx short
  of the minimum on this scene (make_intrinsic_flags_golden.py), so there the device's error is only required not to be above it."""
  z, boards, dets = load_golden(name)
  rounds = []
  real = intrinsics.calibrate_views
  monkeypatch.setattr(intrinsics, "calibrate_views", lambda *a, **k: rounds.append(1) or real(*a, **k))
  cam, err = Camera.calibrate(boards, float(z["limit"]), dets, tuple(int(v) for v in z["image_size"]), model=str(z["model"]),
                              flags=int(z["flags"]), max_iter=int(z["max_iter"]), eps=float(z["eps"]))
  ds = cam.intrinsic_dataset
  assert np.array_equal(np.asarray(ds["board_ids"], np.float64), z["board_ids"])
  assert np.array_equal(np.asarray(ds["image_ids"]), z["image_ids"])
  assert len(rounds) == int(z["rounds"]) > 1
  pv = np.asarray(cam.error_perview).ravel()
  got = dict(per_view=np.abs(pv - z["error_perview"]).max(),
             K=np.abs(cam.intrinsic[[0, 1, 0, 1], [0, 1, 2, 2]] / z["K"][[0, 1, 0, 1], [0, 1, 2, 2]] - 1).max())
  report(f"\ngolden {name} ({len(pv)} views, {len(rounds)} rounds, err {err} against {float(z['err'])}): " +
         ", ".join(f"{k} {v:.2e}" for k, v in got.items()))
  assert pv.shape == z["error_perview"].shape
  if int(z["max_iter"]) >= 500:
    assert got["per_view"] <= 1e-3 and got["K"] <= 1e-3 and err == float(z["err"]), (got, err)
  else:
    assert err <= float(z["err"]) and np.sqrt(np.mean(pv ** 2)) <= np.sqrt(np.mean(z["error_perview"] ** 2)), (err, float(z["err"]))
  fixed, _ = intrinsics.pinhole_flags(int(z["flags"]))
  assert (cam.dist.ravel()[fixed[5:]] == 0).all() and (z["dist"].ravel()[fixed[5:]] == 0).all()


@pytest.mark.parametrize("name", ["intrinsic_flags_loop_40", "intrinsic_flags_loop_40_tight"])
def test_calibrate_loop_with_fix_k3_matches_reference_golden(name, monkeypatch):
  run_golden(name, monkeypatch)


# ---- the engine's mask ------------------------------------------------------------------------------------------------------------
def ba_problem(C=2, F=6, seed=81, boards=False):
  """A bundle adjustment with free intrinsics (standard model): its engine and where camera 0's intrinsics sit in param_vec."""
  from multical_b200.calibration import from_scene
  scene = synthetic.make_scene(C=C, F=F, vis=0.5, seed=seed)
  calib = from_scene(scene).enable(cameras=True, boards=boards)
  eng = calib._upload(calib.inliers)
  n_pts = 3 * eng.desc.B * eng.desc.P if boards else 0
  off_in = eng.num_params - eng.kint * C - n_pts
  return calib, eng, off_in


FIXED = np.array([0, 0, 1, 1, 0, 0, 1, 0, 1, 1], bool)        # cx cy k2 p2 k3: the mask every camera shares


def fixed_columns(eng, off_in, C):
  return np.concatenate([off_in + eng.kint * c + np.flatnonzero(FIXED) for c in range(C)])


def run_engine_linearisation(boards):
  C = 2
  calib, eng, off_in = ba_problem(C=C, boards=boards)
  J0, g0, c0 = eng.linearize()
  eng.set_fixed_intrinsics(FIXED)
  J1, g1, c1 = eng.linearize()
  cols = fixed_columns(eng, off_in, C)
  rest = np.setdiff1d(np.arange(eng.num_params), cols)
  assert (J1[cols] == 0).all() and (J1[:, cols] == 0).all() and (g1[cols] == 0).all()
  assert np.abs(J0[np.ix_(cols, cols)]).max() > 0 and np.abs(g0[cols]).max() > 0         # the columns were not zero before
  if boards:      # board-point rows are added with fp64 atomics in any order: entries within 1e-12 of their Cauchy-Schwarz bound
    dg = np.sqrt(np.abs(np.diag(J0)))[rest]
    assert (np.abs(J1 - J0)[np.ix_(rest, rest)] <= 1e-12 * np.outer(dg, dg)).all()
    assert (np.abs(g1 - g0)[rest] <= 1e-12 * dg * np.sqrt(2 * c0)).all() and abs(c1 / c0 - 1) <= 1e-12
  else:
    assert np.array_equal(J1[np.ix_(rest, rest)], J0[np.ix_(rest, rest)]) and np.array_equal(g1[rest], g0[rest]) and c1 == c0
  return calib, eng, off_in, cols


@pytest.mark.parametrize("boards", [False, True])
def test_mask_zeroes_the_rows_and_columns_of_the_normal_equations(boards):
  run_engine_linearisation(boards)


def run_engine_solves():
  C = 2
  calib, eng, off_in, cols = run_engine_linearisation(False)
  opts = dict(ftol=1e-12, xtol=1e-12, gtol=1e-12, max_nfev=30)
  x0 = eng.param_vec

  def masked_solve():
    calib._upload(calib.inliers)
    eng.set_param_vec(x0)
    eng.set_fixed_intrinsics(FIXED)
    res = eng.solve(**opts)
    return eng.param_vec, res

  def plain_solve():
    calib._upload(calib.inliers)
    eng.set_param_vec(x0)
    res = eng.solve(**opts)
    return eng.param_vec, res

  xp, rp = plain_solve()
  xa, ra = masked_solve()
  xb, rb = masked_solve()
  assert np.array_equal(xa[cols], x0[cols])                                      # held fixed, bit for bit
  assert ra.nfev > 1 and np.abs(xa - x0).max() > 0 and np.abs(xp[cols] - x0[cols]).max() > 0
  assert np.array_equal(xa, xb) and ra.cost == rb.cost and ra.nfev == rb.nfev     # reproducible
  assert ra.cost > rp.cost                                                       # fewer free parameters: a higher minimum
  xq, rq = plain_solve()                                                         # the upload cleared the mask
  assert np.array_equal(xq, xp) and rq.cost == rp.cost and rq.nfev == rp.nfev
  # a mask on a problem whose intrinsics are fixed changes nothing
  calib2 = calib.enable(cameras=False)
  e2 = calib2._upload(calib2.inliers)
  y0 = e2.param_vec
  r0 = e2.solve(**opts)
  y1 = e2.param_vec
  calib2._upload(calib2.inliers)
  e2.set_param_vec(y0)
  e2.set_fixed_intrinsics(FIXED)
  r1 = e2.solve(**opts)
  assert np.array_equal(e2.param_vec, y1) and r1.cost == r0.cost


def test_masked_solves_hold_the_fixed_parameters_and_the_next_upload_clears_the_mask():
  run_engine_solves()


def run_mask_arguments():
  calib, eng, off_in = ba_problem()
  with pytest.raises(AssertionError, match="0 or 1"):
    eng.set_fixed_intrinsics(np.where(FIXED, 2, 0))
  with pytest.raises(AssertionError, match="expected 10 entries"):
    eng.set_fixed_intrinsics(np.zeros(9, bool))
  from multical_b200 import _native as nat
  eng.upload_dense("standard", nat.OPT_BITS["cameras"] | nat.OPT_FIX_ASPECT, np.ones((1, 1, 1, 1), bool), np.zeros((1, 1, 1, 1, 2)),
                   np.zeros((1, 1, 3)))
  with pytest.raises(AssertionError, match="fy follows fx"):
    eng.set_fixed_intrinsics(np.array([0, 1] + [0] * 8, bool))
  eng.set_fixed_intrinsics(np.array([1, 1] + [0] * 8, bool))
  eng.set_fixed_intrinsics(None)


def test_mask_arguments():
  run_mask_arguments()


# ---- refusals (host only) ---------------------------------------------------------------------------------------------------------
def run_refused_flags():
  import cv2
  scene = gi.scene_of(1, 6, 73)
  boards = gi.boards_of(scene)
  dets = gi.detections(scene["points"][0], scene["valid"][0])
  size = scene["image_size"]
  for name in ["CALIB_USE_INTRINSIC_GUESS", "CALIB_FIX_FOCAL_LENGTH", "CALIB_RATIONAL_MODEL", "CALIB_THIN_PRISM_MODEL",
               "CALIB_TILTED_MODEL"]:
    with pytest.raises(NotImplementedError, match=name):
      Camera.calibrate(boards, 1.0, dets, size, flags=getattr(cv2, name) | cv2.CALIB_FIX_K3)
  for bits in [cv2.CALIB_FIX_INTRINSIC, cv2.CALIB_USE_LU, 1 << 30]:
    with pytest.raises(NotImplementedError, match=f"flag bits {bits} "):
      Camera.calibrate(boards, 1.0, dets, size, flags=bits)
  for name in ["CALIB_USE_INTRINSIC_GUESS", "CALIB_CHECK_COND"]:
    with pytest.raises(NotImplementedError, match=name):
      CameraFisheye.calibrate(boards, dets, size, flags=getattr(cv2.fisheye, name))
  for bits in [cv2.fisheye.CALIB_FIX_INTRINSIC, 1 << 30]:
    with pytest.raises(NotImplementedError, match=f"flag bits {bits} "):
      CameraFisheye.calibrate(boards, dets, size, flags=bits)


def test_refused_flags_name_the_flag():
  run_refused_flags()
