"""GPU (-m gpu): the non-overlapping camera initialisation (multical_b200/nonoverlap.py HandEye; include/mcba.h mcba_hand_eye_quads,
mcba_hand_eye_vote; csrc/hand_eye_init_kernels.cuh) against cv2.calibrateRobotWorldHandEye and scipy.stats.gaussian_kde called live,
against the reference's own HandEye.initialise_camera_poses (tests/golden/nonoverlap_*.npz, tests/golden/make_nonoverlap_golden.py)
and against oracle/nonoverlap_oracle.py at cfg4 shape.

Bars: every quadruple -- identical ok, X and Z rotations within 1e-9 element-wise, translations within 1e-9 relative; the vote --
densities within 1e-10 relative, identical argmax; the whole function -- identical reference camera, quadruples and image ids, X and
cam_init within 1e-9.
"""
import json
import os
import pickle

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from conftest import GOLDEN
from multical_b200 import synthetic
from multical_b200.calibration import get_engine
from multical_b200.nonoverlap import HandEye
from multical_b200.structs import Table
from oracle import nonoverlap_oracle

pytestmark = pytest.mark.gpu

SCENES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("nonoverlap_") and f.endswith(".npz"))
BAR = 1e-9
DENSITY_BAR = 1e-10


def golden(name):
  return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def assert_close(got, ref, bar=BAR):
  got, ref = np.asarray(got), np.asarray(ref)
  assert got.shape == ref.shape
  assert np.abs(got[..., :3, :3] - ref[..., :3, :3]).max(initial=0) <= bar
  t, tr = got[..., :3, 3], ref[..., :3, 3]
  assert (np.abs(t - tr) <= bar * np.maximum(1.0, np.abs(tr))).all()


def rigid(R, t):
  T = np.broadcast_to(np.eye(4), (*R.shape[:-2], 4, 4)).copy()
  T[..., :3, :3], T[..., :3, 3] = R, t
  return T


def problem(rng, n, family="random"):
  """A_i (cam_world) and B_i (base_gripper) of one quadruple with A X = Z B up to noise; the degenerate families repeat one rotation
  ("single"), use the identity ("identity"), rotate about one axis ("axis") or alternate two rotations ("two")."""
  X = rigid(Rotation.random(random_state=rng.integers(1 << 31)).as_matrix(), rng.normal(size=3))
  Z = rigid(Rotation.random(random_state=rng.integers(1 << 31)).as_matrix(), rng.normal(size=3))
  if family == "random":
    R = Rotation.random(n, random_state=rng.integers(1 << 31)).as_matrix()
  elif family == "single":
    R = np.broadcast_to(Rotation.random(random_state=rng.integers(1 << 31)).as_matrix(), (n, 3, 3))
  elif family == "identity":
    R = np.broadcast_to(np.eye(3), (n, 3, 3))
  elif family == "axis":
    ax = rng.normal(size=3)
    R = Rotation.from_rotvec(ax / np.linalg.norm(ax) * rng.uniform(-2, 2, (n, 1))).as_matrix()
  else:
    R2 = Rotation.random(2, random_state=rng.integers(1 << 31)).as_matrix()
    R = R2[np.arange(n) % 2]
  A = rigid(R, rng.normal(size=(n, 3)))
  B = np.linalg.inv(Z) @ A @ X
  if family == "random":
    B = B @ synthetic.to_matrix(np.hstack([rng.normal(0, 1e-3, (n, 3)), rng.normal(0, 1e-3, (n, 3))]))
  return A, B


def solve_on_device(problems):
  """one mcba_hand_eye_quads launch: problem k is quadruple (0, 1, k, k) of a two-camera table with poses inv(A), inv(B)."""
  F, K = max(len(a) for a, _ in problems), len(problems)
  poses = np.broadcast_to(np.eye(4), (2, F, K, 4, 4)).copy()
  valid = np.zeros((2, F, K), bool)
  for k, (A, B) in enumerate(problems):
    poses[0, :len(A), k], poses[1, :len(B), k] = np.linalg.inv(A), np.linalg.inv(B)
    valid[:, :len(A), k] = True
  quads = [(0, 1, k, k) for k in range(K)]
  return get_engine().hand_eye_quads(poses, valid, quads), (poses, valid, quads)


def run_quads_against_cv2(sizes, seed=0, degenerate_reps=4):
  rng = np.random.default_rng(seed)
  problems = [problem(rng, n) for n in sizes]
  rejected = [problem(rng, int(rng.integers(3, 30)), fam) for fam in ("single", "identity") for _ in range(degenerate_reps)]
  in_band = [problem(rng, int(rng.integers(3, 30)), fam) for fam in ("axis", "two") for _ in range(degenerate_reps)]
  (X, Z, n, ok), _ = solve_on_device(problems + rejected + in_band)
  worst = [0.0, 0.0]
  for k, (A, B) in enumerate(problems + rejected):
    ref = nonoverlap_oracle.hand_eye_robot_world(A, B)
    assert n[k] == len(A)
    assert ok[k] == (ref is not None), k
    if ref is not None:
      assert_close(X[k], ref[0]); assert_close(Z[k], ref[1])
      worst[0] = max(worst[0], np.abs(X[k][:3, :3] - ref[0][:3, :3]).max(), np.abs(Z[k][:3, :3] - ref[1][:3, :3]).max())
      worst[1] = max(worst[1], (np.abs(X[k][:3, 3] - ref[0][:3, 3]) / np.maximum(1, np.abs(ref[0][:3, 3]))).max())
  assert ok[:len(problems)].all()
  # exactly degenerate motions that OpenCV may accept with an arbitrary singular vector: dropped (DESIGN.md §3f)
  assert not ok[len(problems) + len(rejected):].any()
  return worst


def run_vote_against_scipy(sizes, seed=0):
  rng = np.random.default_rng(seed)
  sets = [rng.normal(size=(n, 3)) * rng.uniform(0.1, 2.0, 3) + rng.normal(size=3) for n in sizes]
  dens, best = get_engine().hand_eye_vote(sets)
  for s, d, b in zip(sets, dens, best):
    ref, ref_best = nonoverlap_oracle.kde_vote(s)
    assert np.abs(d / ref - 1).max() <= DENSITY_BAR, len(s)
    assert b == ref_best, len(s)
    if len(s) == 4:                                  # d + 1 points: equal densities, the tie goes to the lowest index
      assert b == 0 and np.abs(d / d[0] - 1).max() < 1e-12
  for n in (0, 1, 2, 3):
    with pytest.raises(ValueError, match="at least 4"):
      get_engine().hand_eye_vote([rng.normal(size=(5, 3)), rng.normal(size=(n, 3))])
  with pytest.raises(ValueError, match="singular"):
    get_engine().hand_eye_vote([np.repeat(rng.normal(size=(1, 3)), 5, axis=0)])


def table_of(z):
  return Table.create(poses=z["poses"], valid=z["valid"], num_points=z["num_points"])


def names_of(z):
  return [f"cam{c}" for c in range(z["valid"].shape[0])]


def run_golden(name):
  z = golden(name)
  names = names_of(z)
  he = HandEye(table_of(z), names)
  he.initialise_camera_poses()
  assert he.reference_camera == names[int(z["reference_camera"])]
  quads = np.array([(names.index(r["master_cam"]), names.index(r["slave_cam"]), r["boardM"], r["boardS"]) for r in he.handeye_df])
  assert np.array_equal(quads.reshape(-1, 4), z["quads"])
  ids = [z["image_ids"][a:b] for a, b in zip(z["image_start"][:-1], z["image_start"][1:])]
  assert all(np.array_equal(r["image_ids"], i) for r, i in zip(he.handeye_df, ids))
  X = np.array([r["slaveCam_wrt_masterCam"] for r in he.handeye_df])
  assert_close(X, z["X"])
  assert_close(np.array([he.cam_init[k] for k in names]), z["cam_init"])
  assert he.camera_poses["Reference_camera"] == he.reference_camera
  # every vote on the reference's own transforms: the same pick, the density within the bar
  sets = [z["X"][(z["quads"][:, 0] == m) & (z["quads"][:, 1] == s)][:, :3, 3] for m, s in z["pairs"]]
  dens, best = get_engine().hand_eye_vote(sets)
  assert np.array_equal(best, z["pick"])
  got = np.array([d[b] for d, b in zip(dens, best)])
  assert np.abs(got / z["density"] - 1).max() <= DENSITY_BAR
  return np.abs(X - z["X"]).max(), np.abs(np.array([he.cam_init[k] for k in names]) - z["cam_init"]).max()


def run_reproducible(name):
  z = golden(name)
  outs = []
  for _ in range(2):
    he = HandEye(table_of(z), names_of(z))
    he.initialise_camera_poses()
    outs.append((np.array([r["slaveCam_wrt_masterCam"] for r in he.handeye_df]), np.array([he.cam_init[k] for k in names_of(z)])))
  assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
  rng = np.random.default_rng(3)
  problems = [problem(rng, n) for n in (3, 50, 300)]
  a, _ = solve_on_device(problems)
  b, _ = solve_on_device(problems)
  assert all(np.array_equal(x, y) for x, y in zip(a, b))


def run_files(tmp_path, monkeypatch):
  z = golden("nonoverlap_all_boards")
  monkeypatch.chdir(tmp_path)
  he = HandEye(table_of(z), names_of(z))
  he.initialise_camera_poses()
  assert os.listdir(tmp_path) == []
  out = tmp_path / "out"
  out.mkdir()
  he = HandEye(table_of(z), names_of(z), str(out))
  he.initialise_camera_poses()
  assert sorted(os.listdir(out)) == ["camera_groups.pkl", "initial_guess.json"]
  got, ref = json.loads((out / "initial_guess.json").read_text()), json.loads(str(z["initial_guess"]))
  assert list(got) == list(ref) and got["Reference_camera"] == ref["Reference_camera"]
  for k in names_of(z):
    assert list(got[k]) == list(ref[k])
    for s in got[k]:
      assert_close(np.array(got[k][s]), np.array(ref[k][s]))
  with open(out / "camera_groups.pkl", "rb") as f:
    groups = pickle.load(f)
  assert list(groups) == names_of(z) and all(len(groups[k]) == len(names_of(z)) - 1 for k in groups)


def run_raising_scenes():
  """Scenes where the reference raises: every camera sees one board (one solve per camera pair), and a single camera."""
  poses, valid, npts, _ = synthetic.make_pose_table_scene(3, 30, 1, 0.9, seed=5)
  with pytest.raises(ValueError, match="at least 4"):
    nonoverlap_oracle.initialise_camera_poses(poses, valid, ["a", "b", "c"])
  with pytest.raises(ValueError, match="master camera a, slave camera b"):
    HandEye(Table.create(poses=poses, valid=valid, num_points=npts), ["a", "b", "c"]).initialise_camera_poses()
  poses, valid, npts, _ = synthetic.make_pose_table_scene(1, 30, 3, 0.9, seed=6)
  with pytest.raises(ValueError, match="reference camera"):
    nonoverlap_oracle.initialise_camera_poses(poses, valid, ["a"])
  with pytest.raises(ValueError, match="reference camera"):
    HandEye(Table.create(poses=poses, valid=valid, num_points=npts), ["a"]).initialise_camera_poses()


def test_every_quadruple_matches_cv2():
  rot, trans = run_quads_against_cv2([3, 4, 5, 7, 10, 31, 32, 33, 100, 127, 128, 129, 250, 500, 1000, 2000] + [20] * 40)
  print(f"largest difference from cv2: rotation {rot:.2e}, translation {trans:.2e} relative")


def test_vote_matches_gaussian_kde():
  run_vote_against_scipy([4, 4, 5, 6, 7, 25, 31, 32, 33, 64, 65, 300, 1000])


@pytest.mark.parametrize("name", SCENES)
def test_initialise_camera_poses_matches_reference_golden(name):
  x, c = run_golden(name)
  print(f"{name}: X {x:.2e}, cam_init {c:.2e}")


def test_cfg4_shape_matches_oracle():
  """16 cameras x 1000 frames x 5 boards, half the views valid: 6000 quadruples of about 250 images."""
  poses, valid, npts, cam = synthetic.make_pose_table_scene(16, 1000, 5, 0.5, seed=41)
  names = [f"cam{c}" for c in range(16)]
  he = HandEye(Table.create(poses=poses, valid=valid, num_points=npts), names)
  he.initialise_camera_poses()
  ref = nonoverlap_oracle.initialise_camera_poses(poses, valid, names)
  assert he.reference_camera == ref["reference_camera"] and len(he.handeye_df) == len(ref["handeye_df"]) == 6000
  for r, o in zip(he.handeye_df, ref["handeye_df"]):
    assert (r["master_cam"], r["slave_cam"], r["boardM"], r["boardS"]) == (o["master_cam"], o["slave_cam"], o["boardM"], o["boardS"])
  assert_close(np.array([r["slaveCam_wrt_masterCam"] for r in he.handeye_df]), np.array([o["slaveCam_wrt_masterCam"] for o in ref["handeye_df"]]))
  assert_close(np.array([he.cam_init[k] for k in names]), np.array([ref["cam_init"][k] for k in names]))


def test_bit_reproducible():
  run_reproducible("nonoverlap_many_boards")


def test_files_written_only_with_an_image_path(tmp_path, monkeypatch):
  run_files(tmp_path, monkeypatch)


def test_reference_failures_raise_value_error():
  run_raising_scenes()


def test_whole_chain_from_detections():
  """cfg2-sized scene with three boards: intrinsics, pose table, hand-eye camera poses, pose graph and bundle adjustment all through
  this package.  cam_init is the true relative camera pose up to the noise of the views, and the final RMS lands at sigma sqrt(2)."""
  from multical_b200 import workspace
  from multical_b200.board import Board
  from multical_b200 import nonoverlap
  from test_gpu_intrinsics import detections
  scene = synthetic.make_workload("cfg2", seed=5, boards=("charuco", 16, 22, 0.025, 3))
  boards = [Board(p, size=(16, 22), min_points=20) for p in scene["board_points"]]
  dets = [detections(scene["points"][c], scene["valid"][c]) for c in range(scene["C"])]
  cams, _ = workspace.calibrate_single(boards, dets, [scene["image_size"]] * scene["C"], "standard", 1.0)
  table = Table.create(points=scene["points"], valid=scene["valid"])
  seen = {}
  orig = nonoverlap.HandEye.initialise_camera_poses

  def keep(self):
    orig(self)
    seen["cam_init"] = self.cam_init
  nonoverlap.HandEye.initialise_camera_poses = keep
  try:
    calib = workspace.initialise_poses(table, boards, cams, is_non_overlapping=True)
  finally:
    nonoverlap.HandEye.initialise_camera_poses = orig
  cam = scene["gt"]["cam_poses"]
  truth = cam @ np.linalg.inv(cam[0])
  got = np.array([seen["cam_init"][str(c)] for c in range(scene["C"])])
  assert np.abs(got[:, :3, :3] - truth[:, :3, :3]).max() < 5e-3 and np.abs(got[:, :3, 3] - truth[:, :3, 3]).max() < 5e-3
  calib = workspace.calibrate(calib, cameras=True)
  rms = np.sqrt(np.mean(calib.reprojection_error ** 2))
  assert abs(rms - 0.3 * np.sqrt(2)) < 5e-3, rms


def test_bad_inputs():
  import ctypes as C
  eng = get_engine()
  lib = eng.lib
  poses, valid = np.broadcast_to(np.eye(4), (2, 5, 2, 4, 4)).copy(), np.ones((2, 5, 2), bool)
  with pytest.raises(AssertionError, match="dimensions"):
    eng.hand_eye_quads(np.zeros((0, 4, 4)), np.ones((0, 5, 2), bool), [(0, 1, 0, 0)])
  with pytest.raises(AssertionError, match="out of range"):
    eng.hand_eye_quads(poses, valid, [(0, 2, 0, 0)])
  with pytest.raises(AssertionError, match="out of range"):
    eng.hand_eye_quads(poses, valid, [(0, 1, 0, 2)])
  with pytest.raises(AssertionError, match="master == slave"):
    eng.hand_eye_quads(poses, valid, [(1, 1, 0, 1)])
  bad = poses.copy(); bad[1, 2, 0, 0, 3] = np.inf
  with pytest.raises(ValueError, match="non-finite"):
    eng.hand_eye_quads(bad, valid, [(0, 1, 0, 0)])
  with pytest.raises(ValueError, match="non-finite"):
    eng.hand_eye_vote([np.array([[0, 0, np.nan]] + [[1, 2, 3]] * 4)])
  q = np.array([[0, 1, 0, 0]], np.int32)
  rc = lib.mcba_hand_eye_quads(eng.h, 2, 5, 2, None, None, 1, q.ctypes.data_as(C.POINTER(C.c_int32)), None, None, None, None)
  assert rc == 1 and b"null pose table" in lib.mcba_last_error(eng.h)
  pd, vd = poses.ctypes.data_as(C.POINTER(C.c_double)), valid.astype(np.uint8).ctypes.data_as(C.POINTER(C.c_uint8))
  rc = lib.mcba_hand_eye_quads(eng.h, 2, 5, 2, pd, vd, 1, q.ctypes.data_as(C.POINTER(C.c_int32)), None, None, None, None)
  assert rc == 1 and b"null argument" in lib.mcba_last_error(eng.h)
  start = np.array([0, 5], np.int64)
  rc = lib.mcba_hand_eye_vote(eng.h, 1, start.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None)
  assert rc == 1 and b"null" in lib.mcba_last_error(eng.h)
  start = np.array([1, 5], np.int64)
  with pytest.raises(AssertionError, match="offsets"):
    eng._ck(lib.mcba_hand_eye_vote(eng.h, 1, start.ctypes.data_as(C.POINTER(C.c_int64)), None, None, None))
  X, Z, n, ok = eng.hand_eye_quads(poses, valid, np.zeros((0, 4), np.int32))
  assert X.shape == (0, 4, 4) and ok.shape == (0,)
