"""GPU (-m gpu): the pose-graph initialisation (multical_b200/tables.py initialise_poses; include/mcba.h mcba_pose_pairs, mcba_pose_times,
mcba_pose_cluster; csrc/pose_init_kernels.cuh) against the reference's own tables.initialise_poses (tests/golden/pose_init_*.npz,
tests/golden/make_pose_init_golden.py), against scipy's Ward clustering called live, and against oracle/pose_init_oracle.py at cfg4 size.

Bars: every align_transforms_robust call -- identical inlier mask, t within 1e-11 (rotation element-wise, translation relative);
initialise_poses -- camera, board and rig poses within the same bars, identical valid masks, masters and pairs; the largest Ward
cluster -- identical mask.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from multical_b200 import synthetic, tables
from multical_b200.calibration import get_engine
from multical_b200.structs import Table
from oracle import pose_init_oracle

pytestmark = pytest.mark.gpu

SCENES = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith("pose_init_") and f.endswith(".npz"))
SWITCH = 1024         # csrc/pose_init_kernels.cuh PI_SMALL_MAX: rows above it run on the large-item kernel
BAR = 1e-11


def golden(name):
  return dict(np.load(os.path.join(GOLDEN, name + ".npz")))


def assert_poses_close(got, ref):
  got, ref = np.asarray(got), np.asarray(ref)
  assert got.shape == ref.shape
  assert np.abs(got[..., :3, :3] - ref[..., :3, :3]).max(initial=0) <= BAR
  t, tr = got[..., :3, 3], ref[..., :3, 3]
  assert (np.abs(t - tr) <= BAR * np.maximum(1.0, np.abs(tr))).all()
  assert np.array_equal(got[..., 3, :], ref[..., 3, :])


def align(m1, m2, valid):
  """one align_transforms_robust call through mcba_pose_pairs: a two-camera table whose camera 0 holds m1 and camera 1 m2."""
  poses = np.stack([m1, m2])[:, :, None]
  ok = np.stack([valid, np.ones_like(valid)])[:, :, None]
  t, inl, n = get_engine().pose_pairs(poses, ok, 0, [(0, 1)])
  assert n[0] == inl[0].sum()
  return t[0], inl[0]


def run_recorded_calls(name):
  z = golden(name)
  for k in range(int(z["n_calls"])):
    t, inl = align(z[f"call_{k}_m1"], z[f"call_{k}_m2"], z[f"call_{k}_valid"])
    assert np.array_equal(inl, z[f"call_{k}_inliers"]), (name, k)
    assert_poses_close(t, z[f"call_{k}_t"])


def pose_table_of(z):
  return Table.create(poses=z["poses"], valid=z["valid"], num_points=z["num_points"])


def run_whole_function(name):
  z = golden(name)
  table = pose_table_of(z)
  out = tables.initialise_poses(table, camera_poses=z["camera_poses"] if z["has_camera_poses"] else None)
  for k in ("camera", "board", "times"):
    assert np.array_equal(out[k].valid, z[k + "_valid"]), k
    assert_poses_close(out[k].poses, z[k])
  assert np.array_equal(out.times.num_points, np.zeros(len(z["times"]))) and out.times.view_angles.shape == (len(z["times"]), 3)
  for axis, key in ((0, "camera"), (2, "board")):
    master, pairs = tables.select_pairs(tables.pattern_overlaps(z["valid"], z["num_points"], axis))
    assert master == int(z[key + "_master"]) and pairs == [tuple(p) for p in z[key + "_pairs"].tolist()]


def run_cluster_against_scipy(sizes, seed=0):
  rng = np.random.default_rng(seed)
  sets = [rng.normal(size=(n, 6)) * rng.uniform(0.2, 3.0, 6) + rng.normal(size=6) for n in sizes]
  for v, got in zip(sets, get_engine().pose_cluster(sets)):
    assert np.array_equal(got, pose_init_oracle.largest_cluster(v)), len(v)


def run_reproducible(name):
  z = golden(name)
  a = tables.initialise_poses(pose_table_of(z))
  b = tables.initialise_poses(pose_table_of(z))
  for k in ("camera", "board", "times"):
    assert np.array_equal(a[k].poses, b[k].poses) and np.array_equal(a[k].valid, b[k].valid)


@pytest.mark.parametrize("name", SCENES)
def test_every_align_call_matches_reference_golden(name):
  run_recorded_calls(name)


@pytest.mark.parametrize("name", SCENES)
def test_initialise_poses_matches_reference_golden(name):
  run_whole_function(name)


def test_largest_cluster_matches_scipy():
  run_cluster_against_scipy([2, 3, 29, 30, 31, SWITCH - 1, SWITCH, SWITCH + 1, 5000])


def test_full_size_matches_oracle():
  """cfg4 shape: 16 cameras x 1000 frames x 5 boards, half the views valid, 2 % outlier views."""
  poses, valid, npts, _ = synthetic.make_pose_table_scene(16, 1000, 5, 0.5, seed=40, outliers=0.02)
  out = tables.initialise_poses(Table.create(poses=poses, valid=valid, num_points=npts))
  ref = pose_init_oracle.initialise_poses(poses, valid, npts)
  for k in ("camera", "board", "times"):
    assert np.array_equal(out[k].valid, ref[k][1]), k
    assert_poses_close(out[k].poses, ref[k][0])


def test_bit_reproducible():
  run_reproducible("pose_init_large")


def test_whole_chain_from_detections():
  """cfg2-sized scene: intrinsics, pose table, pose graph and bundle adjustment all through this package; the final RMS lands at
  sigma sqrt(2) (tests/test_gpu_parity.py test_large_scene_properties)."""
  from multical_b200 import workspace
  from multical_b200.board import Board
  from test_gpu_intrinsics import detections
  scene = synthetic.make_workload("cfg2", seed=5)
  boards = [Board(p, size=(16, 22), min_points=20) for p in scene["board_points"]]
  dets = [detections(scene["points"][c], scene["valid"][c]) for c in range(scene["C"])]
  cams, _ = workspace.calibrate_single(boards, dets, [scene["image_size"]] * scene["C"], "standard", 1.0)
  table = Table.create(points=scene["points"], valid=scene["valid"])
  calib = workspace.initialise_poses(table, boards, cams)
  calib = workspace.calibrate(calib, cameras=True)
  rms = np.sqrt(np.mean(calib.reprojection_error ** 2))
  assert abs(rms - 0.3 * np.sqrt(2)) < 5e-3, rms


def test_bad_inputs():
  lib, eng = get_engine().lib, get_engine()
  poses, valid = np.broadcast_to(np.eye(4), (2, 3, 1, 4, 4)).copy(), np.ones((2, 3, 1), bool)
  with pytest.raises(AssertionError, match="dimensions"):
    eng.pose_pairs(np.zeros((0, 4, 4)), np.ones((0, 3, 1), bool), 0, [(0, 1)])
  with pytest.raises(AssertionError, match="out of range"):
    eng.pose_pairs(poses, valid, 0, [(0, 2)])
  with pytest.raises(AssertionError, match="out of range"):
    eng.pose_pairs(poses, valid, 0, [(1, 1)])
  with pytest.raises(AssertionError, match="axis"):
    eng.pose_pairs(poses, valid, 1, [(0, 1)])
  bad = poses.copy(); bad[0, 0, 0, 0, 0] = np.nan
  with pytest.raises(ValueError, match="non-finite"):
    eng.pose_pairs(bad, valid, 0, [(0, 1)])
  import ctypes as C
  t, inl, n = np.zeros((1, 4, 4)), np.zeros((1, 3), np.uint8), np.zeros(1, np.int32)
  pairs = np.array([[0, 1]], np.int32)
  rc = lib.mcba_pose_pairs(eng.h, 2, 3, 1, None, None, 0, pairs.ctypes.data_as(C.POINTER(C.c_int32)), 1, t.ctypes.data_as(C.POINTER(C.c_double)),
                           inl.ctypes.data_as(C.POINTER(C.c_uint8)), n.ctypes.data_as(C.POINTER(C.c_int32)))
  assert rc == 1 and b"null pose table" in lib.mcba_last_error(eng.h)
  rc = lib.mcba_pose_times(eng.h, 2, 3, 1, None, None, None, None, None, None, None, None)
  assert rc == 1 and b"null pose table" in lib.mcba_last_error(eng.h)
  with pytest.raises(AssertionError, match="offsets"):
    lib_start = np.array([1, 2], np.int64)
    eng._ck(lib.mcba_pose_cluster(eng.h, 1, lib_start.ctypes.data_as(C.POINTER(C.c_int64)), None, None))
