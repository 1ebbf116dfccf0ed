"""CPU (-m "not gpu"): the pose-graph initialisation of tests/test_gpu_pose_init.py on the SIMT interpreter (tests/simt) at the sizes it
runs in seconds -- the small-item and large-item kernels and the host driver, the same bars -- and oracle/pose_init_oracle.py against
the reference's goldens."""
import numpy as np
import pytest

import test_gpu_pose_init as gp
from oracle import pose_init_oracle
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)

SMALL = [s for s in gp.SCENES if s != "pose_init_large"]


def test_oracle_matches_reference_golden():
  for name in gp.SCENES:
    z = gp.golden(name)
    o = pose_init_oracle.initialise_poses(z["poses"], z["valid"], z["num_points"], z["camera_poses"] if z["has_camera_poses"] else None)
    for k in ("camera", "board", "times"):
      assert np.array_equal(o[k][1], z[k + "_valid"]) and np.abs(o[k][0] - z[k]).max() < 1e-12, (name, k)
    for k in range(int(z["n_calls"])):
      t, inl = pose_init_oracle.align_transforms_robust(z[f"call_{k}_m1"], z[f"call_{k}_m2"], z[f"call_{k}_valid"])
      assert np.array_equal(inl, z[f"call_{k}_inliers"]) and np.abs(t - z[f"call_{k}_t"]).max() < 1e-12, (name, k)


@pytest.mark.parametrize("name", ["pose_init_outliers", "pose_init_dead_camera", "pose_init_large"])
def test_every_align_call_matches_reference_golden(name):
  gp.run_recorded_calls(name)


@pytest.mark.parametrize("name", SMALL)
def test_initialise_poses_matches_reference_golden(name):
  gp.run_whole_function(name)


def test_largest_cluster_matches_scipy_on_both_sides_of_the_switch():
  gp.run_cluster_against_scipy([2, 3, 4, 29, 30, 31, 200, gp.SWITCH - 1, gp.SWITCH, gp.SWITCH + 1])


def test_bit_reproducible():
  gp.run_reproducible("pose_init_cube")


test_bad_inputs = gp.test_bad_inputs
