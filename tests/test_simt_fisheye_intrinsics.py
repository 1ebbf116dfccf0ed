"""CPU (-m "not gpu"): the fisheye intrinsic calibration of tests/test_gpu_fisheye_intrinsics.py on the SIMT interpreter (tests/simt), at
the small sizes the interpreter runs in seconds: 1-2 cameras, at most 20 views each.  The real kernels and host driver, the same bars."""
import pytest

import test_gpu_fisheye_intrinsics as gf
from multical_b200 import intrinsics
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_intrinsics_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(intrinsics, "_engines", {})
  yield
  for eng in intrinsics._engines.values(): eng.close()


def test_initial_camera_matrix_and_poses_are_opencvs():
  gf.run_init(2, 10)


@pytest.mark.parametrize("case", ["plain", "cube"])
def test_converged_solution_matches_opencv(case):
  gf.run_converged(case, 4 if case == "cube" else 20)


def test_calibrate_matches_reference_golden():
  gf.run_golden("fisheye_small_12")


def test_returned_object_and_errors():
  gf.run_returned_object_and_errors(8)


def test_batched_cameras_and_bit_reproducible():
  gf.run_batched_and_reproducible(2, 8)


def test_wide_angle_scene_where_opencv_fails_on_some_hosts():
  gf.run_wide_angle(20)
