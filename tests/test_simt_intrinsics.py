"""CPU (-m "not gpu"): the intrinsic calibration of tests/test_gpu_intrinsics.py on the SIMT interpreter (tests/simt), at the small sizes
the interpreter runs in seconds: 1-2 cameras, at most 20 views each.  The real kernels and host driver, the same bars."""
import pytest

import test_gpu_intrinsics as gi
from multical_b200 import intrinsics
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_intrinsics_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(intrinsics, "_engines", {})
  yield
  for eng in intrinsics._engines.values(): eng.close()


@pytest.mark.parametrize("fix_aspect", [False, True])
def test_initial_camera_matrix_is_initIntrinsicParams2D(fix_aspect):
  gi.run_init(2, 14, fix_aspect)


@pytest.mark.parametrize("case", ["standard", "fix_aspect", "cube"])
def test_converged_solution_matches_opencv(case):
  gi.run_converged(case, 4 if case == "cube" else 20)


def test_calibrate_loop_below_fifteen_views_matches_reference_golden(monkeypatch):
  gi.run_golden("intrinsics_small_12", monkeypatch)


test_unsupported_models_non_planar_boards_and_cameras_without_views = gi.test_unsupported_models_non_planar_boards_and_cameras_without_views


def test_batched_cameras_and_bit_reproducible():
  gi.run_batched_and_reproducible(2, 12)


@pytest.mark.parametrize("motion", ["static", "rolling"])
def test_view_errors_of_a_bundle_adjustment(motion):
  gi.run_view_errors_of_a_bundle_adjustment(motion)
