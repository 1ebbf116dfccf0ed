"""CPU (-m "not gpu"): the fixed-parameter calibration flags of tests/test_gpu_intrinsic_flags.py on the SIMT interpreter (tests/simt), at
the small sizes the interpreter runs in seconds: the engine's mask, one pinhole and one fisheye flag case against OpenCV on the host, and
the refusals.  The real kernels and host driver, the same bars."""
import pytest

import test_gpu_intrinsic_flags as gfl
from multical_b200 import intrinsics
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_intrinsics_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(intrinsics, "_engines", {})
  yield
  for eng in intrinsics._engines.values(): eng.close()


@pytest.mark.parametrize("boards", [False, True])
def test_mask_zeroes_the_rows_and_columns_of_the_normal_equations(boards):
  gfl.run_engine_linearisation(boards)


def test_masked_solves_hold_the_fixed_parameters_and_the_next_upload_clears_the_mask():
  gfl.run_engine_solves()


def test_mask_arguments():
  gfl.run_mask_arguments()


def test_pinhole_fix_k3_and_zero_tangent_dist_matches_opencv():
  gfl.run_pinhole("FIX_K3|ZERO_TANGENT_DIST", 20)


def test_fisheye_fix_k3_and_k4_matches_opencv():
  gfl.run_fisheye("FIX_K3|FIX_K4", 20)


test_refused_flags_name_the_flag = gfl.test_refused_flags_name_the_flag
