"""CPU (-m "not gpu"): the stereo calibration of tests/test_gpu_stereo.py on the SIMT interpreter (tests/simt), at the small sizes the
interpreter runs in seconds: the start against the oracle at an odd and an even view count, one converged case per camera family at 12
views, and the refusals that stop before the solve.  The real kernels and host driver, the same bars."""
import pytest

import test_gpu_stereo as gs
from multical_b200 import intrinsics
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_intrinsics_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(intrinsics, "_engines", {})
  yield
  for eng in intrinsics._engines.values(): eng.close()


@pytest.mark.parametrize("F", [11, 12])
def test_start_is_the_median_relative_pose(F):
  gs.run_start(F)


@pytest.mark.parametrize("model", ["standard", "fisheye"])
def test_converged_solution_matches_opencv(model):
  gs.run_converged(model, True, 12)
