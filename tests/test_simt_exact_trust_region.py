"""CPU (-m "not gpu"): the exact trust-region step (`bundle_adjust(tr_solver="exact")`, the alpha search inside k_lm) on the SIMT
interpreter, with the assertions of tests/test_gpu_exact_trust_region.py on its small scenes: step parity with scipy's
tr_solver='exact' without gauge freedom (static and rolling frames, a robust loss), the converged cost with gauge freedom, two identical
exact solves bit for bit and the default solve untouched by an exact one, and exact mode refused on two ranks."""
import pytest

import test_gpu_exact_trust_region as et
import test_gpu_parity as gp
import test_simt_multirank as mr
from multical_b200 import _native, calibration


@pytest.fixture(autouse=True)
def on_the_interpreter(monkeypatch):
  import simt                     # tests/simt/__init__.py
  monkeypatch.setattr(_native, "LIB_PATH", simt.build())
  monkeypatch.setattr(_native, "_lib", None)
  monkeypatch.setattr(_native, "_allow_interpreter", True)
  monkeypatch.setattr(calibration, "_engines", {})
  yield
  for eng in calibration._engines.values(): eng.close()


@pytest.mark.parametrize("name", ["standard_2x6", "rolling_2x6"])
def test_step_parity_with_scipy_exact(name):
  et.run_step_parity(name)


def test_step_parity_with_a_robust_loss():
  et.run_step_parity("standard_2x6", loss="soft_l1", f_scale=1000.0)


def test_converged_solution_with_gauge_freedom_matches_scipy_exact():
  et.run_gauge_parity("standard_2x6")


def test_exact_solves_are_bit_reproducible_and_leave_the_default_alone():
  et.run_isolation("standard_2x6", max_iterations=12)


def test_exact_mode_on_two_ranks_is_refused(monkeypatch):
  scene, z, calib, prob = gp.make("standard_2x6")
  with pytest.raises(AssertionError, match="NotImplementedError"):
    mr.sharded_solve(calib, 2, True, monkeypatch, tr_solver="exact")
