"""CPU (-m "not gpu"): the blocked reduced solve (n_s > 127: 32-wide panels, each diagonal block factored and inverted by one warp in
csrc/lm_kernel.cuh chol_diag_warp_body) on the SIMT interpreter.  The diagonal block is a loop over its 32 columns with the rows kept
rotated in registers; these sizes put ragged last panels (n_s = 129, 146, 286: 1, 18 and 30 rows, the rest padded with the identity)
and whole panels (n_s = 160) through it, at frames of 6 (static) and 12 (rolling) parameters.  The first step is checked against the
float64 model of oracle/trf_exact_model.py, and two identical solves must agree bit for bit (tests/test_gpu_blocked_cholesky.py)."""
import pytest

import test_gpu_blocked_cholesky as bc
import test_gpu_step_parity as sp
from multical_b200 import _native, calibration


@pytest.fixture(autouse=True)
def on_the_interpreter(monkeypatch):
  import simt                     # tests/simt/__init__.py
  monkeypatch.setattr(_native, "LIB_PATH", simt.build())
  monkeypatch.setattr(_native, "_lib", None)
  monkeypatch.setattr(_native, "_allow_interpreter", True)
  monkeypatch.setattr(calibration, "_engines", {})
  monkeypatch.delenv("SIMT_SMS", raising=False)
  yield
  for eng in calibration._engines.values(): eng.close()


@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("n_s", [129, 160])
def test_first_step_of_the_blocked_reduced_solve(n_s, motion):
  assert sp.run_reduced_solve(n_s, motion, 6, 132) == (8, 1)


@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("n_s", sorted(bc.SHAPES))
def test_first_step_with_a_ragged_last_panel(n_s, motion):
  assert bc.run_first_step(n_s, motion, 6, 132) == (8, 1)


def test_blocked_reduced_solve_at_cfg4s_size_is_bit_reproducible():
  bc.run_bit_reproducible(286, 6)

