"""CPU (-m "not gpu"): the checks of tests/test_gpu_triangulate.py on the SIMT interpreter (tests/simt) at small sizes, and the oracle's
linear solution against live cv2.triangulatePoints."""
import numpy as np
import pytest

import test_gpu_triangulate as gt
from multical_b200 import undistort
from oracle import triangulate_oracle as to
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)


@pytest.fixture(autouse=True)
def fresh_undistort_engines(on_the_interpreter, monkeypatch):  # noqa: F811
  monkeypatch.setattr(undistort, "_engines", {})
  yield
  for eng in undistort._engines.values(): eng.close()


def test_oracle_linear_is_cv2():
  import cv2
  for kind in ("horizontal", "narrow"):
    P1, P2, x1, x2 = gt.linear_pair(kind, 50)
    ours, ref = to.triangulate_linear(P1, P2, x1, x2), cv2.triangulatePoints(P1, P2, x1, x2)
    assert np.allclose(ours[:3] / ours[3], ref[:3] / ref[3], rtol=1e-9, atol=0)


def test_linear_matches_cv2_triangulate_points():
  gt.run_linear([1, 257])


def test_noise_free_recovery_all_models():
  gt.run_noise_free(F=1)


@pytest.mark.parametrize("model", gt.MODELS)
def test_refined_points_match_the_oracle(model):
  gt.run_oracle_parity([model], Cs=(2, 3, 7, 33), F=1, n=40)


def test_validity():
  gt.run_validity()


def test_refusals():
  gt.run_errors()


def test_calibration_triangulate():
  gt.run_calibration(F=2, ba_F=4)


def test_repeated_calls_agree_bit_for_bit():
  gt.run_reproducible(Cs=(3, 40), F=1)
