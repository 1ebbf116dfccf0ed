"""CPU (-m "not gpu"): the exact trust-region step at the paths of k_lm (tests/test_gpu_exact_paths.py) on the SIMT interpreter:
the blocked reduced solve at n_s = 129 and 160 with static and rolling frames on an 8-CTA grid, two SYRK frame chunks on a 32-SM
machine, the full-rank blocked probe and its alpha search after rejected trials (one and two SYRK frame chunks), hand-eye frames
beyond one fold batch, and the degenerate block selections.  Each first step against oracle/trf_exact_model.py `exact_first_step` on
the device's own normal equations."""
import pytest

import test_gpu_exact_paths as ep
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
def test_exact_step_at_the_blocked_reduced_solve(n_s, motion):
  lm_grid, chunks, m = ep.run_reduced_path(n_s, motion, 6, 132)
  assert (lm_grid, chunks) == (8, 1) and not m.full_rank


def test_exact_step_with_several_syrk_chunks(monkeypatch):
  """A 32-SM machine, 40 frames at n_s = 129: F * n_s >= 4096 puts k_lm on all 32 CTAs, 15 tile pairs of the SYRK leave room for
  two frame chunks (set before the first engine of the test is created)."""
  monkeypatch.setenv("SIMT_SMS", "32")
  assert ep.run_reduced_path(129, "static", 40, 32)[:2] == (32, 2)


def test_exact_step_with_hand_eye_frames_beyond_one_fold_batch():
  ep.run_hand_eye(70)


@pytest.mark.parametrize("opt", ep.DEGENERATE)
def test_exact_step_at_degenerate_block_selections(opt):
  ep.run_degenerate(opt)


def test_full_rank_blocked_probe_takes_the_gauss_newton_step():
  ep.run_full_rank_blocked(6, 132)


def test_full_rank_blocked_alpha_search():
  assert ep.run_full_rank_search(6, 132) == (8, 1)


def test_full_rank_blocked_alpha_search_with_several_syrk_chunks(monkeypatch):
  """A 32-SM machine, 40 frames at n_s = 130: k_lm on all 32 CTAs, two SYRK frame chunks."""
  monkeypatch.setenv("SIMT_SMS", "32")
  assert ep.run_full_rank_search(40, 32) == (32, 2)
