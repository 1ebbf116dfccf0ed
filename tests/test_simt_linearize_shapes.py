"""CPU (-m "not gpu"): the launch shapes of k_linearize and its cheap shape cases on the SIMT interpreter (tests/simt), with the bodies
of tests/test_gpu_linearize_shapes.py -- imported, not copied.

  restatement   lin_shape's shared-memory formula against the kernel's own (lin_smem_doubles of csrc/linearize.cuh, compiled for the
                host by tests/host_math), the documented board limits, the scatter-offset bound, the board counts the warp scoring
                used to refuse
  acceptance    every board count up to the limit is accepted by the real host driver, the next one is refused
  shapes        normal equations and first step at the views / boards staged and unstaged, split views, the other models, rolling
                and hand-eye frames, board points, and CTAs that own several frames (one SM)
"""
import pytest

import test_gpu_linearize_shapes as ls
from multical_b200 import _native, calibration
from test_device_math_on_host import hm  # noqa: F401  (fixture)

MODEL_IDS = {"standard": 0, "rational": 1, "thin_prism": 2, "fisheye": 3, "tilted": 4}


@pytest.fixture(scope="session")
def simt_library():
  import simt
  return simt.build()


@pytest.fixture
def on_the_interpreter(simt_library, monkeypatch):
  """Point the ctypes binding at the interpreter build for one test; engines are per-library, so the cache is swapped as well."""
  monkeypatch.setattr(_native, "LIB_PATH", simt_library)
  monkeypatch.setattr(_native, "_lib", None)
  monkeypatch.setattr(_native, "_allow_interpreter", True)
  monkeypatch.setattr(calibration, "_engines", {})
  monkeypatch.delenv("SIMT_SMS", raising=False)
  yield
  for eng in calibration._engines.values(): eng.close()


# ---------------------------------------------------------------------------------------------------------------- restatement
def test_launch_shape_restatement_matches_the_kernel(hm):
  """lin_smem_doubles for every model x motion x warps x board count 1..400 equals the kernel's; the documented limits (DESIGN.md §3b)
  hold; every accepted shape keeps a warp's slice below LIN_WB_FLAG; acceptance is monotone in the board count at every split; the
  former holes are accepted now with fewer warps, where the best-scoring warp count needs more than LIN_SMEM_MAX but less than an SM
  can hold beside the reserve."""
  for model, mid in MODEL_IDS.items():
    for roll in (False, True):
      for warps in (8, 4, 2):
        for B in range(1, 401):
          assert hm.hm_lin_smem_doubles(mid, int(roll), B, warps) == ls.lin_smem_doubles(model, roll, B, warps), (model, roll, warps, B)
      for C in (1, 2, 3, 5, 12):
        accepted = [ls.lin_shape(model, roll, C, B, 132)[4] for B in range(1, 401)]
        limit = accepted.index(False)
        assert not any(accepted[limit:]), (model, roll, C)                                    # no hole below the limit
        for B in range(1, limit + 1):
          split, warps, smem, _, _ = ls.lin_shape(model, roll, C, B, 132)
          assert smem <= ls.LIN_SMEM_MAX and ls.lin_warp_doubles(model, roll, B) < ls.LIN_WB_FLAG
          assert warps == 8 or split == 1
      assert ls.board_limit(model, roll, 5) == ls.BOARD_LIMITS[model][roll]
      assert ls.board_limit(model, roll, 2) == ls.BOARD_LIMITS[model][2 + roll]
      for B in ls.FORMER_HOLES[model][roll]:
        _, warps, smem, _, ok = ls.lin_shape(model, roll, 5, B, 132)
        over = [w for w in (8, 4, 2) if w > warps and ls.LIN_SMEM_MAX < 8 * ls.lin_smem_doubles(model, roll, B, w) <= ls.SM_SHARED - ls.CTA_RESERVE]
        assert ok and over, (model, roll, B, warps)
  assert [ls.BOARD_LIMITS[m][0] for m in ("standard", "tilted")] == [354, 330]
  assert [ls.BOARD_LIMITS[m][2] for m in ("standard", "tilted")] == [63, 39]


# ---------------------------------------------------------------------------------------------------------------- acceptance
@pytest.mark.parametrize("C", [2, 5])
@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("model", sorted(MODEL_IDS))
def test_every_board_count_up_to_the_limit_is_accepted(model, motion, C, on_the_interpreter):
  limit = ls.run_acceptance_scan(model, motion, C)
  assert limit == ls.BOARD_LIMITS[model][(motion == "rolling") + (2 if C == 2 else 0)]


# ---------------------------------------------------------------------------------------------------------------- shapes
# "both unstaged, 96 / 97 / 108" runs as tests/test_simt_kernels.py::test_more_views_per_frame_and_more_boards_than_the_staged_tables_hold
INTERPRETER_SHAPES = [n for n in ls.SHAPES if n not in ("both unstaged, 96 / 97 / 108", "a former hole")]


@pytest.mark.parametrize("name", INTERPRETER_SHAPES)
def test_normal_equations_and_first_step_at_each_path(name, on_the_interpreter):
  ls.run_shape(name, 132)


def test_hand_eye_with_unstaged_boards(on_the_interpreter):
  ls.run_hand_eye_unstaged_boards(132)


def test_board_points_with_unstaged_boards(on_the_interpreter):
  ls.run_board_points_unstaged_boards(132)


def test_ctas_that_own_several_frames_with_unstaged_tables(on_the_interpreter, monkeypatch):
  """One SM: F = 2 x 4 + 3 = 11 frames over 4 CTAs of 4 warps (set before the first engine of the test is created)."""
  monkeypatch.setenv("SIMT_SMS", "1")
  assert ls.run_frames_per_cta_unstaged(1) == 4


def test_two_identical_linearisations_and_solves_agree_bit_for_bit(on_the_interpreter):
  ls.run_bit_reproducibility()
