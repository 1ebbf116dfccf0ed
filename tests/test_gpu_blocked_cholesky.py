"""The blocked reduced solve (n_s > 127: 32-wide panels, each diagonal block factored and inverted by one warp in csrc/lm_kernel.cuh
chol_diag_warp_body) at the sizes where its last panel is padded with the identity: n_s = 129 (a last panel of 1 row), 146 (18 rows),
286 (30 rows: the shape of BASELINE cfg4) and 160 (whole panels).  The diagonal block is a loop over its 32 columns with the rows kept
rotated in registers; the padding rows are where its `k + 1 < nb` pivot test and the zeroed column tail matter.  The device's first step
is checked against the float64 model of oracle/trf_exact_model.py, and two identical solves must agree bit for bit.
tests/test_simt_blocked_cholesky.py runs the same checks on the SIMT interpreter."""
import numpy as np
import pytest

import test_gpu_step_parity as sp
from multical_b200 import synthetic

SHAPES = {   # n_s: (model, cameras, boards, enabled blocks) -- n_s = shared parameters of the Schur complement
  146: ("standard", 8, 3, dict(cameras=True)),        # 16 * 8 + 6 * 3: 5 panels, the last one of 18 rows
  286: ("standard", 16, 5, dict(cameras=True)),       # 16 * 16 + 6 * 5: 9 panels, the last one of 30 rows (cfg4's n_s)
}


def scene_of(n_s, F):
  model, C, B, opt = SHAPES[n_s]
  return synthetic.make_scene(C=C, F=F, vis=0.5, seed=29, model=model, rig="dome", boards=("cube", 4, 4, 0.06, B)), opt


def run_first_step(n_s, motion, F, num_sms):
  """(lm_grid, SYRK chunks) of the run; asserts the device's first step against the model."""
  fb = 12 if motion == "rolling" else 6
  scene, opt = scene_of(n_s, F)
  calib, prob = sp.static_or_rolling(scene, opt, motion=motion)
  eng, _ = sp.upload(calib, prob)
  assert eng.num_params - fb * F == n_s
  lm_grid, chunks = sp.lm_shape(F, n_s, fb, num_sms)
  sp.check_device_step(eng, f"n_s={n_s} FB={fb} F={F} (lm_grid {lm_grid}, SYRK chunks {chunks})")
  return lm_grid, chunks


def run_bit_reproducible(n_s, F):
  scene, opt = scene_of(n_s, F)
  calib, _ = sp.static_or_rolling(scene, opt)
  a, b = (calib.bundle_adjust(tolerance=1e-9, max_iterations=4) for _ in range(2))
  assert a.last_solve.cost == b.last_solve.cost
  assert np.array_equal(np.array(a.last_solve.log, float), np.array(b.last_solve.log, float), equal_nan=True)
  assert np.array_equal(a.param_vec, b.param_vec)


@pytest.mark.gpu
@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("n_s", sorted(SHAPES))
def test_first_step_of_the_blocked_reduced_solve(n_s, motion):
  """6 frames: an 8-CTA grid; 40 frames: the whole machine and several SYRK chunks."""
  import torch
  num_sms = torch.cuda.get_device_properties(0).multi_processor_count
  assert run_first_step(n_s, motion, 6, num_sms) == (8, 1)
  lm_grid, chunks = run_first_step(n_s, motion, 40, num_sms)
  assert lm_grid == num_sms and chunks > 1


@pytest.mark.gpu
def test_blocked_reduced_solve_is_bit_reproducible():
  run_bit_reproducible(286, 40)
