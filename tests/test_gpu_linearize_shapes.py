"""GPU (-m gpu): k_linearize on the paths that the problem's shape selects, against float64 references, and the host's choice of
launch shape at every board count it accepts.

k_linearize (csrc/linearize.cuh) stages a frame's view list in shared memory up to LIN_MAXV = 96 views and reads it from global memory
beyond; it bulk-copies the board pose tables into shared memory up to LIN_MAXB = 8 boards and reads `board_T` beyond; it runs 8, 4 or 2
warps per CTA as the host scores them (csrc/solver.cu setup_problem).  A warp's shared-memory slice grows with the board count, so the
board count also decides how close a CTA comes to the 220 KB of dynamic shared memory it may take, and how large the scatter offsets
of the epilogue grow (int16 tables whose bit LIN_WB_FLAG marks a board-row entry).

  lin_shape        the host's choice restated: split, warps, shared memory, grid, accepted (tests/test_simt_linearize_shapes.py checks
                   its shared-memory formula against the kernel's own through tests/host_math)
  acceptance       every board count up to the limit of its (model, motion, split) is accepted, the next one is refused
  normal equations J^T J, J^T r, cost against fourth-order differences of the oracle, and the first trust-region step against the
                   model, at the bars of tests/test_gpu_step_parity.py, on scenes that take each path

The test bodies take the device's SM count as an argument so that tests/test_simt_linearize_shapes.py runs the cheap shapes on the
interpreter with the same code.
"""
import numpy as np
import pytest

from multical_b200 import synthetic
from multical_b200._native import MOTION_ROLLING, OPT_BITS
from oracle.ba_oracle import Problem
from oracle.trf_exact_model import first_step
from test_gpu_step_parity import (check_normal_equations, check_step, device_first_step, fd5_jacobian, hand_eye,
                                  lin_split, static_or_rolling, upload)

pytestmark = pytest.mark.gpu

MODEL_ND = {"standard": 5, "rational": 8, "thin_prism": 12, "fisheye": 4, "tilted": 14}
LIN_MAXV, LIN_MAXB = 96, 8
LIN_SMEM_MAX = 220 * 1024         # bytes of dynamic shared memory a k_linearize CTA may take
LIN_WB_FLAG = 0x4000              # scatter-table flag: offsets within a warp's slice must stay below it
SM_SHARED, CTA_RESERVE = 227 * 1024, 4 * 1024


# ---------------------------------------------------------------------------------------------------------------- launch shape
def lin_warp_doubles(model, roll, B):
  """Doubles of one warp's shared-memory slice (csrc/linearize.cuh lin_warp_doubles): stage buffer | twist maps | chain | board rows of
  W_f | H_ff, g_f | camera rows of W_f | moment sum | board coupling | tail | view constants."""
  NP = 2 if roll else 1
  KO = FB = 6 * NP
  D = KO + 4 + MODEL_ND[model]
  T = D * (D + 1) // 2 + D + 1
  NC = -(-(D + 1) // 8) * 8
  PT = -(-6 * (NP + 1) // 8)
  EK = 4 * -(-KO // 4)
  EP, MR = 8 * PT + 4, 8 * -(-EK // 8)
  stage = (max(NC * 36, MR * (NC + 4) + 8 * PT * 12) + 1) & ~1
  return (stage + EK * EP + 12 * NP + B * 6 * FB + FB * FB + FB + D * FB + T + (D * 6 + 42) + 6 + 44 + 1) & ~1


def lin_smem_doubles(model, roll, B, warps):
  """Doubles of a CTA's dynamic shared memory: the warps' slices, the frame table twice (double buffer) and the staged board tables."""
  NP = 2 if roll else 1
  return warps * lin_warp_doubles(model, roll, B) + 24 * (2 * NP + min(B, LIN_MAXB))


def lin_shape(model, roll, C, B, num_sms, F=None):
  """(split, warps, smem_bytes, grid, accepted) of k_linearize as the host driver picks them (csrc/solver.cu setup_problem).  With
  `split` > 1 the CTA has 8 warps.  Else the warp count in {8, 4, 2} whose CTA fits LIN_SMEM_MAX and scores highest: resident warps
  per SM (227 KB less 4 KB per CTA, 16 warps of registers) times how evenly the cameras spread over the warps; ties go to more warps.
  grid: the CTAs resident at once (num_sms x CTAs per SM), or with F the smallest grid that keeps every CTA at ceil(F / that) frames."""
  split = lin_split(C)
  warps = 8
  if split == 1:
    best = -1.0
    for wc in (8, 4, 2):
      smem = 8 * lin_smem_doubles(model, roll, B, wc)
      if smem > LIN_SMEM_MAX: continue
      occ = min(SM_SHARED // (smem + CTA_RESERVE), 16 // wc)
      if occ < 1: continue
      score = occ * wc * C / (-(-C // wc) * wc)
      if score > best + 1e-9: best, warps = score, wc
  smem = 8 * lin_smem_doubles(model, roll, B, warps)
  grid = num_sms * max(1, min(SM_SHARED // (smem + CTA_RESERVE), 16 // warps))
  if F is not None:
    per = -(-max(F, 1) // grid)
    grid = -(-max(F, 1) // per)
  return split, warps, smem, grid, smem <= LIN_SMEM_MAX


def board_limit(model, roll, C):
  """The largest board count lin_shape accepts for the rig's split."""
  B = 1
  while lin_shape(model, roll, C, B + 1, 132)[4]: B += 1
  return B


# static / rolling board limits with 5 cameras or more (split 1) and with 2 cameras (split 4: 8 warps)
BOARD_LIMITS = {"standard": (354, 164, 63, 19), "rational": (344, 158, 53, 13), "thin_prism": (340, 156, 49, 10),
                "tilted": (330, 154, 39, 9), "fisheye": (355, 164, 64, 19)}
# board counts that the warp scoring refused before it skipped CTAs over LIN_SMEM_MAX (5 cameras; static, rolling)
FORMER_HOLES = {"standard": ([64, 65, 161, 162, 163], [68]), "rational": ([54, 151, 152], [14, 62, 63]),
                "thin_prism": ([50, 147, 148, 149], [11, 60]), "tilted": ([40, 137, 138, 139], [10, 58, 59]),
                "fisheye": ([65, 162, 163, 164], [20, 69])}


# ---------------------------------------------------------------------------------------------------------------- acceptance
def run_acceptance_scan(model, motion, C):
  """One minimal problem (one frame, one corner per camera on the last board) per board count from 1 to the limit, and one past it:
  every count up to the limit is accepted, the next is refused.  Returns the limit."""
  from multical_b200.calibration import get_engine
  roll = motion == "rolling"
  limit = board_limit(model, roll, C)
  eng = get_engine()
  bits = OPT_BITS["cameras"] | (MOTION_ROLLING if roll else 0)
  obs = np.tile([[960.0, 540.0]], (C, 1))
  for B in range(1, limit + 2):
    idx = np.array([[c, 0, B - 1, 0] for c in range(C)])
    bp = np.zeros((B, 1, 3))
    if B <= limit:
      eng.upload(model, bits, (C, 1, B, 1), idx, obs, bp)
    else:
      with pytest.raises(NotImplementedError, match="too many boards"):
        eng.upload(model, bits, (C, 1, B, 1), idx, obs, bp)
  return limit


@pytest.mark.parametrize("C", [2, 5])
@pytest.mark.parametrize("motion", ["static", "rolling"])
@pytest.mark.parametrize("model", sorted(MODEL_ND))
def test_every_board_count_up_to_the_limit_is_accepted(model, motion, C):
  """5 cameras: split 1, the host chooses the warp count; 2 cameras: split 4, 8 warps."""
  limit = run_acceptance_scan(model, motion, C)
  assert limit == BOARD_LIMITS[model][(motion == "rolling") + (2 if C == 2 else 0)]


# ---------------------------------------------------------------------------------------------------------------- scenes
def tiles_scene(C, B, F=3, views=None, model="standard", seed=41, extent=0.4):
  """C cameras on an arc, B boards of 4 x 3 corners on a near-square grid `extent` metres wide, every (camera, frame, board) view
  present.  views: per frame, the views to keep; the others are dropped round the cameras, view (c, (c + f + k) % B) for k = 0, 1, ..."""
  cols = int(np.ceil(np.sqrt(B)))
  square = extent / (cols * 1.1 * 5)
  scene = synthetic.make_scene(C=C, F=F, vis=1.0, seed=seed, model=model, boards=("tiles", 5, 4, square, B))
  valid = scene["valid"]
  assert valid.any(axis=-1).all(), "a view of the tiles scene is out of the image"
  for f, n in enumerate(views or []):
    drop, k = C * B - n, 0
    while drop > 0:
      for c in range(C):
        if drop == 0: break
        b = (c + f + k) % B
        if valid[c, f, b].any(): valid[c, f, b] = False; drop -= 1
      k += 1
  return scene


def views_per_frame(calib):
  return [int(n) for n in np.asarray(calib.inliers).any(axis=-1).sum(axis=(0, 2))]


def expect_shape(scene, motion, warps, split, num_sms, views=None):
  """Asserts the launch shape (split, warps, views staged per frame, boards staged) the case claims, and the exact view count of every
  frame; returns a label."""
  C, B, F = scene["C"], scene["B"], scene["F"]
  s, w, smem, grid, ok = lin_shape(scene["model"], motion == "rolling", C, B, num_sms, F)
  assert ok and (s, w) == (split, warps), (s, w, split, warps)
  per_frame = [int(n) for n in scene["valid"].any(axis=-1).sum(axis=(0, 2))]
  if views is not None: assert per_frame == list(views), per_frame
  staged = ["staged" if n <= LIN_MAXV else "global" for n in per_frame]
  shown = per_frame if F <= 6 else f"{min(per_frame)}..{max(per_frame)}"
  return (f"{scene['model']} {motion} {C}x{B} F={F} views {shown} ({'/'.join(sorted(set(staged)))}) "
          f"boards {'staged' if B <= LIN_MAXB else 'global'} split {s} warps {w} smem {smem} bytes, grid {grid}")


def check_case(scene, opt, motion, warps, split, num_sms, views=None):
  import time
  label = expect_shape(scene, motion, warps, split, num_sms, views)
  calib, prob = static_or_rolling(scene, opt, motion=motion)
  assert views is None or views_per_frame(calib) == list(views)
  eng, x0 = upload(calib, prob)
  assert np.abs(eng.residuals(x0) - prob.residuals(x0)).max() < 1e-9
  JtJ, Jtr, cost = eng.linearize()
  t0 = time.perf_counter()
  J = fd5_jacobian(prob, x0)
  print(f"[fd5_jacobian] {label}: {time.perf_counter() - t0:.1f} s for {J.shape[1]} columns")
  check_normal_equations(JtJ, Jtr, cost, J, prob.residuals(x0), label)
  check_step(device_first_step(eng)[0], first_step(JtJ, Jtr, eng.param_vec), label)
  return eng


# (C, B, views per frame or None for all, model, motion, split, warps)
SHAPES = {
  "both staged, at both limits": (12, 8, (96, 96, 96), "standard", "static", 1, 4),
  "views unstaged": (13, 8, (104, 104, 104), "standard", "static", 1, 8),
  "boards unstaged": (5, 9, (45, 45, 45), "standard", "static", 1, 2),
  "both unstaged, 96 / 97 / 108": (12, 9, (96, 97, 108), "standard", "static", 1, 4),
  "split 4, views unstaged": (2, 49, (96, 97, 98), "standard", "static", 4, 8),
  "split 2, views unstaged": (4, 25, (96, 97, 100), "standard", "static", 2, 8),
  "fisheye": (12, 9, (108, 108, 108), "fisheye", "static", 1, 4),
  "tilted": (12, 9, (108, 108, 108), "tilted", "static", 1, 2),
  "rolling": (12, 9, (108, 108, 108), "standard", "rolling", 1, 4),
  "a former hole": (5, 64, None, "standard", "static", 1, 2),
}
LIMIT_SHAPES = {"static at the limit": (5, 354, None, "standard", "static", 1, 2),
                "rolling at the limit": (5, 164, None, "standard", "rolling", 1, 2)}


def run_shape(name, num_sms, table=SHAPES):
  C, B, views, model, motion, split, warps = table[name]
  # fisheye: a target 1 m wide, so that the k4 columns (theta^9) stand well above the round-off of the differences (0.4 m: 8e-9)
  scene = tiles_scene(C, B, views=views, model=model, extent=1.0 if model == "fisheye" else 0.4)
  return check_case(scene, dict(cameras=True), motion, warps, split, num_sms, views)


def gpu_sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("name", list(SHAPES))
def test_normal_equations_and_first_step_at_each_path(name):
  run_shape(name, gpu_sms())


@pytest.mark.parametrize("name", list(LIMIT_SHAPES))
def test_normal_equations_and_first_step_at_the_board_limit(name):
  """The largest board count of standard static and rolling frames: a CTA of 2 warps within 400 B of LIN_SMEM_MAX, scatter offsets at
  their largest."""
  C, B, _, model, motion, _, _ = LIMIT_SHAPES[name]
  split, warps, smem, _, ok = lin_shape(model, motion == "rolling", C, B, 132)
  assert ok and B == board_limit(model, motion == "rolling", C) and LIN_SMEM_MAX - smem < 400
  assert lin_warp_doubles(model, motion == "rolling", B) < LIN_WB_FLAG
  run_shape(name, gpu_sms(), LIMIT_SHAPES)


def run_hand_eye_unstaged_boards(num_sms):
  """5 cameras x 9 boards, hand-eye frames with the camera poses fixed and the hand-eye transforms free: the board rows of W_f come from
  board tables read from global memory and go through k_fold_hand_eye."""
  scene = tiles_scene(5, 9)
  label = expect_shape(scene, "static", 2, 1, num_sms, (45, 45, 45))
  calib, prob = hand_eye(scene, dict(camera_poses=False, cameras=True))
  eng, x0 = upload(calib, prob)
  JtJ, Jtr, cost = eng.linearize()
  check_normal_equations(JtJ, Jtr, cost, fd5_jacobian(prob, x0), prob.residuals(x0), "hand-eye " + label)
  check_step(device_first_step(eng)[0], first_step(JtJ, Jtr, eng.param_vec), "hand-eye " + label)


def test_hand_eye_with_unstaged_boards():
  run_hand_eye_unstaged_boards(gpu_sms())


def run_board_points_unstaged_boards(num_sms):
  """5 cameras x 9 boards with the board points free: W_f is zero-filled first (fill_all) and k_point_blocks adds the point rows.  The
  engine holds a slot per (board, point) of the padded table; the oracle has columns for the valid points only."""
  from multical_b200.calibration import from_scene
  scene = tiles_scene(5, 9)
  label = "board points " + expect_shape(scene, "static", 2, 1, num_sms, (45, 45, 45))
  opt = dict(cameras=True, boards=True)
  calib = from_scene(scene).enable(**opt)
  prob = Problem.from_scene(scene, optimize=opt)
  eng = calib._upload(calib.inliers)
  x0 = prob.param_vec
  keep = np.ones(eng.num_params, bool)
  keep[-calib._board_block_slices().size:] = calib._board_block_slices()
  assert keep.sum() == x0.size and np.abs(eng.param_vec[keep] - x0).max() <= 1e-12 * np.abs(x0).max()
  JtJ, Jtr, cost = eng.linearize()
  check_normal_equations(JtJ[np.ix_(keep, keep)], Jtr[keep], cost, fd5_jacobian(prob, x0), prob.residuals(x0), label)
  check_step(device_first_step(eng)[0], first_step(JtJ, Jtr, eng.param_vec), label)


def test_board_points_with_unstaged_boards():
  run_board_points_unstaged_boards(gpu_sms())


def run_frames_per_cta_unstaged(num_sms):
  """12 cameras x 9 boards (108 views per frame, 9 board tables: both read from global memory), F = 2 x (CTAs resident at once) + 3:
  CTAs of 3 frames, so every CTA goes through both halves of the double-buffered frame table and back to the first."""
  _, _, _, max_grid, _ = lin_shape("standard", False, 12, 9, num_sms)
  F = 2 * max_grid + 3
  scene = tiles_scene(12, 9, F=F, seed=43)
  _, _, _, grid, _ = lin_shape("standard", False, 12, 9, num_sms, F)
  assert -(-F // grid) == 3
  check_case(scene, dict(cameras=True), "static", 4, 1, num_sms, (108,) * F)
  return grid


def test_ctas_that_own_several_frames_with_unstaged_tables():
  run_frames_per_cta_unstaged(gpu_sms())


def run_bit_reproducibility():
  """Static frames at 12 x 9: two linearisations and two solves from the same state agree bit for bit."""
  from multical_b200.calibration import from_scene
  scene = tiles_scene(12, 9, seed=47)
  calib = from_scene(scene).enable(cameras=True)
  eng = calib._upload(calib.inliers)
  H0, g0, c0 = eng.linearize()
  H1, g1, c1 = eng.linearize()
  assert np.array_equal(H0, H1) and np.array_equal(g0, g1) and c0 == c1
  x0 = eng.param_vec.copy()
  runs = []
  for _ in range(2):
    eng.set_param_vec(x0)
    res = eng.solve(max_nfev=20, ftol=1e-12, xtol=1e-12, gtol=1e-12)
    runs.append((res.cost, np.array(res.log, float), eng.param_vec.copy()))
  assert runs[0][0] == runs[1][0] and np.array_equal(runs[0][1], runs[1][1], equal_nan=True) and np.array_equal(runs[0][2], runs[1][2])


def test_two_identical_linearisations_and_solves_agree_bit_for_bit():
  run_bit_reproducibility()
