"""GPU (-m gpu): the resident point table (include/mcba.h "resident point table") -- the outlier loop around the hot path
kept on the device (SURVEY §8f rank 1) and the detections -> table wire format (rank 3).

Bars: masks, counts, ranks and thresholds are integer / order-statistic work -> bit exact against numpy on the same
error vector; sums of squares <= 1e-12 relative (summation order); the loop's solves are the solves of the host loop,
so costs agree to 1e-6 relative and per-corner errors to 1e-2 px (poses themselves are gauge-dependent)."""
import numpy as np
import pytest

from conftest import load_golden
from multical_b200 import _native, synthetic
from multical_b200.calibration import from_scene, get_engine, select_threshold
from oracle.ba_oracle import Problem

pytestmark = pytest.mark.gpu


def scene_and_calib(seed=61, **kw):
  args = dict(C=3, F=8, vis=0.5, seed=seed, outlier_fraction=0.02); args.update(kw)
  scene = synthetic.make_scene(**args)
  return scene, from_scene(scene).enable(cameras=True)


def resident_engine(calib):
  eng = get_engine()
  n = eng.table_upload(calib.engine_model, calib._optimize_bits(), calib.valid, np.asarray(calib.point_table.points),
                       calib.board_points.points)
  calib._push_state(eng)
  return eng, n


def test_table_errors_ranks_and_reject_are_numpy_on_the_same_errors():
  scene, calib = scene_and_calib()
  prob = Problem.from_scene(scene, optimize=dict(cameras=True))
  err_host = calib._upload(calib.valid).reprojection_error()            # same kernel, through the packed entry point
  host_rule = calib.reject_outliers(select_threshold(0.9, 1.0)(err_host)).inliers
  eng, n = resident_engine(calib)
  assert n == int(calib.valid.sum()) == err_host.size
  st = eng.table_errors()
  assert (st.n_valid, st.n_inliers) == (n, n)
  assert abs(st.sumsq_valid - np.sum(err_host ** 2)) <= 1e-12 * np.sum(err_host ** 2)
  assert st.sumsq_inliers == st.sumsq_valid
  o_err, o_mask = prob.reprojection_error()                            # and the oracle agrees with the values
  assert np.abs(np.sort(err_host) - np.sort(o_err[o_mask])).max() < 1e-9
  srt = np.sort(err_host)
  ranks = np.array([0, 1, n // 3, n // 2, n - 2, n - 1])
  assert np.array_equal(eng.table_error_ranks("valid", ranks), srt[ranks])
  q = np.array([0.0, 0.25, 0.5, 0.75, 0.95, 1.0])
  assert np.array_equal(eng.table_quantile("valid", n, q), np.quantile(err_host, q))
  thr = select_threshold(0.9, 1.0)(err_host)                           # the initial guess is far off: cut the worst tenth
  assert eng.table_quantile("valid", n, 0.9) * 1.0 == thr
  n_valid, n_keep = eng.table_reject(thr)
  keep = np.zeros(calib.valid.shape, bool); keep[calib.valid] = err_host < thr
  assert (n_valid, n_keep) == (n, int(keep.sum())) and n_keep < n
  assert np.array_equal(eng.table_get_inliers(), keep)
  assert np.array_equal(keep, host_rule)                               # = the host path's rule (calibration.py:240-252)
  # inlier statistics after the rejection; then the inlier selection is what the solver sees
  st2 = eng.table_errors()
  inl = err_host[keep[calib.valid]]
  assert st2.n_inliers == inl.size and abs(st2.sumsq_inliers - np.sum(inl ** 2)) <= 1e-12 * np.sum(inl ** 2)
  assert np.array_equal(eng.table_quantile("inliers", inl.size, q), np.quantile(inl, q))
  assert eng.table_select("inliers") == inl.size
  r_resident = eng.residuals()
  r_host = calib.copy(inlier_mask=keep)._upload(keep).residuals()
  assert np.array_equal(r_resident, r_host)                             # same packing, same state, same kernel


def test_resident_adjust_outliers_equals_host_loop(monkeypatch):
  scene, calib = scene_and_calib(seed=62)
  kw = dict(num_adjustments=3, select_outliers=select_threshold(quantile=0.75, factor=5.0),
            select_scale=select_threshold(quantile=0.75, factor=2.0), loss="soft_l1", tolerance=1e-8, max_iterations=60)
  monkeypatch.setenv("MCBA_HOST_OUTLIERS", "1")
  host = calib.adjust_outliers(**kw)
  monkeypatch.delenv("MCBA_HOST_OUTLIERS")
  res = calib.adjust_outliers(**kw)
  assert np.array_equal(res.inlier_mask, host.inlier_mask) and res.inlier_mask.sum() < calib.valid.sum()
  # The host loop re-enters each solve through 4x4 matrices (rtvec -> matrix -> rtvec, ~1e-16), the resident loop keeps the
  # rotation vectors: same iterations up to that perturbation.  Poses are only defined up to the gauge (a common rigid motion
  # of rig and boards), so the solutions are compared through what they predict: cost and per-corner pixel error.
  assert abs(res.last_solve.cost - host.last_solve.cost) <= 1e-6 * host.last_solve.cost
  assert np.abs(res.reprojection_error - host.reprojection_error).max() < 1e-2
  rms = np.sqrt(np.mean(res.reprojection_inliers ** 2))
  assert 0.3 < rms < 0.6                                               # 0.3 px noise -> 0.3*sqrt(2) expected


def detection_lists(valid, points):
  """What the reference holds before tables.make_point_table: per (camera, frame, board) the detected ids and corners."""
  Cn, F, B, P = valid.shape
  flat_v, flat_p = valid.reshape(-1, P), points.reshape(-1, P, 2)
  counts = flat_v.sum(axis=1)
  start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
  w, ids = np.nonzero(flat_v)
  return start, ids.astype(np.int32), flat_p[w, ids]


def test_table_from_detections_is_make_point_table():
  scene, calib = scene_and_calib(seed=63, F=5, boards=("cube", 6, 6, 0.03, 3))      # several boards of one rig
  valid_pts = np.asarray(calib.point_table.valid)
  pts = np.where(valid_pts[..., None], np.asarray(calib.point_table.points), 0.0)       # fill_sparse leaves zeros
  start, ids, xy = detection_lists(valid_pts, pts)
  rng = np.random.default_rng(0)                                         # detection order inside a list is arbitrary
  for w in range(start.size - 1):
    perm = rng.permutation(start[w + 1] - start[w]) + start[w]
    ids[start[w]:start[w + 1]], xy[start[w]:start[w + 1]] = ids[perm], xy[perm]
  eng = get_engine()
  n = eng.table_from_detections(calib.engine_model, calib._optimize_bits(), valid_pts.shape, start, ids, xy, calib.board_points.points)
  got_valid, got_pts = eng.table_download()
  assert n == int(valid_pts.sum()) and np.array_equal(got_valid, valid_pts) and np.array_equal(got_pts, pts)
  calib._push_state(eng)
  r_table = eng.residuals()
  r_dense = calib._upload(valid_pts).residuals()
  assert np.array_equal(r_table, r_dense)
  # malformed lists are refused, not scattered out of bounds
  bad = ids.copy(); bad[0] = valid_pts.shape[3]
  with pytest.raises(AssertionError):
    eng.table_from_detections(calib.engine_model, calib._optimize_bits(), valid_pts.shape, start, bad, xy, calib.board_points.points)
  bad_start = start.copy(); bad_start[1], bad_start[2] = start[2], start[1]
  if bad_start[1] != bad_start[2]:
    with pytest.raises(AssertionError):
      eng.table_from_detections(calib.engine_model, calib._optimize_bits(), valid_pts.shape, bad_start, ids, xy, calib.board_points.points)


@pytest.mark.parametrize("refusal", ["too many boards", "detection id outside"])
def test_a_refused_upload_leaves_no_problem(refusal):
  """An upload replaces the problem even when it is refused: one refused inside setup_problem (too many boards for k_linearize's
  shared memory) or for its detection lists leaves none, so the next residuals refuse instead of running on the previous problem."""
  scene, calib = scene_and_calib(seed=65)
  eng = calib._upload(calib.valid)
  eng.residuals()
  if refusal == "too many boards":      # 2 cameras: 63 boards at most (tests/test_gpu_linearize_shapes.py BOARD_LIMITS)
    mask = np.zeros((2, 1, 64, 1), bool); mask[:, 0, -1, 0] = True
    with pytest.raises(NotImplementedError, match=refusal):
      eng.upload_dense("standard", calib._optimize_bits(), mask, np.zeros((2, 1, 64, 1, 2)), np.zeros((64, 1, 3)))
  else:
    valid_pts = np.asarray(calib.point_table.valid)
    start, ids, xy = detection_lists(valid_pts, np.asarray(calib.point_table.points))
    ids[0] = valid_pts.shape[3]
    with pytest.raises(AssertionError, match=refusal):
      eng.table_from_detections(calib.engine_model, calib._optimize_bits(), valid_pts.shape, start, ids, xy, calib.board_points.points)
  with pytest.raises(_native.NativeError, match="no problem uploaded"):
    eng.residuals()
  calib._upload(calib.valid).residuals()


def test_a_repeated_detection_id_is_refused():
  """A dense table holds one corner per (view, point id): a detection list that repeats an id is refused."""
  scene, calib = scene_and_calib(seed=66)
  valid_pts = np.asarray(calib.point_table.valid)
  start, ids, xy = detection_lists(valid_pts, np.asarray(calib.point_table.points))
  w = int(np.flatnonzero(np.diff(start) >= 2)[0])
  ids[start[w] + 1] = ids[start[w]]
  with pytest.raises(AssertionError, match="repeats point id"):
    get_engine().table_from_detections(calib.engine_model, calib._optimize_bits(), valid_pts.shape, start, ids, xy,
                                       calib.board_points.points)


def test_table_state_machine_refuses_stale_errors():
  scene, calib = scene_and_calib(seed=64)
  eng = calib._upload(calib.valid)                                       # packed upload: no resident table
  with pytest.raises(_native.NativeError):
    eng.table_errors()
  eng, n = resident_engine(calib)
  with pytest.raises(_native.NativeError):
    eng.table_reject(1.0)                                                # no errors yet
  eng.table_errors()
  calib._push_state(eng)                                                 # parameters changed -> errors are stale
  with pytest.raises(_native.NativeError):
    eng.table_reject(1.0)
  eng.table_errors()
  eng.table_select("inliers")                                            # selection changed -> reject needs the valid packing
  with pytest.raises(_native.NativeError):
    eng.table_reject(1.0)
  # a host mask is and-ed with `valid`; None restores inliers = valid
  everything = np.ones(calib.valid.shape, bool)
  eng.table_set_inliers(everything)
  assert np.array_equal(eng.table_get_inliers(), calib.valid)
  half = calib.valid & (np.arange(calib.valid.shape[1]) % 2 == 0)[None, :, None, None]
  eng.table_set_inliers(half)
  assert eng.table_select("inliers") == int(half.sum())
  eng.table_set_inliers(None)
  assert eng.table_select("inliers") == n
  # rejecting everything leaves an empty, still well-formed problem
  eng.table_errors()
  assert eng.table_reject(0.0) == (n, 0)
  assert eng.table_select("inliers") == 0 and eng.residuals().size == 0


def test_outlier_steps_match_reference_golden():
  """The steps either side of bundle_adjust against what the running reference produced at the same state
  (tests/golden/outliers_3x6.npz, generated by tests/golden/make_golden.py outlier_case)."""
  scene, z = load_golden("outliers_3x6")
  calib = from_scene(scene).enable(cameras=True)
  thr_ref = float(z["thr_q75x5"])
  # the reference-named host API (errors from k_views<MODE_ERROR>)
  assert np.abs(calib.reprojection_error - z["err_valid"]).max() < 1e-9
  assert abs(select_threshold(quantile=0.75, factor=5.0)(calib.reprojection_error) - thr_ref) < 1e-9
  assert np.array_equal(calib.reject_outliers(thr_ref).inliers, z["inliers_thr"])
  assert np.array_equal(calib.reject_outliers_quantile(0.95).inliers, z["inliers_q95"])
  # the same decisions on the resident table
  eng, n = resident_engine(calib)
  st = eng.table_errors()
  assert st.n_valid == z["err_valid"].size
  assert abs(eng.table_quantile("valid", n, 0.75) * 5.0 - thr_ref) < 1e-9
  assert eng.table_reject(thr_ref) == (n, int(z["inliers_thr"].sum()))
  assert np.array_equal(eng.table_get_inliers(), z["inliers_thr"])
  eng.table_errors()
  assert eng.table_reject(eng.table_quantile("valid", n, 0.95)) == (n, int(z["inliers_q95"].sum()))
  assert np.array_equal(eng.table_get_inliers(), z["inliers_q95"])
  # and the whole loop: same inlier set as the reference's adjust_outliers, same inlier RMS
  out = calib.adjust_outliers(num_adjustments=2, select_outliers=select_threshold(quantile=0.75, factor=5.0))
  assert np.array_equal(out.inlier_mask, z["adj_inliers"])
  assert abs(np.sqrt(np.mean(out.reprojection_inliers ** 2)) - float(z["adj_rms"])) < 2e-3


def test_workspace_calibrate_is_enable_plus_the_outlier_loop():
  """multical_b200/workspace.py calibrate = Workspace.calibrate (workspace.py:228-247): the blocks it enables and the selectors it builds."""
  from multical_b200 import workspace
  scene, calib = scene_and_calib()
  base = from_scene(scene)                                   # default blocks: poses only
  out = workspace.calibrate(base, cameras=True, loss="soft_l1", auto_scale=3.0, num_adjustments=2)
  want = base.enable(cameras=True, boards=False, camera_poses=True, motion=True, board_poses=True).adjust_outliers(
    loss="soft_l1", tolerance=1e-4, num_adjustments=2, select_outliers=select_threshold(quantile=0.75, factor=5.0),
    select_scale=select_threshold(quantile=0.75, factor=3.0))
  assert out.optimize == want.optimize and out.optimize["cameras"] is True
  assert np.array_equal(out.inliers, want.inliers) and out.inliers.sum() < calib.valid.sum()
  assert abs(out.last_solve.cost - want.last_solve.cost) <= 1e-12 * want.last_solve.cost
  fixed = workspace.optimize(base, fix_intrinsic=True, fix_board_poses=True)
  assert fixed.optimize["cameras"] is False and fixed.optimize["board_poses"] is False and fixed.optimize["motion"] is True
