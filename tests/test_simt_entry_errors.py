"""CPU (-m "not gpu"): how the C-ABI entry points of include/mcba.h refuse, on the SIMT interpreter build (tests/simt) of the real host
driver.  Every refusal returns its status code and leaves a message for mcba_last_error that names the problem: a null context, no
uploaded problem or resident table (MCBA_ERR_STATE), a bad argument or range.  A host allocation that fails returns MCBA_ERR_CUDA
instead of ending the caller's process, and the context stays usable."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from multical_b200 import _native as nat
from test_simt_kernels import on_the_interpreter, simt_library  # noqa: F401  (fixtures)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ARG, CUDA, STATE, NONFINITE, DEGENERATE = 1, 2, 3, 5, 7
NO_PROBLEM = "no problem uploaded"
NO_TABLE = "no resident table"
NO_ERRORS = "mcba_table_errors has not run"


def p(a):
  """a numpy array as the typed pointer of its dtype"""
  return a.ctypes.data_as(C.POINTER(np.ctypeslib.as_ctypes_type(a.dtype)))


def z(*shape, dtype=np.float64):
  return np.zeros(shape, dtype)


def desc(Cn=1, F=1, B=1, P=4, model=0, optimize=8):
  return C.byref(nat.ProblemDesc(Cn, F, B, P, model, optimize, 0))


def eye(n):
  return np.ascontiguousarray(np.broadcast_to(np.eye(4), (n, 4, 4)))


CAM = np.array([500.0, 500.0, 320.0, 240.0, 0.0, 0, 0, 0, 0, 0])      # standard model: fx fy cx cy skew k1 k2 p1 p2 k3
BP = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]], np.float64)
R3 = np.eye(3)
NAN = np.full(16, np.nan)


def u8pp(n):
  return (C.POINTER(C.c_uint8) * max(n, 1))()


def dets(ids, nv=1):
  """one detection list (w = 0) holding `ids`, the other nv - 1 lists empty"""
  start = np.array([0] + [len(ids)] * nv, np.int64)
  return p(start), p(np.array(ids, np.int32)), p(z(max(len(ids), 1), 2))


# (entry point, what must exist first, call, status, message substring)
ROWS = [
  # ---- communicator and peer memory
  ("mcba_comm_unique_id", None, lambda L, h: L.mcba_comm_unique_id(h, None), ARG, "null id buffer"),
  ("mcba_comm_init", None, lambda L, h: L.mcba_comm_init(h, None, 0, 1), ARG, "null id"),
  ("mcba_comm_init", None, lambda L, h: L.mcba_comm_init(h, b"x", 2, 2), ARG, "bad rank/world"),
  ("mcba_peer_export", None, lambda L, h: L.mcba_peer_export(h, 16, None), ARG, "null handle buffer"),
  ("mcba_peer_export", None, lambda L, h: L.mcba_peer_export(h, 16, C.create_string_buffer(64)), STATE, "initialised communicator"),
  ("mcba_peer_import", None, lambda L, h: L.mcba_peer_import(h, None), ARG, "null handles"),
  ("mcba_peer_import", None, lambda L, h: L.mcba_peer_import(h, C.create_string_buffer(64)), STATE, "mcba_peer_export has not been called"),
  # ---- problem intake
  ("mcba_upload_dense", None, lambda L, h: L.mcba_upload_dense(h, None, p(z(4, dtype=np.uint8)), None, p(z(4, 2)), 0, p(BP), p(z(1, dtype=np.int64))),
   ARG, "null problem description"),
  ("mcba_upload_dense", None, lambda L, h: L.mcba_upload_dense(h, desc(Cn=0), p(z(4, dtype=np.uint8)), None, p(z(4, 2)), 0, p(BP), None),
   ARG, "bad problem dimensions"),
  ("mcba_upload_dense", None, lambda L, h: L.mcba_upload_dense(h, desc(), p(z(4, dtype=np.uint8)), None, p(z(4, 2)), 7, p(BP), None),
   ARG, "unknown point type"),
  ("mcba_table_upload", None, lambda L, h: L.mcba_table_upload(h, None, p(z(4, dtype=np.uint8)), p(z(4, 2)), p(BP), None), ARG, "null problem description"),
  ("mcba_table_upload", None, lambda L, h: L.mcba_table_upload(h, desc(), None, p(z(4, 2)), p(BP), None), ARG, "null dense table"),
  ("mcba_table_from_detections", None, lambda L, h: L.mcba_table_from_detections(h, None, *dets([0]), p(BP), None), ARG, "null problem description"),
  ("mcba_table_from_detections", None, lambda L, h: L.mcba_table_from_detections(h, desc(), *dets([9]), p(BP), None), ARG, "detection id outside [0, P)"),
  ("mcba_table_from_detections", None, lambda L, h: L.mcba_table_from_detections(h, desc(), *dets([1, 2, 1]), p(BP), None),
   ARG, "detection list 0 repeats point id 1"),
  ("mcba_pnp_views", None, lambda L, h: L.mcba_pnp_views(h, None, *dets([0]), p(BP), p(CAM), p(z(5, dtype=np.int32)), p(z(16)), p(z(1)),
                                                         p(z(1, dtype=np.int32)), p(z(1, dtype=np.uint8))), ARG, "null problem description"),
  ("mcba_pnp_views", None, lambda L, h: L.mcba_pnp_views(h, desc(), p(np.array([1, 1], np.int64)), p(z(1, dtype=np.int32)), p(z(1, 2)), p(BP), p(CAM),
                                                         p(np.array([2, 2, 1, 0, 0], np.int32)), p(z(16)), p(z(1)), p(z(1, dtype=np.int32)),
                                                         p(z(1, dtype=np.uint8))), ARG, "bad detection offsets"),
  ("mcba_intrinsic_init", None, lambda L, h: L.mcba_intrinsic_init(h, None, *dets([0]), p(BP), p(np.array([2, 2, 1, 0, 0], np.int32)),
                                                                   p(np.array([640, 480], np.int32)), p(np.ones(1, np.uint8)), p(z(10)), p(z(16)),
                                                                   p(z(1, dtype=np.uint8))), ARG, "null problem description"),
  ("mcba_intrinsic_init", None, lambda L, h: L.mcba_intrinsic_init(h, desc(), *dets([0, 1, 2, 3]), p(BP), p(np.array([2, 2, 1, 0, 0], np.int32)),
                                                                   p(np.array([640, 0], np.int32)), p(np.ones(1, np.uint8)), p(z(10)), p(z(16)),
                                                                   p(z(1, dtype=np.uint8))), ARG, "image sizes must be positive"),
  ("mcba_stereo_init", None, lambda L, h: L.mcba_stereo_init(h, None, *dets([0], 2), p(BP), p(np.tile(CAM, 2)), p(z(6)), p(z(16)),
                                                             p(z(1, dtype=np.uint8))), ARG, "null problem description"),
  ("mcba_stereo_init", None, lambda L, h: L.mcba_stereo_init(h, desc(), *dets([0]), p(BP), p(np.tile(CAM, 2)), p(z(6)), p(z(16)),
                                                             p(z(1, dtype=np.uint8))), ARG, "a stereo pair is 2 cameras"),
  # ---- pose-graph and hand-eye initialisation
  ("mcba_pose_pairs", None, lambda L, h: L.mcba_pose_pairs(h, 0, 1, 1, p(eye(1)), p(np.ones(1, np.uint8)), 0, None, 0, None, None, None),
   ARG, "bad pose table dimensions"),
  ("mcba_pose_pairs", None, lambda L, h: L.mcba_pose_pairs(h, 2, 1, 1, p(eye(2)), p(np.ones(2, np.uint8)), 0, p(np.array([0, 0], np.int32)), 1,
                                                           p(z(16)), p(z(1, dtype=np.uint8)), p(z(1, dtype=np.int32))), ARG, "pair index out of range"),
  ("mcba_pose_pairs", None, lambda L, h: L.mcba_pose_pairs(h, 2, 1, 1, p(np.concatenate([NAN, NAN])), p(np.ones(2, np.uint8)), 0,
                                                           p(np.array([0, 1], np.int32)), 1, p(z(16)), p(z(1, dtype=np.uint8)), p(z(1, dtype=np.int32))),
   NONFINITE, "non-finite pose in the table"),
  ("mcba_pose_times", None, lambda L, h: L.mcba_pose_times(h, 1, 1, 1, None, None, p(eye(1)), p(np.ones(1, np.uint8)), p(eye(1)),
                                                           p(np.ones(1, np.uint8)), p(z(16)), p(z(1, dtype=np.uint8))), ARG, "null pose table"),
  ("mcba_pose_times", None, lambda L, h: L.mcba_pose_times(h, 1, 1, 1, p(NAN), p(np.ones(1, np.uint8)), p(eye(1)), p(np.ones(1, np.uint8)), p(eye(1)),
                                                           p(np.ones(1, np.uint8)), p(z(16)), p(z(1, dtype=np.uint8))), NONFINITE, "non-finite pose"),
  ("mcba_pose_cluster", None, lambda L, h: L.mcba_pose_cluster(h, 1, None, p(z(6)), p(z(1, dtype=np.uint8))), ARG, "null set offsets"),
  ("mcba_pose_cluster", None, lambda L, h: L.mcba_pose_cluster(h, 1, p(np.array([1, 2], np.int64)), p(z(6)), p(z(1, dtype=np.uint8))),
   ARG, "set offsets must start at 0"),
  ("mcba_hand_eye_quads", None, lambda L, h: L.mcba_hand_eye_quads(h, 2, 1, 1, p(eye(2)), p(np.ones(2, np.uint8)), 1, p(np.array([0, 5, 0, 0], np.int32)),
                                                                   p(z(16)), p(z(16)), p(z(1, dtype=np.int32)), p(z(1, dtype=np.uint8))),
   ARG, "quadruple index out of range"),
  ("mcba_hand_eye_quads", None, lambda L, h: L.mcba_hand_eye_quads(h, 2, 1, 1, p(eye(2)), p(np.ones(2, np.uint8)), 1, p(np.array([1, 1, 0, 0], np.int32)),
                                                                   p(z(16)), p(z(16)), p(z(1, dtype=np.int32)), p(z(1, dtype=np.uint8))),
   ARG, "master == slave"),
  ("mcba_hand_eye_vote", None, lambda L, h: L.mcba_hand_eye_vote(h, 1, p(np.array([0, 3], np.int64)), p(z(3, 3)), p(z(3)), p(z(1, dtype=np.int32))),
   DEGENERATE, "set 0 has 3 points"),
  # ---- applying a calibration
  ("mcba_rectify_map", None, lambda L, h: L.mcba_rectify_map(h, 0, p(np.r_[0.0, CAM[1:]]), p(R3), p(R3), 8, 8, None), ARG, "zero focal length"),
  ("mcba_rectify_map", None, lambda L, h: L.mcba_rectify_map(h, 0, p(CAM), p(R3), p(R3), 0, 8, None), ARG, "map size out of range"),
  ("mcba_rectify_images", None, lambda L, h: L.mcba_rectify_images(h, 0, p(CAM), p(R3), p(R3), 8, 8, 1, 8, 8, 1, 1, u8pp(1), u8pp(1)),
   ARG, "unsupported image dtype"),
  ("mcba_project_points", None, lambda L, h: L.mcba_project_points(h, 9, p(CAM), 1, p(z(3)), p(z(2))), ARG, "unknown camera model"),
  ("mcba_rectify_points", None, lambda L, h: L.mcba_rectify_points(h, 0, None, p(R3), p(R3), 1, p(z(2)), p(z(2))), ARG, "null camera"),
  ("mcba_rectify_points", None, lambda L, h: L.mcba_rectify_points(h, 0, p(CAM), p(R3), p(R3), -1, p(z(2)), p(z(2))), ARG,
   "negative point count"),
  ("mcba_remap_cubic_table", None, lambda L, h: L.mcba_remap_cubic_table(h, None), ARG, "null table"),
  ("mcba_rectify_map", None, lambda L, h: L.mcba_rectify_map(h, 0, p(CAM), None, p(R3), 8, 8, None), ARG, "null R or P"),
  ("mcba_rectify_map", None, lambda L, h: L.mcba_rectify_map(h, 0, p(CAM), p(R3), p(z(3, 3)), 8, 8, None), ARG, "P R is singular"),
  ("mcba_rectify_images", None, lambda L, h: L.mcba_rectify_images(h, 0, p(CAM), p(R3), p(R3), 8, 8, 1, 8, 8, 2, 0, u8pp(1), u8pp(1)),
   ARG, "unsupported channel count"),
  ("mcba_rectify_points", None, lambda L, h: L.mcba_rectify_points(h, 0, p(CAM), p(R3), None, 1, p(z(2)), p(z(2))), ARG, "null R or P"),
  ("mcba_triangulate", None, lambda L, h: L.mcba_triangulate(h, 0, 0, p(CAM), p(eye(1)), 1, p(z(2)), p(np.ones(1, np.uint8)), p(z(3)),
                                                             p(z(1, dtype=np.uint8)), p(z(1))), ARG, "camera count out of range"),
  ("mcba_triangulate", None, lambda L, h: L.mcba_triangulate(h, 0, 2, p(np.r_[CAM, 0.0, CAM[1:]]), p(eye(2)), 1, p(z(2, 2)), p(np.ones(2, np.uint8)),
                                                             p(z(3)), p(z(1, dtype=np.uint8)), p(z(1))), ARG, "camera 1: zero focal length"),
  ("mcba_triangulate_linear", None, lambda L, h: L.mcba_triangulate_linear(h, p(NAN[:12]), p(z(12)), 1, p(z(2)), p(z(2)), p(z(4))),
   NONFINITE, "non-finite projection matrix"),
  # ---- resident point table
  ("mcba_table_download", None, lambda L, h: L.mcba_table_download(h, p(z(4, dtype=np.uint8)), None), STATE, NO_TABLE),
  ("mcba_table_set_inliers", None, lambda L, h: L.mcba_table_set_inliers(h, None), STATE, NO_TABLE),
  ("mcba_table_get_inliers", None, lambda L, h: L.mcba_table_get_inliers(h, None), ARG, "null mask"),
  ("mcba_table_get_inliers", None, lambda L, h: L.mcba_table_get_inliers(h, p(z(4, dtype=np.uint8))), STATE, NO_TABLE),
  ("mcba_table_select", None, lambda L, h: L.mcba_table_select(h, 0, None), STATE, NO_TABLE),
  ("mcba_table_select", "table", lambda L, h: L.mcba_table_select(h, 5, None), ARG, "unknown table selection"),
  ("mcba_table_errors", None, lambda L, h: L.mcba_table_errors(h, None), STATE, NO_TABLE),
  ("mcba_table_error_ranks", None, lambda L, h: L.mcba_table_error_ranks(h, 0, None, 1, p(z(1))), ARG, "null ranks or output"),
  ("mcba_table_error_ranks", "table", lambda L, h: L.mcba_table_error_ranks(h, 0, p(z(1, dtype=np.int64)), 1, p(z(1))), STATE, NO_ERRORS),
  ("mcba_table_count_below", None, lambda L, h: L.mcba_table_count_below(h, 0, p(z(1)), 1, None), ARG, "null thresholds or counts"),
  ("mcba_table_count_below", "table", lambda L, h: L.mcba_table_count_below(h, 0, p(z(1)), 1, p(z(1, dtype=np.int64))), STATE, NO_ERRORS),
  ("mcba_table_reject", "table", lambda L, h: L.mcba_table_reject(h, 1.0, None, None), STATE, NO_ERRORS),
  # ---- the uploaded problem's state
  ("mcba_view_errors", None, lambda L, h: L.mcba_view_errors(h, None, p(z(1, dtype=np.int64))), ARG, "null argument"),
  ("mcba_view_errors", None, lambda L, h: L.mcba_view_errors(h, p(z(1)), p(z(1, dtype=np.int64))), STATE, NO_PROBLEM),
  ("mcba_set_params", None, lambda L, h: L.mcba_set_params(h, None, None, None, None), STATE, NO_PROBLEM),
  ("mcba_set_params", "problem", lambda L, h: L.mcba_set_params(h, None, p(z(6)), p(z(6)), p(CAM)), ARG, "null parameter array"),
  ("mcba_get_params", None, lambda L, h: L.mcba_get_params(h, None, None, None, None), STATE, NO_PROBLEM),
  ("mcba_set_state_matrices", None, lambda L, h: L.mcba_set_state_matrices(h, None, None), STATE, NO_PROBLEM),
  ("mcba_set_state_matrices", "problem", lambda L, h: L.mcba_set_state_matrices(h, None, p(CAM)), ARG, "null parameter array"),
  ("mcba_get_state_matrices", None, lambda L, h: L.mcba_get_state_matrices(h, None, None), STATE, NO_PROBLEM),
  ("mcba_set_rolling", None, lambda L, h: L.mcba_set_rolling(h, None, None), STATE, NO_PROBLEM),
  ("mcba_set_rolling", "problem", lambda L, h: L.mcba_set_rolling(h, p(eye(1)), p(np.ones(1))), STATE, "MCBA_MOTION_ROLLING"),
  ("mcba_get_rolling", None, lambda L, h: L.mcba_get_rolling(h, None), ARG, "null parameter array"),
  ("mcba_get_rolling", None, lambda L, h: L.mcba_get_rolling(h, p(eye(1))), STATE, NO_PROBLEM),
  ("mcba_set_hand_eye", None, lambda L, h: L.mcba_set_hand_eye(h, None, None, None), STATE, NO_PROBLEM),
  ("mcba_set_hand_eye", "problem", lambda L, h: L.mcba_set_hand_eye(h, p(eye(1)), p(eye(1)), p(eye(1))), STATE, "MCBA_MOTION_HAND_EYE"),
  ("mcba_get_hand_eye", None, lambda L, h: L.mcba_get_hand_eye(h, None, None), STATE, NO_PROBLEM),
  ("mcba_set_fixed_intrinsics", None, lambda L, h: L.mcba_set_fixed_intrinsics(h, None), STATE, NO_PROBLEM),
  ("mcba_set_fixed_intrinsics", "problem", lambda L, h: L.mcba_set_fixed_intrinsics(h, p(np.full(10, 2, np.uint8))), ARG, "must be 0 or 1"),
  ("mcba_set_trust_region", None, lambda L, h: L.mcba_set_trust_region(h, 0), STATE, NO_PROBLEM),
  ("mcba_set_trust_region", "problem", lambda L, h: L.mcba_set_trust_region(h, 5), ARG, "MCBA_TR_SUBSPACE or MCBA_TR_EXACT"),
  ("mcba_last_alpha_iterations", None, lambda L, h: L.mcba_last_alpha_iterations(h, None), ARG, "null argument"),
  ("mcba_num_params", None, lambda L, h: L.mcba_num_params(h, None), ARG, "null argument"),
  ("mcba_num_params", None, lambda L, h: L.mcba_num_params(h, p(z(1, dtype=np.int64))), STATE, NO_PROBLEM),
  ("mcba_get_param_vec", None, lambda L, h: L.mcba_get_param_vec(h, None), ARG, "null parameter vector"),
  ("mcba_get_param_vec", None, lambda L, h: L.mcba_get_param_vec(h, p(z(64))), STATE, NO_PROBLEM),
  ("mcba_set_param_vec", None, lambda L, h: L.mcba_set_param_vec(h, None), ARG, "null parameter vector"),
  ("mcba_set_param_vec", None, lambda L, h: L.mcba_set_param_vec(h, p(z(64))), STATE, NO_PROBLEM),
  ("mcba_residuals", None, lambda L, h: L.mcba_residuals(h, None, None, None), STATE, NO_PROBLEM),
  ("mcba_linearize", None, lambda L, h: L.mcba_linearize(h, None, None, None, None), STATE, NO_PROBLEM),
  ("mcba_reprojection_error", None, lambda L, h: L.mcba_reprojection_error(h, None), ARG, "null argument"),
  ("mcba_reprojection_error", None, lambda L, h: L.mcba_reprojection_error(h, p(z(4))), STATE, NO_PROBLEM),
  ("mcba_solve", None, lambda L, h: L.mcba_solve(h, None, C.byref(nat.SolveResult()), None, 0), ARG, "null options or result"),
  ("mcba_solve", None, lambda L, h: L.mcba_solve(h, C.byref(nat.SolveOpts(1e-8, 1e-8, 1e-8, 1.0, 10, 0)), C.byref(nat.SolveResult()), None, 0),
   STATE, NO_PROBLEM),
  ("mcba_solve", "problem", lambda L, h: L.mcba_solve(h, C.byref(nat.SolveOpts(1e-8, 1e-8, 1e-8, 1.0, 10, 9)), C.byref(nat.SolveResult()), None, 0),
   ARG, "unknown loss"),
  ("mcba_bench_info", None, lambda L, h: L.mcba_bench_info(h, 0, None, None, None), STATE, NO_PROBLEM),
  ("mcba_bench_launch", None, lambda L, h: L.mcba_bench_launch(h, 0, 1), STATE, NO_PROBLEM),
  ("mcba_bench_launch", "problem", lambda L, h: L.mcba_bench_launch(h, 7, 1), ARG, "unsupported bench kernel"),
]

# entry points without a context argument, or that cannot fail
NO_CONTEXT = {"mcba_create", "mcba_destroy", "mcba_last_error", "mcba_version"}


def test_every_entry_point_has_a_refusal():
  """every entry point that takes a context has a row beyond the null-context one"""
  assert {r[0] for r in ROWS} | {"mcba_set_stream"} | NO_CONTEXT == set(nat.EXPORTS)


@pytest.fixture
def lib():
  return nat.load()


@pytest.fixture
def ctx(lib):
  h = C.c_void_p()
  assert lib.mcba_create(0, C.byref(h)) == 0
  yield h
  lib.mcba_destroy(h)


def make(lib, h, what):
  """a fresh context with nothing, with an uploaded problem (1 camera, 1 frame, 1 board of 4 points) or with that as resident table"""
  valid, pts, n = np.ones(4, np.uint8), z(4, 2), z(1, dtype=np.int64)
  if what == "problem":
    assert lib.mcba_upload_dense(h, desc(), p(valid), None, p(pts), nat.POINTS_F64, p(BP), p(n)) == 0
  elif what == "table":
    assert lib.mcba_table_upload(h, desc(), p(valid), p(pts), p(BP), p(n)) == 0


@pytest.mark.parametrize("name, needs, call, code, msg", [pytest.param(*r, id=f"{r[0]}-{i}") for i, r in enumerate(ROWS)])
def test_refusal_sets_code_and_message(lib, ctx, name, needs, call, code, msg):
  make(lib, ctx, needs)
  rc = call(lib, ctx)
  text = lib.mcba_last_error(ctx).decode()
  assert (rc, msg in text) == (code, True), (name, rc, text)


@pytest.mark.parametrize("name", sorted(set(nat.EXPORTS) - NO_CONTEXT))
def test_null_context_is_refused(lib, name):
  fn = getattr(lib, name)
  args = [None if t is C.c_void_p or t is C.c_char_p or issubclass(t, C._Pointer) else t(0) for t in fn.argtypes]
  assert fn(*args) == ARG


def test_create_refusals(lib):
  assert lib.mcba_create(0, None) == ARG
  assert b"null" in lib.mcba_last_error(None)
  h = C.c_void_p()
  assert lib.mcba_create(5, C.byref(h)) == ARG and not h.value
  assert b"device ordinal out of range" in lib.mcba_last_error(None)


OOM_SCRIPT = r"""
import ctypes as C, resource, sys
import numpy as np
from multical_b200 import _native as nat
nat._allow_interpreter = True
L = nat.load()
h = C.c_void_p()
assert L.mcba_create(0, C.byref(h)) == 0
def pose_pairs(Cn, F, B, n_pairs):
  poses = np.ascontiguousarray(np.broadcast_to(np.eye(4), (Cn * F * B, 4, 4)))
  pairs = np.tile(np.array([0, 1], np.int32), n_pairs)
  R = F * B
  t, inl, n_inl = np.empty((n_pairs, 16)), np.empty(n_pairs * R, np.uint8), np.empty(n_pairs, np.int32)
  dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
  return L.mcba_pose_pairs(h, Cn, F, B, dp(poses), np.ones(Cn * F * B, np.uint8).ctypes.data_as(C.POINTER(C.c_uint8)), 0,
                           pairs.ctypes.data_as(C.POINTER(C.c_int32)), n_pairs, dp(t), inl.ctypes.data_as(C.POINTER(C.c_uint8)),
                           n_inl.ctypes.data_as(C.POINTER(C.c_int32)))
resource.setrlimit(resource.RLIMIT_AS, (4 << 30, 4 << 30))
# 16384 pairs of 65536 rows each: 2^30 gathered rows of 16 bytes on the host, inside the 2^31-row limit the entry point accepts
rc = pose_pairs(2, 1, 65536, 16384)
print("big", rc, L.mcba_last_error(h).decode())
print("small", pose_pairs(2, 1, 4, 1))
L.mcba_destroy(h)
"""


def test_failed_host_allocation_is_an_error_not_an_abort(simt_library):
  """A host allocation the caller's sizes make too large (here under a 4 GB address-space limit) returns MCBA_ERR_CUDA with a message,
  and the next call on the same context succeeds."""
  env = dict(os.environ, MCBA_LIB=simt_library, PYTHONPATH=ROOT, OPENBLAS_NUM_THREADS="1", OMP_NUM_THREADS="1")
  out = subprocess.run([sys.executable, "-c", OOM_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
  assert out.returncode == 0, (out.returncode, out.stdout, out.stderr[-2000:])
  lines = dict(line.split(" ", 1) for line in out.stdout.splitlines())
  rc, msg = lines["big"].split(" ", 1)
  assert int(rc) == CUDA and "host allocation" in msg, lines
  assert lines["small"] == "0", lines
