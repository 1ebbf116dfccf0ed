"""ctypes binding of include/mcba.h (libmcba.so).  Fails loudly when the library or an
H100 (sm_90) device is missing: there is no CPU fallback on the product path."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MCBA_LIB", os.path.join(_HERE, "libmcba.so"))     # MCBA_LIB: developer A/B builds only

MODEL_IDS = {"standard": 0, "rational": 1, "thin_prism": 2, "fisheye": 3, "tilted": 4}
DIST_SIZES = {"standard": 5, "rational": 8, "thin_prism": 12, "fisheye": 4, "tilted": 14}
LOSS_IDS = {"linear": 0, "soft_l1": 1, "huber": 2, "cauchy": 3, "arctan": 4}
OPT_BITS = {"camera_poses": 1, "board_poses": 2, "motion": 4, "cameras": 8, "boards": 16}
OPT_FIX_ASPECT = 256
MOTION_ROLLING, MOTION_HAND_EYE = 1 << 16, 1 << 17        # include/mcba.h MCBA_MOTION_*: or-ed into ProblemDesc.optimize
STATUS_MESSAGES = {
  -1: "Improper input parameters status returned from `leastsq`",
  0: "The maximum number of function evaluations is exceeded.",
  1: "`gtol` termination condition is satisfied.",
  2: "`ftol` termination condition is satisfied.",
  3: "`xtol` termination condition is satisfied.",
  4: "Both `ftol` and `xtol` termination conditions are satisfied.",
}
EXPORTS = ["mcba_create", "mcba_destroy", "mcba_last_error", "mcba_set_stream", "mcba_version",
           "mcba_comm_unique_id", "mcba_comm_init", "mcba_peer_export", "mcba_peer_import", "mcba_upload_dense", "mcba_set_params", "mcba_get_params", "mcba_set_state_matrices", "mcba_get_state_matrices",
           "mcba_set_rolling", "mcba_get_rolling", "mcba_set_hand_eye", "mcba_get_hand_eye", "mcba_set_fixed_intrinsics",
           "mcba_set_trust_region", "mcba_last_alpha_iterations",
           "mcba_num_params", "mcba_get_param_vec", "mcba_set_param_vec", "mcba_residuals",
           "mcba_linearize", "mcba_reprojection_error", "mcba_solve", "mcba_bench_launch", "mcba_bench_info",
           "mcba_table_upload", "mcba_table_from_detections", "mcba_table_download", "mcba_table_set_inliers",
           "mcba_table_get_inliers", "mcba_table_select", "mcba_pnp_views", "mcba_table_errors", "mcba_table_error_ranks", "mcba_table_count_below", "mcba_table_reject",
           "mcba_intrinsic_init", "mcba_view_errors", "mcba_pose_pairs", "mcba_pose_times", "mcba_pose_cluster",
           "mcba_hand_eye_quads", "mcba_hand_eye_vote", "mcba_undistort_map", "mcba_undistort_images", "mcba_project_points",
           "mcba_undistort_points", "mcba_remap_cubic_table", "mcba_stereo_init", "mcba_rectify_map", "mcba_rectify_images",
           "mcba_rectify_points", "mcba_triangulate", "mcba_triangulate_linear"]
IMAGE_UINT8 = 0          # include/mcba.h MCBA_IMAGE_UINT8
POINTS_F64, POINTS_F32 = 0, 1          # include/mcba.h MCBA_POINTS_*
TABLE_VALID, TABLE_INLIERS = 0, 1
TR_SOLVERS = {"lsmr": 0, "exact": 1}    # include/mcba.h MCBA_TR_SUBSPACE / MCBA_TR_EXACT, named after scipy's tr_solver


class ProblemDesc(C.Structure):
  _fields_ = [("C", C.c_int32), ("F", C.c_int32), ("B", C.c_int32), ("P", C.c_int32),
              ("model", C.c_int32), ("optimize", C.c_int32), ("N", C.c_int64)]


class SolveOpts(C.Structure):
  _fields_ = [("ftol", C.c_double), ("xtol", C.c_double), ("gtol", C.c_double), ("f_scale", C.c_double),
              ("max_nfev", C.c_int32), ("loss", C.c_int32)]


class LogRow(C.Structure):
  _fields_ = [("iteration", C.c_int32), ("nfev", C.c_int32), ("cost", C.c_double),
              ("cost_reduction", C.c_double), ("step_norm", C.c_double), ("optimality", C.c_double)]


class SolveResult(C.Structure):
  _fields_ = [("cost", C.c_double), ("initial_cost", C.c_double), ("optimality", C.c_double),
              ("nfev", C.c_int32), ("njev", C.c_int32), ("status", C.c_int32), ("n_log", C.c_int32),
              ("device_ms", C.c_double), ("kernel_launches", C.c_int32), ("chol_retries", C.c_int32)]


class TableStats(C.Structure):
  _fields_ = [("n_valid", C.c_int64), ("n_inliers", C.c_int64), ("sumsq_valid", C.c_double), ("sumsq_inliers", C.c_double)]


class NativeError(RuntimeError):
  pass


_lib = None
_allow_interpreter = False      # set only by tests/test_simt_kernels.py: the product never runs on the test-suite's CPU interpreter build


def load():
  """dlopen libmcba.so (built in-tree by __graft_entry__.build())."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise NativeError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                      "(the engine has no CPU fallback)")
  lib = C.CDLL(LIB_PATH)
  if hasattr(lib, "mcba_simt_build") and not _allow_interpreter:
    raise NativeError(f"{LIB_PATH} is the SIMT-interpreter build of the test-suite (tests/simt), not the CUDA library: "
                      "the engine has no CPU path")
  P, D, I32 = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int32)
  lib.mcba_create.argtypes = [C.c_int, C.POINTER(P)]
  lib.mcba_destroy.argtypes = [P]; lib.mcba_destroy.restype = None
  lib.mcba_last_error.argtypes = [P]; lib.mcba_last_error.restype = C.c_char_p
  lib.mcba_set_stream.argtypes = [P, P]
  lib.mcba_comm_unique_id.argtypes = [P, C.c_char_p]
  lib.mcba_comm_init.argtypes = [P, C.c_char_p, C.c_int, C.c_int]
  lib.mcba_peer_export.argtypes = [P, C.c_int64, C.c_char_p]
  lib.mcba_peer_import.argtypes = [P, C.c_char_p]
  lib.mcba_upload_dense.argtypes = [P, C.POINTER(ProblemDesc), C.POINTER(C.c_uint8), C.POINTER(C.c_uint8), P, C.c_int32, D,
                                    C.POINTER(C.c_int64)]
  lib.mcba_set_params.argtypes = [P, D, D, D, D]
  lib.mcba_get_params.argtypes = [P, D, D, D, D]
  lib.mcba_set_state_matrices.argtypes = [P, D, D]
  lib.mcba_get_state_matrices.argtypes = [P, D, D]
  lib.mcba_set_rolling.argtypes = [P, D, D]
  lib.mcba_get_rolling.argtypes = [P, D]
  lib.mcba_set_hand_eye.argtypes = [P, D, D, D]
  lib.mcba_get_hand_eye.argtypes = [P, D, D]
  lib.mcba_set_fixed_intrinsics.argtypes = [P, C.POINTER(C.c_uint8)]
  lib.mcba_set_trust_region.argtypes = [P, C.c_int32]
  lib.mcba_last_alpha_iterations.argtypes = [P, I32]
  lib.mcba_num_params.argtypes = [P, C.POINTER(C.c_int64)]
  lib.mcba_get_param_vec.argtypes = [P, D]
  lib.mcba_set_param_vec.argtypes = [P, D]
  lib.mcba_residuals.argtypes = [P, D, D, D]
  lib.mcba_linearize.argtypes = [P, D, D, D, D]
  lib.mcba_reprojection_error.argtypes = [P, D]
  lib.mcba_solve.argtypes = [P, C.POINTER(SolveOpts), C.POINTER(SolveResult), C.POINTER(LogRow), C.c_int32]
  lib.mcba_bench_launch.argtypes = [P, C.c_int, C.c_int]
  lib.mcba_bench_info.argtypes = [P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]
  U8, I64 = C.POINTER(C.c_uint8), C.POINTER(C.c_int64)
  lib.mcba_table_upload.argtypes = [P, C.POINTER(ProblemDesc), U8, D, D, I64]
  lib.mcba_table_from_detections.argtypes = [P, C.POINTER(ProblemDesc), I64, I32, D, D, I64]
  lib.mcba_pnp_views.argtypes = [P, C.POINTER(ProblemDesc), I64, I32, D, D, D, I32, D, D, I32, U8]
  lib.mcba_table_download.argtypes = [P, U8, D]
  lib.mcba_table_set_inliers.argtypes = [P, U8]
  lib.mcba_table_get_inliers.argtypes = [P, U8]
  lib.mcba_table_select.argtypes = [P, C.c_int, I64]
  lib.mcba_table_errors.argtypes = [P, C.POINTER(TableStats)]
  lib.mcba_table_error_ranks.argtypes = [P, C.c_int, I64, C.c_int32, D]
  lib.mcba_table_count_below.argtypes = [P, C.c_int, D, C.c_int32, I64]
  lib.mcba_table_reject.argtypes = [P, C.c_double, I64, I64]
  lib.mcba_intrinsic_init.argtypes = [P, C.POINTER(ProblemDesc), I64, I32, D, D, I32, I32, U8, D, D, U8]
  lib.mcba_view_errors.argtypes = [P, D, I64]
  lib.mcba_stereo_init.argtypes = [P, C.POINTER(ProblemDesc), I64, I32, D, D, D, D, D, U8]
  i32 = C.c_int32
  lib.mcba_pose_pairs.argtypes = [P, i32, i32, i32, D, U8, i32, I32, i32, D, U8, I32]
  lib.mcba_pose_times.argtypes = [P, i32, i32, i32, D, U8, D, U8, D, U8, D, U8]
  lib.mcba_pose_cluster.argtypes = [P, i32, I64, D, U8]
  lib.mcba_hand_eye_quads.argtypes = [P, i32, i32, i32, D, U8, i32, I32, D, D, I32, U8]
  lib.mcba_hand_eye_vote.argtypes = [P, i32, I64, D, D, I32]
  U8P = C.POINTER(U8)
  lib.mcba_undistort_map.argtypes = [P, i32, D, i32, i32, C.POINTER(C.c_float)]
  lib.mcba_undistort_images.argtypes = [P, i32, D, i32, i32, i32, i32, i32, i32, i32, U8P, U8P]
  lib.mcba_project_points.argtypes = [P, i32, D, C.c_int64, D, D]
  lib.mcba_undistort_points.argtypes = [P, i32, D, C.c_int64, D, D]
  lib.mcba_remap_cubic_table.argtypes = [P, I32]
  lib.mcba_rectify_map.argtypes = [P, i32, D, D, D, i32, i32, C.POINTER(C.c_float)]
  lib.mcba_rectify_images.argtypes = [P, i32, D, D, D, i32, i32, i32, i32, i32, i32, i32, U8P, U8P]
  lib.mcba_rectify_points.argtypes = [P, i32, D, D, D, C.c_int64, D, D]
  lib.mcba_triangulate.argtypes = [P, i32, i32, D, D, C.c_int64, D, U8, D, U8, D]
  lib.mcba_triangulate_linear.argtypes = [P, D, D, C.c_int64, D, D, D]
  _lib = lib
  return lib


def dptr(a):
  return None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))


def iptr(a):
  return a.ctypes.data_as(C.POINTER(C.c_int32))


def f64(a):
  return np.ascontiguousarray(a, dtype=np.float64)
