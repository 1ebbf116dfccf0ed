"""Python face of libmcba.so: one `Engine` = one C-ABI context on one GPU.

The engine replaces exactly one call of the reference,
`scipy.optimize.least_squares(evaluate, ...)` (multical/optimization/calibration.py:209-210),
together with the `evaluate` closure (204-206) and the reprojection-error pass (tables.py:244-249).
Everything numeric happens in CUDA kernels behind include/mcba.h; numpy is only used to lay
out the packed input arrays."""
import ctypes as C

import numpy as np

from . import _native as nat
from ._native import NativeError


def pack_corners(inliers, points):
  """Dense [C,F,B,P] mask + [C,F,B,P,2] observations -> packed corner arrays in the reference's
  boolean-mask order (np.argwhere(inliers) row-major == `(...)[self.inliers]`, calibration.py:206)."""
  idx = np.argwhere(inliers).astype(np.int32)                     # [N,4] rows (c,f,b,p)
  obs = np.ascontiguousarray(points[inliers], dtype=np.float64)   # [N,2]
  return idx, obs


class SolveInfo(dict):
  __getattr__ = dict.__getitem__


class Engine:
  def __init__(self, device=0, stream=None):
    self.lib = nat.load()
    h = C.c_void_p()
    rc = self.lib.mcba_create(int(device), C.byref(h))
    if rc != 0:
      raise NativeError(f"mcba_create failed ({rc}): {self.lib.mcba_last_error(None).decode()}")
    self.h = h
    self.device = device
    self.desc = None
    if stream is not None:
      self._ck(self.lib.mcba_set_stream(self.h, C.c_void_p(int(stream))))

  def close(self):
    if getattr(self, "h", None):
      self.lib.mcba_destroy(self.h)
      self.h = None

  def __del__(self):
    try: self.close()
    except Exception: pass

  def _ck(self, rc):
    if rc == 0: return
    msg = self.lib.mcba_last_error(self.h).decode()
    if rc == 1: raise AssertionError(msg)            # reference uses `assert` for bad inputs (calibration.py:59-61)
    if rc == 5: raise ValueError(msg)                # scipy: "Residuals are not finite in the initial point."
    if rc == 6: raise NotImplementedError(msg)
    raise NativeError(f"libmcba error {rc}: {msg}")

  # ---- multi-GPU --------------------------------------------------------------------------------
  def comm_unique_id(self):
    buf = C.create_string_buffer(128)
    self._ck(self.lib.mcba_comm_unique_id(self.h, buf))
    return buf.raw

  def comm_init(self, uid, rank, world):
    self._ck(self.lib.mcba_comm_init(self.h, uid, int(rank), int(world)))
    self.rank, self.world = rank, world

  def peer_export(self, cap_doubles):
    """Allocate this rank's NVLink exchange buffer and return its 64-byte IPC handle (include/mcba.h)."""
    buf = C.create_string_buffer(64)
    self._ck(self.lib.mcba_peer_export(self.h, int(cap_doubles), buf))
    return buf.raw

  def peer_import(self, handles):
    """handles: list of the 64-byte IPC handles of all ranks, in rank order."""
    blob = b"".join(handles)
    self._ck(self.lib.mcba_peer_import(self.h, blob))

  # ---- problem ----------------------------------------------------------------------------------
  def upload(self, model, optimize_bits, dims, idx, obs, board_points):
    Cn, F, B, P = (int(v) for v in dims)
    idx = np.ascontiguousarray(idx, dtype=np.int32).reshape(-1, 4)
    cols = [np.ascontiguousarray(idx[:, j]) for j in range(4)]
    obs = nat.f64(obs).reshape(-1, 2)
    bp = nat.f64(board_points).reshape(B, P, 3)
    d = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], int(optimize_bits), idx.shape[0])
    self._ck(self.lib.mcba_upload(self.h, C.byref(d), nat.iptr(cols[0]), nat.iptr(cols[1]), nat.iptr(cols[2]),
                                  nat.iptr(cols[3]), nat.dptr(obs), nat.dptr(bp)))
    self.desc = d
    self.model = model
    self.kint = 5 + nat.DIST_SIZES[model]
    self.N = idx.shape[0]

  def upload_dense(self, model, optimize_bits, mask, points, board_points, view_valid=None):
    """Dense [C,F,B,P] mask + [C,F,B,P,2] observations as the reference holds them (point_table, inliers);
    the packing into frame-major corner arrays happens on the device (csrc/pack_kernels.cuh).  With `view_valid` ([C,F,B]) the
    selection is mask & view_valid[..., None], the conjunction taken on the device (calibration.py:73-81 without the host pass)."""
    mask = np.ascontiguousarray(mask)
    Cn, F, B, P = mask.shape
    u8 = lambda a: a.view(np.uint8) if a.dtype == np.bool_ else np.ascontiguousarray(a, dtype=np.uint8)
    m8 = u8(mask)
    # a float32 table (what make_point_table yields for cv2's float32 corners, tables.py:15-17) goes over as it is; anything else as f64
    f32 = np.asarray(points).dtype == np.float32
    pts = np.ascontiguousarray(points) if f32 else nat.f64(points)
    assert pts.shape == (Cn, F, B, P, 2), f"points {pts.shape} do not match mask {mask.shape}"
    bp = nat.f64(board_points).reshape(B, P, 3)
    d = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], int(optimize_bits), 0)
    n = C.c_int64()
    if f32:
      v8 = None if view_valid is None else u8(np.ascontiguousarray(view_valid))
      self._ck(self.lib.mcba_upload_dense_views_f32(self.h, C.byref(d), m8.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                    None if v8 is None else v8.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                    pts.ctypes.data_as(C.POINTER(C.c_float)), nat.dptr(bp), C.byref(n)))
    elif view_valid is None:
      self._ck(self.lib.mcba_upload_dense(self.h, C.byref(d), m8.ctypes.data_as(C.POINTER(C.c_uint8)), nat.dptr(pts),
                                          nat.dptr(bp), C.byref(n)))
    else:
      v8 = u8(np.ascontiguousarray(view_valid))
      assert v8.shape == (Cn, F, B), f"view_valid {v8.shape} does not match mask {mask.shape}"
      self._ck(self.lib.mcba_upload_dense_views(self.h, C.byref(d), m8.ctypes.data_as(C.POINTER(C.c_uint8)),
                                                v8.ctypes.data_as(C.POINTER(C.c_uint8)), nat.dptr(pts), nat.dptr(bp), C.byref(n)))
    d.N = n.value
    self.desc = d
    self.model = model
    self.kint = 5 + nat.DIST_SIZES[model]
    self.N = n.value

  # ---- resident point table (include/mcba.h "resident point table") ------------------------------
  def _table_ready(self, d, model, n):
    d.N = n
    self.desc, self.model, self.kint, self.N = d, model, 5 + nat.DIST_SIZES[model], n

  def table_upload(self, model, optimize_bits, valid, points, board_points):
    """Keep the whole [C,F,B,P] table on the device: `valid` mask + observations.  Inliers start equal to `valid`,
    which is also the packed selection; returns the number of valid corners."""
    valid = np.ascontiguousarray(valid)
    Cn, F, B, P = valid.shape
    v8 = valid.view(np.uint8) if valid.dtype == np.bool_ else np.ascontiguousarray(valid, dtype=np.uint8)
    pts = nat.f64(points)
    assert pts.shape == (Cn, F, B, P, 2), f"points {pts.shape} do not match mask {valid.shape}"
    bp = nat.f64(board_points).reshape(B, P, 3)
    d = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], int(optimize_bits), 0)
    n = C.c_int64()
    self._ck(self.lib.mcba_table_upload(self.h, C.byref(d), v8.ctypes.data_as(C.POINTER(C.c_uint8)), nat.dptr(pts),
                                        nat.dptr(bp), C.byref(n)))
    self._table_ready(d, model, n.value)
    return n.value

  @staticmethod
  def _detections(dims, det_start, det_ids, det_xy, board_points):
    """Detection lists as the C ABI takes them: list w = (c*F+f)*B+b holds point ids det_ids[det_start[w]:det_start[w+1]] and their
    pixel corners det_xy.  Returns (C, F, B, P), the offsets, ids, corners and board points as contiguous arrays."""
    Cn, F, B, P = (int(v) for v in dims)
    det_start = np.ascontiguousarray(det_start, dtype=np.int64)
    assert det_start.shape == (Cn * F * B + 1,), f"expected {Cn * F * B + 1} list offsets, got {det_start.shape}"
    det_ids = np.ascontiguousarray(det_ids, dtype=np.int32).reshape(-1)
    det_xy = nat.f64(det_xy).reshape(-1, 2)
    assert det_ids.size == det_xy.shape[0] == int(det_start[-1]), "detection arrays do not match the offsets"
    return (Cn, F, B, P), det_start, det_ids, det_xy, nat.f64(board_points).reshape(B, P, 3)

  def table_from_detections(self, model, optimize_bits, dims, det_start, det_ids, det_xy, board_points):
    """Build the table on the device from detection lists: list w = (c*F+f)*B+b holds point ids
    det_ids[det_start[w]:det_start[w+1]] and their pixel corners det_xy (what tables.make_point_table consumes)."""
    (Cn, F, B, P), det_start, det_ids, det_xy, bp = self._detections(dims, det_start, det_ids, det_xy, board_points)
    d = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], int(optimize_bits), 0)
    n = C.c_int64()
    self._ck(self.lib.mcba_table_from_detections(self.h, C.byref(d), det_start.ctypes.data_as(C.POINTER(C.c_int64)),
                                                 nat.iptr(det_ids), nat.dptr(det_xy), nat.dptr(bp), C.byref(n)))
    self._table_ready(d, model, n.value)
    return n.value

  def pnp_views(self, model, dims, det_start, det_ids, det_xy, board_points, intrinsics, board_grid):
    """Batched board-pose initialisation (include/mcba.h mcba_pnp_views): list w = (c*F+f)*B+b of detected point ids and pixel
    corners -> (poses [C,F,B,4,4], reprojection RMS [C,F,B], corner counts [C,F,B], valid [C,F,B])."""
    (Cn, F, B, P), det_start, det_ids, det_xy, bp = self._detections(dims, det_start, det_ids, det_xy, board_points)
    nv = Cn * F * B
    intr = nat.f64(intrinsics).reshape(Cn, 5 + nat.DIST_SIZES[model])
    grid = np.ascontiguousarray(board_grid, dtype=np.int32).reshape(B, 5)
    poses, err = np.zeros((max(nv, 1), 4, 4)), np.zeros(max(nv, 1))
    npts, ok = np.zeros(max(nv, 1), np.int32), np.zeros(max(nv, 1), np.uint8)
    d = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], 0, 0)
    self._ck(self.lib.mcba_pnp_views(self.h, C.byref(d), det_start.ctypes.data_as(C.POINTER(C.c_int64)), nat.iptr(det_ids), nat.dptr(det_xy),
                                     nat.dptr(bp), nat.dptr(intr), nat.iptr(grid), nat.dptr(poses), nat.dptr(err), nat.iptr(npts),
                                     ok.ctypes.data_as(C.POINTER(C.c_uint8))))
    return (poses[:nv].reshape(Cn, F, B, 4, 4), err[:nv].reshape(Cn, F, B), npts[:nv].reshape(Cn, F, B), ok[:nv].reshape(Cn, F, B).astype(bool))

  def intrinsic_init(self, model, dims, det_start, det_ids, det_xy, board_points, board_grid, image_sizes, view_use, fix_aspect=False):
    """Initialisation of single-camera intrinsic calibration (include/mcba.h mcba_intrinsic_init) for every camera at once: list
    w = (c*F+f)*B+b of detected point ids and pixel corners, view_use [C,F,B] the views of this round -> (K0 parameters [C, 5+nd] with
    zero distortion, initial board-wrt-camera poses [C,F,B,4,4], ok [C,F,B])."""
    (Cn, F, B, P), det_start, det_ids, det_xy, bp = self._detections(dims, det_start, det_ids, det_xy, board_points)
    nv = Cn * F * B
    grid = np.ascontiguousarray(board_grid, dtype=np.int32).reshape(B, 5)
    sizes = np.ascontiguousarray(image_sizes, dtype=np.int32).reshape(Cn, 2)
    use = np.ascontiguousarray(view_use, dtype=np.uint8).reshape(nv)
    intr = np.zeros((Cn, 5 + nat.DIST_SIZES[model]))
    poses, ok = np.zeros((max(nv, 1), 4, 4)), np.zeros(max(nv, 1), np.uint8)
    d = nat.ProblemDesc(Cn, F, B, P, nat.MODEL_IDS[model], nat.OPT_FIX_ASPECT if fix_aspect else 0, 0)
    u8 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint8))
    self._ck(self.lib.mcba_intrinsic_init(self.h, C.byref(d), det_start.ctypes.data_as(C.POINTER(C.c_int64)), nat.iptr(det_ids),
                                          nat.dptr(det_xy), nat.dptr(bp), nat.iptr(grid), nat.iptr(sizes), u8(use), nat.dptr(intr),
                                          nat.dptr(poses), u8(ok)))
    return intr, poses[:nv].reshape(Cn, F, B, 4, 4), ok[:nv].reshape(Cn, F, B).astype(bool)

  def view_errors(self):
    """Per-view sums of squared pixel errors and corner counts of the uploaded problem at the current parameters, both [C,F,B]
    (zero where there is no view): include/mcba.h mcba_view_errors."""
    shape = self._dense_shape()[:3]
    n = max(int(np.prod(shape)), 1)
    sumsq, count = np.zeros(n), np.zeros(n, np.int64)
    self._ck(self.lib.mcba_view_errors(self.h, nat.dptr(sumsq), count.ctypes.data_as(C.POINTER(C.c_int64))))
    m = int(np.prod(shape))
    return sumsq[:m].reshape(shape), count[:m].reshape(shape)

  def _dense_shape(self):
    d = self.desc
    return (d.C, d.F, d.B, d.P)

  def table_download(self, points=True):
    valid = np.zeros(self._dense_shape(), dtype=np.uint8)
    pts = np.zeros((*self._dense_shape(), 2)) if points else None
    self._ck(self.lib.mcba_table_download(self.h, valid.ctypes.data_as(C.POINTER(C.c_uint8)), nat.dptr(pts)))
    return valid.astype(bool), pts

  def table_set_inliers(self, mask=None):
    if mask is None:
      self._ck(self.lib.mcba_table_set_inliers(self.h, None)); return
    mask = np.ascontiguousarray(mask)
    assert mask.shape == self._dense_shape(), f"mask {mask.shape} does not match the table {self._dense_shape()}"
    m8 = mask.view(np.uint8) if mask.dtype == np.bool_ else np.ascontiguousarray(mask, dtype=np.uint8)
    self._ck(self.lib.mcba_table_set_inliers(self.h, m8.ctypes.data_as(C.POINTER(C.c_uint8))))

  def table_get_inliers(self):
    mask = np.zeros(self._dense_shape(), dtype=np.uint8)
    self._ck(self.lib.mcba_table_get_inliers(self.h, mask.ctypes.data_as(C.POINTER(C.c_uint8))))
    return mask.astype(bool)

  def table_select(self, which):
    """which: 'valid' or 'inliers' -- the corner set the solver and the residual entry points then work on."""
    n = C.c_int64()
    self._ck(self.lib.mcba_table_select(self.h, {"valid": nat.TABLE_VALID, "inliers": nat.TABLE_INLIERS}[which], C.byref(n)))
    self.N = self.desc.N = n.value
    return n.value

  def table_errors(self):
    """Per-corner pixel error over `valid` at the current parameters; stays on the device, sorted.  Returns the counts and
    sums of squares of the valid and the inlier set (tables.py:244-249, calibration.py:303-310)."""
    st = nat.TableStats()
    self._ck(self.lib.mcba_table_errors(self.h, C.byref(st)))
    self.N = self.desc.N = st.n_valid
    return SolveInfo(n_valid=st.n_valid, n_inliers=st.n_inliers, sumsq_valid=st.sumsq_valid, sumsq_inliers=st.sumsq_inliers)

  def table_error_ranks(self, which, ranks):
    ranks = np.ascontiguousarray(ranks, dtype=np.int64).reshape(-1)
    out = np.zeros(max(ranks.size, 1))
    self._ck(self.lib.mcba_table_error_ranks(self.h, {"valid": nat.TABLE_VALID, "inliers": nat.TABLE_INLIERS}[which],
                                             ranks.ctypes.data_as(C.POINTER(C.c_int64)), ranks.size, nat.dptr(out)))
    return out[:ranks.size]

  def table_count_below(self, which, thresholds):
    """Number of errors of the chosen set below each threshold (binary search in the sorted errors on the device)."""
    t = nat.f64(thresholds).reshape(-1)
    out = np.zeros(max(t.size, 1), np.int64)
    self._ck(self.lib.mcba_table_count_below(self.h, {"valid": nat.TABLE_VALID, "inliers": nat.TABLE_INLIERS}[which], nat.dptr(t), t.size,
                                             out.ctypes.data_as(C.POINTER(C.c_int64))))
    return out[:t.size]

  def table_quantile(self, which, n, q):
    """np.quantile(errors of the chosen set, q), computed from order statistics fetched from the device."""
    from .outliers import quantile_from_sorted
    return quantile_from_sorted(lambda r: self.table_error_ranks(which, r), n, q)

  def table_reject(self, threshold):
    """inliers = valid & (error < threshold) with the errors of the last table_errors(); returns (n_valid, n_keep)."""
    nv, nk = C.c_int64(), C.c_int64()
    self._ck(self.lib.mcba_table_reject(self.h, float(threshold), C.byref(nv), C.byref(nk)))
    return nv.value, nk.value

  def set_params(self, cam_rt, board_rt, frame_rt, intrinsics):
    d = self.desc
    cam_rt, board_rt, intrinsics = nat.f64(cam_rt), nat.f64(board_rt), nat.f64(intrinsics)
    frame_rt = nat.f64(frame_rt) if d.F else np.zeros((1, 6))
    assert cam_rt.size == 6 * d.C and board_rt.size == 6 * d.B and intrinsics.size == self.kint * d.C
    assert d.F == 0 or frame_rt.size == 6 * d.F
    self._ck(self.lib.mcba_set_params(self.h, nat.dptr(cam_rt), nat.dptr(board_rt), nat.dptr(frame_rt), nat.dptr(intrinsics)))

  def set_state_matrices(self, pose_matrices, intrinsics):
    """Parameter state from 4x4 pose matrices f64[C+B+F,4,4] (cameras, boards, frames): the device converts to rtvecs."""
    d = self.desc
    mats, intrinsics = nat.f64(pose_matrices), nat.f64(intrinsics)
    assert mats.shape == (d.C + d.B + d.F, 4, 4) and intrinsics.size == self.kint * d.C
    self._ck(self.lib.mcba_set_state_matrices(self.h, nat.dptr(mats), nat.dptr(intrinsics)))

  def get_state_matrices(self):
    d = self.desc
    mats, intr = np.zeros((d.C + d.B + d.F, 4, 4)), np.zeros((d.C, self.kint))
    self._ck(self.lib.mcba_get_state_matrices(self.h, nat.dptr(mats), nat.dptr(intr)))
    return mats[:d.C], mats[d.C:d.C + d.B], mats[d.C + d.B:], intr

  # ---- motion-model state (include/mcba.h mcba_set_rolling / mcba_set_hand_eye) ----------------------
  def set_rolling(self, end_pose_matrices, image_heights):
    """RollingFrames: end poses f64[F,4,4] (the frames of set_state_matrices are the start poses) and the image height of
    every camera, which turns a corner's observed row into its blend weight (rolling_frames.py:15-19)."""
    d = self.desc
    mats, h = nat.f64(end_pose_matrices), nat.f64(image_heights)
    assert mats.shape == (d.F, 4, 4) and h.shape == (d.C,)
    self._ck(self.lib.mcba_set_rolling(self.h, nat.dptr(mats), nat.dptr(h)))

  def get_rolling(self):
    mats = np.zeros((max(self.desc.F, 1), 4, 4))
    self._ck(self.lib.mcba_get_rolling(self.h, nat.dptr(mats)))
    return mats[:self.desc.F]

  def set_hand_eye(self, base_wrt_gripper, world_wrt_base, gripper_wrt_camera):
    """HandEye: the fixed arm poses f64[F,4,4] and the two optimised transforms f64[4,4] (hand_eye.py:20-33)."""
    arm, w, g = nat.f64(base_wrt_gripper), nat.f64(world_wrt_base), nat.f64(gripper_wrt_camera)
    assert arm.shape == (self.desc.F, 4, 4) and w.shape == (4, 4) and g.shape == (4, 4)
    self._ck(self.lib.mcba_set_hand_eye(self.h, nat.dptr(arm), nat.dptr(w), nat.dptr(g)))

  def get_hand_eye(self):
    w, g = np.zeros((4, 4)), np.zeros((4, 4))
    self._ck(self.lib.mcba_get_hand_eye(self.h, nat.dptr(w), nat.dptr(g)))
    return w, g

  def get_params(self):
    d = self.desc
    out = (np.zeros((d.C, 6)), np.zeros((d.B, 6)), np.zeros((max(d.F, 1), 6)), np.zeros((d.C, self.kint)))
    self._ck(self.lib.mcba_get_params(self.h, *[nat.dptr(a) for a in out]))
    return out[0], out[1], out[2][:d.F], out[3]

  @property
  def num_params(self):
    n = C.c_int64()
    self._ck(self.lib.mcba_num_params(self.h, C.byref(n)))
    return n.value

  @property
  def param_vec(self):
    x = np.zeros(max(self.num_params, 1))
    self._ck(self.lib.mcba_get_param_vec(self.h, nat.dptr(x)))
    return x[:self.num_params]

  def set_param_vec(self, x):
    x = nat.f64(x)
    assert x.size == self.num_params, f"inconsistent parameter sizes, got {x.size}, expected {self.num_params}"
    if x.size: self._ck(self.lib.mcba_set_param_vec(self.h, nat.dptr(x)))

  # ---- parity hooks -----------------------------------------------------------------------------
  def residuals(self, x=None, with_cost=False):
    r = np.zeros(max(2 * self.N, 1))
    cost = C.c_double()
    if x is not None:
      x = nat.f64(x)
      assert x.size == self.num_params
    self._ck(self.lib.mcba_residuals(self.h, nat.dptr(x) if x is not None and x.size else None, nat.dptr(r),
                                     C.cast(C.byref(cost), C.POINTER(C.c_double)) if with_cost else None))
    r = r[:2 * self.N]
    return (r, cost.value) if with_cost else r

  def linearize(self, x=None):
    n = self.num_params
    JtJ, Jtr = np.zeros((max(n, 1), max(n, 1))), np.zeros(max(n, 1))
    cost = C.c_double()
    if x is not None: x = nat.f64(x)
    self._ck(self.lib.mcba_linearize(self.h, nat.dptr(x) if x is not None and x.size else None, nat.dptr(JtJ), nat.dptr(Jtr),
                                     C.cast(C.byref(cost), C.POINTER(C.c_double))))
    return JtJ[:n, :n], Jtr[:n], cost.value

  def reprojection_error(self):
    e = np.zeros(max(self.N, 1))
    self._ck(self.lib.mcba_reprojection_error(self.h, nat.dptr(e)))
    return e[:self.N]

  # ---- the solve --------------------------------------------------------------------------------
  def solve(self, ftol=1e-8, xtol=1e-8, gtol=1e-8, f_scale=1.0, max_nfev=100, loss="linear"):
    if loss not in nat.LOSS_IDS:
      raise ValueError(f"`loss` must be one of {list(nat.LOSS_IDS)} or a callable.")
    opts = nat.SolveOpts(ftol, xtol, gtol, f_scale, int(max_nfev), nat.LOSS_IDS[loss])
    res = nat.SolveResult()
    cap = int(max_nfev) + 2
    log = (nat.LogRow * cap)()
    self._ck(self.lib.mcba_solve(self.h, C.byref(opts), C.byref(res), log, cap))
    rows = [(r.iteration, r.nfev, r.cost, r.cost_reduction, r.step_norm, r.optimality) for r in log[:res.n_log]]
    return SolveInfo(cost=res.cost, initial_cost=res.initial_cost, optimality=res.optimality, nfev=res.nfev,
                     njev=res.njev, status=res.status, message=nat.STATUS_MESSAGES.get(res.status, ""),
                     device_ms=res.device_ms, kernel_launches=res.kernel_launches, log=rows,
                     chol_retries=res.chol_retries)

  # ---- measurement hooks ------------------------------------------------------------------------
  def bench_launch(self, which, repeats=1):
    self._ck(self.lib.mcba_bench_launch(self.h, int(which), int(repeats)))

  def bench_info(self, which):
    a, b, c = C.c_int64(), C.c_int64(), C.c_int32()
    self._ck(self.lib.mcba_bench_info(self.h, int(which), C.byref(a), C.byref(b), C.byref(c)))
    return dict(corners=a.value, bytes_per_launch=b.value, launches_per_call=c.value)


def format_log(rows):
  """scipy's verbose=2 iteration table (scipy/optimize/_lsq/common.py print_header_nonlinear /
  print_iteration_nonlinear), which the reference forwards to its logger (calibration.py:208)."""
  lines = ["{:^15}{:^15}{:^15}{:^15}{:^15}{:^15}".format("Iteration", "Total nfev", "Cost", "Cost reduction", "Step norm", "Optimality")]
  for it, nfev, cost, red, step, opt in rows:
    red_s = " " * 15 if red is None or np.isnan(red) else f"{red:^15.2e}"
    step_s = " " * 15 if step is None or np.isnan(step) else f"{step:^15.2e}"
    lines.append(f"{it:^15}{nfev:^15}{cost:^15.4e}{red_s}{step_s}{opt:^15.2e}")
  return lines
