/* mcba.h — C-ABI of the H100 bundle-adjustment engine (libmcba.so).
 *
 * Drop-in boundary for ONE numeric seam of the reference (multical):
 *     scipy.optimize.least_squares(evaluate, self.param_vec, jac_sparsity=..., x_scale='jac',
 *                                  f_scale=..., ftol=..., max_nfev=..., method='trf', loss=...)
 *     -- multical/optimization/calibration.py:209-210 (inside Calibration.bundle_adjust, 199-212)
 * plus the residual closure it drives (calibration.py:204-206) and the reprojection-error /
 * outlier statistics that bracket every call (calibration.py:134-141, 240-252; tables.py:244-249).
 *
 * Plain C types only: opaque handle, host pointers + sizes, integer status (0 = ok; message via
 * mcba_last_error).  All host arrays are borrowed for the duration of the call and copied.
 * There is no CPU fallback: every entry point fails with MCBA_ERR_CUDA if no sm_90 device works.
 *
 * Index contract (bit-exact with the reference): packed corner k corresponds to row k of
 * np.argwhere(calib.inliers) = (camera, frame, board, point) in row-major order of the dense
 * [C,F,B,P] table (calibration.py:206 boolean-mask order); residual vector element 2k is u, 2k+1 is v.
 * Parameter vector layout = reference order (calibration.py:146-153, parameters.py:104-106):
 *   [camera_poses 6C][board_poses 6B][motion 6F | 12F rolling | 12 hand-eye][cameras (5+nd)C][boards 3*B*P]   (enabled blocks only; the boards
 *   block is the padded stack of tables.stack_boards -- the host strips the padding of boards with fewer points)
 *   pose = [rx ry rz tx ty tz] (transform/rtvec.py:16-27), camera = [fx fy cx cy skew dist...]
 *   (camera.py:144-155).
 */
#ifndef MCBA_H
#define MCBA_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct mcba_ctx mcba_ctx;

/* MCBA_ERR_CUDA: a CUDA call failed, or a host allocation did (the message says which) */
enum { MCBA_OK = 0, MCBA_ERR_ARG = 1, MCBA_ERR_CUDA = 2, MCBA_ERR_STATE = 3, MCBA_ERR_NCCL = 4,
       MCBA_ERR_NONFINITE = 5, MCBA_ERR_UNSUPPORTED = 6,
       MCBA_ERR_DEGENERATE = 7 /* input too degenerate for the estimate asked for (mcba_hand_eye_vote) */ };

/* camera models: camera.py:43-48 (cv2.projectPoints, 5/8/12/14 coefficients) and
 * camera_fisheye.py:113-117 (cv2.fisheye.projectPoints, 4 coefficients) */
enum { MCBA_MODEL_STANDARD = 0, MCBA_MODEL_RATIONAL = 1, MCBA_MODEL_THIN_PRISM = 2, MCBA_MODEL_FISHEYE = 3,
       MCBA_MODEL_TILTED = 4 /* 14 coefficients: thin prism + sensor tilt (tauX, tauY) */ };

/* loss names of scipy.optimize.least_squares (config/arguments.py:59) */
enum { MCBA_LOSS_LINEAR = 0, MCBA_LOSS_SOFT_L1 = 1, MCBA_LOSS_HUBER = 2, MCBA_LOSS_CAUCHY = 3, MCBA_LOSS_ARCTAN = 4 };

/* which parameter blocks are free: Calibration.optimize (calibration.py:28-35,155-161) */
enum { MCBA_OPT_CAMERA_POSES = 1, MCBA_OPT_BOARD_POSES = 2, MCBA_OPT_MOTION = 4, MCBA_OPT_CAMERAS = 8,
       MCBA_OPT_BOARDS = 16 /* board points as parameters (board/charuco.py:112-117); block layout = padded [B][P][3] */,
       MCBA_OPT_FIX_ASPECT = 256 /* camera.py:147-148,159-160 */ };
/* motion model = the `motion` argument of Calibration (calibration.py:44-46), or-ed into mcba_problem_desc.optimize:
 *   (none)                StaticFrames: one rig pose per frame (motion/static_frames.py:29-42)
 *   MCBA_MOTION_ROLLING   RollingFrames: a start and an end pose per frame; a corner is transformed by both and the two
 *                         camera-frame points are blended by its observed row / image height (motion/rolling_frames.py:15-41,
 *                         66-150).  motion block of the parameter vector = [start F x 6 | end F x 6] (135-140).
 *   MCBA_MOTION_HAND_EYE  HandEye: frame pose f = gripper_wrt_camera @ base_wrt_gripper[f] @ world_wrt_base with the arm
 *                         poses fixed (motion/hand_eye.py:14-90).  motion block = [world_wrt_base 6 | gripper_wrt_camera 6]
 *                         (76-81), shared by every residual (89-90).
 */
enum { MCBA_MOTION_ROLLING = 1 << 16, MCBA_MOTION_HAND_EYE = 1 << 17 };

typedef struct {
  int32_t C, F, B, P;       /* Calibration.size (calibration.py:64-67); F = frames held by THIS rank   */
  int32_t model;            /* MCBA_MODEL_*                                                            */
  int32_t optimize;         /* bitmask MCBA_OPT_*                                                      */
  int64_t N;                /* packed inlier corners held by this rank                                 */
} mcba_problem_desc;

typedef struct {
  double ftol, xtol, gtol;  /* scipy defaults 1e-8; the reference passes ftol=tolerance (1e-4)         */
  double f_scale;           /* least_squares f_scale                                                   */
  int32_t max_nfev;         /* max_iterations -> max_nfev (calibration.py:199,210)                     */
  int32_t loss;             /* MCBA_LOSS_*                                                             */
} mcba_solve_opts;

typedef struct {            /* one row of scipy's verbose=2 table (calibration.py:208)                 */
  int32_t iteration, nfev;
  double cost, cost_reduction, step_norm, optimality;
} mcba_log_row;

typedef struct {
  double cost, initial_cost, optimality;
  int32_t nfev, njev, status;   /* scipy termination status -1,0,1,2,3,4 (_lsq/common.py:705-717)      */
  int32_t n_log;                /* rows written to the log buffer                                      */
  double device_ms;             /* CUDA-event time of the solve on the context stream                  */
  int32_t kernel_launches;      /* kernels launched by this solve                                      */
  int32_t chol_retries;
} mcba_solve_result;

/* -- context ------------------------------------------------------------------------------------ */
int  mcba_create(int device_ordinal, mcba_ctx** out);
void mcba_destroy(mcba_ctx* ctx);
const char* mcba_last_error(const mcba_ctx* ctx);   /* ctx may be NULL: returns the creation error     */
int  mcba_set_stream(mcba_ctx* ctx, void* cuda_stream);   /* e.g. torch.cuda.current_stream().cuda_stream */
int  mcba_version(void);

/* -- multi-GPU: one context per process/GPU; frames are sharded across ranks (SURVEY.md §8e) ----
 * mcba_comm_init records (rank, world <= 16); mcba_comm_unique_id is kept for the usual bootstrap shape (rank 0 makes an id, the host
 * broadcasts it) and returns a constant tag.  The exchanges of a solve -- shared gradient / diagonal / cost, g_h^T A g_h, the reduced
 * normal equations S and rhs, the subspace sums: four per LM iteration -- run INSIDE the solver kernel over NVLink peer memory
 * (push to every rank's slot, sequence flag, reduce in rank order: bit-identical results on every rank; csrc/lm_kernel.cuh exchange()).
 * Every rank exports one buffer as an IPC handle (64 bytes), the host all-gathers the handles (torch.distributed / NCCL is the
 * bootstrap), every rank imports all of them.  cap_doubles per slot must hold n_s^2 + 2 n_s + 16; a rank that stops answering makes
 * its peers' solves fail with MCBA_ERR_NCCL after a bounded wait instead of hanging their GPUs. */
int  mcba_comm_unique_id(mcba_ctx* ctx, char out_id[128]);
int  mcba_comm_init(mcba_ctx* ctx, const char id[128], int rank, int world);
int  mcba_peer_export(mcba_ctx* ctx, int64_t cap_doubles, char out_handle[64]);
int  mcba_peer_import(mcba_ctx* ctx, const char* handles /* world x 64 bytes in rank order */);

/* -- problem upload: replaces what `evaluate` closes over (calibration.py:204-206) --------------
 * The reference's own wire format: valid uint8[C][F][B][P] selects the corners (calib.inliers, calibration.py:78-81, or
 * point_table.valid as detected), points [C][F][B][P][2] are their pixels (point_table.points, tables.make_point_table,
 * tables.py:68-81), board_points f64[B][P][3] = tables.stack_boards(boards).points (tables.py:385-394).  view_valid uint8[C][F][B]
 * (may be NULL: all views valid) is the other part the reference builds the mask from (calibration.py:73-81: camera_poses.valid x
 * motion.valid x board_poses.valid); the conjunction valid & view_valid is taken on the device, so the caller hands the detection
 * table over untouched.  point_type MCBA_POINTS_F64 or MCBA_POINTS_F32: make_point_table keeps the dtype of the detector's corners
 * (tables.py:15-17 fill_sparse: `dtype=values.dtype`; cv2's aruco / charuco detectors return float32), so a float32 table IS the
 * reference's table for real detections -- half the bytes over the link; the packed observations are f64 (exact).
 * Packing into the frame-major corner arrays happens on the device; *n_corners receives the number of selected corners.  The packed
 * order seen through mcba_residuals is np.argwhere(valid & view_valid) order (frame ids local to this rank).
 * Every upload (also mcba_table_upload / mcba_table_from_detections) replaces the context's problem: a refused one, for its inputs or
 * later (too many boards for the linearisation kernel: MCBA_ERR_UNSUPPORTED), leaves none, and the entry points that need one fail
 * with MCBA_ERR_STATE until an upload succeeds. */
enum { MCBA_POINTS_F64 = 0, MCBA_POINTS_F32 = 1 };
int  mcba_upload_dense(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const uint8_t* view_valid,
                       const void* points, int32_t point_type, const double* board_points, int64_t* n_corners);

/* full parameter state (also the values of disabled/fixed blocks):
 * cam_rt f64[C][6], board_rt f64[B][6], frame_rt f64[F][6] (PoseSet.params, pose_set.py:51-53),
 * intrinsics f64[C][5+nd] (Camera.params, camera.py:144-155)                                      */
int  mcba_set_params(mcba_ctx* ctx, const double* cam_rt, const double* board_rt,
                     const double* frame_rt, const double* intrinsics);
int  mcba_get_params(mcba_ctx* ctx, double* cam_rt, double* board_rt, double* frame_rt, double* intrinsics);
/* the same state as 4x4 pose matrices, f64[C+B+F][4][4] in the order cameras, boards, frames (PoseSet.poses,
 * pose_set.py:40-42): matrix <-> rtvec (transform/rtvec.py:24-32) is done on the device */
int  mcba_set_state_matrices(mcba_ctx* ctx, const double* pose_matrices, const double* intrinsics);
int  mcba_get_state_matrices(mcba_ctx* ctx, double* pose_matrices, double* intrinsics);
/* motion-model state (after the upload, next to mcba_set_params / mcba_set_state_matrices):
 * rolling: the frames of the calls above are the START poses (mcba_set_params: frame_rt is f64[F][12], start | end of a
 *   frame adjacent); end poses f64[F][4][4] and image heights f64[C] (rolling_times, rolling_frames.py:15-19) come here.
 * hand-eye: the frames of the calls above are ignored on input (mcba_get_state_matrices returns the derived frame poses);
 *   base_wrt_gripper f64[F][4][4] (constants), world_wrt_base and gripper_wrt_camera f64[4][4] (the parameters). */
int  mcba_set_rolling(mcba_ctx* ctx, const double* end_pose_matrices, const double* image_heights);
int  mcba_get_rolling(mcba_ctx* ctx, double* end_pose_matrices);
int  mcba_set_hand_eye(mcba_ctx* ctx, const double* base_wrt_gripper, const double* world_wrt_base,
                       const double* gripper_wrt_camera);
int  mcba_get_hand_eye(mcba_ctx* ctx, double* world_wrt_base, double* gripper_wrt_camera);
/* single intrinsic parameters held fixed (OpenCV's CALIB_FIX_K1..K3, CALIB_ZERO_TANGENT_DIST, CALIB_FIX_PRINCIPAL_POINT, ...):
 * fixed uint8[5+nd] in Camera.params order [fx fy cx cy skew dist...], 1 = fixed, the same for every camera (NULL = none).  A fixed
 * parameter keeps its place in param_vec and its current value: its row and column of J^T J and its entry of J^T r are zero
 * (mcba_linearize shows them), and mcba_solve / mcba_set_param_vec leave it bit for bit.  Harmless without MCBA_OPT_CAMERAS.
 * Entries other than 0 / 1, or fx and fy fixed apart under MCBA_OPT_FIX_ASPECT (fy follows fx), fail with MCBA_ERR_ARG.  Every upload
 * clears the mask. */
int  mcba_set_fixed_intrinsics(mcba_ctx* ctx, const uint8_t* fixed);
/* the trust-region step of mcba_solve (scipy least_squares' tr_solver):
 *   MCBA_TR_SUBSPACE  the exact Gauss-Newton direction, then the step in the 2-D subspace span{g, gn} (the default);
 *   MCBA_TR_EXACT     the full trust-region subproblem, tr_solver='exact': the Gauss-Newton step if A = D J^T J D is nonsingular and it
 *                     lies inside the radius, else Newton iterations on the Levenberg-Marquardt parameter alpha (at most 10, each a
 *                     factorisation of A + alpha I) until ||p(alpha)|| is within 1% of the radius.  Slower per iteration; reaches the
 *                     minimum of long curved valleys where the subspace step stops on xtol above it (the rational intrinsics).
 * Other values fail with MCBA_ERR_ARG.  A solve on several ranks in MCBA_TR_EXACT fails with MCBA_ERR_UNSUPPORTED.  Every upload resets
 * the mode to MCBA_TR_SUBSPACE. */
enum { MCBA_TR_SUBSPACE = 0, MCBA_TR_EXACT = 1 };
int  mcba_set_trust_region(mcba_ctx* ctx, int32_t mode);
/* alpha iterations of the last mcba_solve summed over its trial steps (scipy's n_iter of solve_lsq_trust_region: 0 for a Gauss-Newton
 * step); 0 after a MCBA_TR_SUBSPACE solve */
int  mcba_last_alpha_iterations(mcba_ctx* ctx, int32_t* total);
int  mcba_num_params(mcba_ctx* ctx, int64_t* n);      /* length of param_vec for the enabled blocks    */
int  mcba_get_param_vec(mcba_ctx* ctx, double* x);    /* Parameters.param_vec (parameters.py:44-46)    */
int  mcba_set_param_vec(mcba_ctx* ctx, const double* x);   /* with_param_vec (parameters.py:48-50)     */

/* -- parity hooks -------------------------------------------------------------------------------
 * residuals: r f64[2N] = evaluate(x) (calibration.py:204-206); cost = 0.5*sum(rho) as scipy.       */
int  mcba_residuals(mcba_ctx* ctx, const double* x /*NULL = current params*/, double* r, double* cost);
/* linearize at x: dense J^T J (f64[n][n], row-major, parameter order of param_vec) and J^T r (f64[n])
 * of the (loss-scaled) residual -- what scipy's FD Jacobian + compute_grad produce (trf.py).       */
int  mcba_linearize(mcba_ctx* ctx, const double* x, double* JtJ, double* Jtr, double* cost);
/* per-corner reprojection error norm, f64[N] (tables.py:244-249 restricted to the packed corners)  */
int  mcba_reprojection_error(mcba_ctx* ctx, double* err);

/* -- the solve: replaces scipy.optimize.least_squares(...) at calibration.py:209-210 ------------ */
int  mcba_solve(mcba_ctx* ctx, const mcba_solve_opts* opts, mcba_solve_result* result,
                mcba_log_row* log, int32_t log_capacity);

/* -- resident point table: the outlier loop without host round trips --------------------------------
 * Calibration.adjust_outliers (calibration.py:250-266) alternates  report -> select threshold (np.quantile of the
 * per-corner error over `valid`, calibration.py:37-40) -> reject_outliers (calibration.py:240-252, errors from
 * tables.reprojection_error, tables.py:244-249) -> bundle_adjust.  With the table resident, the dense
 * [C,F,B,P] observations cross PCIe once; each round moves a few order statistics and one mask count.
 *
 * mcba_table_upload: valid uint8[C][F][B][P] = point_table.valid & pose validity (calibration.py:73-76),
 *   points f64[C][F][B][P][2]; the inlier mask starts equal to `valid`; the packed set is `valid`.
 * mcba_table_from_detections: the same table built on the device from the per-image detection lists the
 *   reference keeps before tables.make_point_table (tables.py:68-81; fill_sparse 15-21): list w = (c*F+f)*B+b
 *   holds det_ids[det_start[w]..det_start[w+1]) (point ids on board b) and det_xy (pixel corners).  Ids outside
 *   [0,P), and an id repeated within one list, fail with MCBA_ERR_ARG.
 * Both reset the parameter state to zero like mcba_upload_dense; set it afterwards.                              */
typedef struct mcba_table_stats {
  int64_t n_valid, n_inliers;          /* corners in `valid` / in the current inlier mask                        */
  double  sumsq_valid, sumsq_inliers;  /* sum of squared pixel errors over each set (mse = sumsq / n)            */
} mcba_table_stats;
enum { MCBA_TABLE_VALID = 0, MCBA_TABLE_INLIERS = 1 };

int  mcba_table_upload(mcba_ctx* ctx, const mcba_problem_desc* desc, const uint8_t* valid, const double* points,
                       const double* board_points, int64_t* n_valid);
int  mcba_table_from_detections(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start,
                                const int32_t* det_ids, const double* det_xy, const double* board_points,
                                int64_t* n_valid);
/* read the resident table back (either pointer may be NULL): valid uint8[C][F][B][P], points f64[C][F][B][P][2] */
int  mcba_table_download(mcba_ctx* ctx, uint8_t* valid, double* points);
/* inlier mask uint8[C][F][B][P]; set: NULL restores inliers = valid, otherwise the mask is and-ed with `valid` */
int  mcba_table_set_inliers(mcba_ctx* ctx, const uint8_t* mask);
int  mcba_table_get_inliers(mcba_ctx* ctx, uint8_t* mask);
/* pack `valid` or the inlier mask as the problem the solver / residual entry points work on; the parameter state
 * is kept.  *n_corners (may be NULL) receives the packed count. */
int  mcba_table_select(mcba_ctx* ctx, int which, int64_t* n_corners);
/* per-corner error over `valid` at the current parameters, kept on the device sorted (all valid, and the inlier
 * subset) for mcba_table_error_ranks / mcba_table_reject; selects MCBA_TABLE_VALID as a side effect. */
int  mcba_table_errors(mcba_ctx* ctx, mcba_table_stats* stats);
/* out[i] = ranks[i]-th smallest error (0-based) of the chosen set -- the order statistics np.quantile interpolates */
int  mcba_table_error_ranks(mcba_ctx* ctx, int which, const int64_t* ranks, int32_t n, double* out);
/* counts[i] = number of errors of the chosen set below thresholds[i]: the other half of a quantile over SEVERAL ranks' tables
 * (frames sharded across GPUs: every rank sorts its own errors; ranks and counts are merged on the host) */
int  mcba_table_count_below(mcba_ctx* ctx, int which, const double* thresholds, int32_t n, int64_t* counts);
/* inliers = valid & (error < threshold) (calibration.py:243-244) with the errors of the last mcba_table_errors;
 * MCBA_ERR_STATE if parameters or selection changed since.  Follow with mcba_table_select(MCBA_TABLE_INLIERS). */
int  mcba_table_reject(mcba_ctx* ctx, double threshold, int64_t* n_valid, int64_t* n_keep);

/* -- batched board-pose initialisation (what feeds the path; SURVEY.md §8f rank 4) -------------------------------
 * Replaces the C*F*B calls of board.estimate_pose_points (board/common.py:36-47: camera.undistort_points, then
 * cv2.solvePnPGeneric with the camera matrix and no distortion) that tables.make_pose_table makes (tables.py:44-66).
 * Detection lists as for mcba_table_from_detections; intrinsics f64[C][5+nd] (Camera.params); board_grid int32[B][5] =
 * {id-grid width, height, id divisor (1 ChArUco corner ids, 4 AprilGrid tag corners), min_points, min_rows} of
 * has_min_detections_grid (board/common.py:30-34; charuco.py:104-106, aprilgrid.py:197-199).
 * Out, per list w = (c*F+f)*B+b: pose f64[4][4] (board wrt camera), reprojection RMS over the 2n scalar residuals as
 * solvePnPGeneric reports it, number of corners, valid flag; a view without the minimum detections gets the reference's
 * invalid_pose (identity, 0, 0, false; tables.py:38).  Does not touch the uploaded problem.                       */
int  mcba_pnp_views(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids,
                    const double* det_xy, const double* board_points, const double* intrinsics, const int32_t* board_grid,
                    double* poses, double* errors, int32_t* num_points, uint8_t* valid);

/* -- single-camera intrinsic calibration (Camera.calibrate, camera.py:68-105: cv2.calibrateCameraExtended without an initial matrix) --
 * mcba_intrinsic_init: the initialisation of every camera at once.  Detection lists and board_grid as for mcba_pnp_views;
 * image_sizes int32[C][2] = (width, height); view_use uint8[C*F*B] selects the views of the current round (list w = (c*F+f)*B+b).
 * Per camera: a homography per used view (board plane z = 0 -> pixels; board points and corners rounded to float32): normalised DLT,
 * refined by Levenberg-Marquardt on its pixel reprojection error as cv2.findHomography does,
 * then OpenCV's initIntrinsicParams2D (what cv2.initCameraMatrix2D exposes): principal point ((w-1)/2, (h-1)/2), (1/fx^2, 1/fy^2) by
 * least squares over two vanishing-point rows per view; desc->optimize & MCBA_OPT_FIX_ASPECT gives fx = fy = their mean.
 * Out: intrinsics f64[C][5+nd] = [fx fy cx cy 0 | zeros] (NaN focal lengths for a camera without a usable view), poses f64[C*F*B][4][4]
 * (board wrt camera, k_pnp_views under K0 and zero distortion: OpenCV's findExtrinsicCameraParams2), ok uint8[C*F*B] (0 for unused views).
 * desc->model == MCBA_MODEL_FISHEYE (CameraFisheye.calibrate, camera_fisheye.py:70-94: cv2.fisheye.calibrate without an initial
 * matrix) replaces the homographies and initIntrinsicParams2D by OpenCV's fisheye start, fx = fy = max(w, h) / 2 and principal point
 * (w/2 - 0.5, h/2 - 0.5) whatever the views, and the poses by k_pnp_views<MCBA_MODEL_FISHEYE> under it (fisheye undistortion, exact at
 * zero distortion, then the pinhole PnP); fix_aspect is ignored.
 * Boards with any z != 0 fail with MCBA_ERR_UNSUPPORTED, as OpenCV refuses non-planar rigs without an initial matrix.  Does not touch
 * the uploaded problem.
 * The solve itself is the engine's own: one camera, the used views as frames (frame pose = board wrt camera), camera and board poses at
 * identity and fixed, optimize = MCBA_OPT_MOTION | MCBA_OPT_CAMERAS [| MCBA_OPT_FIX_ASPECT, never for fisheye: OpenCV's fisheye
 * calibration has no aspect constraint].  It iterates to its own tolerances: the
 * minimum OpenCV's LM approaches, not the point where OpenCV's iteration limit stops it.
 * mcba_view_errors: per view of the packed problem at the current parameters, sumsq f64[C*F*B] = sum of squared pixel errors (u and v)
 * and count int64[C*F*B] = corners (both zero where there is no view): calibrateCameraExtended's perViewErrors = sqrt(sumsq / count). */
int  mcba_intrinsic_init(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids,
                         const double* det_xy, const double* board_points, const int32_t* board_grid, const int32_t* image_sizes,
                         const uint8_t* view_use, double* intrinsics, double* poses, uint8_t* ok);
int  mcba_view_errors(mcba_ctx* ctx, double* sumsq, int64_t* count);

/* -- stereo calibration of a camera pair (stereo_calibrate, camera.py:261-286: cv2.stereoCalibrate; stereo_calibrate_fisheye,
 * camera_fisheye.py:180-205: cv2.fisheye.stereoCalibrate) ---------------------------------------------------------------------------
 * mcba_stereo_init: OpenCV's start.  desc = {C = 2, F = views, B = 1, P, model}; detection lists as for mcba_pnp_views, list w = c*F + f
 * (camera 0 the left one), with no minimum-detections rule; board_points f64[P][3] the pair's object points; intrinsics f64[2][5+nd]
 * (Camera.params order) of both cameras.  Per view, k_pnp_views of both cameras under their intrinsics, then for every view where both
 * poses are valid the relative pose R = R2 R1^T, T = T2 - R T1 (x_right = R x_left + T) and its rotation vector; rt0 f64[6] receives
 * the median of each component over those views (the two middle values averaged for an even count; NaN without such a view).  fp64
 * without floating-point sums: bit-reproducible.  Out: also left_poses f64[F][4][4] (board wrt the left camera) and ok uint8[F] (both
 * poses valid).  Non-planar object points (z != 0) fail with MCBA_ERR_UNSUPPORTED, a view with fewer than 4 points in either camera
 * with MCBA_ERR_DEGENERATE naming the view.  Does not touch the uploaded problem.
 * The solve is the engine's own: C = 2, the views as frames, one board; cameras [I, rt0], frames at left_poses, the board at identity;
 * optimize = MCBA_OPT_CAMERA_POSES | MCBA_OPT_MOTION [| MCBA_OPT_CAMERAS [| MCBA_OPT_FIX_ASPECT] with free intrinsics].  The pair's pose is
 * read in gauge-invariant form, T_cam1 T_cam0^-1, and OpenCV's RMS is sqrt(sum of mcba_view_errors' sumsq / (2 x corners per camera)). */
int  mcba_stereo_init(mcba_ctx* ctx, const mcba_problem_desc* desc, const int64_t* det_start, const int32_t* det_ids, const double* det_xy,
                      const double* board_points, const double* intrinsics, double* rt0, double* left_poses, uint8_t* ok);

/* -- pose-graph initialisation (tables.initialise_poses, tables.py:354-377) ---------------------------------------------------------
 * Every call of align_transforms_robust (transform/matrix.py:140-153) that initialise_poses makes, batched: mean_robust of the relative
 * poses (Ward clustering of their rtvecs, transform/common.py:6-19), the inlier test at 1.5 x the upper quartile of the errors over
 * all rows, mean_robust again over the inliers.  The table is poses f64[C][F][B][4][4] and valid uint8[C][F][B] of make_pose_table.
 * mcba_pose_pairs: estimate_transform (tables.py:149-174) for each (parent, child) of pairs int32[n_pairs][2].  axis 0: cameras, rows
 *   (f, b) f-major, m1 = table[parent], m2 = table[child]; axis 2: boards of the inverted table (estimate_relative_poses_inv), rows (c, f)
 *   c-major, m1 = inv(table[:, :, parent]), m2 = inv(table[:, :, child]).  Out: t f64[n_pairs][4][4], inliers uint8[n_pairs][rows]
 *   (rows = F*B or C*F), n_inliers int32[n_pairs].
 * mcba_pose_times: the rig poses (relative_between_inv per frame): rows (c, b) in np.nonzero order with cam_valid[c] & valid[c, f, b] &
 *   board_valid[b]; m1 = inv(cam[c]), m2 = inv(table[c, f, b] inv(board[b])); times[f] = inv(t), or the identity with times_valid[f] = 0
 *   for a frame without rows.
 * mcba_pose_cluster: mean_robust's clustering alone.  Sets of 6-vectors vecs f64[N][6] (CSR offsets set_start int64[n_sets + 1]) ->
 *   mask uint8[N] of each set's largest cluster.
 * Non-finite poses or vectors fail with MCBA_ERR_NONFINITE.  None of these touches the uploaded problem. */
int  mcba_pose_pairs(mcba_ctx* ctx, int32_t C, int32_t F, int32_t B, const double* poses, const uint8_t* valid, int32_t axis,
                     const int32_t* pairs, int32_t n_pairs, double* t, uint8_t* inliers, int32_t* n_inliers);
int  mcba_pose_times(mcba_ctx* ctx, int32_t C, int32_t F, int32_t B, const double* poses, const uint8_t* valid, const double* cam_poses,
                     const uint8_t* cam_valid, const double* board_poses, const uint8_t* board_valid, double* times, uint8_t* times_valid);
int  mcba_pose_cluster(mcba_ctx* ctx, int32_t n_sets, const int64_t* set_start, const double* vecs, uint8_t* mask);

/* -- non-overlapping camera initialisation (HandEye.initialise_camera_poses, hand_eye/hand_eye.py:35-79) -------------------------------
 * mcba_hand_eye_quads: one cv2.calibrateRobotWorldHandEye(..., CALIB_ROBOT_WORLD_HAND_EYE_SHAH) of master_slave_pair per quadruple
 *   quads int32[n][4] = (master, slave, boardM, boardS) over the images where valid[master, :, boardM] & valid[slave, :, boardS], with
 *   A_i = inv(poses[master, i, boardM]), B_i = inv(poses[slave, i, boardS]) and A X = Z B.  Out: X f64[n][4][4] (slaveCam_wrt_masterCam),
 *   Z f64[n][4][4], n_images int32[n], ok uint8[n]: 0 for fewer than 3 images, for a rotation whose determinant OpenCV calls null, and
 *   for a top singular value of sum kron(R_B, R_A) that is not separated from the second (relative gap below 1e-6: DESIGN.md §3f).
 * mcba_hand_eye_vote: probabilistic_guess (hand_eye/helper.py:5-18) per set of points f64[N][3] (CSR offsets set_start int64[n_sets+1]):
 *   scipy.stats.gaussian_kde densities at the points -> density f64[N], best int32[n_sets] = the argmax within the set (ties: the lowest
 *   index within 1e-12 relative of the maximum).  A set of 3 points or fewer, or with a singular covariance, fails with
 *   MCBA_ERR_DEGENERATE.
 * Non-finite poses or points fail with MCBA_ERR_NONFINITE.  Neither touches the uploaded problem. */
int  mcba_hand_eye_quads(mcba_ctx* ctx, int32_t C, int32_t F, int32_t B, const double* poses, const uint8_t* valid, int32_t n_quads,
                         const int32_t* quads, double* X, double* Z, int32_t* n_images, uint8_t* ok);
int  mcba_hand_eye_vote(mcba_ctx* ctx, int32_t n_sets, const int64_t* set_start, const double* points, double* density, int32_t* best);

/* -- applying a finished calibration (Camera.undistort_map / undistort_points / project, camera.py:113-128; undistort_images,
 * camera.py:244-258; the CameraFisheye twins, camera_fisheye.py:102-117) -----------------------------------------------------------
 * camera f64[5+nd] = [fx fy cx cy skew dist...] of `model` (Camera.params order); K = [[fx skew cx] [0 fy cy] [0 0 1]].  Undistortion is
 * the rectification below with R = I and P = K.
 * mcba_project_points: cv2.projectPoints(points, rvec = 0, tvec = 0, K, dist) (cv2.fisheye.projectPoints): camera-frame points
 *   f64[n][3] -> pixels f64[n][2].
 * mcba_remap_cubic_table: the fixed-point bicubic weights the remap uses, int32[1024][16]: entry (Y & 31) * 32 + (X & 31) for the map
 *   position (X, Y) = rint(32 (x, y)), 4x4 taps row-major from ((X >> 5) - 1, (Y >> 5) - 1).
 * Non-finite camera parameters fail with MCBA_ERR_NONFINITE.  None of these touches the uploaded problem. */
enum { MCBA_IMAGE_UINT8 = 0 };
int  mcba_project_points(mcba_ctx* ctx, int32_t model, const double* camera, int64_t n, const double* points, double* pixels);
int  mcba_remap_cubic_table(mcba_ctx* ctx, int32_t* table);

/* -- rectifying a calibrated pair (cv2.initUndistortRectifyMap / cv2.undistortPoints with R and P, after cv2.stereoRectify) ---------------
 * camera as above; R f64[9] (the rectifying rotation, row-major) and P f64[9] (the left 3x3 of the new projection matrix, row-major).
 * mcba_rectify_map: cv2.initUndistortRectifyMap(K, dist, R, P, (width, height), CV_32FC2) (cv2.fisheye.initUndistortRectifyMap for
 *   MCBA_MODEL_FISHEYE; its two CV_32F maps interleaved).  The normalised point of pixel (u, v) of row v is OpenCV's walk along the row
 *   from (P R)^-1 (0, v, 1) in steps of (P R)^-1 (1, 0, 0): blocks of 8 pixels for the pinhole models, one pixel at a time for the
 *   fisheye, as OpenCV's own loops round it; the forward projection uses fx, fy, cx, cy only, as OpenCV's does.  fp64, stored as
 *   float32.  (width, height) is the rectified image's size, which need not be the camera's.  The map stays resident on the context in
 *   its fixed-point form, keyed by the camera, R, P and the size (the most recently used 64 maps are kept); map f32[height][width][2]
 *   receives the float map when not NULL.
 * mcba_rectify_images: cv2.remap(src[i], map, None, INTER_CUBIC) with the constant-zero border for n images of one camera through its
 *   rectification map of (R, P, width, height), host memory to host memory: src[i] uint8[src_height][src_width][channels], dst[i]
 *   uint8[height][width][channels] (the map's size).  Uses the resident map (computed first if it is not resident).  Chunks of images
 *   are staged through pinned buffers on several streams so that the copies in, the remap and the copies out overlap.  dtype must be
 *   MCBA_IMAGE_UINT8 and channels 1 or 3, else MCBA_ERR_ARG.
 * mcba_rectify_points: cv2.undistortPoints(pixels, K, dist, R = R, P = P) (cv2.fisheye.undistortPoints(pixels, K, dist, R, P)):
 *   f64[n][2] -> f64[n][2].  P = I gives normalised coordinates in the rectified frame.
 * (P R)^-1 comes from 3x3 Gaussian elimination with partial pivoting on the host: a singular P R fails with MCBA_ERR_ARG.  Non-finite
 * camera parameters, R or P fail with MCBA_ERR_NONFINITE.  None of these touches the uploaded problem. */
int  mcba_rectify_map(mcba_ctx* ctx, int32_t model, const double* camera, const double* R, const double* P, int32_t width,
                      int32_t height, float* map);
int  mcba_rectify_images(mcba_ctx* ctx, int32_t model, const double* camera, const double* R, const double* P, int32_t width,
                         int32_t height, int32_t n, int32_t src_width, int32_t src_height, int32_t channels, int32_t dtype,
                         const uint8_t* const* src, uint8_t* const* dst);
int  mcba_rectify_points(mcba_ctx* ctx, int32_t model, const double* camera, const double* R, const double* P, int64_t n,
                         const double* pixels, double* rectified);

/* -- triangulating points of a calibrated rig (DESIGN.md §3j) -----------------------------------------------------------------------
 * mcba_triangulate: N points seen by C cameras of one model (1 <= C <= MCBA_TRI_MAX_CAMERAS).  cameras f64[C][5 + nd] as above;
 *   poses f64[C][16] rig -> camera (x_cam = T_c x_rig, row-major 4x4, last row ignored); pixels f64[C][N][2]; valid uint8[C][N]
 *   (non-zero: camera c sees point n).  Out: points f64[N][3] in the rig frame, ok uint8[N], rms f64[N] (pixels, over the point's valid
 *   views).  Each point: the linear (DLT) solution from the undistorted normalised views, refined by Levenberg-Marquardt on the
 *   reprojection error through the full camera model.  A point is invalid (ok = 0, point and rms NaN) with fewer than 2 valid views,
 *   a non-finite valid pixel, a DLT w that is non-finite or zero at working precision, a valid view with z_cam <= 0 at the end, or a
 *   non-finite result.
 * mcba_triangulate_linear: cv2.triangulatePoints(P1, P2, x1, x2): P1, P2 f64[12] (3x4 row-major), x1, x2 f64[2][N] (row 0 x, row 1 y),
 *   out f64[4][N], the homogeneous points of unit norm (the sign is unspecified, as OpenCV's).  No distortion and no refinement.
 * Both work on chunks of points, so the device memory of a call stays within MCBA_TRI_CHUNK_BYTES plus the cameras.  Identical calls
 * agree bit for bit.  Bad arguments fail with MCBA_ERR_ARG; non-finite camera parameters, poses or P with MCBA_ERR_NONFINITE.  Neither
 * touches the uploaded problem. */
enum { MCBA_TRI_MAX_CAMERAS = 256, MCBA_TRI_CHUNK_BYTES = 64 << 20 };
int  mcba_triangulate(mcba_ctx* ctx, int32_t model, int32_t C, const double* cameras, const double* poses, int64_t N,
                      const double* pixels, const uint8_t* valid, double* points, uint8_t* ok, double* rms);
int  mcba_triangulate_linear(mcba_ctx* ctx, const double* P1, const double* P2, int64_t N, const double* x1, const double* x2,
                             double* out);

/* -- measurement hooks (bench.py): launch one kernel family on the context stream -------------- */
enum { MCBA_BENCH_LINEARIZE = 0, MCBA_BENCH_RESIDUAL = 1, MCBA_BENCH_COST = 2,
       MCBA_BENCH_NO_PREPARE = 256 /* or-ed in: reuse the pose tables of the previous call (times the kernel alone) */ };
int  mcba_bench_launch(mcba_ctx* ctx, int which, int repeats);
int  mcba_bench_info(mcba_ctx* ctx, int which, int64_t* corners, int64_t* bytes_per_launch, int32_t* launches_per_call);

#ifdef __cplusplus
}
#endif
#endif
