// kernels.cuh — sm_90a kernels of the bundle-adjustment hot path.
//
// Data layout in HBM (built once per upload from the dense table, on the device by pack_kernels.cuh): corners are stored FRAME-MAJOR, sorted by
// (frame, camera, board, point), so that every "view" (frame,camera,board) is one contiguous run and all
// views of one frame are contiguous (frames are also the multi-GPU sharding unit, SURVEY.md §8e):
//   obs   double2[N]   observed (u,v)                       16 B / corner   (point_table.points, calibration.py:206)
//   pid   uint16[N]    point index inside the board          2 B / corner
//   orig  uint32[N]    canonical packed index (np.argwhere(inliers) row) -- only read by the API hooks
//   view_start int[V+1], view_cam/frame/board int[V]       16 B / view
// Algorithmic bytes of one linearisation pass = 18 B / corner (+16 B / view).
//
// Kernel map (what each replaces in the reference is cited at the kernel):
//   k_prepare          rtvec -> R,t,JL tables of an unchanged state        pose_set.py:55-57, rtvec.py:24-27
//   make_trial_item    x -> trial state + its tables (k_lm; the API hooks through k_trial_state, solver.cu)
//   corner_loss        a corner's robust cost, row weights, scaled residual    common.py:720-731
//   corner_row         a corner's weighted 2 x D local Jacobian rows
//   k_views<MODE>      residual / cost / per-corner error                  calibration.py:204-206
//   k_point_blocks     board-point rows of the normal equations            (boards=True: calibration.py:188-190)
// The linearisation itself (residuals + analytic Jacobian + normal equations) is k_linearize (linearize.cuh), the trust-region loop
// k_lm (lm_kernel.cuh).  It, k_views and k_point_blocks share corner_point, project<>, corner_loss and corner_row.
#pragma once
#include <stdint.h>
#include "geometry.cuh"

namespace mcba {

// ------------------------------------------------------------------------------------------------
struct DeviceProblem {
  int C, F, B, P, model, nd, kint, D, T;   // T = D(D+1)/2 + D + 1 moment entries per view
  int64_t N;
  int V;
  const double2* obs;
  const uint16_t* pid;
  const uint32_t* orig;
  const int* view_start;
  const int* view_cam;
  const int* view_frame;
  const int* view_board;
  const int* frame_view_start;   // [F+1]
  double* board_pts;             // [B][P][3]  (parameters when off_pt >= 0: boards=True, board/charuco.py:112-117)
  // parameter state (full, including fixed blocks): one block laid out by state_layout (solver.cu), board_pts and he_rt included
  double* cam_rt;    // [C][6]   first: the base of the block
  double* board_rt;  // [B][6]
  double* frame_rt;  // [F][6]
  double* intr;      // [C][kint]
  // derived tables
  PoseT* cam_T;
  PoseT* frame_T;
  PoseT* board_T;
  // solver variable layout: x = [shared (n_s) | frames (fb*F if motion free)]
  int n, n_s, n_f;
  int off_cp, off_bp, off_in, off_pt;   // offsets inside shared, -1 when the block is fixed (off_pt: 3 per padded board point)
  int motion_on, fix_aspect;            // motion_on: per-frame blocks are free (static / rolling frames)
  uint32_t fixed_intr;                  // bit i: entry i of every camera's [fx fy cx cy skew dist...] is held at its current value
                                        // (mcba_set_fixed_intrinsics): a dead column, like skew's
  int tr_exact;                         // mcba_solve launches k_lm<FB, true>: scipy's tr_solver='exact' step instead of the 2-D subspace
                                        // one (mcba_set_trust_region; a field here so that it is part of the solve graph's key)
  int frame_blocks;                     // the linearisation emits H_ff, g_f (at g + n_s) and W_f: motion_on, or hand-eye with free
                                        // hand-eye parameters (k_fold_hand_eye folds the frame blocks into them)
  // motion model (the `motion` argument of Calibration, calibration.py:44-46)
  int motion;        // MOTION_STATIC: one rig pose per frame (motion/static_frames.py:29-42)
                     // MOTION_ROLLING: start + end pose per frame, blended per corner by its observed row (motion/rolling_frames.py:15-41,66-150)
                     // MOTION_HAND_EYE: frame pose = gripper_wrt_camera base_wrt_gripper[f] world_wrt_base (motion/hand_eye.py:14-90)
  int npf;           // pose-table entries per frame: frame_T[f*npf + j], frame_rt + 6*(f*npf + j)   (2 for rolling, else 1)
  int fb;            // parameters of one eliminated frame block: 6 (static), 12 (rolling: start | end), 0 (hand-eye: none)
  int koff;          // local Jacobian layout of a residual row: [camera-frame twists (koff = 6 or 12) | fx fy cx cy dist]; D = koff + 4 + nd
  const double* img_h;   // [C] image heights (rolling_times, rolling_frames.py:15-19)
  double* he_rt;     // [12] world_wrt_base | gripper_wrt_camera as rtvecs (HandEye.params, hand_eye.py:76-81)
  PoseT* he_T;       // [2]
  const PoseT* arm_T;    // [F] base_wrt_gripper (R, t only)
  int off_he;        // offset of the 12 hand-eye parameters inside shared, -1 when fixed or not a hand-eye problem
};
enum { MOTION_STATIC = 0, MOTION_ROLLING = 1, MOTION_HAND_EYE = 2 };

__host__ __device__ constexpr int tri_index(int D, int i, int j) { return i * D - (i * (i - 1)) / 2 + (j - i); }
__device__ __forceinline__ double msym(const double* M, int D, int i, int j) {
  return i <= j ? M[tri_index(D, i, j)] : M[tri_index(D, j, i)];
}

// ------------------------------------------------------------------------------------------------
// (R, t) of A B
__host__ __device__ __forceinline__ void se3_mul(const double* Ra, const double* ta, const double* Rb, const double* tb, double* R, double* t) {
  mat3_mul(Ra, Rb, R);
  mat3_vec(Ra, tb, t);
  t[0] += ta[0]; t[1] += ta[1]; t[2] += ta[2];
}
__device__ __forceinline__ void pose_from_rt(const double* rt, PoseT& t) {
  rodrigues(rt, t.R, t.JL);
  t.t[0] = rt[3]; t.t[1] = rt[4]; t.t[2] = rt[5];
  t.pad[0] = t.pad[1] = t.pad[2] = 0;
}
// hand-eye frame pose T_f = G A_f W (motion/hand_eye.py:43-46) from the rtvecs he = [W | G].  A derived pose has no rtvec of its own; its
// left Jacobian is the identity, so that the linearisation treats the frame as a twist-perturbed pose (see hand_eye_frame_map)
__device__ __forceinline__ void hand_eye_frame(const double* he, const PoseT& arm, PoseT& out) {
  PoseT W, G;
  pose_from_rt(he, W);
  pose_from_rt(he + 6, G);
  double Rga[9], tga[3];
  se3_mul(G.R, G.t, arm.R, arm.t, Rga, tga);
  se3_mul(Rga, tga, W.R, W.t, out.R, out.t);
#pragma unroll
  for (int i = 0; i < 9; i++) out.JL[i] = (i % 4 == 0) ? 1.0 : 0.0;
  out.pad[0] = out.pad[1] = out.pad[2] = 0;
}
// M_f (6 x 12, row-major): how the hand-eye parameters he = [W | G] move frame f's pose, as a twist of that pose.  For a view of camera c
// the twist map of the frame pose taken with JL = I, twist_map(R_c, I, t_cf), times M_f is the view's map of he: so H_he,he, H_s,he and
// g_he are M_f folds of the per-frame blocks H_ff, W_f, g_f (k_fold_hand_eye).  With R_GA = R_G R_Af and t_f = translation of T_f:
//   M_f = [ R_GA JL_W   0      JL_G                 0 ]
//         [ 0           R_GA   [(t_G - t_f)x] JL_G   I ]
__host__ __device__ inline void hand_eye_frame_map(const double* RG, const double* RA, const double* JLW, const double* JLG, const double* tG,
                                                   const double* tf, double* M) {
  double RGA[9], RJ[9];
  mat3_mul(RG, RA, RGA);
  mat3_mul(RGA, JLW, RJ);
  const double d[3] = {tG[0] - tf[0], tG[1] - tf[1], tG[2] - tf[2]};
  for (int i = 0; i < 72; i++) M[i] = 0.0;
  for (int r = 0; r < 3; r++) {
    M[12 * (3 + r) + 9 + r] = 1.0;
    for (int c = 0; c < 3; c++) {
      M[12 * r + c] = RJ[3 * r + c];
      M[12 * (3 + r) + 3 + c] = RGA[3 * r + c];
      M[12 * r + 6 + c] = JLG[3 * r + c];
      const double a0 = JLG[c], a1 = JLG[3 + c], a2 = JLG[6 + c];         // (d x column c of JL_G)
      M[12 * (3 + r) + 6 + c] = r == 0 ? d[1] * a2 - d[2] * a1 : r == 1 ? d[2] * a0 - d[0] * a2 : d[0] * a1 - d[1] * a0;
    }
  }
}

// k_prepare: one thread per pose.  rtvec -> (R, t, JL).   pose_set.py:55-57 / transform/rtvec.py:24-27
__global__ void k_prepare(DeviceProblem p, const double* cam_rt, const double* board_rt, const double* frame_rt) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int nfp = p.F * p.npf;
  const double* src; PoseT* dst;
  if (i < p.C) { src = cam_rt + 6 * i; dst = p.cam_T + i; }
  else if (i < p.C + p.B) { src = board_rt + 6 * (i - p.C); dst = p.board_T + (i - p.C); }
  else if (i < p.C + p.B + nfp) {
    const int q = i - p.C - p.B;
    if (p.motion == MOTION_HAND_EYE) { PoseT t; hand_eye_frame(p.he_rt, p.arm_T[q], t); p.frame_T[q] = t; return; }
    src = frame_rt + 6 * q; dst = p.frame_T + q;
  }
  else if (p.motion == MOTION_HAND_EYE && i < p.C + p.B + nfp + 2) { const int j = i - p.C - p.B - nfp; src = p.he_rt + 6 * j; dst = p.he_T + j; }
  else return;
  PoseT t;
  pose_from_rt(src, t);
  *dst = t;
}

// pose matrices <-> rtvec parameter state, one thread per pose (the host never converts rotations itself)
// frame f goes to frame_rt + fstride*f (fstride = 6; 12 for rolling frames, whose start | end poses are adjacent; 0 = frames are
// derived, hand-eye, and not stored)
__global__ void k_matrices_to_state(int C, int B, int F, const double* mats /*[C+B+F][16]*/, double* cam_rt, double* board_rt, double* frame_rt, int fstride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C + B + F) return;
  if (i >= C + B && fstride == 0) return;
  double* dst = i < C ? cam_rt + 6 * i : i < C + B ? board_rt + 6 * (i - C) : frame_rt + fstride * (i - C - B);
  double rt[6];
  matrix_to_rtvec(mats + (size_t)16 * i, rt);
#pragma unroll
  for (int j = 0; j < 6; j++) dst[j] = rt[j];
}
// frame_T != nullptr: frame matrices come from the pose table (hand-eye: derived poses; the table must be current)
__global__ void k_state_to_matrices(int C, int B, int F, const double* cam_rt, const double* board_rt, const double* frame_rt, double* mats, int fstride,
                                    const PoseT* frame_T) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= C + B + F) return;
  double* M = mats + (size_t)16 * i;
  if (i >= C + B && frame_T) {
    const PoseT& t = frame_T[i - C - B];
#pragma unroll
    for (int r = 0; r < 3; r++) { M[4 * r] = t.R[3 * r]; M[4 * r + 1] = t.R[3 * r + 1]; M[4 * r + 2] = t.R[3 * r + 2]; M[4 * r + 3] = t.t[r]; }
    M[12] = 0.0; M[13] = 0.0; M[14] = 0.0; M[15] = 1.0;
    return;
  }
  const double* src = i < C ? cam_rt + 6 * i : i < C + B ? board_rt + 6 * (i - C) : frame_rt + fstride * (i - C - B);
  double R[9], JL[9];
  rodrigues(src, R, JL);
#pragma unroll
  for (int r = 0; r < 3; r++) { M[4 * r] = R[3 * r]; M[4 * r + 1] = R[3 * r + 1]; M[4 * r + 2] = R[3 * r + 2]; M[4 * r + 3] = src[3 + r]; }
  M[12] = 0.0; M[13] = 0.0; M[14] = 0.0; M[15] = 1.0;
}

// trial parameter state = current state with the free blocks replaced by x (internal order), and the pose tables of that state (item i
// of one pass of k_lm).  One item per pose, then one per camera (intrinsics), per board point, and one for the hand-eye pair (which
// must be complete before the derived frame poses: those items recompute it themselves).  `trial` has the layout of the current state.
// The only path from a parameter vector to a state: k_lm calls it for its trial states, set_state_from_x (solver.cu) for the API hooks.
__device__ __forceinline__ void make_trial_item(const DeviceProblem& p, const double* x, double* trial, int i) {
  const int nfp = p.F * p.npf;
  const int np = p.C + p.B + nfp;
  auto to_trial = [&](const double* cur) { return trial + (cur - p.cam_rt); };      // the twin of a current-state entry
  if (i < np) {
    const double* cur; const double* src = nullptr; double* dst; PoseT* tab;
    if (i < p.C) { cur = p.cam_rt + 6 * i; dst = to_trial(cur); tab = p.cam_T + i; if (p.off_cp >= 0) src = x + p.off_cp + 6 * i; }
    else if (i < p.C + p.B) { const int b = i - p.C; cur = p.board_rt + 6 * b; dst = to_trial(cur); tab = p.board_T + b; if (p.off_bp >= 0) src = x + p.off_bp + 6 * b; }
    else {
      const int q = i - p.C - p.B;
      if (p.motion == MOTION_HAND_EYE) {
        double he[12];
#pragma unroll
        for (int j = 0; j < 12; j++) he[j] = p.off_he >= 0 ? __ldcg(&x[p.off_he + j]) : p.he_rt[j];
        PoseT t; hand_eye_frame(he, p.arm_T[q], t); p.frame_T[q] = t;
        return;
      }
      cur = p.frame_rt + 6 * q; dst = to_trial(cur); tab = p.frame_T + q; if (p.motion_on) src = x + p.n_s + 6 * q;
    }
    if (!src) src = cur;
    double v[6];
#pragma unroll
    for (int j = 0; j < 6; j++) { v[j] = __ldcg(&src[j]); dst[j] = v[j]; }      // (x may have been written by another CTA of the same launch: k_lm)
    PoseT t;
    pose_from_rt(v, t);
    *tab = t;
  } else if (i < np + p.C) {
    const int c = i - np;
    const double* src = p.off_in >= 0 ? x + p.off_in + p.kint * c : p.intr + p.kint * c;
    double* dst = to_trial(p.intr + p.kint * c);
    for (int j = 0; j < p.kint; j++) {
      double v = __ldcg(&src[j]);
      if (j == 1 && p.fix_aspect && p.off_in >= 0) v = __ldcg(&src[0]);      // fy follows fx (camera.py:159-160)
      if ((p.fixed_intr >> j) & 1u) v = __ldcg(&p.intr[p.kint * c + j]);     // held fixed: keeps the current value
      dst[j] = v;
    }
  } else if (i < np + p.C + p.B * p.P) {
    const int q = i - np - p.C;                                       // padded board point index b*P + p
    const double* src = p.off_pt >= 0 ? x + p.off_pt + 3 * q : p.board_pts + 3 * q;
    double* dst = to_trial(p.board_pts + 3 * q);
    dst[0] = __ldcg(&src[0]); dst[1] = __ldcg(&src[1]); dst[2] = __ldcg(&src[2]);
  } else if (i < np + p.C + p.B * p.P + 2 && p.motion == MOTION_HAND_EYE) {
    const int j = i - np - p.C - p.B * p.P;
    const double* src = p.off_he >= 0 ? x + p.off_he + 6 * j : p.he_rt + 6 * j;
    double* dst = to_trial(p.he_rt + 6 * j);
    double v[6];
#pragma unroll
    for (int k = 0; k < 6; k++) { v[k] = __ldcg(&src[k]); dst[k] = v[k]; }
    PoseT t;
    pose_from_rt(v, t);
    p.he_T[j] = t;
  }
}

// compose T_cfb = T_c T_f T_b for one view (every lane of the warp computes the same small product)
struct ViewPose { double R[9]; double t[3]; };
__device__ __forceinline__ void compose_view(const PoseT& c, const PoseT& f, const PoseT& b, ViewPose& o) {
  double Rcf[9], tcf[3];
  mat3_mul(c.R, f.R, Rcf);
  mat3_vec(c.R, f.t, tcf);
  tcf[0] += c.t[0]; tcf[1] += c.t[1]; tcf[2] += c.t[2];
  mat3_mul(Rcf, b.R, o.R);
  mat3_vec(Rcf, b.t, o.t);
  o.t[0] += tcf[0]; o.t[1] += tcf[1]; o.t[2] += tcf[2];
}

// the view's chain(s): static / hand-eye frames have one pose table entry per frame, rolling frames two (start, end)
template <bool ROLL>
__device__ __forceinline__ void compose_views(const DeviceProblem& p, int c, int f, int b, ViewPose& vp, ViewPose& vpe) {
  if constexpr (ROLL) {
    compose_view(p.cam_T[c], p.frame_T[2 * f], p.board_T[b], vp);
    compose_view(p.cam_T[c], p.frame_T[2 * f + 1], p.board_T[b], vpe);
  } else {
    compose_view(p.cam_T[c], p.frame_T[f], p.board_T[b], vp);
  }
}
// camera-frame point of a corner.  Rolling shutter (rolling_frames.py:21-41 transformed_linear + interpolate.py:6-8 lerp): the
// board point is transformed by the start and by the end chain and the two are blended by tau = observed row / image height.
template <bool ROLL>
__device__ __forceinline__ void corner_point(const ViewPose& vp, const ViewPose& vpe, const double* X, double tau,
                                             double* Xc, double* Xs, double* Xe) {
  mat3_vec(vp.R, X, Xc);
  Xc[0] += vp.t[0]; Xc[1] += vp.t[1]; Xc[2] += vp.t[2];
  if constexpr (ROLL) {
    mat3_vec(vpe.R, X, Xe);
    Xe[0] += vpe.t[0]; Xe[1] += vpe.t[1]; Xe[2] += vpe.t[2];
#pragma unroll
    for (int i = 0; i < 3; i++) { Xs[i] = Xc[i]; Xc[i] = Xs[i] * (1.0 - tau) + Xe[i] * tau; }
  }
}

struct ViewKernelArgs {
  int loss;
  double f_scale;
  double* view_cost;   // MODE_COST   : [V]
  double* resid;       // MODE_RESID  : [2N] canonical order
  double* err;         // MODE_ERROR  : [N]  canonical order
};
enum { MODE_COST = 0, MODE_RESID = 1, MODE_ERROR = 2 };

constexpr int VIEW_WARPS = 4;          // warps per CTA for k_views
constexpr double SCIPY_EPS = 2.220446049250313e-16;
constexpr double TRIGGS_FLOOR = 0.1;

// robust loss per scalar residual (least_squares.py construct_loss_function, common.py:720-731) of a corner's residual pair (ru, rv):
// adds its 0.5 sum rho to `cost` and returns the weights wu, wv of its u and v rows (Triggs' correction, floored) with the residuals
// scaled to match.  loss == 0: cost 0.5 (ru^2 + rv^2), weights 1, residuals unchanged.  (Values in, a struct out: through references
// the compiler orders k_linearize's instructions differently.)
struct CornerLoss { double ru, rv, wu, wv; };
__device__ __forceinline__ CornerLoss corner_loss(int loss, double f_scale, double ru, double rv, double& cost) {
  double wu = 1.0, wv = 1.0;
  if (loss == 0) {
    cost += 0.5 * (ru * ru + rv * rv);
  } else {
    const double is = 1.0 / f_scale, fs2 = f_scale * f_scale;
    double zu = ru * is, zv = rv * is;
    zu *= zu; zv *= zv;
    double r0u, r1u, r2u, r0v, r1v, r2v;
    loss_rho(loss, zu, r0u, r1u, r2u);
    loss_rho(loss, zv, r0v, r1v, r2v);
    cost += 0.5 * fs2 * (r0u + r0v);
    double ju = r1u + 2.0 * r2u * zu, jv = r1v + 2.0 * r2v * zv;
    ju = fmax(fmax(ju, TRIGGS_FLOOR * r1u), SCIPY_EPS);
    jv = fmax(fmax(jv, TRIGGS_FLOOR * r1v), SCIPY_EPS);
    wu = sqrt(ju); wv = sqrt(jv);
    ru *= r1u / wu; rv *= r1v / wv;
  }
  return {ru, rv, wu, wv};
}

// the weighted local Jacobian rows of a corner, columns [0, D): twist block(s) (6; rolling: start | end, 12) then [fx fy cx cy dist].
// Xc = camera-frame point (rolling: Xs, Xe = the start / end chain's point, tau = the blend), Ju, Jv / ku, kv = d(u, v) / d(Xc) and
// d(u, v) / d(intrinsics) from project<MODEL, true>.  The four structural zeros (fy, cy of the u row; fx, cx of the v row) are not
// written: the caller zeroes the rows first (k_linearize needs zero rows for its idle lanes anyway, and stores of the zeros here would
// change its instruction schedule).
template <int MODEL, bool ROLL>
__device__ __forceinline__ void corner_row(const double* Xc, const double* Xs, const double* Xe, double tau, const double* Ju, const double* Jv,
                                           const double* ku, const double* kv, double wu, double wv, double* gu, double* gv) {
  constexpr int ND = model_nd(MODEL), KO = ROLL ? 12 : 6;
  if constexpr (!ROLL) {
    gu[0] = (Xc[1] * Ju[2] - Xc[2] * Ju[1]) * wu; gu[1] = (Xc[2] * Ju[0] - Xc[0] * Ju[2]) * wu; gu[2] = (Xc[0] * Ju[1] - Xc[1] * Ju[0]) * wu;
    gv[0] = (Xc[1] * Jv[2] - Xc[2] * Jv[1]) * wv; gv[1] = (Xc[2] * Jv[0] - Xc[0] * Jv[2]) * wv; gv[2] = (Xc[0] * Jv[1] - Xc[1] * Jv[0]) * wv;
#pragma unroll
    for (int i = 0; i < 3; i++) { gu[3 + i] = Ju[i] * wu; gv[3 + i] = Jv[i] * wv; }
  } else {
    const double su = (1.0 - tau) * wu, sv = (1.0 - tau) * wv, eu = tau * wu, ev = tau * wv;
    gu[0] = (Xs[1] * Ju[2] - Xs[2] * Ju[1]) * su; gu[1] = (Xs[2] * Ju[0] - Xs[0] * Ju[2]) * su; gu[2] = (Xs[0] * Ju[1] - Xs[1] * Ju[0]) * su;
    gv[0] = (Xs[1] * Jv[2] - Xs[2] * Jv[1]) * sv; gv[1] = (Xs[2] * Jv[0] - Xs[0] * Jv[2]) * sv; gv[2] = (Xs[0] * Jv[1] - Xs[1] * Jv[0]) * sv;
    gu[6] = (Xe[1] * Ju[2] - Xe[2] * Ju[1]) * eu; gu[7] = (Xe[2] * Ju[0] - Xe[0] * Ju[2]) * eu; gu[8] = (Xe[0] * Ju[1] - Xe[1] * Ju[0]) * eu;
    gv[6] = (Xe[1] * Jv[2] - Xe[2] * Jv[1]) * ev; gv[7] = (Xe[2] * Jv[0] - Xe[0] * Jv[2]) * ev; gv[8] = (Xe[0] * Jv[1] - Xe[1] * Jv[0]) * ev;
#pragma unroll
    for (int i = 0; i < 3; i++) { gu[3 + i] = Ju[i] * su; gv[3 + i] = Jv[i] * sv; gu[9 + i] = Ju[i] * eu; gv[9 + i] = Jv[i] * ev; }
  }
  gu[KO] = ku[0] * wu; gu[KO + 2] = wu;
  gv[KO + 1] = kv[1] * wv; gv[KO + 3] = wv;
#pragma unroll
  for (int i = 0; i < ND; i++) { gu[KO + 4 + i] = ku[4 + i] * wu; gv[KO + 4 + i] = kv[4 + i] * wv; }
}

// k_views: one warp per view, lanes stride over the view's corners (one thread per corner per step).
//   MODE_COST    -> 0.5*sum rho(f) per view               (cost hook of mcba_residuals)
//   MODE_RESID   -> residual vector in canonical order     (calibration.py:204-206)
//   MODE_ERROR   -> per-corner ||proj - obs||              (tables.py:244-249)
// (the linearisation -- residuals + analytic Jacobian + normal equations -- is k_linearize, linearize.cuh)
template <int MODEL, int MODE, bool ROLL = false>
__global__ void __launch_bounds__(VIEW_WARPS * 32)
k_views(DeviceProblem p, ViewKernelArgs a) {
  constexpr int ND = model_nd(MODEL);
  constexpr int KINT = 5 + ND;
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int gw = blockIdx.x * VIEW_WARPS + warp;
  const int nw = gridDim.x * VIEW_WARPS;
  for (int v = gw; v < p.V; v += nw) {
    const int c = p.view_cam[v], f = p.view_frame[v], b = p.view_board[v];
    const int beg = p.view_start[v], end = p.view_start[v + 1];
    ViewPose vp, vpe;
    compose_views<ROLL>(p, c, f, b, vp, vpe);
    const double inv_h = ROLL ? 1.0 / p.img_h[c] : 0.0;
    double k[KINT];
#pragma unroll
    for (int i = 0; i < KINT; i++) k[i] = p.intr[c * KINT + i];
    const double* bp = p.board_pts + (size_t)b * p.P * 3;
    double acc = 0.0;
    for (int idx = beg + lane; idx < end; idx += 32) {
      const double2 ob = p.obs[idx];
      const int pi = p.pid[idx];
      const double X[3] = {bp[3 * pi], bp[3 * pi + 1], bp[3 * pi + 2]};
      double Xc[3], Xs[3], Xe[3];
      corner_point<ROLL>(vp, vpe, X, ob.y * inv_h, Xc, Xs, Xe);
      double u, w_;
      double Ju[3], Jv[3], ku[4 + ND], kv[4 + ND];
      project<MODEL, false>(Xc, k, u, w_, Ju, Jv, ku, kv);
      const double ru = u - ob.x, rv = w_ - ob.y;           // projected - observed (calibration.py:206)
      if constexpr (MODE == MODE_RESID) {
        const uint32_t o = p.orig[idx];
        a.resid[2 * (size_t)o] = ru;
        a.resid[2 * (size_t)o + 1] = rv;
      } else if constexpr (MODE == MODE_ERROR) {
        a.err[p.orig[idx]] = sqrt(ru * ru + rv * rv);
      } else {
        corner_loss(a.loss, a.f_scale, ru, rv, acc);
      }
    }
    if constexpr (MODE == MODE_COST) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) a.view_cost[v] = acc;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// fp64 tensor-core steps (mma.sync "DMMA"; wgmma has no fp64 kind): the 16x8 C fragment += A (16xK) B (Kx8), K = 8 or 4.
// k_linearize accumulates its per-view moment SYRKs and the view epilogue's products with them, k_lm the Schur complement.  Fragments
// (PTX ISA "Matrix fragments for mma.m16n8k*", .f64), lane = 4 grp + tig:
//   a[i] = A[grp + 8 (i & 1)][tig + 4 (i >> 1)]     b[i] = B[tig + 4 i][grp]     c[i] = C[grp + 8 (i >> 1)][2 tig + (i & 1)]
// On an H100 (SXM, 700 W) the m16n8k* shapes run at 128 MAC/clk/SM, twice the rate of m8n8k4 (scripts/dmma_shapes.cu).  A host build
// of the sources (no __CUDA_ARCH__) composes each shape from m8n8k4 steps: rows grp and grp + 8 are two m8n8k4 with the same B.
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void dmma1688(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
#ifdef __CUDA_ARCH__
  asm __volatile__("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                   : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
#else
  dmma884(c[0], c[1], a[0], b[0]); dmma884(c[2], c[3], a[1], b[0]);      // k = tig
  dmma884(c[0], c[1], a[2], b[1]); dmma884(c[2], c[3], a[3], b[1]);      // k = tig + 4
#endif
}
__device__ __forceinline__ void dmma1684(double (&c)[4], const double (&a)[2], const double (&b)[1]) {
#ifdef __CUDA_ARCH__
  asm __volatile__("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                   : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
#else
  dmma884(c[0], c[1], a[0], b[0]); dmma884(c[2], c[3], a[1], b[0]);
#endif
}
// C += A B over K = 4 NQ: m16n8k8 steps, and m16n8k4 for an odd last quad.  a[q][h] = A[grp + 8 h][4 q + tig], b[q] = B[4 q + tig][grp].
template <int NQ>
__device__ __forceinline__ void dmma_quads(double (&c)[4], const double (&a)[NQ][2], const double (&b)[NQ]) {
#pragma unroll
  for (int q = 0; q + 1 < NQ; q += 2) {
    const double a8[4] = {a[q][0], a[q][1], a[q + 1][0], a[q + 1][1]}, b8[2] = {b[q], b[q + 1]};
    dmma1688(c, a8, b8);
  }
  if constexpr (NQ % 2 == 1) {
    const double a4[2] = {a[NQ - 1][0], a[NQ - 1][1]}, b4[1] = {b[NQ - 1]};
    dmma1684(c, a4, b4);
  }
}
// columns of a staged residual row [G | r]: the local Jacobian (D, plus 6 for the second twist block of rolling frames) and r, padded to 8
__host__ __device__ constexpr int mma_nc(int model, bool roll = false) { return ((model_D(model) + (roll ? 6 : 0) + 1 + 7) / 8) * 8; }

__device__ __forceinline__ int intr_param_index(const DeviceProblem& p, int local /*0..3+nd*/) {
  // local [fx fy cx cy dist...] -> index in [fx fy cx cy skew dist...]; fix_aspect folds fy onto fx (camera.py:159-160); -1 for a
  // parameter held fixed (DeviceProblem::fixed_intr): its column is zero, and every caller skips it
  const int q = (local == 1 && p.fix_aspect) ? 0 : local < 4 ? local : local + 1;
  return ((p.fixed_intr >> q) & 1u) ? -1 : q;
}

__device__ __forceinline__ void view_chain(const PoseT& pc, const PoseT& pf, double* Rcf, double* tcf) {
  mat3_mul(pc.R, pf.R, Rcf);
  mat3_vec(pc.R, pf.t, tcf);
  tcf[0] += pc.t[0]; tcf[1] += pc.t[1]; tcf[2] += pc.t[2];
}

// NP = twist blocks of the local row / pose-table entries per frame: 1 (static, hand-eye), 2 (rolling: start, end).  A parameter
// block reaches the local twists through NP 6x6 maps (camera pose: the same map for every block; board pose: one map per chain;
// frame pose j: its own map into block j only).
// the view's twist maps: Ac (camera pose), Af[j] (frame pose j), Ab[j] (board pose through chain j); lanes 0 .. 2 NP of the warp
template <int NP>
__device__ __forceinline__ void view_twist_maps(const DeviceProblem& p, int c, int f, int b, int lane, double* Ac, double* Af, double* Ab) {
  if (lane > 2 * NP) return;
  const PoseT& pc = p.cam_T[c];
  if (lane == 0) { if (Ac) { const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; twist_map(I3, pc.JL, pc.t, Ac); } return; }
  const int j = (lane - 1) % NP;
  const PoseT& pf = p.frame_T[f * NP + j];
  double Rcf[9], tcf[3];
  view_chain(pc, pf, Rcf, tcf);
  if (lane <= NP) { if (Af) twist_map(pc.R, pf.JL, tcf, Af + 36 * j); return; }
  if (!Ab) return;
  const PoseT& pb = p.board_T[b];
  double tb[3];
  mat3_vec(Rcf, pb.t, tb);
  tb[0] += tcf[0]; tb[1] += tcf[1]; tb[2] += tcf[2];
  twist_map(Rcf, pb.JL, tb, Ab + 36 * j);
}

// k_point_blocks (boards=True only): board points as shared parameters (3 per padded point).  One warp per view, one
// thread per corner: d r / d X_board = J_proj R_cfb (rolling: the blend (1-tau) R_start + tau R_end); the point's own 3x3 block,
// its gradient and its couplings with the camera pose / intrinsics / board pose (H_ss) and the frame block (W_f; hand-eye: k_fold_hand_eye
// carries them on to the hand-eye pair) are added with fp64 atomics on top of what k_linearize / k_reduce_shared wrote.  Replaces the
// axis-3 column block of the reference's sparsity pattern (calibration.py:188-190).  NP = 2: rolling frames (two twist blocks per row,
// 12-wide frame block).
template <int MODEL, int NP>
__global__ void __launch_bounds__(VIEW_WARPS * 32)
k_point_blocks(DeviceProblem p, ViewKernelArgs a, double* Hss, double* W, double* g) {
  constexpr bool ROLL = NP == 2;
  constexpr int ND = model_nd(MODEL);
  constexpr int KINT = 5 + ND;
  constexpr int NIN = 4 + ND;
  constexpr int KO = 6 * NP, FB = 6 * NP;
  __shared__ double maps[VIEW_WARPS][36 + 72 * NP];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gw = blockIdx.x * VIEW_WARPS + warp, nw = gridDim.x * VIEW_WARPS;
  const int n_s = p.n_s;
  double* Ac = maps[warp]; double* Af = Ac + 36; double* Ab = Af + 36 * NP;
  for (int v = gw; v < p.V; v += nw) {
    const int c = p.view_cam[v], f = p.view_frame[v], b = p.view_board[v];
    const int beg = p.view_start[v], end = p.view_start[v + 1];
    ViewPose vp, vpe;
    compose_views<ROLL>(p, c, f, b, vp, vpe);
    const double inv_h = ROLL ? 1.0 / p.img_h[c] : 0.0;
    __syncwarp();
    view_twist_maps<NP>(p, c, f, b, lane, Ac, Af, Ab);
    __syncwarp();
    double k[KINT];
#pragma unroll
    for (int i = 0; i < KINT; i++) k[i] = p.intr[c * KINT + i];
    const double* bp = p.board_pts + (size_t)b * p.P * 3;
    const int cp = p.off_cp >= 0 ? p.off_cp + 6 * c : -1;
    const int bpo = p.off_bp >= 0 ? p.off_bp + 6 * b : -1;
    const int in0 = p.off_in >= 0 ? p.off_in + p.kint * c : -1;
    for (int idx = beg + lane; idx < end; idx += 32) {
      const double2 ob = p.obs[idx];
      const int pi = p.pid[idx];
      const double X[3] = {bp[3 * pi], bp[3 * pi + 1], bp[3 * pi + 2]};
      const double tau = ob.y * inv_h;
      double Xc[3], Xs[3], Xe[3];
      corner_point<ROLL>(vp, vpe, X, tau, Xc, Xs, Xe);
      double u, w_, Ju[3], Jv[3], ku[4 + ND], kv[4 + ND];
      project<MODEL, true>(Xc, k, u, w_, Ju, Jv, ku, kv);
      double cost = 0.0;         // unused: k_linearize sums the cost
      const CornerLoss cl = corner_loss(a.loss, a.f_scale, u - ob.x, w_ - ob.y, cost);
      const double ru = cl.ru, rv = cl.rv, wu = cl.wu, wv = cl.wv;
      // local rows: twist block(s) (KO) then [fx fy cx cy dist] (NIN), as k_linearize stages them
      double gu[KO + NIN] = {}, gv[KO + NIN] = {};
      corner_row<MODEL, ROLL>(Xc, Xs, Xe, tau, Ju, Jv, ku, kv, wu, wv, gu, gv);
      // point rows: d r / d X_board = J_proj R_cfb  (rolling: R = (1 - tau) R_start + tau R_end)
      double xu[3], xv[3];
#pragma unroll
      for (int j = 0; j < 3; j++) {
        double r0 = vp.R[j], r1 = vp.R[3 + j], r2 = vp.R[6 + j];
        if constexpr (ROLL) {
          r0 = r0 * (1.0 - tau) + vpe.R[j] * tau; r1 = r1 * (1.0 - tau) + vpe.R[3 + j] * tau; r2 = r2 * (1.0 - tau) + vpe.R[6 + j] * tau;
        }
        xu[j] = (Ju[0] * r0 + Ju[1] * r1 + Ju[2] * r2) * wu;
        xv[j] = (Jv[0] * r0 + Jv[1] * r1 + Jv[2] * r2) * wv;
      }
      const int pt = p.off_pt + 3 * (b * p.P + pi);
      auto addS = [&](int i, int j, double val) {
        atomicAdd(&Hss[(size_t)i * n_s + j], val);
        atomicAdd(&Hss[(size_t)j * n_s + i], val);
      };
#pragma unroll
      for (int r = 0; r < 3; r++) {
        atomicAdd(&g[pt + r], xu[r] * ru + xv[r] * rv);
#pragma unroll
        for (int q = r; q < 3; q++) {
          const double val = xu[r] * xu[q] + xv[r] * xv[q];
          if (q == r) atomicAdd(&Hss[(size_t)(pt + r) * n_s + pt + r], val); else addS(pt + r, pt + q, val);
        }
        double Q[KO];
#pragma unroll
        for (int kk = 0; kk < KO; kk++) Q[kk] = xu[r] * gu[kk] + xv[r] * gv[kk];
#pragma unroll
        for (int j = 0; j < 6; j++) {
          double vc = 0.0, vb = 0.0;
#pragma unroll
          for (int kk = 0; kk < KO; kk++) { vc += Q[kk] * Ac[(kk % 6) * 6 + j]; vb += Q[kk] * Ab[36 * (kk / 6) + (kk % 6) * 6 + j]; }
          if (cp >= 0) addS(pt + r, cp + j, vc);
          if (bpo >= 0) addS(pt + r, bpo + j, vb);
        }
        if (p.frame_blocks) {
#pragma unroll
          for (int col = 0; col < FB; col++) {
            double vf = 0.0;
#pragma unroll
            for (int kk = 0; kk < 6; kk++) vf += Q[6 * (col / 6) + kk] * Af[36 * (col / 6) + kk * 6 + col % 6];
            atomicAdd(&W[((size_t)f * n_s + pt + r) * FB + col], vf);
          }
        }
        if (in0 >= 0) {
#pragma unroll
          for (int i = 0; i < NIN; i++) {
            const double val = xu[r] * gu[KO + i] + xv[r] * gv[KO + i];
            const int q = intr_param_index(p, i);
            if (val != 0.0 && q >= 0) addS(pt + r, in0 + q, val);
          }
        }
      }
    }
  }
}

}  // namespace mcba
