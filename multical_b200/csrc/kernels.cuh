// kernels.cuh — sm_90a kernels of the bundle-adjustment hot path.
//
// Data layout in HBM (built once by mcba_upload, solver.cu): corners are stored FRAME-MAJOR, sorted by
// (frame, camera, board, point), so that every "view" (frame,camera,board) is one contiguous run and all
// views of one frame are contiguous (frames are also the multi-GPU sharding unit, SURVEY.md §8e):
//   obs   double2[N]   observed (u,v)                       16 B / corner   (point_table.points, calibration.py:206)
//   pid   uint16[N]    point index inside the board          2 B / corner
//   orig  uint32[N]    canonical packed index (np.argwhere(inliers) row) -- only read by the API hooks
//   view_start int[V+1], view_cam/frame/board int[V]       16 B / view
// Algorithmic bytes of one linearisation pass = 18 B / corner (+16 B / view).
//
// Kernel map (what each replaces in the reference is cited at the kernel):
//   k_prepare          rtvec -> R,t,JL tables                     pose_set.py:55-57, rtvec.py:24-27
//   k_views<MODE>      residual / cost / per-view moments          calibration.py:204-206 + scipy FD Jacobian
//   k_expand_frames    per-frame Hessian blocks H_ff, W_f, g_f     (J^T J restricted to one motion pose; pose_set.py:59-60)
//   k_expand_shared    shared blocks H_ss, g_s                     (camera pose / board pose / intrinsics columns)
//   k_scale, k_quad, k_schur_*, k_chol_solve, k_backsub, k_step    scipy _lsq/trf.py trf_no_bounds (LSMR replaced by an
//                                                                   exact damped solve through the Schur complement)
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
  const int* cam_view_start;     // [C+1]
  const int* cam_view_list;      // [V] view ids grouped by camera
  double* board_pts;             // [B][P][3]  (parameters when off_pt >= 0: boards=True, board/charuco.py:112-117)
  // parameter state (full, including fixed blocks)
  double* cam_rt;    // [C][6]
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
// hand-eye frame pose T_f = G A_f W (motion/hand_eye.py:43-46) from the rtvecs he = [W | G]; JL is not used for derived poses
__device__ __forceinline__ void hand_eye_frame(const double* he, const PoseT& arm, PoseT& out) {
  PoseT W, G;
  pose_from_rt(he, W);
  pose_from_rt(he + 6, G);
  double Rga[9], tga[3];
  se3_mul(G.R, G.t, arm.R, arm.t, Rga, tga);
  se3_mul(Rga, tga, W.R, W.t, out.R, out.t);
#pragma unroll
  for (int i = 0; i < 9; i++) out.JL[i] = 0.0;
  out.pad[0] = out.pad[1] = out.pad[2] = 0;
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

// k_make_trial: trial parameter state = current state with the free blocks replaced by x (internal order), and the
// pose tables of that state, in one launch.  One thread per pose, then one per camera (intrinsics), per board point, and one
// for the hand-eye pair (which must be complete before the derived frame poses: those threads recompute it themselves).
__device__ __forceinline__ void make_trial_item(const DeviceProblem& p, const double* x, double* cam_o, double* board_o, double* frame_o, double* intr_o,
                                                double* bpts_o, double* he_o, int i) {
  const int nfp = p.F * p.npf;
  const int np = p.C + p.B + nfp;
  if (i < np) {
    const double* cur; const double* src = nullptr; double* dst; PoseT* tab;
    if (i < p.C) { cur = p.cam_rt + 6 * i; dst = cam_o + 6 * i; tab = p.cam_T + i; if (p.off_cp >= 0) src = x + p.off_cp + 6 * i; }
    else if (i < p.C + p.B) { const int b = i - p.C; cur = p.board_rt + 6 * b; dst = board_o + 6 * b; tab = p.board_T + b; if (p.off_bp >= 0) src = x + p.off_bp + 6 * b; }
    else {
      const int q = i - p.C - p.B;
      if (p.motion == MOTION_HAND_EYE) {
        double he[12];
#pragma unroll
        for (int j = 0; j < 12; j++) he[j] = p.off_he >= 0 ? __ldcg(&x[p.off_he + j]) : p.he_rt[j];
        PoseT t; hand_eye_frame(he, p.arm_T[q], t); p.frame_T[q] = t;
        return;
      }
      cur = p.frame_rt + 6 * q; dst = frame_o + 6 * q; tab = p.frame_T + q; if (p.motion_on) src = x + p.n_s + 6 * q;
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
    for (int j = 0; j < p.kint; j++) {
      double v = __ldcg(&src[j]);
      if (j == 1 && p.fix_aspect && p.off_in >= 0) v = __ldcg(&src[0]);      // fy follows fx (camera.py:159-160)
      intr_o[p.kint * c + j] = v;
    }
  } else if (i < np + p.C + p.B * p.P) {
    const int q = i - np - p.C;                                       // padded board point index b*P + p
    const double* src = p.off_pt >= 0 ? x + p.off_pt + 3 * q : p.board_pts + 3 * q;
    bpts_o[3 * q] = __ldcg(&src[0]); bpts_o[3 * q + 1] = __ldcg(&src[1]); bpts_o[3 * q + 2] = __ldcg(&src[2]);
  } else if (i < np + p.C + p.B * p.P + 2 && p.motion == MOTION_HAND_EYE) {
    const int j = i - np - p.C - p.B * p.P;
    const double* src = p.off_he >= 0 ? x + p.off_he + 6 * j : p.he_rt + 6 * j;
    double v[6];
#pragma unroll
    for (int k = 0; k < 6; k++) { v[k] = __ldcg(&src[k]); he_o[6 * j + k] = v[k]; }
    PoseT t;
    pose_from_rt(v, t);
    p.he_T[j] = t;
  }
}
__global__ void k_make_trial(DeviceProblem p, const double* x, double* cam_o, double* board_o, double* frame_o, double* intr_o, double* bpts_o, double* he_o) {
  make_trial_item(p, x, cam_o, board_o, frame_o, intr_o, bpts_o, he_o, blockIdx.x * blockDim.x + threadIdx.x);
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
  double* moments;     // MODE_MOMENTS: [V][T]
  double* view_cost;   // MODE_COST   : [V]
  double* resid;       // MODE_RESID  : [2N] canonical order
  double* err;         // MODE_ERROR  : [N]  canonical order
};
enum { MODE_COST = 0, MODE_MOMENTS = 1, MODE_RESID = 2, MODE_ERROR = 3 };

constexpr int VIEW_WARPS = 4;          // warps per CTA for k_views
constexpr double SCIPY_EPS = 2.220446049250313e-16;
constexpr double TRIGGS_FLOOR = 0.1;

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
        // robust loss per scalar residual (least_squares.py construct_loss_function, common.py:720-731)
        if (a.loss == 0) acc += 0.5 * (ru * ru + rv * rv);
        else {
          const double is = 1.0 / a.f_scale, fs2 = a.f_scale * a.f_scale;
          double zu = ru * is, zv = rv * is;
          zu *= zu; zv *= zv;
          double r0u, r1u, r2u, r0v, r1v, r2v;
          loss_rho(a.loss, zu, r0u, r1u, r2u);
          loss_rho(a.loss, zv, r0v, r1v, r2v);
          acc += 0.5 * fs2 * (r0u + r0v);
        }
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
// k_views_mma: the per-view moment accumulation as what it is -- a small fp64 SYRK.  Per 32-corner chunk the warp
// stages Gt = [G | r] (64 residual rows x NC columns, NC = D+1 padded to a multiple of 8) in shared memory and
// accumulates M += Gt^T Gt on the fp64 tensor path (mma.sync m8n8k4 "DMMA"; wgmma has no fp64 kind).  The 8x8 C
// fragments ARE the per-view accumulators (2 doubles per lane and tile), so one pass produces all D(D+1)/2 + D
// moments: no register-limited PART split, no cross-lane reduction.  Same outputs as k_views<MODE_MOMENTS>.
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

#ifndef MMA_MIN_CTAS
#define MMA_MIN_CTAS 4
#endif
constexpr int MMA_KPAD = 68;     // 64 residual rows + 4: (column stride mod 16 doubles) == 4 -> conflict-free fragment loads
__host__ __device__ constexpr int mma_nc(int model, bool roll = false) { return ((model_D(model) + (roll ? 6 : 0) + 1 + 7) / 8) * 8; }

// WPV = warps per view: 1 (one warp owns a view; many views) or VIEW_WARPS (the CTA's warps split one view's chunks and meet in
// shared memory once: few, long views -- e.g. 4 cameras x 200 frames -- would otherwise leave most of the machine idle).
// ROLL (RollingFrames): the local row has two twist blocks, [xi_start (6) | xi_end (6) | fx fy cx cy dist], weighted by
// (1 - tau) and tau -- d x_cam = (1-tau) (omega_s x X_s + v_s) + tau (omega_e x X_e + v_e).
template <int MODEL, int WPV, bool ROLL = false>
__global__ void __launch_bounds__(VIEW_WARPS * 32, ((MODEL == MODEL_TILTED || ROLL) ? 2 : MMA_MIN_CTAS))
k_views_mma(DeviceProblem p, ViewKernelArgs a) {
  constexpr int ND = model_nd(MODEL);
  constexpr int KO = ROLL ? 12 : 6;              // offset of the intrinsics in the local row
  constexpr int D = KO + 4 + ND;
  constexpr int E = D * (D + 1) / 2;
  constexpr int T = E + D + 1;
  constexpr int NC = mma_nc(MODEL, ROLL);
  constexpr int NT = NC / 8;
  constexpr int NPAIR = NT * (NT + 1) / 2;
  constexpr int KINT = 5 + ND;
  extern __shared__ double stage_all[];

  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int gw = (WPV == 1) ? blockIdx.x * VIEW_WARPS + warp : blockIdx.x;
  const int nw = (WPV == 1) ? gridDim.x * VIEW_WARPS : gridDim.x;
  double* stage = stage_all + (size_t)warp * NC * MMA_KPAD;      // [NC][MMA_KPAD], element (row k, col j) at j*KPAD + k
  double* xred = stage_all + (size_t)VIEW_WARPS * NC * MMA_KPAD; // WPV > 1: [warp][2*NPAIR + 1][32]
  const int grp = lane >> 2, tig = lane & 3;
  const int sub = (WPV == 1) ? 0 : warp;

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

    double acc[NPAIR][2];
#pragma unroll
    for (int i = 0; i < NPAIR; i++) { acc[i][0] = 0.0; acc[i][1] = 0.0; }
    double cost_acc = 0.0;

    for (int base = beg + 32 * sub; base < end; base += 32 * WPV) {
      const int idx = base + lane;
      double gu[NC], gv[NC];
#pragma unroll
      for (int i = 0; i < NC; i++) { gu[i] = 0.0; gv[i] = 0.0; }
      if (idx < end) {
        const double2 ob = p.obs[idx];
        const int pi = p.pid[idx];
        const double X[3] = {bp[3 * pi], bp[3 * pi + 1], bp[3 * pi + 2]};
        const double tau = ob.y * inv_h;
        double Xc[3], Xs[3], Xe[3];
        corner_point<ROLL>(vp, vpe, X, tau, Xc, Xs, Xe);
        double u, w_;
        double Ju[3], Jv[3], ku[4 + ND], kv[4 + ND];
        project<MODEL, true>(Xc, k, u, w_, Ju, Jv, ku, kv);
        double ru = u - ob.x, rv = w_ - ob.y;
        double wu = 1.0, wv = 1.0;
        if (a.loss == 0) {
          cost_acc += 0.5 * (ru * ru + rv * rv);
        } else {
          const double is = 1.0 / a.f_scale, fs2 = a.f_scale * a.f_scale;
          double zu = ru * is, zv = rv * is;
          zu *= zu; zv *= zv;
          double r0u, r1u, r2u, r0v, r1v, r2v;
          loss_rho(a.loss, zu, r0u, r1u, r2u);
          loss_rho(a.loss, zv, r0v, r1v, r2v);
          cost_acc += 0.5 * fs2 * (r0u + r0v);
          double ju = r1u + 2.0 * r2u * zu, jv = r1v + 2.0 * r2v * zv;
          ju = fmax(fmax(ju, TRIGGS_FLOOR * r1u), SCIPY_EPS);
          jv = fmax(fmax(jv, TRIGGS_FLOOR * r1v), SCIPY_EPS);
          wu = sqrt(ju); wv = sqrt(jv);
          ru *= r1u / wu; rv *= r1v / wv;
        }
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
        gu[D] = ru; gv[D] = rv;                      // residual column: Gt^T Gt then carries G^T r as well
      }
      // stage: rows 2*lane (u) and 2*lane+1 (v); one 16-byte store per column, consecutive lanes -> consecutive addresses
#pragma unroll
      for (int j = 0; j < NC; j++)
        *reinterpret_cast<double2*>(stage + j * MMA_KPAD + 2 * lane) = make_double2(gu[j], gv[j]);
      __syncwarp();
      // 16 k-steps of 4 residual rows; fragment of column tile I = Gt[k0 + tig][8 I + grp] serves as A (row tile) and B (col tile)
      const int ksteps = (2 * min(32, end - base) + 3) >> 2;       // ragged last chunk: skip all-zero row groups
#pragma unroll 4
      for (int ks = 0; ks < ksteps; ks++) {
        double fr[NT];
#pragma unroll
        for (int I = 0; I < NT; I++) fr[I] = stage[(8 * I + grp) * MMA_KPAD + 4 * ks + tig];
        int t = 0;
#pragma unroll
        for (int I = 0; I < NT; I++)
#pragma unroll
          for (int J = I; J < NT; J++) { dmma884(acc[t][0], acc[t][1], fr[I], fr[J]); t++; }
      }
      __syncwarp();
    }

#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cost_acc += __shfl_xor_sync(0xffffffffu, cost_acc, o);
    if constexpr (WPV > 1) {       // meet: warp 0 adds the other warps' fragments (same lane -> same matrix element)
      __syncthreads();
      if (warp > 0) {
#pragma unroll
        for (int t = 0; t < NPAIR; t++) { xred[((warp * (2 * NPAIR + 1)) + 2 * t) * 32 + lane] = acc[t][0]; xred[((warp * (2 * NPAIR + 1)) + 2 * t + 1) * 32 + lane] = acc[t][1]; }
        if (lane == 0) xred[(warp * (2 * NPAIR + 1) + 2 * NPAIR) * 32] = cost_acc;
      }
      __syncthreads();
      if (warp > 0) continue;
#pragma unroll
      for (int w = 1; w < WPV; w++) {
#pragma unroll
        for (int t = 0; t < NPAIR; t++) { acc[t][0] += xred[((w * (2 * NPAIR + 1)) + 2 * t) * 32 + lane]; acc[t][1] += xred[((w * (2 * NPAIR + 1)) + 2 * t + 1) * 32 + lane]; }
        cost_acc += xred[(w * (2 * NPAIR + 1) + 2 * NPAIR) * 32];
      }
    }
    // ---- write the view's moments in the layout the expand kernels read
    double* out = a.moments + (size_t)v * T;
    {
      int t = 0;
#pragma unroll
      for (int I = 0; I < NT; I++)
#pragma unroll
        for (int J = I; J < NT; J++) {
#pragma unroll
          for (int h = 0; h < 2; h++) {
            const int i = 8 * I + grp, j = 8 * J + 2 * tig + h;
            const double val = acc[t][h];
            if (i < D && j < D && i <= j) out[tri_index(D, i, j)] = val;
            else if (i < D && j == D) out[E + i] = val;
          }
          t++;
        }
    }
    if (lane == 0) { out[T - 1] = cost_acc; if (a.view_cost) a.view_cost[v] = cost_acc; }     // compact copy for the acceptance test
  }
}

// ------------------------------------------------------------------------------------------------
// Block maps shared by the two expand kernels.
struct SolverBuffers {
  double* moments;   // [V][T]
  double* Hss;       // [n_s][n_s] full symmetric (local contribution of this rank)
  double* g;         // [n] gradient J^T f  (shared part local until all-reduced)
  double* Hff;       // [F][36]
  double* W;         // [F][n_s][6]   H[shared, frame f]
  double* cost_part; // per-CTA partial costs of k_expand_shared
  int zero_shared;   // unused
};

__device__ __forceinline__ int intr_param_index(const DeviceProblem& p, int local /*0..3+nd*/) {
  // local [fx fy cx cy dist...] -> index in [fx fy cx cy skew dist...]; fix_aspect folds fy onto fx (camera.py:159-160)
  if (local == 1 && p.fix_aspect) return 0;
  return local < 4 ? local : local + 1;
}

__device__ __forceinline__ int intr_param_index(const DeviceProblem& p, int local);

// Both expand kernels work warp-per-view: a warp pulls one view's moment record (T doubles) into its private shared
// memory slice, builds the 6x6 twist maps it needs, and does the small products with lane-owned outputs -- only
// __syncwarp inside the view loop; warps of a CTA run different views concurrently and meet once at the end.
constexpr int EXP_THREADS = 128;
constexpr int EXP_WARPS = EXP_THREADS / 32;

__device__ __forceinline__ void view_chain(const PoseT& pc, const PoseT& pf, double* Rcf, double* tcf) {
  mat3_mul(pc.R, pf.R, Rcf);
  mat3_vec(pc.R, pf.t, tcf);
  tcf[0] += pc.t[0]; tcf[1] += pc.t[1]; tcf[2] += pc.t[2];
}

// NP = twist blocks of the local row / pose-table entries per frame: 1 (static, hand-eye), 2 (rolling: start, end).  A parameter
// block reaches the local twists through NP 6x6 maps (camera pose: the same map for every block; board pose: one map per chain;
// frame pose j: its own map into block j only), so every product below is the static one summed over the NP blocks.
// per-warp shared slice of k_expand_frames: Ms[T] | Tm[D*FB] | Ac[36] | Af[NP*36] | Ab[NP*36] | Wb[B*6*FB]
__host__ __device__ inline int expf_warp_doubles(int T, int D, int B, int NP) { return T + D * 6 * NP + 36 + 72 * NP + B * 36 * NP; }

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

// The same maps computed by the WHOLE warp (opt-in MCBA_EXPAND=parallel): view_twist_maps leaves 3 (5) lanes with ~300 dependent
// flops each while 29 wait, once per view -- the longest serial piece of the expand kernels, which at 80 views per frame (cfg4) cost
// more than the moment kernel.  Three short phases instead: chain products (R_c R_f, t_cf) / R·J_L products and t_b / the 36 entries
// of every map, each entry by one lane from at most two products.  scr: 33 NP doubles of shared memory per warp.
//   A = twist_map(Rl, JL, t):  rows 0-2 = [Rl JL | 0],  rows 3-5 = [t x (Rl JL) columns | Rl]
template <int NP>
__device__ __forceinline__ void view_twist_maps_par(const DeviceProblem& p, int c, int f, int b, int lane, double* Ac, double* Af, double* Ab, double* scr) {
  const PoseT& pc = p.cam_T[c];
  const PoseT& pb = p.board_T[b];
  double* Rcf = scr;                    // [NP][9]
  double* tcf = Rcf + 9 * NP;           // [NP][3]
  double* tb = tcf + 3 * NP;            // [NP][3]
  double* RJf = tb + 3 * NP;            // [NP][9]  R_c JL_f
  double* RJb = RJf + 9 * NP;           // [NP][9]  R_cf JL_b
  // phase A: the chain up to the frame pose(s)
  for (int o = lane; o < 12 * NP; o += 32) {
    const int j = o / 12, e = o % 12;
    const PoseT& pf = p.frame_T[f * NP + j];
    if (e < 9) { const int r = e / 3, cc = e % 3; Rcf[9 * j + e] = pc.R[3 * r] * pf.R[cc] + pc.R[3 * r + 1] * pf.R[3 + cc] + pc.R[3 * r + 2] * pf.R[6 + cc]; }
    else { const int r = e - 9; tcf[3 * j + r] = pc.R[3 * r] * pf.t[0] + pc.R[3 * r + 1] * pf.t[1] + pc.R[3 * r + 2] * pf.t[2] + pc.t[r]; }
  }
  __syncwarp();
  // phase B: R J_L products and the chain translation up to the board pose
  for (int o = lane; o < 21 * NP; o += 32) {
    const int j = o / 21, e = o % 21;
    const PoseT& pf = p.frame_T[f * NP + j];
    const double* Rc = Rcf + 9 * j;
    if (e < 9) { const int r = e / 3, cc = e % 3; RJf[9 * j + e] = pc.R[3 * r] * pf.JL[cc] + pc.R[3 * r + 1] * pf.JL[3 + cc] + pc.R[3 * r + 2] * pf.JL[6 + cc]; }
    else if (e < 18) { const int q = e - 9, r = q / 3, cc = q % 3; RJb[9 * j + q] = Rc[3 * r] * pb.JL[cc] + Rc[3 * r + 1] * pb.JL[3 + cc] + Rc[3 * r + 2] * pb.JL[6 + cc]; }
    else { const int r = e - 18; tb[3 * j + r] = Rc[3 * r] * pb.t[0] + Rc[3 * r + 1] * pb.t[1] + Rc[3 * r + 2] * pb.t[2] + tcf[3 * j + r]; }
  }
  __syncwarp();
  // phase C: map entries.  m = 0: camera pose (Rl = I, RJ = JL_c, t = t_c); 1 .. NP: frame pose j; NP+1 .. 2NP: board pose through chain j
  const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int o = lane; o < 36 * (1 + 2 * NP); o += 32) {
    const int m = o / 36, e = o % 36, kk = e / 6, col = e % 6;
    const double* RJ; const double* Rl; const double* t; double* out;
    if (m == 0) { RJ = pc.JL; Rl = I3; t = pc.t; out = Ac; }
    else if (m <= NP) { const int j = m - 1; RJ = RJf + 9 * j; Rl = pc.R; t = tcf + 3 * j; out = Af ? Af + 36 * j : nullptr; }
    else { const int j = m - 1 - NP; RJ = RJb + 9 * j; Rl = Rcf + 9 * j; t = tb + 3 * j; out = Ab ? Ab + 36 * j : nullptr; }
    if (!out) continue;
    double val;
    if (kk < 3) val = col < 3 ? RJ[3 * kk + col] : 0.0;
    else {
      const int r = kk - 3;
      if (col < 3) {
        const double a0 = RJ[col], a1 = RJ[3 + col], a2 = RJ[6 + col];
        val = r == 0 ? t[1] * a2 - t[2] * a1 : r == 1 ? t[2] * a0 - t[0] * a2 : t[0] * a1 - t[1] * a0;
      } else val = Rl[3 * r + col - 3];
    }
    out[e] = val;
  }
}

// hand-eye twist maps of one view into Eh[6][12] = [A_W | A_G] (see k_expand_hand_eye): `role` 0 computes the W half, 1 the G half
__device__ __forceinline__ void hand_eye_twist_maps(const DeviceProblem& p, int c, int f, int role, double* Eh) {
  const PoseT& pc = p.cam_T[c];
  const PoseT& pW = p.he_T[0];
  const PoseT& pG = p.he_T[1];
  double A[36];
  if (role == 0) {           // W: left part T_c G A_f, chain translation up to and including W = t(T_c T_f)
    const PoseT& pf = p.frame_T[f];
    const PoseT& pa = p.arm_T[f];
    double Rcf[9], tcf[3], Rcg[9], Rl[9];
    view_chain(pc, pf, Rcf, tcf);
    mat3_mul(pc.R, pG.R, Rcg);
    mat3_mul(Rcg, pa.R, Rl);
    twist_map(Rl, pW.JL, tcf, A);
    for (int kk = 0; kk < 6; kk++) for (int j = 0; j < 6; j++) Eh[kk * 12 + j] = A[kk * 6 + j];
  } else {                   // G: left part T_c, chain translation up to and including G = R_c t_G + t_c
    double tcg[3];
    mat3_vec(pc.R, pG.t, tcg);
    tcg[0] += pc.t[0]; tcg[1] += pc.t[1]; tcg[2] += pc.t[2];
    twist_map(pc.R, pG.JL, tcg, A);
    for (int kk = 0; kk < 6; kk++) for (int j = 0; j < 6; j++) Eh[kk * 12 + 6 + j] = A[kk * 6 + j];
  }
}

// k_point_blocks (boards=True only): board points as shared parameters (3 per padded point).  One warp per view, one
// thread per corner: d r / d X_board = J_proj R_cfb (rolling: the blend (1-tau) R_start + tau R_end); the point's own 3x3 block,
// its gradient and its couplings with the camera pose / intrinsics / board pose / hand-eye pair (H_ss) and the frame block (W_f)
// are added with fp64 atomics on top of what the expand kernels wrote.  Replaces the axis-3 column block of the reference's
// sparsity pattern (calibration.py:188-190).  NP = 2: rolling frames (two twist blocks per row, 12-wide frame block).
template <int MODEL, int NP>
__global__ void __launch_bounds__(VIEW_WARPS * 32)
k_point_blocks(DeviceProblem p, ViewKernelArgs a, double* Hss, double* W, double* g) {
  constexpr bool ROLL = NP == 2;
  constexpr int ND = model_nd(MODEL);
  constexpr int KINT = 5 + ND;
  constexpr int NIN = 4 + ND;
  constexpr int KO = 6 * NP, FB = 6 * NP;
  __shared__ double maps[VIEW_WARPS][36 + 72 * NP + 72];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gw = blockIdx.x * VIEW_WARPS + warp, nw = gridDim.x * VIEW_WARPS;
  const int n_s = p.n_s;
  double* Ac = maps[warp]; double* Af = Ac + 36; double* Ab = Af + 36 * NP; double* Eh = Ab + 36 * NP;
  for (int v = gw; v < p.V; v += nw) {
    const int c = p.view_cam[v], f = p.view_frame[v], b = p.view_board[v];
    const int beg = p.view_start[v], end = p.view_start[v + 1];
    ViewPose vp, vpe;
    compose_views<ROLL>(p, c, f, b, vp, vpe);
    const double inv_h = ROLL ? 1.0 / p.img_h[c] : 0.0;
    __syncwarp();
    view_twist_maps<NP>(p, c, f, b, lane, Ac, Af, Ab);
    if (p.off_he >= 0 && (lane == 8 || lane == 9)) hand_eye_twist_maps(p, c, f, lane - 8, Eh);
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
      double ru = u - ob.x, rv = w_ - ob.y, wu = 1.0, wv = 1.0;
      if (a.loss != 0) {
        const double is = 1.0 / a.f_scale;
        double zu = ru * is, zv = rv * is;
        zu *= zu; zv *= zv;
        double r0u, r1u, r2u, r0v, r1v, r2v;
        loss_rho(a.loss, zu, r0u, r1u, r2u);
        loss_rho(a.loss, zv, r0v, r1v, r2v);
        double ju = r1u + 2.0 * r2u * zu, jv = r1v + 2.0 * r2v * zv;
        ju = fmax(fmax(ju, TRIGGS_FLOOR * r1u), SCIPY_EPS);
        jv = fmax(fmax(jv, TRIGGS_FLOOR * r1v), SCIPY_EPS);
        wu = sqrt(ju); wv = sqrt(jv);
        ru *= r1u / wu; rv *= r1v / wv;
      }
      // local rows: twist block(s) (KO) then [fx fy cx cy dist] (NIN) -- the layout of k_views_mma
      double gu[KO + NIN], gv[KO + NIN];
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
#pragma unroll
      for (int i = 0; i < NIN; i++) { gu[KO + i] = 0.0; gv[KO + i] = 0.0; }
      gu[KO] = ku[0] * wu; gu[KO + 2] = wu; gv[KO + 1] = kv[1] * wv; gv[KO + 3] = wv;
#pragma unroll
      for (int i = 0; i < ND; i++) { gu[KO + 4 + i] = ku[4 + i] * wu; gv[KO + 4 + i] = kv[4 + i] * wv; }
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
        if (p.motion_on) {
#pragma unroll
          for (int col = 0; col < FB; col++) {
            double vf = 0.0;
#pragma unroll
            for (int kk = 0; kk < 6; kk++) vf += Q[6 * (col / 6) + kk] * Af[36 * (col / 6) + kk * 6 + col % 6];
            atomicAdd(&W[((size_t)f * n_s + pt + r) * FB + col], vf);
          }
        }
        if (p.off_he >= 0) {
#pragma unroll
          for (int j = 0; j < 12; j++) {
            double vh = 0.0;
#pragma unroll
            for (int kk = 0; kk < 6; kk++) vh += Q[kk] * Eh[kk * 12 + j];
            addS(pt + r, p.off_he + j, vh);
          }
        }
        if (in0 >= 0) {
#pragma unroll
          for (int i = 0; i < NIN; i++) {
            const double val = xu[r] * gu[KO + i] + xv[r] * gv[KO + i];
            if (val != 0.0) addS(pt + r, in0 + intr_param_index(p, i), val);
          }
        }
      }
    }
  }
}

// per-warp shared slice of k_expand_shared: Ms[T] | Um[D*6] | Ab[NP*36] | Ub[B*D*6] | Hbb[B*36] | gb[B*6]
__host__ __device__ inline int exps_warp_doubles(int T, int D, int B, int NP) { return T + D * 6 + 36 * NP + B * (D * 6 + 42); }

// k_expand_shared: one CTA per (camera, chunk of that camera's views).  The camera's own (pose+intrinsics) block is a
// plain sum of moment records (its twist map does not depend on the view) kept lane-distributed in registers; the
// camera-board and board-board blocks need the per-view board twist map(s).  Per-warp partials are summed once at the
// end and added into H_ss / g_s with fp64 atomics.
template <int NP>
__global__ void __launch_bounds__(EXP_THREADS)
k_expand_shared(DeviceProblem p, SolverBuffers s, int chunks) {
  constexpr int KO = 6 * NP;
  extern __shared__ double sh[];
  const int D = p.D, T = p.T, B = p.B, n_s = p.n_s;
  const int E = D * (D + 1) / 2;
  const int c = blockIdx.x / chunks, chunk = blockIdx.x % chunks;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wd = exps_warp_doubles(T, D, B, NP);
  double* Ms = sh + (size_t)warp * wd;
  double* Um = Ms + T;
  double* Ab = Um + D * 6;
  double* Ub = Ab + 36 * NP;
  double* Hbb = Ub + (size_t)B * D * 6;
  double* gb = Hbb + B * 36;
  double* Msum = sh + (size_t)EXP_WARPS * wd;          // [T] block total
  double* Ac = Msum + T;                                // 36
  for (int i = lane; i < B * (D * 6 + 42); i += 32) Ub[i] = 0.0;
  constexpr int MAXT = NP == 1 ? 11 : 16;                // ceil(T/32): tilted model, D = 24 (T = 325) / rolling tilted, D = 30 (T = 496)
  double macc[MAXT];
#pragma unroll
  for (int q = 0; q < MAXT; q++) macc[q] = 0.0;
  __syncwarp();

  const int l0 = p.cam_view_start[c], l1 = p.cam_view_start[c + 1];
  const int per = (l1 - l0 + chunks - 1) / chunks;
  const int a0 = l0 + chunk * per, a1 = min(l1, a0 + per);
  const PoseT& pc = p.cam_T[c];
  for (int li = a0 + warp; li < a1; li += EXP_WARPS) {
    const int v = p.cam_view_list[li];
    const int f = p.view_frame[v], b = p.view_board[v];
#pragma unroll
    for (int q = 0; q < MAXT; q++) {
      const int i = lane + 32 * q;
      if (i < T) { const double m = s.moments[(size_t)v * T + i]; Ms[i] = m; macc[q] += m; }
    }
    if (p.off_bp >= 0) {
      view_twist_maps<NP>(p, c, f, b, lane, nullptr, nullptr, Ab);
      __syncwarp();
      for (int o = lane; o < D * 6; o += 32) {           // Um = sum_a M[:, xi_a] Ab_a
        const int i = o / 6, j = o % 6; double acc = 0.0;
#pragma unroll
        for (int kk = 0; kk < KO; kk++) acc += msym(Ms, D, i, kk) * Ab[36 * (kk / 6) + (kk % 6) * 6 + j];
        Um[o] = acc;
        Ub[(size_t)b * D * 6 + o] += acc;
      }
      __syncwarp();
      for (int o = lane; o < 42; o += 32) {
        if (o < 36) { const int i = o / 6, j = o % 6; double acc = 0.0;
#pragma unroll
          for (int kk = 0; kk < KO; kk++) acc += Ab[36 * (kk / 6) + (kk % 6) * 6 + i] * Um[kk * 6 + j];
          Hbb[b * 36 + o] += acc; }
        else { const int i = o - 36; double acc = 0.0;
#pragma unroll
          for (int kk = 0; kk < KO; kk++) acc += Ab[36 * (kk / 6) + (kk % 6) * 6 + i] * Ms[E + kk];
          gb[b * 6 + i] += acc; }
      }
    }
    __syncwarp();
  }
  // ---- meet: block totals (warp 0's slice becomes the sum)
#pragma unroll
  for (int q = 0; q < MAXT; q++) { const int i = lane + 32 * q; if (i < T) Ms[i] = macc[q]; }
  __syncthreads();
  for (int i = tid; i < T; i += EXP_THREADS) {
    double acc = 0.0;
#pragma unroll
    for (int w = 0; w < EXP_WARPS; w++) acc += sh[(size_t)w * wd + i];
    Msum[i] = acc;
  }
  const int nb_part = B * (D * 6 + 42);
  const int part_off = T + D * 6 + 36 * NP;
  for (int i = tid; i < nb_part; i += EXP_THREADS) {
    double acc = 0.0;
#pragma unroll
    for (int w = 1; w < EXP_WARPS; w++) acc += sh[(size_t)w * wd + part_off + i];
    sh[part_off + i] += acc;                             // warp 0's Ub | Hbb | gb now hold the block totals
  }
  if (tid == 0) { const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; twist_map(I3, pc.JL, pc.t, Ac); }
  __syncthreads();
  Um = sh + T;                                           // warp 0's Um, reused by the whole block
  Ub = sh + part_off; Hbb = Ub + (size_t)B * D * 6; gb = Hbb + B * 36;
  if (tid == 0) s.cost_part[blockIdx.x] = Msum[T - 1];
  for (int o = tid; o < D * 6; o += EXP_THREADS) {       // Um = sum_a Msum[:, xi_a] Ac  (the camera's map is the same for every chain)
    const int i = o / 6, j = o % 6; double acc = 0.0;
#pragma unroll
    for (int kk = 0; kk < KO; kk++) acc += msym(Msum, D, i, kk) * Ac[(kk % 6) * 6 + j];
    Um[o] = acc;
  }
  __syncthreads();
  const int nin = 4 + p.nd;
  const int cp = p.off_cp >= 0 ? p.off_cp + 6 * c : -1;
  const int in0 = p.off_in >= 0 ? p.off_in + p.kint * c : -1;
  auto addH = [&](int i, int j, double val) {
    atomicAdd(&s.Hss[(size_t)i * n_s + j], val);
    if (i != j) atomicAdd(&s.Hss[(size_t)j * n_s + i], val);
  };
  if (cp >= 0) {
    for (int o = tid; o < 36; o += EXP_THREADS) {
      const int i = o / 6, j = o % 6;
      if (j < i) continue;
      double acc = 0.0;
#pragma unroll
      for (int kk = 0; kk < KO; kk++) acc += Ac[(kk % 6) * 6 + i] * Um[kk * 6 + j];
      addH(cp + i, cp + j, acc);
    }
    if (tid < 6) {
      double acc = 0.0;
#pragma unroll
      for (int kk = 0; kk < KO; kk++) acc += Ac[(kk % 6) * 6 + tid] * Msum[E + kk];
      atomicAdd(&s.g[cp + tid], acc);
    }
  }
  if (in0 >= 0) {
    if (cp >= 0)
      for (int o = tid; o < nin * 6; o += EXP_THREADS) {
        const int i = o / 6, j = o % 6;
        addH(in0 + intr_param_index(p, i), cp + j, Um[(KO + i) * 6 + j]);
      }
    for (int o = tid; o < nin * nin; o += EXP_THREADS) {
      const int i = o / nin, j = o % nin;
      atomicAdd(&s.Hss[(size_t)(in0 + intr_param_index(p, i)) * n_s + in0 + intr_param_index(p, j)], msym(Msum, D, KO + i, KO + j));
    }
    for (int i = tid; i < nin; i += EXP_THREADS) atomicAdd(&s.g[in0 + intr_param_index(p, i)], Msum[E + KO + i]);
  }
  if (p.off_bp >= 0) {
    for (int b = 0; b < B; b++) {
      const int bp = p.off_bp + 6 * b;
      const double* U = Ub + (size_t)b * D * 6;
      if (cp >= 0)
        for (int o = tid; o < 36; o += EXP_THREADS) {     // camera pose x board pose = sum_a Ac^T U_xi_a
          const int i = o / 6, j = o % 6; double acc = 0.0;
#pragma unroll
          for (int kk = 0; kk < KO; kk++) acc += Ac[(kk % 6) * 6 + i] * U[kk * 6 + j];
          if (acc != 0.0) addH(cp + i, bp + j, acc);
        }
      if (in0 >= 0)
        for (int o = tid; o < nin * 6; o += EXP_THREADS) { // intrinsics x board pose = U_k
          const int i = o / 6, j = o % 6; const double val = U[(KO + i) * 6 + j];
          if (val != 0.0) addH(in0 + intr_param_index(p, i), bp + j, val);
        }
      for (int o = tid; o < 36; o += EXP_THREADS) {
        const double val = Hbb[b * 36 + o];
        if (val != 0.0) atomicAdd(&s.Hss[(size_t)(bp + o / 6) * n_s + bp + o % 6], val);
      }
      if (tid < 6 && gb[b * 6 + tid] != 0.0) atomicAdd(&s.g[bp + tid], gb[b * 6 + tid]);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Hand-eye motion (motion/hand_eye.py:14-90): the frame pose is G A_f W with the arm pose A_f fixed, so the "motion" block is
// 12 SHARED parameters he = [W = world_wrt_base (6) | G = gripper_wrt_camera (6)] that every residual depends on
// (hand_eye.py:89-90) and there are no per-frame blocks to eliminate.  The per-view moments are the static ones (the chain
// T_c T_f T_b only changed how T_f is obtained); this kernel adds the he rows and columns of H_ss / g_s on top of
// k_expand_shared<1>.  Twist maps of one view (camera c, frame f):
//   W: left part T_c G A_f, chain translation up to and including W = t(T_c T_f)      -> twist_map(R_c R_G R_Af, JL_W, t_cf)
//   G: left part T_c,       chain translation up to and including G = R_c t_G + t_c   -> twist_map(R_c, JL_G, t_cG)
// per-warp shared slice: Ms[T] | Eh[6*12] | Ab[36] | Uh[D*12] | UhS[D*12] | Hhh[144] | gh[12] | Hbh[B*72]
__host__ __device__ inline int exph_warp_doubles(int T, int D, int B) { return T + 72 + 36 + 2 * D * 12 + 156 + B * 72; }

__global__ void __launch_bounds__(EXP_THREADS)
k_expand_hand_eye(DeviceProblem p, SolverBuffers s, int chunks) {
  extern __shared__ double sh[];
  const int D = p.D, T = p.T, B = p.B, n_s = p.n_s;
  const int E = D * (D + 1) / 2;
  const int c = blockIdx.x / chunks, chunk = blockIdx.x % chunks;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wd = exph_warp_doubles(T, D, B);
  double* Ms = sh + (size_t)warp * wd;
  double* Eh = Ms + T;                 // [6][12]
  double* Ab = Eh + 72;
  double* Uh = Ab + 36;                // [D][12]  M[:, xi] Eh of the current view
  double* UhS = Uh + D * 12;           // [D][12]  summed over this warp's views
  double* Hhh = UhS + D * 12;          // [12][12]
  double* gh = Hhh + 144;              // [12]
  double* Hbh = gh + 12;               // [B][6][12]
  const int npart = D * 12 + 156 + B * 72;
  for (int i = lane; i < npart; i += 32) UhS[i] = 0.0;
  __syncwarp();

  const int l0 = p.cam_view_start[c], l1 = p.cam_view_start[c + 1];
  const int per = (l1 - l0 + chunks - 1) / chunks;
  const int a0 = l0 + chunk * per, a1 = min(l1, a0 + per);
  const PoseT& pc = p.cam_T[c];
  for (int li = a0 + warp; li < a1; li += EXP_WARPS) {
    const int v = p.cam_view_list[li];
    const int f = p.view_frame[v], b = p.view_board[v];
    for (int i = lane; i < T; i += 32) Ms[i] = s.moments[(size_t)v * T + i];
    if (lane < 2) hand_eye_twist_maps(p, c, f, lane, Eh);
    else if (lane == 2 && p.off_bp >= 0) {
      const PoseT& pf = p.frame_T[f];
      const PoseT& pb = p.board_T[b];
      double Rcf[9], tcf[3], tb[3];
      view_chain(pc, pf, Rcf, tcf);
      mat3_vec(Rcf, pb.t, tb);
      tb[0] += tcf[0]; tb[1] += tcf[1]; tb[2] += tcf[2];
      twist_map(Rcf, pb.JL, tb, Ab);
    }
    __syncwarp();
    for (int o = lane; o < D * 12; o += 32) {            // Uh = M[:, xi] Eh
      const int i = o / 12, j = o % 12; double acc = 0.0;
#pragma unroll
      for (int kk = 0; kk < 6; kk++) acc += msym(Ms, D, i, kk) * Eh[kk * 12 + j];
      Uh[o] = acc;
      UhS[o] += acc;
    }
    __syncwarp();
    for (int o = lane; o < 156; o += 32) {               // Hhh += Eh^T Uh_xi ; gh += Eh^T g_xi
      double acc = 0.0;
      if (o < 144) { const int i = o / 12, j = o % 12;
#pragma unroll
        for (int kk = 0; kk < 6; kk++) acc += Eh[kk * 12 + i] * Uh[kk * 12 + j];
      } else { const int i = o - 144;
#pragma unroll
        for (int kk = 0; kk < 6; kk++) acc += Eh[kk * 12 + i] * Ms[E + kk];
      }
      Hhh[o] += acc;                                     // gh follows Hhh in the slice
    }
    if (p.off_bp >= 0)
      for (int o = lane; o < 72; o += 32) {              // board pose x he = Ab^T Uh_xi
        const int i = o / 12, j = o % 12; double acc = 0.0;
#pragma unroll
        for (int kk = 0; kk < 6; kk++) acc += Ab[kk * 6 + i] * Uh[kk * 12 + j];
        Hbh[b * 72 + o] += acc;
      }
    __syncwarp();
  }
  // ---- meet: warp 0's partials become the block totals
  __syncthreads();
  const int part_off = T + 72 + 36 + D * 12;
  for (int i = tid; i < npart; i += EXP_THREADS) {
    double acc = 0.0;
#pragma unroll
    for (int w = 1; w < EXP_WARPS; w++) acc += sh[(size_t)w * wd + part_off + i];
    sh[part_off + i] += acc;
  }
  double* Ac = sh + T;                                    // warp 0's Eh slot is free now
  if (tid == 0) { const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; twist_map(I3, pc.JL, pc.t, Ac); }
  __syncthreads();
  UhS = sh + part_off; Hhh = UhS + D * 12; gh = Hhh + 144; Hbh = gh + 12;
  const int he = p.off_he;
  const int nin = 4 + p.nd;
  const int cp = p.off_cp >= 0 ? p.off_cp + 6 * c : -1;
  const int in0 = p.off_in >= 0 ? p.off_in + p.kint * c : -1;
  auto addS = [&](int i, int j, double val) {             // off-diagonal block: both triangles
    atomicAdd(&s.Hss[(size_t)i * n_s + j], val);
    atomicAdd(&s.Hss[(size_t)j * n_s + i], val);
  };
  for (int o = tid; o < 144; o += EXP_THREADS) atomicAdd(&s.Hss[(size_t)(he + o / 12) * n_s + he + o % 12], Hhh[o]);
  if (tid < 12) atomicAdd(&s.g[he + tid], gh[tid]);
  if (cp >= 0)
    for (int o = tid; o < 72; o += EXP_THREADS) {         // camera pose x he = Ac^T UhS_xi
      const int i = o / 12, j = o % 12; double acc = 0.0;
#pragma unroll
      for (int kk = 0; kk < 6; kk++) acc += Ac[kk * 6 + i] * UhS[kk * 12 + j];
      addS(cp + i, he + j, acc);
    }
  if (in0 >= 0)
    for (int o = tid; o < nin * 12; o += EXP_THREADS) {   // intrinsics x he = UhS_k
      const int i = o / 12, j = o % 12;
      addS(in0 + intr_param_index(p, i), he + j, UhS[(6 + i) * 12 + j]);
    }
  if (p.off_bp >= 0)
    for (int o = tid; o < B * 72; o += EXP_THREADS) {
      const int b = o / 72, i = (o % 72) / 12, j = o % 12;
      const double val = Hbh[o];
      if (val != 0.0) addS(p.off_bp + 6 * b + i, he + j, val);
    }
}

}  // namespace mcba
