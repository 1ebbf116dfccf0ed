// linearize.cuh — the fused linearisation pass: residuals, analytic Jacobian rows, per-view moments on the fp64 tensor path AND their
// expansion into the block-arrow normal equations, in ONE kernel that reads every corner once and writes nothing per corner or per view.
//
//   k_linearize<MODEL, ROLL>   one CTA per frame (persistent, static frame -> CTA map), warps own the frame's views by camera:
//                              per view   M = sum [G r]^T [G r]  (mma.sync.m16n8k4.f64, view_chunk below)
//                              epilogue   the view's 6x6 twist maps (camera / frame / board pose -> camera-frame twist) applied to M:
//                                         H_ff, g_f, W_f (this frame's block row of the arrow) are COMPLETE when the CTA leaves the frame and
//                                         are stored once; the shared-parameter blocks are accumulated per (CTA, camera) in a record that
//                                         only this CTA's owning warp ever touches (plain read-modify-write in L2, no atomics).
//   k_reduce_shared<NP>        sums the per-CTA records in CTA order (fixed -> bit-reproducible run to run) and stores H_ss, g_s, cost.
//   k_fold_hand_eye            hand-eye frames: the 12 hand-eye rows and columns of H_ss, g_s as per-frame folds of H_ff, W_f, g_f
//                              (the frames are derived poses; their blocks are emitted for the fold only), summed in frame order.
// Every motion model goes through these kernels, and none of them adds to H or g with atomics: two identical linearisations agree bit for
// bit (only the board-point blocks of boards=True, k_point_blocks in kernels.cuh, are added with fp64 atomics).
// Reference semantics: the Jacobian scipy builds by finite differences over calibration.py:173-196's sparsity pattern, here analytic.
#pragma once
#include "solver_kernels.cuh"

namespace mcba {

constexpr int LIN_WARPS = 8;           // at most; the host takes fewer when two CTAs of 8 would not fit an SM's shared memory
constexpr int LIN_THREADS = LIN_WARPS * 32;
constexpr int LIN_KPAD = 36;           // 32 staged residual rows + 4: (column stride mod 16 doubles) == 4 -> conflict-free fragment loads
constexpr int LIN_MAXV = 96;           // views of a frame staged in shared memory (more: the list is read from global memory)
constexpr int LIN_MAXC = 1024;         // cameras tracked by the per-frame presence mask (more: W_f is zero-filled first)
constexpr int LIN_MAXB = 8;            // board pose tables staged per frame (more boards: the tables are read from global memory)
constexpr int LIN_TSTR = 12;           // row stride of T^t in the epilogue (stride mod 16 == 12: conflict-free fragment loads)
constexpr int LIN_VC = 44;             // per-warp view constants: 12 doubles per chain + the intrinsics
constexpr int LIN_WB_FLAG = 0x4000;    // scatter-table entry: add the view's board offset (rows of W_f that belong to board b)
constexpr int LIN_SMEM_MAX = 220 * 1024;   // dynamic shared memory of a CTA at most (bytes; the static part and the per-CTA reserve fit beside it)

// compile-time shape of a residual row's local Jacobian [twist block(s) | fx fy cx cy dist | r]
template <int MODEL, bool ROLL>
struct LinShape {
  static constexpr int ND = model_nd(MODEL);
  static constexpr int NP = ROLL ? 2 : 1;
  static constexpr int KO = 6 * NP;                 // twist columns
  static constexpr int NIN = 4 + ND;                // intrinsic columns
  static constexpr int D = KO + NIN;
  static constexpr int E = D * (D + 1) / 2;
  static constexpr int T = E + D + 1;               // moment record: upper triangle | G^T r | cost
  static constexpr int NC = mma_nc(MODEL, ROLL);    // staged columns (D + 1 padded to 8)
  static constexpr int NT = NC / 8;                 // 8-column tiles of M
  static constexpr int NMB = (NC + 15) / 16;        // 16-row blocks of M
  static constexpr int NBLK = NMB * NT - NMB * (NMB - 1);   // 16 x 8 C blocks on or above the diagonal: (mb, J) with J >= 2 mb
  static constexpr int KINT = 5 + ND;
  static constexpr int FB = KO;                     // parameters of one eliminated frame block
  static constexpr int UB = D * 6 + 42;             // per (camera, board): M[:,xi] Ab (D x 6) | Ab^T M Ab (36) | Ab^T g (6)
};

// One 32-corner chunk of a view: every lane computes its corner's residual pair and 2 x D Jacobian rows (fp64), the warp stages
// [G | r] (64 rows x NC columns) in shared memory and accumulates M += [G r]^T [G r] into the DMMA C fragments `acc`: block t = (mb, J)
// of the enumeration mb = 0.., J = 2 mb .. NT-1 holds M[16 mb .. 16 mb + 15][8 J .. 8 J + 7].
template <int MODEL, bool ROLL>
__device__ __forceinline__ void view_chunk(const DeviceProblem& p, int loss, double f_scale, const ViewPose& vp, const ViewPose& vpe, const double* k,
                                           const double* bp, double inv_h, int base, int end, int lane, double* stage,
                                           double (&acc)[LinShape<MODEL, ROLL>::NBLK][4], double& cost_acc, double2 ob, int pi) {
  using S = LinShape<MODEL, ROLL>;
  constexpr int ND = S::ND, D = S::D, NC = S::NC, NT = S::NT, NMB = S::NMB;
  const int grp = lane >> 2, tig = lane & 3;
  const int idx = base + lane;
  double gu[NC], gv[NC];
#pragma unroll
  for (int i = 0; i < NC; i++) { gu[i] = 0.0; gv[i] = 0.0; }
  if (idx < end) {
    const double X[3] = {bp[3 * pi], bp[3 * pi + 1], bp[3 * pi + 2]};
    const double tau = ob.y * inv_h;
    double Xc[3], Xs[3], Xe[3];
    corner_point<ROLL>(vp, vpe, X, tau, Xc, Xs, Xe);
    double u, w_;
    double Ju[3], Jv[3], ku[4 + ND], kv[4 + ND];
    project<MODEL, true>(Xc, k, u, w_, Ju, Jv, ku, kv);
    const CornerLoss cl = corner_loss(loss, f_scale, u - ob.x, w_ - ob.y, cost_acc);      // projected - observed (calibration.py:206)
    corner_row<MODEL, ROLL>(Xc, Xs, Xe, tau, Ju, Jv, ku, kv, cl.wu, cl.wv, gu, gv);
    gu[D] = cl.ru; gv[D] = cl.rv;                // residual column: Gt^T Gt then carries G^T r as well
  }
  // The 64 residual rows of the chunk go through the stage buffer in two halves of 32 (lanes 0-15, then lanes 16-31): half the shared
  // memory per warp, so that twice the warps fit an SM (the pass is latency-bound per warp: resident warps are what hides it).
  // rows 2*l (u) and 2*l+1 (v) of a half; one 16-byte store per column, consecutive lanes -> consecutive addresses.
  const int cnt = min(32, end - base);
#pragma unroll
  for (int half = 0; half < 2; half++) {
    if ((lane >> 4) == half) {
#pragma unroll
      for (int j = 0; j < NC; j++)
        *reinterpret_cast<double2*>(stage + j * LIN_KPAD + 2 * (lane & 15)) = make_double2(gu[j], gv[j]);
    }
    __syncwarp();
    // m16n8k4 steps of 4 residual rows; fr[I] = Gt[k0 + tig][8 I + grp] of column tile I: tiles 2 mb, 2 mb + 1 are the A fragment of row
    // block mb (a tile past NC reads as zero), tile J is the B fragment of block (mb, J)
    const int rows = 2 * max(0, min(16, cnt - 16 * half));
    const int ksteps = (rows + 3) >> 2;                          // ragged last chunk: skip all-zero row groups
#pragma unroll
    for (int ks = 0; ks < 8; ks++) {
      if (ks >= ksteps) break;
      double fr[2 * NMB];
#pragma unroll
      for (int I = 0; I < 2 * NMB; I++) fr[I] = I < NT ? stage[(8 * I + grp) * LIN_KPAD + 4 * ks + tig] : 0.0;
      int t = 0;
#pragma unroll
      for (int mb = 0; mb < NMB; mb++)
#pragma unroll
        for (int J = 2 * mb; J < NT; J++) {
          const double a[2] = {fr[2 * mb], fr[2 * mb + 1]}, b[1] = {fr[J]};
          dmma1684(acc[t], a, b);
          t++;
        }
    }
    __syncwarp();
  }
}

struct LinArgs {
  int loss; double f_scale;
  int split;             // warps per view: LIN_WARPS / split camera slots per CTA (split > 1 when the rig has fewer cameras than a CTA has warps)
  double* Hff;           // [F][FB*FB]
  double* g;             // [n]: frame parts written here (shared part by k_reduce_shared)
  double* W;             // [F][n_s][FB]
  double* spart;         // [grid][C][rec]   rec = T + B*UB   per-(CTA, camera) partial sums of the shared blocks
  double* frame_cost;    // [F]
};

__host__ __device__ inline int lin_record_doubles(int T, int D, int B) { return T + B * (D * 6 + 42); }
// dynamic shared memory of k_linearize in doubles
__host__ __device__ inline size_t lin_warp_doubles(int NC, int T, int D, int FB, int nin, int B, int NP) {
  (void)nin;
  const int KO = 6 * NP, PC = 6 * (NP + 1);
  const int PT = (PC + 7) / 8, EK = 4 * ((KO + 3) / 4), EP = 8 * PT + 4, MR = 8 * ((EK + 7) / 8);
  const int need = MR * (NC + 4) + 8 * PT * LIN_TSTR, chunk = NC * LIN_KPAD;
  return ((size_t)(((chunk > need ? chunk : need) + 1) & ~1)      // stage (chunk loop, 32 rows at a time) = Ms | T^t (epilogue)
       + EK * EP + 12 * NP                // E: twist maps of the view [EK][EP], zero padded | chain R_cf, t_cf
       + (size_t)B * 6 * FB               // Wb: this warp's partial board rows of W_f
       + FB * FB + FB                     // hacc: H_ff | g_f partial
       + D * FB                           // wacc: sum over the camera's boards of M[:, xi] Af
       + T                                // macc: raw moment sum of the current camera
       + (D * 6 + 42)                     // ub: board coupling of the current (camera, board)
       + 6                                // cost of this frame's views | cur_cam | cur_board | wdirty | chain frame | chain camera
       + LIN_VC                           // pose and intrinsics of the view in progress
       + 1) & ~(size_t)1;                 // even: every warp's stage buffer takes 16-byte stores
}
// dynamic shared memory of a CTA of `warps` warps: the warps' slices, then the pose tables staged per frame (frame [NP] | boards [min(B, LIN_MAXB)])
__host__ __device__ inline size_t lin_smem_doubles(int NC, int T, int D, int FB, int nin, int B, int NP, int warps) {
  return (size_t)warps * lin_warp_doubles(NC, T, D, FB, nin, B, NP) + (size_t)24 * (2 * NP + (B < LIN_MAXB ? B : LIN_MAXB));      // frame table x 2 (double buffer) | board tables
}

// fire-and-forget fp64 add to global memory.  Every address of a CTA's records is only ever updated by ONE lane of ONE warp of that CTA,
// and a thread's operations on one address are applied in program order: the sums are as reproducible as with load-add-store, without
// paying the L2 round trip per update (the records live in L2; nothing waits for them until k_reduce_shared).
__device__ __forceinline__ void red_add(double* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}

// per-warp shared-memory layout of k_linearize (doubles from the warp's base).  The epilogue's per-view scratch aliases the stage
// buffer of the chunk loop; what must survive from view to view lies behind it.
template <int MODEL, bool ROLL>
struct LinLayout {
  using S = LinShape<MODEL, ROLL>;
  static constexpr int PC = 6 * (S::NP + 1);                    // columns of the map matrix E: frame-pose block(s) | board-pose block
  static constexpr int PT = (PC + 7) / 8;                       // 8-row tiles of T^t = E^T M[xi, :] (rows of T^t held, columns of E)
  static constexpr int PM = (PC + 15) / 16;                     // 16-row blocks of the products: rows past 8 PT are zero, never loaded or stored
  static constexpr int KS = (S::KO + 3) / 4;                    // quads of twist components: m16n8k8 steps, m16n8k4 for an odd last quad
  static constexpr int EK = 4 * KS;                             // rows of E (twist components), zero padded to the k-steps
  static constexpr int EP = 8 * PT + 4;                         // row stride of E; strides mod 16 == 4 or 12: the mma fragment loads
  static constexpr int MSTR = S::NC + 4;                        //   (address = 4-lane group x stride + lane in group) hit 16 different banks
  static constexpr int MR = 8 * ((EK + 7) / 8);                 // rows of M the epilogue multiplies with: the twist rows
  static constexpr int Ms = 0;                                  // [MR][MSTR] rows xi of the view's moment matrix, column D = G^T r
  static constexpr int Tt = Ms + MR * MSTR;                     // [8 PT][LIN_TSTR]   T^t[:, xi]
  static constexpr int stage_need = Tt + 8 * PT * LIN_TSTR;     // what the epilogue needs
  static constexpr int stage_end = ((S::NC * LIN_KPAD > stage_need ? S::NC * LIN_KPAD : stage_need) + 1) & ~1;
  static_assert((4 * S::NBLK + 1) * 32 <= stage_end, "the fragments of a view part must fit the warp's stage buffer");
  static_assert(EK <= LIN_TSTR && (MSTR % 16 == 4 || MSTR % 16 == 12) && (EP % 16 == 4 || EP % 16 == 12), "fragment strides");
  static constexpr int NHF = S::FB * S::FB + S::FB;             // H_ff | g_f
  static constexpr int NWC = S::D * S::FB;                      // sum over the camera's boards of Tf = M[:, xi] Af (D x FB)
  // scatter tables (per CTA, one entry per lane): where the C fragments of the epilogue's products and of the moment tiles are added
  static constexpr int NTT = PM * S::NT * 4, NTP = PM * PT * 4, NTM = S::NBLK * 4;
  // after the stage buffer: E [EK][EP] | chain (R_cf 9, t_cf 3) x NP | Wb [B][6][FB] | hacc [NHF] | wacc [NWC] | macc [T] | ub [UB] | tail [6]
  static constexpr int E = stage_end;
  static constexpr int chain = E + EK * EP;
  static constexpr int Wb = chain + 12 * S::NP;
  __device__ static int hacc(int B) { return Wb + B * 6 * S::FB; }
  __device__ static int wacc(int B) { return hacc(B) + NHF; }
  __device__ static int macc(int B) { return wacc(B) + NWC; }
  __device__ static int ub(int B) { return macc(B) + S::T; }
  __device__ static int tail(int B) { return ub(B) + S::UB; }      // [0] frame cost of this warp's views, [1] cur_cam, [2] cur_board, [3] wdirty, [4] [5] frame / camera of the chain cache
  __device__ static int vc(int B) { return tail(B) + 6; }          // constants of the view in progress: pose R, t [12 NP] | intrinsics [KINT]  (LIN_VC doubles)
};

// one entry e = kk*6 + col of the 6x6 twist map of a pose (geometry.cuh twist_map): RJ = R_left J_L, Rl = R_left, t = chain translation
__device__ __forceinline__ double twist_entry(const double* RJ, const double* Rl, const double* t, int kk, int col) {
  if (kk < 3) return col < 3 ? RJ[3 * kk + col] : 0.0;
  const int r = kk - 3;
  if (col >= 3) return Rl[3 * r + col - 3];
  const double a0 = RJ[col], a1 = RJ[3 + col], a2 = RJ[6 + col];
  return r == 0 ? t[1] * a2 - t[2] * a1 : r == 1 ? t[2] * a0 - t[0] * a2 : t[0] * a1 - t[1] * a0;
}

// running sums -> this CTA's records / this frame's W_f rows (leader warps)
template <int MODEL, bool ROLL>
__device__ __forceinline__ void lin_flush_ub(const DeviceProblem& p, double* w, double* myrec, int lane) {
  using S = LinShape<MODEL, ROLL>; using L = LinLayout<MODEL, ROLL>;
  const int B = p.B;
  double* tl = w + L::tail(B);
  const int cam = (int)tl[1], board = (int)tl[2];
  if (cam < 0 || board < 0 || p.off_bp < 0) return;
  double* ub = w + L::ub(B);
  double* r = myrec + (size_t)cam * lin_record_doubles(S::T, S::D, B) + S::T + (size_t)board * S::UB;
  for (int i = lane; i < S::UB; i += 32) { red_add(r + i, ub[i]); ub[i] = 0.0; }
}
template <int MODEL, bool ROLL>
__device__ __forceinline__ void lin_flush_macc(const DeviceProblem& p, double* w, double* myrec, int lane) {
  using S = LinShape<MODEL, ROLL>; using L = LinLayout<MODEL, ROLL>;
  const int B = p.B;
  const int cam = (int)(w + L::tail(B))[1];
  if (cam < 0) return;
  double* macc = w + L::macc(B);
  double* r = myrec + (size_t)cam * lin_record_doubles(S::T, S::D, B);
  for (int i = lane; i < S::T; i += 32) { red_add(r + i, macc[i]); macc[i] = 0.0; }
}
// camera rows of W_f: pose rows = sum_a Ac^T wacc[xi_a rows] (the camera's own map does not depend on the view: applied once per
// camera and frame), intrinsics rows = wacc[kappa rows]
template <int MODEL, bool ROLL>
__device__ __forceinline__ void lin_flush_wacc(const DeviceProblem& p, const LinArgs& a, double* w, int f, int lane, unsigned* seen) {
  using S = LinShape<MODEL, ROLL>; using L = LinLayout<MODEL, ROLL>;
  constexpr int FB = S::FB, KO = S::KO, NIN = S::NIN;
  const int B = p.B;
  double* tl = w + L::tail(B);
  const int cam = (int)tl[1];
  if (cam < 0 || !p.frame_blocks || tl[3] == 0.0) return;
  __syncwarp();
  if (lane == 0) tl[3] = 0.0;
  double* wacc = w + L::wacc(B);
  double* Wf = a.W + (size_t)f * p.n_s * FB;
  if (p.off_cp >= 0) {
    const PoseT& pc = p.cam_T[cam];
    const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int o = lane; o < 6 * FB; o += 32) {
      const int i = o / FB, col = o % FB;
      double s = 0.0;
#pragma unroll
      for (int kk = 0; kk < KO; kk++) s += twist_entry(pc.JL, I3, pc.t, kk % 6, i) * wacc[kk * FB + col];
      Wf[(size_t)(p.off_cp + 6 * cam + i) * FB + col] = s;
    }
  }
  if (p.off_in >= 0) {
    for (int o = lane; o < NIN * FB; o += 32) {
      const int i = o / FB, col = o % FB;
      const double val = wacc[(KO + i) * FB + col];
      if (p.fix_aspect && i == 1) { Wf[(size_t)(p.off_in + p.kint * cam + 1) * FB + col] = 0.0; continue; }      // fy follows fx (camera.py:159-160): folded onto fx, its own row is dead
      const int q = intr_param_index(p, i);
      if (q < 0) { Wf[(size_t)(p.off_in + p.kint * cam + (i < 4 ? i : i + 1)) * FB + col] = 0.0; continue; }      // held fixed: dead row
      const double v2 = (p.fix_aspect && i == 0) ? val + wacc[(KO + 1) * FB + col] : val;
      Wf[(size_t)(p.off_in + p.kint * cam + q) * FB + col] = v2;
    }
    for (int col = lane; col < FB; col += 32) Wf[(size_t)(p.off_in + p.kint * cam + 4) * FB + col] = 0.0;             // skew: ignored by cv2.projectPoints, dead column
  }
  if (lane == 0) atomicOr(&seen[cam >> 5], 1u << (cam & 31));
  __syncwarp();
  for (int o = lane; o < L::NWC; o += 32) wacc[o] = 0.0;
}

// entry (r, c) of the 3x3 product A B
__device__ __forceinline__ double mat3_entry(const double* A, const double* B, int r, int c) {
  return A[3 * r] * B[c] + A[3 * r + 1] * B[3 + c] + A[3 * r + 2] * B[6 + c];
}
// The 27 structurally non-zero entries of a 6x6 twist map (geometry.cuh twist_map) with R_left = Rl, left Jacobian JL and chain translation
// t, one per lane: e < 9 -> (rotation rows, rotation columns) = Rl JL, e < 18 -> (translation rows, translation columns) = Rl,
// else (translation rows, rotation columns) = t x (Rl JL).  Returns the value, row kk and column col.
__device__ __forceinline__ double twist_nonzero(const double* Rl, const double* JL, const double* t, int e, int& kk, int& col) {
  if (e < 9) { kk = e / 3; col = e % 3; return mat3_entry(Rl, JL, kk, col); }
  if (e < 18) { const int q = e - 9; kk = 3 + q / 3; col = 3 + q % 3; return Rl[q]; }
  const int q = e - 18, r = q / 3;
  col = q % 3; kk = 3 + r;
  const double a0 = mat3_entry(Rl, JL, 0, col), a1 = mat3_entry(Rl, JL, 1, col), a2 = mat3_entry(Rl, JL, 2, col);
  return r == 0 ? t[1] * a2 - t[2] * a1 : r == 1 ? t[2] * a0 - t[0] * a2 : t[0] * a1 - t[1] * a0;
}

// The noinline helpers below take the problem description by POINTER to the CTA's copy in shared memory: a reference to the kernel's own
// parameter would force the compiler to keep a local-memory copy of it and to reach every table of the kernel through that copy.
// what: 1 = board coupling of the current (camera, board), 2 = the camera's rows of W_f, 4 = the camera's raw moment sum
template <int MODEL, bool ROLL>
__device__ __noinline__ void lin_flush(const DeviceProblem* p, const LinArgs* a, double* w, double* myrec, unsigned* seen, int f, int what) {
  const int lane = threadIdx.x & 31;
  if (what & 1) lin_flush_ub<MODEL, ROLL>(*p, w, myrec, lane);
  if (what & 2) lin_flush_wacc<MODEL, ROLL>(*p, *a, w, f, lane, seen);
  if (what & 4) lin_flush_macc<MODEL, ROLL>(*p, w, myrec, lane);
  __syncwarp();
}

// Epilogue of one view (camera c, frame f, board b), leader warp.  In: rows xi of the view's moment matrix in Ms (column D = G^T r), the
// chain R_cf, t_cf of (camera, frame) in the warp's slice.  With E = [Af_0 .. | Ab] the 6 x 6 twist maps of the view stacked by columns
// (rows = twist components):
//     T^t = E^T M[xi, :]      rows f: Tf^t (-> W_f camera / intrinsics rows, g_f)      rows b: Tb^t (-> camera x board blocks, board gradient)
//     P   = T^t[:, xi] E      (f,f) -> H_ff      (b,f) -> W_f board rows      (b,b) -> board x board block
// both products on the fp64 tensor path (m16n8k8, 2 + 2 instructions for static frames; rolling frames' 12 twist components add an
// m16n8k4 per C block); every lane adds its C fragments
// to the warp's running sums at offsets it reads from the CTA's scatter tables (no index arithmetic, no branches on the element's role).
// A call, not inlined: the chunk loop of the kernel keeps its registers.
template <int MODEL, bool ROLL>
__device__ __noinline__ void lin_view_epilogue(int B, bool frames_on, bool boards_on, const PoseT* pcam, double* w, const PoseT* ftab, const PoseT* btab,
                                               const short (*tabT)[32], const short (*tabP)[32], int b, double cost_acc, bool new_chain) {
  using S = LinShape<MODEL, ROLL>; using L = LinLayout<MODEL, ROLL>;
  constexpr int NP = S::NP, T = S::T, NT = S::NT, FB = S::FB;
  constexpr int PT = L::PT, PM = L::PM, KS = L::KS, EP = L::EP, MSTR = L::MSTR, EK = L::EK;
  const int lane = threadIdx.x & 31, grp = lane >> 2, tig = lane & 3;
  double* Ms = w + L::Ms; double* Tt = w + L::Tt;
  double* Em = w + L::E; const double* chain = w + L::chain;
  double* tl = w + L::tail(B);
  if (lane == 0) { (w + L::macc(B))[T - 1] += cost_acc; tl[0] += cost_acc; tl[3] = 1.0; }
  if (!(frames_on || boards_on)) { __syncwarp(); return; }
  // ---- twist maps: the frame block(s) of E change with (camera, frame), the board block with the view.  Entries that are structurally
  // zero (and the blocks of parameter groups that are switched off) were zeroed when the kernel started and are never written.
  const PoseT& pc = *pcam;
  if (frames_on && new_chain)
    for (int o = lane; o < 27 * NP; o += 32) {
      const int j = o / 27; int kk, col;
      const double val = twist_nonzero(pc.R, ftab[j].JL, chain + 12 * j + 9, o % 27, kk, col);
      Em[(6 * j + kk) * EP + 6 * j + col] = val;            // block j of the twist components only reaches frame pose j
    }
  if (boards_on) {
    const PoseT& pb = btab[b];
    for (int o = lane; o < 27 * NP; o += 32) {
      const int j = o / 27; int kk, col;
      const double* Rc = chain + 12 * j;
      double t[3];
      mat3_vec(Rc, pb.t, t);
      t[0] += Rc[9]; t[1] += Rc[10]; t[2] += Rc[11];
      const double val = twist_nonzero(Rc, pb.JL, t, o % 27, kk, col);
      Em[(6 * j + kk) * EP + 6 * NP + col] = val;
    }
  }
  __syncwarp();
  // ---- T^t = E^T M[xi, :]
#pragma unroll
  for (int I = 0; I < PM; I++) {
    double fa[KS][2];
#pragma unroll
    for (int ks = 0; ks < KS; ks++)
#pragma unroll
      for (int h = 0; h < 2; h++) fa[ks][h] = 16 * I + 8 * h < 8 * PT ? Em[(4 * ks + tig) * EP + 16 * I + 8 * h + grp] : 0.0;
#pragma unroll
    for (int J = 0; J < NT; J++) {
      double fb[KS], c[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int ks = 0; ks < KS; ks++) fb[ks] = Ms[(4 * ks + tig) * MSTR + 8 * J + grp];
      dmma_quads<KS>(c, fa, fb);
#pragma unroll
      for (int h = 0; h < 2; h++)
        if (16 * I + 8 * h < 8 * PT && 8 * J < EK && 8 * J + 2 * tig < EK)
          *reinterpret_cast<double2*>(Tt + (16 * I + 8 * h + grp) * LIN_TSTR + 8 * J + 2 * tig) = make_double2(c[2 * h], c[2 * h + 1]);
#pragma unroll
      for (int i = 0; i < 4; i++) { const int o = tabT[(I * NT + J) * 4 + i][lane]; if (o >= 0) w[o] += c[i]; }
    }
  }
  __syncwarp();
  // ---- P = T^t[:, xi] E
  const int wb = b * 6 * FB;
#pragma unroll
  for (int I = 0; I < PM; I++) {
    double fa[KS][2];
#pragma unroll
    for (int ks = 0; ks < KS; ks++)
#pragma unroll
      for (int h = 0; h < 2; h++) fa[ks][h] = 16 * I + 8 * h < 8 * PT ? Tt[(16 * I + 8 * h + grp) * LIN_TSTR + 4 * ks + tig] : 0.0;
#pragma unroll
    for (int J = 0; J < PT; J++) {
      double fb[KS], c[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int ks = 0; ks < KS; ks++) fb[ks] = Em[(4 * ks + tig) * EP + 8 * J + grp];
      dmma_quads<KS>(c, fa, fb);
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int o = tabP[(I * PT + J) * 4 + i][lane];
        if (o >= 0) w[(o & (LIN_WB_FLAG - 1)) + ((o & LIN_WB_FLAG) ? wb : 0)] += c[i];
      }
    }
  }
  __syncwarp();
}


template <int MODEL, bool ROLL>
__global__ void __launch_bounds__(LIN_THREADS, 2)
k_linearize(DeviceProblem p, LinArgs a) {
  using S = LinShape<MODEL, ROLL>; using L = LinLayout<MODEL, ROLL>;
  constexpr int NIN = S::NIN, D = S::D, T = S::T, NC = S::NC, NT = S::NT, NBLK = S::NBLK, KINT = S::KINT, FB = S::FB, NP = S::NP;
  extern __shared__ double lsm[];
  __shared__ int fv_cam[LIN_MAXV], fv_board[LIN_MAXV], fv_start[LIN_MAXV + 1];
  __shared__ int any_view;
  __shared__ DeviceProblem ps;                       // copies for the noinline helpers (lin_flush)
  __shared__ LinArgs as_;
  __shared__ unsigned cam_seen[LIN_MAXC / 32];       // cameras with a view in the frame in progress (their W_f rows are written by the owning warp)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nthreads = blockDim.x, nwarps = nthreads >> 5;
  const int grp = lane >> 2, tig = lane & 3;
  const int B = p.B, n_s = p.n_s;
  const int split = a.split, slots = nwarps / split, slot = warp / split, sub = warp % split;
  const bool leader = sub == 0;
  const bool frames_on = p.frame_blocks != 0;
  const size_t wd = lin_warp_doubles(NC, T, D, FB, NIN, B, NP);
  double* w = lsm + (size_t)warp * wd;          // this warp's slice; w[0 .. NC*LIN_KPAD) is the stage buffer of the chunk loop
  // pose tables staged in shared memory by bulk asynchronous copies: the frame's [NP] (double buffered: the next frame's is in flight
  // while this one is worked on), then the boards' (they do not change during the launch)
  __shared__ __align__(8) unsigned long long tbar[3];
  PoseT* ftab2 = reinterpret_cast<PoseT*>(lsm + (size_t)nwarps * wd);       // [2][NP]
  const bool boards_staged = B <= LIN_MAXB;
  const PoseT* btab = boards_staged ? ftab2 + 2 * NP : p.board_T;
  if (tid == 0) { mbar_init(&tbar[0], 1); mbar_init(&tbar[1], 1); mbar_init(&tbar[2], 1); fence_barrier_init(); ps = p; as_ = a; }
  static_assert(12 * NP + KINT <= LIN_VC, "view constants");
  // scatter tables: for every C-fragment slot of the epilogue's two products and of the moment tiles, the offset (from the warp's
  // slice) of the running sum the lane's element belongs to, or -1
  __shared__ short tabT[L::NTT][32], tabP[L::NTP][32], tabM[L::NTM][32];
  {
    constexpr int PC = L::PC, PT = L::PT, E_ = S::E;
    const bool boards_on = p.off_bp >= 0;
    // C fragment slot i of a 16 x 8 block: row grp + 8 (i >> 1), column 2 tig + (i & 1)
    for (int o = tid; o < L::NTT * 32; o += nthreads) {
      const int e = o >> 5, l = o & 31, I = (e >> 2) / NT, J = (e >> 2) % NT, i = e & 3;
      const int pp = 16 * I + (l >> 2) + 8 * (i >> 1), j = 8 * J + 2 * (l & 3) + (i & 1);
      int off = -1;
      if (pp < 6 * NP) { if (frames_on) { if (j < D) off = L::wacc(B) + j * FB + pp; else if (j == D) off = L::hacc(B) + FB * FB + pp; } }
      else if (pp < PC && boards_on) { const int r = pp - 6 * NP; if (j < D) off = L::ub(B) + j * 6 + r; else if (j == D) off = L::ub(B) + D * 6 + 36 + r; }
      tabT[e][l] = (short)off;
    }
    for (int o = tid; o < L::NTP * 32; o += nthreads) {
      const int e = o >> 5, l = o & 31, I = (e >> 2) / PT, J = (e >> 2) % PT, i = e & 3;
      const int pp = 16 * I + (l >> 2) + 8 * (i >> 1), q = 8 * J + 2 * (l & 3) + (i & 1);
      int off = -1;
      if (pp < FB) { if (frames_on && q < FB) off = L::hacc(B) + pp * FB + q; }
      else if (pp < PC && boards_on) {
        const int r = pp - FB;
        if (q < FB) { if (frames_on) off = (L::Wb + r * FB + q) | LIN_WB_FLAG; }
        else if (q < PC) off = L::ub(B) + D * 6 + r * 6 + (q - FB);
      }
      tabP[e][l] = (short)off;
    }
    for (int o = tid; o < L::NTM * 32; o += nthreads) {
      const int e = o >> 5, l = o & 31, s = e & 3;
      int t = e >> 2, mb = 0;
      while (t >= NT - 2 * mb) { t -= NT - 2 * mb; mb++; }
      const int J = 2 * mb + t, i = 16 * mb + (l >> 2) + 8 * (s >> 1), j = 8 * J + 2 * (l & 3) + (s & 1);      // i > j below the diagonal
      int off = -1;
      if (i < D && j < D && i <= j) off = L::macc(B) + tri_index(D, i, j);
      else if (i < D && j == D) off = L::macc(B) + E_ + i;
      tabM[e][l] = (short)off;
    }
  }
  const int rec = lin_record_doubles(T, D, B);
  double* myrec = a.spart + (size_t)blockIdx.x * p.C * rec;

  // this CTA's records start at zero; the leader warps' running sums too
  for (int i = tid; i < p.C * rec; i += nthreads) myrec[i] = 0.0;
  if (leader) for (int i = L::E + lane; i < L::tail(B); i += 32) w[i] = 0.0;       // E | chain | Wb | hacc | wacc | macc | ub
  if (lane == 0) { double* tl = w + L::tail(B); tl[0] = 0.0; tl[1] = -1.0; tl[2] = -1.0; tl[3] = 0.0; tl[4] = -1.0; tl[5] = -1.0; }
  __syncthreads();
  if (tid == 0) {
    if (boards_staged) { mbar_expect_tx(&tbar[2], (unsigned)(sizeof(PoseT) * B)); bulk_g2s(ftab2 + 2 * NP, p.board_T, (unsigned)(sizeof(PoseT) * B), &tbar[2]); }
    if ((int)blockIdx.x < p.F) { mbar_expect_tx(&tbar[0], (unsigned)(sizeof(PoseT) * NP)); bulk_g2s(ftab2, p.frame_T + (size_t)blockIdx.x * NP, (unsigned)(sizeof(PoseT) * NP), &tbar[0]); }
  }
  if (boards_staged) mbar_wait(&tbar[2], 0);

  int it = 0;
  for (int f = blockIdx.x; f < p.F; f += gridDim.x, it++) {
    const PoseT* ftab = ftab2 + (it & 1) * NP;
    if (tid == 0 && f + (int)gridDim.x < p.F) {       // the next frame's table -> the other buffer (every warp left it at the end of the previous frame)
      unsigned long long* nb = &tbar[(it + 1) & 1];
      mbar_expect_tx(nb, (unsigned)(sizeof(PoseT) * NP));
      bulk_g2s(ftab2 + ((it + 1) & 1) * NP, p.frame_T + (size_t)(f + gridDim.x) * NP, (unsigned)(sizeof(PoseT) * NP), nb);
    }
    const int v0 = p.frame_view_start[f], v1 = p.frame_view_start[f + 1];
    const bool staged = v1 - v0 <= LIN_MAXV;
    if (staged) {
      for (int i = tid; i <= v1 - v0; i += nthreads) {
        fv_start[i] = p.view_start[v0 + i];
        if (i < v1 - v0) { fv_cam[i] = p.view_cam[v0 + i]; fv_board[i] = p.view_board[v0 + i]; }
      }
    }
    // W_f is written once: camera rows by the warp that owns the camera, board rows at the end of the frame, zeros only where nobody writes
    // (cameras without a view in this frame; board points as parameters: k_point_blocks adds to zeroed rows afterwards)
    const bool fill_all = frames_on && (p.C > LIN_MAXC || p.off_pt >= 0);
    if (fill_all) {
      double* Wf = a.W + (size_t)f * n_s * FB;
      for (int i = tid; i < n_s * FB; i += nthreads) Wf[i] = 0.0;
    }
    for (int i = tid; i < LIN_MAXC / 32; i += nthreads) cam_seen[i] = 0u;
    mbar_wait(&tbar[it & 1], (unsigned)((it >> 1) & 1));       // this frame's pose table(s) have landed
    if (leader) {
      for (int i = L::Wb + lane; i < L::wacc(B); i += 32) w[i] = 0.0;      // Wb | hacc
      if (lane == 0) (w + L::tail(B))[0] = 0.0;
    }
    __syncthreads();

    // next view (at or after `from`) of this warp's cameras (c == slot mod slots; slots is a power of two): 32 views per look
    auto next_view = [&](int from) {
      while (from < v1) {
        const int q = from + lane;
        const int cq = q < v1 ? (staged ? fv_cam[q - v0] : p.view_cam[q]) : -1;
        const unsigned m = __ballot_sync(0xffffffffu, q < v1 && (cq & (slots - 1)) == slot);
        if (m) return from + __ffs(m) - 1;
        from += 32;
      }
      return v1;
    };
    // first chunk of a view: observation and point id of this lane's corner.  Requested one view ahead (before the previous view's
    // epilogue), so that the DRAM round trip of a view's first corners is not on the warp's critical path
    double2 ob_n = make_double2(0.0, 0.0); int pi_n = 0;
    auto prefetch_view = [&](int vv) {
      if (vv >= v1) return;
      const int beg = staged ? fv_start[vv - v0] : p.view_start[vv], end = staged ? fv_start[vv - v0 + 1] : p.view_start[vv + 1];
      const int i0 = beg + 32 * sub + lane;
      if (i0 < end) { ob_n = p.obs[i0]; pi_n = p.pid[i0]; }
    };
    int v = next_view(v0);
    prefetch_view(v);
    while (true) {
      const bool have = v < v1;
      if (split == 1) { if (!have) break; }
      else {
        // the warps of a slot walk the same views; the CTA meets twice per round, so every warp runs the same number of rounds
        if (tid == 0) any_view = 0;
        __syncthreads();
        if (have && lane == 0 && leader) any_view = 1;
        __syncthreads();
        if (!any_view) break;
      }
      double acc[NBLK][4];
#pragma unroll
      for (int t = 0; t < NBLK; t++)
#pragma unroll
        for (int i = 0; i < 4; i++) acc[t][i] = 0.0;
      double cost_acc = 0.0;
      int c = 0, b = 0;
      bool new_chain = false;
      if (have) {
        c = staged ? fv_cam[v - v0] : p.view_cam[v]; b = staged ? fv_board[v - v0] : p.view_board[v];
        const int beg = staged ? fv_start[v - v0] : p.view_start[v], end = staged ? fv_start[v - v0 + 1] : p.view_start[v + 1];
        // R_cf, t_cf of (camera, frame): kept in the warp's slice while the warp stays with the pair (all boards of the frame)
        double* chain = w + L::chain; double* tl = w + L::tail(B);
        new_chain = (int)tl[4] != f || (int)tl[5] != c;
        if (new_chain) {
          const PoseT& pc = p.cam_T[c];
          __syncwarp();
          for (int o = lane; o < 12 * NP; o += 32) {
            const int j = o / 12, e = o % 12;
            const PoseT& pf = ftab[j];
            if (e < 9) chain[12 * j + e] = mat3_entry(pc.R, pf.R, e / 3, e % 3);
            else { const int r = e - 9; chain[12 * j + e] = pc.R[3 * r] * pf.t[0] + pc.R[3 * r + 1] * pf.t[1] + pc.R[3 * r + 2] * pf.t[2] + pc.t[r]; }
          }
          if (lane == 0) { tl[4] = f; tl[5] = c; }
          __syncwarp();
        }
        // the view's constants -- pose(s) T_c T_f T_b and the camera's intrinsics -- go to the warp's slice: the chunk loop reads them from
        // shared memory where it needs them instead of holding 22 doubles in registers (they would be spilled to local memory)
        double* vc = w + L::vc(B);
        {
          const PoseT& pb = btab[b];
          for (int o = lane; o < 12 * NP + KINT; o += 32) {
            if (o < 12 * NP) {
              const int j = o / 12, e = o % 12;
              const double* Rc = chain + 12 * j;
              if (e < 9) vc[o] = mat3_entry(Rc, pb.R, e / 3, e % 3);
              else { const int r = e - 9; vc[o] = Rc[3 * r] * pb.t[0] + Rc[3 * r + 1] * pb.t[1] + Rc[3 * r + 2] * pb.t[2] + Rc[9 + r]; }
            } else vc[o] = p.intr[c * KINT + o - 12 * NP];
          }
          __syncwarp();
        }
        const ViewPose& vp = *reinterpret_cast<const ViewPose*>(vc);
        const ViewPose& vpe = *reinterpret_cast<const ViewPose*>(vc + (ROLL ? 12 : 0));
        const double* k = vc + 12 * NP;
        const double inv_h = ROLL ? 1.0 / p.img_h[c] : 0.0;
        const double* bp = p.board_pts + (size_t)b * p.P * 3;
        // the next chunk's observation / point id are in flight while this chunk is computed (one L2 round trip less per chunk on the
        // dependent chain  point id -> board point -> projection)
        for (int base = beg + 32 * sub; base < end; base += 32 * split) {
          const double2 ob = ob_n; const int pi = pi_n;
          const int i1 = base + 32 * split + lane;
          if (i1 < end) { ob_n = p.obs[i1]; pi_n = p.pid[i1]; }
          view_chunk<MODEL, ROLL>(p, a.loss, a.f_scale, vp, vpe, k, bp, inv_h, base, end, lane, w, acc, cost_acc, ob, pi);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cost_acc += __shfl_xor_sync(0xffffffffu, cost_acc, o);
      }
      const int v_next = have ? next_view(v + 1) : v1;
      prefetch_view(v_next);
      if (split > 1) {        // meet: the slot's leader adds the other warps' fragments in warp order (same lane -> same matrix element)
        if (have && !leader) {
          double* xr = w;                      // this warp's stage buffer is free between two views
#pragma unroll
          for (int t = 0; t < NBLK; t++)
#pragma unroll
            for (int i = 0; i < 4; i++) xr[(4 * t + i) * 32 + lane] = acc[t][i];
          if (lane == 0) xr[4 * NBLK * 32] = cost_acc;
        }
        __syncthreads();
        if (have && leader) {
          for (int q = 1; q < split; q++) {
            const double* xr = lsm + (size_t)(warp + q) * wd;
#pragma unroll
            for (int t = 0; t < NBLK; t++)
#pragma unroll
              for (int i = 0; i < 4; i++) acc[t][i] += xr[(4 * t + i) * 32 + lane];
            cost_acc += xr[4 * NBLK * 32];
          }
        }
      }
      if (have && leader) {
        {   // the warp moves on to a view of camera c / board b: running sums of the previous camera / board go out first
          double* tl = w + L::tail(B);
          if (c != (int)tl[1]) {
            lin_flush<MODEL, ROLL>(&ps, &as_, w, myrec, cam_seen, f, 7);
            if (lane == 0) { tl[1] = c; tl[2] = b; }
            __syncwarp();
          } else if (b != (int)tl[2]) {
            lin_flush<MODEL, ROLL>(&ps, &as_, w, myrec, cam_seen, f, 1);
            if (lane == 0) tl[2] = b;
            __syncwarp();
          }
        }
        // the camera's raw moment sum (upper triangle | G^T r) straight from the fragments; rows xi of M -> Ms for the epilogue's products
        double* Ms = w + L::Ms;
        // (the 8 x 8 tile of a diagonal block below the diagonal, I > J, is the mirror of a tile above it: neither summed nor stored)
        int t = 0;
#pragma unroll
        for (int mb = 0; mb < S::NMB; mb++)
#pragma unroll
          for (int J = 2 * mb; J < NT; J++) {
#pragma unroll
            for (int s = 0; s < 4; s++) {
              const int o = tabM[4 * t + s][lane];
              if (o >= 0) w[o] += acc[t][s];
              const int I = 2 * mb + (s >> 1), i = 8 * I + grp, j = 8 * J + 2 * tig + (s & 1);
              if (I <= J && 8 * I < L::EK) Ms[i * L::MSTR + j] = acc[t][s];
              if (I < J && 8 * J < L::EK) Ms[j * L::MSTR + i] = acc[t][s];
            }
            t++;
          }
        __syncwarp();
        lin_view_epilogue<MODEL, ROLL>(B, frames_on, p.off_bp >= 0, p.cam_T + c, w, ftab, btab, tabT, tabP, b, cost_acc, new_chain);
      }
      v = v_next;
    }
    // ---- end of the frame: camera rows out, then the CTA sums the slots' partials in slot order
    if (leader) lin_flush<MODEL, ROLL>(&ps, &as_, w, myrec, cam_seen, f, 2);
    __syncthreads();
    if (frames_on && !fill_all) {
      double* Wf = a.W + (size_t)f * n_s * FB;
      for (int c = 0; c < p.C; c++) {
        if (cam_seen[c >> 5] & (1u << (c & 31))) continue;
        if (p.off_cp >= 0) for (int i = tid; i < 6 * FB; i += nthreads) Wf[(size_t)(p.off_cp + 6 * c) * FB + i] = 0.0;
        if (p.off_in >= 0) for (int i = tid; i < p.kint * FB; i += nthreads) Wf[(size_t)(p.off_in + p.kint * c) * FB + i] = 0.0;
      }
    }
    if (frames_on) {
      for (int o = tid; o < L::NHF; o += nthreads) {
        double s = 0.0;
        for (int q = 0; q < slots; q++) s += lsm[(size_t)(q * split) * wd + L::hacc(B) + o];
        if (o < FB * FB) a.Hff[(size_t)f * FB * FB + o] = s; else a.g[n_s + FB * f + o - FB * FB] = s;
      }
      if (p.off_bp >= 0) {
        double* Wf = a.W + (size_t)f * n_s * FB;
        for (int o = tid; o < B * 6 * FB; o += nthreads) {
          double s = 0.0;
          for (int q = 0; q < slots; q++) s += lsm[(size_t)(q * split) * wd + L::Wb + o];
          const int bb = o / (6 * FB), i = (o % (6 * FB)) / FB, j = o % FB;
          Wf[(size_t)(p.off_bp + 6 * bb + i) * FB + j] = s;
        }
      }
    }
    if (tid == 0) {
      double s = 0.0;
      for (int q = 0; q < slots; q++) s += lsm[(size_t)(q * split) * wd + L::tail(B)];
      a.frame_cost[f] = s;
    }
    __syncthreads();
  }
  if (leader) lin_flush<MODEL, ROLL>(&ps, &as_, w, myrec, cam_seen, 0, 5);
}

// ------------------------------------------------------------------------------------------------
// k_reduce_shared: the per-CTA records of k_linearize -> H_ss, g_s, cost.  No atomics on data: two runs give bit-identical results.
//   step 1  grid = cameras x slices of 32 record entries; 256 threads = 32 entries x 8 groups: group g adds records g, g+8, ... in
//           order, the 8 group sums are added in order -> the camera's summed record (global scratch `sred`)
//   step 2  the LAST slice CTA of a camera (arrival counter) applies the camera's own twist map (it does not depend on the view) and
//           STORES the camera's blocks of H_ss / g_s: (pose | intrinsics) x (pose | intrinsics), and x every board pose
//   step 3  board x board blocks and board gradients are sums over the cameras: the last camera to finish step 2 adds the per-camera
//           partials in camera order, and the per-frame costs in frame order
constexpr int RED_THREADS = 256;
constexpr int RED_ENT = 32, RED_GROUPS = RED_THREADS / RED_ENT;
struct ReduceArgs {
  const double* spart; int nparts;            // [nparts][C][rec]
  double* sred;                               // [C][rec]
  double* Hss; double* g;
  double* bpart;                              // [C][B][42]
  const double* frame_cost; int F; double* cost_out;
  unsigned* cam_counter;                      // [C + 1]: slices done per camera | cameras done
};
__host__ __device__ inline int reduce_slices(int rec) { return (rec + RED_ENT - 1) / RED_ENT; }
// the camera's moment sum | Um | Ac: the per-board parts of the record are read from `sred` where they are used, so that the CTA's
// shared memory does not grow with the board count
__host__ __device__ inline size_t reduce_smem_doubles(int T, int D) { return (size_t)T + D * 6 + 36; }

template <int NP>
__global__ void __launch_bounds__(RED_THREADS)
k_reduce_shared(DeviceProblem p, ReduceArgs a) {
  constexpr int KO = 6 * NP;
  extern __shared__ double rsm[];
  __shared__ double sm[32];
  __shared__ double gsum[RED_GROUPS][RED_ENT];
  __shared__ int is_last;
  const int D = p.D, T = p.T, B = p.B, n_s = p.n_s;
  const int E = D * (D + 1) / 2;
  const int UB = D * 6 + 42;
  const int rec = lin_record_doubles(T, D, B);
  const int nsl = reduce_slices(rec);
  const int c = blockIdx.x / nsl, slice = blockIdx.x % nsl, tid = threadIdx.x;
  // ---- step 1
  {
    const int e = slice * RED_ENT + (tid % RED_ENT), grp = tid / RED_ENT;
    double s = 0.0;
    if (e < rec) {
      const double* src = a.spart + (size_t)c * rec + e;
      const size_t stride = (size_t)p.C * rec;
      int q = grp;
      for (; q + 3 * RED_GROUPS < a.nparts; q += 4 * RED_GROUPS) {       // four loads in flight, added in record order
        const double v0 = src[(size_t)q * stride], v1 = src[(size_t)(q + RED_GROUPS) * stride];
        const double v2 = src[(size_t)(q + 2 * RED_GROUPS) * stride], v3 = src[(size_t)(q + 3 * RED_GROUPS) * stride];
        s = (((s + v0) + v1) + v2) + v3;
      }
      for (; q < a.nparts; q += RED_GROUPS) s += src[(size_t)q * stride];
    }
    gsum[grp][tid % RED_ENT] = s;
    __syncthreads();
    if (tid < RED_ENT && slice * RED_ENT + tid < rec) {
      double t = 0.0;
#pragma unroll
      for (int gq = 0; gq < RED_GROUPS; gq++) t += gsum[gq][tid];
      a.sred[(size_t)c * rec + slice * RED_ENT + tid] = t;
    }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) { const unsigned t = atomicAdd(a.cam_counter + c, 1u); is_last = (t == (unsigned)nsl - 1); }
  __syncthreads();
  if (!is_last) return;
  if (tid == 0) a.cam_counter[c] = 0;
  __threadfence();
  // ---- step 2: this camera's blocks
  double* Msum = rsm;                         // [T]
  double* Um = rsm + T;                       // [D][6]
  double* Ac = Um + D * 6;                    // 36
  for (int i = tid; i < T; i += RED_THREADS) Msum[i] = __ldcg(&a.sred[(size_t)c * rec + i]);
  if (tid == 0) { const PoseT& pc = p.cam_T[c]; const double I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; twist_map(I3, pc.JL, pc.t, Ac); }
  __syncthreads();
  for (int o = tid; o < D * 6; o += RED_THREADS) {       // Um = sum_a Msum[:, xi_a] Ac  (the camera's map is the same for every chain)
    const int i = o / 6, j = o % 6; double acc = 0.0;
    for (int kk = 0; kk < KO; kk++) acc += msym(Msum, D, i, kk) * Ac[(kk % 6) * 6 + j];
    Um[o] = acc;
  }
  __syncthreads();
  const int nin = 4 + p.nd;
  const int cp = p.off_cp >= 0 ? p.off_cp + 6 * c : -1;
  const int in0 = p.off_in >= 0 ? p.off_in + p.kint * c : -1;
  auto put = [&](int i, int j, double val) { a.Hss[(size_t)i * n_s + j] = val; a.Hss[(size_t)j * n_s + i] = val; };
  if (cp >= 0) {
    for (int o = tid; o < 36; o += RED_THREADS) {
      const int i = o / 6, j = o % 6;
      if (j < i) continue;
      double acc = 0.0;
      for (int kk = 0; kk < KO; kk++) acc += Ac[(kk % 6) * 6 + i] * Um[kk * 6 + j];
      put(cp + i, cp + j, acc);
    }
    if (tid < 6) {
      double acc = 0.0;
      for (int kk = 0; kk < KO; kk++) acc += Ac[(kk % 6) * 6 + tid] * Msum[E + kk];
      a.g[cp + tid] = acc;
    }
  }
  if (in0 >= 0) {
    // one thread per TARGET parameter pair: rows folded onto one parameter (fix_aspect: fy onto fx, camera.py:159-160) are added in a fixed order;
    // a parameter held fixed maps to -1, which no target matches: its row, column and gradient entry are written as zero
    const int kint = p.kint;
    if (cp >= 0)
      for (int o = tid; o < kint * 6; o += RED_THREADS) {
        const int pi = o / 6, j = o % 6;
        double acc = 0.0;
        for (int i = 0; i < nin; i++) if (intr_param_index(p, i) == pi) acc += Um[(KO + i) * 6 + j];
        put(in0 + pi, cp + j, acc);
      }
    for (int o = tid; o < kint * kint; o += RED_THREADS) {
      const int pi = o / kint, pj = o % kint;
      double acc = 0.0;
      for (int i = 0; i < nin; i++) if (intr_param_index(p, i) == pi)
        for (int j = 0; j < nin; j++) if (intr_param_index(p, j) == pj) acc += msym(Msum, D, KO + i, KO + j);
      a.Hss[(size_t)(in0 + pi) * n_s + in0 + pj] = acc;
    }
    for (int pi = tid; pi < kint; pi += RED_THREADS) {
      double acc = 0.0;
      for (int i = 0; i < nin; i++) if (intr_param_index(p, i) == pi) acc += Msum[E + KO + i];
      a.g[in0 + pi] = acc;
    }
  }
  if (p.off_bp >= 0) {
    for (int b = 0; b < B; b++) {
      const int bp = p.off_bp + 6 * b;
      const double* U = a.sred + (size_t)c * rec + T + (size_t)b * UB;      // [D][6] | Hbb 36 | gb 6 (summed by step 1 of this launch)
      if (cp >= 0)
        for (int o = tid; o < 36; o += RED_THREADS) {     // camera pose x board pose = sum_a Ac^T U_xi_a
          const int i = o / 6, j = o % 6; double acc = 0.0;
          for (int kk = 0; kk < KO; kk++) acc += Ac[(kk % 6) * 6 + i] * __ldcg(&U[kk * 6 + j]);
          put(cp + i, bp + j, acc);
        }
      if (in0 >= 0)
        for (int o = tid; o < p.kint * 6; o += RED_THREADS) { // intrinsics x board pose = U_kappa
          const int pi = o / 6, j = o % 6;
          double acc = 0.0;
          for (int i = 0; i < nin; i++) if (intr_param_index(p, i) == pi) acc += __ldcg(&U[(KO + i) * 6 + j]);
          put(in0 + pi, bp + j, acc);
        }
      for (int o = tid; o < 42; o += RED_THREADS) a.bpart[((size_t)c * B + b) * 42 + o] = __ldcg(&U[D * 6 + o]);
    }
  }
  // ---- step 3 (last camera): board x board blocks, board gradients (camera order) and the cost (frame order)
  __threadfence();
  __syncthreads();
  if (tid == 0) { const unsigned t = atomicAdd(a.cam_counter + p.C, 1u); is_last = (t == (unsigned)p.C - 1); }
  __syncthreads();
  if (!is_last) return;
  if (tid == 0) a.cam_counter[p.C] = 0;
  __threadfence();
  if (p.off_bp >= 0)
    for (int o = tid; o < B * 42; o += RED_THREADS) {
      const int b = o / 42, q = o % 42;
      double acc = 0.0;
      for (int cc = 0; cc < p.C; cc++) acc += __ldcg(&a.bpart[((size_t)cc * B + b) * 42 + q]);
      const int bp = p.off_bp + 6 * b;
      if (q < 36) a.Hss[(size_t)(bp + q / 6) * n_s + bp + q % 6] = acc; else a.g[bp + q - 36] = acc;
    }
  double cs = 0.0;
  for (int f = tid; f < a.F; f += RED_THREADS) cs += a.frame_cost[f];
  cs = block_sum(cs, sm);
  if (tid == 0) *a.cost_out = cs;
}

// ------------------------------------------------------------------------------------------------
// k_fold_hand_eye: hand-eye frames with free hand-eye parameters he = [W | G].  Every residual of frame f reaches he through the frame's
// twist, J_he = J_f M_f (hand_eye_frame_map), so with the frame blocks k_linearize emitted (frame_blocks) and k_point_blocks completed
//     H_he,he = sum_f M_f^T H_ff M_f      H_s,he = sum_f W_f[s, :] M_f   (every shared row s outside he)      g_he = sum_f M_f^T g_f
// One CTA per row s of H_s,he (he rows: the upper triangle of H_he,he; row n_s: g_he); thread (slice, j) sums column j over the frames
// f == slice mod FOLD_SLICES in frame order, and the slices' partials are added in slice order: fixed order, no atomics.  The CTA builds
// the maps of FOLD_FRAMES frames at a time in shared memory.  The he block, both triangles of every coupling and g_he are stored (nothing
// else writes them); the he rows of W_f are never written or read.
constexpr int FOLD_SLICES = 16;
constexpr int FOLD_THREADS = FOLD_SLICES * 16;
constexpr int FOLD_FRAMES = 64;
__global__ void __launch_bounds__(FOLD_THREADS)
k_fold_hand_eye(DeviceProblem p, const double* Hff, const double* W, double* Hss, double* g) {
  __shared__ double Mf[FOLD_FRAMES][72];
  __shared__ double part[FOLD_SLICES][16];
  const int n_s = p.n_s, he = p.off_he;
  const int r = blockIdx.x, j = threadIdx.x % 16, slice = threadIdx.x / 16;
  const int q = r - he;
  const bool hrow = q >= 0 && q < 12;
  const bool live = j < 12 && !(hrow && j < q);
  double acc = 0.0;
  for (int f0 = 0; f0 < p.F; f0 += FOLD_FRAMES) {
    const int nf = min(FOLD_FRAMES, p.F - f0);
    __syncthreads();
    if ((int)threadIdx.x < nf) {
      const PoseT& pw = p.he_T[0]; const PoseT& pg = p.he_T[1];
      const int f = f0 + threadIdx.x;
      hand_eye_frame_map(pg.R, p.arm_T[f].R, pw.JL, pg.JL, pg.t, p.frame_T[f].t, Mf[threadIdx.x]);
    }
    __syncthreads();
    if (!live) continue;
    for (int i = slice; i < nf; i += FOLD_SLICES) {
      const double* M = Mf[i];
      const int f = f0 + i;
      if (r == n_s) {
        const double* gf = g + n_s + 6 * f;
        for (int k = 0; k < 6; k++) acc += M[12 * k + j] * gf[k];
      } else if (hrow) {
        const double* H = Hff + 36 * f;
        for (int k = 0; k < 6; k++) {
          double t = 0.0;
          for (int l = 0; l < 6; l++) t += M[12 * l + q] * H[6 * l + k];
          acc += t * M[12 * k + j];
        }
      } else {
        const double* w = W + ((size_t)f * n_s + r) * 6;
        for (int k = 0; k < 6; k++) acc += w[k] * M[12 * k + j];
      }
    }
  }
  part[slice][j] = acc;
  __syncthreads();
  if (slice != 0 || !live) return;
  for (int s = 1; s < FOLD_SLICES; s++) acc += part[s][j];
  if (r == n_s) g[he + j] = acc;
  else {
    Hss[(size_t)r * n_s + he + j] = acc;
    Hss[(size_t)(he + j) * n_s + r] = acc;
  }
}

}  // namespace mcba
