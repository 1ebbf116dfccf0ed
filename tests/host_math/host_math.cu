// TEST INFRASTRUCTURE ONLY: host-callable wrappers around the __host__ __device__ math of csrc/geometry.cuh and
// csrc/solver_kernels.cuh so that CPU tests can check the exact source the kernels run (projection + analytic Jacobians
// against cv2, Rodrigues / twist maps against finite differences, the 2-D trust-region solve against scipy).
// Not part of libmcba.so and never loaded by multical_b200.
#include "solver_kernels.cuh"
#include "pnp_kernels.cuh"
#include "linearize.cuh"

using namespace mcba;

template <int MODEL>
static void project_all(int n, const double* X, const double* k, double* uv, double* J, double* Jk) {
  constexpr int ND = model_nd(MODEL);
  for (int i = 0; i < n; i++) {
    double u, v, Ju[3], Jv[3], ku[4 + ND], kv[4 + ND];
    for (int j = 0; j < 4 + ND; j++) { ku[j] = 0.0; kv[j] = 0.0; }
    project<MODEL, true>(X + 3 * i, k, u, v, Ju, Jv, ku, kv);
    uv[2 * i] = u; uv[2 * i + 1] = v;
    for (int j = 0; j < 3; j++) { J[(2 * i) * 3 + j] = Ju[j]; J[(2 * i + 1) * 3 + j] = Jv[j]; }
    for (int j = 0; j < 4 + ND; j++) { Jk[(2 * i) * (4 + ND) + j] = ku[j]; Jk[(2 * i + 1) * (4 + ND) + j] = kv[j]; }
    double u2, v2;
    project<MODEL, false>(X + 3 * i, k, u2, v2, nullptr, nullptr, nullptr, nullptr);
    if (u2 != u || v2 != v) { uv[2 * i] = NAN; }      // the residual-only and the Jacobian paths must agree bit for bit
  }
}

template <int MODEL>
static void undistort_all(int n, const double* uv, const double* k, double* out) {
  for (int i = 0; i < n; i++) undistort_pixel<MODEL>(k, uv[2 * i], uv[2 * i + 1], out[2 * i], out[2 * i + 1]);
}

template <int MODEL, bool ROLL>
static size_t lin_smem_of(int B, int warps) {
  using S = LinShape<MODEL, ROLL>;
  return lin_smem_doubles(S::NC, S::T, S::D, S::FB, S::NIN, B, S::NP, warps);
}

extern "C" {
int hm_undistort(int model, int n, const double* uv, const double* k, double* out) {
  switch (model) {
    case MODEL_STANDARD: undistort_all<MODEL_STANDARD>(n, uv, k, out); return 0;
    case MODEL_RATIONAL: undistort_all<MODEL_RATIONAL>(n, uv, k, out); return 0;
    case MODEL_THIN_PRISM: undistort_all<MODEL_THIN_PRISM>(n, uv, k, out); return 0;
    case MODEL_FISHEYE: undistort_all<MODEL_FISHEYE>(n, uv, k, out); return 0;
    case MODEL_TILTED: undistort_all<MODEL_TILTED>(n, uv, k, out); return 0;
  }
  return 1;
}
void hm_pose_from_homography(const double* H, double* R, double* t) { pose_from_homography(H, R, t); }
int hm_spd_solve8(double* A, double* b) { return spd_solve<8>(A, b) ? 1 : 0; }
int hm_project(int model, int n, const double* X, const double* k, double* uv, double* J, double* Jk) {
  switch (model) {
    case MODEL_STANDARD: project_all<MODEL_STANDARD>(n, X, k, uv, J, Jk); return 0;
    case MODEL_RATIONAL: project_all<MODEL_RATIONAL>(n, X, k, uv, J, Jk); return 0;
    case MODEL_THIN_PRISM: project_all<MODEL_THIN_PRISM>(n, X, k, uv, J, Jk); return 0;
    case MODEL_FISHEYE: project_all<MODEL_FISHEYE>(n, X, k, uv, J, Jk); return 0;
    case MODEL_TILTED: project_all<MODEL_TILTED>(n, X, k, uv, J, Jk); return 0;
  }
  return 1;
}
void hm_rodrigues(const double* r, double* R, double* JL) { rodrigues(r, R, JL); }
void hm_matrix_to_rtvec(const double* T, double* rt) { matrix_to_rtvec(T, rt); }
void hm_twist_map(const double* Rl, const double* JL, const double* t, double* A) { twist_map(Rl, JL, t, A); }
void hm_hand_eye_frame_map(const double* RG, const double* RA, const double* JLW, const double* JLG, const double* tG, const double* tf, double* M) {
  hand_eye_frame_map(RG, RA, JLW, JLG, tG, tf, M);
}
void hm_tr2d(double b11, double b12, double b22, double g1, double g2, double Delta, double* p) { solve_tr_2d(b11, b12, b22, g1, g2, Delta, p[0], p[1]); }
void hm_loss(int loss, double z, double* r) { loss_rho(loss, z, r[0], r[1], r[2]); }
// dynamic shared memory of a k_linearize CTA in doubles, as the host driver sizes the launch (lin_smem_for in csrc/solver.cu)
size_t hm_lin_smem_doubles(int model, int roll, int B, int warps) {
  switch (model) {
    case MODEL_STANDARD: return roll ? lin_smem_of<MODEL_STANDARD, true>(B, warps) : lin_smem_of<MODEL_STANDARD, false>(B, warps);
    case MODEL_RATIONAL: return roll ? lin_smem_of<MODEL_RATIONAL, true>(B, warps) : lin_smem_of<MODEL_RATIONAL, false>(B, warps);
    case MODEL_THIN_PRISM: return roll ? lin_smem_of<MODEL_THIN_PRISM, true>(B, warps) : lin_smem_of<MODEL_THIN_PRISM, false>(B, warps);
    case MODEL_FISHEYE: return roll ? lin_smem_of<MODEL_FISHEYE, true>(B, warps) : lin_smem_of<MODEL_FISHEYE, false>(B, warps);
    case MODEL_TILTED: return roll ? lin_smem_of<MODEL_TILTED, true>(B, warps) : lin_smem_of<MODEL_TILTED, false>(B, warps);
  }
  return 0;
}
}
