// hand_eye_init_kernels.cuh — the non-overlapping camera initialisation of HandEye.initialise_camera_poses (hand_eye/hand_eye.py) on
// the device.
//
// k_he_quads: one quadruple (master m, slave s, board bM, board bS) per CTA, one cv2.calibrateRobotWorldHandEye(SHAH) call of
// HandEye.master_slave_pair over the images i where both views are valid.  A_i = inv(P[m, i, bM]), B_i = inv(P[s, i, bS]) (rigid
// inverses), A X = Z B:
//   T = sum_i kron(R_B_i, R_A_i) (9x9);  v, u = top right / left singular vectors of T;  R_X ~ reshape_F(v), R_Z ~ reshape_F(u)
//   R <- orthonormal polar factor of sign(det R) R (= U V^T of normalizeRotation after its cube-root scale, whose det is then +1)
//   translations: least squares of -R_A_i t_X + t_Z = t_A_i - R_Z t_B_i, normal matrix [[n I, -S^T], [-S, n I]], S = sum_i R_A_i.
// v is the top eigenvector of T^T T (cyclic Jacobi, fp64, one thread), u = T v / |T v|.  A quadruple is dropped (ok = 0) with fewer
// than 3 images, where OpenCV raises "determinant(R) is null" (|det reshape_F(v or u)| < FLT_EPSILON), and where the top singular
// value is not separated, (s1 - s2) / s1 < HE_GAP_MIN: there the singular vector is arbitrary and OpenCV's answer is decided by its
// rounding (DESIGN.md §3f).
// k_he_vote: one warp per (master, slave) set of accepted translations: scipy.stats.gaussian_kde (Scott's factor n^(-1/7), unbiased
// covariance, Cholesky whitening) evaluated at every point, and the argmax (lowest index within HE_TIE_REL of the maximum).
// Every sum runs in a fixed order: two identical calls agree bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "pose_init_kernels.cuh"

namespace mcba {

constexpr int HE_THREADS = 128;
constexpr int HE_VOTE_WARPS = 4;
constexpr double HE_DET_MIN = 1.1920928955078125e-07;   // FLT_EPSILON, normalizeRotation's null-determinant test
constexpr double HE_GAP_MIN = 1e-6;                     // relative gap of the top two singular values of T
constexpr double HE_TIE_REL = 1e-12;

struct HandEyeArgs {
  int C, F, B;
  const double* poses; const uint8_t* valid;       // [C*F*B][4][4], [C*F*B]
  const int32_t* quads;                            // [n][4]: master, slave, boardM, boardS
  double* X; double* Z;                            // [n][4][4]
  int32_t* n_images; uint8_t* ok;                  // [n]
};

struct HandEyeVoteArgs {
  int n_sets;
  const int64_t* start;                            // [n_sets + 1]
  const double* points;                            // [N][3]
  double* density;                                 // [N]
  int32_t* best;                                   // [n_sets]: index within the set, -1 for a singular covariance
};

// cyclic Jacobi on the symmetric n x n row-major A (destroyed: eigenvalues on the diagonal); V <- eigenvectors in its columns
__device__ inline void he_jacobi(double* A, double* V, int n) {
  for (int i = 0; i < n * n; i++) V[i] = (i % (n + 1)) == 0 ? 1.0 : 0.0;
  double total = 0.0;
  for (int i = 0; i < n * n; i++) total += A[i] * A[i];
  for (int sweep = 0; sweep < 50; sweep++) {
    double off = 0.0;
    for (int p = 0; p < n; p++) for (int q = p + 1; q < n; q++) off += A[n * p + q] * A[n * p + q];
    if (!(off > 1e-34 * total)) break;
    for (int p = 0; p < n; p++) for (int q = p + 1; q < n; q++) {
      const double apq = A[n * p + q];
      if (apq == 0.0) continue;
      const double th = (A[n * q + q] - A[n * p + p]) / (2.0 * apq);
      const double t = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int k = 0; k < n; k++) {                // A <- A J (columns p, q)
        const double kp = A[n * k + p], kq = A[n * k + q];
        A[n * k + p] = c * kp - s * kq; A[n * k + q] = s * kp + c * kq;
      }
      for (int k = 0; k < n; k++) {                // A <- J^T A (rows p, q)
        const double pk = A[n * p + k], qk = A[n * q + k];
        A[n * p + k] = c * pk - s * qk; A[n * q + k] = s * pk + c * qk;
      }
      for (int k = 0; k < n; k++) {
        const double kp = V[n * k + p], kq = V[n * k + q];
        V[n * k + p] = c * kp - s * kq; V[n * k + q] = s * kp + c * kq;
      }
    }
  }
}

__device__ inline double he_det3(const double* M) {
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// orthonormal polar factor of sign(det M) M (Newton: R <- (R + R^-T) / 2), row-major 3x3 in place
__device__ inline void he_polar(double* R) {
  if (he_det3(R) < 0.0) for (int k = 0; k < 9; k++) R[k] = -R[k];
  for (int it = 0; it < 100; it++) {
    const double d = he_det3(R);
    double N[9], ch = 0.0;
    for (int i = 0; i < 3; i++) {
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;  // row i of the cofactor matrix = row i1 x row i2
      for (int j = 0; j < 3; j++) {
        const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        const double cof = R[3 * i1 + j1] * R[3 * i2 + j2] - R[3 * i1 + j2] * R[3 * i2 + j1];
        N[3 * i + j] = 0.5 * (R[3 * i + j] + cof / d);
      }
    }
    for (int k = 0; k < 9; k++) { ch = fmax(ch, fabs(N[k] - R[k])); R[k] = N[k]; }
    if (ch < 1e-15) break;
  }
}

// the common images of the quadruple in the tile [f0, f0 + NT): A_i, B_i (3x4) compacted into sA, sB in image order; returns the count
template <int NT>
__device__ int he_gather(const HandEyeArgs& a, int m, int s, int bm, int bs, int f0, double (*sA)[12], double (*sB)[12]) {
  const int f = f0 + threadIdx.x;
  const size_t vm = ((size_t)m * a.F + f) * a.B + bm, vs = ((size_t)s * a.F + f) * a.B + bs;
  const bool p = f < a.F && a.valid[vm] && a.valid[vs];
  int tot;
  const int pos = pi_scan<NT>(p ? 1 : 0, tot);
  if (p) { pi_inv34(a.poses + 16 * vm, sA[pos]); pi_inv34(a.poses + 16 * vs, sB[pos]); }
  __syncthreads();
  return tot;
}

__global__ void __launch_bounds__(HE_THREADS) k_he_quads(HandEyeArgs a) {
  constexpr int NT = HE_THREADS;
  __shared__ double sA[NT][12], sB[NT][12];
  __shared__ double sT[90];                        // T row-major (81), then S = sum R_A (9)
  __shared__ double sM[81], sV[81];
  __shared__ double sRX[9], sRZ[9], sg[6];
  __shared__ int s_ok;
  const int q = blockIdx.x, t = threadIdx.x;
  const int m = a.quads[4 * q], s = a.quads[4 * q + 1], bm = a.quads[4 * q + 2], bs = a.quads[4 * q + 3];
  double acc = 0.0;
  int n = 0;
  for (int f0 = 0; f0 < a.F; f0 += NT) {
    const int tot = he_gather<NT>(a, m, s, bm, bs, f0, sA, sB);
    if (t < 81) {                                  // kron(R_B, R_A)[i][j] = R_B[i/3][j/3] R_A[i%3][j%3]
      const int i = t / 9, j = t % 9, b = 4 * (i / 3) + j / 3, c = 4 * (i % 3) + j % 3;
      for (int k = 0; k < tot; k++) acc += sB[k][b] * sA[k][c];
    } else if (t < 90) {
      const int e = t - 81, c = 4 * (e / 3) + e % 3;
      for (int k = 0; k < tot; k++) acc += sA[k][c];
    }
    n += tot;
    __syncthreads();
  }
  double* X = a.X + 16 * (size_t)q; double* Z = a.Z + 16 * (size_t)q;
  if (t < 16) { X[t] = t % 5 == 0 ? 1.0 : 0.0; Z[t] = X[t]; }
  if (t == 0) a.n_images[q] = n;
  if (n < 3) { if (t == 0) a.ok[q] = 0; return; }
  if (t < 90) sT[t] = acc;
  __syncthreads();
  if (t < 81) {                                    // T^T T
    const int i = t / 9, j = t % 9;
    double v = 0.0;
    for (int k = 0; k < 9; k++) v += sT[9 * k + i] * sT[9 * k + j];
    sM[t] = v;
  }
  __syncthreads();
  if (t == 0) {
    he_jacobi(sM, sV, 9);
    int i1 = 0;
    for (int i = 1; i < 9; i++) if (sM[10 * i] > sM[10 * i1]) i1 = i;
    double l2 = -INFINITY;
    for (int i = 0; i < 9; i++) if (i != i1) l2 = fmax(l2, sM[10 * i]);
    const double s1 = sqrt(fmax(sM[10 * i1], 0.0)), s2 = sqrt(fmax(l2, 0.0));
    double v[9], u[9], nu = 0.0;
    for (int k = 0; k < 9; k++) v[k] = sV[9 * k + i1];
    for (int k = 0; k < 9; k++) {
      double x = 0.0;
      for (int j = 0; j < 9; j++) x += sT[9 * k + j] * v[j];
      u[k] = x; nu += x * x;
    }
    nu = sqrt(nu);
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) { sRX[3 * r + c] = v[3 * c + r]; sRZ[3 * r + c] = u[3 * c + r] / nu; }
    const bool ok = s1 > 0.0 && (s1 - s2) / s1 >= HE_GAP_MIN && fabs(he_det3(sRX)) >= HE_DET_MIN && fabs(he_det3(sRZ)) >= HE_DET_MIN;
    if (ok) { he_polar(sRX); he_polar(sRZ); }
    s_ok = ok;
    a.ok[q] = ok;
  }
  __syncthreads();
  if (!s_ok) return;
  acc = 0.0;                                       // t < 3: sum r_i; 3 <= t < 6: -sum R_A_i^T r_i, r_i = t_A_i - R_Z t_B_i
  for (int f0 = 0; f0 < a.F; f0 += NT) {
    const int tot = he_gather<NT>(a, m, s, bm, bs, f0, sA, sB);
    if (t < tot) {
      double r[3];
      for (int i = 0; i < 3; i++) r[i] = sA[t][4 * i + 3] - (sRZ[3 * i] * sB[t][3] + sRZ[3 * i + 1] * sB[t][7] + sRZ[3 * i + 2] * sB[t][11]);
      for (int i = 0; i < 3; i++) sB[t][i] = r[i];
    }
    __syncthreads();
    if (t < 3) for (int k = 0; k < tot; k++) acc += sB[k][t];
    else if (t < 6) {
      const int e = t - 3;
      for (int k = 0; k < tot; k++) acc -= sA[k][e] * sB[k][0] + sA[k][4 + e] * sB[k][1] + sA[k][8 + e] * sB[k][2];
    }
    __syncthreads();
  }
  if (t < 6) sg[t] = acc;
  __syncthreads();
  if (t == 0) {
    // (n^2 I - S^T S) t_X = n g1 + S^T g2,  t_Z = (g2 + S t_X) / n,  g1 = -sum R_A^T r, g2 = sum r
    const double* S = sT + 81;
    const double nd = (double)n;
    double M[9], rhs[3], tx[3], tz[3];
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) M[3 * i + j] = (i == j ? nd * nd : 0.0) - (S[i] * S[j] + S[3 + i] * S[3 + j] + S[6 + i] * S[6 + j]);
      rhs[i] = nd * sg[3 + i] + S[i] * sg[0] + S[3 + i] * sg[1] + S[6 + i] * sg[2];
    }
    const double d = he_det3(M);
    for (int i = 0; i < 3; i++) {                  // Cramer's rule with the cofactors of the symmetric M
      const int i1 = (i + 1) % 3, i2 = (i + 2) % 3;
      double x = 0.0;
      for (int j = 0; j < 3; j++) {
        const int j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        x += (M[3 * j1 + i1] * M[3 * j2 + i2] - M[3 * j1 + i2] * M[3 * j2 + i1]) * rhs[j];
      }
      tx[i] = x / d;
    }
    for (int i = 0; i < 3; i++) tz[i] = (sg[i] + S[3 * i] * tx[0] + S[3 * i + 1] * tx[1] + S[3 * i + 2] * tx[2]) / nd;
    for (int i = 0; i < 3; i++) {
      for (int j = 0; j < 3; j++) { X[4 * i + j] = sRX[3 * i + j]; Z[4 * i + j] = sRZ[3 * i + j]; }
      X[4 * i + 3] = tx[i]; Z[4 * i + 3] = tz[i];
    }
  }
}

__device__ inline double he_warp_sum(double v) {  // fixed-order tree; lane 0's total broadcast to the warp
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return __shfl_sync(0xffffffffu, v, 0);
}

__global__ void __launch_bounds__(32 * HE_VOTE_WARPS) k_he_vote(HandEyeVoteArgs a) {
  const int set = blockIdx.x * HE_VOTE_WARPS + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (set >= a.n_sets) return;                     // whole warps leave together
  const int64_t s0 = a.start[set];
  const int n = (int)(a.start[set + 1] - s0);
  const double* P = a.points + 3 * s0;
  double* dens = a.density + s0;
  double mu[3];
  for (int c = 0; c < 3; c++) {
    double x = 0.0;
    for (int i = lane; i < n; i += 32) x += P[3 * i + c];
    mu[c] = he_warp_sum(x) / n;
  }
  double cv[6];                                    // xx yy zz xy xz yz
  const int ca[6] = {0, 1, 2, 0, 0, 1}, cb[6] = {0, 1, 2, 1, 2, 2};
  for (int k = 0; k < 6; k++) {
    double x = 0.0;
    for (int i = lane; i < n; i += 32) x += (P[3 * i + ca[k]] - mu[ca[k]]) * (P[3 * i + cb[k]] - mu[cb[k]]);
    cv[k] = he_warp_sum(x) / (n - 1);
  }
  const double f2 = pow((double)n, -2.0 / 7.0);   // Scott's factor squared, d = 3
  // Cholesky L of cov f^2
  const double l00 = sqrt(cv[0] * f2), l10 = cv[3] * f2 / l00, l20 = cv[4] * f2 / l00;
  const double l11 = sqrt(cv[1] * f2 - l10 * l10), l21 = (cv[5] * f2 - l20 * l10) / l11;
  const double l22 = sqrt(cv[2] * f2 - l20 * l20 - l21 * l21);
  if (!(l00 > 0.0 && l11 > 0.0 && l22 > 0.0)) {   // singular covariance (scipy: LinAlgError)
    for (int i = lane; i < n; i += 32) dens[i] = NAN;
    if (lane == 0) a.best[set] = -1;
    return;
  }
  const double norm = 1.0 / (n * 15.749609945722419 * l00 * l11 * l22);   // (2 pi)^(3/2)
  double dmax = -INFINITY;
  for (int i = lane; i < n; i += 32) {
    double acc = 0.0;
    for (int j = 0; j < n; j++) {
      const double d0 = P[3 * i] - P[3 * j], d1 = P[3 * i + 1] - P[3 * j + 1], d2 = P[3 * i + 2] - P[3 * j + 2];
      const double y0 = d0 / l00, y1 = (d1 - l10 * y0) / l11, y2 = (d2 - l20 * y0 - l21 * y1) / l22;
      acc += exp(-0.5 * (y0 * y0 + y1 * y1 + y2 * y2));
    }
    dens[i] = acc * norm;
    dmax = fmax(dmax, acc * norm);
  }
  for (int o = 16; o > 0; o >>= 1) dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
  __syncwarp();
  int b = 0x7fffffff;
  for (int i = lane; i < n; i += 32) if (dens[i] >= dmax * (1.0 - HE_TIE_REL)) { b = i; break; }
  for (int o = 16; o > 0; o >>= 1) b = min(b, __shfl_xor_sync(0xffffffffu, b, o));
  if (lane == 0) a.best[set] = b;
}

}  // namespace mcba
