// triangulate_kernels.cuh — 3-D points from pixels seen by several calibrated cameras (DESIGN.md §3j):
//   k_triangulate<MODEL, LANES>   N-view triangulation through the full camera model: linear start, then Levenberg-Marquardt on X
//   k_triangulate_linear          cv2.triangulatePoints: the linear solution of two pixel projection matrices
//
// One group of LANES lanes per point (LANES a power of two from 2 to 32, the smallest >= min(C, 32)); lane l owns the point's views
// c = l, l + LANES, ...  Every sum over views is a lane-local sum in view order followed by an xor-shuffle tree over the group, so all
// lanes of a group hold the same bits and two identical calls agree bit for bit.  Every warp-collective is executed by all 32 lanes:
// the loops run while any group of the warp still works, and a group that has finished computes but no longer changes its state, so a
// point's result does not depend on its neighbours.
//
// The linear solution (group_dlt): the rows x T3 - T1 and y T3 - T2 of each view (T the 3x4 projection), 2n x 4, by one-sided Jacobi
// SVD: column pairs are rotated until every pair is orthogonal to working precision, each column dot product one group reduction.  The
// right singular vector of the smallest column norm is the homogeneous point, of unit norm.  (The eigenvectors of A^T A would square the
// condition number.)  A lane keeps its rows in shared memory; it is the only one that reads or writes them.
#pragma once
#include <stdint.h>
#include <float.h>
#include "geometry.cuh"
#include "pnp_kernels.cuh"

namespace mcba {

constexpr int TRI_THREADS = 256;
constexpr int TRI_KD = 5 + 14;               // camera vector [fx fy cx cy skew dist...], distortion padded to 14
constexpr int TRI_SWEEPS = 30;               // Jacobi sweeps at most (4 columns converge in about 6)
constexpr double TRI_JACOBI_TOL = 4.0 * DBL_EPSILON;
constexpr int TRI_MAX_ITERS = 50;
constexpr double TRI_XTOL = 1e-12, TRI_FTOL = 1e-15;

// dynamic shared memory of a CTA: 8 doubles (2 rows of 4) per view a lane owns
__host__ __device__ __forceinline__ size_t tri_smem(int nk) { return (size_t)TRI_THREADS * 8 * nk * sizeof(double); }

// the lanes of a group for C cameras
__host__ __device__ __forceinline__ int tri_lanes(int C) {
  int l = 2;
  while (l < C && l < 32) l *= 2;
  return l;
}

template <int LANES>
__device__ __forceinline__ double group_sum(double v) {
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one-sided Jacobi SVD of the group's rows; A points at this lane's first entry, entry (row slot r < 2 nk, column j) at
// A[(j * 2 nk + r) * stride].  Xh: the right singular vector of the smallest singular value, unit norm, the same in every lane of the
// group; NaN when a row of the group is not finite.
template <int LANES>
__device__ void group_dlt(double* A, int nk, int stride, double* Xh) {
  const int nr = 2 * nk;
  double V[16];
#pragma unroll
  for (int i = 0; i < 16; i++) V[i] = i % 5 == 0 ? 1.0 : 0.0;
  bool finite = true;
  for (int r = 0; r < nr; r++)
    for (int j = 0; j < 4; j++) finite = finite && isfinite(A[(j * nr + r) * stride]);
  const bool bad = group_sum<LANES>(finite ? 0.0 : 1.0) != 0.0;
  bool done = bad;
  for (int sweep = 0; sweep < TRI_SWEEPS && __ballot_sync(0xffffffffu, !done) != 0; sweep++) {
    bool rotated = false;
    for (int p = 0; p < 3; p++)
      for (int q = p + 1; q < 4; q++) {
        double a = 0.0, b = 0.0, g = 0.0;
        for (int r = 0; r < nr; r++) {
          const double x = A[(p * nr + r) * stride], y = A[(q * nr + r) * stride];
          a += x * x; b += y * y; g += x * y;
        }
        a = group_sum<LANES>(a); b = group_sum<LANES>(b); g = group_sum<LANES>(g);
        if (done || !(fabs(g) > TRI_JACOBI_TOL * sqrt(a) * sqrt(b))) continue;
        const double zeta = (b - a) / (2.0 * g);
        const double t = copysign(1.0, zeta) / (fabs(zeta) + hypot(1.0, zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
        for (int r = 0; r < nr; r++) {
          double& x = A[(p * nr + r) * stride];
          double& y = A[(q * nr + r) * stride];
          const double xp = x, yp = y;
          x = c * xp - s * yp; y = s * xp + c * yp;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const double xp = V[4 * i + p], yp = V[4 * i + q];
          V[4 * i + p] = c * xp - s * yp; V[4 * i + q] = s * xp + c * yp;
        }
        rotated = true;
      }
    if (!rotated) done = true;
  }
  double nrm[4];
  for (int j = 0; j < 4; j++) {
    double s = 0.0;
    for (int r = 0; r < nr; r++) { const double x = A[(j * nr + r) * stride]; s += x * x; }
    nrm[j] = group_sum<LANES>(s);
  }
  int m = 0;
  for (int j = 1; j < 4; j++) if (nrm[j] < nrm[m]) m = j;
  const double s = 1.0 / sqrt(V[m] * V[m] + V[4 + m] * V[4 + m] + V[8 + m] * V[8 + m] + V[12 + m] * V[12 + m]);
  for (int i = 0; i < 4; i++) Xh[i] = bad ? NAN : V[4 * i + m] * s;
}

// the two DLT rows of pixel or normalised point (x, y) under the 3x4 row-major T, written to this lane's row slots 2k, 2k + 1
__device__ __forceinline__ void dlt_rows(double* A, int nk, int k, int stride, double x, double y, const double* T) {
  const int nr = 2 * nk;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    A[(j * nr + 2 * k) * stride] = x * T[8 + j] - T[j];
    A[(j * nr + 2 * k + 1) * stride] = y * T[8 + j] - T[4 + j];
  }
}

struct TriArgs {
  int C, nk;                   // cameras, views per lane (ceil(C / LANES))
  int64_t n;                   // points of this chunk
  const double* cams;          // [C][TRI_KD]
  const double* poses;         // [C][16] rig -> camera, row-major
  const double2* px;           // [C][n]
  const uint8_t* valid;        // [C][n]
  double* points;              // [n][3]
  uint8_t* ok;                 // [n]
  double* rms;                 // [n]
};

// The sums of the point's residuals at rig point X over its valid views, reduced over the group: s = [H00 H01 H02 H11 H12 H22 g0 g1 g2
// cost behind] with residual e = project(R X + t) - pixel, J = [Ju; Jv] R, H = J^T J, g = J^T e, cost = |e|^2 and `behind` the number of
// views with z_cam <= 0.  A lane with on = false adds nothing (but takes part in the reductions).
template <int MODEL, int LANES>
__device__ void tri_eval(const TriArgs& a, int64_t p, bool on, int lane, const double* X, double* s) {
  double loc[11];
#pragma unroll
  for (int i = 0; i < 11; i++) loc[i] = 0.0;
  for (int k = 0; k < a.nk; k++) {
    const int c = k * LANES + lane;
    if (!on || c >= a.C || !a.valid[(size_t)c * a.n + p]) continue;
    const double* T = a.poses + 16 * c;
    const double Xc[3] = {T[0] * X[0] + T[1] * X[1] + T[2] * X[2] + T[3], T[4] * X[0] + T[5] * X[1] + T[6] * X[2] + T[7],
                          T[8] * X[0] + T[9] * X[1] + T[10] * X[2] + T[11]};
    double u, v, Ju[3], Jv[3], ku[4 + 14], kv[4 + 14];
    project<MODEL, true>(Xc, a.cams + TRI_KD * c, u, v, Ju, Jv, ku, kv);
    const double2 q = a.px[(size_t)c * a.n + p];
    const double eu = u - q.x, ev = v - q.y;
    double ju[3], jv[3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
      ju[j] = Ju[0] * T[j] + Ju[1] * T[4 + j] + Ju[2] * T[8 + j];
      jv[j] = Jv[0] * T[j] + Jv[1] * T[4 + j] + Jv[2] * T[8 + j];
    }
    loc[0] += ju[0] * ju[0] + jv[0] * jv[0]; loc[1] += ju[0] * ju[1] + jv[0] * jv[1]; loc[2] += ju[0] * ju[2] + jv[0] * jv[2];
    loc[3] += ju[1] * ju[1] + jv[1] * jv[1]; loc[4] += ju[1] * ju[2] + jv[1] * jv[2]; loc[5] += ju[2] * ju[2] + jv[2] * jv[2];
    loc[6] += ju[0] * eu + jv[0] * ev; loc[7] += ju[1] * eu + jv[1] * ev; loc[8] += ju[2] * eu + jv[2] * ev;
    loc[9] += eu * eu + ev * ev;
    loc[10] += Xc[2] <= 0.0 ? 1.0 : 0.0;
  }
#pragma unroll
  for (int i = 0; i < 11; i++) s[i] = group_sum<LANES>(loc[i]);
}

// One group per point; grid ceil(n LANES / TRI_THREADS) of TRI_THREADS, dynamic shared memory tri_smem(nk).
//  1. Each valid view's pixel is undistorted to normalised coordinates by undistort_pixel<MODEL> under K = I after the division by the
//     focal lengths (k_rectify_points with R = P = I); its DLT rows use T = the camera's pose.  A fisheye pixel whose undistortion fails
//     (OpenCV's -1e6 sentinel) gives no rows; a non-finite pixel gives non-finite rows, so the point is invalid.
//  2. X = the DLT's (x, y, z) / w.
//  3. Levenberg-Marquardt on X: (H + lambda diag(H)) d = -g by spd_solve<3>, lambda from 1e-3, x10 on a rejected step, x0.1 on an
//     accepted one; a step is accepted only if the cost decreases.  Stops on |d| <= TRI_XTOL |X|, on an accepted step that lowers the
//     cost by at most TRI_FTOL of it, or after TRI_MAX_ITERS steps.
//  4. The point is valid with at least 2 valid views, a finite non-zero w (|w| > DBL_EPSILON, w of the unit vector), every view at
//     z_cam > 0 at the end and finite results; otherwise its point and rms are NaN.  rms = sqrt(cost / views).
template <int MODEL, int LANES>
__global__ void __launch_bounds__(TRI_THREADS) k_triangulate(TriArgs a) {
  extern __shared__ double tri_rows[];
  const int lane = threadIdx.x % LANES;
  const int64_t p = ((int64_t)blockIdx.x * TRI_THREADS + threadIdx.x) / LANES;
  const bool active = p < a.n;
  double* A = tri_rows + threadIdx.x;
  double nv = 0.0;
  for (int k = 0; k < a.nk; k++) {
    const int c = k * LANES + lane;
    double x = 0.0, y = 0.0;
    const double* T = nullptr;
    if (active && c < a.C && a.valid[(size_t)c * a.n + p]) {
      nv += 1.0;
      const double2 q = a.px[(size_t)c * a.n + p];
      const double* kc = a.cams + TRI_KD * c;
      double kn[TRI_KD];
      kn[0] = 1.0; kn[1] = 1.0; kn[2] = 0.0; kn[3] = 0.0; kn[4] = 0.0;
      for (int d = 0; d < 14; d++) kn[5 + d] = kc[5 + d];
      if (isfinite(q.x) && isfinite(q.y)) {
        undistort_pixel<MODEL>(kn, (q.x - kc[2]) / kc[0], (q.y - kc[3]) / kc[1], x, y);
        if (!(MODEL == MODEL_FISHEYE && x == -1000000.0 && y == -1000000.0)) T = a.poses + 16 * c;
      } else {
        x = NAN; y = NAN; T = a.poses + 16 * c;
      }
    }
    const double zero[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    dlt_rows(A, a.nk, k, TRI_THREADS, T ? x : 0.0, T ? y : 0.0, T ? T : zero);
  }
  nv = group_sum<LANES>(nv);
  double Xh[4];
  group_dlt<LANES>(A, a.nk, TRI_THREADS, Xh);
  const bool start = active && nv >= 2.0 && isfinite(Xh[3]) && fabs(Xh[3]) > DBL_EPSILON;
  double X[3] = {0.0, 0.0, 0.0};
  if (start) { X[0] = Xh[0] / Xh[3]; X[1] = Xh[1] / Xh[3]; X[2] = Xh[2] / Xh[3]; }
  double s[11];
  tri_eval<MODEL, LANES>(a, p, start, lane, X, s);
  bool done = !start;
  double lambda = 1e-3;
  int it = 0;
  while (__ballot_sync(0xffffffffu, !done) != 0) {
    double Xt[3] = {X[0], X[1], X[2]}, step = 0.0;
    bool solved = false;
    if (!done) {
      double M[9] = {s[0], s[1], s[2], s[1], s[3], s[4], s[2], s[4], s[5]}, d[3] = {-s[6], -s[7], -s[8]};
      M[0] += lambda * s[0]; M[4] += lambda * s[3]; M[8] += lambda * s[5];
      solved = spd_solve<3>(M, d);
      if (solved) {
        for (int j = 0; j < 3; j++) Xt[j] = X[j] + d[j];
        step = sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
      }
    }
    double st[11];
    tri_eval<MODEL, LANES>(a, p, !done && solved, lane, Xt, st);
    if (done) continue;
    const double xn = sqrt(X[0] * X[0] + X[1] * X[1] + X[2] * X[2]);
    if (solved && st[9] < s[9]) {
      const double decrease = s[9] - st[9], before = s[9];
      for (int j = 0; j < 3; j++) X[j] = Xt[j];
      for (int i = 0; i < 11; i++) s[i] = st[i];
      lambda *= 0.1;
      if (decrease <= TRI_FTOL * before) done = true;
    } else {
      lambda *= 10.0;
    }
    if (solved && step <= TRI_XTOL * xn) done = true;
    if (++it >= TRI_MAX_ITERS) done = true;
  }
  if (!active || lane != 0) return;
  const double r = sqrt(s[9] / nv);
  const bool good = start && s[10] == 0.0 && isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]) && isfinite(r);
  for (int j = 0; j < 3; j++) a.points[3 * p + j] = good ? X[j] : NAN;
  a.rms[p] = good ? r : NAN;
  a.ok[p] = good ? 1 : 0;
}

struct TriLinearArgs {
  double P[2][12];             // the two 3x4 projection matrices, row-major
  int64_t n;
  const double* x[2];          // [2][n] each: row 0 x, row 1 y
  double* out;                 // [4][n]
};

// cv2.triangulatePoints(P1, P2, x1, x2): group_dlt of the 4 x 4 system, a group of 2 lanes per point (lane l: view l); grid
// ceil(2 n / TRI_THREADS) of TRI_THREADS, dynamic shared memory tri_smem(1).
__global__ void __launch_bounds__(TRI_THREADS) k_triangulate_linear(TriLinearArgs a) {
  extern __shared__ double tri_rows[];
  const int lane = threadIdx.x & 1;
  const int64_t p = ((int64_t)blockIdx.x * TRI_THREADS + threadIdx.x) >> 1;
  const bool active = p < a.n;
  double* A = tri_rows + threadIdx.x;
  const double* x = a.x[lane];
  dlt_rows(A, 1, 0, TRI_THREADS, active ? x[p] : 0.0, active ? x[a.n + p] : 0.0, a.P[lane]);
  double Xh[4];
  group_dlt<2>(A, 1, TRI_THREADS, Xh);
  if (active && lane == 0)
    for (int j = 0; j < 4; j++) a.out[j * a.n + p] = Xh[j];
}

}  // namespace mcba
