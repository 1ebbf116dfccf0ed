// intrinsics_kernels.cuh — the initialisation of single-camera intrinsic calibration (Camera.calibrate, camera.py:68-105 ->
// cv2.calibrateCameraExtended without an initial matrix), batched over every view of every camera, and the per-view error sums that
// follow each solve.
//
//   k_view_homography   one warp per used detection list: homography board plane (X, Y) -> pixels, normalised DLT refined by
//                       Levenberg-Marquardt on its pixel reprojection error (what cv2.findHomography does)
//   k_zhang_init        one CTA per camera: OpenCV's initIntrinsicParams2D (cv2.initCameraMatrix2D) from those homographies
//   (the initial per-view poses are k_pnp_views, pnp_kernels.cuh, given K0 and zero distortion: OpenCV's findExtrinsicCameraParams2)
//   k_fisheye_k0        one thread per camera: the start of cv2.fisheye.calibrate (CameraFisheye.calibrate, camera_fisheye.py:70-94),
//                       whose initial per-view poses are k_pnp_views<MODEL_FISHEYE> under it (exact fisheye undistortion at k = 0)
//   k_view_sumsq        per view of the packed problem: sum of squared pixel errors (k_views<MODE_COST>, kernels.cuh) and corner count
//
// K0 only seeds the trust-region solve, which iterates to its own tolerances.
// All sums are fp64 in a fixed order (lane-strided, then the xor butterfly of warp_sum; per camera: contiguous chunks of views in order,
// then the chunks in order), so two identical calls agree bit for bit.
#pragma once
#include <stdint.h>
#include "kernels.cuh"
#include "pnp_kernels.cuh"

namespace mcba {

constexpr int HOMOG_WARPS = 4;
constexpr int ZHANG_THREADS = 128;

struct HomographyArgs {
  int n_used, B, P;
  const int32_t* used;          // [n_used] list w = (c*F+f)*B+b, grouped by camera
  const int64_t* det_start;     // [C*F*B+1] CSR
  const int32_t* det_ids;
  const double2* det_xy;
  const double* board_pts;      // [B][P][3], z = 0 (checked on the host)
  double* H;                    // [n_used][9] row-major, h33 = 1, maps (X, Y, 1) to pixels
  uint8_t* ok;                  // [n_used]
};

// Normalise both point sets (centroid to the origin, mean distance sqrt 2), solve the 8x8 normal equations of the DLT with h33 = 1, refine,
// undo the normalisations.  Pixels and board points are rounded to float32 first, as calibration_points hands them to OpenCV.
__global__ void __launch_bounds__(HOMOG_WARPS * 32)
k_view_homography(HomographyArgs a) {
  const int lane = threadIdx.x & 31;
  const int u = blockIdx.x * HOMOG_WARPS + (threadIdx.x >> 5);
  if (u >= a.n_used) return;
  const int w = a.used[u], b = w % a.B;
  const int64_t beg = a.det_start[w], end = a.det_start[w + 1];
  const int n = (int)(end - beg);
  const double* bp = a.board_pts + (size_t)b * a.P * 3;
  double* Hout = a.H + (size_t)9 * u;
  auto board_xy = [&](int64_t i, double& X, double& Y) {
    const int id = a.det_ids[i];
    X = (double)(float)bp[3 * id]; Y = (double)(float)bp[3 * id + 1];
  };
  auto pixel = [&](int64_t i, double& x, double& y) {
    const double2 q = a.det_xy[i];
    x = (double)(float)q.x; y = (double)(float)q.y;
  };
  double mX = 0, mY = 0, mx = 0, my = 0;
  for (int64_t i = beg + lane; i < end; i += 32) {
    double X, Y, x, y;
    board_xy(i, X, Y); pixel(i, x, y);
    mX += X; mY += Y; mx += x; my += y;
  }
  mX = warp_sum(mX) / n; mY = warp_sum(mY) / n; mx = warp_sum(mx) / n; my = warp_sum(my) / n;
  double dB = 0, dP = 0;
  for (int64_t i = beg + lane; i < end; i += 32) {
    double X, Y, x, y;
    board_xy(i, X, Y); pixel(i, x, y);
    dB += sqrt((X - mX) * (X - mX) + (Y - mY) * (Y - mY));
    dP += sqrt((x - mx) * (x - mx) + (y - my) * (y - my));
  }
  dB = warp_sum(dB) / n; dP = warp_sum(dP) / n;
  const double sB = dB > 0 ? 1.4142135623730951 / dB : 1.0, sP = dP > 0 ? 1.4142135623730951 / dP : 1.0;

  double N[44];                                                       // upper triangle of A^T A (36) | A^T b (8)
#pragma unroll
  for (int i = 0; i < 44; i++) N[i] = 0.0;
  for (int64_t i = beg + lane; i < end; i += 32) {
    double X, Y, x, y;
    board_xy(i, X, Y); pixel(i, x, y);
    X = (X - mX) * sB; Y = (Y - mY) * sB; x = (x - mx) * sP; y = (y - my) * sP;
    const double ru[8] = {X, Y, 1, 0, 0, 0, -x * X, -x * Y}, rv[8] = {0, 0, 0, X, Y, 1, -y * X, -y * Y};
    int e = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
#pragma unroll
      for (int s = r; s < 8; s++) { N[e] += ru[r] * ru[s] + rv[r] * rv[s]; e++; }
      N[36 + r] += ru[r] * x + rv[r] * y;
    }
  }
#pragma unroll
  for (int i = 0; i < 44; i++) N[i] = warp_sum(N[i]);
  double A[64], h[8];
  {
    int e = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
#pragma unroll
      for (int s = r; s < 8; s++) { A[r * 8 + s] = N[e]; A[s * 8 + r] = N[e]; e++; }
      h[r] = N[36 + r];
    }
  }
  bool solved = n >= 4 && spd_solve<8>(A, h);

  // Levenberg-Marquardt on the reprojection error of the homography, as cv2.findHomography refines its DLT.  The pixel normalisation is
  // isotropic, so the minimiser in normalised coordinates is the pixel-space one.
  auto cost_of = [&](const double* g) {
    double s = 0.0;
    for (int64_t i = beg + lane; i < end; i += 32) {
      double X, Y, x, y;
      board_xy(i, X, Y); pixel(i, x, y);
      X = (X - mX) * sB; Y = (Y - mY) * sB; x = (x - mx) * sP; y = (y - my) * sP;
      const double iw = 1.0 / (g[6] * X + g[7] * Y + 1.0);
      const double ru = (g[0] * X + g[1] * Y + g[2]) * iw - x, rv = (g[3] * X + g[4] * Y + g[5]) * iw - y;
      s += ru * ru + rv * rv;
    }
    return warp_sum(s);
  };
  double lambda = 1e-3, cost = solved ? cost_of(h) : 0.0;
  for (int it = 0; solved && it < 30; it++) {
#pragma unroll
    for (int i = 0; i < 44; i++) N[i] = 0.0;
    for (int64_t i = beg + lane; i < end; i += 32) {
      double X, Y, x, y;
      board_xy(i, X, Y); pixel(i, x, y);
      X = (X - mX) * sB; Y = (Y - mY) * sB; x = (x - mx) * sP; y = (y - my) * sP;
      const double iw = 1.0 / (h[6] * X + h[7] * Y + 1.0);
      const double u = (h[0] * X + h[1] * Y + h[2]) * iw, v = (h[3] * X + h[4] * Y + h[5]) * iw;
      const double ru = u - x, rv = v - y;
      const double ju[8] = {X * iw, Y * iw, iw, 0, 0, 0, -u * X * iw, -u * Y * iw}, jv[8] = {0, 0, 0, X * iw, Y * iw, iw, -v * X * iw, -v * Y * iw};
      int e = 0;
#pragma unroll
      for (int r = 0; r < 8; r++) {
#pragma unroll
        for (int s = r; s < 8; s++) { N[e] += ju[r] * ju[s] + jv[r] * jv[s]; e++; }
        N[36 + r] += ju[r] * ru + jv[r] * rv;
      }
    }
#pragma unroll
    for (int i = 0; i < 44; i++) N[i] = warp_sum(N[i]);
    bool improved = false, stop = false;
    for (int tries = 0; tries < 12 && !improved && !stop; tries++) {
      double M[64], d[8];
      int e = 0;
#pragma unroll
      for (int r = 0; r < 8; r++) {
#pragma unroll
        for (int s = r; s < 8; s++) { M[r * 8 + s] = N[e]; M[s * 8 + r] = N[e]; e++; }
        d[r] = -N[36 + r];
      }
#pragma unroll
      for (int r = 0; r < 8; r++) M[r * 9] += lambda * fmax(M[r * 9], 1e-30);
      if (!spd_solve<8>(M, d)) { lambda *= 10.0; continue; }
      double hn[8], step2 = 0.0, h2 = 0.0;
#pragma unroll
      for (int r = 0; r < 8; r++) { hn[r] = h[r] + d[r]; step2 += d[r] * d[r]; h2 += h[r] * h[r]; }
      const double cn = cost_of(hn);
      if (cn <= cost) {
        stop = (cost - cn) <= 1e-15 * cost || step2 <= 1e-30 * h2;
#pragma unroll
        for (int r = 0; r < 8; r++) h[r] = hn[r];
        cost = cn;
        lambda = fmax(lambda * 0.1, 1e-12);
        improved = true;
      } else {
        stop = step2 <= 1e-30 * h2;
        lambda *= 10.0;
      }
    }
    if (stop || !improved) break;
  }

  // H = Tp^-1 Hn Tb with Tb = [sB 0 -sB mX; 0 sB -sB mY; 0 0 1], Tp^-1 = [1/sP 0 mx; 0 1/sP my; 0 0 1]
  const double Hn[9] = {h[0], h[1], h[2], h[3], h[4], h[5], h[6], h[7], 1.0};
  double G[9];                                                        // Hn Tb
#pragma unroll
  for (int r = 0; r < 3; r++) {
    G[3 * r] = Hn[3 * r] * sB;
    G[3 * r + 1] = Hn[3 * r + 1] * sB;
    G[3 * r + 2] = Hn[3 * r + 2] - sB * (Hn[3 * r] * mX + Hn[3 * r + 1] * mY);
  }
  double H[9];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    H[c] = G[c] / sP + mx * G[6 + c];
    H[3 + c] = G[3 + c] / sP + my * G[6 + c];
    H[6 + c] = G[6 + c];
  }
  const double s = 1.0 / H[8];
  bool finite = solved;
#pragma unroll
  for (int i = 0; i < 9; i++) { H[i] *= s; finite = finite && isfinite(H[i]); }
  if (lane < 9) Hout[lane] = H[lane];
  if (lane == 0) a.ok[u] = finite ? 1 : 0;
}

struct ZhangArgs {
  int kint, fix_aspect;
  const int32_t* cam_start;     // [C+1] CSR of the used views of each camera (rows of H)
  const int32_t* image_size;    // [C][2] = width, height
  const double* H;              // [n_used][9]
  const uint8_t* ok;            // [n_used]
  double* intr;                 // [C][kint] out: fx fy cx cy 0 | zero distortion
};

// initIntrinsicParams2D: principal point ((w-1)/2, (h-1)/2); per view the homography with the principal point moved to the origin,
// h = column 1, v = column 2, d1 = (h+v)/2, d2 = (h-v)/2, each scaled to unit length, gives two rows
//   [h0 v0, h1 v1] f = -h2 v2,   [d1_0 d2_0, d1_1 d2_1] f = -d1_2 d2_2
// and f = (1/fx^2, 1/fy^2) is their least-squares solution (normal equations); fx, fy = sqrt|1/f|.  Under fix_aspect (OpenCV's
// CALIB_FIX_ASPECT_RATIO with an identity input matrix: aspect ratio 1) both become their mean.  A camera without a usable view gets NaN.
__global__ void __launch_bounds__(ZHANG_THREADS)
k_zhang_init(ZhangArgs a) {
  const int c = blockIdx.x, t = threadIdx.x;
  const int v0 = a.cam_start[c], v1 = a.cam_start[c + 1], nv = v1 - v0;
  const double cx = (a.image_size[2 * c] - 1) * 0.5, cy = (a.image_size[2 * c + 1] - 1) * 0.5;
  __shared__ double part[ZHANG_THREADS][6];
  __shared__ int bad_any;
  if (t == 0) bad_any = 0;
  __syncthreads();
  // AtA = [s00 s01; s01 s11], Atb = [r0; r1]
  double s00 = 0, s01 = 0, s11 = 0, r0 = 0, r1 = 0;
  int bad = 0;
  const int per = (nv + ZHANG_THREADS - 1) / ZHANG_THREADS;
  const int lo = v0 + t * per, hi = min(v1, lo + per);
  for (int v = lo; v < hi; v++) {
    if (!a.ok[v]) { bad = 1; continue; }
    double H[9];
#pragma unroll
    for (int i = 0; i < 9; i++) H[i] = a.H[(size_t)9 * v + i];
    H[0] -= H[6] * cx; H[1] -= H[7] * cx; H[2] -= H[8] * cx;
    H[3] -= H[6] * cy; H[4] -= H[7] * cy; H[5] -= H[8] * cy;
    double h[3], vv[3], d1[3], d2[3], n0 = 0, n1 = 0, n2 = 0, n3 = 0;
#pragma unroll
    for (int j = 0; j < 3; j++) {
      const double t0 = H[3 * j], t1 = H[3 * j + 1];
      h[j] = t0; vv[j] = t1; d1[j] = (t0 + t1) * 0.5; d2[j] = (t0 - t1) * 0.5;
      n0 += t0 * t0; n1 += t1 * t1; n2 += d1[j] * d1[j]; n3 += d2[j] * d2[j];
    }
    n0 = 1.0 / sqrt(n0); n1 = 1.0 / sqrt(n1); n2 = 1.0 / sqrt(n2); n3 = 1.0 / sqrt(n3);
#pragma unroll
    for (int j = 0; j < 3; j++) { h[j] *= n0; vv[j] *= n1; d1[j] *= n2; d2[j] *= n3; }
    const double a0 = h[0] * vv[0], a1 = h[1] * vv[1], b0 = -h[2] * vv[2];
    const double a2 = d1[0] * d2[0], a3 = d1[1] * d2[1], b1 = -d1[2] * d2[2];
    s00 += a0 * a0 + a2 * a2; s01 += a0 * a1 + a2 * a3; s11 += a1 * a1 + a3 * a3;
    r0 += a0 * b0 + a2 * b1; r1 += a1 * b0 + a3 * b1;
  }
  part[t][0] = s00; part[t][1] = s01; part[t][2] = s11; part[t][3] = r0; part[t][4] = r1;
  if (bad) atomicOr(&bad_any, 1);
  __syncthreads();
  if (t == 0) {
    double S[5] = {0, 0, 0, 0, 0};
    for (int i = 0; i < ZHANG_THREADS; i++)
#pragma unroll
      for (int j = 0; j < 5; j++) S[j] += part[i][j];
    const double det = S[0] * S[2] - S[1] * S[1];
    const double f0 = (S[2] * S[3] - S[1] * S[4]) / det, f1 = (S[0] * S[4] - S[1] * S[3]) / det;
    double fx = sqrt(fabs(1.0 / f0)), fy = sqrt(fabs(1.0 / f1));
    if (a.fix_aspect) { const double m = (fx + fy) * 0.5; fx = m; fy = m; }
    if (nv == 0 || bad_any || !(det != 0.0)) { fx = fy = nan(""); }
    double* k = a.intr + (size_t)c * a.kint;
    k[0] = fx; k[1] = fy; k[2] = cx; k[3] = cy;
    for (int i = 4; i < a.kint; i++) k[i] = 0.0;
  }
}

// cv2.fisheye.calibrate's start without an initial matrix: fx = fy = max(w, h) / 2, principal point (w/2 - 0.5, h/2 - 0.5), zero skew
// (CALIB_FIX_SKEW) and zero distortion -- what OpenCV 4.13 returns when its loop runs no iteration (DESIGN.md §3d).  It needs no view;
// one thread per camera.
__global__ void k_fisheye_k0(int C, int kint, const int32_t* image_size, double* intr) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const int w = image_size[2 * c], h = image_size[2 * c + 1];
  const double f = max(w, h) / 2.0;
  double* k = intr + (size_t)c * kint;
  k[0] = f; k[1] = f; k[2] = w / 2.0 - 0.5; k[3] = h / 2.0 - 0.5;
  for (int i = 4; i < kint; i++) k[i] = 0.0;
}

// per-view sums of squared pixel errors (u and v) and corner counts, dense over (camera, frame, board), from the per-view costs of
// k_views<MODE_COST> under the linear loss (0.5 sum, halved exactly): for the intrinsic calibration the per-view RMS sqrt(sumsq / count)
// of calibrateCameraExtended's perViewErrors; for a bundle adjustment per-(camera, frame, board) view errors
__global__ void k_view_sumsq(DeviceProblem p, const double* view_cost, double* sumsq, int64_t* count) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= p.V) return;
  const size_t o = ((size_t)p.view_cam[v] * p.F + p.view_frame[v]) * p.B + p.view_board[v];
  sumsq[o] = 2.0 * view_cost[v];
  count[o] = p.view_start[v + 1] - p.view_start[v];
}

}  // namespace mcba
