// stereo_kernels.cuh — the start of stereo calibration (stereo_calibrate, camera.py:261-286 -> cv2.stereoCalibrate; the fisheye twin
// camera_fisheye.py:180-205 -> cv2.fisheye.stereoCalibrate).
//
//   (the per-view poses of both cameras are k_pnp_views, pnp_kernels.cuh, under the cameras' own intrinsics, in one launch)
//   k_stereo_start   one CTA: for every view where both poses are valid the relative pose R = R2 R1^T, T = T2 - R T1 and its rotation
//                    vector; then OpenCV's start, the median of each of the 6 components over those views (the two middle values
//                    averaged for an even count)
//
// The medians come from ranks, not from a parallel sort: the value of view i goes to position #{usable j : v_j < v_i, or v_j == v_i
// and j < i}.  No floating-point sum is involved, so two identical calls agree bit for bit whatever the thread schedule.
#pragma once
#include <stdint.h>
#include "geometry.cuh"

namespace mcba {

constexpr int STEREO_THREADS = 256;

struct StereoStartArgs {
  int F;
  const double* poses;          // [2][F][16] board wrt camera (k_pnp_views over lists w = c*F + f, one board)
  const uint8_t* ok;            // [2][F]
  double* rel;                  // scratch [6][F]: the relative rtvec of view f, component-major
  double* sorted;               // scratch [6][F]: each component's usable values in ascending order
  double* rt0;                  // [6] the start (NaN without a usable view)
  uint8_t* both;                // [F] both poses of the view are valid
};

__global__ void __launch_bounds__(STEREO_THREADS)
k_stereo_start(StereoStartArgs a) {
  const int F = a.F;
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    const bool use = a.ok[f] && a.ok[F + f];
    a.both[f] = use ? 1 : 0;
    if (!use) continue;
    const double* T1 = a.poses + (size_t)16 * f;
    const double* T2 = a.poses + (size_t)16 * ((size_t)F + f);
    // R = R2 R1^T, T = T2 - R T1 as a 4x4 (row-major, last row unused)
    double T[16];
#pragma unroll
    for (int i = 0; i < 3; i++) {
#pragma unroll
      for (int j = 0; j < 3; j++) T[4 * i + j] = T2[4 * i] * T1[4 * j] + T2[4 * i + 1] * T1[4 * j + 1] + T2[4 * i + 2] * T1[4 * j + 2];
    }
#pragma unroll
    for (int i = 0; i < 3; i++) T[4 * i + 3] = T2[4 * i + 3] - (T[4 * i] * T1[3] + T[4 * i + 1] * T1[7] + T[4 * i + 2] * T1[11]);
    double rt[6];
    matrix_to_rtvec(T, rt);
#pragma unroll
    for (int k = 0; k < 6; k++) a.rel[(size_t)k * F + f] = rt[k];
  }
  __syncthreads();
  __shared__ int count[STEREO_THREADS];
  int mine = 0;
  for (int f = threadIdx.x; f < F; f += blockDim.x) mine += a.both[f];
  count[threadIdx.x] = mine;
  __syncthreads();
  int n = 0;
  for (int t = 0; t < (int)blockDim.x; t++) n += count[t];
  for (int e = threadIdx.x; e < 6 * F; e += blockDim.x) {
    const int k = e / F, i = e % F;
    if (!a.both[i]) continue;
    const double* v = a.rel + (size_t)k * F;
    const double vi = v[i];
    int rank = 0;
    for (int j = 0; j < F; j++) rank += (a.both[j] && (v[j] < vi || (v[j] == vi && j < i))) ? 1 : 0;
    a.sorted[(size_t)k * F + rank] = vi;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    const double* s = a.sorted + (size_t)threadIdx.x * F;
    a.rt0[threadIdx.x] = n == 0 ? nan("") : (n % 2 ? s[n / 2] : (s[n / 2 - 1] + s[n / 2]) * 0.5);
  }
}

}  // namespace mcba
