// undistort_kernels.cuh — applying a finished calibration, what the reference does with OpenCV on the host:
//   Camera.undistort_map    camera.py:113-117, camera_fisheye.py:102-106   cv2.initUndistortRectifyMap(K, dist, None, K, size, CV_32FC2)
//                                                                          / cv2.fisheye.initUndistortRectifyMap
//   undistort_images        camera.py:244-258                              cv2.remap(image, map, None, INTER_CUBIC) per image
//   Camera.undistort_points camera.py:119-122, camera_fisheye.py:108-111   cv2.undistortPoints(pts, K, dist, P=K)
//   Camera.project          camera.py:124-128, camera_fisheye.py:113-117   cv2.projectPoints(pts, 0, 0, K, dist)
//
// The undistortion map and points are the rectification ones below at R = I, P = K (k_rectify_map, k_rectify_points).  Map entries are
// fp64 in a fixed order with no fused multiply-adds (dmul/dadd below), cast to float32 at the end; the map kernel also writes the
// resident fixed-point form remap reads.
//
// Remap (k_remap_cubic): cv2.remap's fixed-point bicubic for uint8 with the constant-zero border.  X = rint(32 x), Y = rint(32 y) (ties
// to even); the 4x4 taps start at (X >> 5) - 1, (Y >> 5) - 1 and their weights are entry (Y & 31) * 32 + (X & 31) of a 32 x 32 table of
// 4 x 4 integers that sum to 2^15 (k_cubic_table).  acc = sum of tap * weight in int32 with taps outside the image counted as 0;
// out = clamp((acc + 2^14) >> 15, 0, 255).
//
// Resident map form: 6 bytes per pixel, the tap origin (X >> 5, Y >> 5) as two int16 saturated like OpenCV's CV_16SC2 map (4 bytes) and
// the table index (2 bytes).  The float map (8 bytes per pixel) is written only when the caller asks for it.
//
// Everything is integer arithmetic or fp64 / fp32 in a fixed order: repeated calls agree bit for bit.
#pragma once
#include <stdint.h>
#include <limits.h>
#include "geometry.cuh"
#include "pnp_kernels.cuh"

namespace mcba {

constexpr int UND_TAB = 32;                  // sub-pixel positions per pixel (OpenCV INTER_TAB_SIZE)
constexpr int UND_COEF_BITS = 15;            // fixed-point weights (INTER_REMAP_COEF_BITS)
constexpr int UND_TAB_ENTRIES = UND_TAB * UND_TAB;
constexpr int UND_THREADS = 256;

// rounded, unfused arithmetic: nvcc would otherwise contract a * b + c into one FMA, which rounds once instead of twice
__host__ __device__ __forceinline__ double dmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ float fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}

// cvRound of a float: nearest, ties to even; NaN and values outside int32 give INT_MIN, as the x86 conversion OpenCV uses does
__host__ __device__ __forceinline__ int round_to_int(float v) {
  if (!(v >= -2147483648.0f && v < 2147483648.0f)) return INT_MIN;
  return (int)rintf(v);
}

// OpenCV's 1-D cubic weights at sub-position x, in float32 (A = -0.75)
__host__ __device__ inline void cubic_coeffs(float x, float* c) {
  const float A = -0.75f, x1 = fadd(x, 1.0f), y = fadd(1.0f, -x);
  c[0] = fadd(fmul(fadd(fmul(fadd(fmul(A, x1), -5.0f * A), x1), 8.0f * A), x1), -4.0f * A);
  c[1] = fadd(fmul(fmul(fadd(fmul(A + 2.0f, x), -(A + 3.0f)), x), x), 1.0f);
  c[2] = fadd(fmul(fmul(fadd(fmul(A + 2.0f, y), -(A + 3.0f)), y), y), 1.0f);
  c[3] = fadd(fadd(fadd(1.0f, -c[0]), -c[1]), -c[2]);
}

// tab int32[1024][16]: entry (i, j) = rounded 2^15 * (y weights at i/32) x (x weights at j/32); a sum off 2^15 is put on one of the
// four central taps (the largest when the sum is short, the smallest when it is over), as OpenCV's initInterTab2D does.  One thread
// per entry.
__global__ void k_cubic_table(int32_t* tab) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= UND_TAB_ENTRIES) return;
  const int i = e / UND_TAB, j = e % UND_TAB;
  float cy[4], cx[4];
  cubic_coeffs(fmul((float)i, 1.0f / UND_TAB), cy);
  cubic_coeffs(fmul((float)j, 1.0f / UND_TAB), cx);
  int t[16], sum = 0;
  for (int a = 0; a < 4; a++)
    for (int b = 0; b < 4; b++) { t[4 * a + b] = round_to_int(fmul(fmul(cy[a], cx[b]), (float)(1 << UND_COEF_BITS))); sum += t[4 * a + b]; }
  const int diff = sum - (1 << UND_COEF_BITS);
  if (diff) {
    int mk = 10, Mk = 10;                     // tap (2, 2)
    for (int a = 2; a < 4; a++)
      for (int b = 2; b < 4; b++) {
        const int k = 4 * a + b;
        if (t[k] < t[mk]) mk = k;
        else if (t[k] > t[Mk]) Mk = k;
      }
    if (diff < 0) t[Mk] -= diff;
    else t[mk] -= diff;
  }
  for (int k = 0; k < 16; k++) tab[16 * e + k] = t[k];
}

// the camera of a map: [fx fy cx cy skew dist...] with the distortion padded to 14 (zeros), and the sensor tilt matrix (identity
// unless MODEL_TILTED) computed on the host
struct UndistortCamera {
  double k[5 + 14];
  double tilt[9];
  int w, h;
};

// the map entry of the normalised point (x, y): OpenCV's distortion and projection (fx, fy, cx, cy; K[0][1] unused), cast to float32
template <int MODEL>
__host__ __device__ inline void distorted_pixel(const UndistortCamera& c, double x, double y, float& mx, float& my) {
  const double fx = c.k[0], fy = c.k[1], cx = c.k[2], cy = c.k[3];
  const double* d = c.k + 5;
  double mu, mv;
  if constexpr (MODEL == MODEL_FISHEYE) {
    // cv2.fisheye.initUndistortRectifyMap: theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8), scale = theta_d / r
    const double r = sqrt(dadd(dmul(x, x), dmul(y, y)));
    const double th = atan(r);
    const double t2 = dmul(th, th), t4 = dmul(t2, t2), t6 = dmul(t4, t2), t8 = dmul(t4, t4);
    const double poly = dadd(dadd(dadd(dadd(1.0, dmul(d[0], t2)), dmul(d[1], t4)), dmul(d[2], t6)), dmul(d[3], t8));
    const double thd = dmul(th, poly);
    const double scale = r == 0.0 ? 1.0 : thd / r;
    mu = dadd(dmul(dmul(fx, x), scale), cx);
    mv = dadd(dmul(dmul(fy, y), scale), cy);
  } else {
    // cv2.initUndistortRectifyMap: rational radial term, tangential, thin prism, then the tilt's perspective division
    const double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4], k4 = d[5], k5 = d[6], k6 = d[7];
    const double s1 = d[8], s2 = d[9], s3 = d[10], s4 = d[11];
    const double x2 = dmul(x, x), y2 = dmul(y, y), r2 = dadd(x2, y2), xy2 = dmul(dmul(2.0, x), y);
    const double num = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k3, r2), k2), r2), k1), r2));
    const double den = dadd(1.0, dmul(dadd(dmul(dadd(dmul(k6, r2), k5), r2), k4), r2));
    const double kr = num / den;
    const double xd = dadd(dadd(dadd(dadd(dmul(x, kr), dmul(p1, xy2)), dmul(p2, dadd(r2, dmul(2.0, x2)))), dmul(s1, r2)), dmul(dmul(s2, r2), r2));
    const double yd = dadd(dadd(dadd(dadd(dmul(y, kr), dmul(p1, dadd(r2, dmul(2.0, y2)))), dmul(p2, xy2)), dmul(s3, r2)), dmul(dmul(s4, r2), r2));
    const double* M = c.tilt;
    const double t0 = dadd(dadd(dmul(M[0], xd), dmul(M[1], yd)), M[2]);
    const double t1 = dadd(dadd(dmul(M[3], xd), dmul(M[4], yd)), M[5]);
    const double t2 = dadd(dadd(dmul(M[6], xd), dmul(M[7], yd)), M[8]);
    const double ip = t2 != 0.0 ? 1.0 / t2 : 1.0;
    mu = dadd(dmul(dmul(fx, ip), t0), cx);
    mv = dadd(dmul(dmul(fy, ip), t1), cy);
  }
  mx = (float)mu;
  my = (float)mv;
}

// the fixed-point form of one map entry: tap origin (X >> 5, Y >> 5) saturated to int16 and packed (x low, y high), table index
__host__ __device__ __forceinline__ void fixed_point_entry(float mx, float my, uint32_t& org, uint16_t& idx) {
  const int X = round_to_int(mx * (float)UND_TAB), Y = round_to_int(my * (float)UND_TAB);
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767);
  org = (uint32_t)(uint16_t)(int16_t)sx | ((uint32_t)(uint16_t)(int16_t)sy << 16);
  idx = (uint16_t)((Y & (UND_TAB - 1)) * UND_TAB + (X & (UND_TAB - 1)));
}

struct RemapArgs {
  const uint8_t* src;          // [n][hs][ws][CN]
  uint8_t* dst;                // [n][hm][wm][CN]
  const uint32_t* org;         // [hm][wm] packed tap origin
  const uint16_t* idx;         // [hm][wm] table index
  const int32_t* tab;          // [1024][16]
  int ws, hs, wm, hm;
};

// cv2.remap(src, map, None, INTER_CUBIC) with the constant-zero border; one thread per output pixel, grid (ceil(wm / UND_THREADS), hm, n)
template <int CN>
__global__ void __launch_bounds__(UND_THREADS) k_remap_cubic(RemapArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= a.wm) return;
  const size_t p = (size_t)y * a.wm + x;
  const uint32_t o = __ldg(a.org + p);
  const int sx = (int)(int16_t)(o & 0xffffu) - 1, sy = (int)(int16_t)(o >> 16) - 1;
  const int32_t* w = a.tab + 16 * (int)__ldg(a.idx + p);
  const uint8_t* src = a.src + (size_t)blockIdx.z * a.hs * a.ws * CN;
  int acc[CN];
#pragma unroll
  for (int ch = 0; ch < CN; ch++) acc[ch] = 0;
  if (sx >= 0 && sy >= 0 && sx + 4 <= a.ws && sy + 4 <= a.hs) {
#pragma unroll
    for (int ky = 0; ky < 4; ky++) {
      const uint8_t* row = src + ((size_t)(sy + ky) * a.ws + sx) * CN;
#pragma unroll
      for (int kx = 0; kx < 4; kx++) {
        const int wk = __ldg(w + 4 * ky + kx);
#pragma unroll
        for (int ch = 0; ch < CN; ch++) acc[ch] += (int)__ldg(row + kx * CN + ch) * wk;
      }
    }
  } else if (sx < a.ws && sy < a.hs && sx + 4 > 0 && sy + 4 > 0) {       // the window overlaps the image: taps outside count as 0
#pragma unroll
    for (int ky = 0; ky < 4; ky++) {
      const int yy = sy + ky;
      if (yy < 0 || yy >= a.hs) continue;
#pragma unroll
      for (int kx = 0; kx < 4; kx++) {
        const int xx = sx + kx;
        if (xx < 0 || xx >= a.ws) continue;
        const int wk = __ldg(w + 4 * ky + kx);
        const uint8_t* px = src + ((size_t)yy * a.ws + xx) * CN;
#pragma unroll
        for (int ch = 0; ch < CN; ch++) acc[ch] += (int)__ldg(px + ch) * wk;
      }
    }
  }
  uint8_t* out = a.dst + ((size_t)blockIdx.z * a.hm * a.wm + p) * CN;
#pragma unroll
  for (int ch = 0; ch < CN; ch++) out[ch] = (uint8_t)min(max((acc[ch] + (1 << (UND_COEF_BITS - 1))) >> UND_COEF_BITS, 0), 255);
}

// cv2.projectPoints(X, rvec = 0, tvec = 0, K, dist) / cv2.fisheye.projectPoints: project<MODEL> of the camera frame point, one thread each
template <int MODEL>
__global__ void __launch_bounds__(UND_THREADS) k_project_points(UndistortCamera c, int64_t n, const double* xyz, double* uv) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double X[3] = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]};
  double u, v;
  project<MODEL, false>(X, c.k, u, v, nullptr, nullptr, nullptr, nullptr);
  uv[2 * i] = u; uv[2 * i + 1] = v;
}

// ---- rectification: initUndistortRectifyMap(K, dist, R, P) and undistortPoints(pts, K, dist, R, P) --------------------------------------
// ir = (P[:, :3] R)^-1 and rr = P[:, :3] R, both row-major fp64 from the host (its 3x3 Gaussian elimination); cam.w, cam.h are the map size.
// Undistortion (initUndistortRectifyMap(K, dist, None, K), undistortPoints(P = K)) is this at R = I, P = K.
//
// Map (k_rectify_map): OpenCV walks each row i from (x, y, w) = i * ir[1, 4, 7] + ir[2, 5, 8] in steps of ir[0, 3, 6], and the
// walk's rounding reaches the float32 map.  Pinhole (undistort.simd.hpp, 2 vectors of 4 doubles): blocks of RECT_BLOCK = 8 pixels
// start at `cur`, pixel k of a block is cur + k * step, then cur += 8 * step while a whole block is left; the last W mod 8 pixels take
// cur, then cur += step, one at a time.  x = _x * (1 / _w).  Fisheye (fisheye.cpp): one pixel at a time, cur += step, x = _x / _w, and
// _w <= 0 gives an infinite map entry.  The walk of a row is a list of entries (block starts, then tail pixels; every pixel for the
// fisheye), taken RECT_SEG at a time: three threads of the row's CTA write a segment's entries into shared memory, carrying `cur` over
// from the segment before, the CTA synchronises, every thread finishes the segment's pixels with distorted_pixel<MODEL>, and the CTA
// synchronises again before the next segment.  So a map has no width limit.
constexpr int RECT_BLOCK = 8;
constexpr int RECT_SEG = 512;                      // walk entries per segment: 12 KB of shared memory for x, y and w

struct RectifyCamera {
  UndistortCamera cam;
  double ir[9], rr[9];
};

// one CTA of UND_THREADS per map row.  fmap (float2 [h][w]) may be null.
template <int MODEL>
__global__ void __launch_bounds__(UND_THREADS) k_rectify_map(RectifyCamera c, float2* fmap, uint32_t* org, uint16_t* idx) {
  __shared__ double walk[3][RECT_SEG];
  constexpr int B = MODEL == MODEL_FISHEYE ? 1 : RECT_BLOCK;
  const int w = c.cam.w, i = blockIdx.x;
  const int nb = w / B, n = nb + (w - nb * B);           // whole blocks; walk entries
  const int r = threadIdx.x;                             // walker r < 3: 0 x, 1 y, 2 w
  double cur = r < 3 ? dadd(dmul((double)i, c.ir[3 * r + 1]), c.ir[3 * r + 2]) : 0.0;
  for (int e0 = 0; e0 < n; e0 += RECT_SEG) {
    const int e1 = min(n, e0 + RECT_SEG);
    if (r < 3) {
      const double step = c.ir[3 * r], bstep = dmul((double)B, step);
      int e = e0;
      for (; e < min(e1, nb); e++) { walk[r][e - e0] = cur; cur = dadd(cur, bstep); }
      for (; e < e1; e++) { walk[r][e - e0] = cur; cur = dadd(cur, step); }
    }
    __syncthreads();
    // entry e < nb starts the pixels e B .. e B + B - 1, entry e >= nb is the pixel nb B + e - nb
    const int j0 = min(e0, nb) * B + max(e0 - nb, 0), j1 = min(e1, nb) * B + max(e1 - nb, 0);
    for (int j = j0 + threadIdx.x; j < j1; j += blockDim.x) {
      double v[3];
      const int b = j / B, k = j - b * B;
      const int e = (b < nb ? b : nb + (j - nb * B)) - e0;
#pragma unroll
      for (int q = 0; q < 3; q++) {
        if (MODEL == MODEL_FISHEYE) v[q] = walk[q][e];
        else v[q] = b < nb ? dadd(walk[q][e], dmul((double)k, c.ir[3 * q])) : walk[q][e];
      }
      float mx, my;
      if constexpr (MODEL == MODEL_FISHEYE) {
        if (v[2] <= 0.0) {
          mx = v[0] > 0.0 ? -INFINITY : INFINITY;
          my = v[1] > 0.0 ? -INFINITY : INFINITY;
        } else {
          distorted_pixel<MODEL>(c.cam, v[0] / v[2], v[1] / v[2], mx, my);
        }
      } else {
        const double iw = 1.0 / v[2];
        distorted_pixel<MODEL>(c.cam, dmul(v[0], iw), dmul(v[1], iw), mx, my);
      }
      const size_t p = (size_t)i * w + j;
      if (fmap) { float2 f; f.x = mx; f.y = my; fmap[p] = f; }
      fixed_point_entry(mx, my, org[p], idx[p]);
    }
    __syncthreads();
  }
}

// cv2.undistortPoints(pts, K, dist, R = R, P = P) / cv2.fisheye.undistortPoints(pts, K, dist, R, P), one thread each: the normalised
// undistorted point is undistort_pixel<MODEL> under K = I after the division by the focal lengths (both exact in IEEE arithmetic), then
// OpenCV's (xx, yy, ww) = rr (x, y, 1), pixel (xx, yy) / ww.  A fisheye point whose Newton iteration fails keeps the -1e6 sentinel.
template <int MODEL>
__global__ void __launch_bounds__(UND_THREADS) k_rectify_points(RectifyCamera c, int64_t n, const double* in, double* out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double kn[5 + 14];
  kn[0] = 1.0; kn[1] = 1.0; kn[2] = 0.0; kn[3] = 0.0; kn[4] = 0.0;
  for (int d = 0; d < model_nd(MODEL); d++) kn[5 + d] = c.cam.k[5 + d];
  const double* k = c.cam.k;
  double x, y;
  undistort_pixel<MODEL>(kn, (in[2 * i] - k[2]) / k[0], (in[2 * i + 1] - k[3]) / k[1], x, y);
  if (MODEL == MODEL_FISHEYE && x == -1000000.0 && y == -1000000.0) { out[2 * i] = x; out[2 * i + 1] = y; return; }
  const double* R = c.rr;
  const double xx = R[0] * x + R[1] * y + R[2], yy = R[3] * x + R[4] * y + R[5], ww = R[6] * x + R[7] * y + R[8];
  if (MODEL == MODEL_FISHEYE) { out[2 * i] = xx / ww; out[2 * i + 1] = yy / ww; }
  else { const double iw = 1.0 / ww; out[2 * i] = xx * iw; out[2 * i + 1] = yy * iw; }
}

}  // namespace mcba
