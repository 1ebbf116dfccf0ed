// table_kernels.cuh — the resident point table: detection lists -> dense table, error statistics and outlier
// rejection on the device.
//
// The reference keeps the [C,F,B,P] table in numpy and re-masks it on the host around every bundle adjustment:
//   tables.make_point_table / fill_sparse   tables.py:15-21,68-81     -> k_table_fill
//   tables.reprojection_error               tables.py:244-249         -> k_views<MODE_ERROR> (kernels.cuh)
//   Calibration.reject_outliers             calibration.py:240-252    -> k_table_reject
//   error_stats (mse over valid / inliers)  calibration.py:303-310    -> k_table_stats
// All kernels here are one warp per packed view of the VALID selection; they are HBM-streaming byte/double work
// (17 B of table per corner), so the only design rules are coalesced lane-strided access and a grid that covers the SMs.
#pragma once
#include <stdint.h>
#include <math.h>

namespace mcba {

constexpr int TABLE_WARPS = 8;

// one warp per detection list w = (c*F+f)*B+b: dense[ids] = corners, mask[ids] = true (tables.py:15-21)
__global__ void k_table_fill(const int64_t* det_start, const int32_t* det_ids, const double2* det_xy, int nv, int P,
                             uint8_t* mask, double2* points, int* bad) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= nv) return;
  const int64_t beg = det_start[w], end = det_start[w + 1];
  for (int64_t i = beg + lane; i < end; i += 32) {
    const int id = det_ids[i];
    if (id < 0 || id >= P) { atomicExch(bad, 1); continue; }
    mask[(size_t)w * P + id] = 1;
    points[(size_t)w * P + id] = det_xy[i];
  }
}

__global__ void k_mask_and(const uint8_t* a, const uint8_t* b, size_t n, uint8_t* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (a[i] && b[i]) ? 1 : 0;
}

// Over the packed VALID selection: err[] holds the pixel error of every valid corner in canonical (boolean-mask) order.
//   err_inl[o]  = error if the corner is in the inlier mask, +inf otherwise (sorted afterwards: inliers come first)
//   part[v]     = { sum e^2 over the view, sum e^2 over its inliers, number of its inliers }   (summed by k_sum_partials)
__global__ void __launch_bounds__(TABLE_WARPS * 32)
k_table_stats(DeviceProblem p, const double* err, const uint8_t* inl, double* err_inl, double* part) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * TABLE_WARPS + (threadIdx.x >> 5), nw = gridDim.x * TABLE_WARPS;
  for (int v = gw; v < p.V; v += nw) {
    const int c = p.view_cam[v], f = p.view_frame[v], b = p.view_board[v];
    const size_t dense0 = ((size_t)(c * p.F + f) * p.B + b) * p.P;
    double s_all = 0.0, s_in = 0.0, n_in = 0.0;
    for (int idx = p.view_start[v] + lane; idx < p.view_start[v + 1]; idx += 32) {
      const uint32_t o = p.orig[idx];
      const double e = err[o];
      const bool on = inl[dense0 + p.pid[idx]] != 0;
      err_inl[o] = on ? e : INFINITY;
      s_all += e * e;
      if (on) { s_in += e * e; n_in += 1.0; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s_all += __shfl_xor_sync(0xffffffffu, s_all, o);
      s_in += __shfl_xor_sync(0xffffffffu, s_in, o);
      n_in += __shfl_xor_sync(0xffffffffu, n_in, o);
    }
    if (lane == 0) { part[3 * (size_t)v] = s_all; part[3 * (size_t)v + 1] = s_in; part[3 * (size_t)v + 2] = n_in; }
  }
}

// inliers = (errors < threshold) & valid (calibration.py:243-244).  `inl` was cleared beforehand, so the entries outside
// `valid` stay 0; part[v] = corners of the view that were kept.
__global__ void __launch_bounds__(TABLE_WARPS * 32)
k_table_reject(DeviceProblem p, const double* err, double threshold, uint8_t* inl, double* part) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * TABLE_WARPS + (threadIdx.x >> 5), nw = gridDim.x * TABLE_WARPS;
  for (int v = gw; v < p.V; v += nw) {
    const int c = p.view_cam[v], f = p.view_frame[v], b = p.view_board[v];
    const size_t dense0 = ((size_t)(c * p.F + f) * p.B + b) * p.P;
    double kept = 0.0;
    for (int idx = p.view_start[v] + lane; idx < p.view_start[v + 1]; idx += 32) {
      const bool keep = err[p.orig[idx]] < threshold;        // NaN compares false: rejected, as in numpy
      inl[dense0 + p.pid[idx]] = keep ? 1 : 0;
      kept += keep ? 1.0 : 0.0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
    if (lane == 0) part[v] = kept;
  }
}

__global__ void k_gather_ranks(const double* sorted, const int64_t* ranks, int n, double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = sorted[ranks[i]];
}

// out[i] = number of entries of sorted[0, count) that are < thresholds[i] (lower bound): with k_gather_ranks this is all a
// multi-rank quantile needs from each rank's sorted error vector (multical_b200/distributed.py merged_order_statistics)
__global__ void k_count_below(const double* sorted, int64_t count, const double* thresholds, int n, int64_t* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double t = thresholds[i];
  int64_t lo = 0, hi = count;
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (sorted[mid] < t) lo = mid + 1; else hi = mid; }
  out[i] = lo;
}

}  // namespace mcba
