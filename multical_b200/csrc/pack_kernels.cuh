// pack_kernels.cuh — dense point table -> packed, frame-major corner arrays, on the device.
//
// Replaces the host-side masking of the reference (`(...)[self.inliers]`, calibration.py:206, over the dense
// [C,F,B,P] table built by tables.make_point_table, tables.py:68-81) and keeps the reference's index contract:
// orig[k_internal] = rank of the corner in row-major boolean-mask order (np.argwhere(inliers)).
#pragma once
#include <stdint.h>

namespace mcba {

// one warp per view (c,f,b): number of selected points, written in canonical (c,f,b) and frame-major (f,c,b) order, and whether the
// view has any (frame-major order).  view_valid (may be null): views whose camera / frame / board pose is invalid select nothing
// (calibration.py:73-79)
__global__ void k_pack_count(const uint8_t* mask, const uint8_t* view_valid, int C, int F, int B, int P, int* cnt_can, int* cnt_fm, int* flag_fm) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= C * F * B) return;
  const int b = w % B, f = (w / B) % F, c = w / (B * F);
  const uint8_t* m = mask + (size_t)w * P;
  int n = 0;
  if (!view_valid || view_valid[w])
    for (int p = lane; p < P; p += 32) n += m[p] ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if (lane == 0) {
    const int wf = (f * C + c) * B + b;
    cnt_can[w] = n; cnt_fm[wf] = n; flag_fm[wf] = n > 0;
  }
}

// in-place exclusive scan of int32 arrays of n (+1 slot for the total) elements, one CTA per array (arrays `stride` apart)
__global__ void k_scan_exclusive(int* data_all, int n, int stride) {
  int* data = data_all + (size_t)blockIdx.x * stride;
  __shared__ int warp_sums[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, nt = blockDim.x;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += nt) {
    const int i = base + tid;
    const int v = i < n ? data[i] : 0;
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += t; }
    if (lane == 31) warp_sums[w] = s;
    __syncthreads();
    if (w == 0) {
      int ws = lane < (nt >> 5) ? warp_sums[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, ws, o); if (lane >= o) ws += t; }
      warp_sums[lane] = ws;
    }
    __syncthreads();
    const int prefix = carry + (w > 0 ? warp_sums[w - 1] : 0) + s - v;
    if (i < n) data[i] = prefix;
    __syncthreads();
    if (tid == nt - 1) carry += warp_sums[(nt >> 5) - 1];
    __syncthreads();
  }
  if (tid == 0) data[n] = carry;
}

struct PackOut {
  double2* obs; uint16_t* pid; uint32_t* orig;
  int* view_start; int* view_cam; int* view_frame; int* view_board;
  int* frame_view_start;
};

// one warp per view: scatter the selected corners to their frame-major slot; lane 0 emits the view record
// PT = double2, or float2: the reference's table keeps the dtype of the detector's corners (tables.py:15-17 fill_sparse; cv2 returns
// float32), the packed observations are f64 either way (exact)
template <typename PT>
__global__ void k_pack_scatter(const uint8_t* mask, const PT* points, int C, int F, int B, int P,
                               const int* off_can, const int* off_fm, const int* vid_fm, PackOut o) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  const int nv = C * F * B;
  if (w >= nv) return;
  const int b = w % B, f = (w / B) % F, c = w / (B * F);
  const int wf = (f * C + c) * B + b;
  if (lane == 0) {
    if (b == 0 && c == 0) o.frame_view_start[f] = vid_fm[wf];
    if (w == nv - 1) { o.frame_view_start[F] = vid_fm[nv]; o.view_start[vid_fm[nv]] = off_fm[nv]; }
  }
  const int base_fm = off_fm[wf], base_can = off_can[w];
  const int count = off_can[w + 1] - base_can;
  if (count == 0) return;
  if (lane == 0) {
    const int vid = vid_fm[wf];
    o.view_start[vid] = base_fm; o.view_cam[vid] = c; o.view_frame[vid] = f; o.view_board[vid] = b;
  }
  const uint8_t* m = mask + (size_t)w * P;
  const PT* pt = points + (size_t)w * P;
  int running = 0;
  for (int p0 = 0; p0 < P; p0 += 32) {
    const int p = p0 + lane;
    const bool on = p < P && m[p];
    const unsigned bal = __ballot_sync(0xffffffffu, on);
    if (on) {
      const int r = running + __popc(bal & ((1u << lane) - 1u));
      const PT q = pt[p];
      o.obs[base_fm + r] = make_double2((double)q.x, (double)q.y);
      o.pid[base_fm + r] = (uint16_t)p;
      o.orig[base_fm + r] = (uint32_t)(base_can + r);
    }
    running += __popc(bal);
  }
}

}  // namespace mcba
