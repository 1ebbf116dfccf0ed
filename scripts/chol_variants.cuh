// Single-CTA Cholesky variants that were measured against the shipping ones and dropped (scripts/chol_bench.cu): kept here, next to
// the micro-benchmark that times them (scripts/chol_bench.cu), not in the product's headers.
//   chol_small_body   the round-1 scheme: matrix cyclically distributed in registers, two block barriers per column
//   chol_diag_body    the 32 x 32 diagonal block by 256 threads (the product uses one warp: chol_diag_warp_body)
//   chol_v3_body      one block barrier per column with look-ahead (the product uses the rotating-register version chol_rot_body)
#pragma once
#include "lm_kernel.cuh"
namespace mcba {

// reduced solve, n_s <= CHOL_SMALL_MAX: one CTA, matrix cyclically distributed in registers (the round-1 k_chol_small scheme)
template <int R>
__device__ __forceinline__ void chol_small_body(int n, const double* Sg, const double* rhs, const double* gh, double reg, int* chol_fail, double* out, double* shm) {
  const int ld = n | 1;
  double* Lm = shm;
  double* colbuf = Lm + (size_t)n * ld;
  double* invd = colbuf + n;
  double* piv = invd + n;
  const int tid = threadIdx.x, ty = tid & 15, tx = tid >> 4;
  double a[R][R];
#pragma unroll
  for (int p = 0; p < R; p++)
#pragma unroll
    for (int q = 0; q < R; q++) {
      const int i = ty + 16 * p, j = tx + 16 * q;
      a[p][q] = (i < n && j < n) ? __ldcg(&Sg[(size_t)j * n + i]) + (i == j ? reg : 0.0) : 0.0;
    }
  __syncthreads();
  if (tid == 0) piv[0] = a[0][0];
  __syncthreads();
  for (int k = 0; k < n; k++) {
    const int kq = k >> 4, kt = k & 15;
    if (tx == kt) {
      const double akk = piv[0];
      if (ty == kt && !(akk > 0.0)) *chol_fail += 1;
      const double rs = rsqrt(fmax(akk, 1e-300));
      if (ty == kt) invd[k] = rs;
#define MCBA_SCALE_Q(Q) case Q: if constexpr (Q < R) { _Pragma("unroll") for (int p = 0; p < R; p++) { const int i = ty + 16 * p; \
        if (i >= k && i < n) { const double l = a[p][Q < R ? Q : 0] * rs; a[p][Q < R ? Q : 0] = l; colbuf[i] = l; } } } break;
      switch (kq) { MCBA_SCALE_Q(0) MCBA_SCALE_Q(1) MCBA_SCALE_Q(2) MCBA_SCALE_Q(3) MCBA_SCALE_Q(4) MCBA_SCALE_Q(5) MCBA_SCALE_Q(6) MCBA_SCALE_Q(7) }
#undef MCBA_SCALE_Q
    }
    __syncthreads();
    double ci[R], cj[R];
#pragma unroll
    for (int p = 0; p < R; p++) { const int i = ty + 16 * p; ci[p] = (i > k && i < n) ? colbuf[i] : 0.0; }
#pragma unroll
    for (int q = 0; q < R; q++) { const int j = tx + 16 * q; cj[q] = (j > k && j < n) ? colbuf[j] : 0.0; }
#pragma unroll
    for (int p = 0; p < R; p++)
#pragma unroll
      for (int q = 0; q < R; q++) a[p][q] -= ci[p] * cj[q];
    {
      const int k1 = k + 1, q1 = k1 >> 4, t1 = k1 & 15;
      if (k1 < n && ty == t1 && tx == t1) {
#pragma unroll
        for (int p = 0; p < R; p++) if (p == q1) piv[0] = a[p][p];
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int p = 0; p < R; p++)
#pragma unroll
    for (int q = 0; q < R; q++) {
      const int i = ty + 16 * p, j = tx + 16 * q;
      if (i < n && j <= i) Lm[i * ld + j] = a[p][q];
    }
  __syncthreads();
  if (tid < 32) {
    constexpr int RS = (R * 16 + 31) / 32;
    const int lane = tid;
    double bs[RS];
#pragma unroll
    for (int s2 = 0; s2 < RS; s2++) { const int i = lane + 32 * s2; bs[s2] = i < n ? __ldcg(&rhs[i]) + gh[i] : 0.0; }
#pragma unroll
    for (int s1 = 0; s1 < RS; s1++) {
      for (int kk = 0; kk < 32; kk++) {
        const int k = 32 * s1 + kk;
        if (k >= n) break;
        const double yk = __shfl_sync(0xffffffffu, bs[s1] * invd[k], kk);
        if (lane == kk) bs[s1] = yk;
#pragma unroll
        for (int s2 = s1; s2 < RS; s2++) { const int i = lane + 32 * s2; if (i > k && i < n) bs[s2] -= Lm[i * ld + k] * yk; }
      }
    }
#pragma unroll
    for (int s1 = RS - 1; s1 >= 0; s1--) {
      for (int kk = 31; kk >= 0; kk--) {
        const int k = 32 * s1 + kk;
        if (k >= n) continue;
        const double xk = __shfl_sync(0xffffffffu, bs[s1] * invd[k], kk);
        if (lane == kk) bs[s1] = xk;
#pragma unroll
        for (int s2 = 0; s2 <= s1; s2++) { const int i = lane + 32 * s2; if (i < k) bs[s2] -= Lm[k * ld + i] * xk; }
      }
    }
#pragma unroll
    for (int s2 = 0; s2 < RS; s2++) { const int i = lane + 32 * s2; if (i < n) out[i] = bs[s2]; }
  }
  __syncthreads();
}

__device__ __forceinline__ void chol_diag_body(int n, int kb, double* S, double* Linv_all, int* chol_fail, double* sh) {
  double (*Lm)[CHOL_NB + 1] = reinterpret_cast<double (*)[CHOL_NB + 1]>(sh);
  double* colbuf = sh + CHOL_NB * (CHOL_NB + 1);
  double* invd = colbuf + CHOL_NB;
  double* piv = invd + CHOL_NB;
  const int nb = min(CHOL_NB, n - kb);
  const int tid = threadIdx.x, ty = tid & 15, tx = tid >> 4;
  double a[2][2];
  __syncthreads();                       // the block may just have been updated by this CTA (look-ahead tile of the previous panel)
#pragma unroll
  for (int p = 0; p < 2; p++)
#pragma unroll
    for (int q = 0; q < 2; q++) {
      const int i = ty + 16 * p, j = tx + 16 * q;
      a[p][q] = (i < nb && j < nb) ? (j <= i ? __ldcg(&S[(size_t)(kb + i) * n + kb + j]) : __ldcg(&S[(size_t)(kb + j) * n + kb + i])) : (i == j ? 1.0 : 0.0);
    }
  __syncthreads();
  if (tid == 0) piv[0] = a[0][0];
  __syncthreads();
  for (int k = 0; k < CHOL_NB; k++) {
    const int kq = k >> 4, kt = k & 15;
    if (tx == kt) {
      const double akk = piv[0];
      if (ty == kt && k < nb && !(akk > 0.0)) *chol_fail += 1;
      const double rs = fast_rsqrt(fmin(fmax(akk, 1e-30), 1e30));
      if (ty == kt) invd[k] = rs;
#pragma unroll
      for (int p = 0; p < 2; p++) {
        const int i = ty + 16 * p;
        if (i >= k) {
          if (kq == 0) { const double l = a[p][0] * rs; a[p][0] = l; colbuf[i] = l; }
          else { const double l = a[p][1] * rs; a[p][1] = l; colbuf[i] = l; }
        }
      }
    }
    __syncthreads();
    double ci[2], cj[2];
#pragma unroll
    for (int p = 0; p < 2; p++) { const int i = ty + 16 * p; ci[p] = i > k ? colbuf[i] : 0.0; }
#pragma unroll
    for (int q = 0; q < 2; q++) { const int j = tx + 16 * q; cj[q] = j > k ? colbuf[j] : 0.0; }
#pragma unroll
    for (int p = 0; p < 2; p++)
#pragma unroll
      for (int q = 0; q < 2; q++) a[p][q] -= ci[p] * cj[q];
    {
      const int k1 = k + 1, q1 = k1 >> 4, t1 = k1 & 15;
      if (k1 < CHOL_NB && ty == t1 && tx == t1) piv[0] = q1 == 0 ? a[0][0] : a[1][1];
    }
    __syncthreads();
  }
#pragma unroll
  for (int p = 0; p < 2; p++)
#pragma unroll
    for (int q = 0; q < 2; q++) {
      const int i = ty + 16 * p, j = tx + 16 * q;
      Lm[i][j] = j <= i ? a[p][q] : 0.0;
      if (i < nb && j <= i) S[(size_t)(kb + i) * n + kb + j] = a[p][q];
    }
  __syncthreads();
  if (tid < CHOL_NB) {
    const int j = tid;
    double z[CHOL_NB];
#pragma unroll
    for (int i = 0; i < CHOL_NB; i++) {
      double t = (i == j) ? 1.0 : 0.0;
#pragma unroll
      for (int k2 = 0; k2 < CHOL_NB; k2++) if (k2 < i) t -= Lm[i][k2] * z[k2];
      z[i] = (i >= j) ? t * invd[i] : 0.0;
    }
    double* Li = Linv_all + (size_t)(kb / CHOL_NB) * CHOL_NB * CHOL_NB;
#pragma unroll
    for (int i = 0; i < CHOL_NB; i++) Li[i * CHOL_NB + j] = z[i];
  }
  __syncthreads();
}
// ---- reduced solve, n <= CHOL_V3_MAX: one CTA, ONE block barrier per column.  Warp w owns the columns j == w (mod 8), lane l the rows
// i == l (mod 32); the matrix lives in registers (a[q][r] = A[l + 32 r][w + 8 q]).  Per column k: every thread applies the rank-1
// update of the scaled column k (read from shared memory), but the warp that owns column k+1 updates THAT column first, takes its
// pivot, scales it and publishes it in the other half of the double-buffered column store -- so the next step can start right after
// the barrier (look-ahead), and the remaining updates are off the critical path.  The right-hand side rides along as row n (forward
// substitution for free); the backward substitution is done by warp 0 from the factor in shared memory.
constexpr int CHOL_V3_MAX = 127;
__host__ __device__ inline size_t chol_v3_smem_doubles(int n) { return (size_t)n * (n | 1) + 2 * 160 + 160; }
template <int CQ>
__device__ __forceinline__ void chol_v3_body(int n, const double* Sg, const double* rhs, const double* gh, double reg, int* chol_fail, double* out, double* shm) {
  const int ld = n | 1;
  double* Lm = shm;                                   // [n][ld] factor, written at the end
  double* colbuf = Lm + (size_t)n * ld;               // [2][160] scaled columns (rows 0..n)
  double* invd = colbuf + 2 * 160;                    // [160] 1 / L_kk
  const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
  double a[CQ][4];
#pragma unroll
  for (int q = 0; q < CQ; q++)
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int i = l + 32 * r, j = w + 8 * q;
      double v = 0.0;
      if (j < n) {
        if (i < n) { if (i >= j) v = __ldcg(&Sg[(size_t)i * n + j]) + (i == j ? reg : 0.0); }
        else if (i == n) v = __ldcg(&rhs[j]) + gh[j];
      }
      a[q][r] = v;
    }
  // scale column k (held in slot q of this warp) and publish it in colbuf[buf]: executed by the owning warp only (warp-uniform)
#define V3_SCALE_CASE(Q) case Q: if constexpr (Q < CQ) { \
    const double pv = rk == 0 ? a[Q < CQ ? Q : 0][0] : rk == 1 ? a[Q < CQ ? Q : 0][1] : rk == 2 ? a[Q < CQ ? Q : 0][2] : a[Q < CQ ? Q : 0][3]; \
    const double piv = __shfl_sync(0xffffffffu, pv, lk); \
    if (l == 0 && !(piv > 0.0)) *chol_fail += 1; \
    const double rs = rsqrt(fmax(piv, 1e-300)); \
    if (l == 0) invd[k1] = rs; \
    _Pragma("unroll") for (int r = 0; r < 4; r++) { const int i = l + 32 * r; if (i >= k1 && i <= n) { const double v = a[Q < CQ ? Q : 0][r] * rs; a[Q < CQ ? Q : 0][r] = v; cb[i] = v; } } } break;
#define V3_UPDATE_CASE(Q) case Q: if constexpr (Q < CQ) { _Pragma("unroll") for (int r = 0; r < 4; r++) a[Q < CQ ? Q : 0][r] -= ci[r] * cjn; } break;
  {
    __syncthreads();
    if (w == 0) {
      const int k1 = 0, rk = 0, lk = 0; double* cb = colbuf;
      switch (0) { V3_SCALE_CASE(0) }
    }
    __syncthreads();
  }
  for (int k = 0; k < n; k++) {
    const double* cur = colbuf + (k & 1) * 160;
    double ci[4];
#pragma unroll
    for (int r = 0; r < 4; r++) { const int i = l + 32 * r; ci[r] = (i > k && i <= n) ? cur[i] : 0.0; }
    const int k1 = k + 1;
    const int q1 = k1 >> 3;
    const bool owner = k1 < n && (k1 & 7) == w;
    if (owner) {
      // look-ahead: column k+1 first, then its pivot / scaling / publication
      const double cjn = cur[k1];
      switch (q1) { V3_UPDATE_CASE(0) V3_UPDATE_CASE(1) V3_UPDATE_CASE(2) V3_UPDATE_CASE(3) V3_UPDATE_CASE(4) V3_UPDATE_CASE(5) V3_UPDATE_CASE(6) V3_UPDATE_CASE(7)
                    V3_UPDATE_CASE(8) V3_UPDATE_CASE(9) V3_UPDATE_CASE(10) V3_UPDATE_CASE(11) V3_UPDATE_CASE(12) V3_UPDATE_CASE(13) V3_UPDATE_CASE(14) V3_UPDATE_CASE(15) }
      const int rk = k1 >> 5, lk = k1 & 31; double* cb = colbuf + (k1 & 1) * 160;
      switch (q1) { V3_SCALE_CASE(0) V3_SCALE_CASE(1) V3_SCALE_CASE(2) V3_SCALE_CASE(3) V3_SCALE_CASE(4) V3_SCALE_CASE(5) V3_SCALE_CASE(6) V3_SCALE_CASE(7)
                    V3_SCALE_CASE(8) V3_SCALE_CASE(9) V3_SCALE_CASE(10) V3_SCALE_CASE(11) V3_SCALE_CASE(12) V3_SCALE_CASE(13) V3_SCALE_CASE(14) V3_SCALE_CASE(15) }
    }
    // the other columns j > k of this warp (column k+1 is done if this warp owns it)
#pragma unroll
    for (int q = 0; q < CQ; q++) {
      const int j = w + 8 * q;
      if (j > k && j < n && !(owner && q == q1)) {
        const double cj = cur[j];
#pragma unroll
        for (int r = 0; r < 4; r++) a[q][r] -= ci[r] * cj;
      }
    }
    __syncthreads();
  }
#undef V3_SCALE_CASE
#undef V3_UPDATE_CASE
  // factor -> shared memory (lower triangle incl. the diagonal), y = row n
#pragma unroll
  for (int q = 0; q < CQ; q++)
#pragma unroll
    for (int r = 0; r < 4; r++) {
      const int i = l + 32 * r, j = w + 8 * q;
      if (j < n && i < n && i >= j) Lm[i * ld + j] = a[q][r];
      if (j < n && i == n) colbuf[j] = a[q][r];          // y = L^-1 b
    }
  __syncthreads();
  if (tid < 32) {
    constexpr int RS = 4;
    const int lane = tid;
    double bs[RS];
#pragma unroll
    for (int s2 = 0; s2 < RS; s2++) { const int i = lane + 32 * s2; bs[s2] = i < n ? colbuf[i] : 0.0; }
    // backward: L^T x = y
#pragma unroll
    for (int s1 = RS - 1; s1 >= 0; s1--) {
      for (int kk = 31; kk >= 0; kk--) {
        const int k = 32 * s1 + kk;
        if (k >= n) continue;
        const double xk = __shfl_sync(0xffffffffu, bs[s1] * invd[k], kk);
        if (lane == kk) bs[s1] = xk;
#pragma unroll
        for (int s2 = 0; s2 <= s1; s2++) { const int i = lane + 32 * s2; if (i < k) bs[s2] -= Lm[k * ld + i] * xk; }
      }
    }
#pragma unroll
    for (int s2 = 0; s2 < RS; s2++) { const int i = lane + 32 * s2; if (i < n) out[i] = bs[s2]; }
  }
  __syncthreads();
}

}  // namespace mcba
