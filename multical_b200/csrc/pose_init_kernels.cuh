// pose_init_kernels.cuh — the pose-graph initialisation of tables.initialise_poses (tables.py:354-377) on the device.
//
// Every call of the reference's align_transforms_robust (transform/matrix.py:140-153) is one item: a run of rows (m1, m2, mask)
//   m    = mean_robust(m2[mask] @ inv(m1[mask]))
//   errs = |m @ m1 - m2|_F over all rows;  inliers = (errs < 1.5 np.quantile(errs, 0.75)) & mask
//   t    = mean_robust(m2[inliers] @ inv(m1[inliers]))
// with mean_robust (transform/common.py:6-19) = mean of the largest cluster of
//   fcluster(linkage(whiten(rtvecs), 'ward'), t = max(n // 10, 3), 'maxclust'), ties to the cluster holding the lowest row.
// k_pose_gather forms the rows of every item from the uploaded table (the relative poses of estimate_transform, the inverted table of
// estimate_relative_poses_inv, the camera poses broadcast over the boards of relative_between_inv); k_pose_align runs one item per CTA.
//
// Ward clustering without a distance matrix: parallel reciprocal nearest neighbours on centroids and sizes.  Each round every stale
// cluster finds its nearest neighbour (Ward distance sqrt(2ab/(a+b)) |c_A - c_B|, ties to the lower index) and every reciprocal pair
// merges.  Ward is reducible, so only clusters that merged or whose neighbour merged need a new search.  The merge of cluster j into
// i is recorded at j (par[j] = i, height hj[j]); heights are monotone along the tree, so the maxclust cut is "every merge with a height
// <= the (n - t)-th smallest" -- scipy's own rule (cluster_maxclust_monocrit), ties included -- and the cluster labels are the roots of
// the merges kept.  Working memory is O(n).
//
// Two size classes, by item rows R: up to PI_SMALL_MAX rows the whole working set (PI_ROW_BYTES a row) lives in shared memory, 256
// threads per CTA; above it the working set lives in global memory (L2-resident) and the neighbour search tiles the candidates
// through shared memory, 512 threads per CTA.  Every sum runs in a fixed order: two identical calls agree bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "geometry.cuh"

namespace mcba {

enum { PI_ROW_PAIR = 0 /* m1 = T[a], m2 = T[b] */, PI_ROW_PAIR_INV = 1 /* m1 = inv(T[a]), m2 = inv(T[b]) */,
       PI_ROW_FRAME = 2 /* view a = (c, f, b): m1 = inv(cam[c]), m2 = inv(T[a] inv(board[b])) */ };
constexpr int PI_SMALL_MAX = 1024;                 // rows: 1024 x PI_ROW_BYTES = 152 KiB of shared memory
constexpr int PI_SMALL_THREADS = 256, PI_LARGE_THREADS = 512, PI_TILE = 512;
constexpr int PI_ROW_BYTES = 15 * 8 + 8 * 4;       // x 6, cen 6, sz, nnw, hj doubles; 8 int arrays

struct PoseRow { int32_t kind, a, b, pad; };

struct PoseAlignArgs {
  int C, F, B;
  const double* poses; const uint8_t* valid;       // [C*F*B][4][4], [C*F*B]
  const double* cam; const double* board;          // [C][4][4], [B][4][4] (PI_ROW_FRAME)
  const PoseRow* rows; int64_t n_rows;
  double* m1; double* m2; uint8_t* mask;           // gathered rows: [n_rows][3][4] twice, [n_rows]
  const int64_t* row_start;                        // [items + 1]
  const int32_t* items;                            // the items of this launch
  const double* vecs;                              // cluster-only: [n_rows][6] -> inl = mask of the largest cluster
  char* work;                                      // large items: PI_ROW_BYTES per row, at row_start
  double* t;                                       // [items][4][4]
  uint8_t* inl;                                    // [n_rows]
  int32_t* n_inl;                                  // [items]
};

struct ClusterWork {
  double *x, *cen, *sz, *nnw, *hj;
  int *idx, *nn, *alive, *alive2, *par, *mround, *slist, *cnt;
};

__host__ __device__ inline ClusterWork pi_carve(char* p, int R) {
  ClusterWork w;
  double* d = (double*)p;
  w.x = d; w.cen = d + 6 * (size_t)R; w.sz = d + 12 * (size_t)R; w.nnw = d + 13 * (size_t)R; w.hj = d + 14 * (size_t)R;
  int* i = (int*)(d + 15 * (size_t)R);
  w.idx = i; w.nn = i + R; w.alive = i + 2 * R; w.alive2 = i + 3 * R; w.par = i + 4 * R; w.mround = i + 5 * R; w.slist = i + 6 * R;
  w.cnt = i + 7 * R;
  return w;
}

// 3x4 blocks of row-major 4x4 poses (last row [0 0 0 1])
__host__ __device__ inline void pi_inv34(const double* A, double* O) {
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) O[4 * i + j] = A[4 * j + i];
  for (int i = 0; i < 3; i++) O[4 * i + 3] = -(O[4 * i] * A[3] + O[4 * i + 1] * A[7] + O[4 * i + 2] * A[11]);
}
__host__ __device__ inline void pi_mul34(const double* A, const double* B, double* O) {
  for (int i = 0; i < 3; i++) {
    for (int j = 0; j < 4; j++) O[4 * i + j] = A[4 * i] * B[j] + A[4 * i + 1] * B[4 + j] + A[4 * i + 2] * B[8 + j];
    O[4 * i + 3] += A[4 * i + 3];
  }
}

__global__ void k_pose_gather(PoseAlignArgs a) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < a.n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    const PoseRow d = a.rows[r];
    double A[12], B[12], T[12];
    uint8_t ok = 1;
    if (d.kind == PI_ROW_FRAME) {
      const int FB = a.F * a.B, c = d.a / FB, b = d.a % a.B;
      pi_inv34(a.cam + 16 * (size_t)c, A);
      pi_inv34(a.poses + 16 * (size_t)d.a, T);
      pi_mul34(a.board + 16 * (size_t)b, T, B);
    } else {
      const double* P = a.poses + 16 * (size_t)d.a; const double* Q = a.poses + 16 * (size_t)d.b;
      if (d.kind == PI_ROW_PAIR_INV) { pi_inv34(P, A); pi_inv34(Q, B); }
      else for (int k = 0; k < 12; k++) { A[k] = P[k]; B[k] = Q[k]; }
      ok = a.valid[d.a] && a.valid[d.b];
    }
    for (int k = 0; k < 12; k++) { a.m1[12 * r + k] = A[k]; a.m2[12 * r + k] = B[k]; }
    a.mask[r] = ok;
  }
}

// ---- block primitives (NT threads, every thread calls) ---------------------------------------------------------------------------
template <int NT>
__device__ int pi_scan(int v, int& total) {      // exclusive prefix sum of v over the block
  __shared__ int ws[NT / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) ws[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int s = lane < NT / 32 ? ws[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
    if (lane < NT / 32) ws[lane] = s;
  }
  __syncthreads();
  const int excl = x - v + (wid ? ws[wid - 1] : 0);
  total = ws[NT / 32 - 1];
  __syncthreads();
  return excl;
}

// stable compaction of positions [0, m) that satisfy pred: emit(position, output slot); returns the count
template <int NT, class Pred, class Emit>
__device__ int pi_compact(int m, Pred pred, Emit emit) {
  int base = 0;
  for (int c0 = 0; c0 < m; c0 += NT) {
    const int k = c0 + threadIdx.x;
    const bool p = k < m && pred(k);
    int tot;
    const int pos = pi_scan<NT>(p ? 1 : 0, tot);
    if (p) emit(k, base + pos);
    base += tot;
  }
  __syncthreads();
  return base;
}

template <int NT>
__device__ double pi_sum(double v) {             // fixed-order tree: bit-reproducible for a fixed NT
  __shared__ double s[NT];
  s[threadIdx.x] = v;
  __syncthreads();
  for (int h = NT / 2; h > 0; h >>= 1) { if ((int)threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h]; __syncthreads(); }
  const double r = s[0];
  __syncthreads();
  return r;
}

__device__ __forceinline__ unsigned long long pi_bits(double v) { unsigned long long u; memcpy(&u, &v, 8); return u; }

// k-th smallest (0-based) of v[0, n), all >= 0 (their bit patterns order like the values): radix select, 8 bits a pass
template <int NT>
__device__ double pi_select(const double* v, int n, int k) {
  __shared__ unsigned hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k;
  unsigned long long prefix = 0, pmask = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += NT) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += NT) {
      const unsigned long long u = pi_bits(v[i]);
      if ((u & pmask) == prefix) atomicAdd(&hist[(u >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int kk = k, dg = 0;
      for (; dg < 255; dg++) { if (kk < (int)hist[dg]) break; kk -= (int)hist[dg]; }
      s_prefix = prefix | ((unsigned long long)dg << shift); s_k = kk;
    }
    __syncthreads();
    prefix = s_prefix; k = s_k; pmask |= 255ull << shift;
    __syncthreads();
  }
  double r; memcpy(&r, &prefix, 8);
  return r;
}

// nearest neighbour (Ward distance, ties to the lower index) of each of the ns clusters in slist among the m alive ones.  G lanes share
// a cluster when there are few; large items load the candidates tile by tile into shared memory.
template <int NT, bool LARGE>
__device__ void pi_search(const ClusterWork& w, const int* al, int m, int ns) {
  __shared__ double tc[LARGE ? PI_TILE * 7 : 1];
  __shared__ int ti[LARGE ? PI_TILE : 1];
  int G = 32;
  while (G > 1 && NT / G < ns) G >>= 1;
  const int groups = NT / G, g = threadIdx.x % G;
  for (int base = 0; base < ns; base += groups) {
    const int s = base + threadIdx.x / G;
    const bool have = s < ns;
    const int i = have ? w.slist[s] : -1;
    double ci[6], si = 1.0;
    for (int c = 0; c < 6; c++) ci[c] = have ? w.cen[6 * i + c] : 0.0;
    if (have) si = w.sz[i];
    double bw = INFINITY; int bj = -1;
    auto consider = [&](int j, const double* cj, double sj) {
      if (j == i) return;
      double d2 = 0.0;
      for (int c = 0; c < 6; c++) { const double d = ci[c] - cj[c]; d2 += d * d; }
      const double wv = si * sj / (si + sj) * d2;
      if (wv < bw || (wv == bw && j < bj)) { bw = wv; bj = j; }
    };
    if constexpr (LARGE) {
      for (int t0 = 0; t0 < m; t0 += PI_TILE) {
        const int tn = min(PI_TILE, m - t0);
        __syncthreads();
        for (int k = threadIdx.x; k < tn; k += NT) {
          const int j = al[t0 + k];
          ti[k] = j;
          for (int c = 0; c < 6; c++) tc[7 * k + c] = w.cen[6 * j + c];
          tc[7 * k + 6] = w.sz[j];
        }
        __syncthreads();
        if (have) for (int k = g; k < tn; k += G) consider(ti[k], tc + 7 * k, tc[7 * k + 6]);
      }
    } else {
      if (have) for (int k = g; k < m; k += G) { const int j = al[k]; consider(j, w.cen + 6 * j, w.sz[j]); }
    }
    for (int o = G / 2; o > 0; o >>= 1) {
      const double ow = __shfl_xor_sync(0xffffffffu, bw, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (oj >= 0 && (bj < 0 || ow < bw || (ow == bw && oj < bj))) { bw = ow; bj = oj; }
    }
    if (have && g == 0) { w.nn[i] = bj; w.nnw[i] = bw; }
  }
  __syncthreads();
}

// mean_robust's cluster of the n rtvecs in w.x: returns the label (lowest row) of the largest cluster; w.nn[k] = label of row k
template <int NT, bool LARGE>
__device__ int pi_cluster(const ClusterWork& w, int n) {
  __shared__ double s_sd[6];
  __shared__ int s_merges, s_changed, s_best;
  const int t = max(n / 10, 3);
  if (n <= t) {                                    // every row its own cluster: the first one wins
    for (int k = threadIdx.x; k < n; k += NT) w.nn[k] = k;
    __syncthreads();
    return 0;
  }
  for (int c = 0; c < 6; c++) {                    // whiten: population std per column, 1 where it is zero
    double acc = 0.0;
    for (int k = threadIdx.x; k < n; k += NT) acc += w.x[6 * k + c];
    const double mean = pi_sum<NT>(acc) / n;
    acc = 0.0;
    for (int k = threadIdx.x; k < n; k += NT) { const double d = w.x[6 * k + c] - mean; acc += d * d; }
    const double sd = sqrt(pi_sum<NT>(acc) / n);
    if (threadIdx.x == 0) s_sd[c] = sd == 0.0 ? 1.0 : sd;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < n; k += NT) {
    for (int c = 0; c < 6; c++) w.cen[6 * k + c] = w.x[6 * k + c] / s_sd[c];
    w.sz[k] = 1.0; w.alive[k] = k; w.par[k] = k; w.hj[k] = INFINITY; w.mround[k] = -1; w.nn[k] = -1;
  }
  __syncthreads();
  int* al = w.alive; int* al2 = w.alive2;
  int m = n;
  for (int round = 0; m > 1; round++) {
    const int ns = pi_compact<NT>(m, [&](int p) {
      const int k = al[p], j = w.nn[k];
      return round == 0 || j < 0 || w.mround[k] == round - 1 || w.mround[j] == round - 1 || w.par[j] != j;
    }, [&](int p, int o) { w.slist[o] = al[p]; });
    pi_search<NT, LARGE>(w, al, m, ns);
    if (threadIdx.x == 0) s_merges = 0;
    __syncthreads();
    for (int p = threadIdx.x; p < m; p += NT) {
      const int i = al[p], j = w.nn[i];
      if (j > i && w.nn[j] == i) {
        const double a = w.sz[i], b = w.sz[j], s = a + b;
        for (int c = 0; c < 6; c++) w.cen[6 * i + c] = (a * w.cen[6 * i + c] + b * w.cen[6 * j + c]) / s;
        w.sz[i] = s; w.hj[j] = sqrt(2.0 * w.nnw[i]); w.par[j] = i; w.mround[i] = round;
        atomicAdd(&s_merges, 1);
      }
    }
    __syncthreads();
    if (s_merges == 0) break;                      // only on non-finite input, which the host rejects
    m = pi_compact<NT>(m, [&](int p) { return w.par[al[p]] == al[p]; }, [&](int p, int o) { al2[o] = al[p]; });
    int* tmp = al; al = al2; al2 = tmp;
  }
  const double cut = pi_select<NT>(w.hj, n, n - t - 1);
  for (int k = threadIdx.x; k < n; k += NT) { w.nn[k] = w.hj[k] <= cut ? w.par[k] : k; w.cnt[k] = 0; }
  __syncthreads();
  for (;;) {                                       // labels = roots of the merges kept (pointer jumping)
    if (threadIdx.x == 0) s_changed = 0;
    __syncthreads();
    for (int k = threadIdx.x; k < n; k += NT) {
      const int l = w.nn[k], ll = w.nn[l];
      if (ll != l) { w.nn[k] = ll; s_changed = 1; }
    }
    __syncthreads();
    if (!s_changed) break;
    __syncthreads();
  }
  for (int k = threadIdx.x; k < n; k += NT) atomicAdd(&w.cnt[w.nn[k]], 1);
  if (threadIdx.x == 0) s_best = 0;
  __syncthreads();
  // largest cluster, ties to the lowest label (= lowest row of the cluster)
  int bc = 0, bl = 0x7fffffff;
  for (int k = threadIdx.x; k < n; k += NT) if (w.cnt[k] > bc) { bc = w.cnt[k]; bl = k; }
  const int key_hi = bc;
  __shared__ int s_bc[NT], s_bl[NT];
  s_bc[threadIdx.x] = key_hi; s_bl[threadIdx.x] = bl;
  __syncthreads();
  for (int h = NT / 2; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) {
      const int oc = s_bc[threadIdx.x + h], ol = s_bl[threadIdx.x + h];
      if (oc > s_bc[threadIdx.x] || (oc == s_bc[threadIdx.x] && ol < s_bl[threadIdx.x])) { s_bc[threadIdx.x] = oc; s_bl[threadIdx.x] = ol; }
    }
    __syncthreads();
  }
  const int best = s_bl[0];
  __syncthreads();
  return best;
}

// mean_robust of the n rtvecs in w.x -> 3x4 pose in T (shared); NaN when n == 0
template <int NT, bool LARGE>
__device__ void pi_mean_robust(const ClusterWork& w, int n, double* T) {
  if (n == 0) {
    if (threadIdx.x == 0) for (int k = 0; k < 12; k++) T[k] = NAN;
    __syncthreads();
    return;
  }
  const int best = pi_cluster<NT, LARGE>(w, n);
  __shared__ double s_mean[6];
  double cntd = 0.0;
  for (int k = threadIdx.x; k < n; k += NT) cntd += w.nn[k] == best ? 1.0 : 0.0;
  const double cnt = pi_sum<NT>(cntd);
  for (int c = 0; c < 6; c++) {
    double acc = 0.0;
    for (int k = threadIdx.x; k < n; k += NT) if (w.nn[k] == best) acc += w.x[6 * k + c];
    const double s = pi_sum<NT>(acc);
    if (threadIdx.x == 0) s_mean[c] = s / cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double R[9], JL[9];
    rodrigues(s_mean, R, JL);
    for (int i = 0; i < 3; i++) { for (int j = 0; j < 3; j++) T[4 * i + j] = R[3 * i + j]; T[4 * i + 3] = s_mean[3 + i]; }
  }
  __syncthreads();
}

// rtvecs of m2 inv(m1) for the rows in w.idx[0, n)
__device__ inline void pi_rel_rtvecs(const ClusterWork& w, int n, const double* M1, const double* M2, int NT) {
  for (int k = threadIdx.x; k < n; k += NT) {
    const int r = w.idx[k];
    double I[12], Rl[12];
    pi_inv34(M1 + 12 * (size_t)r, I);
    pi_mul34(M2 + 12 * (size_t)r, I, Rl);
    matrix_to_rtvec(Rl, w.x + 6 * (size_t)k);
  }
  __syncthreads();
}

template <int NT, bool LARGE>
__global__ void __launch_bounds__(NT) k_pose_align(PoseAlignArgs a) {
  extern __shared__ double pi_dyn[];
  __shared__ double s_T[12];
  const int item = a.items[blockIdx.x];
  const int64_t r0 = a.row_start[item];
  const int R = (int)(a.row_start[item + 1] - r0);
  const ClusterWork w = pi_carve(LARGE ? a.work + r0 * PI_ROW_BYTES : (char*)pi_dyn, R);
  if (a.vecs) {                                    // cluster only: the mask of mean_robust's cluster
    for (int k = threadIdx.x; k < 6 * R; k += NT) w.x[k] = a.vecs[6 * r0 + k];
    __syncthreads();
    const int best = pi_cluster<NT, LARGE>(w, R);
    for (int k = threadIdx.x; k < R; k += NT) a.inl[r0 + k] = w.nn[k] == best;
    return;
  }
  const double* M1 = a.m1 + 12 * r0; const double* M2 = a.m2 + 12 * r0;
  const uint8_t* mk = a.mask + r0;
  int n = pi_compact<NT>(R, [&](int r) { return mk[r] != 0; }, [&](int r, int o) { w.idx[o] = r; });
  pi_rel_rtvecs(w, n, M1, M2, NT);
  pi_mean_robust<NT, LARGE>(w, n, s_T);
  for (int r = threadIdx.x; r < R; r += NT) {      // error_transform over every row, masked or not
    double P[12], e = 0.0;
    pi_mul34(s_T, M1 + 12 * (size_t)r, P);
    for (int k = 0; k < 12; k++) { const double d = P[k] - M2[12 * (size_t)r + k]; e += d * d; }
    w.hj[r] = sqrt(e);
  }
  __syncthreads();
  // np.quantile(errs, 0.75), method 'linear' (numpy's _lerp)
  const double vi = 0.75 * (R - 1);
  const int lo = (int)floor(vi);
  const double gm = vi - lo;
  const double qa = pi_select<NT>(w.hj, R, lo);
  double q = qa;
  if (gm > 0.0) {
    const double qb = pi_select<NT>(w.hj, R, min(lo + 1, R - 1));
    const double diff = qb - qa;
    q = gm >= 0.5 ? qb - diff * (1.0 - gm) : qa + diff * gm;
  }
  const double thr = q * 1.5;
  n = pi_compact<NT>(R, [&](int r) {
    const bool in = mk[r] && w.hj[r] < thr;
    a.inl[r0 + r] = in;
    return in;
  }, [&](int r, int o) { w.idx[o] = r; });
  pi_rel_rtvecs(w, n, M1, M2, NT);
  pi_mean_robust<NT, LARGE>(w, n, s_T);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 12; k++) a.t[16 * (size_t)item + k] = s_T[k];
    a.t[16 * (size_t)item + 12] = 0.0; a.t[16 * (size_t)item + 13] = 0.0; a.t[16 * (size_t)item + 14] = 0.0; a.t[16 * (size_t)item + 15] = 1.0;
    a.n_inl[item] = n;
  }
}

}  // namespace mcba
